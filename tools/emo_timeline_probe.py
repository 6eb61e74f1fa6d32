"""Cost of an emotion timeline over one hour (`GigaAMEmo.emotion_timeline`, INTEGRATION.md, "Emotions over time").

    python tools/emo_timeline_probe.py [--minutes 60] [--batch-size 16]

The synthetic GigaAM-Emo checkpoint (full-depth v1 encoder, random weights, fp16 encoder as load_model gives it) and synthetic
audio of the given length at 16 kHz; windows of 30 s with 4 s overlap, spans of 4 s every 1 s.  One warm-up call over the
first two minutes, then:
  - the wall time of three timed calls (host clock around the call, which ends in device-to-host copies), median;
  - one more call with gam_profile_* armed: the GPU time per kernel class, split into the encoder (every class but the two
    below), emo_frame_logits and emo_spans, with their launch counts;
  - emo_frame_logits' effective bandwidth: the bytes it must move (every kept frame's 768 fp32 values read once, C fp32
    logits written) over its measured time.
The card's name, power limit and SM clocks are read in the same run.  The last line is one JSON record of everything printed."""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402

dev = torch.device("cuda", 0)
SR = 16000


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=60.0)
    ap.add_argument("--batch-size", type=int, default=16)
    args = ap.parse_args()
    model = gigaam.load_model("emo", device=dev, synthetic=True)
    wav = gigaam.synthetic_audio(1, 60.0 * args.minutes, seed=1)[0][0]
    kw = dict(window=30.0, overlap=4.0, span=4.0, hop=1.0, batch_size=args.batch_size)
    model.emotion_timeline(wav[:120 * SR], **kw)            # warm-up: module loads, workspaces, pinned staging
    times = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tl = model.emotion_timeline(wav, **kw)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    eng = model._get_engine()
    eng.profile_begin()
    model.emotion_timeline(wav, **kw)
    prof = eng.profile_end()
    T, C = tl.frame_logits.shape
    own = {k: prof.get(k, (0.0, 0)) for k in ("emo_frame_logits", "emo_spans")}
    encoder_ms = sum(ms for k, (ms, _) in prof.items() if k not in own)
    fl_ms = own["emo_frame_logits"][0]
    fl_bytes = T * (768 + C) * 4
    rec = dict(card=card(), minutes=args.minutes, batch_size=args.batch_size, frames=T, classes=C, spans=len(tl.spans),
               wall_s_median=statistics.median(times), wall_s=times, encoder_gpu_ms=encoder_ms,
               emo_frame_logits_ms=fl_ms, emo_frame_logits_launches=own["emo_frame_logits"][1],
               emo_spans_ms=own["emo_spans"][0], emo_spans_launches=own["emo_spans"][1],
               emo_frame_logits_bytes=fl_bytes, emo_frame_logits_gb_per_s=fl_bytes / (fl_ms * 1e-3) / 1e9 if fl_ms else None,
               kernel_share_of_gpu_time=(fl_ms + own["emo_spans"][0]) / (encoder_ms + fl_ms + own["emo_spans"][0]))
    print(f"card: {rec['card']}")
    print(f"{args.minutes:g} min, T = {T} frames, {len(tl.spans)} spans; wall {rec['wall_s_median']:.2f} s (median of 3)")
    print(f"GPU time: encoder and front end {encoder_ms:.1f} ms; emo_frame_logits {fl_ms:.3f} ms in {rec['emo_frame_logits_launches']} "
          f"launches ({fl_bytes / 1e6:.0f} MB, {rec['emo_frame_logits_gb_per_s'] or 0:.0f} GB/s); emo_spans {rec['emo_spans_ms']:.3f} ms")
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
