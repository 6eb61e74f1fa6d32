"""Cost of scored greedy decoding (gam_*_greedy_scored) against the unscored decoders, with CUDA events.

    python tools/score_probe.py

For each shape the encoder output of synthetic audio (a 2-layer synthetic model) is decoded by `Engine.greedy` with and
without `scores=True`, alternating, after a warm-up; each figure is the median of the repetitions.  Shapes:
v2_ctc 64 x 251, v3_e2e_ctc (257 classes) 64 x 251, v2_rnnt 32 x 376 and v3_e2e_rnnt (1025 classes) 32 x 251 (B x T').
The card name, power limit and SM clock are read in the same run.  The last line is one JSON record of everything printed.
"""
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402

dev = torch.device("cuda", 0)
SHAPES = [("v2_ctc", 64, 10.0), ("v3_e2e_ctc", 64, 10.0), ("v2_rnnt", 32, 15.0), ("v3_e2e_rnnt", 32, 10.0)]


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(dev)


def timed(fn, reps):
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def probe(name, B, seconds, warmup=5, reps=30):
    ck = gigaam.synthetic_checkpoint(name, seed=0, n_layers=2)
    model = gigaam.load_model(name, device=dev, checkpoint=ck)
    wav, wav_len = gigaam.synthetic_audio(B, seconds, seed=1)
    with torch.inference_mode():
        enc, enc_len = model(wav.to(dev), wav_len.to(dev))
        x = enc.transpose(1, 2).contiguous()
        eng = model._get_engine()
        plain = lambda: eng.greedy(x, enc_len)                  # noqa: E731
        scored = lambda: eng.greedy(x, enc_len, scores=True)    # noqa: E731
        for _ in range(warmup):
            plain()
            scored()
        torch.cuda.synchronize()
        tp, ts = [], []
        for _ in range(reps):                                   # alternate, so drift hits both arms alike
            tp += timed(plain, 1)
            ts += timed(scored, 1)
    mp, ms = statistics.median(tp), statistics.median(ts)
    rec = dict(shape=f"{name} {B}x{x.shape[1]}", classes=eng.num_classes, unscored_ms=round(mp, 4), scored_ms=round(ms, 4),
               overhead_pct=round(100.0 * (ms - mp) / mp, 2),
               unscored_range=[round(min(tp), 4), round(max(tp), 4)], scored_range=[round(min(ts), 4), round(max(ts), 4)])
    print(rec)
    return rec


def main():
    gpu = card()
    print("card (name, power limit, SM clock, max SM clock):", gpu)
    recs = [probe(*s) for s in SHAPES]
    print(json.dumps(dict(card=gpu, shapes=recs)))


if __name__ == "__main__":
    main()
