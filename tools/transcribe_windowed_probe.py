"""Cost of GigaAMASR.transcribe_windowed (window encoding, resumable greedy decoding, word grouping and host segmentation),
with device-synchronised wall clocks.

    python tools/transcribe_windowed_probe.py [--quick]

Synthetic 16-layer models (fp16 encoder) v2_ctc, v2_rnnt and v3_e2e_rnnt over 10 and 60 minutes of synthetic audio (10
minutes only with --quick), batch_size 16, scores on:
  encode  -- longform.window_batches alone (upload + model.forward of every batch of windows);
  decode  -- longform.decode_windows (the same encoding plus gam_*_greedy_resume over each window's kept frames) minus encode;
  words   -- the whole transcribe_windowed(word_timestamps=True, confidence=True) minus decode_windows: gam_group_words, the
             read-back, segment_cuts and windowed_segments;
  peak    -- torch.cuda.max_memory_allocated over the whole call, above what was allocated before it.
The card's name, power limit and SM clocks are read in the same run; the last line is one JSON record of everything printed."""
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402
from gigaam_b200 import longform  # noqa: E402

dev = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(dev)


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    quick = "--quick" in sys.argv
    print(card(), flush=True)
    rows = []
    for name in ("v2_ctc", "v2_rnnt", "v3_e2e_rnnt"):
        ck = gigaam.synthetic_checkpoint(name, seed=0)
        model = gigaam.load_model(name, fp16_encoder=True, device=dev, checkpoint=ck)
        for minutes in ((10,) if quick else (10, 60)):
            wav = gigaam.synthetic_audio(1, 60.0 * minutes, seed=minutes)[0][0]
            max_frames = model._max_frames
            windows, T = longform.plan_windows(wav.numel(), 30.0, 4.0, model._encoded_length, max_frames)
            host = wav.to(model._dtype).pin_memory()

            def encode_only():
                with torch.inference_mode():
                    for _, encoded in longform.window_batches(model, host, windows, 16):
                        del encoded

            def decode():
                with torch.inference_mode():
                    return longform.decode_windows(model, host, windows, T, 16, scores=True)

            def whole():
                return model.transcribe_windowed(wav, word_timestamps=True, confidence=True)

            whole()                                           # warm every window shape and workspace
            t_enc, _ = wall(encode_only)
            t_dec, out = wall(decode)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            t_all, res = wall(whole)
            peak = torch.cuda.max_memory_allocated() - base
            r = dict(model=name, minutes=minutes, frames=T, windows=len(windows), tokens=int(out.counts[0]),
                     segments=len(res.segments), encode_s=round(t_enc, 3), decode_s=round(t_dec - t_enc, 3),
                     decode_us_per_frame=round((t_dec - t_enc) * 1e6 / T, 2), words_s=round(t_all - t_dec, 3),
                     total_s=round(t_all, 3), peak_mib=round(peak / 2**20, 1))
            rows.append(r)
            print(f"{name:12s} {minutes:3d} min T'={T:6d}: encode {t_enc:7.3f} s, decode {t_dec - t_enc:7.3f} s "
                  f"({r['decode_us_per_frame']:.1f} us/frame), words+segments {t_all - t_dec:6.3f} s, whole call {t_all:7.3f} s, "
                  f"{r['tokens']} tokens, {r['segments']} segments, peak {peak / 2**20:.0f} MiB", flush=True)
        del model
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=card(), rows=rows)))


if __name__ == "__main__":
    main()
