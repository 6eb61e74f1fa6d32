"""Speed of gam_resample (Engine.resample_spans), with CUDA events around each call.

    python tools/resample_probe.py [--reps N]

One hour of audio in a batch of 64 rows (56.25 s each) of seeded noise at 8, 44.1 and 48 kHz, resampled to 16 kHz in one
launch.  Reported per rate: the table (n x K taps), milliseconds per call (median of N after a warm-up), bytes moved (every
input sample read once, every output written once, the table once) over time against the H100 SXM data sheet's 3.35 TB/s,
and FMAs (K per output, the taps the definition sums) over time as FLOP/s (2 per FMA) against its 67 TFLOP/s fp32 figure.
The card's name and power limit are read in the same run; the last line is one JSON record of everything printed."""
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402
from gigaam_b200.preprocess import resampled_length  # noqa: E402

dev = torch.device("cuda", 0)
RATES = (8000, 44100, 48000)
ROWS, SECONDS = 64, 3600.0 / 64
HBM_BYTES_S, FP32_FLOP_S = 3.35e12, 67e12


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(dev)


def main():
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 20
    name = card()
    print(name, flush=True)
    model = gigaam.load_model("v2_ctc", fp16_encoder=False, device=dev,
                              checkpoint=gigaam.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1))
    eng = model._get_engine()
    rows = []
    for sr in RATES:
        table, o, n, w = eng.resample_plan(sr)
        K = table.shape[0]
        L = int(round(SECONDS * sr))
        N = resampled_length(L, sr)
        g = torch.Generator(device=dev).manual_seed(sr)
        x = torch.rand((ROWS, L), device=dev, generator=g) * 2 - 1
        y = torch.empty((ROWS, N), device=dev)
        spans = torch.tensor([[0] * ROWS, [L] * ROWS, [0] * ROWS, [N] * ROWS], dtype=torch.int64, device=dev)
        for _ in range(3):
            eng.resample_spans(x, spans, sr, y)
        times = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            eng.resample_spans(x, spans, sr, y)
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b))
        ms = statistics.median(times)
        nbytes = 4 * (ROWS * (L + N) + table.numel())
        fma = ROWS * N * K
        row = dict(rate=sr, o=o, n=n, taps=K, ms=round(ms, 3), spread_ms=[round(min(times), 3), round(max(times), 3)],
                   bytes_per_s=nbytes / (ms * 1e-3), hbm_share=nbytes / (ms * 1e-3) / HBM_BYTES_S,
                   flop_per_s=2 * fma / (ms * 1e-3), fp32_share=2 * fma / (ms * 1e-3) / FP32_FLOP_S,
                   realtime=ROWS * SECONDS / (ms * 1e-3))
        rows.append(row)
        print(f"{sr:6d} Hz  {n:4d} x {K:3d} taps  {ms:8.3f} ms  {row['bytes_per_s'] / 1e9:7.1f} GB/s ({100 * row['hbm_share']:.1f} % "
              f"of 3.35 TB/s)  {row['flop_per_s'] / 1e12:6.2f} TFLOP/s ({100 * row['fp32_share']:.1f} % of 67)  "
              f"{row['realtime']:.0f}x real time", flush=True)
        del x, y
    print(json.dumps(dict(card=name, rows=rows)))


if __name__ == "__main__":
    main()
