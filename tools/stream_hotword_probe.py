"""Cost of hotwords in live streams (`GigaAMASR.streaming(hotwords=...)`, INTEGRATION.md §7i).

    python tools/stream_hotword_probe.py [--quick]

A synthetic full-depth v2_ctc model (random weights, fp32 encoder), N streams of synthetic audio at W / V = 8 / 4 s,
batch_size 64.  Every stream first holds one window; each step then receives H = 4 s per stream, so every step encodes and
decodes one window of every stream.  Each setting runs without hotwords and with K hotwords (near misses of the model's own
greedy words, threshold 0.1, so splices happen).  Reported per setting: the median step time over 5 timed steps after 2
warm-up steps (host clock, `step()` call to return); the GPU time of the bias-resume calls (CUDA events around each
`Engine.ctc_bias_resume` call, summed per step, median); the distribution of C - R, the frames each stream holds back after a
step (min / median / p95 / max over streams and timed steps); and the peak device memory above the model's.  The card's
name, power limit and SM clocks are read in the same run.  The last line is one JSON record of everything printed."""
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402

dev = torch.device("cuda", 0)
SR = 16000


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(dev)


def hotwords_of(model, audio, K):
    plain = model.transcribe_windowed(audio[0, :60 * SR], window=8.0, overlap=4.0)
    words = sorted({w for s in plain.segments for w in s.text.split() if 2 <= len(w) <= 60})
    hot = sorted({w[:i] + c + w[i + 1:] for w in words for i in (0, len(w) // 2) for c in "аеиорст" if c != w[i]})
    rng = np.random.default_rng(K)
    while len(hot) < K:   # a transcript with few words: random words fill the list
        hot.append("".join(rng.choice(list("абвгдежзиклмнопрст"), int(rng.integers(3, 9)))))
    return hot[:K]


def run(model, audio, N, hot, warmup=2, reps=5):
    eng = model._get_engine()
    spans = []
    real = eng.ctc_bias_resume

    def timed(*a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = real(*a, **kw)
        e1.record()
        spans.append((e0, e1))
        return out
    eng.ctc_bias_resume = timed
    try:
        srv = model.streaming(window=8.0, overlap=4.0, batch_size=64, hotwords=hot, hotword_threshold=0.1)
        ids = [srv.open() for _ in range(N)]
        pos = 8 * SR + 1
        for i, a in enumerate(ids):
            srv.push(a, audio[i % audio.shape[0], :pos].numpy())
        srv.step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        times, kernel, lag = [], [], []
        for r in range(warmup + reps):
            for i, a in enumerate(ids):
                srv.push(a, audio[i % audio.shape[0], pos:pos + 4 * SR].numpy())
            spans.clear()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            srv.step()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            pos += 4 * SR
            if r >= warmup:
                times.append(dt * 1e3)
                kernel.append(sum(e0.elapsed_time(e1) for e0, e1 in spans))
                lag += [0 if srv._streams[a].hw_rows is None else int(srv._streams[a].hw_rows.shape[0]) for a in ids] if hot else []
        peak = (torch.cuda.max_memory_allocated() - base) / 2**20
        for a in ids:
            srv.close(a)
    finally:
        eng.ctc_bias_resume = real
    rec = {"streams": N, "hotwords": len(hot or []), "step_ms": round(statistics.median(times), 2),
           "bias_resume_ms": round(statistics.median(kernel), 3) if hot else None, "peak_mib": round(peak, 1)}
    if hot:
        q = np.percentile(lag, [0, 50, 95, 100])
        rec["held_frames"] = {"min": int(q[0]), "median": float(q[1]), "p95": float(q[2]), "max": int(q[3])}
    return rec


def main():
    quick = "--quick" in sys.argv
    ck = gigaam.synthetic_checkpoint("v2_ctc", seed=0)
    model = gigaam.load_model("v2_ctc", fp16_encoder=False, device=dev, checkpoint=ck)
    audio, _ = gigaam.synthetic_audio(8, 100.0, seed=3)
    out = {"card": card(), "runs": []}
    print(out["card"])
    for N in ((16,) if quick else (16, 128)):
        for K in (0, 10, 100):
            hot = hotwords_of(model, audio, K) if K else None
            rec = run(model, audio, N, hot)
            out["runs"].append(rec)
            print(rec, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
