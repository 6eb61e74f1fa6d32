"""Step time of the live-stream server (`GigaAMASR.streaming`), with a host clock around whole steps.

    python tools/stream_probe.py [--quick]

Synthetic full-depth v2_ctc and v2_rnnt models (random weights, fp32 encoder), S streams of synthetic audio at W / V = 8 / 4
and 30 / 4 s, batch_size 64.  Every stream first holds one window; each step then receives H = W - V seconds per stream,
so every step encodes and decodes one window of every stream: the steady state of live audio.  A step's time runs from
the `step()` call to its return, which has copied every result to the host.  Each figure is the median of 5 timed steps
after 2 warm-up steps.  CTC runs with and without 100 keywords of 3 to 12 tokens.  Then, at 8 / 4 without keywords, S
doubles from 256 up to 4096 until a step takes longer than H: the largest S whose step stays under H is the capacity of one
card for that setting (median of 3 steps after 1).  The card's name, power limit and SM clocks are read in the same run.  The last line is one JSON record
of everything printed."""
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


def step_ms(model, audio, S, window, overlap, keywords, warmup=2, reps=5):
    W, H = int(window * SR), int((window - overlap) * SR)
    srv = model.streaming(window=window, overlap=overlap, batch_size=64, keywords=keywords, threshold=0.5)
    ids = [srv.open() for _ in range(S)]
    offs = [(i * 7919 * 16) % (audio.numel() - W - H * (warmup + reps + 1)) for i in range(S)]
    pos = [0] * S

    def feed(n):
        for i, a in enumerate(ids):
            srv.push(a, audio[offs[i] + pos[i]: offs[i] + pos[i] + n])
            pos[i] += n

    feed(W)
    times = []
    for k in range(warmup + reps):
        feed(H)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ups = srv.step()
        t1 = time.perf_counter()
        assert len(ups) == S
        if k >= warmup:
            times.append((t1 - t0) * 1e3)
    return statistics.median(times)


def main(quick):
    rec = {"card_before": card(), "rows": [], "capacity": {}}
    print(f"card: {rec['card_before']}")
    wav, _ = gigaam.synthetic_audio(1, 600.0, seed=3)
    audio = wav[0]
    g = torch.Generator().manual_seed(0)
    counts = (1, 16, 64) if quick else (1, 16, 64, 256)
    for name in ("v2_ctc", "v2_rnnt"):
        model = gigaam.load_model(name, fp16_encoder=False, device=dev, checkpoint=gigaam.synthetic_checkpoint(name, seed=0))
        V = len(model.decoding.tokenizer)
        kws = [torch.randint(0, V, (int(n),), generator=g).tolist() for n in torch.randint(3, 13, (100,), generator=g)]
        for window, overlap in ((8.0, 4.0), (30.0, 4.0)):
            for keywords in ((None, kws) if name == "v2_ctc" else (None,)):
                for S in counts:
                    ms = step_ms(model, audio, S, window, overlap, keywords)
                    row = dict(model=name, window=window, overlap=overlap, keywords=0 if keywords is None else len(keywords),
                               streams=S, step_ms=round(ms, 2), hop_ms=(window - overlap) * 1e3)
                    rec["rows"].append(row)
                    print(f"{name:8s} W/V = {window:4.1f}/{overlap:.1f} s, {row['keywords']:3d} keywords, {S:4d} streams: "
                          f"step {ms:9.2f} ms  (hop {row['hop_ms']:.0f} ms)")
        if quick:
            continue
        S, best = 256, None
        while S <= 4096:
            ms = step_ms(model, audio, S, 8.0, 4.0, None, warmup=1, reps=3)
            print(f"{name:8s} capacity search, 8/4 s: {S:5d} streams: step {ms:9.2f} ms")
            rec["rows"].append(dict(model=name, window=8.0, overlap=4.0, keywords=0, streams=S, step_ms=round(ms, 2), hop_ms=4000.0))
            if ms >= 4000.0:
                break
            best = S
            S *= 2
        rec["capacity"][name] = best
        print(f"{name:8s} largest stream count measured whose step stays under the 4 s hop: {best}")
        del model
        torch.cuda.empty_cache()
    rec["card_after"] = card()
    print(f"card after: {rec['card_after']}")
    print(json.dumps(rec))


if __name__ == "__main__":
    main("--quick" in sys.argv)
