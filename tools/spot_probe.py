"""Cost of CTC keyword spotting (gam_ctc_spot), with CUDA events.

    python tools/spot_probe.py [--quick]

The kernel alone, on random log_softmax rows [1, T, V+1] standing in for stitched long-form log-probs: 10 and 60 minutes of
audio (T = 15 000 and 90 000 frames of 40 ms) at V + 1 = 34 (v2_ctc) and 257 (v3_e2e_ctc), for 10, 100 and 1000 random
keywords of 3 to 12 tokens, threshold 0.5, max_det 64.  Each figure is the median of 5 timed calls after 2 warm-up calls.
The card's name, power limit and SM clocks are read in the same run, before and after; the kernel's registers and spills
come from the ptxas report of the in-tree build.  The last line is one JSON record of everything printed."""
import json
import re
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402

dev = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(dev)


def registers():
    """ptxas' line for ctc_spot_kernel in the build log: registers, spills."""
    log = ROOT / "gigaam_b200" / "build" / "spot.cu.log"
    if not log.exists():
        return "not available (no build log)"
    text = log.read_text()
    m = re.search(r"ctc_spot_kernel.*?(\d+) bytes spill stores, (\d+) bytes spill loads.*?Used (\d+) registers", text, re.S)
    return f"{m.group(3)} registers, {m.group(1)} B spill stores, {m.group(2)} B spill loads" if m else "not found"


def median_ms(fn, warmup=2, reps=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def main(quick):
    rec = {"card_before": card(), "kernel": registers(), "rows": []}
    print(f"card: {rec['card_before']}\nctc_spot_kernel: {rec['kernel']}")
    g = torch.Generator().manual_seed(0)
    for name in ("v2_ctc", "v3_e2e_ctc"):
        ck = gigaam.synthetic_checkpoint(name, seed=0, n_layers=1)
        eng = gigaam.load_model(name, fp16_encoder=False, device=dev, checkpoint=ck)._get_engine()
        V1 = eng.num_classes
        for minutes in ((10,) if quick else (10, 60)):
            T = minutes * 60 * 25
            lp = torch.randn(1, T, V1, generator=g).mul_(2.0).log_softmax(-1).to(dev)
            enc_len = torch.tensor([T], dtype=torch.int32, device=dev)
            for K in ((10, 100) if quick else (10, 100, 1000)):
                lens = torch.randint(3, 13, (K,), generator=g, dtype=torch.int32)
                kw = torch.randint(0, V1 - 1, (K, 12), generator=g, dtype=torch.int32)
                kw_d, lens_d = kw.to(dev), lens.to(dev)
                ms = median_ms(lambda: eng.ctc_spot(lp, enc_len, kw_d, lens_d, 0.5, 64))
                row = dict(V1=V1, minutes=minutes, frames=T, keywords=K, ms=round(ms, 3),
                           us_per_frame=round(ms * 1e3 / T, 4), lp_MB=round(T * V1 * 4 / 1e6, 1))
                rec["rows"].append(row)
                print(f"V+1 = {V1:4d}, {minutes:2d} min ({T} frames, log-probs {row['lp_MB']} MB), K = {K:4d}: "
                      f"{ms:9.3f} ms  ({row['us_per_frame']} us per frame)")
            del lp
    rec["card_after"] = card()
    print(f"card after: {rec['card_after']}")
    print(json.dumps(rec))


if __name__ == "__main__":
    main("--quick" in sys.argv)
