"""Isolated timing of the head kernels (csrc/heads.cu) at user sizes, with CUDA events.

    python tools/head_probe.py

  - CTC log-probs at the c2 shape (64 x 251 frames), V+1 = 34 (v2_ctc) and 257 (v3_e2e_ctc);
  - the joint lattice (both projections + the lattice kernel) at B = 8, T = 251, U = 100, V+1 = 34 and 1025;
  - one greedy-search step at B = 32, U = 1: predict, joint, and the two together, called from Python (what a search
    loop pays per step, call overhead included) and replayed from a CUDA graph (device time).

Achieved FP32 FLOP/s and HBM bytes/s are computed from the shapes (the arithmetic the algorithm needs, and each input and
output crossing HBM once) over the median kernel time, against the H100 SXM data-sheet 67 TFLOP/s FP32 and 3.35 TB/s.
The card name and power limit are read in the same run.  The last line is one JSON record of everything printed.
"""
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402

PEAK_FLOPS, PEAK_BYTES = 67e12, 3.35e12
dev = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(dev)


def time_us(fn, reps=20, warmup=3):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def model(name):
    ck = gigaam.synthetic_checkpoint(name, n_layers=1)
    return gigaam.load_model(name, fp16_encoder=False, device=dev, checkpoint=ck)


records = []


def report(what, us, flops, nbytes):
    r = dict(what=what, us=round(us, 1), tflops=round(flops / us / 1e6, 2), tbps=round(nbytes / us / 1e6, 3),
             pct_fp32_peak=round(100 * flops / us / 1e-6 / PEAK_FLOPS, 1), pct_hbm_peak=round(100 * nbytes / us / 1e-6 / PEAK_BYTES, 1))
    records.append(r)
    print(f"{what:44s} {us:10.1f} us  {r['tflops']:7.2f} TFLOP/s ({r['pct_fp32_peak']:5.1f}% of 67)  "
          f"{r['tbps']:6.3f} TB/s ({r['pct_hbm_peak']:5.1f}% of 3.35)", flush=True)


@torch.inference_mode()
def main():
    info = card()
    print(f"device: {info}", flush=True)
    g = torch.Generator().manual_seed(0)
    d, H, J = 768, 320, 320

    B, T = 64, 251
    enc = torch.randn(B, T, d, generator=g).to(dev)
    for name in ("v2_ctc", "v3_e2e_ctc"):
        m = model(name)
        V1 = m.cfg["head"]["num_classes"]
        encoded = enc.transpose(1, 2)
        us = time_us(lambda: m.head(encoded))
        report(f"ctc_log_probs B={B} T={T} V+1={V1}", us, 2.0 * B * T * d * V1, 4.0 * (B * T * d + V1 * d + B * T * V1))
        del m

    B, T, U = 8, 251, 100
    enc = torch.randn(B, T, d, generator=g).to(dev)
    dec = (torch.rand(B, U, H, generator=g) * 2 - 1).to(dev)
    steps = {}
    for name in ("v2_rnnt", "v3_e2e_rnnt"):
        m = model(name)
        V1 = m.cfg["head"]["joint"]["num_classes"]
        us = time_us(lambda: m.head.joint.joint(enc, dec), reps=10)
        flops = 2.0 * (B * T * J * d + B * U * J * H + B * T * U * J * V1)
        report(f"rnnt_joint B={B} T={T} U={U} V+1={V1}", us, flops, 4.0 * (B * T * d + B * U * H + V1 * J + B * T * U * V1))
        steps[name] = m

    m = steps["v2_rnnt"]
    V1 = m.cfg["head"]["joint"]["num_classes"]
    B = 32
    x = torch.randint(0, V1, (B, 1), generator=g).to(dev)
    h, c = torch.randn(1, B, H, generator=g).to(dev), torch.randn(1, B, H, generator=g).to(dev)
    f = torch.randn(B, 1, d, generator=g).to(dev)
    gp, _ = m.head.decoder.predict(x, (h, c))
    us_p = time_us(lambda: m.head.decoder.predict(x, (h, c)), reps=50)
    report(f"rnnt_predict B={B} U=1", us_p, 2.0 * B * H * 4 * H, 4.0 * (H * 4 * H + V1 * 4 * H + 4 * B * H))
    us_j = time_us(lambda: m.head.joint.joint(f, gp), reps=50)
    report(f"rnnt_joint B={B} T=1 U=1 V+1={V1}", us_j, 2.0 * B * J * (d + H + V1), 4.0 * (J * (d + H + V1) + B * (d + H + V1)))

    def step():
        g1, _ = m.head.decoder.predict(x, (h, c))
        return m.head.joint.joint(f, g1)
    us_s = time_us(step, reps=50)
    step_flops = 2.0 * B * (H * 4 * H + J * (d + H + V1))
    report(f"predict + joint step B={B}", us_s, step_flops, 0.0)
    # the same step replayed from a CUDA graph: device time without the Python / ctypes call overhead
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    report(f"predict + joint step B={B}, graph replay", time_us(graph.replay, reps=50), step_flops, 0.0)
    print(json.dumps(dict(device=info, results=records)), flush=True)


if __name__ == "__main__":
    main()
