"""Isolated timing of the wgmma GEMM (L2 flushed between launches, CUDA events), written as one JSON file together with the
card name and power limit read in the same run.  Development aid:

    python tools/gemm_probe.py --json OUT.json [--label NAME]

Three sets of measurements:
  * shapes:  every GEMM of the bench step at R = 64 x 251 = 16064 rows (FFN up / down, QKV as one dual-A launch, proj,
             pw1 + GLU, sub_out) and the conv2 implicit GEMM (A_CONV, B = 64, T' = 251, packed rows).
  * rounds:  one round of the persistent grid with 33, 66 and 132 tiles at (N, K) = (768, 3072), and with 36, 72 and 132
             tiles at (3072, 768) (12 n-blocks: 33 and 66 are not multiples of 12).  A one-round time that grows with the
             number of busy SMs means the operand feed is a resource the SMs share (L2); a flat one means each SM is
             limited on its own.
  * ksweep:  M = 16064, N = 768, K = 768 .. 6144 (the FFN-down epilogue): the slope is the mainloop cost per k-block, the
             intercept the fixed cost per tile (pipeline fill + epilogue)."""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from gigaam_b200 import synthetic  # noqa: E402
from gigaam_b200.engine import Engine  # noqa: E402

KINDS = {0: "bias->f16", 1: "bias+silu->f16", 2: "bias+glu->f16", 3: "res+scale*(acc+bias)->f32", 4: "bias->f32"}
R = 64 * 251
ITERS = 11


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, plim, clk = [s.strip() for s in out.splitlines()[0].split(",")]
    return {"name": name, "power_limit": plim, "clocks_max_sm": clk}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", required=True, help="output file")
    ap.add_argument("--label", default="")
    args = ap.parse_args()

    dev = torch.device("cuda", 0)
    ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1)
    eng = Engine(ck["cfg"], ck["state_dict"], dev)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(launch):
        ts = []
        for it in range(ITERS):
            flush.fill_(it)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = launch()
            e1.record()
            torch.cuda.synchronize()
            assert rc == 0, eng.lib.gam_last_error(eng.handle)
            ts.append(e0.elapsed_time(e1) * 1e3)
        ts = sorted(ts[1:])
        return ts[len(ts) // 2], ts[0], ts[-1]

    def gemm(M, N, K, kind, dual_n1=0, name=""):
        g = torch.Generator(device=dev).manual_seed(M + N + K)
        A = (torch.randn(M, K, generator=g, device=dev) * 0.5).half()
        A2 = (torch.randn(M, K, generator=g, device=dev) * 0.5).half() if dual_n1 else None
        W = (torch.randn(N, K, generator=g, device=dev) / K ** 0.5).half()
        bias = torch.randn(N, generator=g, device=dev)
        ncol = N // 2 if kind == 2 else N
        out = torch.zeros(M, ncol, dtype=torch.float32 if kind >= 3 else torch.float16, device=dev)
        us, lo, hi = timed(lambda: eng.lib.gam_test_gemm(
            eng.handle, kind, A.data_ptr(), A2.data_ptr() if dual_n1 else None, dual_n1, W.data_ptr(), bias.data_ptr(),
            out.data_ptr() if kind == 3 else None, out.data_ptr(), M, N, K, ncol, 0, 0.5, 0, None, st))
        tiles = -(-M // 128) * (N // 256)
        r = {"name": name, "M": M, "N": N, "K": K, "epilogue": KINDS[kind] + (" dual-A" if dual_n1 else ""), "tiles": tiles,
             "us": round(us, 2), "us_min": round(lo, 2), "us_max": round(hi, 2), "tflops": round(2.0 * M * N * K / us / 1e6, 1)}
        print(json.dumps(r), flush=True)
        return r

    def conv2(B=64, T2=251, Cc=768, N=768):
        T1 = 2 * T2 - 1                       # 3x3, stride 2, pad 1: T2 = (T1 - 1) // 2 + 1
        g = torch.Generator(device=dev).manual_seed(5)
        x = torch.rand((B, T1, 32, Cc), generator=g, device=dev).half()
        W = (torch.randn(N, 9 * Cc, generator=g, device=dev) / (9 * Cc) ** 0.5).half()
        bias = torch.randn(N, generator=g, device=dev) * 0.1
        lens = torch.full((B,), T2, dtype=torch.int32, device=dev)
        cu = torch.arange(B, dtype=torch.int32, device=dev) * T2
        out = torch.empty((B * T2 * 16, N), dtype=torch.float16, device=dev)
        us, lo, hi = timed(lambda: eng.lib.gam_test_gemm_conv(
            eng.handle, 0, x.data_ptr(), W.data_ptr(), bias.data_ptr(), lens.data_ptr(), cu.data_ptr(), lens.data_ptr(),
            out.data_ptr(), B * T2, B, T1, 32, Cc, 9, N, 0, st))
        M, K = B * T2 * 16, 9 * Cc
        r = {"name": "conv2", "M": M, "N": N, "K": K, "epilogue": "A_CONV packed, relu+mask->f16", "tiles": (M // 128) * (N // 256),
             "us": round(us, 2), "us_min": round(lo, 2), "us_max": round(hi, 2), "tflops": round(2.0 * M * N * K / us / 1e6, 1)}
        print(json.dumps(r), flush=True)
        return r

    res = {"label": args.label, "card": card(), "iters": ITERS, "stat": "median of launches 2..N, L2 flushed before each"}
    res["shapes"] = [
        gemm(R, 3072, 768, 1, name="ffn_up"), gemm(R, 768, 3072, 3, name="ffn_down"),
        gemm(R, 2304, 768, 0, dual_n1=1536, name="qkv"), gemm(R, 768, 768, 3, name="proj_pw2"),
        gemm(R, 1536, 768, 2, name="pw1_glu"), gemm(R, 768, 20 * 768, 4, name="sub_out"), conv2()]
    res["rounds"] = ([gemm(128 * t // 3, 768, 3072, 3, name=f"round_{t}") for t in (33, 66, 132)]
                     + [gemm(128 * t // 12, 3072, 768, 1, name=f"round_{t}") for t in (36, 72, 132)])
    res["ksweep"] = [gemm(R, 768, K, 3, name=f"k{K}") for K in (768, 1536, 3072, 6144)]
    res["card_after"] = card()
    Path(args.json).parent.mkdir(parents=True, exist_ok=True)
    Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
