"""Isolated timing of the wgmma GEMM's epilogue kinds at the BASELINE config-2 shapes (L2 flushed between launches).
Development aid:   python tools/gemm_probe.py [M]"""
import ctypes as C
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from gigaam_b200 import synthetic  # noqa: E402
from gigaam_b200.engine import Engine  # noqa: E402

dev = torch.device("cuda", 0)
ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1)
eng = Engine(ck["cfg"], ck["state_dict"], dev)
M = int(sys.argv[1]) if len(sys.argv) > 1 else 16064
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
KINDS = {0: "bias->f16", 1: "bias+silu->f16", 2: "bias+glu->f16", 3: "res+scale*(acc+bias)->f32", 4: "bias->f32"}
for (N, K, kinds) in ((768, 768, (3,)), (768, 3072, (3,)), (3072, 768, (1,)), (2304, 768, (0,)), (1536, 768, (2,))):
    A = (torch.randn(M, K) * 0.5).half().to(dev)
    W = (torch.randn(N, K) / K ** 0.5).half().to(dev)
    bias = torch.randn(N).to(dev)
    for kind in kinds:
        ncol = N // 2 if kind == 2 else N
        out = torch.zeros(M, ncol, dtype=torch.float32 if kind >= 3 else torch.float16, device=dev)
        ts = []
        for it in range(7):
            flush.fill_(it)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = eng.lib.gam_test_gemm(eng.handle, kind, A.data_ptr(), None, 0, W.data_ptr(), bias.data_ptr(),
                                       out.data_ptr() if kind == 3 else None, out.data_ptr(), M, N, K, ncol, 0, 0.5, 0, None, st)
            e1.record()
            torch.cuda.synchronize()
            assert rc == 0
            ts.append(e0.elapsed_time(e1) * 1e3)
        us = sorted(ts[1:])[2]
        print(f"M={M} N={N} K={K} {KINDS[kind]:28s} {us:8.1f} us  {2.0 * M * N * K / us / 1e6:7.0f} TFLOP/s", flush=True)
