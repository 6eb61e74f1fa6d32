"""Unit tests of the encoder's kernels one at a time (need an H100): the wgmma GEMM in every mode gam_encode runs it in,
the implicit-convolution GEMMs of the subsampling, the row kernels of rowops.cu, the packed-row plan and the front-end
subsampling kernels, each called through its gam_test_* entry point and compared with a float64 restatement of the same
operation.

The encoder-level tests compare 16 layers against the oracle with a relative Frobenius bar over the whole batch, which
dilutes an error confined to a few rows (one tile, one block, one utterance boundary).  Here every element is held to a
worst-case bound derived from the arithmetic, so a single wrong row fails, and rows / columns a kernel must not write are
filled with a sentinel (NaN where a read of them must not happen either) and must come back unchanged.

Bounds use these terms (u = 2^-24, the unit roundoff of fp32):
  * fp32 sums and dot products: a sum of n terms evaluated in any tree of depth d is within d * u * sum |terms| of the
    exact sum.  A k-deep chain of fp32 FMAs is a tree of depth k; the GEMM is bounded with depth K (|A||W|^T * K * u).
  * one fp16 rounding of the stored value: 2^-11 |value| (+ 2^-25 absolute below the normal range).
  * tanh.approx.f32 (SiLU and the GLU sigmoid): the PTX ISA gives a maximum relative error of about 2^-11; TANH_REL
    rounds that up to 2^-10.5.
  * __expf (the conv LayerNorm variant's SiLU): CUDA Math API, 2 + floor(|1.173 x|) ulp.
  * rsqrtf: 2 ulp.
A worst-case bound cannot fail by chance on a correct kernel; where it is meaningful a tight aggregate check (relative
Frobenius norm) is added to catch small systematic errors that stay inside the elementwise bound."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from gigaam_b200 import _lib, synthetic  # noqa: E402
from gigaam_b200.engine import (Engine, fold_batchnorm, glu_row_permutation, pack_conv1d_weight,  # noqa: E402
                                pack_conv2_weight, pack_sub_out_weight, rotary_half_tables, split_dft_basis)
from oracle import gigaam_oracle as orc  # noqa: E402

U = 2.0 ** -24                 # fp32 unit roundoff
U16 = 2.0 ** -11               # fp16 rounding, relative
F16_ABS = 2.0 ** -25           # fp16 rounding below the normal range, absolute
TANH_REL = 2.0 ** -10.5        # tanh.approx.f32, relative (PTX ISA: about 2^-11)
RSQRT_REL = 2.0 ** -22         # rsqrtf: 2 ulp
LN_EPS = 1e-5
D = 768
F32_FRO = 1e-5                 # aggregate: relative Frobenius error of fp32 outputs against float64
F16_FRO = 1e-3                 # aggregate: fp16 outputs (rms of one rounding is ~2.8e-4)
SENT16 = -4096.0               # sentinels: exact in fp16 and fp32, never produced by the tested data
SENT32 = -12345.0
NAN = float("nan")


# ------------------------------------------------------------------------------------------ plumbing
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (there is no CPU fallback to test instead)"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def eng(dev):
    ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1)
    return Engine(ck["cfg"], ck["state_dict"], dev)


@pytest.fixture(scope="module")
def nsm(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def _call(eng, fn, *args):
    """Call a gam_test_* entry point; tensor arguments are passed as device pointers and stay referenced alive here
    until the call has finished."""
    ptrs = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    rc = getattr(eng.lib, fn)(eng.handle, *ptrs, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    _lib.check(eng.lib, eng.handle, rc, fn)


def _i32(x, dev):
    return torch.as_tensor(x, dtype=torch.int32).to(dev)


def _gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _randn(shape, g, dev, scale=1.0):
    return torch.randn(shape, generator=g, device=dev, dtype=torch.float32) * scale


def _assert_within(got, want, tol, what):
    """Every element of got within tol of want (NaN in got fails); reports the worst element."""
    got, want = got.double(), want.double()
    err = (got - want).abs()
    bad = ~(err <= tol)
    if bool(bad.any()):
        idx = tuple(int(i) for i in bad.nonzero()[0])
        ratio = float((err / tol)[~torch.isnan(err)].max()) if bool((~torch.isnan(err)).any()) else float("nan")
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} elements outside the bound; first at {idx}: "
                             f"got {float(got[idx])!r}, want {float(want[idx])!r}, bound {float(tol[idx]):.3e} "
                             f"(worst err / bound {ratio:.2f})")


def _rel_fro(got, want):
    return float((got.double() - want.double()).norm() / want.double().norm().clamp_min(1e-300))


def _f16_store(v):
    """Bound of one fp16 rounding of the value v (float64)."""
    return U16 * v.abs() + F16_ABS


def _same_bits(a, b, what):
    assert torch.equal(a.view(torch.int16) if a.dtype == torch.float16 else a.view(torch.int32),
                       b.view(torch.int16) if b.dtype == torch.float16 else b.view(torch.int32)), f"{what}: changed"


# ------------------------------------------------------------------------------------------ GEMM (2-D operands)
def _gemm(eng, kind, A, W, bias, out, M, N, K, *, A2=None, n1=0, res=None, ldo=None, col0=0, scale=1.0, reverse=0, m_dev=None):
    _call(eng, "gam_test_gemm", kind, A, A2, n1, W, bias, res, out, M, N, K,
          out.shape[1] if ldo is None else ldo, col0, C.c_float(scale), reverse, m_dev)


def _acc_ref(A, W, K):
    """float64 product of the fp16 operands and the fp32-accumulation bound K * u * |A||W|^T."""
    a, w = A.double(), W.double()
    return a @ w.t(), (a.abs() @ w.abs().t()) * (K * U)


def _epilogue_ref(kind, acc, dacc, bias, res=None, scale=1.0):
    """(want, bound) of epilogue `kind` GemmKind in float64, columns in natural (un-permuted) order for the GLU."""
    x = acc + bias.double()
    dx = dacc + U * x.abs()                                   # + the rounding of the bias add
    if kind in (0, 4):
        want, tol = x, dx
    elif kind == 1:
        # silu = h + h tanh(h), h = x/2: tanh error |h| TANH_REL, one FMA rounding, |silu'| <= 1.1 carries dx
        want = x * torch.sigmoid(x)
        tol = 1.1 * dx + 0.5 * TANH_REL * x.abs() + U * want.abs()
    elif kind == 2:
        # value * sigmoid(gate), sigmoid = 0.5 + 0.5 tanh(gate/2): error 0.5 TANH_REL + u, |sigmoid'| <= 1/4
        n = x.shape[1] // 2
        a, b, da, db = x[:, :n], x[:, n:], dx[:, :n], dx[:, n:]
        sg = torch.sigmoid(b)
        want = a * sg
        tol = a.abs() * (0.5 * TANH_REL + U + 0.25 * db) + sg * da + U * want.abs()
    elif kind == 3:
        want = res.double() + scale * x
        tol = scale * dx + U * want.abs()
    else:
        raise ValueError(kind)
    if kind in (0, 1, 2):
        tol = tol + _f16_store(want)
    return want, tol


def _gemm_operands(M, N, K, dev, seed):
    g = _gen(dev, seed)
    A = _randn((M, K), g, dev, 0.5).half()
    W = _randn((N, K), g, dev, 1.0 / math.sqrt(K)).half()
    bias = _randn((N,), g, dev)
    res = _randn((M, N), g, dev)
    return A, W, bias, res


def _rows(m, nsm):
    """M of a shape: an int, or a tile count relative to the SM count (with N = 256 one 128-row block is one tile)."""
    return {"sms": 128 * nsm, "sms+1": 128 * nsm + 1, "2sms-1": 128 * (2 * nsm - 1) - 5}.get(m, m) if isinstance(m, str) else m


GEMM_SHAPES = [
    # the shapes of the former encoder-file test
    (128, 256, 64), (1000, 768, 768), (777, 768, 3072), (300, 1536, 768), (1, 256, 128),
    # row tails around the 128-row block, every N and K the encoder uses
    (127, 2304, 768), (129, 3072, 64), (255, 768, 3072), (257, 1536, 768),
    # config 2 (64 x 251 rows): FFN up / down, QKV, and the sub_out GEMM with K = F2 * d = 15360
    (16064, 3072, 768), (16064, 768, 3072), (16064, 2304, 768), (16064, 768, 15360),
    # tile counts equal to, one above, and just under twice the SM count
    ("sms", 256, 768), ("sms+1", 256, 768), ("2sms-1", 256, 64),
]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_epilogues(eng, dev, nsm, M, N, K):
    """Kinds 0-4 against float64, once dense (ldo = cols) and once reversed with a device row count of M into columns
    [64, 64 + cols) of a wider buffer whose other columns must keep their sentinel.  The GLU runs on the real
    glu_row_permutation of its weight rows."""
    M = _rows(M, nsm)
    A, W, bias, res = _gemm_operands(M, N, K, dev, 1000 + N + K + M % 997)
    acc, dacc = _acc_ref(A, W, K)
    perm = glu_row_permutation(N // 2).to(dev)
    m_dev = _i32([M], dev)
    for kind in range(5):
        Wk, bk = (W[perm].contiguous(), bias[perm].contiguous()) if kind == 2 else (W, bias)
        want, tol = _epilogue_ref(kind, acc, dacc, bias, res, 0.5)   # natural order: the GLU pairs row j with row N/2 + j
        ncol = want.shape[1]
        dt = torch.float16 if kind < 3 else torch.float32
        for reverse, wide in ((0, False), (1, True)):
            col0, ldo = (64, ncol + 128) if wide else (0, ncol)
            sent = SENT16 if kind < 3 else SENT32
            out = torch.full((M, ldo), sent, dtype=dt, device=dev)
            r = None
            if kind == 3:
                r = torch.full((M, ldo), SENT32, dtype=torch.float32, device=dev)
                r[:, col0:col0 + ncol] = res
            _gemm(eng, kind, A, Wk, bk, out, M, N, K, res=r, ldo=ldo, col0=col0, scale=0.5, reverse=reverse,
                  m_dev=m_dev if wide else None)
            what = f"kind {kind} M={M} N={N} K={K} reverse={reverse}"
            got = out[:, col0:col0 + ncol]
            _assert_within(got, want, tol, what)
            assert _rel_fro(got, want) < (F16_FRO if kind < 3 else F32_FRO), what
            if wide:
                assert bool((out[:, :col0] == sent).all() and (out[:, col0 + ncol:] == sent).all()), f"{what}: wrote outside its columns"


def test_gemm_sub_out_weight_layout(eng, dev):
    """pre_encode.out (K = F2 * d = 15360): the conv2d stage writes its rows in (f, c) order and pack_sub_out_weight
    reorders the reference weight's (c, f) K index to match, so the product is the reference's Linear over (c, f)."""
    M, F2 = 2001, 16
    K = F2 * D
    g = _gen(dev, 15)
    A = _randn((M, F2, D), g, dev, 0.5).half()                   # [rows, f, c] as the conv epilogue writes it
    Wr = _randn((D, D * F2), g, dev, 1.0 / math.sqrt(K)).half()  # pre_encode.out.weight, K index c * F2 + f
    bias = _randn((D,), g, dev)
    Wp = pack_sub_out_weight(Wr.float(), D).half().contiguous()
    acc, dacc = _acc_ref(A.permute(0, 2, 1).reshape(M, K), Wr, K)
    want, tol = _epilogue_ref(4, acc, dacc, bias)
    out = torch.full((M, D), SENT32, device=dev)
    _gemm(eng, 4, A.reshape(M, K), Wp, bias, out, M, D, K, m_dev=_i32([M], dev))
    _assert_within(out, want, tol, "sub_out")
    assert _rel_fro(out, want) < F32_FRO


@pytest.mark.parametrize("reverse", [0, 1])
@pytest.mark.parametrize("live", ["null", "M", "below", "zero", "above"])
def test_gemm_device_row_count(eng, dev, reverse, live):
    """The layer GEMMs read their row count from the device and most walk the tiles in reverse.  Rows at or past the
    live count (m_dev, clamped to [0, M]) keep their sentinel; every row below it is computed."""
    M, N, K = 16064, 768, 768
    A, W, bias, _ = _gemm_operands(M, N, K, dev, 7 + reverse)
    n_live = {"null": M, "M": M, "below": 5001, "zero": 0, "above": M}[live]
    m_dev = None if live == "null" else _i32([{"M": M, "below": 5001, "zero": 0, "above": M + 1000}[live]], dev)
    acc, dacc = _acc_ref(A[:max(n_live, 1)], W, K)
    want, tol = _epilogue_ref(0, acc, dacc, bias)
    out = torch.full((M, N + 256), SENT16, dtype=torch.float16, device=dev)
    _gemm(eng, 0, A, W, bias, out, M, N, K, col0=128, reverse=reverse, m_dev=m_dev)
    if n_live:
        _assert_within(out[:n_live, 128:128 + N], want[:n_live], tol[:n_live], f"live={live} reverse={reverse}")
    assert bool((out[n_live:] == SENT16).all()), "rows at or past the live count were written"
    assert bool((out[:, :128] == SENT16).all() and (out[:, 128 + N:] == SENT16).all()), "columns outside [col0, col0 + N) were written"


@pytest.mark.parametrize("scale", [0.5, 1.0])
def test_gemm_residual_in_place(eng, dev, scale):
    """x += scale * (A W^T + b) with res == out, as the FFN-down / projection GEMMs run: reversed, device row count below
    M, into a column window of a wider fp32 buffer.  Rows past the live count keep the residual bit for bit."""
    M, N, K, live = 4000, 768, 3072, 3001
    A, W, bias, res = _gemm_operands(M, N, K, dev, 31 + int(scale * 2))
    buf = torch.full((M, N + 256), SENT32, dtype=torch.float32, device=dev)
    buf[:, 64:64 + N] = res
    before = buf.clone()
    acc, dacc = _acc_ref(A[:live], W, K)
    want, tol = _epilogue_ref(3, acc, dacc, bias, res[:live], scale)
    _gemm(eng, 3, A, W, bias, buf, M, N, K, res=buf, col0=64, scale=scale, reverse=1, m_dev=_i32([live], dev))
    _assert_within(buf[:live, 64:64 + N], want, tol, f"in-place residual, scale {scale}")
    assert _rel_fro(buf[:live, 64:64 + N], want) < F32_FRO
    _same_bits(buf[live:], before[live:], "rows past the live count")
    _same_bits(buf[:, :64], before[:, :64], "columns left of the window")
    _same_bits(buf[:, 64 + N:], before[:, 64 + N:], "columns right of the window")


@pytest.mark.parametrize("M,live,reverse", [(16064, 16064, 1), (16064, 9999, 1), (257, 130, 0)])
def test_gemm_dual_a(eng, dev, M, live, reverse):
    """gam_encode's q/k/v projection: one launch, columns [0, 2d) from rope(u) A1 and [2d, 3d) from u (A2).  A2 is
    independent of A1, so any n-block that reads the wrong operand is off by O(1)."""
    N, K, n1 = 3 * D, D, 2 * D
    g = _gen(dev, M + live)
    A1 = _randn((M, K), g, dev, 0.5).half()
    A2 = _randn((M, K), g, dev, 0.5).half()
    W = _randn((N, K), g, dev, 1.0 / math.sqrt(K)).half()
    bias = _randn((N,), g, dev)
    acc1, d1 = _acc_ref(A1[:live], W[:n1], K)
    acc2, d2 = _acc_ref(A2[:live], W[n1:], K)
    want, tol = _epilogue_ref(0, torch.cat([acc1, acc2], 1), torch.cat([d1, d2], 1), bias)
    out = torch.full((M, N), SENT16, dtype=torch.float16, device=dev)
    _gemm(eng, 0, A1, W, bias, out, M, N, K, A2=A2, n1=n1, reverse=reverse, m_dev=_i32([live], dev))
    _assert_within(out[:live], want, tol, "dual-A q/k/v")
    assert bool((out[live:] == SENT16).all())


def test_gemm_power_spectrum(eng, dev):
    """The tensor-core log-mel's DFT GEMM: split-precision frames [hi | lo | hi] x split_dft_basis with the |X|^2
    epilogue, against the float64 product of the same operands and, loosely, against a float64 FFT of the frames
    (which checks split_dft_basis itself)."""
    n_fft, M = 400, 1001
    kp = (n_fft + 63) // 64 * 64
    g = _gen(dev, 5)
    x = (torch.randn((M, n_fft), generator=g, device=dev, dtype=torch.float64) * 0.1)      # windowed frames
    s = x * 2048.0                                                                           # frames_split_kernel's scale
    hi = s.to(torch.float16)
    lo = (s - hi.double()).to(torch.float16)
    A = torch.zeros((M, 3 * kp), dtype=torch.float16, device=dev)
    A[:, :n_fft], A[:, kp:kp + n_fft], A[:, 2 * kp:2 * kp + n_fft] = hi, lo, hi
    W = split_dft_basis(n_fft).to(dev)
    K = 3 * kp
    acc, dacc = _acc_ref(A, W, K)
    pick = lambda t, j: t.view(M, 2, 2, 128)[:, :, j, :].reshape(M, 256)   # noqa: E731  tile = [128 cos | 128 sin] rows
    re, im, dre, dim = pick(acc, 0), pick(acc, 1), pick(dacc, 0), pick(dacc, 1)
    sc = 2.0 ** -28
    want = (re * re + im * im) * sc
    tol = sc * (2 * re.abs() * dre + 2 * im.abs() * dim + dre * dre + dim * dim + 2 * U * (re * re + im * im))
    out = torch.full((M, 256 + 64), SENT32, dtype=torch.float32, device=dev)
    _gemm(eng, 7, A, W, None, out, M, 512, K, col0=32)
    _assert_within(out[:, 32:288], want, tol, "power epilogue")
    assert _rel_fro(out[:, 32:288], want) < F32_FRO
    assert bool((out[:, :32] == SENT32).all() and (out[:, 288:] == SENT32).all())
    nb = n_fft // 2 + 1
    fft = torch.fft.rfft(x, dim=-1)
    # the split operands keep ~22 bits and drop lo x lo: a few 1e-6 of relative error against the exact DFT
    assert _rel_fro(want[:, :nb], fft.real ** 2 + fft.imag ** 2) < 1e-4
    assert bool((want[:, nb:] == 0).all())


# ------------------------------------------------------------------------------------------ implicit-convolution GEMMs
def _packing(plen, gap, tail):
    """cu of utterances packed with `gap` unused frames between them and `tail` behind the last; total frames."""
    cu, r = [], 0
    for p in plen:
        cu.append(r)
        r += p + gap
    return cu, r - gap + tail


def _conv_check(out, want, tol, len_out, plen, cu, T_out, rows_per_frame, sent, what):
    """Frames t < plen[b] packed or t < T_out padded hold the reference (0 past len_out); every other row is sentinel."""
    B = len(len_out)
    written = torch.zeros(out.shape[0], dtype=torch.bool, device=out.device)
    for b in range(B):
        n = plen[b] if cu is not None else T_out
        r0 = (cu[b] if cu is not None else b * T_out) * rows_per_frame
        if n == 0:
            continue
        w = want[b, :n].reshape(n * rows_per_frame, -1)
        _assert_within(out[r0:r0 + n * rows_per_frame], w, tol[b, :n].reshape(n * rows_per_frame, -1), f"{what} utterance {b}")
        written[r0:r0 + n * rows_per_frame] = True
    assert bool((out[~written] == sent).all()), f"{what}: rows outside the utterances were written"


@pytest.mark.parametrize("packed", [False, True])
def test_gemm_conv2d_subsampling(eng, dev, packed):
    """A_CONV: the stage-2 3x3 / stride-2 / pad-1 conv over channels-last fp16 [B, T1, 32, 768] (4-D strided TMA), with
    bias, ReLU and the time mask, against float64 F.conv2d.  Lengths 0, 1, 7, 8, 9 straddle the 8-frame row block.
    Packed: frame (b, t < plen) -> row cu[b] + t, with unused frames between utterances that must keep the sentinel."""
    B, T1, F1, Cc, N = 6, 41, 32, D, D
    T2 = int(orc.sub_out_len(torch.tensor([T1]), 3, 1)[0])
    len2 = [0, 1, 7, 8, 9, T2]
    g = _gen(dev, 11)
    x = torch.rand((B, T1, F1, Cc), generator=g, device=dev).half()
    w2 = _randn((N, Cc, 3, 3), g, dev, 1.0 / math.sqrt(9 * Cc)).half()
    bias = _randn((N,), g, dev, 0.1)
    Wp = pack_conv2_weight(w2.float()).half().contiguous()
    xin = x.double().permute(0, 3, 1, 2)
    acc = F.conv2d(xin, w2.double(), stride=2, padding=1) + bias.double()[None, :, None, None]     # [B, N, T2, 16]
    dacc = F.conv2d(xin.abs(), w2.double().abs(), stride=2, padding=1) * (9 * Cc * U) + U * acc.abs()
    live = (torch.arange(T2, device=dev)[None, :] < torch.tensor(len2, device=dev)[:, None])[:, None, :, None]
    want = torch.where(live, acc.clamp_min(0), torch.zeros_like(acc)).permute(0, 2, 3, 1)        # [B, T2, 16, N]
    tol = (dacc + _f16_store(acc)).permute(0, 2, 3, 1)
    if packed:
        plen = [3, 1, 7, 12, 9, T2]            # plen > len2 for utterances 0 and 3: their extra frames are written as 0
        cu, frames = _packing(plen, 2, 3)
        cu_d, plen_d = _i32(cu, dev), _i32(plen, dev)
    else:
        plen, cu, frames, cu_d, plen_d = None, None, B * T2, None, None
    out = torch.full((frames * 16, N), SENT16, dtype=torch.float16, device=dev)
    _call(eng, "gam_test_gemm_conv", 0, x, Wp, bias, _i32(len2, dev), cu_d, plen_d, out, frames,
          B, T1, F1, Cc, 9, N, 0)
    _conv_check(out, want, tol, len2, plen, cu, T2, 16, SENT16, f"A_CONV packed={packed}")


def test_gemm_conv2d_rejects_other_frequency_widths(eng, dev):
    x = torch.zeros((1, 9, 30, D), dtype=torch.float16, device=dev)
    w = torch.zeros((D, 9 * D), dtype=torch.float16, device=dev)
    b = torch.zeros(D, device=dev)
    out = torch.zeros((5 * 16, D), dtype=torch.float16, device=dev)
    with pytest.raises(_lib.GamError, match="F1 = 32"):
        _call(eng, "gam_test_gemm_conv", 0, x, w, b, _i32([5], dev), None, None, out, 5, 1, 9, 30, D, 9, D, 0)


@pytest.mark.parametrize("taps,f32_out,packed,c_in", [(3, 0, False, 64), (5, 0, True, 64), (3, 1, True, D), (5, 1, False, D)])
def test_gemm_conv1d_subsampling(eng, dev, taps, f32_out, packed, c_in):
    """A_CONV1D: a k-tap / stride-2 conv1d over time-major fp16 [B, T_in, C] (3-D strided TMA) with bias, ReLU and the
    time mask, fp16 or fp32 out, against float64 F.conv1d.  Weights go through pack_conv1d_weight's (tap, channel)
    order; lengths 127, 128, 129 straddle the 128-frame row block."""
    B, T_in, N = 6, 600, D
    pad = (taps - 1) // 2
    T_out = int(orc.sub_out_len(torch.tensor([T_in]), taps, 1)[0])
    lens = [0, 1, 127, 128, 129, T_out]
    g = _gen(dev, 100 + taps + c_in)
    x = _randn((B, T_in, c_in), g, dev).half()
    w = _randn((N, c_in, taps), g, dev, 1.0 / math.sqrt(taps * c_in)).half()
    bias = _randn((N,), g, dev, 0.1)
    Wp = pack_conv1d_weight(w.float()).half().contiguous()
    xin = x.double().transpose(1, 2)
    acc = F.conv1d(xin, w.double(), stride=2, padding=pad) + bias.double()[None, :, None]          # [B, N, T_out]
    dacc = F.conv1d(xin.abs(), w.double().abs(), stride=2, padding=pad) * (taps * c_in * U) + U * acc.abs()
    live = (torch.arange(T_out, device=dev)[None, :] < torch.tensor(lens, device=dev)[:, None])[:, None, :]
    want = torch.where(live, acc.clamp_min(0), torch.zeros_like(acc)).transpose(1, 2)               # [B, T_out, N]
    tol = dacc.transpose(1, 2)
    if not f32_out:
        tol = tol + _f16_store(acc.transpose(1, 2))
    if packed:
        plen = [5, 1, 127, 200, 129, T_out]
        cu, frames = _packing(plen, 3, 7)
        cu_d, plen_d = _i32(cu, dev), _i32(plen, dev)
    else:
        plen, cu, frames, cu_d, plen_d = None, None, B * T_out, None, None
    sent = SENT32 if f32_out else SENT16
    out = torch.full((frames, N), sent, dtype=torch.float32 if f32_out else torch.float16, device=dev)
    _call(eng, "gam_test_gemm_conv", 1, x, Wp, bias, _i32(lens, dev), cu_d, plen_d, out, frames,
          B, T_in, 0, c_in, taps, N, f32_out)
    _conv_check(out, want, tol, lens, plen, cu, T_out, 1, sent, f"A_CONV1D taps={taps} f32={f32_out} packed={packed}")
    if f32_out:
        valid = torch.cat([want[b, :(plen[b] if packed else T_out)] for b in range(B)])
        got = torch.cat([out[(cu[b] if packed else b * T_out):][:(plen[b] if packed else T_out)] for b in range(B)])
        assert _rel_fro(got, valid) < F32_FRO


# ------------------------------------------------------------------------------------------ LayerNorm kernels
def _ln_ref(x, g, b, dx=None, depth=13):
    """float64 LayerNorm(768, eps 1e-5) of the rows of x and the bound of the kernel's fp32 result (before any fp16 store).
    The kernels sum a row in a tree of depth 13 (2 inside a float4, 6 float4 per lane, 5 shuffle levels; depth 29 for
    the depthwise kernel's 24 channels per lane); dx is an elementwise error already carried by the kernel's input."""
    x = x.double()
    g, b = g.double(), b.double()
    dx = torch.zeros_like(x) if dx is None else dx
    mu = x.mean(-1, keepdim=True)
    xc = x - mu
    var = (xc * xc).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + LN_EPS)
    y = xc * rstd * g + b
    dmu = dx.amax(-1, keepdim=True) + (depth + 3) * U * x.abs().mean(-1, keepdim=True)
    e = dx + dmu                                                          # error of x - mean as the kernel forms it
    dvar = 2 * torch.sqrt(var) * e.amax(-1, keepdim=True) + e.amax(-1, keepdim=True) ** 2 + (depth + 3) * U * var
    drstd = rstd * (0.5 * dvar / (var + LN_EPS) + RSQRT_REL + U)
    dy = g.abs() * (e * rstd + xc.abs() * drstd) + 4 * U * ((xc * rstd * g).abs() + b.abs())
    return y, dy


def _ln_rows(R, dev, seed):
    """Rows of four kinds, cycling: a large common offset (mean 1e3, std 0.1) that a one-pass variance cannot survive,
    constant rows (rstd = eps^-1/2), variance ~1e-4 where eps = 1e-5 moves the result by percents, and plain N(0, 1)."""
    g = _gen(dev, seed)
    z = _randn((R, D), g, dev)
    kind = torch.arange(R, device=dev)[:, None] % 4
    off = 1e3 + 10 * _randn((R, 1), g, dev)
    x = torch.where(kind == 0, off + 0.1 * z,
        torch.where(kind == 1, (0.7 + _randn((R, 1), g, dev)).expand(R, D),
        torch.where(kind == 2, 0.3 + 1e-2 * z, z)))
    gamma = 1.0 + 0.1 * _randn((D,), g, dev)
    beta = 0.1 * _randn((D,), g, dev)
    return x.contiguous(), gamma, beta


LIVE_MODES = [(0, "all"), (1, "all"), (1, "below"), (0, "below"), (1, "zero"), (0, "above")]


def _live(mode, R, dev):
    n = {"all": None, "below": R - 357, "zero": 0, "above": R + 100}[mode]
    return (R if n is None else min(max(n, 0), R)), (None if n is None else _i32([n], dev))


@pytest.mark.parametrize("reverse,live", LIVE_MODES)
def test_layernorm_f16(eng, dev, reverse, live):
    R = 1003
    x, gamma, beta = _ln_rows(R, dev, 1)
    n, rows_dev = _live(live, R, dev)
    out = torch.full((R, D), SENT16, dtype=torch.float16, device=dev)
    _call(eng, "gam_test_layernorm", x, gamma, beta, out, R, rows_dev, reverse)
    y, dy = _ln_ref(x[:n], gamma, beta)
    _assert_within(out[:n], y, dy + _f16_store(y), f"LayerNorm reverse={reverse} live={live}")
    assert bool((out[n:] == SENT16).all()), "rows at or past rows_dev were written"


@pytest.mark.parametrize("in_place,with_y", [(True, True), (False, True), (True, False)])
@pytest.mark.parametrize("reverse,live", [(1, "all"), (0, "below"), (1, "below")])
def test_ln_out_ln(eng, dev, in_place, with_y, reverse, live):
    """x = LN_out(r) in fp32 (in place over r as gam_encode runs it) fused with y = LN_next(x) in fp16; y is checked
    against the float64 LayerNorm of the kernel's own x."""
    R = 1003
    r, g1, b1 = _ln_rows(R, dev, 2)
    _, g2, b2 = _ln_rows(8, dev, 3)
    n, rows_dev = _live(live, R, dev)
    r0 = r.clone()
    x = r if in_place else torch.full((R, D), SENT32, device=dev)
    y = torch.full((R, D), SENT16, dtype=torch.float16, device=dev) if with_y else None
    _call(eng, "gam_test_ln_out_ln", r, g1, b1, g2, b2, x, y, R, rows_dev, reverse)
    want, tol = _ln_ref(r0[:n], g1, b1)
    _assert_within(x[:n], want, tol, "x = LN_out(r)")
    # aggregate on the N(0, 1) rows only: on the offset rows the fp32 mean of values near 1e3 alone is ~1e-3 of their std
    plain = torch.arange(n, device=dev) % 4 == 3
    assert _rel_fro(x[:n][plain], want[plain]) < F32_FRO
    if in_place:
        _same_bits(x[n:], r0[n:], "rows past rows_dev")
    else:
        assert bool((x[n:] == SENT32).all())
        _same_bits(r, r0, "the input r")
    if with_y:
        wy, ty = _ln_ref(x[:n], g2, b2)
        _assert_within(y[:n], wy, ty + _f16_store(wy), "y = LN_next(x)")
        assert bool((y[n:] == SENT16).all())


def _plan(eng, dev, mel_len, M, k=3):
    """Run gam_test_pack_plan; returns its outputs as CPU int64 tensors (row maps cut to the live rows)."""
    B = len(mel_len)
    T1 = int(orc.sub_out_len(torch.tensor([M]), k, 1)[0])
    T2 = int(orc.sub_out_len(torch.tensor([M]), k, 2)[0])
    bufs = {n: torch.full((B,), -7, dtype=torch.int32, device=dev) for n in ("len0", "len1", "len2", "plen", "run1")}
    bufs["cu"] = torch.full((B + 1,), -7, dtype=torch.int32, device=dev)
    bufs["rows_dev"] = torch.full((1,), -7, dtype=torch.int32, device=dev)
    bufs["row_b"] = torch.full((B * T2,), -7, dtype=torch.int32, device=dev)
    bufs["row_t"] = torch.full((B * T2,), -7, dtype=torch.int32, device=dev)
    ml = torch.as_tensor(mel_len, dtype=torch.int64).to(dev)
    _call(eng, "gam_test_pack_plan", ml, B, k, M, *[bufs[n] for n in ("len0", "len1", "len2", "plen", "run1", "cu",
                                                                            "rows_dev", "row_b", "row_t")])
    return {n: t.long().cpu() for n, t in bufs.items()}, T1, T2


def _rope_tables64(dk, base, dev):
    inv = 1.0 / (base ** (torch.arange(0, dk, 2, dtype=torch.float64, device=dev) / dk))
    return inv


def rope_ref(y, dy, t, dk, base):
    """The oracle's rotary formula (x * cos + rotate_half(x) * sin) on float64 tables, applied per head of dk to the rows
    y (with their error dy) at positions t, and the bound of the kernel's fp32 result with the engine's fp32
    rotary_half_tables (before the fp16 store)."""
    n = y.shape[0]
    inv = _rope_tables64(dk, base, y.device)
    ang = t.double()[:, None] * torch.cat([inv, inv])[None, :]                     # [n, dk]
    c, s = torch.cos(ang)[:, None, :], torch.sin(ang)[:, None, :]
    yh, dyh = y.view(n, D // dk, dk), dy.view(n, D // dk, dk)
    want = (yh * c + orc._rtt_half(yh) * s).reshape(n, D)
    # fp32 tables: the rounded exponent 2i/dk moves base^e by ln(5000) e u <= 8.5 u, pow (1 ulp) and the reciprocal add
    # 3 u, the product t * inv_freq one more; cos / sin of the fp32 angle within 1 ulp + rounding:
    # |table error| <= 16 u * angle + 3 u
    dtab = 16 * U * ang.abs()[:, None, :] + 3 * U
    yp = orc._rtt_half(yh).abs()
    tol = (dyh * c.abs() + orc._rtt_half(dyh).abs() * s.abs() + (yh.abs() + yp) * dtab
           + 2 * U * (yh.abs() * c.abs() + yp * s.abs())).reshape(n, D)
    return want, tol


@pytest.mark.parametrize("positions", ["plan", "row_mod_T"])
@pytest.mark.parametrize("reverse", [0, 1])
def test_ln_rope(eng, dev, positions, reverse):
    """LN + rotary embedding: out_u = LN(x), out_r = rope(LN(x)) at the row's frame position, with the engine's fp32
    rotary_half_tables, against the oracle's rotary formula (x * cos + rotate_half(x) * sin) on float64 tables.
    Positions come from a real packed plan (they restart at every utterance) or, without row_t, from row % T."""
    dk, base = D // 16, 5000
    cos, sin = (t.to(dev).contiguous() for t in rotary_half_tables(dk, base, base))
    if positions == "plan":
        plan, _, T = _plan(eng, dev, [1000, 37, 0, 1000, 501, 4, 999], 1000)
        n = int(plan["rows_dev"][0])
        R = 7 * T
        row_t = _i32(plan["row_t"][:n], dev)
        rows_dev = _i32([n], dev)
        t = plan["row_t"][:n].to(dev)
    else:
        T, R = 251, 1003
        n, row_t, rows_dev = R, None, None
        t = torch.arange(R, device=dev) % T
    x, gamma, beta = _ln_rows(R, dev, 4)
    ou = torch.full((R, D), SENT16, dtype=torch.float16, device=dev)
    orr = torch.full((R, D), SENT16, dtype=torch.float16, device=dev)
    _call(eng, "gam_test_ln_rope", x, gamma, beta, cos, sin, cos.shape[0], dk // 2, ou, orr, R,
          rows_dev, row_t, T, reverse)
    y, dy = _ln_ref(x[:n], gamma, beta)
    _assert_within(ou[:n], y, dy + _f16_store(y), "out_u")
    want, tol = rope_ref(y, dy, t, dk, base)
    _assert_within(orr[:n], want, tol + _f16_store(want), f"out_r positions={positions}")
    assert bool((ou[n:] == SENT16).all() and (orr[n:] == SENT16).all())


@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("reverse", [0, 1])
def test_unpack_rows(eng, dev, norm, reverse):
    """Packed fp32 rows -> the caller's padded [B, T, 768]: frame t < plen[b] from row cu[b] + t (LayerNorm'd for the
    last layer, a bit-exact copy for the pre_encode output), zeros for every other frame.  Rows between utterances are
    NaN: reading one shows."""
    B, T = 5, 40
    plen = [0, 1, 39, 40, 17]
    cu, rows = _packing(plen, 2, 4)
    x, gamma, beta = _ln_rows(rows, dev, 5)
    owned = torch.zeros(rows, dtype=torch.bool, device=dev)
    for b in range(B):
        owned[cu[b]:cu[b] + plen[b]] = True
    x[~owned] = NAN
    out = torch.full((B, T, D), NAN, device=dev)
    _call(eng, "gam_test_unpack_rows", x, gamma if norm else None, beta if norm else None, _i32(cu, dev),
          _i32(plen, dev), out, B, T, rows, reverse)
    for b in range(B):
        src = x[cu[b]:cu[b] + plen[b]]
        if norm and plen[b]:
            y, dy = _ln_ref(src, gamma, beta)
            _assert_within(out[b, :plen[b]], y, dy, f"utterance {b}")
        elif plen[b]:
            _same_bits(out[b, :plen[b]], src, f"utterance {b} copy")
        assert bool((out[b, plen[b]:] == 0).all()), f"utterance {b}: frames past plen are not zero"


# ------------------------------------------------------------------------------------------ depthwise conv
def _dw_case(dev, kw, seed):
    g = _gen(dev, seed)
    dw = _randn((D, kw), g, dev, 1.0 / math.sqrt(kw))
    db = 0.1 * _randn((D,), g, dev)
    bn = dict(gamma=1.0 + 0.1 * _randn((D,), g, dev), beta=0.1 * _randn((D,), g, dev), mean=0.1 * _randn((D,), g, dev),
              var=0.5 + torch.rand((D,), generator=g, device=dev))
    return dw, db, bn


def _dw_ref(frames, L, P, dw, db, bn, norm, cn):
    """float64 reference of one utterance: the first L of its P >= L frames exist (the others read as zero), output
    frames [0, P): conv1d(groups=768) + BatchNorm(eval) + SiLU, or + LayerNorm over channels + SiLU; and the bound."""
    kw = dw.shape[1]
    h = (kw - 1) // 2
    z = torch.zeros((P, D), dtype=torch.float64, device=dw.device)
    z[:L] = frames[:L].double()
    z = z.t()[None]
    w = dw.double()[:, None, :]
    acc = F.conv1d(z, w, db.double(), padding=h, groups=D)[0, :, :P].t()                           # [P, D]
    sab = F.conv1d(z.abs(), w.abs(), padding=h, groups=D)[0, :, :P].t()
    if not norm:
        s = bn["gamma"].double() / torch.sqrt(bn["var"].double() + 1e-5)
        a = (acc - bn["mean"].double()) * s + bn["beta"].double()
        # folded weights carry ~4 u each (fold_batchnorm in fp32); then a kw-deep FMA chain from the folded bias
        da = (kw + 6) * U * (sab * s.abs() + (db.double().abs() + bn["mean"].double().abs()) * s.abs() + bn["beta"].double().abs())
        want = a * torch.sigmoid(a)
        tol = 1.1 * da + 0.5 * TANH_REL * a.abs() + U * want.abs()
    else:
        da = (kw + 1) * U * (sab + db.double().abs())
        y, dy = _ln_ref(acc, cn[0], cn[1], da, depth=29)
        want = y * torch.sigmoid(y)
        # x / (1 + __expf(-x)): __expf within (2 + 1.173 |x|) ulp, one add, one IEEE division
        tol = 1.1 * dy + ((2 + 1.2 * y.abs()) * 2 * U + 3 * U) * want.abs()
    return want, tol + _f16_store(want)


@pytest.mark.parametrize("layout", ["packed", "padded", "single"])
@pytest.mark.parametrize("kw", [5, 31])
@pytest.mark.parametrize("norm", [False, True])
def test_dwconv(eng, dev, norm, kw, layout):
    """Depthwise conv + (folded BatchNorm | LayerNorm over channels) + SiLU, each utterance against its own float64
    conv1d.  Lengths 0, 1, 31, 32, 33 straddle the 32-frame time tile.  Every utterance is run with all other rows --
    its neighbours' and the rows behind the stream -- set to NaN, so a halo that crosses a boundary shows.  Frames at or
    past len that stay in the stream (padded layout, and the batch of one, whose plen is T) are NaN too: they must be
    read as zero."""
    T = 70
    lens = [45] if layout == "single" else [0, 1, 31, 32, 33, T]
    B = len(lens)
    dw, db, bn = _dw_case(dev, kw, 10 * kw + norm)
    cn = (1.0 + 0.1 * _randn((D,), _gen(dev, 3), dev), 0.1 * _randn((D,), _gen(dev, 4), dev))
    if norm:
        w_k, b_k = dw.t().contiguous(), db
    else:
        wf, bf = fold_batchnorm(dw, db, bn["gamma"], bn["beta"], bn["mean"], bn["var"])
        w_k, b_k = wf.t().contiguous(), bf
    if layout == "padded":
        plen, cu, rows = [T] * B, [b * T for b in range(B)], B * T
    else:
        plen = [T] if layout == "single" else lens                  # the encoder's rule: plen = len, a batch of one keeps T
        cu, n = _packing(plen, 0, 0)
        rows = max(B * T, n) + 8
    n_live = cu[-1] + plen[-1]
    row_b = torch.full((rows,), -1, dtype=torch.int32)
    row_t = torch.full((rows,), -1, dtype=torch.int32)
    for b in range(B):
        row_b[cu[b]:cu[b] + plen[b]] = b
        row_t[cu[b]:cu[b] + plen[b]] = torch.arange(plen[b], dtype=torch.int32)
    data = _randn((rows, D), _gen(dev, 77), dev).half()
    packed = layout != "padded"
    args_tail = (_i32(lens, dev), _i32(cu, dev) if packed else None, _i32(plen, dev) if packed else None,
                 row_b[:n_live].contiguous().to(dev) if packed else None, row_t[:n_live].contiguous().to(dev) if packed else None,
                 _i32([n_live], dev) if packed else None)
    for b in range(B):
        if plen[b] == 0:
            continue
        g = torch.full((rows, D), NAN, dtype=torch.float16, device=dev)
        g[cu[b]:cu[b] + lens[b]] = data[cu[b]:cu[b] + lens[b]]      # frames past len stay NaN
        out = torch.full((rows, D), SENT16, dtype=torch.float16, device=dev)
        _call(eng, "gam_test_dwconv", int(norm), g, w_k, b_k, cn[0] if norm else None, cn[1] if norm else None,
              *args_tail, out, B, T, rows, kw)
        want, tol = _dw_ref(data[cu[b]:cu[b] + lens[b]], lens[b], plen[b], dw, db, bn, norm, cn)
        _assert_within(out[cu[b]:cu[b] + plen[b]], want, tol, f"norm={norm} kw={kw} {layout} utterance {b} (len {lens[b]})")
        if not norm:   # the BatchNorm kernel writes only frames that exist (the LayerNorm one also runs the NaN rows)
            others = torch.ones(rows, dtype=torch.bool, device=dev)
            for bb in range(B):
                others[cu[bb]:cu[bb] + plen[bb]] = False
            assert bool((out[others] == SENT16).all()), "rows outside every utterance were written"


# ------------------------------------------------------------------------------------------ packed-row plan
def _plan_ref(mel_len, M, k=3):
    """float32 restatement of the stage lengths (gigaam/encoder.py:77-90, as oracle.sub_out_len) and of the plan rules of
    pack_plan_kernel / row_map_kernel."""
    ml = torch.as_tensor(mel_len, dtype=torch.int64)
    B = ml.numel()
    T1 = int(orc.sub_out_len(torch.tensor([M]), k, 1)[0])
    T2 = int(orc.sub_out_len(torch.tensor([M]), k, 2)[0])
    len1 = orc.sub_out_len(ml, k, 1).long()
    len2 = orc.sub_out_len(ml, k, 2).long()
    plen = len2.clamp(0, T2) if B > 1 else torch.full((B,), T2, dtype=torch.int64)
    run1 = torch.minimum(torch.tensor(T1), 2 * ((plen + 7) // 8 * 8) + 2) if B > 1 else torch.full((B,), T1, dtype=torch.int64)
    cu = torch.cat([torch.zeros(1, dtype=torch.int64), plen.cumsum(0)])
    n = int(cu[-1])
    row_b = torch.repeat_interleave(torch.arange(B), plen)
    row_t = torch.arange(n) - cu[:-1][row_b] if n else torch.zeros(0, dtype=torch.int64)
    return dict(len0=ml.clamp(max=M), len1=len1, len2=len2, plen=plen, run1=run1, cu=cu, rows_dev=cu[-1:], row_b=row_b, row_t=row_t)


@pytest.mark.parametrize("B", [1, 2, 31, 33, 1023, 1024, 1025, 3000])
def test_pack_plan(eng, dev, B):
    """Every output of the plan, exactly.  B > 1024 takes the kernel's chunked prefix sum with a carried total, which no
    benchmark batch reaches.  Lengths include 0, 1 (the shortest that still gives a frame) and the maximum."""
    M = 1500
    g = torch.Generator().manual_seed(B)
    ml = torch.randint(0, M + 1, (B,), generator=g)
    special = torch.tensor([0, 1, M, 1, 0, M])
    ml[:min(B, 6)] = special[:min(B, 6)]
    ml = ml[torch.randperm(B, generator=g)]
    want = _plan_ref(ml.tolist(), M)
    got, _, T2 = _plan(eng, dev, ml.tolist(), M)
    n = int(want["cu"][-1])
    for name in ("len0", "len1", "len2", "plen", "run1", "cu", "rows_dev"):
        assert torch.equal(got[name], want[name]), f"{name} differs (B={B})"
    assert torch.equal(got["row_b"][:n], want["row_b"]) and torch.equal(got["row_t"][:n], want["row_t"])
    assert bool((got["row_b"][n:] == -7).all() and (got["row_t"][n:] == -7).all()), "row maps written past the live rows"


# ------------------------------------------------------------------------------------------ front-end subsampling
@pytest.mark.parametrize("with_run1", [False, True])
def test_subsample_conv1(eng, dev, with_run1):
    """Stage 1 of the conv2d subsampling (1 -> 768 channels, 3x3 / stride 2 / pad 1, fp32 CUDA cores, channels-last
    fp16 out) against float64 F.conv2d on the time-masked mel, with ragged len0 / len1.  run1 skips whole 8-frame
    blocks from run1[b] on: those rows keep the sentinel."""
    B, Fm, M, Cc = 5, 64, 203, D
    len0 = [0, 1, 2, 150, M]
    T1 = int(orc.sub_out_len(torch.tensor([M]), 3, 1)[0])
    F1 = int(orc.sub_out_len(torch.tensor([Fm]), 3, 1)[0])
    len1 = orc.sub_out_len(torch.tensor(len0), 3, 1).tolist()
    run1 = [min(T1, r) for r in (2, 3, 10, 77, 200)] if with_run1 else None
    g = _gen(dev, 21)
    mel = _randn((B, Fm, M), g, dev, 3.0)
    w = _randn((Cc, 1, 3, 3), g, dev, 1.0 / 3)
    bias = 0.1 * _randn((Cc,), g, dev)
    out = torch.full((B, T1, F1, Cc), SENT16, dtype=torch.float16, device=dev)
    _call(eng, "gam_test_subsample_conv1", mel, _i32(len0, dev), _i32(len1, dev), _i32(run1, dev) if run1 else None,
          (w.reshape(Cc, 9).contiguous()), bias, out, B, Fm, M, Cc)
    t = torch.arange(M, device=dev)
    x = torch.where(t[None, None, :] < torch.tensor(len0, device=dev)[:, None, None], mel, torch.zeros_like(mel))
    xin = x.double().transpose(1, 2)[:, None]                                                       # [B, 1, M, F]
    acc = F.conv2d(xin, w.double(), bias.double(), stride=2, padding=1)                            # [B, C, T1, F1]
    dacc = F.conv2d(xin.abs(), w.double().abs(), bias.double().abs(), stride=2, padding=1) * (10 * U)
    live = (torch.arange(T1, device=dev)[None, :] < torch.tensor(len1, device=dev)[:, None])[:, None, :, None]
    want = torch.where(live, acc.clamp_min(0), torch.zeros_like(acc)).permute(0, 2, 3, 1)
    tol = (dacc + _f16_store(acc)).permute(0, 2, 3, 1)
    for b in range(B):
        n = T1 if run1 is None else min(T1, (run1[b] + 7) // 8 * 8)
        _assert_within(out[b, :n], want[b, :n], tol[b, :n], f"utterance {b}")
        assert bool((out[b, n:] == SENT16).all()), f"utterance {b}: blocks past run1 were written"


def test_mel_to_tmajor(eng, dev):
    """mel [B, F, M] f32 -> time-major fp16 [B, M, F] with frames >= len0 zeroed, bit-exact against mel.half();
    F and M are not multiples of the 32 x 32 transpose tile."""
    B, Fm, M = 3, 70, 333
    len0 = [0, 100, 400]
    mel = _randn((B, Fm, M), _gen(dev, 9), dev, 4.0)
    out = torch.full((B, M, Fm), NAN, dtype=torch.float16, device=dev)
    _call(eng, "gam_test_mel_to_tmajor", mel, _i32(len0, dev), out, B, Fm, M)
    keep = torch.arange(M, device=dev)[None, :, None] < torch.tensor(len0, device=dev)[:, None, None]
    want = torch.where(keep, mel.transpose(1, 2), torch.zeros((), device=dev)).half()
    _same_bits(out, want.contiguous(), "mel_to_tmajor")
