"""Unit tests of the log-mel front end against a float64 STFT (GPU tests need an H100): frames_split_kernel and
mel_log_kernel one at a time through their gam_test_* entry points, and the two whole paths -- the tensor-core
gam_logmel_tc (frames -> fp16 split -> DFT GEMM -> sparse mel) and the fused CUDA-core gam_logmel -- at the lengths,
batch shapes, signals and amplitudes where a front end goes wrong.

The float64 reference restates gigaam/preprocess.py:43-50: reflect padding for center=True (plain frames otherwise),
frames x the checkpoint's window, torch.fft.rfft, |X|^2, @ fb, clamp to [1e-9, 1e9] (NaN stays NaN), log.

Bounds use u = 2^-24 (fp32) and these terms, per (utterance, frame, bin) with G = sum_j |x_j w_j| |cos or sin(2 pi k j / n)|:
  * tensor-core DFT, in the frame's own units: the dropped lo x lo product, the roundings of lo and d_lo (2^-22 |term|
    each) and the fp32 accumulation over K = 3 Kp (K u sum |terms|), plus 2^-25 per fp16 element below the normal range:
    |re error| <= (K u + 3 * 2^-22 + u) G + 2^-23 (n 2^-e + sum |x w| / 8), the same for im (test_gemm_power_spectrum
    derives the product part on given operands).  The fused kernel's DFT is an fp32 FMA chain of depth n/2 + 1 over folded
    samples: (n/2 + 5) u G.
  * |X|^2: 2 |re| dre + dre^2 (+ im) and the epilogue's roundings, 3 u |X|^2.
  * mel projection: an fp32 FMA chain of depth mel_hi - mel_lo (tensor-core path) or n/2 + 1 (fused), so
    dmel = depth u (P + dP) . fb + dP . fb.
  * clamp is 1-Lipschitz and log' = 1/x: dlog = dmel / clamp(mel - dmel), plus one fp32 rounding of the clamped value
    (u) and logf's 1 ulp (CUDA Math API), 2^-23 |log|.
A worst-case bound cannot fail by chance on a correct kernel; a relative Frobenius check of the mel powers on top catches
small systematic errors that stay inside it."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gigaam_b200 import _lib, synthetic
from gigaam_b200.engine import Engine
from oracle import gigaam_oracle as orc

gpu = pytest.mark.gpu

U = 2.0 ** -24                 # fp32 unit roundoff
F32_FRO = 1e-5                 # aggregate: relative Frobenius error against float64 (mel powers for the whole paths)
SENT32 = -12345.0              # sentinels: exact in fp32 and fp16, never produced by the tested data
SENT16 = -4096.0
NAN = float("nan")
CLAMP_LO, CLAMP_HI = float(np.float32(1e-9)), float(np.float32(1e9))   # the fp32 constants the kernels clamp with
GEOMETRY = {"v2": dict(n_fft=400, hop=160, center=True), "v3": dict(n_fft=320, hop=160, center=False)}
# v2: the smallest length reflect padding accepts (n_fft/2 + 1) and its neighbours, one and three frames around n_fft,
# then lengths giving M = 31 .. 129 frames around the 32-row mel_log block and the 64 / 128-row blocks
LENGTHS = {
    "v2": [201, 202, 399, 400, 401, 479, 480, 481] + [(m - 1) * 160 + 37 for m in (31, 32, 33, 63, 64, 65, 127, 128, 129)],
    "v3": [320, 321, 479, 480, 481] + [320 + (m - 1) * 160 + 11 for m in (31, 32, 33, 63, 64, 65, 127, 128, 129)],
}
AMPLITUDES = [1.0, 15.9, 31.9, 32.0, 33.0, 1000.0, 32767.0, 2.0 ** 31]
_RATIOS = {}                   # worst err / bound per bound, printed by each test (pytest -s)


# ------------------------------------------------------------------------------------------ plumbing
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (there is no CPU fallback to test instead)"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def engines(dev):
    out = {}
    for geo, name in (("v2", "v2_ctc"), ("v3", "v3_ctc")):
        ck = synthetic.synthetic_checkpoint(name, seed=0, n_layers=1)
        out[geo] = (Engine(ck["cfg"], ck["state_dict"], dev), ck["state_dict"])
    return out


@pytest.fixture(scope="module")
def log_floor(dev):
    """logf(1e-9f) as the GPU computes it: the value every silent frame must hold exactly."""
    v = float(torch.log(torch.tensor([CLAMP_LO], dtype=torch.float32, device=dev))[0])
    assert abs(v - math.log(CLAMP_LO)) <= 2.0 ** -23 * abs(v)
    return v


def _call(eng, fn, *args):
    ptrs = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    rc = getattr(eng.lib, fn)(eng.handle, *ptrs, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    _lib.check(eng.lib, eng.handle, rc, fn)


def _i32(x, dev):
    return torch.as_tensor(x, dtype=torch.int32).to(dev)


def _rel_fro(got, want):
    return float((got.double() - want.double()).norm() / want.double().norm().clamp_min(1e-300))


def _ratio(name, err, tol):
    finite = torch.isfinite(err)
    r = float((err[finite] / tol[finite]).max()) if bool(finite.any()) else 0.0
    _RATIOS[name] = max(_RATIOS.get(name, 0.0), r)
    return r


def _assert_within(got, want, tol, what, name):
    """Every element of got within tol of want (NaN in got fails); reports the worst element."""
    got, want = got.double(), want.double()
    err = (got - want).abs()
    bad = ~(err <= tol)
    if bool(bad.any()):
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} elements outside the bound; first at {idx}: "
                             f"got {float(got[idx])!r}, want {float(want[idx])!r}, bound {float(tol[idx]):.3e} "
                             f"(worst err / bound {_ratio(name, err, tol):.2f})")
    _ratio(name, err, tol)


def _report():
    print("worst err / bound: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(_RATIOS.items())))


# ------------------------------------------------------------------------------------------ float64 reference
def _frames(wav, n_fft, hop, center):
    """[B, M, n_fft] frames of wav (any dtype) as torch.stft / the reference cut them: reflect-padded by n_fft/2 when centered."""
    x = wav
    if center:
        x = F.pad(x[:, None], (n_fft // 2, n_fft // 2), mode="reflect")[:, 0]
    return x.unfold(-1, n_fft, hop)


def _basis(n_fft, dev):
    j = torch.arange(n_fft, dtype=torch.float64, device=dev)
    k = torch.arange(n_fft // 2 + 1, dtype=torch.float64, device=dev)
    ang = 2.0 * math.pi * torch.outer(j, k) / n_fft
    return torch.cos(ang).abs(), torch.sin(ang).abs()          # [n, nb]


def _frame_exponent(v):
    """frames_split_kernel's per-frame power of two: 11 unless max |x.w| (NaN ignored) x 2^11 rounds to inf in fp16, then
    14 - ilogb(max), so that every hi stays below 2^15."""
    amax = torch.nan_to_num(v.float().abs(), nan=0.0).amax(-1)
    e_big = 14 - (torch.frexp(amax)[1] - 1)
    return torch.where(amax * 2048.0 < 65520.0, torch.full_like(e_big, 11), e_big.clamp_min(-126)).to(torch.int32)


def _mel_bound(P, dP, fb, depth):
    """float64 mel sums and the bound of their fp32 evaluation (FMA chains of `depth` per mel) on power P +- dP."""
    fb = fb.double()
    mel = P @ fb
    dmel = ((P + dP) @ fb) * (depth.double() * U)[None, None, :] + dP @ fb
    return mel, dmel


def _log_bound(mel, dmel):
    """(want, bound) of logf(clamp(fp32 mel)) for float64 mel within dmel: NaN stays NaN."""
    want = torch.log(mel.clamp(CLAMP_LO, CLAMP_HI))
    low = (mel - dmel).clamp(CLAMP_LO, CLAMP_HI)
    return want, dmel / low + U + 2.0 ** -23 * want.abs()


def _reference(wav, sd, geo, path, mel_lo=None, mel_hi=None):
    """float64 log-mel [B, n_mels, M] of wav and the bound of `path` ('tc' | 'fused') per element."""
    g = GEOMETRY[geo]
    n = g["n_fft"]
    window = sd["preprocessor.featurizer.0.spectrogram.window"].to(wav.device)
    fb = sd["preprocessor.featurizer.0.mel_scale.fb"].to(wav.device)
    x = _frames(wav.double(), n, g["hop"], g["center"])
    xw = x * window.double()
    spec = torch.fft.rfft(xw, dim=-1)
    re, im = spec.real.abs(), spec.imag.abs()
    P = re * re + im * im
    nan_frame = torch.isnan(xw).any(-1)
    A = torch.nan_to_num(xw, nan=0.0).abs()
    cb, sb = _basis(n, wav.device)
    Gc, Gs = A @ cb, A @ sb
    if path == "tc":
        kp = (n + 63) // 64 * 64
        e = _frame_exponent(_frames(wav.float(), n, g["hop"], g["center"]) * window.float()).double()[..., None]
        c1 = 3 * kp * U * (1 + 2.0 ** -9) + 3 * 2.0 ** -22 * (1 + 2.0 ** -9) + U
        a = 2.0 ** -23 * (n * torch.exp2(-e) + A.sum(-1, keepdim=True) / 8.0)
        dre, dim_ = c1 * Gc + a, c1 * Gs + a
        sub = 2.0 ** -149 * torch.exp2(22 - 2 * e)              # the epilogue's output below the fp32 normal range
        depth = (mel_hi - mel_lo).to(wav.device)
    else:
        c1 = (n // 2 + 5) * U
        dre, dim_ = c1 * Gc, c1 * Gs
        sub = 2.0 ** -149
        depth = torch.full((fb.shape[1],), n // 2 + 1, device=wav.device)
    dP = 2 * re * dre + dre * dre + 2 * im * dim_ + dim_ * dim_ + 3 * U * ((re + dre) ** 2 + (im + dim_) ** 2) + sub
    P = torch.where(nan_frame[..., None], torch.full_like(P, NAN), P)
    mel, dmel = _mel_bound(P, dP, fb, depth)
    want, tol = _log_bound(mel, dmel)
    return want.transpose(1, 2), tol.transpose(1, 2), nan_frame, (xw != 0).any(-1) & ~nan_frame


# ------------------------------------------------------------------------------------------ running the paths
def _run(eng, wav, fused):
    """One path over [B, N] into a buffer with a sentinel guard behind [B, n_mels, M]; the tensor-core path gets a
    NaN-filled workspace so that a read of a workspace byte it did not write shows."""
    B, N = wav.shape
    M = eng.logmel_frames(N)
    total = B * eng.n_mels * M
    out = torch.full((total + 1024,), SENT32, dtype=torch.float32, device=wav.device)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if fused:
        rc = eng.lib.gam_logmel(eng.handle, wav.data_ptr(), B, N, out.data_ptr(), stream)
    else:
        ws = torch.full((int(eng.lib.gam_logmel_workspace_bytes(eng.handle, B, N)),), 255, dtype=torch.uint8, device=wav.device)
        rc = eng.lib.gam_logmel_tc(eng.handle, wav.data_ptr(), B, N, out.data_ptr(), ws.data_ptr(), ws.numel(), stream)
    torch.cuda.synchronize()
    _lib.check(eng.lib, eng.handle, rc, "gam_logmel" if fused else "gam_logmel_tc")
    assert bool((out[total:] == SENT32).all()), "written past [B, n_mels, M]"
    return out[:total].view(B, eng.n_mels, M)


def _mel_ranges(sd):
    fb = sd["preprocessor.featurizer.0.mel_scale.fb"]
    nz = fb != 0
    lo = torch.where(nz.any(0), nz.float().argmax(0), torch.zeros(fb.shape[1], dtype=torch.long))
    hi = torch.where(nz.any(0), fb.shape[0] - nz.flip(0).float().argmax(0), torch.zeros(fb.shape[1], dtype=torch.long))
    return lo, hi


def _check_path(eng, sd, geo, wav, path, log_floor, what):
    got = _run(eng, wav, path == "fused")
    lo, hi = _mel_ranges(sd)
    want, tol, nan_frame, seen = _reference(wav, sd, geo, path, lo, hi)
    name = f"{path} {geo}"
    empty = (lo == hi).to(wav.device)                       # mels whose filter has no bin
    want_nan = nan_frame[:, None, :].expand_as(want)
    if path == "tc":                                        # the sparse loop never multiplies an empty filter's zeros
        want_nan = want_nan & ~empty[None, :, None]
    assert torch.equal(torch.isnan(got), want_nan), f"{what}: NaN where the reference has none, or the reverse"
    if path == "tc" and bool(empty.any()):
        assert bool((got[:, empty][nan_frame[:, None, :].expand(-1, int(empty.sum()), -1)] == log_floor).all())
    ok = ~want_nan & ~torch.isnan(want)
    _assert_within(got[ok], want[ok], tol[ok], what, name)
    silent = ~seen[:, None, :].expand_as(got) & ~want_nan
    assert bool((got[silent] == log_floor).all()), f"{what}: a frame no sample reaches is not exactly logf(1e-9f)"
    if bool(ok.any()):                                      # on the mel powers: the loud bins, where the split keeps ~22 bits
        agg = _rel_fro(got[ok].double().exp(), want[ok].exp())
        _RATIOS[f"{name} rel-fro"] = max(_RATIOS.get(f"{name} rel-fro", 0.0), agg)
        assert agg < F32_FRO, f"{what}: relative Frobenius error of the mel powers {agg:.2e}"
    return got


# ------------------------------------------------------------------------------------------ signals
def _signal(kind, B, n, seed, dev, amp=1.0):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n, dtype=torch.float64)
    if kind == "zeros":
        x = torch.zeros(B, n, dtype=torch.float64)
    elif kind == "impulse":                                 # per row: sample 0, n - 1, a hop boundary, one past it
        x = torch.zeros(B, n, dtype=torch.float64)
        for b in range(B):
            x[b, [0, n - 1, 160 * max(1, n // 320), min(160 * max(1, n // 320) + 1, n - 1)][b % 4]] = 1.0
    elif kind == "noise":
        x = 0.3 * torch.randn(B, n, generator=g, dtype=torch.float64)
    elif kind == "tones":
        x = synthetic.synthetic_audio(B, n / synthetic.SAMPLE_RATE, seed=seed)[0].double()
    elif kind == "square":                                  # +-amp: |x w| reaches amp where the window is 1
        f = 150.0 + 70.0 * torch.arange(B, dtype=torch.float64)[:, None]
        x = torch.where(torch.sin(2 * math.pi * f * t[None, :] / 16000.0) >= 0, 1.0, -1.0)
    elif kind == "dither":                                  # one int16 step
        x = torch.randint(-1, 2, (B, n), generator=g).double() * (1.0 / 32768.0)
    else:
        raise ValueError(kind)
    return (x * amp).float().to(dev)


SIGNALS = ["zeros", "impulse", "noise", "tones", "square", "dither"]


# ------------------------------------------------------------------------------------------ frames_split_kernel
def _split_ref(wav, window, n_fft, hop, center):
    """A' = [hi | lo | hi] and the per-frame exponent, restated in torch: v = fp32(x w) 2^e, hi = fp16(v),
    lo = fp16(v - hi), columns [n_fft, Kp) zero."""
    kp = (n_fft + 63) // 64 * 64
    v = _frames(wav, n_fft, hop, center) * window                     # fp32 products, as the kernel forms them
    B, M, _ = v.shape
    e = _frame_exponent(v)
    s = v * torch.exp2(e.float())[..., None]
    hi = s.half()
    lo = (s - hi.float()).half()
    A = torch.zeros((B * M, 3 * kp), dtype=torch.float16, device=wav.device)
    A[:, :n_fft], A[:, kp:kp + n_fft], A[:, 2 * kp:2 * kp + n_fft] = hi.reshape(B * M, -1), lo.reshape(B * M, -1), hi.reshape(B * M, -1)
    return A, e.reshape(-1)


def _same_bits_nan(got, want, what):
    gn, wn = torch.isnan(got), torch.isnan(want)
    assert torch.equal(gn, wn), f"{what}: NaN positions differ"
    assert torch.equal(got[~gn].view(torch.int16), want[~wn].view(torch.int16)), f"{what}: bits differ"


@gpu
@pytest.mark.parametrize("geo", ["v2", "v3"])
@pytest.mark.parametrize("kind,amp", [("noise", 1.0), ("tones", 31.9), ("square", 32.0), ("square", 33.0), ("tones", 32767.0),
                                      ("square", 2.0 ** 31), ("dither", 1.0), ("nan", 1.0)])
def test_frames_split_bits(engines, dev, geo, kind, amp):
    """A' and the per-frame exponents bit for bit, with rows of different amplitude in one batch (one row at 1 keeps
    e = 11 beside loud rows), at lengths around the 8-frame block; rows behind the last frame keep their sentinel."""
    eng, sd = engines[geo]
    g = GEOMETRY[geo]
    window = sd["preprocessor.featurizer.0.spectrogram.window"].to(dev)
    kp = (g["n_fft"] + 63) // 64 * 64
    for n in LENGTHS[geo][:3] + [LENGTHS[geo][-1]]:
        wav = _signal("noise" if kind == "nan" else kind, 3, n, n, dev, amp)
        wav[0] = _signal("noise", 1, n, n + 1, dev)[0]
        if kind == "nan":
            wav[1, n // 2] = NAN
        M = eng.logmel_frames(n)
        A = torch.full((3 * M + 8, 3 * kp), SENT16, dtype=torch.float16, device=dev)
        fexp = torch.full((3 * M + 8,), -999, dtype=torch.int32, device=dev)
        _call(eng, "gam_test_frames_split", wav, 3, n, A, fexp)
        want_a, want_e = _split_ref(wav, window, g["n_fft"], g["hop"], g["center"])
        what = f"{geo} {kind} x{amp} n={n}"
        assert torch.equal(fexp[:3 * M], want_e), f"{what}: exponents differ"
        _same_bits_nan(A[:3 * M], want_a, what)
        assert bool((A[3 * M:] == SENT16).all() and (fexp[3 * M:] == -999).all()), f"{what}: wrote past the last frame"
        assert bool(torch.isfinite(A[:3 * M][~torch.isnan(A[:3 * M])]).all()), f"{what}: a split value overflowed"
        if amp <= 31.9:
            assert bool((fexp[:3 * M] == 11).all())


# ------------------------------------------------------------------------------------------ mel_log_kernel
def _filterbanks():
    """(name, fb [nbins, 64]): the synthetic v2 (201 bins) and v3 (161 bins) HTK banks, and the v2 bank with mel 5 emptied."""
    v2 = synthetic.mel_filterbank(201, 64, 16000)
    v3 = synthetic.mel_filterbank(161, 64, 16000)
    z = v2.clone()
    z[:, 5] = 0.0
    return [("v2", v2), ("v3", v3), ("v2-empty-mel", z)]


@gpu
@pytest.mark.parametrize("fb_name", ["v2", "v3", "v2-empty-mel"])
def test_mel_log(engines, dev, log_floor, fb_name):
    """Power rows -> log mel against float64, on frame counts around the 32-row block, with per-frame exponents from
    -16 to 11 (the 2^(22 - 2e) undo must be exact) and rows of silence, of power past the 1e9 clamp and of NaN."""
    eng, _ = engines["v2"]
    fb = dict(_filterbanks())[fb_name].to(dev)
    nb = fb.shape[0]
    nz = fb.cpu() != 0
    lo = torch.where(nz.any(0), nz.float().argmax(0), torch.zeros(64, dtype=torch.long))
    hi = torch.where(nz.any(0), nb - nz.flip(0).float().argmax(0), torch.zeros(64, dtype=torch.long))
    empty = (lo == hi).to(dev)
    assert bool(empty.any()) == (fb_name == "v2-empty-mel")
    for B, M in ((1, 1), (3, 31), (2, 33), (1, 64), (2, 97)):
        g = torch.Generator(device=dev).manual_seed(B * 100 + M)
        e = torch.randint(-16, 12, (B * M,), generator=g, device=dev, dtype=torch.int32)
        e[::3] = 11
        true = torch.rand((B * M, 256), generator=g, device=dev, dtype=torch.float64) * torch.exp2(
            torch.randint(-40, 30, (B * M, 1), generator=g, device=dev).double())
        true[0, :nb] = 0.0                                        # silence
        if B * M > 2:
            true[1, :nb] = 1e12                                   # past the upper clamp
            true[2, :nb] = NAN                                    # a frame with a NaN sample has NaN in every bin
        P = (true * torch.exp2(2 * e.double() - 22)[:, None]).float()   # what the GEMM epilogue stores
        P[:, nb:] = SENT32                                        # columns past nbins must not be read
        Pd = P.double() * torch.exp2(22 - 2 * e.double())[:, None]      # the exact power the kernel sees after the undo
        out = torch.full((B * 64 * M + 64,), SENT32, device=dev)
        _call(eng, "gam_test_mel_log", P, e, B, M, nb, fb, _i32(lo, dev), _i32(hi, dev), 64, out)
        got = out[:B * 64 * M].view(B, 64, M)
        assert bool((out[B * 64 * M:] == SENT32).all()), "written past [B, 64, M]"
        Pm = Pd[:, :nb].view(B, M, nb)
        mel, dmel = _mel_bound(Pm, torch.zeros_like(Pm), fb, (hi - lo).to(dev))
        want, tol = _log_bound(mel, dmel)
        want, tol = want.transpose(1, 2), tol.transpose(1, 2)
        nan_rows = torch.isnan(Pm).any(-1)[:, None, :] & ~empty[None, :, None]
        what = f"{fb_name} B={B} M={M}"
        assert torch.equal(torch.isnan(got), nan_rows), f"{what}: NaN rows"
        ok = ~torch.isnan(want)
        _assert_within(got[ok], want[ok], tol[ok], what, "mel_log")
        assert _rel_fro(got[ok], want[ok]) < F32_FRO
        assert bool((got[0, :, 0] == log_floor).all()), f"{what}: silence is not exactly logf(1e-9f)"
        if bool(empty.any()):                                     # lo = hi = 0: logf(1e-9f) even in the NaN row
            assert bool((got[:, empty] == log_floor).all())
    _report()


def test_mel_log_filterbanks_have_no_empty_mel():
    """Neither real-geometry bank has a mel with an empty filter, so the NaN exception of the sparse loop (an empty mel stays
    at logf(1e-9f) in a NaN frame while the dense reference gives NaN) does not arise on the shipped configurations."""
    for name, fb in _filterbanks()[:2]:
        assert bool((fb != 0).any(0).all()), name


# ------------------------------------------------------------------------------------------ whole paths
@gpu
@pytest.mark.parametrize("path", ["tc", "fused"])
@pytest.mark.parametrize("geo", ["v2", "v3"])
@pytest.mark.parametrize("kind", SIGNALS)
def test_logmel_paths(engines, dev, log_floor, path, geo, kind):
    """Both paths against float64 at every length of LENGTHS with three different utterances per batch."""
    eng, sd = engines[geo]
    for n in LENGTHS[geo]:
        wav = _signal(kind, 3, n, 7 * n + len(kind), dev)
        _check_path(eng, sd, geo, wav, path, log_floor, f"{path} {geo} {kind} n={n}")
    _report()


@gpu
@pytest.mark.parametrize("path", ["tc", "fused"])
@pytest.mark.parametrize("geo", ["v2", "v3"])
@pytest.mark.parametrize("amp", AMPLITUDES)
def test_logmel_amplitudes(engines, dev, log_floor, path, geo, amp):
    """Square waves and tones at amplitudes up to 2^31: frames with |x w| >= 32 used to store an fp16 hi of inf, which
    made every bin NaN and the clamp turned that into silence (logf(1e-9f)) on the tensor-core path."""
    eng, sd = engines[geo]
    for n in (LENGTHS[geo][1], LENGTHS[geo][-4]):
        for kind in ("square", "tones"):
            wav = _signal(kind, 3, n, n, dev, amp)
            _check_path(eng, sd, geo, wav, path, log_floor, f"{path} {geo} {kind} x{amp} n={n}")
    _report()


@gpu
@pytest.mark.parametrize("path", ["tc", "fused"])
@pytest.mark.parametrize("geo", ["v2", "v3"])
def test_logmel_batch_of_64(engines, dev, log_floor, path, geo):
    """B = 64 utterances of M = 65 frames: the 128-row GEMM tiles and 64-frame blocks hold frames of two utterances; every
    row has its own content and amplitude, so a frame read from the wrong utterance or exponent shows."""
    eng, sd = engines[geo]
    n = LENGTHS[geo][-4]
    wav = _signal("noise", 64, n, 5, dev)
    wav *= torch.tensor([[AMPLITUDES[b % len(AMPLITUDES)] / 0.3 if b % 3 else 1.0] for b in range(64)], device=dev)
    _check_path(eng, sd, geo, wav, path, log_floor, f"{path} {geo} B=64")
    _report()


@gpu
@pytest.mark.parametrize("path", ["tc", "fused"])
@pytest.mark.parametrize("geo", ["v2", "v3"])
def test_logmel_nan_sample(engines, dev, log_floor, path, geo):
    """One NaN sample: the frames the reference lets it reach are NaN (every mel: neither bank has an empty filter, see
    test_mel_log_filterbanks_have_no_empty_mel), and every other frame is bit-identical to the run with that sample at 0.
    Without centering the last samples of an utterance may lie in no frame: then nothing changes at all."""
    eng, sd = engines[geo]
    reached = 0
    for n in (LENGTHS[geo][0], LENGTHS[geo][-1]):
        for pos in (0, n // 2, n - 1):
            wav = _signal("noise", 3, n, pos, dev)
            clean = wav.clone()
            clean[1, pos] = 0.0
            wav[1, pos] = NAN
            got = _check_path(eng, sd, geo, wav, path, log_floor, f"{path} {geo} NaN at {pos} n={n}")
            ref = _run(eng, clean, path == "fused")
            nan_frame = torch.isnan(_frames(wav, GEOMETRY[geo]["n_fft"], GEOMETRY[geo]["hop"], GEOMETRY[geo]["center"])).any(-1)
            reached += int(nan_frame.sum())
            assert bool(torch.isnan(got).all(1)[nan_frame].all())
            keep = ~nan_frame[:, None, :].expand_as(got)
            assert torch.equal(got[keep].view(torch.int32), ref[keep].view(torch.int32)), "a frame without the NaN changed"
    assert reached > 0


# ------------------------------------------------------------------------------------------ public level
@gpu
def test_int16_scaled_ndarray_matches_oracle(dev):
    """An int16 array (soundfile / scipy without rescaling) is accepted as is: FeatureExtractor and transcribe see samples
    up to 32767 and must match the oracle -- features within test_logmel_matches_oracle's tolerance, CTC frame labels
    wherever the oracle's top-2 margin clears test_ctc_ids_margin_aware_larger_batch's 0.01."""
    import gigaam_b200 as gigaam
    ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=4)
    model = gigaam.load_model("v2_ctc", fp16_encoder=False, device=dev, checkpoint=ck)
    wav, _ = synthetic.synthetic_audio(1, 3.0, seed=17)
    pcm = np.round(wav[0].numpy() * 32767.0).astype(np.int16)
    x = torch.from_numpy(pcm.astype(np.float32))[None]
    n = torch.tensor([x.shape[1]])
    sd, cfg = ck["state_dict"], ck["cfg"]
    with torch.inference_mode():
        feats, _ = model.preprocessor(x.to(dev), n.to(dev))
        want = orc.log_mel(x, sd, cfg["preprocessor"])
        assert float((feats.cpu() - want).abs().max()) < 5e-3 and float((feats.cpu() - want).abs().mean()) < 1e-4
        enc, enc_len = model.embed_audio(pcm)
        enc_o, len_o = orc.model_forward(x, n, sd, cfg)
        assert torch.equal(enc_len.cpu(), len_o)
        logits = orc.ctc_logits(enc_o, sd)
        top2 = logits.topk(2, dim=-1).values
        safe = (top2[..., 0] - top2[..., 1]) > 0.01
        lab = F.conv1d(enc.cpu(), sd["head.decoder_layers.0.weight"], sd["head.decoder_layers.0.bias"]).argmax(1)
        assert int(safe.sum()) > 0.5 * safe.numel()
        assert torch.equal(lab[safe], logits.argmax(-1)[safe])
        text = model.transcribe(pcm).text
        if bool(safe.all()):
            ids, _ = orc.ctc_greedy(enc_o, len_o, sd)[0]
            assert text == model.decoding.tokenizer.decode(ids)


def test_create_refuses_more_than_64_mels():
    """gam_create refuses n_mels > 64 (the log-mel kernels hold 64 mel rows) with a message naming n_mels, before any
    device work -- so this runs without a GPU.  A conv1d model with feat_in 128 is otherwise a valid configuration.  The
    weights are null pointers behind one layer record: nothing here may be read or launched."""
    lib = _lib.load()
    cfg = _lib.GamConfig(sample_rate=16000, n_mels=128, n_fft=320, win_length=320, hop_length=160, center=0, feat_in=128,
                         n_layers=1, d_model=768, n_heads=16, d_ff=3072, subsampling=1, subs_kernel_size=5, conv_kernel_size=5,
                         conv_norm=1, self_attention=0, pos_emb_max_len=5000, head=1, num_classes=257, max_symbols=10)
    layers = (_lib.GamLayerWeights * 1)()
    w = _lib.GamWeights(layers=C.cast(layers, C.POINTER(_lib.GamLayerWeights)))
    h = C.c_void_p()
    rc = lib.gam_create(C.byref(cfg), C.byref(w), 0, C.byref(h))
    try:
        msg = lib.gam_last_error(h).decode()
        assert rc != 0 and "n_mels" in msg, (rc, msg)
    finally:
        lib.gam_destroy(h)
