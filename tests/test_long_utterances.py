"""Utterances longer than 768 encoder frames (30.7 s), up to the encoder's 5000-row position tables, on a model loaded
with `max_encoded_frames`.

CPU: the oracle pinned to the reference beyond 768 frames (what the GPU parity tests below lean on), a protocol model of
the rotary attention kernel's K / V ring, and the load-time validation of the limit.
GPU: both attention kernels against float64 at T' up to 5000, encoder parity against the oracle at full depth, the
reference's TensorRT envelope (32 x 50 s), the heads and decoders on T' = 5000 activations, SSL embeddings of 120 s,
the refusal past the limit and CUDA-graph replay."""
import random
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, synthetic
from gigaam_b200.engine import Engine, max_encoded_frames_config
from test_attention_protocol_model import Barrier, ProtocolError, _schedule

MAX_T = 5000                  # pos_emb_max_len of every shipped checkpoint
N_MAX = 3_199_519             # samples at 16 kHz that encode to T' = 5000 (3 199 360 ... 3 199 999 all do)
N_OVER = 3_200_000            # the fewest samples that encode to T' = 5001


# ------------------------------------------------------------------------------------------ oracle vs the reference
def _reference_vs_oracle(which, n_layers, secs=None, samples=None):
    """Runs the byte-compiled reference archive and the oracle on the same waveforms in a subprocess (as
    test_oracle_golden.py does) and returns its stdout; asserts equal lengths and encoder outputs on every valid frame."""
    from oracle import ref_loader
    if not ref_loader.ARCHIVE.is_file():
        pytest.skip("oracle/_ref/gigaam_ref.zip not built (oracle/build_ref.py needs /root/reference)")
    lens = samples if samples is not None else [int(s * 16000) for s in secs]
    code = (
        "import sys, torch\n"
        f"sys.path.insert(0, {str(ref_loader.ROOT)!r})\n"
        "from oracle.ref_loader import build_reference, reference_root\n"
        "from oracle import gigaam_oracle as orc\n"
        "from gigaam_b200 import synthetic\n"
        "assert reference_root().endswith('gigaam_ref.zip')\n"
        f"ck = synthetic.synthetic_checkpoint({which!r}, seed=0, n_layers={n_layers})\n"
        "root, dec = build_reference(ck['cfg'], ck['state_dict'])\n"
        f"lens = {lens!r}\n"
        "wav, _ = synthetic.synthetic_audio(len(lens), max(lens) / 16000.0, seed=2024)\n"
        "wav = wav[:, :max(lens)].contiguous()\n"
        "wl = torch.tensor(lens)\n"
        "for b, n in enumerate(lens): wav[b, n:] = 0.0\n"
        "with torch.inference_mode():\n"
        "    mel, ml = root.preprocessor(wav, wl); enc, el = root.encoder(mel, ml)\n"
        "    enc_o, el_o = orc.model_forward(wav, wl, ck['state_dict'], ck['cfg'])\n"
        "assert torch.equal(el.long(), el_o.long()), (el, el_o)\n"
        "valid = torch.arange(enc.shape[2])[None, :] < el[:, None]\n"
        "a, b = enc_o.transpose(1, 2)[valid], enc.transpose(1, 2)[valid]\n"
        "rel = float((a - b).norm() / b.norm())\n"
        "worst = max(float((enc_o[i, :, :int(el[i])] - enc[i, :, :int(el[i])]).norm() / enc[i, :, :int(el[i])].norm()) for i in range(len(lens)))\n"
        "assert rel < 1e-5 and worst < 1e-4, (rel, worst)\n"
        "print('long ok', el.tolist(), rel, worst)\n")
    env = dict(**__import__("os").environ, GIGAAM_REFERENCE_ARCHIVE_ONLY="1")
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=1800)
    assert res.returncode == 0 and "long ok" in res.stdout, (res.stdout[-500:], res.stderr[-2000:])
    return res.stdout


@pytest.mark.parametrize("which", ["v2_ctc", "v1_ctc"])
@pytest.mark.parametrize("case", ["60s", "60s+7s"])
def test_oracle_matches_the_reference_beyond_768_frames(which, case):
    """Rotary (v2) and rel_pos (v1) encoders, two layers: the oracle slices its rotary / relative-position tables like
    the reference's forward (gigaam/encoder.py:312-361) at T' = 1501, alone and in a ragged batch."""
    out = _reference_vs_oracle(which, 2, secs=[60.0] if case == "60s" else [60.0, 7.0])
    assert "[1501" in out


@pytest.mark.parametrize("which", ["v2_ctc", "v1_ctc"])
def test_oracle_matches_the_reference_at_the_5000_frame_ceiling(which):
    """3 199 519 samples encode to T' = 5000, the last frame the reference's 5000-row tables serve (one layer)."""
    out = _reference_vs_oracle(which, 1, samples=[N_MAX])
    assert "[5000]" in out


def test_the_5000_frame_ceiling_in_samples():
    """The oracle's length arithmetic (pinned to the reference above): 19 997 to 19 999 mel frames (hop 160, centred) all
    subsample to 5000 frames, so 3 199 360 ... 3 199 999 samples give T' = 5000 and 3 200 000 is the first count past it."""
    from oracle import gigaam_oracle as orc
    for which in ("v2_ctc", "v1_ctc"):
        cfg = synthetic.synthetic_checkpoint(which, seed=0, n_layers=1)["cfg"]
        pre, enc = cfg["preprocessor"], cfg["encoder"]
        sr = pre["sample_rate"]
        n = torch.tensor([3_199_359, 3_199_360, N_MAX, N_MAX + 1, N_OVER - 1, N_OVER])
        mel = orc.logmel_out_len(n, pre.get("hop_length", sr // 100), pre.get("win_length", sr // 40), pre.get("center", True))
        t = orc.sub_out_len(mel, enc["subs_kernel_size"], 2)
        assert t.tolist() == [MAX_T - 1, MAX_T, MAX_T, MAX_T, MAX_T, MAX_T + 1], which


# ------------------------------------------------------------------------------------------ protocol model of the rotary ring
class RotaryRing:
    """attention_kernel (gigaam_b200/csrc/attention_sm90.cu): thread 0 issues key blocks 0 .. min(nk, 6) - 1 into stages
    0 .. 5, every warp waits kv_full[kb % 6] for its completion kb / 6, reads K (S = QK^T) and then V (P.V) of the stage,
    and block kb + 6 is issued into the same stage only after a __syncthreads that follows every warp's reads of block kb.
    A partial last block is zeroed between two __syncthreads; its stage is never refilled."""

    S = 6

    def __init__(self, nk, partial, nwarps, rng, refill_sync=True):
        self.nk, self.partial, self.nwarps, self.rng, self.refill_sync = nk, partial, nwarps, rng, refill_sync
        ns = min(nk, self.S)
        self.kv_full = [Barrier(f"kv_full[{s}]", 1) for s in range(ns)]
        self.stage = [None] * ns
        self.readers = [0] * ns
        self.zeroed = [False] * ns
        self.tma = []
        self.sync_gen, self.sync_arrived = 0, 0
        self.blocks_read = [[] for _ in range(nwarps)]

    def syncthreads(self):
        gen = self.sync_gen
        self.sync_arrived += 1
        if self.sync_arrived == self.nwarps:
            self.sync_gen, self.sync_arrived = self.sync_gen + 1, 0
        yield lambda: self.sync_gen > gen

    def issue_block(self, kb):
        st = kb % self.S
        if self.readers[st]:
            raise ProtocolError(f"block {kb} issued into stage {st} while {self.readers[st]} warp(s) read block {self.stage[st]}")
        if self.zeroed[st]:
            raise ProtocolError(f"block {kb} issued into stage {st}, which holds the zeroed last block")
        self.stage[st] = "loading"

        def landed(st=st, kb=kb):
            self.stage[st] = kb
            self.kv_full[st].arrive("tma")
        self.tma.append(landed)

    def _check(self, w, st, kb, what):
        if self.stage[st] != kb:
            raise ProtocolError(f"warp {w} {what}: stage {st} holds {self.stage[st]}, wanted block {kb}")

    def warp(self, w):
        if w == 0:
            for kb in range(min(self.nk, self.S)):
                self.issue_block(kb)
        yield from self.syncthreads()
        for kb in range(self.nk):
            st = kb % self.S
            yield lambda st=st, j=kb // self.S: self.kv_full[st].ready(j)        # mbar_wait(kv_full[kb % 6], (kb / 6) & 1)
            self._check(w, st, kb, "after the wait")
            if self.partial and kb == self.nk - 1:                                  # V rows past klen -> 0
                yield from self.syncthreads()
                if self.readers[st]:
                    raise ProtocolError("V tail zeroed while the stage is read")
                self._check(w, st, kb, "zeroing the V tail")
                self.zeroed[st] = True
                yield from self.syncthreads()
            self.readers[st] += 1
            yield lambda: True                                                      # K reads of S = QK^T
            self._check(w, st, kb, "reading K")
            yield lambda: True                                                      # V reads of P.V
            self._check(w, st, kb, "reading V")
            self.readers[st] -= 1
            self.blocks_read[w].append(kb)
            if kb + self.S < self.nk:
                if self.refill_sync:
                    yield from self.syncthreads()
                if w == 0:
                    self.issue_block(kb + self.S)

    def run(self):
        _schedule(self.rng, {f"warp{w}": self.warp(w) for w in range(self.nwarps)}, {"tma": (self.tma, False)})
        if self.blocks_read != [list(range(self.nk))] * self.nwarps:
            raise ProtocolError(f"blocks read: {self.blocks_read}")


@pytest.mark.parametrize("partial", [True, False])
@pytest.mark.parametrize("nk_range", [(1, 7), (7, 14), (14, 27), (27, 41)])
def test_rotary_kv_ring_has_no_deadlock_aliasing_or_hazard(nk_range, partial):
    """8 warps, 1 to 40 key blocks (T' up to 5120): no deadlock, no parity aliasing (a stage completes up to seven times),
    and every read sees the block it expects."""
    rng = random.Random(1000 * nk_range[0] + partial)
    for nk in range(*nk_range):
        for _ in range(12):
            RotaryRing(nk, partial, nwarps=8, rng=rng).run()


def test_the_model_catches_a_rotary_refill_without_syncthreads():
    """Sanity of the checker: issuing block kb + 6 without the __syncthreads lets the refill overwrite a stage that another
    warp still reads (or hands a warp the wrong block)."""
    rng = random.Random(17)
    with pytest.raises(ProtocolError):
        for _ in range(200):
            RotaryRing(14, False, 8, rng, refill_sync=False).run()


# ------------------------------------------------------------------------------------------ load-time validation
@pytest.mark.parametrize("bad", [5001, 100, 767])
def test_load_model_refuses_a_limit_outside_the_tables(bad):
    ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1)
    with pytest.raises(ValueError, match="max_encoded_frames"):
        gigaam.load_model("v2_ctc", device="cpu", checkpoint=ck, max_encoded_frames=bad)


def test_default_limit_leaves_the_config_field_zero():
    ck = synthetic.synthetic_checkpoint("v1_ctc", seed=0, n_layers=1)
    model = gigaam.load_model("v1_ctc", device="cpu", checkpoint=ck)
    assert model.__dict__["_max_encoded_frames"] is None
    assert max_encoded_frames_config(None, 5000) == 0
    assert _lib.GamConfig().max_encoded_frames == 0
    assert _lib.GamConfig._fields_[-1][0] == "max_encoded_frames"
    model = gigaam.load_model("v1_ctc", device="cpu", checkpoint=ck, max_encoded_frames=MAX_T)
    assert model.__dict__["_max_encoded_frames"] == MAX_T
    model = model.float()                                     # survives the engine invalidation of .to() / _apply
    assert model.__dict__["_max_encoded_frames"] == MAX_T
    assert max_encoded_frames_config(MAX_T, 5000) == MAX_T and max_encoded_frames_config(768, 5000) == 768


# ============================================================================================ GPU
ENC_REL_TOL = 1e-3


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (there is no CPU fallback to test instead)"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def eng_rot(dev):
    ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1)
    return Engine(ck["cfg"], ck["state_dict"], dev, max_encoded_frames=MAX_T)


@pytest.fixture(scope="module")
def eng_rel(dev):
    ck = synthetic.synthetic_checkpoint("v1_ctc", seed=0, n_layers=1)
    return Engine(ck["cfg"], ck["state_dict"], dev, max_encoded_frames=MAX_T)


def _stream():
    import ctypes as C
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


_ATT_CASES = [(2, 769, [769, 1]), (3, 896, [896, 0, 700]), (2, 1537, [1537, 768]), (1, 5000, None), (2, 5000, [4999, 1153])]


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,lens", _ATT_CASES)
def test_rotary_attention_beyond_768_matches_float64_softmax(eng_rot, dev, B, T, lens):
    """The K / V ring (key block kb in stage kb % 6, refilled after every warp's P.V) at 7 to 40 key blocks, with ragged
    lengths inside a T > 768 batch: 0, 1, <= 768, T - 1 and T."""
    g = torch.Generator().manual_seed(B * 1000 + T)
    d, H, dk = 768, 16, 48
    qkv = torch.randn(B * T, 3 * d, generator=g).half().to(dev)
    out = torch.zeros(B * T, d, dtype=torch.float16, device=dev)
    klen = torch.tensor(lens, dtype=torch.int32, device=dev) if lens else None
    rc = eng_rot.lib.gam_test_attention(eng_rot.handle, qkv.data_ptr(), klen.data_ptr() if lens else None, out.data_ptr(), B, T,
                                        _stream())
    torch.cuda.synchronize()
    assert rc == 0, eng_rot.lib.gam_last_error(eng_rot.handle)
    assert torch.isfinite(out).all()
    x = qkv.double().view(B, T, 3, H, dk)
    for b in range(B):
        q, k, v = (x[b, :, i].transpose(0, 1) for i in range(3))
        n = lens[b] if lens else T
        got = out.view(B, T, d)[b].float()
        if n == 0:
            assert float(got.abs().max()) == 0.0          # no valid key -> zeros
            continue
        sc = q @ k[:, :n].transpose(-1, -2) / dk ** 0.5
        want = (torch.softmax(sc, -1) @ v[:, :n]).transpose(0, 1).reshape(T, d)
        assert rel(got, want) < 1e-3, (b, n)


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,lens", [(1, 1537, None), (2, 2000, [2000, 1300]), (1, 5000, None)])
def test_rotary_attention_peaked_rows_beyond_768(eng_rot, dev, B, T, lens):
    """Score rows whose spread grows along the key axis (the inputs of test_attention_peaked_rows_move_the_softmax_reference)
    move the lazy softmax reference again and again after the first wrap of the ring, i.e. at key blocks read from refilled
    stages.  The number of moves grows with the score range, not with the block count, so it is counted past block 6."""
    g = torch.Generator().manual_seed(B * 77 + T)
    d, H, dk = 768, 16, 48
    x = torch.randn(B, T, 3, H, dk, generator=g)
    x[:, :, 0] *= 6.0
    x[:, :, 1] *= (0.1 + 2.4 * torch.arange(T) / T)[None, :, None, None]
    qkv = x.reshape(B * T, 3 * d).half().to(dev)
    out = torch.zeros(B * T, d, dtype=torch.float16, device=dev)
    klen = torch.tensor(lens, dtype=torch.int32, device=dev) if lens else None
    rc = eng_rot.lib.gam_test_attention(eng_rot.handle, qkv.data_ptr(), klen.data_ptr() if lens else None, out.data_ptr(), B, T,
                                        _stream())
    torch.cuda.synchronize()
    assert rc == 0
    assert torch.isfinite(out).all()
    xf = qkv.double().view(B, T, 3, H, dk)
    nblk = (T + 127) // 128
    for b in range(B):
        n = lens[b] if lens else T
        q, k, v = (xf[b, :, i].transpose(0, 1) for i in range(3))
        sc = q @ k[:, :n].transpose(-1, -2) / dk ** 0.5
        l2 = sc * 1.4426950408889634
        nb = (n + 127) // 128
        bmax = F.pad(l2, (0, nb * 128 - n), value=float("-inf")).view(H, T, nb, 128).amax(-1)
        mc, moves, late = bmax[..., 0].clone(), torch.zeros_like(bmax[..., 0]), torch.zeros_like(bmax[..., 0])
        for j in range(1, nb):
            move = bmax[..., j] > mc + 8.0
            moves += move
            late += move * (j >= 6)
            mc = torch.where(move, bmax[..., j], mc)
        print(f"softmax reference moves per row: {float(moves.mean()):.2f} over {nb} of {nblk} key blocks, "
              f"{float(late.mean()):.2f} of them past block 6")
        # measured: 2.08 / 2.80 / 1.30 / 4.76 late moves per row, at least 93 % of the rows moving, for the four utterances
        assert float(late.mean()) >= 1.0 and float((late > 0).double().mean()) > 0.9
        want = (torch.softmax(sc, -1) @ v[:, :n]).transpose(0, 1).reshape(T, d)
        assert rel(out.view(B, T, d)[b].float(), want) < 2e-3, b


def _relpos_want(xb, pos, L, n, H, dk):
    """float64 reference formula (gigaam/encoder.py:216-228) with the reference's pad/view rel_shift, n valid frames."""
    qu, qv, k, v = (xb[:, i].transpose(0, 1) for i in range(4))
    T = xb.shape[0]
    p = pos.double()[L - T: L + T - 1].view(2 * T - 1, H, dk).transpose(0, 1)           # positions T-1 ... -(T-1)
    bd = qv @ p.transpose(-1, -2)
    bd = F.pad(bd, (1, 0)).view(H, -1, T)[:, 1:].reshape(H, T, 2 * T - 1)[..., :T]      # rel_shift, encoder.py:202-206
    sc = (qu @ k.transpose(-1, -2) + bd) / dk ** 0.5
    sc[..., n:] = float("-inf")
    return (torch.softmax(sc, -1) @ v).transpose(0, 1).reshape(T, -1)


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,lens", _ATT_CASES)
def test_relpos_attention_beyond_768_matches_float64_softmax(eng_rel, dev, B, T, lens):
    """A 2 * 5000 - 1 row position table; T' = 5000 exactly puts the last query tile's window start below row 0 (5000 is
    not a multiple of 128), where TMA zero-fills rows that only meet queries >= T."""
    g = torch.Generator().manual_seed(B * 1000 + T + 7)
    d, H, dk, L = 768, 16, 48, MAX_T
    qkv = torch.randn(B * T, 4 * d, generator=g).half().to(dev)
    pos = torch.randn(2 * L - 1, d, generator=g).half().to(dev)
    out = torch.zeros(B * T, d, dtype=torch.float16, device=dev)
    klen = torch.tensor(lens, dtype=torch.int32, device=dev) if lens else None
    rc = eng_rel.lib.gam_test_attention_relpos(eng_rel.handle, qkv.data_ptr(), pos.data_ptr(), klen.data_ptr() if lens else None,
                                               out.data_ptr(), B, T, _stream())
    torch.cuda.synchronize()
    assert rc == 0, eng_rel.lib.gam_last_error(eng_rel.handle)
    assert torch.isfinite(out).all()
    x = qkv.double().view(B, T, 4, H, dk)
    for b in range(B):
        n = lens[b] if lens else T
        got = out.view(B, T, d)[b].float()
        if n == 0:
            assert float(got.abs().max()) == 0.0
            continue
        want = _relpos_want(x[b], pos, L, n, H, dk)
        assert rel(got, want) < 1e-3, (b, n)


@pytest.mark.gpu
@pytest.mark.parametrize("relpos", [False, True])
@pytest.mark.parametrize("T,lens", [(5000, [5000, 1, 769, 0, 4097]), (1537, [300, 1537, 768, 1300])])
def test_attention_varlen_beyond_768(request, dev, relpos, T, lens):
    """Packed rows (the path gam_encode takes) past 768 frames; the rows behind each utterance -- the next utterance's, and
    NaN behind the last one -- must not leak in, and nothing is stored behind the stream."""
    eng = request.getfixturevalue("eng_rel" if relpos else "eng_rot")
    B, d, H, dk, L = len(lens), 768, 16, 48, MAX_T
    parts = 4 if relpos else 3
    g = torch.Generator().manual_seed(T + 17 * B + relpos)
    rows = sum(lens)
    qkv = torch.full((rows + 300, parts * d), float("nan"), dtype=torch.float16)
    qkv[:rows] = torch.randn(rows, parts * d, generator=g).half()
    qkv = qkv.to(dev)
    pos = torch.randn(2 * L - 1, d, generator=g).half().to(dev)
    out = torch.full((rows + 300, d), 7.0, dtype=torch.float16, device=dev)
    klen = torch.tensor(lens, dtype=torch.int32, device=dev)
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    cu_d = torch.tensor(cu, dtype=torch.int32, device=dev)
    rc = eng.lib.gam_test_attention_varlen(eng.handle, qkv.data_ptr(), pos.data_ptr() if relpos else None, klen.data_ptr(),
                                           cu_d.data_ptr(), out.data_ptr(), B, T, rows + 300, _stream())
    torch.cuda.synchronize()
    assert rc == 0, eng.lib.gam_last_error(eng.handle)
    assert torch.isfinite(out).all()
    assert bool((out[rows:] == 7.0).all())
    for b, n in enumerate(lens):
        if n == 0:
            continue
        xb = qkv[cu[b]: cu[b] + n].double().view(n, parts, H, dk)
        if relpos:
            want = _relpos_want(xb, pos, L, n, H, dk)
        else:
            q, k, v = (xb[:, i].transpose(0, 1) for i in range(3))
            want = (torch.softmax(q @ k.transpose(-1, -2) / dk ** 0.5, -1) @ v).transpose(0, 1).reshape(n, d)
        assert rel(out[cu[b]: cu[b] + n].float(), want) < 1e-3, (b, n)


@pytest.mark.gpu
def test_test_entry_points_refuse_past_the_handle_limit(eng_rot, eng_rel, dev):
    out = torch.zeros(1, dtype=torch.float16, device=dev)
    assert eng_rot.lib.gam_test_attention(eng_rot.handle, out.data_ptr(), None, out.data_ptr(), 1, MAX_T + 1, _stream()) != 0
    assert b"limit" in eng_rot.lib.gam_last_error(eng_rot.handle)
    assert eng_rel.lib.gam_test_attention_relpos(eng_rel.handle, out.data_ptr(), out.data_ptr(), None, out.data_ptr(), 1, MAX_T + 1,
                                                 _stream()) != 0
    assert b"limit" in eng_rel.lib.gam_last_error(eng_rel.handle)


# ------------------------------------------------------------------------------------------ the encoder end to end
def _encoder_parity(model, ckpt, wav, wav_len, dev):
    """The criteria of test_gpu_parity._encoder_parity: the benchmarked fp16 mode against the oracle on fp16-rounded encoder
    parameters, relative error <= 1e-3 over all valid frames and <= 1.5e-3 for the worst utterance."""
    from oracle import gigaam_oracle as orc
    sd16 = {k: (v.half().float() if k.startswith("encoder.") and v.is_floating_point() else v) for k, v in ckpt["state_dict"].items()}
    enc, enc_len = model(wav.to(dev), wav_len.to(dev))
    with torch.inference_mode():
        enc_o, len_o = orc.model_forward(wav, wav_len, sd16, ckpt["cfg"])
    assert torch.equal(enc_len.cpu(), len_o)
    assert torch.isfinite(enc).all()
    got, want = enc.cpu().transpose(1, 2), enc_o.transpose(1, 2)
    valid = torch.arange(want.shape[1])[None, :] < len_o[:, None]
    r_all = rel(got[valid], want[valid])
    r_utt = max(rel(got[i, : int(len_o[i])], want[i, : int(len_o[i])]) for i in range(wav.shape[0]))
    print(f"encoder rel: all {r_all:.3e}, worst utterance {r_utt:.3e}")
    assert r_all < ENC_REL_TOL and r_utt < 1.5 * ENC_REL_TOL
    return enc, enc_len, enc_o, len_o, sd16


_CKPTS = {}


def _ckpt(which):
    if which not in _CKPTS:
        _CKPTS[which] = synthetic.synthetic_checkpoint(which, seed=0)
    return _CKPTS[which]


def _ragged(secs, seed):
    lens = [int(s * 16000) for s in secs]
    wav, _ = synthetic.synthetic_audio(len(lens), max(lens) / 16000.0, seed=seed)
    wav = wav[:, : max(lens)].contiguous()
    for b, n in enumerate(lens):
        wav[b, n:] = 0.0
    return wav, torch.tensor(lens)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["v2_ctc", "v3_e2e_rnnt", "v1_ctc"])
def test_encoder_parity_on_a_ragged_60s_pair(dev, which):
    ck = _ckpt(which)
    model = gigaam.load_model(which, device=dev, checkpoint=ck, max_encoded_frames=MAX_T)
    wav, wav_len = _ragged([60.0, 12.0], seed=61)
    enc, enc_len, _, _, _ = _encoder_parity(model, ck, wav, wav_len, dev)
    assert enc.shape[2] >= 1500


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["v2_ctc", "v1_ctc"])
def test_encoder_parity_at_5000_frames_and_refusal_at_5001(dev, which):
    ck = _ckpt(which)
    model = gigaam.load_model(which, device=dev, checkpoint=ck, max_encoded_frames=MAX_T)
    assert model._get_engine().gam_config.max_encoded_frames == MAX_T
    wav, wav_len = _ragged([N_MAX / 16000.0], seed=50)
    assert int(wav_len[0]) == N_MAX
    enc, enc_len, _, _, _ = _encoder_parity(model, ck, wav, wav_len, dev)
    assert enc.shape[2] == MAX_T and int(enc_len[0]) == MAX_T
    with pytest.raises(Exception, match="T'=5001 exceeds the attention kernels' 5000-frame limit"):
        model(torch.zeros(1, N_OVER, device=dev), torch.tensor([N_OVER], device=dev))


@pytest.mark.gpu
def test_default_model_keeps_the_768_frame_limit(dev):
    ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1)
    model = gigaam.load_model("v2_ctc", device=dev, checkpoint=ck)
    eng = model._get_engine()
    assert eng.gam_config.max_encoded_frames == 0 and eng.max_encoded_frames == 768
    with pytest.raises(Exception, match=r"T'=\d+ exceeds the attention kernels' 768-frame limit"):
        model(torch.zeros(1, 31 * 16000, device=dev), torch.tensor([31 * 16000], device=dev))


@pytest.mark.gpu
def test_tensorrt_envelope_32_utterances_up_to_50s(dev):
    """The reference's serving profile (32 x 64 x 5000 mel frames, triton_scripts/run_convert_trt.sh): 32 ragged
    utterances up to 50 s (T' = 1251) through model(wav, len) + decoding.decode.  Each utterance's valid frames are
    bit-identical to the same utterance encoded in a batch of 4 over the same buffer: every kernel of the path computes
    a frame from its own utterance's rows in an order that does not depend on the batch (row-wise GEMM tiles with a fixed
    K order, per-utterance attention tiles and depthwise windows, per-row LayerNorm)."""
    ck = _ckpt("v2_ctc")
    model = gigaam.load_model("v2_ctc", device=dev, checkpoint=ck, max_encoded_frames=MAX_T)
    rng = random.Random(32)
    secs = [50.0] + [round(rng.uniform(0.5, 50.0), 2) for _ in range(31)]
    wav, wav_len = _ragged(secs, seed=320)
    enc, enc_len = model(wav.to(dev), wav_len.to(dev))
    hyps = model.decoding.decode(model.head, enc, enc_len)
    assert enc.shape[2] == 1251 and torch.isfinite(enc).all() and len(hyps) == 32
    exact = 0
    for g0 in range(0, 32, 4):
        e4, l4 = model(wav[g0: g0 + 4].to(dev), wav_len[g0: g0 + 4].to(dev))
        assert torch.equal(l4, enc_len[g0: g0 + 4])
        for i in range(4):
            n = int(l4[i])
            exact += int(torch.equal(e4[i, :, :n], enc[g0 + i, :, :n]))
    print(f"{exact} of 32 utterances bit-identical to their batch-of-4 run")
    assert exact == 32
    _encoder_parity(model, ck, wav[:4], wav_len[:4], dev)


@pytest.mark.gpu
def test_heads_and_decoders_on_5000_frame_activations(dev):
    """Identical fp32 activations at T' = 5000 on both sides: CTC and RNN-T greedy hypotheses bit-exact with the oracle's,
    CTC log-probs of model.head within the 1e-4 of test_head_forward.py."""
    from oracle import gigaam_oracle as orc
    ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1)
    model = gigaam.load_model("v2_ctc", fp16_encoder=False, device=dev, checkpoint=ck, max_encoded_frames=MAX_T)
    sd = ck["state_dict"]
    g = torch.Generator().manual_seed(5000)
    enc = torch.randn(2, MAX_T, 768, generator=g)
    enc_len = torch.tensor([MAX_T, 3001], dtype=torch.int32)
    enc[1, 3001:] = 0
    eng = model._get_engine()
    ids, frames, counts = eng.greedy(enc.to(dev), enc_len.to(dev))
    want = orc.ctc_greedy(enc.transpose(1, 2), enc_len, sd)
    for b in range(2):
        n = int(counts[b])
        assert n > 0 and ids[b, :n].tolist() == want[b][0] and frames[b, :n].tolist() == want[b][1], b
    with torch.inference_mode():
        lp = model.head(enc.to(dev).transpose(1, 2)).cpu()
    want_lp = torch.log_softmax(orc.ctc_logits(enc.transpose(1, 2), sd), dim=-1)
    valid = torch.arange(MAX_T)[None, :] < enc_len[:, None]
    assert float((lp[valid] - want_lp[valid]).abs().max()) <= 1e-4

    ck = synthetic.synthetic_checkpoint("v2_rnnt", seed=0, n_layers=1)
    model = gigaam.load_model("v2_rnnt", fp16_encoder=False, device=dev, checkpoint=ck, max_encoded_frames=MAX_T)
    mean = torch.as_tensor(synthetic._rnnt_calibration("v2_rnnt")["enc_mean"])
    enc = mean + torch.randn(1, MAX_T, 768, generator=g) * 0.3
    enc_len = torch.tensor([MAX_T], dtype=torch.int32)
    ids, frames, counts = model._get_engine().greedy(enc.to(dev).contiguous(), enc_len.to(dev))
    want = orc.rnnt_greedy(enc.transpose(1, 2), enc_len, ck["state_dict"], 10)
    n = int(counts[0])
    assert n > 0 and ids[0, :n].tolist() == want[0][0] and frames[0, :n].tolist() == want[0][1]


@pytest.mark.gpu
def test_ssl_embeddings_of_a_120s_recording(dev):
    ck = synthetic.synthetic_checkpoint("v2_ssl", seed=0)
    model = gigaam.load_model("v2_ssl", device=dev, checkpoint=ck, max_encoded_frames=MAX_T)
    wav, wav_len = synthetic.synthetic_audio(1, 120.0, seed=120)
    enc, enc_len = model.embed_audio(wav[0])
    assert enc.shape == (1, 768, 3001) and int(enc_len[0]) == 3001
    _, _, enc_o, _, _ = _encoder_parity(model, ck, wav, wav_len, dev)
    assert rel(enc.cpu(), enc_o) < ENC_REL_TOL


@pytest.mark.gpu
def test_cuda_graph_of_a_120s_step_replays_bit_identically(dev):
    """The launch sequence of a step depends only on the host-known padded T' (lengths stay on the device), so a captured
    graph of a 120 s batch replays the eager result exactly, and the limit + 1 is still refused."""
    ck = synthetic.synthetic_checkpoint("v1_ctc", seed=0, n_layers=2)
    model = gigaam.load_model("v1_ctc", device=dev, checkpoint=ck, max_encoded_frames=3001)
    wav, wav_len = _ragged([120.0, 77.0], seed=7)
    wav, wav_len = wav.to(dev), wav_len.to(dev)
    with torch.inference_mode():
        eager, eager_len = model(wav, wav_len)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            model(wav, wav_len)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out, out_len = model(wav, wav_len)
        graph.replay()
        torch.cuda.synchronize()
    assert eager.shape[2] == 3001
    assert torch.equal(out, eager) and torch.equal(out_len, eager_len)
    with pytest.raises(Exception, match=r"T'=\d+ exceeds the attention kernels' 3001-frame limit"):
        model(torch.zeros(1, 1_920_640, device=dev), torch.tensor([1_920_640], device=dev))   # T' = 3002
