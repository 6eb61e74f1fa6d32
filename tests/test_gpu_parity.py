"""Parity tests proper (need an H100): every stage of the CUDA path, called through the C ABI, against the CPU oracle
on the same seeded inputs, against the golden fixtures generated from the real reference, and -- at the full
BASELINE sizes -- through size-independent properties (batch-vs-single consistency, run-to-run determinism).

Tolerances (north_star: encoder activations within 1e-3 relative with fp16 tensor-core operands; CTC token ids
bit-exact): relative Frobenius error on valid frames <= 1e-3 for the encoder, exact ids wherever the oracle's
top-2 logit margin exceeds the fp16 operand noise (and exact, unconditionally, when the head is fed identical
activations)."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import gigaam_b200 as gigaam  # noqa: E402
from gigaam_b200 import synthetic  # noqa: E402
from gigaam_b200.engine import Engine  # noqa: E402
from oracle import gigaam_oracle as orc  # noqa: E402

ENC_REL_TOL = 1e-3


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.fixture(scope="session")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (there is no CPU fallback to test instead)"
    return torch.device("cuda", 0)


@pytest.fixture(scope="session")
def eng_ctc(dev, v2_ctc_ckpt):
    return Engine(v2_ctc_ckpt["cfg"], v2_ctc_ckpt["state_dict"], dev)


@pytest.fixture(scope="session")
def eng_rnnt(dev, v2_rnnt_ckpt):
    return Engine(v2_rnnt_ckpt["cfg"], v2_rnnt_ckpt["state_dict"], dev)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------ kernels in isolation
# (the GEMM, row, subsampling and packing kernels have float64 unit tests of their own in test_kernel_units.py)
@pytest.mark.parametrize("B,T,lens", [(1, 128, None), (2, 51, [51, 30]), (3, 251, [251, 200, 97]), (2, 376, [376, 129]),
                                      (1, 626, None), (2, 5, [5, 1]), (2, 129, [129, 128]), (2, 751, [751, 640]), (1, 768, None)])
def test_attention_matches_masked_softmax(eng_ctc, dev, B, T, lens):
    g = torch.Generator().manual_seed(B * 1000 + T)
    d, H, dk = 768, 16, 48
    qkv = torch.randn(B * T, 3 * d, generator=g).half().to(dev)
    out = torch.zeros(B * T, d, dtype=torch.float16, device=dev)
    klen = torch.tensor(lens, dtype=torch.int32, device=dev) if lens else None
    rc = eng_ctc.lib.gam_test_attention(eng_ctc.handle, qkv.data_ptr(), klen.data_ptr() if lens else None, out.data_ptr(), B, T, _stream())
    torch.cuda.synchronize()
    assert rc == 0
    x = qkv.float().view(B, T, 3, H, dk)
    q, k, v = (x[:, :, i].transpose(1, 2) for i in range(3))
    sc = q @ k.transpose(-1, -2) / dk ** 0.5
    if lens:
        valid = torch.arange(T, device=dev)[None, :] < klen[:, None]
        sc = sc.masked_fill(~valid[:, None, None, :], float("-inf"))
    want = (torch.softmax(sc, -1) @ v).transpose(1, 2).reshape(B * T, d)
    assert torch.isfinite(out).all()
    assert rel(out.float(), want) < 1e-3


@pytest.mark.parametrize("B,T,lens", [(2, 251, [251, 140]), (2, 626, [626, 417]), (1, 128, None), (1, 768, None),
                                      (3, 512, [512, 385, 300])])
def test_attention_peaked_rows_move_the_softmax_reference(eng_ctc, dev, B, T, lens):
    """attention_sm90.cu takes the exact maximum of a row's first 128-key block as its softmax reference point and moves it
    at a later block only when that block's maximum exceeds it by more than 2^8; a move rescales O and the row sum.  Score
    rows whose spread grows along the key axis (key norms ramp up, queries are scaled) move the reference at block after
    block, so every multi-block shape here exercises that rescaling -- repeatedly at 4 to 6 blocks.  The single-block shape
    checks the same peaked rows where the first block's exact maximum is the only reference."""
    g = torch.Generator().manual_seed(B * 77 + T)
    d, H, dk = 768, 16, 48
    x = torch.randn(B, T, 3, H, dk, generator=g)
    x[:, :, 0] *= 6.0                                                      # queries: scores ~ N(0, 6^2 * |k|^2 / 48)
    x[:, :, 1] *= (0.1 + 2.4 * torch.arange(T) / T)[None, :, None, None]   # key norms ramp up along the sequence
    qkv = x.reshape(B * T, 3 * d).half().to(dev)
    out = torch.zeros(B * T, d, dtype=torch.float16, device=dev)
    klen = torch.tensor(lens, dtype=torch.int32, device=dev) if lens else None
    rc = eng_ctc.lib.gam_test_attention(eng_ctc.handle, qkv.data_ptr(), klen.data_ptr() if lens else None, out.data_ptr(), B, T, _stream())
    torch.cuda.synchronize()
    assert rc == 0
    xf = qkv.float().view(B, T, 3, H, dk)
    q, k, v = (xf[:, :, i].transpose(1, 2) for i in range(3))
    sc = q @ k.transpose(-1, -2) / dk ** 0.5
    if lens:
        valid = torch.arange(T, device=dev)[None, :] < klen[:, None]
        sc = sc.masked_fill(~valid[:, None, None, :], float("-inf"))
    # the test must do what it says: per row, replay the kernel's rule over the valid keys and count the moves
    l2 = sc * 1.4426950408889634
    nblk = (T + 127) // 128
    bmax = F.pad(l2, (0, nblk * 128 - T), value=float("-inf")).view(B, H, T, nblk, 128).amax(-1)
    mc, moves = bmax[..., 0].clone(), torch.zeros_like(bmax[..., 0])
    for j in range(1, nblk):
        move = bmax[..., j] > mc + 8.0
        moves += move
        mc = torch.where(move, bmax[..., j], mc)
    rows = torch.arange(T, device=dev)[None, None, :] < (klen[:, None, None] if lens else T)
    mean_moves = float(moves[rows.expand_as(moves)].mean())
    print(f"softmax reference moves per row: {mean_moves:.2f} over {nblk} key blocks")
    assert mean_moves >= 0.5 * (nblk - 1) and (nblk > 1 or mean_moves == 0.0)
    want = (torch.softmax(sc, -1) @ v).transpose(1, 2).reshape(B * T, d)
    assert torch.isfinite(out).all()
    assert rel(out.float(), want) < 2e-3


@pytest.mark.parametrize("B,sec,ragged", [(2, 2.0, True), (3, 10.0, False), (1, 0.5, False), (1, 0.2, False), (1, 0.3125, False)])
def test_logmel_matches_oracle(eng_ctc, v2_ctc_ckpt, B, sec, ragged):
    wav, _ = synthetic.synthetic_audio(B, sec, seed=11, ragged=ragged)
    want = orc.log_mel(wav, v2_ctc_ckpt["state_dict"], v2_ctc_ckpt["cfg"]["preprocessor"])
    got = eng_ctc.logmel(wav.cuda()).cpu()
    assert got.shape == want.shape
    # fp32 DFT vs pocketfft: power-spectrum rounding is amplified by log near the 1e-9 clamp only
    assert float((got - want).abs().max()) < 5e-3
    assert float((got - want).abs().mean()) < 1e-4


def test_logmel_fused_cuda_core_kernel_still_matches(eng_ctc, v2_ctc_ckpt):
    """The single fused kernel (gam_logmel) and the tensor-core split-precision path (gam_logmel_tc) agree."""
    wav, _ = synthetic.synthetic_audio(2, 3.0, seed=13, ragged=True)
    want = orc.log_mel(wav, v2_ctc_ckpt["state_dict"], v2_ctc_ckpt["cfg"]["preprocessor"])
    tc = eng_ctc.logmel(wav.cuda()).cpu()
    fused = eng_ctc.logmel(wav.cuda(), fused=True).cpu()
    for got in (tc, fused):
        assert float((got - want).abs().max()) < 5e-3 and float((got - want).abs().mean()) < 1e-4
    assert float((tc - fused).abs().max()) < 5e-3


# ------------------------------------------------------------------------------------------ encoder
@pytest.fixture(scope="session")
def golden_ctc(golden_dir):
    return np.load(golden_dir / "v2_ctc_b2_2s.npz")


def test_encoder_stagewise_against_oracle(eng_ctc, v2_ctc_ckpt, golden_ctc):
    g = golden_ctc
    cfg, sd = v2_ctc_ckpt["cfg"], v2_ctc_ckpt["state_dict"]
    mel, mel_len = torch.from_numpy(g["mel"]), torch.from_numpy(g["mel_len"])
    with torch.inference_mode():
        _, len_o, stages = orc.encoder_forward(mel, mel_len, sd, cfg["encoder"], return_all=True)
    valid = torch.arange(stages[0].shape[1])[None, :] < len_o[:, None]
    for n in (0, 1, 2, 8, 16):
        enc, enc_len = eng_ctc.encode(mel.cuda(), mel_len.cuda(), n_layers_run=n)
        assert torch.equal(enc_len.cpu(), len_o)
        assert torch.isfinite(enc).all()
        assert rel(enc.cpu()[valid], stages[n][valid]) < ENC_REL_TOL, f"after {n} layers"


def test_end_to_end_against_reference_golden(eng_ctc, golden_ctc):
    """wav -> ids through the CUDA path vs outputs of the REAL reference (tests/golden, oracle/make_golden.py)."""
    g = golden_ctc
    wav, wav_len = synthetic.synthetic_audio(2, 2.0, seed=1234, ragged=True)
    mel = eng_ctc.logmel(wav.cuda())
    assert float((mel.cpu() - torch.from_numpy(g["mel"])).abs().max()) < 5e-3
    enc, enc_len = eng_ctc.encode(mel, torch.from_numpy(g["mel_len"]).cuda())
    assert np.array_equal(enc_len.cpu().numpy(), g["enc_len"])
    want = torch.from_numpy(g["enc"]).transpose(1, 2)
    valid = torch.arange(want.shape[1])[None, :] < torch.from_numpy(g["enc_len"])[:, None]
    assert rel(enc.cpu()[valid], want[valid]) < ENC_REL_TOL
    ids, frames, counts = eng_ctc.greedy(enc, enc_len)
    for b in range(2):
        n = int(counts[b])
        # golden margins are >= 3.6e-3 on every valid frame, far above the ~1e-4 logit noise -> ids must be bit-exact
        assert ids[b, :n].tolist() == g[f"ids_{b}"].tolist()
        assert frames[b, :n].tolist() == g[f"frames_{b}"].tolist()


def test_ctc_ids_margin_aware_larger_batch(eng_ctc, v2_ctc_ckpt):
    """Bit-exact CTC ids wherever the oracle's top-2 margin exceeds the FIXED margin CTC_MARGIN_EPS (derived from the
    1e-3 activation budget, see the BASELINE-size tests below); sub-margin frames are counted (SURVEY 7 'hard parts')."""
    cfg, sd = v2_ctc_ckpt["cfg"], v2_ctc_ckpt["state_dict"]
    wav, wav_len = synthetic.synthetic_audio(4, 5.0, seed=99, ragged=True)
    with torch.inference_mode():
        enc_o, len_o = orc.model_forward(wav, wav_len, sd, cfg)
        logits = orc.ctc_logits(enc_o, sd)
    mel = eng_ctc.logmel(wav.cuda())
    enc, enc_len = eng_ctc.encode(mel, orc.logmel_out_len(wav_len, 160, 400, True).cuda())
    assert torch.equal(enc_len.cpu(), len_o)
    eng_ctc.greedy(enc, enc_len)
    lab_gpu = (F.conv1d(enc.cpu().transpose(1, 2), sd["head.decoder_layers.0.weight"], sd["head.decoder_layers.0.bias"])).argmax(1)
    top2 = logits.topk(2, dim=-1).values
    margin = top2[..., 0] - top2[..., 1]
    valid = torch.arange(logits.shape[1])[None, :] < len_o[:, None]
    safe = valid & (margin > CTC_MARGIN_EPS)
    print(f"CTC: {int((valid & ~safe).sum())} of {int(valid.sum())} frames below the {CTC_MARGIN_EPS} margin")
    assert torch.equal(lab_gpu[safe], logits.argmax(-1)[safe])
    assert float((valid & ~safe).sum()) / float(valid.sum()) < CTC_SUBMARGIN_MAX


def test_batch_vs_single_consistency(eng_ctc):
    """Property from the reference's tests/test_batching.py:70-83: valid frames of a padded batch equal the
    single-utterance run (atol 0.03 there; much tighter here)."""
    wav, wav_len = synthetic.synthetic_audio(3, 3.0, seed=5, ragged=True)
    mel = eng_ctc.logmel(wav.cuda())
    mel_len = (wav_len // 160 + 1).cuda()
    enc_b, len_b = eng_ctc.encode(mel, mel_len)
    for i in range(3):
        n = int(wav_len[i])
        mel_i = eng_ctc.logmel(wav[i:i + 1, :n].cuda())
        enc_i, len_i = eng_ctc.encode(mel_i, torch.tensor([mel_i.shape[2]]).cuda())
        L = int(len_i[0])
        assert L == int(len_b[i])
        # the batched front end reflects at the *buffer* end, the single run at the utterance end: the last frames
        # of a short utterance legitimately differ (SURVEY 7), so compare away from the tail like the reference
        # test does by running the front end per sample
        mel_fair = mel[i:i + 1, :, : mel_i.shape[2]].contiguous()
        enc_f, _ = eng_ctc.encode(mel_fair, torch.tensor([mel_i.shape[2]]).cuda())
        assert float((enc_f[0, :L] - enc_b[i, :L]).abs().max()) < 0.03
        assert rel(enc_f[0, :L], enc_b[i, :L]) < 2e-3


def test_run_to_run_determinism(eng_ctc):
    wav, wav_len = synthetic.synthetic_audio(4, 4.0, seed=21, ragged=True)
    outs = []
    for _ in range(2):
        mel = eng_ctc.logmel(wav.cuda())
        enc, enc_len = eng_ctc.encode(mel, (wav_len // 160 + 1).cuda())
        ids, frames, counts = eng_ctc.greedy(enc, enc_len)
        outs.append((enc.clone(), ids.clone(), frames.clone(), counts.clone()))
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.equal(outs[0][3], outs[1][3])
    for b in range(4):
        n = int(outs[0][3][b])
        assert torch.equal(outs[0][1][b, :n], outs[1][1][b, :n]) and torch.equal(outs[0][2][b, :n], outs[1][2][b, :n])


def test_max_length_utterance_25s(eng_ctc, v2_ctc_ckpt):
    """T' = 626 (the 25 s limit of transcribe, gigaam/model.py:13,135-136): 5 key blocks in the attention kernel."""
    cfg, sd = v2_ctc_ckpt["cfg"], v2_ctc_ckpt["state_dict"]
    wav, wav_len = synthetic.synthetic_audio(1, 25.0, seed=3)
    with torch.inference_mode():
        enc_o, len_o = orc.model_forward(wav, wav_len, sd, cfg)
    mel = eng_ctc.logmel(wav.cuda())
    enc, enc_len = eng_ctc.encode(mel, torch.tensor([mel.shape[2]]).cuda())
    assert int(enc_len[0]) == 626 == int(len_o[0])
    assert rel(enc.cpu()[0], enc_o.transpose(1, 2)[0]) < ENC_REL_TOL


# ------------------------------------------------------------------------------------------ decoders on identical activations
@pytest.mark.parametrize("B,T,lens", [(2, 51, [51, 30]), (5, 251, [251, 250, 1, 0, 100]), (1, 1, [1])])
def test_ctc_greedy_bit_exact(eng_ctc, v2_ctc_ckpt, B, T, lens):
    g = torch.Generator().manual_seed(T)
    enc = torch.randn(B, T, 768, generator=g)
    enc_len = torch.tensor(lens, dtype=torch.int32)
    want = orc.ctc_greedy(enc.transpose(1, 2), enc_len, v2_ctc_ckpt["state_dict"])
    ids, frames, counts = eng_ctc.greedy(enc.cuda(), enc_len.cuda())
    for b in range(B):
        n = int(counts[b])
        assert ids[b, :n].tolist() == want[b][0] and frames[b, :n].tolist() == want[b][1]


def test_rnnt_greedy_matches_reference_golden(eng_rnnt, golden_dir):
    g = np.load(golden_dir / "v2_rnnt_b2_2s.npz")
    enc = torch.from_numpy(g["enc"]).transpose(1, 2).contiguous()
    ids, frames, counts = eng_rnnt.greedy(enc.cuda(), torch.from_numpy(g["enc_len"]).cuda())
    for b in range(2):
        n = int(counts[b])
        assert n == len(g[f"ids_{b}"]) and n > 0
        assert ids[b, :n].tolist() == g[f"ids_{b}"].tolist()
        assert frames[b, :n].tolist() == g[f"frames_{b}"].tolist()


def test_rnnt_blank_then_emit_patterns(eng_rnnt, v2_rnnt_ckpt):
    """Emissions that follow runs of blank frames consume a prediction-network state computed many steps earlier
    (the synthetic audio never produces this: its encoder output is almost constant in time).  Random, time-varying
    activations give hypotheses whose frame lists have gaps of both parities; ids and frames must still be exact."""
    sd = v2_rnnt_ckpt["state_dict"]
    # the calibrated joint network cancels the mean encoder frame (oracle/calibrate_rnnt.py): frames = that mean + noise
    mean = torch.as_tensor(synthetic._rnnt_calibration("v2_rnnt")["enc_mean"])
    gaps_seen = set()
    for seed, scale in [(8, 0.3), (9, 0.3), (10, 0.25), (11, 0.35)]:
        g = torch.Generator().manual_seed(seed)
        enc = mean + torch.randn(6, 40, 768, generator=g) * scale
        enc_len = torch.tensor([40, 33, 0, 17, 40, 9], dtype=torch.int32)
        want = orc.rnnt_greedy(enc.transpose(1, 2), enc_len, sd, 10)
        ids, frames, counts = eng_rnnt.greedy(enc.cuda(), enc_len.cuda())
        for b in range(6):
            n = int(counts[b])
            assert ids[b, :n].tolist() == want[b][0], (seed, b)
            assert frames[b, :n].tolist() == want[b][1], (seed, b)
            fr = want[b][1]
            gaps_seen |= {(y - x) % 2 for x, y in zip(fr, fr[1:]) if y - x > 1}
    assert gaps_seen == {0, 1}, "the test inputs no longer exercise blank runs of both parities"


def test_rnnt_edge_lengths(eng_rnnt, v2_rnnt_ckpt):
    g = torch.Generator().manual_seed(8)
    enc = torch.as_tensor(synthetic._rnnt_calibration("v2_rnnt")["enc_mean"]) + 0.3 * torch.randn(3, 20, 768, generator=g)
    enc_len = torch.tensor([20, 0, 1], dtype=torch.int32)
    want = orc.rnnt_greedy(enc.transpose(1, 2), enc_len, v2_rnnt_ckpt["state_dict"], 10)
    ids, frames, counts = eng_rnnt.greedy(enc.cuda(), enc_len.cuda())
    for b in range(3):
        n = int(counts[b])
        assert ids[b, :n].tolist() == want[b][0] and frames[b, :n].tolist() == want[b][1]
    assert int(counts[1]) == 0


@pytest.mark.parametrize("which,B", [("v2", 40), ("v3", 40), ("v2", 61)])
def test_rnnt_large_batches_against_oracle_and_small_groups(which, B, eng_rnnt, v2_rnnt_ckpt, request):
    """A batch too large for one 4-utterance group per cluster takes the 8-utterance kernel variant (two float4 halves,
    ragged last group); it must give the oracle's hypotheses and exactly what the 4-utterance variant gives when the
    same utterances are decoded in batches of 3.  v3 = 1025 classes: part of W_o stays in L2 (the prefetch path).
    B = 61 needs more groups than clusters can be resident (a few on an H100): clusters decode a second group after their first."""
    if which == "v2":
        eng, sd = eng_rnnt, v2_rnnt_ckpt["state_dict"]
    else:
        eng, sd = request.getfixturevalue("eng_v3"), request.getfixturevalue("v3_ckpt")["state_dict"]
    g = torch.Generator().manual_seed(21)
    T = 24
    mean = torch.as_tensor(synthetic._rnnt_calibration("v2_rnnt" if which == "v2" else "v3_e2e_rnnt")["enc_mean"])
    enc = mean + torch.randn(B, T, 768, generator=g) * 0.3      # blank runs, single tokens and max_symbols bursts
    enc_len = torch.randint(0, T + 1, (B,), generator=g, dtype=torch.int32)
    enc_len[0], enc_len[7] = T, 0
    ids, frames, counts = (x.cpu() for x in eng.greedy(enc.cuda(), enc_len.cuda()))
    want = orc.rnnt_greedy(enc[:12].transpose(1, 2), enc_len[:12], sd, 10)
    for b in range(12):
        n = int(counts[b])
        assert ids[b, :n].tolist() == want[b][0] and frames[b, :n].tolist() == want[b][1], b
    for b0 in range(0, B, 3):
        i3, f3, c3 = (x.cpu() for x in eng.greedy(enc[b0:b0 + 3].contiguous().cuda(), enc_len[b0:b0 + 3].cuda()))
        for j in range(min(3, B - b0)):
            n = int(c3[j])
            assert n == int(counts[b0 + j])
            assert torch.equal(i3[j, :n], ids[b0 + j, :n]) and torch.equal(f3[j, :n], frames[b0 + j, :n])
    if which == "v2":
        assert int(counts.sum()) > 0


# ------------------------------------------------------------------------------------------ word grouping on the device
class _Pieces:
    """Stand-in tokenizer: id -> piece (charwise vocabularies and SentencePiece models both reduce to this)."""

    def __init__(self, pieces):
        self.pieces = pieces

    def __len__(self):
        return len(self.pieces)

    def id_to_str(self, i):
        return self.pieces[i]


@pytest.mark.parametrize("kind", ["char", "sentencepiece"])
def test_word_grouping_on_device_matches_reference_semantics(eng_ctc, dev, kind):
    """gam_group_words (csrc/words.cu) against the host restatement of gigaam/timestamps_utils.py:13-53 on random
    hypotheses: leading / trailing / repeated delimiters, bare U+2581 pieces, whitespace-only pieces, empty utterances,
    utterances longer than one 32-token chunk."""
    from gigaam_b200.timestamps_utils import frames_to_words, token_flag_table, words_from_device
    if kind == "char":
        tok = _Pieces([" "] + [chr(c) for c in range(ord("a"), ord("a") + 20)])
    else:
        tok = _Pieces(["\u2581", "\u2581ab", "cd", "\u2581e", "f", "\u2581 ", "g", "\u2581hij", "k", " ", "\t", "lm"])
    g = torch.Generator().manual_seed(len(tok))
    B, max_out = 9, 100
    counts = torch.tensor([0, 1, 5, 31, 32, 33, 64, 100, 77], dtype=torch.int32)
    p_delim = 0.25 if kind == "char" else 0.1
    ids = torch.randint(1 if kind == "char" else 0, len(tok), (B, max_out), generator=g, dtype=torch.int32)
    ids[torch.rand(B, max_out, generator=g) < p_delim] = 0 if kind == "char" else 9
    ids[2, :5] = torch.tensor([0, 0, 3, 0, 0] if kind == "char" else [9, 0, 5, 10, 9], dtype=torch.int32)
    frames = torch.sort(torch.randint(0, 400, (B, max_out), generator=g, dtype=torch.int32), dim=1).values
    flags = token_flag_table(tok)
    rec = eng_ctc.group_words(ids.to(dev), frames.to(dev), counts.to(dev), flags)
    ws, we, wf, wn, nw = (t.cpu() for t in rec)
    seen_words = 0
    for b in range(B):
        n, k = int(counts[b]), int(nw[b])
        row = ids[b, :n].tolist()
        want = frames_to_words(tok, row, frames[b, :n].tolist(), 0.04)
        got = words_from_device(tok, row, ws[b, :k].tolist(), we[b, :k].tolist(), wf[b, :k].tolist(), wn[b, :k].tolist(), 0.04)
        assert [(w.text, w.start, w.end) for w in got] == [(w.text, w.start, w.end) for w in want], b
        seen_words += k
    assert seen_words > 20


# ------------------------------------------------------------------------------------------ public API (drop-in surface)
def test_public_api_drop_in(dev, v2_ctc_ckpt):
    model = gigaam.load_model("v2_ctc", device=dev, checkpoint=v2_ctc_ckpt)     # reference default: fp16 encoder
    assert model._device.type == "cuda" and model._dtype == torch.float16
    wav, wav_len = synthetic.synthetic_audio(2, 2.0, seed=1234, ragged=True)
    enc, enc_len = model(wav.to(dev), wav_len.to(dev))
    assert enc.shape == (2, 768, 51) and enc.dtype == torch.float32 and enc_len.dtype == torch.int32
    hyps = model.decoding.decode(model.head, enc, enc_len)
    assert len(hyps) == 2 and all(isinstance(t, str) and len(i) == len(f) for t, i, f in hyps)
    assert all(t == "".join(model.decoding.tokenizer.vocab[k] for k in i) for t, i, _ in hyps)
    assert model.decoding.blank_id == 33
    # single-utterance surface: transcribe / embed_audio from an in-memory waveform
    res = model.transcribe(wav[0])
    assert isinstance(res, gigaam.TranscriptionResult) and res.words is None and isinstance(str(res), str)
    res_w = model.transcribe(wav[0], word_timestamps=True)
    assert res_w.text == res.text and all(w.end > w.start for w in res_w.words)
    emb, emb_len = model.embed_audio(wav[0])
    assert emb.shape[:2] == (1, 768) and int(emb_len[0]) == emb.shape[2]
    with pytest.raises(ValueError, match="Too long"):
        model.transcribe(torch.zeros(25 * 16000 + 1))
    # components reachable like the reference's tests do (tests/test_batching.py:39-64)
    feats, flen = model.preprocessor(wav.to(dev), wav_len.to(dev))
    pre, plen = model.encoder.pre_encode(x=feats.transpose(1, 2), lengths=flen)
    assert pre.shape == (2, 51, 768) and torch.equal(plen.cpu(), enc_len.cpu())


def test_fp16_encoder_weights_stay_within_tolerance(dev, v2_ctc_ckpt):
    """load_model(fp16_encoder=True) rounds *all* encoder parameters to fp16 like the reference (gigaam/__init__.py:
    188-189); the result must stay close to the fp32-weight run."""
    wav, wav_len = synthetic.synthetic_audio(2, 2.0, seed=1234, ragged=True)
    m16 = gigaam.load_model("v2_ctc", device=dev, checkpoint=v2_ctc_ckpt)
    m32 = gigaam.load_model("v2_ctc", fp16_encoder=False, device=dev, checkpoint=v2_ctc_ckpt)
    e16, l16 = m16(wav.to(dev), wav_len.to(dev))
    e32, l32 = m32(wav.to(dev), wav_len.to(dev))
    assert torch.equal(l16, l32)
    valid = torch.arange(e32.shape[2], device=dev)[None, :] < l32[:, None]
    assert rel(e16.transpose(1, 2)[valid], e32.transpose(1, 2)[valid]) < 3e-3


# ------------------------------------------------------------------------------------------ BASELINE sizes, benchmarked mode
# Every BASELINE.json config at its stated per-GPU size, through load_model(...) with the DEFAULT fp16_encoder=True (the
# mode bench.py times), against the oracle run on the same fp16-rounded-then-float encoder parameters
# (gigaam/__init__.py:188-189: `model.encoder.half()` rounds every encoder tensor, the head stays fp32).
# Fixed logit margin, derived once from the activation budget: a relative error of 1e-3 on a frame of norm ~27.7 moves a
# logit (head-row norm ~2.3) by 2.3 * 0.0277 / sqrt(768) = 2.3e-3 rms and a top-2 difference by 3.3e-3 rms -> 3 sigma.
CTC_MARGIN_EPS = 0.01
# The synthetic head on the stationary test signal has many near-ties: 3.6 % of config 2's frames (oracle alone, CPU
# measurement) sit below the margin; they are counted and reported, not compared.
CTC_SUBMARGIN_MAX = 0.06


def _fp16_rounded(sd):
    return {k: (v.half().float() if k.startswith("encoder.") and v.is_floating_point() else v) for k, v in sd.items()}


def _encoder_parity(model, ckpt, wav, wav_len, dev):
    sd16 = _fp16_rounded(ckpt["state_dict"])
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


def test_config2_full_size_against_oracle(dev, v2_ctc_ckpt):
    """BASELINE.json configs[1]: v2_ctc, 64 x 10 s (R = 16 064 rows: three GEMM waves, the benchmarked shape)."""
    model = gigaam.load_model("v2_ctc", device=dev, checkpoint=v2_ctc_ckpt)
    assert model._dtype == torch.float16
    wav, wav_len = synthetic.synthetic_audio(64, 10.0, seed=1234)
    enc, enc_len, enc_o, len_o, sd16 = _encoder_parity(model, v2_ctc_ckpt, wav, wav_len, dev)
    assert enc.shape == (64, 768, 251)
    # CTC ids: frame labels from the GPU activations == oracle labels wherever the oracle margin exceeds the FIXED eps
    logits = orc.ctc_logits(enc_o, sd16)
    top2 = logits.topk(2, dim=-1).values
    margin = top2[..., 0] - top2[..., 1]
    lab_gpu = F.conv1d(enc.cpu(), sd16["head.decoder_layers.0.weight"], sd16["head.decoder_layers.0.bias"]).argmax(1)
    valid = torch.arange(logits.shape[1])[None, :] < len_o[:, None]
    safe = valid & (margin > CTC_MARGIN_EPS)
    n_sub = int((valid & ~safe).sum())
    print(f"CTC: {n_sub} of {int(valid.sum())} frames below the {CTC_MARGIN_EPS} margin; "
          f"{int((lab_gpu != logits.argmax(-1))[valid].sum())} label differences in total")
    assert torch.equal(lab_gpu[safe], logits.argmax(-1)[safe])
    assert n_sub / float(valid.sum()) < CTC_SUBMARGIN_MAX
    # the device decoder on its own activations == the oracle decoder on the same activations (bit exact away from fp32 ties)
    ids, frames, counts = (t.cpu() for t in model.decoding.decode_device(model.head, enc, enc_len))
    want = orc.ctc_greedy(enc.cpu(), enc_len.cpu(), sd16)
    lg = orc.ctc_logits(enc.cpu(), sd16).topk(2, dim=-1).values
    tie_free = ((lg[..., 0] - lg[..., 1]) > 1e-4).all(1)
    assert int(tie_free.sum()) >= 48      # utterances whose own top-2 margins leave no room for an fp32 summation-order tie
    for b in range(64):
        n = int(counts[b])
        if tie_free[b]:
            assert ids[b, :n].tolist() == want[b][0] and frames[b, :n].tolist() == want[b][1], b
    # determinism and batch independence at this size
    enc2, _ = model(wav.to(dev), wav_len.to(dev))
    assert torch.equal(enc, enc2)
    enc_s, _ = model(wav[:2].to(dev), wav_len[:2].to(dev))
    assert rel(enc_s, enc[:2]) < 1e-6 or float((enc_s - enc[:2]).abs().max()) < 1e-3


def _rnnt_on_oracle_activations(model, enc_o, len_o, sd, max_symbols, dev):
    ids, frames, counts = (t.cpu() for t in model.decoding.decode_device(model.head, enc_o.to(dev), len_o.to(dev)))
    want = orc.rnnt_greedy(enc_o, len_o, sd, max_symbols)
    total = 0
    for b in range(enc_o.shape[0]):
        n = int(counts[b])
        total += n
        assert ids[b, :n].tolist() == want[b][0] and frames[b, :n].tolist() == want[b][1], b
    rate = total / float(len_o.sum())
    print(f"RNN-T: {total} tokens, {rate:.3f} tokens/frame")
    return rate


def test_config3_full_size_against_oracle(dev, v2_rnnt_ckpt):
    """BASELINE.json configs[2]: v2_rnnt, 32 x 15 s.  Encoder vs oracle; the device RNN-T loop fed the ORACLE's activations
    must reproduce the oracle's hypotheses for all 32 utterances."""
    model = gigaam.load_model("v2_rnnt", device=dev, checkpoint=v2_rnnt_ckpt)
    wav, wav_len = synthetic.synthetic_audio(32, 15.0, seed=77)
    enc, enc_len, enc_o, len_o, sd16 = _encoder_parity(model, v2_rnnt_ckpt, wav, wav_len, dev)
    assert enc.shape == (32, 768, 376)
    rate = _rnnt_on_oracle_activations(model, enc_o, len_o, sd16, 10, dev)
    assert 0.1 < rate < 2.0          # calibrated head (oracle/calibrate_rnnt.py), target 0.5
    ids, frames, counts = model.decoding.decode_device(model.head, enc, enc_len)
    assert bool((counts <= 376 * 10).all()) and int(counts.sum()) > 0


def test_config4_per_gpu_size_against_oracle(dev, v3_ckpt):
    """BASELINE.json configs[3]: v3_e2e_rnnt 256 x 10 s over 8 GPUs = 32 x 10 s per GPU (conv1d subsampling, LayerNorm conv
    module, 1025 classes: part of W_o streams from L2 in the RNN-T kernel)."""
    model = gigaam.load_model("v3_e2e_rnnt", device=dev, checkpoint=v3_ckpt)
    wav, wav_len = synthetic.synthetic_audio(32, 10.0, seed=1234)
    enc, enc_len, enc_o, len_o, sd16 = _encoder_parity(model, v3_ckpt, wav, wav_len, dev)
    assert enc.shape == (32, 768, 250)
    rate = _rnnt_on_oracle_activations(model, enc_o, len_o, sd16, 10, dev)
    assert 0.03 < rate < 1.0         # target 0.2


def test_config5_slice_against_oracle(dev):
    """BASELINE.json configs[4]: v2_ssl embed path, 25 s utterances (T' = 626: five key blocks, one K / V set per CTA in the attention kernel; s1 of
    0.5 G elements per 16 utterances); a 16-utterance slice of the 128 x 25 s batch."""
    ck = synthetic.synthetic_checkpoint("v2_ssl", seed=0)
    model = gigaam.load_model("v2_ssl", device=dev, checkpoint=ck)
    wav, wav_len = synthetic.synthetic_audio(16, 25.0, seed=1234)
    enc, enc_len, _, _, _ = _encoder_parity(model, ck, wav, wav_len, dev)
    assert enc.shape == (16, 768, 626)


def test_segment_of_30s_runs_and_matches_oracle(dev, v2_ctc_ckpt):
    """The reference's VAD emits segments of up to 30 s (gigaam/vad_utils.py:85,105-118) and forward() has no length
    guard: T' = 751 (six key blocks)."""
    model = gigaam.load_model("v2_ctc", device=dev, checkpoint=v2_ctc_ckpt)
    wav, wav_len = synthetic.synthetic_audio(2, 30.0, seed=31, ragged=True)
    enc, enc_len, _, _, _ = _encoder_parity(model, v2_ctc_ckpt, wav, wav_len, dev)
    assert enc.shape[2] == 751
    with pytest.raises(Exception, match="limit"):
        model(torch.zeros(1, 31 * 16000, device=dev), torch.tensor([31 * 16000], device=dev))


# ------------------------------------------------------------------------------------------ v3 shape (conv1d / LN conv-norm / k5 / n_fft 320)
@pytest.fixture(scope="session")
def v3_ckpt():
    return synthetic.synthetic_checkpoint("v3_e2e_rnnt", seed=0)


@pytest.fixture(scope="session")
def eng_v3(dev, v3_ckpt):
    return Engine(v3_ckpt["cfg"], v3_ckpt["state_dict"], dev)


def test_v3_frontend_and_encoder_against_reference_golden(eng_v3, v3_ckpt, golden_dir):
    """conv1d subsampling as two strided-TMA implicit GEMMs, LayerNorm conv-norm, depthwise k=5, center=False log-mel."""
    g = np.load(golden_dir / "v3_e2e_rnnt_b2_2s.npz")
    cfg, sd = v3_ckpt["cfg"], v3_ckpt["state_dict"]
    wav, wav_len = synthetic.synthetic_audio(2, 2.0, seed=1234, ragged=True)
    mel = eng_v3.logmel(wav.cuda())
    assert mel.shape == g["mel"].shape
    assert float((mel.cpu() - torch.from_numpy(g["mel"])).abs().max()) < 5e-3
    mel_len = torch.from_numpy(g["mel_len"])
    with torch.inference_mode():
        _, len_o, stages = orc.encoder_forward(torch.from_numpy(g["mel"]), mel_len, sd, cfg["encoder"], return_all=True)
    valid = torch.arange(stages[0].shape[1])[None, :] < len_o[:, None]
    for n in (0, 1, 16):
        enc, enc_len = eng_v3.encode(torch.from_numpy(g["mel"]).cuda(), mel_len.cuda(), n_layers_run=n)
        assert np.array_equal(enc_len.cpu().numpy(), g["enc_len"])
        assert rel(enc.cpu()[valid], stages[n][valid]) < ENC_REL_TOL, f"v3 after {n} layers"
    want = torch.from_numpy(g["enc"]).transpose(1, 2)
    assert rel(enc.cpu()[valid], want[valid]) < ENC_REL_TOL


def test_v3_rnnt_greedy_matches_reference_golden(eng_v3, golden_dir):
    g = np.load(golden_dir / "v3_e2e_rnnt_b2_2s.npz")
    enc = torch.from_numpy(g["enc"]).transpose(1, 2).contiguous()
    ids, frames, counts = eng_v3.greedy(enc.cuda(), torch.from_numpy(g["enc_len"]).cuda())
    total = 0
    for b in range(2):
        n = int(counts[b])
        total += n
        assert ids[b, :n].tolist() == g[f"ids_{b}"].tolist()
        assert frames[b, :n].tolist() == g[f"frames_{b}"].tolist()
    assert total > 0


# ------------------------------------------------------------------------------------------ v1 shape: rel_pos attention
@pytest.fixture(scope="session")
def eng_v1(dev, v1_ctc_ckpt):
    return Engine(v1_ctc_ckpt["cfg"], v1_ctc_ckpt["state_dict"], dev)


@pytest.mark.parametrize("B,T,lens", [(1, 128, None), (2, 51, [51, 30]), (3, 251, [251, 200, 97]), (2, 376, [376, 129]),
                                      (1, 626, None), (2, 5, [5, 1]), (2, 129, [129, 128]), (3, 300, [300, 0, 257]), (1, 640, None),
                                      (2, 751, [751, 700])])
def test_relpos_attention_matches_shifted_softmax(eng_v1, dev, B, T, lens):
    """gam_test_attention_relpos vs the reference formula (gigaam/encoder.py:216-228) in torch fp32, with the
    reference's own pad/view rel_shift, on the same fp16 operands."""
    from gigaam_b200 import _lib
    g = torch.Generator().manual_seed(B * 1000 + T + 7)
    d, H, dk, L = 768, 16, 48, _lib.REL_POS_MAX_T
    qkv = torch.randn(B * T, 4 * d, generator=g).half().to(dev)
    pos = torch.randn(2 * L - 1, d, generator=g).half().to(dev)
    out = torch.zeros(B * T, d, dtype=torch.float16, device=dev)
    klen = torch.tensor(lens, dtype=torch.int32, device=dev) if lens else None
    rc = eng_v1.lib.gam_test_attention_relpos(eng_v1.handle, qkv.data_ptr(), pos.data_ptr(), klen.data_ptr() if lens else None,
                                              out.data_ptr(), B, T, _stream())
    torch.cuda.synchronize()
    assert rc == 0
    x = qkv.float().view(B, T, 4, H, dk)
    qu, qv, k, v = (x[:, :, i].transpose(1, 2) for i in range(4))
    p = pos.float()[L - T: L + T - 1].view(2 * T - 1, H, dk).transpose(0, 1)            # positions T-1 ... -(T-1)
    bd = qv @ p.transpose(-1, -2)                                                        # [B, H, T, 2T-1]
    bd = F.pad(bd, (1, 0)).view(B, H, -1, T)[:, :, 1:].reshape(B, H, T, 2 * T - 1)[..., :T]   # rel_shift, encoder.py:202-206
    sc = (qu @ k.transpose(-1, -2) + bd) / dk ** 0.5
    valid = torch.ones(B, T, dtype=torch.bool, device=dev)
    if lens:
        valid = torch.arange(T, device=dev)[None, :] < klen[:, None]
        sc = sc.masked_fill(~valid[:, None, None, :], float("-inf"))
    want = (torch.softmax(sc, -1).nan_to_num(0.0) @ v).transpose(1, 2).reshape(B, T, d)
    got = out.float().view(B, T, d)
    assert torch.isfinite(out).all()
    has_keys = (valid.sum(1) > 0)
    assert rel(got[has_keys], want[has_keys]) < 1e-3
    assert float(got[~has_keys].abs().max()) == 0.0 if (~has_keys).any() else True   # no valid key -> zeros


def test_v1_rel_pos_encoder_against_reference_golden(eng_v1, v1_ctc_ckpt, golden_dir):
    """wav -> ids of the rel_pos model vs outputs of the REAL reference (tests/golden/v1_ctc_b2_6s.npz)."""
    g = np.load(golden_dir / "v1_ctc_b2_6s.npz")
    cfg, sd = v1_ctc_ckpt["cfg"], v1_ctc_ckpt["state_dict"]
    wav, wav_len = synthetic.synthetic_audio(2, 6.0, seed=1234, ragged=True)
    mel = eng_v1.logmel(wav.cuda())
    assert float((mel.cpu() - torch.from_numpy(g["mel"])).abs().max()) < 5e-3
    mel_ref, mel_len = torch.from_numpy(g["mel"]), torch.from_numpy(g["mel_len"])
    with torch.inference_mode():
        _, len_o, stages = orc.encoder_forward(mel_ref, mel_len, sd, cfg["encoder"], n_layers_run=2, return_all=True)
    valid = torch.arange(stages[0].shape[1])[None, :] < len_o[:, None]
    for n in (1, 2):
        e, _ = eng_v1.encode(mel_ref.cuda(), mel_len.cuda(), n_layers_run=n)
        assert rel(e.cpu()[valid], stages[n][valid]) < ENC_REL_TOL, f"after {n} layers"
    enc, enc_len = eng_v1.encode(mel, mel_len.cuda())
    assert np.array_equal(enc_len.cpu().numpy(), g["enc_len"])
    want = torch.from_numpy(g["enc"]).transpose(1, 2)
    assert torch.isfinite(enc).all()
    assert rel(enc.cpu()[valid], want[valid]) < ENC_REL_TOL
    ids, frames, counts = eng_v1.greedy(enc, enc_len)
    margin = torch.from_numpy(g["ctc_margin"])
    for b in range(2):
        n = int(counts[b])
        if float(margin[b][: int(g["enc_len"][b])].min()) > 2e-3:
            assert ids[b, :n].tolist() == g[f"ids_{b}"].tolist()
            assert frames[b, :n].tolist() == g[f"frames_{b}"].tolist()


def test_v1_batch_vs_single_and_long(eng_v1):
    """rel_pos path: a ragged batch agrees with its utterances run alone (atol 0.03 is the reference's own bar,
    tests/test_batching.py:70), and a 25 s utterance (T' = 626, five key blocks) stays finite."""
    wav, wav_len = synthetic.synthetic_audio(3, 4.0, seed=5, ragged=True)
    mel = eng_v1.logmel(wav.cuda())
    mel_len = torch.tensor([eng_v1.logmel_frames(int(n)) for n in wav_len])
    enc, enc_len = eng_v1.encode(mel, mel_len.cuda())
    for b in range(3):
        m = int(mel_len[b])
        e1, l1 = eng_v1.encode(mel[b:b + 1, :, :m].contiguous(), torch.tensor([m]).cuda())   # same front-end frames, alone
        n = int(l1[0])
        assert n == int(enc_len[b])
        assert float((e1[0, :n] - enc[b, :n]).abs().max()) < 0.03
        assert rel(e1[0, :n], enc[b, :n]) < 2e-3
    wav, _ = synthetic.synthetic_audio(1, 25.0, seed=6)
    mel = eng_v1.logmel(wav.cuda())
    enc, enc_len = eng_v1.encode(mel, torch.tensor([mel.shape[2]]).cuda())
    assert int(enc_len[0]) == 626 and torch.isfinite(enc).all()


# ------------------------------------------------------------------------------------------ serving loop
@pytest.mark.parametrize("use_graph", [False, True])
def test_batch_pipeline_equals_direct_calls(dev, v2_ctc_ckpt, use_graph):
    """gigaam_b200.pipeline.BatchPipeline (overlapped copies, CUDA-graph replay per shape) returns exactly what the
    plain `model(wav, len)` + `model.decoding.decode(...)` calls return, batch after batch, across two shapes."""
    from gigaam_b200.pipeline import BatchPipeline
    model = gigaam.load_model("v2_ctc", device=dev, checkpoint=v2_ctc_ckpt)
    batches = []
    for i, (B, sec) in enumerate([(3, 2.0), (3, 2.0), (2, 3.0), (3, 2.0), (2, 3.0)]):
        wav, wav_len = synthetic.synthetic_audio(B, sec, seed=100 + i, ragged=True)
        batches.append((wav.pin_memory(), wav_len))
    want = []
    for wav, wav_len in batches:
        enc, enc_len = model(wav.to(dev), wav_len.to(dev))
        want.append(model.decoding.decode(model.head, enc, enc_len))
    got = list(BatchPipeline(model, use_graph=use_graph).run(iter(batches)))
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g == w
    assert sum(len(h[1]) for hyps in want for h in hyps) > 0


def test_batch_pipeline_many_shapes_keeps_graph_workspaces_alive(dev, v2_ctc_ckpt):
    """More input shapes than the engine's workspace cache holds (4 per kind), revisited in a round robin: every cached
    graph keeps writing into scratch memory it owns, so replays after the engine has forgotten the shape still give the
    plain-call results, and device memory stays bounded."""
    from gigaam_b200.pipeline import BatchPipeline
    model = gigaam.load_model("v2_ctc", device=dev, checkpoint=v2_ctc_ckpt)
    shapes = [(2, 1.0), (2, 1.5), (3, 1.0), (1, 2.0), (2, 2.5), (3, 0.8)]
    batches = []
    for rnd in range(3):
        for i, (B, sec) in enumerate(shapes):
            wav, wav_len = synthetic.synthetic_audio(B, sec, seed=300 + 10 * rnd + i, ragged=True)
            batches.append((wav.pin_memory(), wav_len))
    want = []
    for wav, wav_len in batches:
        enc, enc_len = model(wav.to(dev), wav_len.to(dev))
        want.append(model.decoding.decode(model.head, enc, enc_len))
    pipe = BatchPipeline(model, use_graph=True, max_graphs=len(shapes))
    got = list(pipe.run(iter(batches)))
    assert got == want
    eng = model._get_engine()
    assert len(eng._ws_enc) <= eng.WS_CACHE and len(eng._ws_mel) <= eng.WS_CACHE and len(eng._ws_dec) <= eng.WS_CACHE


def test_many_distinct_lengths_do_not_leak_workspaces(dev, v2_ctc_ckpt):
    """transcribe() over many different lengths (what eval / long-form loops do): the engine's scratch caches are bounded
    per kind, so allocated device memory levels off instead of growing with the number of shapes seen."""
    model = gigaam.load_model("v2_ctc", device=dev, checkpoint=synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=2))
    wav, _ = synthetic.synthetic_audio(1, 6.0, seed=5)
    peaks = []
    for i in range(24):
        model.transcribe(wav[0, : 16000 + 3217 * ((7 * i) % 24)])      # 24 distinct lengths, shuffled
        torch.cuda.synchronize()
        peaks.append(torch.cuda.memory_allocated(dev))
    assert max(peaks[12:]) <= max(peaks[:12]) * 1.5 + (64 << 20)


def test_packed_weight_cache_and_triton_contract(dev, v2_ctc_ckpt, tmp_path):
    """SURVEY 8f-4: (a) a checkpoint FILE loads through `load_model(download_root=...)`; the second load finds the packed
    weights cached next to it (keyed by the file's md5) and gives bit-identical results; (b) the Triton ensemble's I/O
    contract (audio_batch FP32 concat + INT64 lengths -> texts) served by one call chain on the GPU."""
    from gigaam_b200.serving.triton_backend import config_pbtxt, transcribe_concatenated
    ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=2)
    torch.save(ck, tmp_path / "v2_ctc.ckpt")
    m1 = gigaam.load_model("v2_ctc", device=dev, download_root=str(tmp_path))
    wav, wav_len = synthetic.synthetic_audio(3, 2.0, seed=8, ragged=True)
    e1, l1 = m1(wav.to(dev), wav_len.to(dev))
    assert m1._get_engine().pack_cache_hit is False
    assert len(list(tmp_path.glob("v2_ctc.*.float16.b200pack"))) == 1
    m2 = gigaam.load_model("v2_ctc", device=dev, download_root=str(tmp_path))
    e2, l2 = m2(wav.to(dev), wav_len.to(dev))
    assert m2._get_engine().pack_cache_hit is True and torch.equal(e1, e2) and torch.equal(l1, l2)
    # Triton contract: concatenated utterances in, one text per utterance out, in request order
    lens = [int(n) for n in wav_len]
    concat = np.concatenate([wav[i, : lens[i]].numpy() for i in range(3)])
    texts = transcribe_concatenated(m2, concat, np.asarray(lens, dtype=np.int64), max_utterances=2)
    alone = [str(m2.transcribe(wav[i, : lens[i]])) for i in range(3)]
    assert texts[0] == alone[0] and len(texts) == 3 and all(isinstance(t, str) for t in texts)
    assert [t[:-3] for t in texts] == [a[: len(t[:-3])] for t, a in zip(texts, alone)]    # padded members may differ in the tail
    cfg = config_pbtxt(model_name="v2_ctc")
    assert 'name: "audio_batch"' in cfg and "TYPE_INT64" in cfg and "TYPE_STRING" in cfg
    with pytest.raises(ValueError):
        transcribe_concatenated(m2, concat, [concat.size, 5])


def test_transcribe_longform_against_oracle(dev):
    """transcribe_longform (gigaam/model.py:195-259) over pre-cut segments against the ORACLE: every segment's text and word
    timestamps must equal the CPU oracle's greedy decode of that segment (fp16-rounded waveform and encoder parameters, as
    the reference does on CUDA), shifted by the segment start.  Segments were picked (2-layer synthetic model) so that the
    oracle's top-2 logit margin stays above 0.02 on every frame -- asserted here, so the comparison can be exact."""
    from gigaam_b200.longform import plan_batches
    from gigaam_b200.timestamps_utils import frames_to_words
    ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=2)
    model = gigaam.load_model("v2_ctc", device=dev, checkpoint=ck)
    sd16, cfg = _fp16_rounded(ck["state_dict"]), ck["cfg"]
    vocab = cfg["decoding"]["vocabulary"]
    seeds = [203, 211, 217, 241, 249, 252, 212, 226, 250, 242]
    segments = [synthetic.synthetic_audio(1, 2.0 + (sd % 5) * 0.7, seed=sd)[0][0] for sd in seeds]
    bounds, t0 = [], 0.0
    for s in segments:
        bounds.append((t0, t0 + s.numel() / 16000.0))
        t0 += s.numel() / 16000.0 + 0.25

    def oracle(wav, wav_len):
        with torch.inference_mode():
            enc, enc_len = orc.model_forward(wav.half().float(), wav_len, sd16, cfg)
        top2 = orc.ctc_logits(enc, sd16).topk(2, dim=-1).values
        margin = top2[..., 0] - top2[..., 1]
        ok = [float(margin[i, : int(enc_len[i])].min()) > 0.02 for i in range(wav.shape[0])]
        return orc.ctc_greedy(enc, enc_len, sd16), enc_len, ok

    # one segment per batch: no padding, exact for every segment
    res = model.transcribe_longform(None, word_timestamps=True, fr_batch_size=1, segments=segments, boundaries=bounds)
    assert len(res) == len(segments) and res.has_word_timestamps
    for seg, wav, (s0, e0) in zip(res, segments, bounds):
        hyp, enc_len, ok = oracle(wav[None], torch.tensor([wav.numel()]))
        assert ok[0], "test segment lost its margin: pick another seed"
        ids, frames = hyp[0]
        assert seg.text == "".join(vocab[i] for i in ids) and (seg.start, seg.end) == (s0, e0)
        want = frames_to_words(model.decoding.tokenizer, ids, frames, wav.numel() / 16000.0 / int(enc_len[0]))
        assert [w.text for w in seg.words] == [w.text for w in want]
        for a, b in zip(seg.words, want):
            assert a.start == pytest.approx(b.start + s0, abs=2e-3) and a.end == pytest.approx(b.end + s0, abs=2e-3)
    # length-bucketed batches of 4: the oracle runs the SAME padded batches (padding semantics are part of the path)
    res4 = model.transcribe_longform(None, fr_batch_size=4, segments=segments, boundaries=bounds)
    lengths = [s.numel() for s in segments]
    compared = 0
    for batch in plan_batches(lengths, 4):
        wav = torch.zeros(len(batch), max(lengths[i] for i in batch))
        for row, i in enumerate(batch):
            wav[row, : lengths[i]] = segments[i]
        hyp, _, ok = oracle(wav, torch.tensor([lengths[i] for i in batch]))
        for row, i in enumerate(batch):
            if ok[row]:
                assert res4.segments[i].text == "".join(vocab[k] for k in hyp[row][0]), i
                compared += 1
    assert compared >= 5


def test_transcribe_longform_equals_per_segment_transcribe(dev, v2_ctc_ckpt):
    """transcribe_longform (gigaam/model.py:195-259) over pre-cut segments == transcribe() of every segment alone, in
    recording order, with word timestamps shifted by the segment start; the built-in splitter handles a 50 s waveform
    that transcribe() itself refuses (>25 s, model.py:135-136)."""
    model = gigaam.load_model("v2_ctc", device=dev, checkpoint=v2_ctc_ckpt)
    wavs, lens = synthetic.synthetic_audio(5, 4.0, seed=77, ragged=True)
    segments = [wavs[i, : int(lens[i])] for i in range(5)]
    bounds, t0 = [], 0.0
    for s in segments:
        bounds.append((t0, t0 + s.numel() / 16000.0))
        t0 += s.numel() / 16000.0 + 0.5
    res = model.transcribe_longform(None, word_timestamps=True, fr_batch_size=1, segments=segments, boundaries=bounds)
    assert isinstance(res, gigaam.LongformTranscriptionResult) and len(res) == 5 and res.has_word_timestamps
    alone = [model.transcribe(wav, word_timestamps=True) for wav in segments]
    for seg, one, (s0, e0) in zip(res, alone, bounds):
        assert seg.text == one.text and (seg.start, seg.end) == (s0, e0)
        assert [w.text for w in seg.words] == [w.text for w in one.words]
        for a, b in zip(seg.words, one.words):
            assert a.start == pytest.approx(b.start + s0, abs=2e-3) and a.end == pytest.approx(b.end + s0, abs=2e-3)
    # length-bucketed batches of 2: the padded member's last mel frames see zeros instead of the reflection a lone run
    # sees (same as the reference's padded batches), so only its tail may differ
    res2 = model.transcribe_longform(None, fr_batch_size=2, segments=segments, boundaries=bounds)
    assert len(res2) == 5 and not res2.has_word_timestamps
    for seg, one, (s0, e0) in zip(res2, alone, bounds):
        assert (seg.start, seg.end) == (s0, e0) and seg.text[:-3] == one.text[: len(seg.text[:-3])]
    long_wav, _ = synthetic.synthetic_audio(1, 50.0, seed=78)
    with pytest.raises(ValueError):
        model.transcribe(long_wav[0])
    res = model.transcribe_longform(long_wav[0])
    assert len(res) >= 3 and res.segments[0].start == 0.0 and res.segments[-1].end == pytest.approx(50.0)
    assert all(s.end - s.start <= 22.0 + 1e-6 for s in res) and isinstance(res.text, str)


# ------------------------------------------------------------------------------------------ varlen (packed-row) execution, SURVEY 8 a19
def _pack(x_btc, lens):
    return torch.cat([x_btc[b, :n] for b, n in enumerate(lens)], 0)


_MIXED_251 = [int(x) for x in np.random.default_rng(5).integers(0, 252, size=44)]    # 704 items: ~5 per persistent CTA,
_MIXED_626 = [int(x) for x in np.random.default_rng(6).integers(0, 627, size=24)]    # 1-/2-tile and empty utterances interleaved


@pytest.mark.parametrize("relpos", [False, True])
@pytest.mark.parametrize("T,lens", [(251, [251, 97, 1, 0, 128, 129, 200]), (128, [5, 128, 64]), (751, [751, 129, 640, 300]),
                                    (376, [0, 376, 257, 31]), (251, _MIXED_251), (626, _MIXED_626)])
def test_attention_varlen_packed_rows(request, dev, relpos, T, lens):
    """The cu_seqlens contract of apply_masked_flash_attn (gigaam/utils.py:103-155): q / k / v rows of the utterances lie
    back to back, every utterance attends to its own frames only, nothing is computed for frames that do not exist.  The
    rows behind the last utterance are poisoned with NaN: a tile that reaches past the stream must not let them in."""
    from gigaam_b200 import _lib
    eng = request.getfixturevalue("eng_v1" if relpos else "eng_ctc")
    B, d, H, dk, L = len(lens), 768, 16, 48, _lib.REL_POS_MAX_T
    parts = 4 if relpos else 3
    g = torch.Generator().manual_seed(T + 17 * B + relpos)
    x = torch.randn(B, T, parts * d, generator=g).half()
    rows = sum(lens)
    qkv = torch.full((rows + 300, parts * d), float("nan"), dtype=torch.float16)
    qkv[:rows] = _pack(x, lens)
    qkv = qkv.to(dev)
    pos = torch.randn(2 * L - 1, d, generator=g).half().to(dev)
    out = torch.full((rows + 300, d), 7.0, dtype=torch.float16, device=dev)
    klen = torch.tensor(lens, dtype=torch.int32, device=dev)
    cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=dev)
    rc = eng.lib.gam_test_attention_varlen(eng.handle, qkv.data_ptr(), pos.data_ptr() if relpos else None, klen.data_ptr(),
                                           cu.data_ptr(), out.data_ptr(), B, T, rows + 300, _stream())
    torch.cuda.synchronize()
    assert rc == 0, eng.lib.gam_last_error(eng.handle)
    assert torch.isfinite(out).all()
    assert bool((out[rows:] == 7.0).all())                 # nothing stored behind the stream
    for b, n in enumerate(lens):
        if n == 0:
            continue
        xb = x[b, :n].float().to(dev).view(n, parts, H, dk)
        if relpos:
            qu, qv, k, v = (xb[:, i].transpose(0, 1) for i in range(4))
            p = pos.float()[L - n: L + n - 1].view(2 * n - 1, H, dk).transpose(0, 1)
            bd = qv @ p.transpose(-1, -2)
            bd = F.pad(bd, (1, 0)).view(H, -1, n)[:, 1:].reshape(H, n, 2 * n - 1)[..., :n]      # rel_shift, encoder.py:202-206
            sc = (qu @ k.transpose(-1, -2) + bd) / dk ** 0.5
        else:
            q, k, v = (xb[:, i].transpose(0, 1) for i in range(3))
            sc = q @ k.transpose(-1, -2) / dk ** 0.5
        want = (torch.softmax(sc, -1) @ v).transpose(0, 1).reshape(n, d)
        got = out[int(cu[b]): int(cu[b]) + n].float()
        assert rel(got, want) < 1e-3, (b, n)


@pytest.mark.parametrize("which", ["v2_ctc", "v3_e2e_rnnt", "v1_ctc"])
def test_varlen_ragged_batch_against_oracle(request, dev, which):
    """A strongly ragged batch (10 s down to a single encoder frame) through load_model(...) in the benchmarked fp16 mode vs
    the oracle on the valid frames, for the three encoder shapes (conv2d + BatchNorm + rotary; conv1d + LayerNorm;
    rel_pos).  Only sum(len) rows run through the blocks; frames that do not exist come back as zeros; a second call
    with the scratch memory poisoned with NaN gives bit-identical results (nothing stale is ever read)."""
    ck = {"v2_ctc": "v2_ctc_ckpt", "v3_e2e_rnnt": "v3_ckpt", "v1_ctc": "v1_ctc_ckpt"}[which]
    ckpt = request.getfixturevalue(ck)
    model = gigaam.load_model(which, device=dev, checkpoint=ckpt)
    secs = [10.0, 0.06, 3.3, 7.77, 0.5, 10.0, 1.29, 5.12]
    wav, _ = synthetic.synthetic_audio(len(secs), 10.0, seed=4321)
    wav_len = torch.tensor([int(s * 16000) for s in secs])
    for b, n in enumerate(wav_len.tolist()):
        wav[b, n:] = 0.0
    enc, enc_len, enc_o, len_o, _ = _encoder_parity(model, ckpt, wav, wav_len, dev)
    assert int(len_o.min()) <= 2 and int(len_o.max()) >= 250
    pad = torch.arange(enc.shape[2], device=dev)[None, :] >= enc_len[:, None]
    assert float(enc.transpose(1, 2)[pad].abs().max()) == 0.0
    eng = model._get_engine()
    for cache in (eng._ws_enc, eng._ws_mel, eng._ws_dec):
        for t in cache.tensors():
            t.view(torch.float16).fill_(float("nan"))
    enc2, _ = model(wav.to(dev), wav_len.to(dev))
    assert torch.equal(enc, enc2)


def test_varlen_rows_scale_with_audio_not_with_padding(dev, v2_ctc_ckpt):
    """Size-independent property at the BASELINE config-2 shape: 64 utterances of which 48 are 1 s long inside a 10 s
    buffer.  Each utterance equals its run inside a batch of its own kind (lengths alone decide the result, padding does
    not), and the step is much cheaper than the 64 x 10 s one because only the existing frames are computed."""
    model = gigaam.load_model("v2_ctc", device=dev, checkpoint=v2_ctc_ckpt)
    wav, _ = synthetic.synthetic_audio(64, 10.0, seed=99)
    full_len = torch.full((64,), 160000)
    rag_len = full_len.clone()
    rag_len[16:] = 16000
    wav_r = wav.clone()
    wav_r[16:, 16000:] = 0.0
    eng = model._get_engine()
    mel = eng.logmel(wav_r.to(dev))
    mel_len = (rag_len // 160 + 1).to(dev)
    m1 = int(mel_len[16])
    enc_r, len_r = eng.encode(mel, mel_len)
    enc_s, len_s = eng.encode(mel[16:, :, :m1].contiguous(), mel_len[16:])       # the short ones alone: no padded frame anywhere
    n = int(len_s[0])
    assert torch.equal(len_r[16:], len_s) and n == 26
    assert rel(enc_r[16:, :n], enc_s[:, :n]) < 1e-5 or float((enc_r[16:, :n] - enc_s[:, :n]).abs().max()) < 1e-3
    assert float(enc_r[16:, n:].abs().max()) == 0.0
    enc_f, _ = eng.encode(mel[:16].contiguous(), mel_len[:16])                    # the long ones alone
    assert rel(enc_r[:16], enc_f) < 1e-5 or float((enc_r[:16] - enc_f).abs().max()) < 1e-3

    def kernel_ms(w, l):
        """Sum of the kernels' own durations (CUDA events around every launch, gam_profile_*): what the GPU spends on the
        batch, free of the host's launch pace -- an eager step of 237 launches is launch-bound on a busy host."""
        w, l = w.to(dev), l.to(dev)
        model(w, l)
        best = float("inf")
        for _ in range(3):
            eng.profile_begin()
            model(w, l)
            best = min(best, sum(ms for ms, _ in eng.profile_end().values()))
        return best
    t_full, t_rag = kernel_ms(wav, full_len), kernel_ms(wav_r, rag_len)
    frac = float(rag_len.sum()) / float(full_len.sum())
    print(f"kernel time, 64 x 10 s: {t_full:.2f} ms; 16 x 10 s + 48 x 1 s in the same buffer ({frac:.2f} of the audio): {t_rag:.2f} ms")
    # 0.33 of the audio; measured 0.51 of the kernel time: the front end and the CTC head run over the whole buffer, the short
    # utterances still cost a 128 x 128 attention tile per head and a 256-row GEMM tile granularity, and kernels have floors
    assert t_rag < 0.62 * t_full
