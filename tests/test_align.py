"""Alignment of known transcripts (gam_ctc_align, gam_rnnt_align_scores, gam_rnnt_align; include/gigaam_b200.h has the
definitions, INTEGRATION.md §7d the user's view).

The work is checked in two stages.  Stage 1 (the per-frame / per-node scores) is gam_ctc_log_probs, tested elsewhere, or the
gathered joint, which must be bit-identical to the lattice of gam_rnnt_joint.  Stage 2 (the dynamic programme) runs on
planted fp32 scores.  Its Viterbi recursion is a fixed sequence of fp32 adds and strict compares, so the numpy float32 replay
below reproduces frames, token log-probs, path scores and path rows bit for bit; only the forward (log-sum-exp) recursion is
approximate, and it is compared with float64 within bounds derived in `ctc_forward_bound` / `rnnt_forward_bound`.

CPU: the float64 definitions against F.ctc_loss and torchaudio's rnnt_loss, the replay's tie rules on hand-built scores,
Tokenizer.encode, the Alignment record and the refusals of align_batch.  GPU: stage 2 of both heads against the replay at up
to T = 5000 and U = 4096, stage 1 against the lattice, the public calls end to end on one-layer synthetic models, batch
independence, determinism and a CUDA-graph replay."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gigaam_b200 as gigaam
from gigaam_b200 import decoding, synthetic
from gigaam_b200.decoding import Tokenizer
from gigaam_b200.timestamps_utils import compute_frame_shift, frames_to_words, mean_logp_confidence, path_confidence
from gigaam_b200.types import Alignment, Word

U32 = 2.0 ** -24          # unit roundoff of fp32
INF, NAN = float("inf"), float("nan")
F32 = np.float32


# ------------------------------------------------------------------------------------------ the oracle: float32 replay
def _empty_result(U, value):
    return np.full(U, -1, np.int32), np.full(U, value, F32)


def ctc_replay(lp, Tb, y, U=None):
    """Stage 2 of CTC for one utterance in numpy float32, the header's arithmetic step for step.  lp [T, V+1] float32, Tb its
    frame count, y its target ids.  -> (frames [U], token_logp [U], viterbi_logp, path_rows); U = the row pitch (>= len(y))."""
    lp = np.asarray(lp, F32)
    V1 = lp.shape[1]
    blank, n = V1 - 1, len(y)
    U = n if U is None else U
    frames, tok = _empty_result(U, -INF)
    if any(not 0 <= i < blank for i in y):
        tok[:n] = NAN
        return frames, tok, F32(NAN), Tb
    if Tb == 0:
        return frames, tok, F32(-INF), Tb
    read = lp[:Tb][:, [blank] + list(y)]
    if np.isnan(read).any():
        tok[:n] = NAN
        return frames, tok, F32(NAN), Tb
    S = 2 * n + 1
    lab = np.full(S, blank, np.int64)
    lab[1::2] = y
    skip = np.zeros(S, bool)
    skip[3::2] = np.asarray(y[1:], np.int64) != np.asarray(y[:-1], np.int64)
    v = np.full(S, -INF, F32)
    v[:2] = lp[0, lab[:2]]
    code = np.zeros((Tb, S), np.int8)
    ninf = np.array([-INF, -INF], F32)
    with np.errstate(invalid="ignore"):
        for t in range(1, Tb):
            best = v.copy()
            c1 = np.concatenate([ninf[:1], v[:-1]])
            m1 = c1 > best
            best[m1] = c1[m1]
            code[t, m1] = 1
            c2 = np.concatenate([ninf, v[:-2]])[:S]
            m2 = skip & (c2 > best)
            best[m2] = c2[m2]
            code[t, m2] = 2
            v = lp[t, lab] + best
    s = S - 1
    if S >= 2 and v[S - 2] > v[S - 1]:
        s = S - 2
    vit = v[s]
    if vit == -INF:
        return frames, tok, vit, Tb
    for t in range(Tb - 1, -1, -1):
        if s & 1:
            frames[s >> 1] = t
        if t > 0:
            s -= int(code[t, s])
    tok[:n] = lp[frames[:n], y]
    return frames, tok, vit, Tb


def rnnt_replay(blank, label, Tb, Ub, U=None):
    """Stage 2 of RNN-T for one utterance in numpy float32, walking the anti-diagonals as the kernel does (each node is one
    add per candidate, so the order of nodes does not change the bits).  blank / label [T, U+1] float32."""
    blank, label = np.asarray(blank, F32), np.asarray(label, F32)
    U = Ub if U is None else U
    frames, tok = _empty_result(U, -INF)
    if Tb == 0:
        return frames, tok, F32(-INF), Ub
    read_nan = (np.isnan(blank[:Tb - 1, :Ub + 1]).any() or np.isnan(label[:Tb, :Ub]).any() or np.isnan(blank[Tb - 1, Ub]))
    if read_nan:
        tok[:Ub] = NAN
        return frames, tok, F32(NAN), Tb + Ub
    v = np.full((Tb, Ub + 1), -INF, F32)
    take = np.zeros((Tb, Ub + 1), bool)
    v[0, 0] = 0
    with np.errstate(invalid="ignore"):
        for d in range(1, Tb + Ub):
            u = np.arange(max(0, d - (Tb - 1)), min(Ub, d) + 1)
            t = d - u
            tb, ul = np.maximum(t - 1, 0), np.maximum(u - 1, 0)
            cb = np.where(t > 0, v[tb, u] + blank[tb, u], F32(-INF)).astype(F32)
            cl = np.where(u > 0, v[t, ul] + label[t, ul], F32(-INF)).astype(F32)
            tk = (u > 0) & ((t == 0) | (cl > cb))
            v[t, u] = np.where(tk, cl, cb)
            take[t, u] = tk
    vit = v[Tb - 1, Ub] + blank[Tb - 1, Ub]
    if vit == -INF:
        return frames, tok, vit, Tb + Ub
    t, u = Tb - 1, Ub
    while t + u > 0:
        if take[t, u]:
            frames[u - 1] = t
            u -= 1
        else:
            t -= 1
    tok[:Ub] = label[frames[:Ub], np.arange(Ub)]
    return frames, tok, vit, Tb + Ub


# ------------------------------------------------------------------------------------------ float64 definitions
def ctc_forward64(lp, Tb, y):
    """log p(y | lp) over the CTC paths in float64, and the largest finite |f(t, s)| of every frame (for the bound)."""
    lp = np.asarray(lp, np.float64)
    blank, n = lp.shape[1] - 1, len(y)
    if Tb == 0:
        return -INF, []
    S = 2 * n + 1
    lab = np.full(S, blank, np.int64)
    lab[1::2] = y
    skip = np.zeros(S, bool)
    skip[3::2] = np.asarray(y[1:], np.int64) != np.asarray(y[:-1], np.int64)
    f = np.full(S, -INF)
    f[:2] = lp[0, lab[:2]]
    mags = [np.abs(f[np.isfinite(f)]).max(initial=0.0)]
    with np.errstate(invalid="ignore", divide="ignore"):
        for t in range(1, Tb):
            a = np.concatenate([[-INF], f[:-1]])
            b = np.where(skip, np.concatenate([[-INF, -INF], f[:-2]])[:S], -INF)
            f = np.logaddexp(np.logaddexp(f, a), b) + lp[t, lab]
            mags.append(np.abs(f[np.isfinite(f)]).max(initial=0.0))
    ll = np.logaddexp(f[S - 1], f[S - 2]) if S >= 2 else f[0]
    return float(ll), mags


def rnnt_forward64(blank, label, Tb, Ub):
    """log p(y | lattice) in float64 over the RNN-T paths, and the largest finite |f| of every anti-diagonal."""
    blank, label = np.asarray(blank, np.float64), np.asarray(label, np.float64)
    if Tb == 0:
        return -INF, []
    f = np.full((Tb, Ub + 1), -INF)
    f[0, 0] = 0.0
    mags = [0.0]
    with np.errstate(invalid="ignore"):
        for d in range(1, Tb + Ub):
            u = np.arange(max(0, d - (Tb - 1)), min(Ub, d) + 1)
            t = d - u
            tb, ul = np.maximum(t - 1, 0), np.maximum(u - 1, 0)
            a = np.where(t > 0, f[tb, u] + blank[tb, u], -INF)
            b = np.where(u > 0, f[t, ul] + label[t, ul], -INF)
            f[t, u] = np.logaddexp(a, b)
            fin = f[t, u][np.isfinite(f[t, u])]
            mags.append(np.abs(fin).max(initial=0.0))
    ll = f[Tb - 1, Ub] + blank[Tb - 1, Ub]
    return float(ll), mags


def ctc_forward_bound(mags, ll):
    """Error of the kernel's fp32 forward recursion against the float64 one on the same fp32 scores.  One frame of state s:
    lse3 = m + logf(sum of three expf(x - m)): each difference is rounded (an exponent error of at most |x - m| u on a term
    e^(x-m), and x e^-x <= 1/e), each expf is within 2 ulp (4u relative), the two adds of terms in [1, 3] give 2u, logf adds 2 ulp
    of a value below log 3 (4u), so the log term is off by at most 3 (4u + u/e) + 2u + 4u < 20u; the add of m and the add of lp
    round once each, at most u |f| apiece.  log-sum-exp is 1-Lipschitz in the max norm, so per-frame errors add up along t:
    sum_t (20 + 2 max_s |f(t, s)|) u, plus one final lse2 (at most 10u + u |ll|)."""
    return U32 * (sum(20.0 + 2.0 * m for m in mags) + 10.0 + abs(ll)) * 1.01


def rnnt_forward_bound(mags, ll):
    """As ctc_forward_bound for one RNN-T node: two candidate adds (u |f| each), lse2 = m + log1pf(expf(min - m)) with a rounded
    difference (u/e), expf (4u relative, so at most 4u absolute in log1p), log1pf (2 ulp of a value below log 2: 2u) and the add
    of m (u |f|): at most 8u + 3u |f| per anti-diagonal, summed along the T + U - 1 diagonals, plus the final add."""
    return U32 * (sum(8.0 + 3.0 * m for m in mags) + abs(ll)) * 1.01


# ------------------------------------------------------------------------------------------ CPU
def test_ctc_definition_in_float64_matches_ctc_loss():
    rng = np.random.default_rng(0)
    cases = [(30, [3, 1, 4, 1, 5]), (12, [2, 2, 2]), (5, [1, 1, 1]), (4, [1, 2, 3, 4, 5]), (9, []), (1, [7])]
    for T, y in cases:
        V1 = 9
        lp = torch.from_numpy(rng.standard_normal((T, V1)) * 2).log_softmax(-1)
        ll, _ = ctc_forward64(lp.numpy(), T, y)
        want = -F.ctc_loss(lp[:, None, :], torch.tensor([y], dtype=torch.long), torch.tensor([T]), torch.tensor([len(y)]),
                           blank=V1 - 1, reduction="none", zero_infinity=False)
        assert float(want) == pytest.approx(ll, abs=1e-9, rel=1e-12) or (ll == -INF and float(want) == -INF), (T, y)
    assert ctc_forward64(np.zeros((4, 9)), 4, [1, 2, 3, 4, 5])[0] == -INF        # infeasible: T < U
    assert ctc_forward64(np.zeros((3, 9)), 3, [1, 1, 2])[0] == -INF              # T < U + repeats
    assert ctc_forward64(np.zeros((4, 9)), 4, [1, 1, 2])[0] == 0.0               # exactly one path
    assert ctc_forward64(np.zeros((4, 9)), 0, [])[0] == -INF


def test_rnnt_definition_in_float64_matches_rnnt_loss():
    ta = pytest.importorskip("torchaudio.functional")
    rng = np.random.default_rng(1)
    for T, y in ((7, [1, 2, 2, 0]), (1, [3, 1]), (9, [4]), (5, [0, 1, 2, 3, 4, 5, 6, 7, 0])):
        V1 = 9
        lat = torch.from_numpy(rng.standard_normal((T, len(y) + 1, V1)) * 2).float().log_softmax(-1)
        blank = lat[..., V1 - 1].double().numpy()
        label = np.full((T, len(y) + 1), -INF)
        label[:, :len(y)] = lat[:, np.arange(len(y)), y].double().numpy()
        ll, _ = rnnt_forward64(blank, label, T, len(y))
        want = -ta.rnnt_loss(lat[None], torch.tensor([y], dtype=torch.int32), torch.tensor([T], dtype=torch.int32),
                             torch.tensor([len(y)], dtype=torch.int32), blank=V1 - 1, reduction="none", fused_log_softmax=False)
        assert float(want) == pytest.approx(ll, rel=1e-5, abs=1e-4), (T, y)
    # U = 0: the all-blank path
    blank = rng.standard_normal((6, 1))
    assert rnnt_forward64(blank, np.full((6, 1), -INF), 6, 0)[0] == pytest.approx(blank.sum(), abs=1e-12)
    assert rnnt_forward64(blank, np.full((6, 1), -INF), 0, 0)[0] == -INF


def test_replay_tie_rules_on_hand_built_scores():
    # CTC, all scores equal: staying wins every tie, so the path takes the label at frame 0 and stays in the final blank
    fr, tok, vit, rows = ctc_replay(np.zeros((4, 3), F32), 4, [1])
    assert fr.tolist() == [0] and tok.tolist() == [0.0] and vit == 0.0 and rows == 4
    # ... and between the two final states S - 1 wins a tie: token 0 ends the path only if strictly better
    lp = np.full((3, 3), -1.0, F32)
    fr, _, vit, _ = ctc_replay(lp, 3, [0, 1])
    assert fr.tolist() == [0, 1] and vit == F32(-3.0)
    # a label reached through the blank between two labels: frames are the first frame of each token's run
    lp = np.array([[0, -5, -1], [0, -5, 0], [-5, 0, -5], [-5, -5, 0]], F32)
    fr, tok, vit, _ = ctc_replay(lp, 4, [0, 1])
    assert fr.tolist() == [0, 2] and tok.tolist() == [0.0, 0.0] and vit == F32(0.0)
    # repeated labels need a blank between them
    fr, _, vit, _ = ctc_replay(np.zeros((3, 3), F32), 3, [1, 1])
    assert fr.tolist() == [0, 2] and vit == 0.0
    fr, tok, vit, _ = ctc_replay(np.zeros((2, 3), F32), 2, [1, 1])
    assert fr.tolist() == [-1, -1] and vit == -INF and np.all(tok == -INF)
    # RNN-T, all scores equal: the blank edge wins every tie, so every token is emitted at frame 0
    fr, tok, vit, rows = rnnt_replay(np.zeros((5, 4), F32), np.zeros((5, 4), F32), 5, 3)
    assert fr.tolist() == [0, 0, 0] and vit == 0.0 and rows == 8
    # a strictly better label edge is taken
    label = np.zeros((5, 4), F32)
    blank = np.full((5, 4), -1.0, F32)
    label[2, 1] = 1.0
    fr, _, _, _ = rnnt_replay(blank, label, 5, 3)
    assert fr[1] == 2
    # no path / NaN
    assert rnnt_replay(np.zeros((5, 4), F32), np.zeros((5, 4), F32), 0, 3)[0].tolist() == [-1, -1, -1]
    blank = np.zeros((5, 4), F32)
    blank[4, 0] = NAN                          # not read when U_b = 3: (T_b - 1, 0) has no blank edge out of it
    assert rnnt_replay(blank, np.zeros((5, 4), F32), 5, 3)[2] == 0.0
    blank[3, 0] = NAN                          # read
    assert math.isnan(rnnt_replay(blank, np.zeros((5, 4), F32), 5, 3)[2])


CHARS = [" ", "а", "б", "в", "е", "ж", "и", "к", "о"]


def test_tokenizer_encode_charwise_normalises_and_drops():
    tok = Tokenizer(CHARS)
    text = "  Ёжик\t\tИ  БОБЁР-7 "
    assert tok.normalize(text) == "ежик и бобе"
    assert tok.encode(text) == [CHARS.index(c) for c in "ежик и бобе"]
    assert tok.decode(tok.encode(text)) == tok.normalize(text)
    assert tok.encode("xyz") == [] and tok.encode("") == []


def test_tokenizer_encode_sentencepiece_round_trip(tmp_path):
    spm = pytest.importorskip("sentencepiece")
    corpus = tmp_path / "corpus.txt"
    lines = ["привет как дела", "все хорошо спасибо", "ежик в тумане", "где мой телефон", "сегодня хорошая погода"] * 40
    corpus.write_text("\n".join(lines), encoding="utf-8")
    spm.SentencePieceTrainer.train(input=str(corpus), model_prefix=str(tmp_path / "m"), vocab_size=32, model_type="unigram",
                                   character_coverage=1.0, minloglevel=2)
    tok = Tokenizer([], str(tmp_path / "m.model"))
    for text in ("Привет  как ДЕЛА", "Ёжик в  тумане", "сегодня", " где\tМОЙ телефон "):
        ids = tok.encode(text)
        assert ids == list(tok.model.encode(tok.normalize(text)))
        assert all(0 <= i < len(tok) for i in ids)
        assert tok.decode(ids) == tok.normalize(text)
    assert tok.normalize("Ёжик\n В  ТУМАНЕ ") == "ежик в тумане"


def test_alignment_record():
    w = [Word("аб", 0.0, 0.08, 0.5)]
    a = Alignment("аб", w, -1.5, 0.75)
    assert a == Alignment(text="аб", words=[Word("аб", 0.0, 0.08, 0.5)], log_likelihood=-1.5, confidence=0.75)
    assert a != Alignment("аб", None, -1.5, 0.75)
    assert repr(a) == ("Alignment(text='аб', words=[Word(text='аб', start=0.0, end=0.08, confidence=0.5)], "
                       "log_likelihood=-1.5, confidence=0.75)")
    assert str(a) == "аб" and Alignment("x", log_likelihood=0.0, confidence=1.0).words is None


def test_align_batch_refuses_bad_input_before_device_work():
    model = gigaam.load_model("v2_ctc", device="cpu", checkpoint=synthetic.synthetic_checkpoint("v2_ctc", n_layers=1))
    V = len(model.decoding.tokenizer)
    wav, lens = torch.zeros(2, 1600), torch.tensor([1600, 1600])
    with pytest.raises(ValueError, match="empty batch"):
        model.align_batch(torch.zeros(0, 1600), torch.zeros(0), [])
    with pytest.raises(ValueError, match="texts for a batch"):
        model.align_batch(wav, lens, ["а"])
    with pytest.raises(ValueError, match="outside"):
        model.align_batch(wav, lens, ["а", [0, V]])
    with pytest.raises(ValueError, match="outside"):
        model.align_batch(wav, lens, [[-1], "а"])
    with pytest.raises(ValueError, match="exceed"):
        model.align_batch(wav, lens, ["а", [1] * 4097])


# ------------------------------------------------------------------------------------------ GPU helpers
def _dev():
    return torch.device("cuda", 0)


_MODELS = {}


def _model(name):
    if name not in _MODELS:
        ck = synthetic.synthetic_checkpoint(name, seed=0, n_layers=1)
        _MODELS[name] = (gigaam.load_model(name, fp16_encoder=False, device=_dev(), checkpoint=ck), ck)
    return _MODELS[name]


def _check_ctc_batch(eng, lp, enc_len, targets, target_len, forward=True):
    """Run gam_ctc_align on host arrays and check every utterance against the replay (bit for bit) and float64 (bound)."""
    B, T, _ = lp.shape
    out = eng.ctc_align(torch.from_numpy(lp).to(_dev()), torch.tensor(enc_len), torch.from_numpy(targets), torch.tensor(target_len))
    fr, tok, vit, ll, rows = (t.cpu().numpy() for t in out)
    U = targets.shape[1]
    for b in range(B):
        Tb, Ub = min(max(enc_len[b], 0), T), target_len[b]
        y = targets[b, :Ub].tolist()
        r_fr, r_tok, r_vit, r_rows = ctc_replay(lp[b], Tb, y, U)
        assert np.array_equal(fr[b], r_fr), b
        assert np.array_equal(tok[b].view(np.uint32), r_tok.view(np.uint32)) or (np.isnan(r_tok).any() and np.array_equal(
            np.isnan(tok[b]), np.isnan(r_tok))), b
        assert np.array_equal(np.float32(vit[b]).view(np.uint32), F32(r_vit).view(np.uint32)) or (math.isnan(r_vit) and math.isnan(vit[b])), b
        assert rows[b] == r_rows
        if math.isnan(r_vit):
            assert math.isnan(ll[b])
        elif forward:
            want, mags = ctc_forward64(lp[b], Tb, y)
            if want == -INF:
                assert ll[b] == -INF
            else:
                assert abs(ll[b] - want) <= ctc_forward_bound(mags, want), (b, ll[b], want)
    return out


def _check_rnnt_batch(eng, blank, label, enc_len, target_len):
    B, T, U1 = blank.shape
    out = eng.rnnt_align(torch.from_numpy(blank).to(_dev()), torch.from_numpy(label).to(_dev()), torch.tensor(enc_len),
                         torch.tensor(target_len))
    fr, tok, vit, ll, rows = (t.cpu().numpy() for t in out)
    for b in range(B):
        Tb, Ub = min(max(enc_len[b], 0), T), target_len[b]
        r_fr, r_tok, r_vit, r_rows = rnnt_replay(blank[b], label[b], Tb, Ub, U1 - 1)
        assert np.array_equal(fr[b], r_fr), b
        assert np.array_equal(tok[b].view(np.uint32), r_tok.view(np.uint32)) or (np.isnan(r_tok).any() and np.array_equal(
            np.isnan(tok[b]), np.isnan(r_tok))), b
        assert np.array_equal(np.float32(vit[b]).view(np.uint32), F32(r_vit).view(np.uint32)) or (math.isnan(r_vit) and math.isnan(vit[b])), b
        assert rows[b] == r_rows
        if math.isnan(r_vit):
            assert math.isnan(ll[b])
        else:
            want, mags = rnnt_forward64(blank[b], label[b], Tb, Ub)
            if want == -INF:
                assert ll[b] == -INF
            else:
                assert abs(ll[b] - want) <= rnnt_forward_bound(mags, want), (b, ll[b], want)
    return out


def _log_probs(rng, shape, scale=3.0, ties=False):
    z = torch.from_numpy(rng.standard_normal(shape) * scale)
    if ties:
        z = torch.round(z)
    lp = z.log_softmax(-1).float().numpy()
    if ties:   # planted scores need not be normalised: quarter steps make exact ties common
        lp = (np.round(lp * 4) / 4).astype(F32)
    return lp


# ------------------------------------------------------------------------------------------ GPU: stage 2, CTC
@pytest.mark.gpu
@pytest.mark.parametrize("V1", [34, 257])
def test_ctc_stage2_ragged_batch_against_replay(V1):
    eng = _model("v2_ctc" if V1 == 34 else "v3_e2e_ctc")[0]._get_engine()
    rng = np.random.default_rng(V1)
    B, T, U = 12, 300, 100
    for ties in (False, True):
        lp = _log_probs(rng, (B, T, V1), ties=ties)
        targets = rng.integers(0, V1 - 1, (B, U)).astype(np.int32)
        targets[1, 10:20] = targets[1, 10]                              # repeats
        enc_len = [300, 250, 200, 120, 300, 40, 0, 300, 300, 300, 150, 301]
        target_len = [100, 60, 80, 100, 0, 50, 10, 30, 30, 30, 40, 20]
        lp[2, 5, :] = -INF                                              # a frame with no finite score
        lp[3, :, targets[3, 0]] = -INF                                  # the first token can never be emitted
        lp[7, 40, targets[7, 3]] = NAN                                  # NaN in a used entry
        lp[8, 250, :] = NAN                                             # NaN in frames past T_b ...
        enc_len[8] = 250
        unused = sorted(set(range(V1 - 1)) - set(targets[9, :30].tolist()))[0]
        lp[9, :, unused] = NAN                                          # ... and in a class the utterance never reads
        targets[10, 5] = V1 - 1                                         # blank is not a valid target id
        targets[11, 3] = -4
        out = _check_ctc_batch(eng, lp, enc_len, targets, target_len)
        vit = out[2].cpu()
        assert math.isnan(vit[7]) and math.isnan(vit[10]) and math.isnan(vit[11])
        assert math.isfinite(vit[8]) and math.isfinite(vit[9]) and vit[3] == -INF and vit[6] == -INF and vit[5] == -INF


@pytest.mark.gpu
def test_ctc_stage2_long_utterance_at_the_token_limit():
    eng = gigaam.load_model("v3_e2e_ctc", fp16_encoder=False, device=_dev(), max_encoded_frames=5000,
                            checkpoint=synthetic.synthetic_checkpoint("v3_e2e_ctc", seed=0, n_layers=1))._get_engine()
    rng = np.random.default_rng(7)
    T, U, V1 = 5000, 4096, 257
    lp = _log_probs(rng, (2, T, V1))
    targets = rng.integers(0, V1 - 1, (2, U)).astype(np.int32)
    _check_ctc_batch(eng, lp, [T, 4500], targets, [U, 2000])
    with pytest.raises(ValueError):
        eng.ctc_align(torch.zeros(1, T, V1, device=_dev()), torch.tensor([T]), torch.zeros(1, U + 1, dtype=torch.int32),
                      torch.tensor([U + 1]))


# ------------------------------------------------------------------------------------------ GPU: stage 2, RNN-T
def _rnnt_scores(rng, B, T, U1, ties=False):
    blank = -rng.exponential(1.0, (B, T, U1))
    label = -rng.exponential(1.0, (B, T, U1))
    if ties:
        blank, label = np.round(blank * 2) / 2, np.round(label * 2) / 2
    return blank.astype(F32), label.astype(F32)


@pytest.mark.gpu
def test_rnnt_stage2_ragged_batch_against_replay():
    eng = _model("v2_rnnt")[0]._get_engine()
    rng = np.random.default_rng(3)
    B, T, U = 10, 200, 70
    for ties in (False, True):
        blank, label = _rnnt_scores(rng, B, T, U + 1, ties)
        enc_len = [200, 150, 1, 0, 200, 100, 200, 200, 201, 180]
        target_len = [70, 30, 5, 4, 0, 70, 20, 20, 10, 40]
        if ties:
            blank[6], label[6] = 0.0, 0.0                                  # everything ties
        blank[5, 50, :] = -INF                                              # -inf edges
        label[5, :, 3] = -INF                                               # token 3 cannot be emitted: no path of finite score
        label[7, 10, 5] = NAN                                               # NaN in a used entry
        blank[1, 149, 0] = NAN                                              # unused: no blank edge out of (T_b - 1, 0)
        label[1, :, 30:] = NAN                                              # unused: past U_b
        blank[9, 179, 40] = NAN                                             # only the closing blank edge (T_b - 1, U_b)
        out = _check_rnnt_batch(eng, blank, label, enc_len, target_len)
        vit, tok = out[2].cpu(), out[1].cpu()
        assert math.isnan(vit[7]) and math.isfinite(vit[1]) and vit[3] == -INF and vit[5] == -INF
        assert math.isnan(vit[9]) and math.isnan(out[3][9]) and bool(tok[9, :40].isnan().all()) and bool((out[0][9] == -1).all())


@pytest.mark.gpu
def test_rnnt_stage2_long_utterances():
    eng = gigaam.load_model("v2_rnnt", fp16_encoder=False, device=_dev(), max_encoded_frames=5000,
                            checkpoint=synthetic.synthetic_checkpoint("v2_rnnt", seed=0, n_layers=1))._get_engine()
    rng = np.random.default_rng(4)
    blank, label = _rnnt_scores(rng, 2, 5000, 4097)
    _check_rnnt_batch(eng, blank, label, [5000, 3000], [4096, 1000])


# ------------------------------------------------------------------------------------------ GPU: stage 1, RNN-T
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_rnnt", "v3_e2e_rnnt"])
def test_rnnt_scores_bit_identical_to_the_lattice(name):
    model, _ = _model(name)
    eng = model._get_engine()
    V1 = eng.num_classes
    torch.manual_seed(0)
    for B, T, U in ((2, 37, 100), (3, 20, 1), (1, 9, 0)):
        enc = torch.randn(B, T, eng.d_model, device=_dev())
        targets = torch.randint(0, V1 - 1, (B, U), device=_dev())
        targets[0, :U // 2] = 1                                      # repeats
        x = torch.cat([torch.full((B, 1), V1 - 1, dtype=torch.int64, device=_dev()), targets], 1).contiguous()
        dec, _, _ = eng.rnnt_predict(x, None, None)
        lat = eng.rnnt_joint(enc, dec)
        blank, label = eng.rnnt_align_scores(enc, dec, targets)
        assert torch.equal(blank, lat[..., V1 - 1])
        gathered = lat[..., :U, :].gather(-1, targets[:, None, :, None].expand(B, T, U, 1))[..., 0]
        assert torch.equal(label[..., :U], gathered)
        assert bool((label[..., U] == -INF).all())
        if B > 1 and U > 1:   # an id outside [0, V) gives NaN in its own entries only, and reads no table row
            bad = targets.clone()
            bad[0, 1] = V1 - 1
            _, lab2 = eng.rnnt_align_scores(enc, dec, bad)
            assert bool(lab2[0, :, 1].isnan().all()) and torch.equal(lab2[0, :, 2:U], gathered[0, :, 2:])
            assert torch.equal(lab2[1:, :, :U], gathered[1:])


@pytest.mark.gpu
def test_rnnt_scores_beyond_2_31_lattice_elements_at_sampled_nodes():
    """T = 5000, U = 500 and V + 1 = 1025 give a lattice of 2.6e9 elements, which is never built.  Sampled nodes are compared
    with float64 from the same fp32 enc / dec.  Bound: the projections E = W_e enc + b_e and P = W_p dec + b_p are fp32 dot
    products, off by at most (K + 1) u (|W| |x| + |b|); the hidden h = relu(E + P) adds one rounding; each logit
    z = W_o h + b_o is off by |W_o| e_h + (J + 1) u (|W_o| |h| + |b_o|); log_softmax moves by at most 2 max_c e_z plus its own
    fp32 evaluation ((V + 16) u relative to the log-sum, and one rounding of the result)."""
    model = gigaam.load_model("v3_e2e_rnnt", fp16_encoder=False, device=_dev(), max_encoded_frames=5000,
                              checkpoint=synthetic.synthetic_checkpoint("v3_e2e_rnnt", seed=0, n_layers=1))
    eng = model._get_engine()
    sd = {k: v.double().cpu() for k, v in model.state_dict().items() if k.startswith("head.")}
    V1, T, U = eng.num_classes, 5000, 500
    short = _model("v3_e2e_rnnt")[0]._get_engine()        # the default limit of 768 frames refuses T = 769
    with pytest.raises(ValueError):
        short.rnnt_align_scores(torch.zeros(1, 769, eng.d_model, device=_dev()), torch.zeros(1, 1, eng.pred_hidden, device=_dev()),
                                torch.zeros(1, 0, dtype=torch.int32, device=_dev()))
    assert T * (U + 1) * V1 > 2 ** 31
    g = torch.Generator().manual_seed(5)
    enc = torch.randn(1, T, eng.d_model, generator=g).to(_dev())
    targets = torch.randint(0, V1 - 1, (1, U), generator=g).to(_dev())
    x = torch.cat([torch.full((1, 1), V1 - 1, device=_dev()), targets], 1).long().contiguous()
    dec, _, _ = eng.rnnt_predict(x, None, None)
    blank, label = eng.rnnt_align_scores(enc, dec, targets)
    We, be = sd["head.joint.enc.weight"], sd["head.joint.enc.bias"]
    Wp, bp = sd["head.joint.pred.weight"], sd["head.joint.pred.bias"]
    Wo, bo = sd["head.joint.joint_net.1.weight"], sd["head.joint.joint_net.1.bias"]
    e64, d64 = enc[0].double().cpu(), dec[0].double().cpu()
    ts = torch.randint(0, T, (64,), generator=g)
    us = torch.randint(0, U + 1, (64,), generator=g)
    ts[:2], us[:2] = torch.tensor([T - 1, 0]), torch.tensor([U, 0])
    J, d, H = We.shape[0], We.shape[1], Wp.shape[1]
    for t, u in zip(ts.tolist(), us.tolist()):
        E, P = e64[t] @ We.t() + be, d64[u] @ Wp.t() + bp
        eE = (d + 1) * U32 * (We.abs() @ e64[t].abs() + be.abs())
        eP = (H + 1) * U32 * (Wp.abs() @ d64[u].abs() + bp.abs())
        h = (E + P).clamp(min=0)
        eh = eE + eP + U32 * (E + P).abs()
        z = h @ Wo.t() + bo
        ez = Wo.abs() @ eh + (J + 1) * U32 * (Wo.abs() @ h.abs() + bo.abs())
        lp = z.log_softmax(-1)
        lse = float(torch.logsumexp(z, -1))
        tol = 2 * float(ez.max()) + (V1 + 16) * U32 * (1 + abs(lse))
        assert abs(float(blank[0, t, u]) - float(lp[V1 - 1])) <= tol + U32 * abs(float(lp[V1 - 1]))
        if u < U:
            k = int(targets[0, u])
            assert abs(float(label[0, t, u]) - float(lp[k])) <= tol + U32 * abs(float(lp[k]))


# ------------------------------------------------------------------------------------------ GPU: end to end
def _encoded(model, B=4, seconds=2.0, seed=11):
    wav, lens = synthetic.synthetic_audio(B, seconds, seed=seed, ragged=True)
    with torch.inference_mode():
        enc, enc_len = model(wav.to(_dev()), lens.to(_dev()))
    return wav, lens, enc, enc_len


def _pad(rows, U=None):
    U = max(len(r) for r in rows) if U is None else U
    t = torch.zeros((len(rows), U), dtype=torch.int32)
    for b, r in enumerate(rows):
        t[b, :len(r)] = torch.tensor(r, dtype=torch.int32)
    return t, torch.tensor([len(r) for r in rows], dtype=torch.int32)


def _ctc_lp64(enc, sd):
    W = sd["head.decoder_layers.0.weight"].double().cpu()[:, :, 0]
    b = sd["head.decoder_layers.0.bias"].double().cpu()
    x = enc.double().cpu().transpose(1, 2)
    z = x @ W.t() + b
    ez = (W.shape[1] + 1) * U32 * (x.abs() @ W.abs().t() + b.abs())
    return z, ez


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v3_e2e_ctc"])
def test_ctc_end_to_end(name):
    """decoding.align against float64 log-probs of the same encoder output.  Bound per frame: the logits are fp32 dot products
    (ez = (d + 1) u (|W| |x| + |b|)), so every log-prob is within 2 max_c ez + (V + 16) u (1 + |lse|) of float64 (as in
    test_rnnt_scores_beyond_2_31_lattice_elements_at_sampled_nodes); a path score sums T_b of them with one rounding per add."""
    model, ck = _model(name)
    wav, lens, enc, enc_len = _encoded(model)
    hyps = model.decoding.decode(model.head, enc, enc_len, return_scores=True)
    targets, tlen = _pad([h[1] for h in hyps])
    frames, tok, vit, ll, rows = (t.cpu() for t in decoding.align(model.head, enc, enc_len, targets, tlen))
    z, ez = _ctc_lp64(enc, ck["state_dict"])
    lp64 = z.log_softmax(-1)
    for b, h in enumerate(hyps):
        Tb, y = int(enc_len[b]), h[1]
        lse = torch.logsumexp(z[b, :Tb], -1)
        e_lp = 2 * ez[b, :Tb].max(-1).values + (z.shape[-1] + 16) * U32 * (1 + lse.abs())
        ll64, mags = ctc_forward64(lp64[b].numpy(), Tb, y)
        tol = float(e_lp.sum()) + ctc_forward_bound(mags, ll64)
        assert abs(float(ll[b]) - ll64) <= tol, (b, float(ll[b]), ll64, tol)
        assert int(rows[b]) == Tb == h[5]
        # the greedy path collapses to its own hypothesis: aligning it reproduces the greedy frames when every frame's
        # maximum is unique by more than the fp32 error of the log-probs
        top2 = z[b, :Tb].topk(2, -1).values
        if bool(((top2[:, 0] - top2[:, 1]) > 2 * e_lp).all()):
            assert frames[b, :len(y)].tolist() == h[2]
            assert abs(float(vit[b]) - h[4]) <= 2 * float(e_lp.sum()) + U32 * Tb * abs(h[4]), b
        assert float(vit[b]) <= float(ll[b]) + tol
    # the public call: words equal frames_to_words on the host from the same frames, confidences from token_logp
    _check_public_words(model, wav, lens, enc_len, hyps, frames, tok, vit, ll, rows)
    tokz = model.decoding.tokenizer
    text = " " + "".join(tokz.id_to_str(i) for i in hyps[0][1][:6]).upper() + "  "
    a = model.align(wav[0, :int(lens[0])], text)
    assert a.text == tokz.normalize(text) and len(a.words) <= 6 and math.isfinite(a.log_likelihood)


def _rnnt_lattice64(enc_b, dec_b, sd):
    """float64 blank / label entries from the same fp32 enc [T, d] / dec [U+1, H], and a per-entry error bound of the fp32
    stage 1 (see test_rnnt_scores_beyond_2_31_lattice_elements_at_sampled_nodes)."""
    We, be = sd["head.joint.enc.weight"], sd["head.joint.enc.bias"]
    Wp, bp = sd["head.joint.pred.weight"], sd["head.joint.pred.bias"]
    Wo, bo = sd["head.joint.joint_net.1.weight"], sd["head.joint.joint_net.1.bias"]
    e64, d64 = enc_b.double().cpu(), dec_b.double().cpu()
    E, P = e64 @ We.t() + be, d64 @ Wp.t() + bp
    eE = (We.shape[1] + 1) * U32 * (e64.abs() @ We.abs().t() + be.abs())
    eP = (Wp.shape[1] + 1) * U32 * (d64.abs() @ Wp.abs().t() + bp.abs())
    S = E[:, None, :] + P[None, :, :]
    h = S.clamp(min=0)
    eh = eE[:, None, :] + eP[None, :, :] + U32 * S.abs()
    z = h @ Wo.t() + bo
    ez = (eh @ Wo.abs().t() + (Wo.shape[1] + 1) * U32 * (h.abs() @ Wo.abs().t() + bo.abs())).amax(-1)
    lse = torch.logsumexp(z, -1)
    err = 2 * ez + (z.shape[-1] + 16) * U32 * (1 + lse.abs())
    return z.log_softmax(-1), err


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_rnnt", "v3_e2e_rnnt"])
def test_rnnt_end_to_end(name):
    """decoding.align against float64 entries of the same encoder output and prediction-network output.  Each entry is within
    err(t, u) of float64 (_rnnt_lattice64); a path adds T_b + U_b of them, so the forward score is within
    (T_b + U_b) max err + rnnt_forward_bound.  The Viterbi score is at least the fp32 sum, in path order, of any path's
    entries (rounding is monotone), in particular the greedy path's when it hit no max_symbols cap; and the greedy decoder's
    path_logp is the float64 sum of its own evaluation of the same rows, so viterbi_logp >= path_logp - bound."""
    model, ck = _model(name)
    eng = model._get_engine()
    sd = {k: v.double().cpu() for k, v in model.state_dict().items() if k.startswith("head.")}
    wav, lens, enc, enc_len = _encoded(model, B=3)
    hyps = model.decoding.decode(model.head, enc, enc_len, return_scores=True)
    targets, tlen = _pad([h[1] for h in hyps])
    frames, tok, vit, ll, rows = (t.cpu() for t in decoding.align(model.head, enc, enc_len, targets, tlen))
    V1 = eng.num_classes
    enc_btd = decoding._as_btd(enc)
    for b, h in enumerate(hyps):
        Tb, y = int(enc_len[b]), h[1]
        x = torch.tensor([[V1 - 1] + y], dtype=torch.int64, device=_dev())
        dec, _, _ = eng.rnnt_predict(x, None, None)
        lp64, err = _rnnt_lattice64(enc_btd[b, :Tb], dec[0], sd)
        blank64 = lp64[..., V1 - 1].numpy()
        label64 = np.full(blank64.shape, -INF)
        label64[:, :len(y)] = lp64[:, np.arange(len(y)), y].numpy()
        ll64, mags = rnnt_forward64(blank64, label64, Tb, len(y))
        emax = float(err.max())
        tol = (Tb + len(y)) * emax + rnnt_forward_bound(mags, ll64)
        assert abs(float(ll[b]) - ll64) <= tol, (b, float(ll[b]), ll64, tol)
        assert int(rows[b]) == Tb + len(y)
        # the greedy path is a path of the lattice when every frame closes with a blank
        capped = any(h[2].count(t) >= model.decoding.max_symbols for t in set(h[2]))
        if not capped:
            blank_d, label_d = eng.rnnt_align_scores(enc_btd[b:b + 1, :Tb].contiguous(), dec, x[:, 1:])
            bl, lb = blank_d[0].cpu().numpy(), label_d[0].cpu().numpy()
            s, u = F32(0), 0
            for t in range(Tb):
                while u < len(y) and h[2][u] == t:
                    s = F32(s + lb[t, u])
                    u += 1
                s = F32(s + bl[t, u])
            assert float(vit[b]) >= float(s)
            assert float(vit[b]) >= h[4] - 2 * int(h[5]) * emax - U32 * int(h[5]) * abs(h[4]), b
    _check_public_words(model, wav, lens, enc_len, hyps, frames, tok, vit, ll, rows)


def _check_public_words(model, wav, lens, enc_len, hyps, frames, tok, vit, ll, rows):
    """align_batch on the same audio with the hypotheses' ids: its words equal frames_to_words on the host from the frames
    of decoding.align, each word's confidence is exp(mean token_logp) over its tokens, and the record's scores are the
    device's."""
    res = model.align_batch(wav.to(_dev()), lens.to(_dev()), [h[1] for h in hyps])
    tokz = model.decoding.tokenizer
    for b, (a, h) in enumerate(zip(res, hyps)):
        n = len(h[1])
        shift = compute_frame_shift(int(lens[b]), int(enc_len[b]))
        want = frames_to_words(tokz, h[1], frames[b, :n].tolist(), shift)
        assert [(w.text, w.start, w.end) for w in a.words] == [(w.text, w.start, w.end) for w in want]
        assert a.text == tokz.decode(h[1]) and a.log_likelihood == float(ll[b])
        assert a.confidence == path_confidence(float(vit[b]), int(rows[b]))
        if len(a.words) == 1 and tokz.id_to_str(h[1][0]).strip():
            assert a.words[0].confidence == mean_logp_confidence(tok[b, :n].tolist())
        assert all(math.isfinite(w.confidence) for w in a.words)


# ------------------------------------------------------------------------------------------ GPU: batch independence, graphs
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v3_e2e_rnnt"])
def test_batch_independence_determinism_and_graph_replay(name):
    model, _ = _model(name)
    V = len(model.decoding.tokenizer)
    _, _, enc, enc_len = _encoded(model, B=8, seed=21)
    g = torch.Generator().manual_seed(2)
    tl = torch.randint(0, 25, (8,), generator=g)
    tl[3] = 0
    targets = torch.randint(0, V, (8, 25), generator=g, dtype=torch.int32)
    dev_args = (enc, enc_len, targets.to(_dev()), tl.to(_dev(), torch.int32))
    full = [t.clone() for t in decoding.align(model.head, *dev_args)]
    again = decoding.align(model.head, *dev_args)
    assert all(torch.equal(a, b) for a, b in zip(full, again))
    for b in (0, 3, 7):
        Ub = int(tl[b])
        one = decoding.align(model.head, enc[b:b + 1], enc_len[b:b + 1], targets[b:b + 1, :max(Ub, 1)].to(_dev()),
                             tl[b:b + 1].to(_dev(), torch.int32))
        assert torch.equal(one[0][0, :Ub], full[0][b, :Ub]) and torch.equal(one[1][0, :Ub], full[1][b, :Ub])
        for k in (2, 3, 4):
            assert torch.equal(one[k][0], full[k][b]), (b, k)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        decoding.align(model.head, *dev_args)          # warm-up: workspaces exist before capture
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            captured = decoding.align(model.head, *dev_args)
    torch.cuda.current_stream().wait_stream(stream)
    for t in captured:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(full, captured))
