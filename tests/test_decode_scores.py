"""Scored greedy decoding (gam_ctc_greedy_scored, gam_rnnt_greedy_scored): token log-probabilities, path log-probability
and word / utterance confidence.

The definitions (include/gigaam_b200.h, INTEGRATION.md "Confidence"): a decision row is one logit row the greedy rule
evaluates (CTC: every frame t < len; RNN-T: every joint row of gigaam/decoding.py:184-205, emissions and blanks alike).
l(row) = log_softmax(row)[label] for the label the greedy rule picks, NaN on a row with a NaN or +inf logit or only -inf
logits.  token_logp = l of the row that emitted the token (CTC: the first frame of its run), path_logp = sum of l over
all decision rows, path_rows = their count.  Word.confidence = exp(mean token_logp over the word), utterance / segment
confidence = exp(path_logp / path_rows).

CPU: a float64 statement of the definitions against torch, path rows and sums on oracle traces of hand-built rows
(a max_symbols cap hit, len = 0, non-finite rows), word confidence against a hand computation, and the records' repr / ==.

GPU: CTC through an engine with custom head weights and RNN-T through gam_test_rnnt_greedy_scored against float64 within
derived bounds; ids / frames / counts identical to the unscored kernels; non-finite rows; batch independence and
determinism; and the public API (transcribe / transcribe_longform with confidence=True, and a CUDA-graph replay)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, synthetic
from gigaam_b200.decoding import Tokenizer
from gigaam_b200.timestamps_utils import mean_logp_confidence, path_confidence, words_from_device
from gigaam_b200.types import LongformTranscriptionResult, Segment, TranscriptionResult, Word
from oracle import gigaam_oracle as orc
from test_greedy_decisions import H, JOINT_TIE, T_SWEEP, _dev_weights, _oracle_setup, make_encproj, make_lens, make_weights

U32 = 2.0 ** -24        # unit roundoff of fp32
INF, NAN = float("inf"), float("nan")


# ------------------------------------------------------------------------------------------ float64 definitions
def ell(z, label):
    """l(row) in float64: log_softmax(row)[label] on a finite row, NaN otherwise."""
    z = np.asarray(z, dtype=np.float64)
    if not np.isfinite(z).all():
        return NAN
    m = z.max()
    return float(z[label] - m - np.log(np.exp(z - m).sum()))


def greedy_label(z):
    """The decision contract: first maximal index of a finite row, 0 otherwise."""
    z = np.asarray(z, dtype=np.float64)
    return int(z.argmax()) if np.isfinite(z).all() else 0


def ctc_scores(z, L):
    """float64 CTC scoring of one utterance's [T, V1] logits over t < L: (ids, frames, token l, path sum, rows)."""
    blank = z.shape[1] - 1
    labels = [greedy_label(z[t]) for t in range(z.shape[0])]
    ids, frames, tok = [], [], []
    path = 0.0
    for t in range(L):
        lab = labels[t]
        path += ell(z[t], lab)
        if lab != blank and (t == 0 or lab != labels[t - 1]):
            ids.append(lab)
            frames.append(t)
            tok.append(ell(z[t], lab))
    return ids, frames, tok, path, L


def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def rnnt_scores(W, encproj, L, max_symbols, ids, frames):
    """Walk the reference's greedy rule for one utterance in float64 along the trace (ids, frames) and score it:
    ([(token l, row logits)] per emission, [row logits] of every decision row)."""
    emb_gates, whhT, wpT, bp, wo, bo = (np.asarray(W[k], dtype=np.float64) for k in ("emb_gates", "whhT", "wpT", "bp", "wo", "bo"))
    blank = wo.shape[0] - 1
    n = len(ids)

    def lstm(label, h, c):
        i, f, g, o = np.split(emb_gates[label] + h @ whhT, 4)
        c2 = _sig(f) * c + _sig(i) * np.tanh(g)
        return _sig(o) * np.tanh(c2), c2

    hn, cn = lstm(blank, np.zeros(H), np.zeros(H))
    pg = hn @ wpT + bp
    pos = 0
    rows, emitted = [], []
    with np.errstate(invalid="ignore", over="ignore"):
        for t in range(L):
            for _ in range(max_symbols):
                z = np.asarray(encproj[t], dtype=np.float64) + pg
                z = wo @ np.where(z < 0, 0.0, z) + bo
                k = ids[pos] if pos < n and frames[pos] == t else blank
                rows.append((z, k))
                if k == blank:
                    break
                emitted.append(len(rows) - 1)
                pos += 1
                hn, cn = lstm(k, hn, cn)
                pg = hn @ wpT + bp
    assert pos == n
    return rows, emitted


def lse_eval_bound(z, runs):
    """Bound on the error of evaluating -log sum_c exp(z_c - z_max) in fp32 the kernels' way, relative to the exact value
    on the same fp32 logits: every term gets one expf (2 ulp) of a rounded difference (relative error |x| u, at most X u
    in the exp-weighted average, X = z_max - z_min), a running sum is rescaled at most `runs` times by an expf and a
    multiply (each (X + 4) u), two folds add an expf, a multiply and an add each, and the sum of V1 positive terms adds
    (V1 + 8) u; logf adds 2 ulp of the result."""
    z = np.asarray(z, dtype=np.float64)
    X = float(z.max() - z.min())
    lse = float(np.log(np.exp(z - z.max()).sum()))
    rel = U32 * ((X + 4) * (runs + 2) + 2 * X + len(z) + 8)
    return rel / (1 - rel) + 2 * U32 * lse


# ------------------------------------------------------------------------------------------ CPU
def test_definitions_in_float64_match_torch():
    rng = np.random.default_rng(0)
    for V1 in (2, 5, 34, 257):
        for scale in (0.01, 1.0, 30.0):
            z = rng.standard_normal(V1) * scale
            k = greedy_label(z)
            want = float(torch.log_softmax(torch.from_numpy(z), -1)[k])
            assert ell(z, k) == pytest.approx(want, abs=1e-12)
            assert ell(z, k) <= 0.0
            assert int(torch.from_numpy(z).log_softmax(-1).argmax()) == k
    for row in ([0.0, NAN, 1.0], [0.0, INF, 1.0], [-INF, -INF, -INF], [INF, NAN, -INF]):
        assert greedy_label(row) == int(torch.tensor(row).log_softmax(-1).argmax()) == 0
        assert math.isnan(ell(row, 0)) and bool(torch.tensor(row, dtype=torch.float64).log_softmax(-1)[0].isnan())
    assert path_confidence(-3.0, 0) != path_confidence(-3.0, 0)          # NaN for a path without rows
    assert path_confidence(-3.0, 6) == pytest.approx(math.exp(-0.5), rel=1e-15)


def _ctc_sd(V1, D=4):
    ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1)
    sd = dict(ck["state_dict"])
    w = torch.zeros(V1, D, 1)
    w[:, :, 0] = torch.eye(V1, D)
    sd["head.decoder_layers.0.weight"], sd["head.decoder_layers.0.bias"] = w, torch.zeros(V1)
    return sd


def test_ctc_oracle_traces_hand_built_rows():
    """Head = identity, so every frame's logits are the hand-built encoder column: the oracle's trace, its rows and the
    path sum, including a repeated label (one token, two rows), blank frames, len = 0, len < T and a NaN frame."""
    V1, T = 4, 6                                   # blank = 3
    rows = np.array([[2.0, 0, 0, 0], [2.0, 0, 0, 0], [0, 0, 0, 5.0], [0, 1.5, 1.0, 0], [0, 0, 3.0, 0], [9.0, 0, 0, 0]])
    enc = torch.from_numpy(np.stack([rows.T, rows.T, rows.T])).float()
    enc[2, :, 3] = NAN
    lens = torch.tensor([6, 0, 5])
    sd = _ctc_sd(V1)
    hyps = orc.ctc_greedy(enc, lens, sd)
    assert hyps[0] == ([0, 1, 2, 0], [0, 3, 4, 5]) and hyps[1] == ([], [])
    z = enc.double().transpose(1, 2).numpy()
    l = [ell(z[0, t], greedy_label(z[0, t])) for t in range(T)]
    hand = [2 - math.log(math.exp(2) + 3), 2 - math.log(math.exp(2) + 3), 5 - math.log(math.exp(5) + 3),
            1.5 - math.log(math.exp(1.5) + math.exp(1) + 2), 3 - math.log(math.exp(3) + 3), 9 - math.log(math.exp(9) + 3)]
    assert l == pytest.approx(hand, abs=1e-12)
    for b in range(3):
        ids, frames, tok, path, n = ctc_scores(z[b], int(lens[b]))
        assert (ids, frames) == hyps[b] and n == int(lens[b])
        if b == 0:
            assert tok == pytest.approx([hand[0], hand[3], hand[4], hand[5]], abs=1e-12)
            assert path == pytest.approx(sum(hand), abs=1e-12)
        if b == 1:
            assert path == 0.0 and math.isnan(path_confidence(path, n))
        if b == 2:      # frame 3 is NaN: label 0 (a token), l NaN there and on the path
            assert ids[-2:] == [0, 2] and frames[-2:] == [3, 4] and math.isnan(tok[-2]) and math.isnan(path)
            assert not any(math.isnan(x) for x in tok[:-2] + tok[-1:])


@pytest.mark.parametrize("max_symbols", [1, 2, 10])
def test_rnnt_oracle_traces_rows_and_path(max_symbols):
    """On the oracle's traces: a frame with k < max_symbols tokens has k + 1 decision rows, a frame that hits the cap has
    max_symbols (no closing blank), len = 0 has none; the path sum is the sum of l over exactly those rows."""
    sd, W, enc, encproj, lens = _oracle_setup(seed=5 + max_symbols)
    hyps = orc.rnnt_greedy(enc, torch.from_numpy(lens), sd, max_symbols=max_symbols)
    capped = 0
    for b, (ids, frames) in enumerate(hyps):
        L = int(lens[b])
        per = np.bincount(np.asarray(frames, dtype=np.int64), minlength=L)[:L] if L else np.zeros(0, np.int64)
        want_rows = int(sum(k if k == max_symbols else k + 1 for k in per))
        capped += int((per == max_symbols).sum())
        rows, emitted = rnnt_scores(W, encproj[b], L, max_symbols, ids, frames)
        assert len(rows) == want_rows and len(emitted) == len(ids)
        assert all(k == greedy_label(z) or z.max() - z[k] < JOINT_TIE for z, k in rows)
        path = sum(ell(z, k) for z, k in rows)
        assert path <= 0.0
        if L == 0:
            assert rows == [] and path == 0
    assert capped > 0 and (lens == 0).any()


def test_word_confidence_host_code_against_hand_computation():
    tok = Tokenizer([" ", "a", "b", "c"])
    ids = [1, 2, 0, 3, 1, 0, 2]
    logp = [-0.1, -0.3, -2.0, -0.05, -0.25, -1.0, -0.7]
    words = words_from_device(tok, ids, [0, 3, 6], [2, 5, 7], [0, 3, 6], [2, 2, 1], 0.04, logp)
    assert [w.text for w in words] == ["ab", "ca", "b"]
    assert [w.confidence for w in words] == pytest.approx([math.exp(-0.2), math.exp(-0.15), math.exp(-0.7)], rel=1e-15)
    assert all(w.confidence is None for w in words_from_device(tok, ids, [0], [2], [0], [2], 0.04))
    assert math.isnan(mean_logp_confidence([-0.1, NAN])) and math.isnan(mean_logp_confidence([]))


def test_records_repr_and_equality_with_confidence():
    w = Word("hi", 0.0, 0.5)
    assert repr(w) == "Word(text='hi', start=0.0, end=0.5)" and w.confidence is None
    wc = Word("hi", 0.0, 0.5, confidence=0.75)
    assert repr(wc) == "Word(text='hi', start=0.0, end=0.5, confidence=0.75)"
    assert w != wc and wc == Word(text="hi", start=0.0, end=0.5, confidence=0.75) and wc != Word("hi", 0.0, 0.5, 0.7)
    r = TranscriptionResult(text="hi")
    assert repr(r) == "TranscriptionResult(text='hi', words=None)" and str(r) == "hi"
    rc = TranscriptionResult(text="hi", confidence=0.5)
    assert repr(rc) == "TranscriptionResult(text='hi', words=None, confidence=0.5)" and rc != r
    s = Segment("hi", 0.0, 1.0)
    assert repr(s) == "Segment(text='hi', start=0.0, end=1.0, words=None)"
    sc = Segment("hi", 0.0, 1.0, None, 0.25)
    assert repr(sc).endswith("confidence=0.25)") and sc != s and sc == Segment("hi", 0.0, 1.0, confidence=0.25)
    lf = LongformTranscriptionResult(segments=[sc])
    assert lf.text == "hi" and lf.segments[0].confidence == 0.25


# ------------------------------------------------------------------------------------------ GPU plumbing
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (there is no CPU fallback to test instead)"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def eng(dev):
    from gigaam_b200.engine import Engine
    ck = synthetic.synthetic_checkpoint("v2_rnnt", seed=0, n_layers=1)
    return Engine(ck["cfg"], ck["state_dict"], dev)


def _call(eng, fn, *args):
    ptrs = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    rc = getattr(eng.lib, fn)(eng.handle, *ptrs, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    _lib.check(eng.lib, eng.handle, rc, fn)


def run_rnnt(eng, Wd, V1, encproj, lens, max_symbols, scored=True):
    """gam_test_rnnt_greedy[_scored] -> dict of host arrays (ids, frames, counts[, token_logp, path_logp, path_rows], plan)."""
    dev = eng.device
    B, T, _ = encproj.shape
    max_out = T * max_symbols
    out = {k: torch.full((B, max_out), -7, dtype=torch.int32, device=dev) for k in ("ids", "frames")}
    out["counts"] = torch.full((B,), -7, dtype=torch.int32, device=dev)
    plan = (C.c_int32 * 7)()
    e = torch.from_numpy(np.ascontiguousarray(encproj, dtype=np.float32)).to(dev)
    ln = torch.from_numpy(np.asarray(lens, dtype=np.int32)).to(dev)
    args = [e, ln, *Wd, B, T, V1, max_symbols, max_out, out["ids"], out["frames"], out["counts"]]
    if scored:
        out["token_logp"] = torch.full((B, max_out), 7.0, dtype=torch.float32, device=dev)
        out["path_logp"] = torch.full((B,), 7.0, dtype=torch.float32, device=dev)
        out["path_rows"] = torch.full((B,), -7, dtype=torch.int32, device=dev)
        args += [out["token_logp"], out["path_logp"], out["path_rows"]]
    _call(eng, "gam_test_rnnt_greedy_scored" if scored else "gam_test_rnnt_greedy", *args, C.cast(plan, C.c_void_p))
    res = {k: v.cpu().numpy() for k, v in out.items()}
    res["plan"] = dict(zip(("NH", "GLOB", "rows_smem", "cls_per", "nu", "groups", "clusters"), list(plan)))
    return res


def _utt(res, b):
    """One utterance's (ids, frames, token_logp bits, path bits, rows) for bit comparisons."""
    n = int(res["counts"][b])
    return (res["ids"][b, :n].tolist(), res["frames"][b, :n].tolist(), res["token_logp"][b, :n].view(np.int32).tolist(),
            int(res["path_logp"][b:b + 1].view(np.int32)[0]), int(res["path_rows"][b]))


# ------------------------------------------------------------------------------------------ GPU: CTC
_CTC = {}


def _ctc_model(V1, dev):
    """A one-layer v2_ctc model with a custom head of V1 classes; columns 700-702 make non-finite rows (as in
    test_greedy_decisions: partial NaN, +inf from class 1 on, all -inf)."""
    if V1 not in _CTC:
        ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1)
        ck["cfg"]["head"]["num_classes"] = V1
        ck["cfg"]["decoding"]["vocabulary"] = [f"<{i}>" for i in range(V1 - 1)]
        rng = np.random.default_rng(V1)
        w = rng.standard_normal((V1, 768)) * 0.05
        b = rng.standard_normal(V1) * 0.5
        cls = np.arange(V1)
        w[:, 700] = np.where(cls % 2 == 0, 0.01, -0.01)
        w[V1 // 2, 700] = 0.0
        w[:, 701] = np.where(cls < 1, -0.01, 0.01)
        w[:, 702] = -np.abs(w[:, 702]) - 1e-4
        sd = ck["state_dict"]
        sd["head.decoder_layers.0.weight"] = torch.from_numpy(w.astype(np.float32)).unsqueeze(-1)
        sd["head.decoder_layers.0.bias"] = torch.from_numpy(b.astype(np.float32))
        model = gigaam.load_model("v2_ctc", fp16_encoder=False, device=dev, checkpoint=ck)
        _CTC[V1] = (model, sd)
    return _CTC[V1]


def _ctc_inputs(V1, sd, B, T, seed):
    """Encoder rows from near-ties to confident: 0.05 noise plus alpha * W[target] with alpha in {0, 0.3, 1, 3}, features
    700-702 kept at 0 so that only the planted non-finite rows are non-finite."""
    W = sd["head.decoder_layers.0.weight"][..., 0]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, 768, generator=g) * 0.05
    target = torch.randint(0, V1, (B, T), generator=g)
    alpha = torch.tensor([0.0, 0.3, 1.0, 3.0])[torch.randint(0, 4, (B, T), generator=g)]
    x += alpha[..., None] * W[target]
    x[..., 700:703] = 0
    return x


def _ctc_run(eng, x, lens, scores):
    out = eng.greedy(x, lens, scores=scores)
    torch.cuda.synchronize()
    return [t.cpu() for t in out]


def _ctc_bound(x, W, bias, labels):
    """Per-row bound of |l_kernel - l_float64| and l in float64: the fp32 dot-product bound gamma_{D+1} (sum |w x| + |b|)
    per logit (twice: the label's logit and the log-sum-exp move by at most the largest), plus the evaluation bound with
    as many rescales as the longest run of new maxima in one class group of 9-class slices of 36-class tiles."""
    D = x.shape[-1]
    gam = (D + 1) * U32 / (1 - (D + 1) * U32)
    xd, Wd, bd = x.double(), W.double(), bias.double()
    z = (xd @ Wd.T + bd).numpy()
    A = (xd.abs() @ Wd.abs().T + bd.abs()).numpy()
    V1 = z.shape[-1]
    group = (np.arange(V1) % 36) // 9
    B, T = labels.shape
    tol = np.zeros((B, T))
    l64 = np.zeros((B, T))
    for b in range(B):
        for t in range(T):
            row = z[b, t]
            l64[b, t] = ell(row, int(labels[b, t]))
            if not np.isfinite(row).all():
                continue
            E = gam * A[b, t].max()
            runs = 0
            for gi in range(4):
                best, n = -INF, 0
                for v in row[group == gi]:
                    if v > best - 2 * E:
                        n += 1
                    best = max(best, v)
                runs = max(runs, n)
            tol[b, t] = 2 * E + lse_eval_bound(row, runs)
    return l64, tol


@pytest.mark.gpu
@pytest.mark.parametrize("V1", [34, 100, 257])
def test_ctc_scores_against_float64(dev, V1):
    model, sd = _ctc_model(V1, dev)
    eng = model._get_engine()
    B, T = 6, 64
    x = _ctc_inputs(V1, sd, B, T, V1)
    lens = torch.tensor([T, 0, 1, T, 37, 50], dtype=torch.int32)
    xd, ld = x.to(dev).contiguous(), lens.to(dev)
    ids0, fr0, cn0 = _ctc_run(eng, xd, ld, False)
    ids, fr, cn, tok, path, rows = _ctc_run(eng, xd, ld, True)
    labels = eng._ws_dec.peek((B, T))[: B * T * 4].view(torch.int32).view(B, T).cpu().numpy()
    assert torch.equal(cn, cn0)
    for b in range(B):
        n = int(cn[b])
        assert torch.equal(ids[b, :n], ids0[b, :n]) and torch.equal(fr[b, :n], fr0[b, :n])
    assert torch.equal(rows, lens)
    W, bias = sd["head.decoder_layers.0.weight"][..., 0], sd["head.decoder_layers.0.bias"]
    l64, tol = _ctc_bound(x, W, bias, labels)
    assert tol.max() < 1e-3, tol.max()
    worst = 0.0
    for b in range(B):
        n, L = int(cn[b]), int(lens[b])
        f = fr[b, :n].numpy()
        got = tok[b, :n].double().numpy()
        err = np.abs(got - l64[b, f])
        assert (err <= tol[b, f]).all(), (b, err.max(), tol[b, f].max())
        worst = max(worst, float((err / np.maximum(tol[b, f], 1e-30)).max(initial=0)))
        want_path = l64[b, :L].sum()
        assert abs(float(path[b]) - want_path) <= tol[b, :L].sum() + abs(want_path) * U32 + 1e-12, (b, float(path[b]), want_path)
        if L == 0:
            assert float(path[b]) == 0.0
    live = lens.numpy()[:, None] > np.arange(T)[None]
    ls = l64[live]
    zs = np.sort((x.double() @ W.double().T + bias.double()).numpy()[live], -1)
    near = int((zs[:, -1] - zs[:, -2] < 0.05).sum())
    print(f"V1={V1}: worst error / bound {worst:.3g}, bound max {tol.max():.3g}, l in [{ls.min():.3g}, {ls.max():.3g}], "
          f"{near} near ties")
    assert near > 0 and math.exp(ls.max()) > 0.75        # near-tie rows and confident rows are both present


@pytest.mark.gpu
@pytest.mark.parametrize("V1", [34, 257])
def test_ctc_nonfinite_rows_batch_independence_and_determinism(dev, V1):
    model, sd = _ctc_model(V1, dev)
    eng = model._get_engine()
    B, T = 5, 48
    x = _ctc_inputs(V1, sd, B, T, 100 + V1)
    lens = torch.tensor([T, 40, 1, T, 0], dtype=torch.int32)
    keys = ("ids", "frames", "counts", "token_logp", "path_logp", "path_rows")
    res = {k: v.numpy() for k, v in zip(keys, _ctc_run(eng, x.to(dev), lens.to(dev), True))}
    again = {k: v.numpy() for k, v in zip(keys, _ctc_run(eng, x.to(dev), lens.to(dev), True))}
    assert all(_utt(again, b) == _utt(res, b) for b in range(B))      # entries past counts[b] are not defined
    for b in range(B):      # alone, and in a batch of a different size and order
        one = {k: v.numpy() for k, v in zip(res, _ctc_run(eng, x[b:b + 1].to(dev), lens[b:b + 1].to(dev), True))}
        assert _utt(one, 0) == _utt(res, b), b
    perm = [3, 0, 4, 1, 2, 0]
    mix = {k: v.numpy() for k, v in zip(res, _ctc_run(eng, x[perm].to(dev), lens[perm].to(dev), True))}
    assert all(_utt(mix, i) == _utt(res, b) for i, b in enumerate(perm))
    bad = x.clone()
    bad[0, 5] = NAN
    bad[0, 9, 701] = INF
    bad[1, 7, 700] = INF
    bad[1, 45, 702] = INF          # beyond len = 40: not a decision row
    bad_rows = {(0, 5), (0, 9), (1, 7)}
    out = {k: v.numpy() for k, v in zip(res, _ctc_run(eng, bad.to(dev), lens.to(dev), True))}
    for b in (0, 1):
        n = int(out["counts"][b])
        fr, tl = out["frames"][b, :n], out["token_logp"][b, :n]
        assert np.array_equal(np.isnan(tl), np.array([(b, int(f)) in bad_rows for f in fr])), b
        assert any((b, int(f)) in bad_rows for f in fr)
        assert math.isnan(float(out["path_logp"][b]))
    for b in (2, 3, 4):
        assert _utt(out, b) == _utt(res, b), b


# ------------------------------------------------------------------------------------------ GPU: RNN-T
@pytest.fixture(scope="module")
def geometry(eng, dev):
    """The scored kernel's launch geometry probed on the device with all lengths 0: the NH = 1 / 2 batch switch,
    resident clusters, and per NH the largest V1 whose class rows all fit in shared memory next to the scored state."""
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    b_switch = 4 * max(1, sms // 16 - 2)
    Vmax = 8192
    Wz = {k: np.zeros_like(v) for k, v in make_weights(2, 0).items()}
    Wz["emb_gates"] = np.zeros((Vmax, 4 * H), np.float32)
    Wz["wo"] = np.zeros((Vmax, H), np.float32)
    Wz["bo"] = np.zeros(Vmax, np.float32)
    Wd = _dev_weights(Wz, dev)

    def plan(V1, B):
        return run_rnnt(eng, Wd, V1, np.zeros((B, 1, H), np.float32), np.zeros(B, np.int32), 1)["plan"]

    out = dict(b_switch=b_switch, clusters=plan(2, 400)["clusters"])
    for nh, B in ((1, 1), (2, b_switch + 1)):
        assert plan(2, B)["NH"] == nh and plan(2, B)["GLOB"] == 0 and plan(Vmax, B)["GLOB"] == 1
        lo, hi = 2, Vmax
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if plan(mid, B)["GLOB"]:
                hi = mid
            else:
                lo = mid
        out[f"last_smem_{nh}"] = lo
        rs = plan(lo + 1, B)["rows_smem"]
        out[f"l2_gt32_{nh}"] = 16 * (rs + 40) + 1
    print("scored geometry:", out)
    return out


def _check_rnnt_case(W, enc, lens, ms, res, what):
    """Every emission's l and every path against the float64 replay: per row 2 JOINT_TIE (the logits' fp32 error the
    decision replay allows) plus the log-sum-exp evaluation bound with one rescale per class of the busiest warp."""
    V1 = W["wo"].shape[0]
    runs = -(-(-(-V1 // 16)) // 16) + 1
    stats = dict(rows=0, worst=0.0, bound=0.0)
    for b in range(enc.shape[0]):
        n = int(res["counts"][b])
        ids, frames = res["ids"][b, :n].tolist(), res["frames"][b, :n].tolist()
        rows, emitted = rnnt_scores(W, enc[b], int(lens[b]), ms, ids, frames)
        assert int(res["path_rows"][b]) == len(rows), (what, b)
        tols = [2 * JOINT_TIE + (lse_eval_bound(z, runs) if np.isfinite(z).all() else 0) for z, _ in rows]
        ls = [ell(z, k) for z, k in rows]
        for i, r in enumerate(emitted):
            got = float(res["token_logp"][b, i])
            if math.isnan(ls[r]):
                assert math.isnan(got), (what, b, i)
            else:
                assert abs(got - ls[r]) <= tols[r], (what, b, i, got, ls[r], tols[r])
        path = float(res["path_logp"][b])
        want = sum(ls)
        if math.isnan(want):
            assert math.isnan(path), (what, b)
        else:
            assert abs(path - want) <= sum(tols) + abs(want) * U32, (what, b, path, want)
        stats["rows"] += len(rows)
        stats["bound"] = max([stats["bound"]] + tols)
    return stats


@pytest.mark.gpu
def test_rnnt_scores_sweep_against_float64(eng, dev, geometry):
    g = geometry
    vs = sorted({2, 17, 34, 257, 1025, 4097, g["last_smem_1"], g["last_smem_1"] + 1, g["last_smem_2"], g["last_smem_2"] + 1,
                 g["l2_gt32_1"], g["l2_gt32_2"]})
    bs = g["b_switch"]
    b_ragged = 8 * g["clusters"] + 3
    nh1_B, nh2_B = [1, bs - 1, bs], [bs + 1, b_ragged]
    cases = []
    for i, V1 in enumerate(vs):
        cases.append((V1, nh1_B[i % 3], (1, 2, 10)[i % 3], 1))
        cases.append((V1, nh2_B[i % 2], (10, 1, 2)[i % 3], 2))
    paths, rows = set(), 0
    for ci, (V1, B, ms, nh) in enumerate(cases):
        W = make_weights(V1, V1)
        Wd = _dev_weights(W, dev)
        enc, lens = make_encproj(B, T_SWEEP, 3000 + ci), make_lens(B, T_SWEEP, 3000 + ci)
        res = run_rnnt(eng, Wd, V1, enc, lens, ms)
        plain = run_rnnt(eng, Wd, V1, enc, lens, ms, scored=False)
        plan = res["plan"]
        assert plan["NH"] == nh and plan["GLOB"] == int(V1 > g[f"last_smem_{nh}"]), (V1, B, plan)
        l2 = plan["cls_per"] - plan["rows_smem"]
        paths.add((nh, plan["GLOB"], "L2>32" if l2 > 32 else ("L2>0" if l2 > 0 else "smem")))
        assert np.array_equal(res["counts"], plain["counts"])
        for b in range(B):
            n = int(res["counts"][b])
            assert np.array_equal(res["ids"][b, :n], plain["ids"][b, :n]) and np.array_equal(res["frames"][b, :n], plain["frames"][b, :n])
        rows += _check_rnnt_case(W, enc, lens, ms, res, (V1, B, ms))["rows"]
        for b in range(B):          # alone: the same bits
            one = run_rnnt(eng, Wd, V1, enc[b:b + 1], lens[b:b + 1], ms)
            assert _utt(one, 0) == _utt(res, b), (V1, B, ms, b)
        if ci % 4 == 0:             # repeated call: the same bits
            again = run_rnnt(eng, Wd, V1, enc, lens, ms)
            assert all(_utt(again, b) == _utt(res, b) for b in range(B))
    print("paths:", sorted(map(str, paths)), "rows:", rows)
    for want in ((1, 0, "smem"), (1, 1, "L2>32"), (2, 0, "smem"), (2, 1, "L2>32")):
        assert want in paths, want


@pytest.mark.gpu
@pytest.mark.parametrize("V1,nh", [(34, 1), (1025, 2)])
def test_rnnt_nonfinite_rows_scores(eng, dev, geometry, V1, nh):
    W = make_weights(V1, 7)
    wo = W["wo"]
    cls = np.arange(V1)
    wo[:, 1] = np.where(cls % 2 == 0, 0.3, -0.3)
    wo[:, 2] = np.where(cls % 3 == 0, -0.2, 0.2)
    wo[:, 3] = -np.abs(wo[:, 3]) - 1e-3
    wo[:, 5] = np.where(cls < 5, -0.3, 0.3)
    B = 5 if nh == 1 else geometry["b_switch"] + 3
    T = T_SWEEP
    clean = make_encproj(B, T, 190 + V1)
    lens = np.full(B, T, np.int32)
    bad = clean.copy()
    bad[0, 2, :] = NAN
    bad[1, 3, 1] = bad[1, 3, 2] = INF
    bad[2, 1, 3] = INF
    bad[3, 5, 5] = INF
    Wd = _dev_weights(W, dev)
    res = run_rnnt(eng, Wd, V1, bad, lens, 10)
    ref = run_rnnt(eng, Wd, V1, clean, lens, 10)
    assert res["plan"]["NH"] == nh
    _check_rnnt_case(W, bad, lens, 10, res, ("nonfinite", V1))
    for b in range(4):
        assert math.isnan(float(res["path_logp"][b])), b
        n = int(res["counts"][b])
        rows, emitted = rnnt_scores(W, bad[b], T, 10, res["ids"][b, :n].tolist(), res["frames"][b, :n].tolist())
        want_nan = [not np.isfinite(rows[r][0]).all() for r in emitted]
        assert np.array_equal(np.isnan(res["token_logp"][b, :n]), np.array(want_nan, dtype=bool)), b
    for b in range(4, B):
        assert _utt(res, b) == _utt(ref, b), b


# ------------------------------------------------------------------------------------------ GPU: public API
def _word_token_ranges(tok, ids):
    """Host grouping of token indices into words (timestamps_utils.frames_to_words' rule)."""
    words, cur, text = [], [], []
    for i, t in enumerate(ids):
        piece = tok.id_to_str(t)
        if piece == " " or piece.startswith("▁"):
            if "".join(text).strip():
                words.append(cur)
            cur, text = [], []
            if piece == " ":
                continue
            piece = piece[1:]
        cur.append(i)
        text.append(piece)
    if "".join(text).strip():
        words.append(cur)
    return words


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v2_rnnt", "v3_e2e_rnnt"])
def test_public_api_confidence(dev, name):
    ck = synthetic.synthetic_checkpoint(name, seed=0, n_layers=2)
    model = gigaam.load_model(name, device=dev, checkpoint=ck)
    wavs, lens = synthetic.synthetic_audio(4, 3.0, seed=11, ragged=True)
    segs = [wavs[i, : int(lens[i])] for i in range(4)]
    segs.append(segs[1].clone())                      # a repeated shape: the longform pipeline replays a CUDA graph
    tok = model.decoding.tokenizer
    alone = []
    for wav in segs:
        plain = model.transcribe(wav, word_timestamps=True)
        res = model.transcribe(wav, word_timestamps=True, confidence=True)
        assert res.text == plain.text and res.confidence is not None and 0.0 < res.confidence <= 1.0
        assert [(w.text, w.start, w.end) for w in res.words] == [(w.text, w.start, w.end) for w in plain.words]
        assert model.transcribe(wav, confidence=True).confidence == res.confidence
        with torch.inference_mode():
            w, n = model.prepare_wav(wav)
            enc, enc_len = model.forward(w, n)
            text, ids, frames, tl, path, rows = model.decoding.decode(model.head, enc, enc_len, return_scores=True)[0]
        assert text == res.text
        assert rows == int(enc_len[0]) if name.endswith("ctc") else rows >= int(enc_len[0])
        assert res.confidence == math.exp(path / rows)
        ranges = _word_token_ranges(tok, ids)
        assert len(ranges) == len(res.words)
        for word, r in zip(res.words, ranges):
            assert 0.0 < word.confidence <= 1.0
            assert word.confidence == pytest.approx(math.exp(float(np.mean([tl[i] for i in r]))), rel=1e-12, abs=0)
        alone.append(res)
    bounds, t0 = [], 0.0
    for s in segs:
        bounds.append((t0, t0 + s.numel() / 16000.0))
        t0 += s.numel() / 16000.0 + 0.5
    lf = model.transcribe_longform(None, word_timestamps=True, fr_batch_size=1, segments=segs, boundaries=bounds, confidence=True)
    for seg, one in zip(lf, alone):
        assert seg.text == one.text and seg.confidence == one.confidence
        assert [w.confidence for w in seg.words] == [w.confidence for w in one.words]
    lf0 = model.transcribe_longform(None, fr_batch_size=1, segments=segs, boundaries=bounds)
    assert [s.text for s in lf0] == [s.text for s in lf] and all(s.confidence is None for s in lf0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v2_rnnt"])
def test_graph_replay_of_scored_step_is_bit_identical(dev, name):
    from gigaam_b200.pipeline import BatchPipeline
    ck = synthetic.synthetic_checkpoint(name, seed=0, n_layers=2)
    model = gigaam.load_model(name, device=dev, checkpoint=ck)
    wavs, lens = synthetic.synthetic_audio(3, 2.5, seed=5, ragged=True)
    batches = [(wavs.clone().pin_memory(), lens.clone()) for _ in range(3)]
    eager = list(BatchPipeline(model, use_graph=False, with_words=True, with_scores=True).run_raw(iter(batches)))
    graph = list(BatchPipeline(model, use_graph=True, with_words=True, with_scores=True).run_raw(iter(batches)))
    assert len(eager) == len(graph) == 3
    for e, g in zip(eager, graph):
        assert len(e) == len(g) == 12
        counts = e[2]
        for i, (a, b) in enumerate(zip(e, g)):
            if i in (0, 1, 9):      # ids, frames, token_logp: the first counts[b] entries of every row are defined
                for r in range(a.shape[0]):
                    n = int(counts[r])
                    assert torch.equal(a[r, :n].view(torch.int32), b[r, :n].view(torch.int32)), (i, r)
            elif i in (4, 5, 6, 7):  # word records past n_words are not defined: compared through n_words
                continue
            else:
                assert torch.equal(a.view(torch.int32), b.view(torch.int32)), i
    assert not any(math.isnan(float(v)) for v in eager[0][10])
