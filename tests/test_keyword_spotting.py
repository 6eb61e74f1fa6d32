"""CTC keyword spotting: gam_ctc_spot (include/gigaam_b200.h has the definition), `decoding.spot`, `GigaAMASR.spot_batch` and
`GigaAMASR.spot` for recordings of any length (INTEGRATION.md §7g).

CPU: a float32 oracle of the definition, written line by line, checked against a float64 brute force that enumerates every
path on tiny inputs; the keyword checks and refusals, all before device work; the exported symbols.
GPU: bit identity with the oracle over vocabularies, keyword lengths, thresholds, ragged / empty / NaN recordings and
overflow past max_det; invariance to the batch, the keyword order and the warps per CTA; planted greedy paths; every greedy
word found where transcribe puts it; long recordings; refusals.
"""
import itertools
import math

import numpy as np
import pytest
import torch

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, decoding, synthetic
from gigaam_b200.longform import plan_windows, stitch_ctc_log_probs
from gigaam_b200.types import Detection

F32 = np.float32
NEG = F32(-np.inf)


# ------------------------------------------------------------------------------------------ the float32 oracle
def tau_of(U, threshold):
    """tau = fp32(U) * fp32(log threshold), the log taken on the fp32 threshold and rounded once."""
    return F32(U) * F32(np.log(np.float64(F32(threshold))))


def spot_frames(lp, Tb, y):
    """E(t) and a(t) for t < Tb (float32 / int arrays): the recursion of gam_ctc_spot, one fp32 operation at a time."""
    V1 = lp.shape[1]
    U = len(y)
    S = 2 * U - 1
    lab = np.array([y[s // 2] if s % 2 == 0 else V1 - 1 for s in range(S)])
    skip = np.array([s % 2 == 0 and s >= 2 and y[s // 2] != y[s // 2 - 1] for s in range(S)])
    v = np.full(S, NEG, F32)
    a = np.zeros(S, np.int64)
    E = np.full(Tb, NEG, F32)
    A = np.zeros(Tb, np.int64)
    for t in range(Tb):
        row = lp[t]
        if np.isnan(row).any():              # a barrier
            v = np.full(S, NEG, F32)
            a = np.full(S, t, np.int64)
        else:
            m = F32(row.max() + F32(0))     # exact; a zero max is +0
            c = (row[lab] - m).astype(F32)
            best, start = v.copy(), a.copy()
            c1 = np.concatenate([[NEG], v[:-1]]).astype(F32)
            a1 = np.concatenate([[0], a[:-1]])
            take = c1 > best                 # order s, s - 1, s - 2; strictly greater replaces
            best, start = np.where(take, c1, best), np.where(take, a1, start)
            c2 = np.concatenate([[NEG, NEG], v[:-2]])[:S].astype(F32)
            a2 = np.concatenate([[0, 0], a[:-2]])[:S]
            take = skip & (c2 > best)
            best, start = np.where(take, c2, best), np.where(take, a2, start)
            if F32(0) > best[0]:             # state 0: a fresh path starts at t; a tie continues
                best[0], start[0] = F32(0), t
            v = (c + best).astype(F32)
            a = start
        E[t], A[t] = v[S - 1], a[S - 1]
    return E, A


def scan(E, A, tau):
    """The detection scan: [(start, end, score)] in time order."""
    out, pend = [], None
    for t in range(len(E)):
        if not E[t] >= tau:
            continue
        if pend is not None and A[t] < pend[1]:
            if E[t] > pend[2]:
                pend = (int(A[t]), t + 1, E[t])
        else:
            if pend is not None:
                out.append(pend)
            pend = (int(A[t]), t + 1, E[t])
    if pend is not None:
        out.append(pend)
    return out


def spot_oracle(lp, enc_len, keywords, threshold, max_det, V, frames=None):
    """Outputs of gam_ctc_spot (start, end, score [B, K, max_det], count [B, K]) for lp [B, T, V+1] f32 and keywords as lists
    (a keyword with an id outside [0, V) or no tokens gets NaN rows and count 0).  `frames`: a dict that keeps spot_frames'
    results across thresholds."""
    frames = {} if frames is None else frames
    B, T, _ = lp.shape
    K = len(keywords)
    st = np.full((B, K, max_det), -1, np.int32)
    en = np.full((B, K, max_det), -1, np.int32)
    sc = np.full((B, K, max_det), NEG, F32)
    cnt = np.zeros((B, K), np.int32)
    for b in range(B):
        Tb = min(max(int(enc_len[b]), 0), T)
        for k, y in enumerate(keywords):
            if not 1 <= len(y) <= 64 or any(not 0 <= i < V for i in y):
                sc[b, k] = np.nan
                continue
            if (b, k) not in frames:
                frames[b, k] = spot_frames(lp[b], Tb, y)
            E, A = frames[b, k]
            dets = scan(E, A, tau_of(len(y), threshold))
            cnt[b, k] = len(dets)
            for i, (s, e, x) in enumerate(dets[:max_det]):
                st[b, k, i], en[b, k, i], sc[b, k, i] = s, e, x
    return st, en, sc, cnt


# ------------------------------------------------------------------------------------------ CPU: oracle vs brute force
def brute_force(lp, Tb, y):
    """float64 E(t) and the starts of every path reaching the maximum, by enumerating every state sequence [a, t]."""
    V1 = lp.shape[1]
    U = len(y)
    S = 2 * U - 1
    lab = [y[s // 2] if s % 2 == 0 else V1 - 1 for s in range(S)]
    lp64 = lp.astype(np.float64)
    nan = [bool(np.isnan(lp64[t]).any()) for t in range(Tb)]
    cost = [lp64[t] - lp64[t].max() if not nan[t] else None for t in range(Tb)]
    ends = {}

    def walk(start, t, s, acc):
        if nan[t]:
            return
        acc = acc + cost[t][lab[s]]
        if s == S - 1:
            ends.setdefault(t, []).append((acc, start))
        if t + 1 >= Tb:
            return
        nxt = [s, s + 1]
        if s + 2 < S and (s + 2) % 2 == 0 and y[(s + 2) // 2] != y[(s + 2) // 2 - 1]:
            nxt.append(s + 2)
        for n in nxt:
            if n < S:
                walk(start, t + 1, n, acc)

    for start in range(Tb):
        walk(start, start, 0, 0.0)
    return ends


@pytest.mark.parametrize("seed", range(24))
def test_oracle_agrees_with_the_float64_brute_force(seed):
    rng = np.random.default_rng(seed)
    V1 = int(rng.integers(3, 6))
    Tb = int(rng.integers(1, 8))
    U = int(rng.integers(1, 4))
    y = [int(i) for i in rng.integers(0, V1 - 1, U)]
    if seed % 4 == 0 and U >= 2:
        y[1] = y[0]                                           # a repeated token: no skip
    logits = rng.normal(0, 1.5, (Tb, V1))
    for t in range(Tb):                                       # plant the keyword's tokens here and there
        if rng.random() < 0.4:
            logits[t, y[int(rng.integers(0, U))]] += 3
    lp = torch.tensor(logits).log_softmax(-1).numpy().astype(F32)
    if seed % 5 == 0 and Tb > 2:
        lp[int(rng.integers(0, Tb)), 0] = np.nan              # a barrier
    E, A = spot_frames(lp, Tb, y)
    ends = brute_force(lp, Tb, y)
    tol = 1e-5 * (Tb + 1)
    for t in range(Tb):
        if t not in ends:
            assert E[t] == NEG, (t, E[t])
            continue
        best = max(p[0] for p in ends[t])
        assert abs(float(E[t]) - best) <= tol, (t, float(E[t]), best)
        starts = {p[1] for p in ends[t] if p[0] >= best - 2 * tol}
        if len(starts) == 1:
            assert int(A[t]) in starts, (t, int(A[t]), starts)
    # the scan over the brute force's scores gives the oracle's detections wherever no two scores, or a score and tau, tie
    for theta in (0.05, 0.3, 1.0):
        tau = tau_of(U, theta)
        e64 = [max(p[0] for p in ends[t]) if t in ends else -np.inf for t in range(Tb)]
        finite = [x for x in e64 if np.isfinite(x)] + [float(tau)]
        if all(abs(p - q) > 2 * tol for p, q in itertools.combinations(finite, 2)) and \
                all(len({p[1] for p in ends[t] if p[0] >= e64[t] - 2 * tol}) == 1 for t in ends):
            a64 = [next(p[1] for p in ends[t] if p[0] == e64[t]) if t in ends else 0 for t in range(Tb)]
            want = [(s, e) for s, e, _ in scan(np.array(e64), np.array(a64), float(tau))]
            assert [(s, e) for s, e, _ in scan(E, A, tau)] == want


def test_oracle_rules_on_hand_built_rows():
    V1 = 4                                                     # tokens 0..2, blank 3
    big, small = F32(0.0), F32(-5.0)

    def rows(labels):
        lp = np.full((len(labels), V1), small, F32)
        for t, l in enumerate(labels):
            lp[t, l] = big
        return lp
    lp = rows([3, 0, 0, 1, 3, 1, 2, 2, 3, 0, 1])
    # keyword (0, 1): the greedy path spells it at frames 1..3 and again at 9..10
    assert [(s, e, float(x)) for s, e, x in scan(*spot_frames(lp, 11, [0, 1]), tau_of(2, 1.0))] == [(1, 4, 0.0), (9, 11, 0.0)]
    # a repeated token needs the blank between its copies: (1, 1) at 3..5 (1, blank, 1)
    assert [(s, e) for s, e, _ in scan(*spot_frames(lp, 11, [1, 1]), tau_of(2, 1.0))] == [(3, 6)]
    # U = 1: every run of token 2 and of token 0
    assert [(s, e) for s, e, _ in scan(*spot_frames(lp, 11, [2]), tau_of(1, 1.0))] == [(6, 7)]
    assert [(s, e) for s, e, _ in scan(*spot_frames(lp, 11, [0]), tau_of(1, 1.0))] == [(1, 2), (9, 10)]
    # a NaN row cuts the second occurrence
    lp2 = lp.copy()
    lp2[10, 3] = np.nan
    assert [(s, e) for s, e, _ in scan(*spot_frames(lp2, 11, [0, 1]), tau_of(2, 1.0))] == [(1, 4)]
    # a keyword longer than the recording, and T_b = 0
    assert scan(*spot_frames(lp, 2, [0, 1, 2]), tau_of(3, 0.01)) == []
    assert scan(*spot_frames(lp, 0, [0]), tau_of(1, 0.01)) == []
    # oracle outputs: overflow keeps the true count; a bad id gives NaN rows
    st, en, sc, cnt = spot_oracle(lp[None], [11], [[0], [7]], 1.0, 1, 3)
    assert cnt.tolist() == [[2, 0]] and st[0, 0].tolist() == [1] and np.isnan(sc[0, 1]).all()


# ------------------------------------------------------------------------------------------ CPU: refusals and surface
_CPU_MODELS = {}


def _cpu_model(name):
    if name not in _CPU_MODELS:
        _CPU_MODELS[name] = gigaam.load_model(name, device="cpu", checkpoint=synthetic.synthetic_checkpoint(name, n_layers=1))
    return _CPU_MODELS[name]


def test_keywords_are_tokenised_as_align_does():
    model = _cpu_model("v2_ctc")
    tok = model.decoding.tokenizer
    names, ids = model._keyword_ids(["  Ёлка  ", [3, 4, 5], "да"], 0.5)
    assert names == [tok.normalize("  Ёлка  "), tok.decode([3, 4, 5]), "да"]
    assert ids == [tok.encode("  Ёлка  "), [3, 4, 5], tok.encode("да")]
    assert ids[0] == tok.encode("елка")                       # no space at the ends: a charwise keyword matches inside words
    names, ids = model._keyword_ids("да", 1.0)                # one string is one keyword
    assert names == ["да"]


def test_spot_refuses_before_device_work():
    model = _cpu_model("v2_ctc")
    V = len(model.decoding.tokenizer)
    wav = np.zeros(16000, np.float32)
    bad = [([], "no keywords"), (["123"], "no tokens"), ([[]], "without tokens"), (["а" * 65], "65 tokens"),
           ([[0, V]], "outside"), ([[-1]], "outside")]
    for kws, match in bad:
        with pytest.raises(ValueError, match=match):
            model.spot(wav, kws)
        with pytest.raises(ValueError, match=match):
            model.spot_batch(torch.zeros(1, 16000), torch.tensor([16000]), kws)
    for theta in (0.0, -0.5, 1.5, float("nan"), 1e-50):
        with pytest.raises(ValueError, match="threshold"):
            model.spot(wav, ["да"], threshold=theta)
    with pytest.raises(ValueError, match="max_det"):
        model.spot_batch(torch.zeros(1, 16000), torch.tensor([16000]), ["да"], max_det=0)
    with pytest.raises(ValueError, match="empty"):
        model.spot(np.zeros(0, np.float32), ["да"])
    with pytest.raises(ValueError, match="multiple"):
        model.spot(wav, ["да"], window=30.01)
    with pytest.raises(ValueError, match="overlap"):
        model.spot(wav, ["да"], window=10.0, overlap=10.0)
    with pytest.raises(ValueError, match="max_encoded_frames"):
        model.spot(wav, ["да"], window=31.0)
    with pytest.raises(ValueError, match="batch_size"):
        model.spot(wav, ["да"], batch_size=0)
    assert not hasattr(gigaam.GigaAM, "spot")


def test_rnnt_models_refuse():
    for name in ("v2_rnnt", "v3_e2e_rnnt"):
        model = _cpu_model(name)
        with pytest.raises(NotImplementedError, match="_ctc"):
            model.spot(np.zeros(16000, np.float32), ["a"])
        with pytest.raises(NotImplementedError, match="CTC head"):
            model.spot_batch(torch.zeros(1, 16000), torch.tensor([16000]), [[1]])


def test_detection_record_and_exports():
    d = Detection("да", 0, 1.0, 1.5, -0.25, math.exp(-0.125))
    assert d == Detection(keyword="да", keyword_index=0, start=1.0, end=1.5, score=-0.25, confidence=math.exp(-0.125))
    assert "Detection" in gigaam.__all__ and gigaam.Detection is Detection
    lib = _lib.load()
    for name in ("gam_ctc_spot", "gam_test_ctc_spot"):
        assert name in _lib.EXPORTS and hasattr(lib, name)
    assert hasattr(decoding, "spot")


# ------------------------------------------------------------------------------------------ GPU helpers
def _dev():
    return torch.device("cuda", 0)


_MODELS = {}


def _model(name, max_frames=None):
    key = (name, max_frames)
    if key not in _MODELS:
        _MODELS[key] = gigaam.load_model(name, fp16_encoder=False, device=_dev(), max_encoded_frames=max_frames,
                                         checkpoint=synthetic.synthetic_checkpoint(name, seed=0, n_layers=1))
    return _MODELS[key]


def _engine_for(V1):
    if V1 in (34, 257):
        return _model("v2_ctc" if V1 == 34 else "v3_e2e_ctc")._get_engine()
    return _spot_engine(V1)


def _pad(keywords):
    Umax = max(max(len(y) for y in keywords), 1)
    kw = torch.zeros((len(keywords), Umax), dtype=torch.int32)
    for k, y in enumerate(keywords):
        kw[k, :len(y)] = torch.tensor(y, dtype=torch.int32)
    return kw, torch.tensor([len(y) for y in keywords], dtype=torch.int32)


def _run(eng, lp, enc_len, keywords, threshold, max_det, warps=None):
    """Engine.ctc_spot on host arrays -> host arrays."""
    kw, kw_len = _pad(keywords)
    lp_d = torch.as_tensor(lp).to(_dev()).contiguous()
    return [t.cpu().numpy() for t in eng.ctc_spot(lp_d, torch.as_tensor(enc_len), kw, kw_len, threshold, max_det, warps)]


def _same(got, want):
    for g, w in zip(got, want):
        if g.dtype == np.float32:
            assert np.array_equal(np.isnan(g), np.isnan(w))
            g, w = np.where(np.isnan(g), 0, g).view(np.int32), np.where(np.isnan(w), 0, w).astype(F32).view(np.int32)
        assert np.array_equal(g, w), np.argwhere(g != w)[:5]


def _random_case(rng, V1, B, T):
    """log_softmax rows with keywords planted (boosted, not always argmax) here and there; keywords of 1, 2, 63 and 64 tokens
    with repeats, and a few random ones."""
    V = V1 - 1
    keywords = [[int(rng.integers(0, V))], [int(rng.integers(0, V))] * 2, [int(i) for i in rng.integers(0, V, 2)]]
    long = [int(i) for i in rng.integers(0, min(V, 6), 63)]
    long[10:13] = [long[9]] * 3                                      # runs of a repeated token
    keywords += [long, long + [long[-1]], [int(i) for i in rng.integers(0, V, 5)], [int(i) for i in rng.integers(0, V, 17)]]
    logits = rng.normal(0, 1.0, (B, T, V1)).astype(np.float64)
    logits[..., V] += 1.5                                            # blank-heavy, as CTC models are
    for b in range(B):
        for j in range(8):
            y = keywords[3 + j % 2] if j < 2 else keywords[int(rng.integers(0, len(keywords)))]
            t = int(rng.integers(0, T))
            for tok in y:
                for _ in range(int(rng.integers(1, 3))):
                    if t < T:
                        logits[b, t, tok] += rng.choice([2.0, 6.0])
                        t += 1
                if rng.random() < 0.5 and t < T:
                    t += 1
    lp = torch.tensor(logits).float().log_softmax(-1).numpy()
    return lp, keywords


# ------------------------------------------------------------------------------------------ GPU: bit identity with the oracle
@pytest.mark.gpu
@pytest.mark.parametrize("V1", [34, 257, 1025])
def test_bit_identical_to_the_oracle(V1):
    rng = np.random.default_rng(V1)
    B, T = 5, 260
    lp, keywords = _random_case(rng, V1, B, T)
    lp[2, 40, 7] = np.nan                                            # barriers in recording 2
    lp[2, 150] = np.nan
    enc_len = [T, 0, 200, 1, 10_000]                                 # ragged, empty, one frame, clamped to T
    keywords += [[V1 - 1], [0, V1 + 3]]                              # bad ids: NaN rows, count 0
    eng = _engine_for(V1)
    assert eng.num_classes == V1
    saw_overflow = saw_det = False
    cache = {}
    for theta in (0.05, 0.3, 0.7, 1.0):
        for max_det in (2, 40):
            got = _run(eng, lp, enc_len, keywords, theta, max_det)
            want = spot_oracle(lp, enc_len, keywords, theta, max_det, V1 - 1, cache)
            _same(got, want)
            saw_overflow |= bool((want[3] > max_det).any())
            saw_det |= bool((want[3][:, 3:5] > 0).any())
    assert saw_overflow and saw_det


_SPOT_ENGINES = {}


def _spot_engine(V1):
    """A CTC engine with V + 1 = V1 classes (a synthetic v2 encoder with a head of that width)."""
    if V1 not in _SPOT_ENGINES:
        ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1)
        vocab = [f"<{i}>" for i in range(V1 - 1)]
        ck["cfg"]["head"]["num_classes"] = V1
        ck["cfg"]["decoding"]["vocabulary"] = vocab
        sd = ck["state_dict"]
        w = sd["head.decoder_layers.0.weight"]
        g = torch.Generator().manual_seed(V1)
        sd["head.decoder_layers.0.weight"] = torch.randn((V1,) + tuple(w.shape[1:]), generator=g) * 0.05
        sd["head.decoder_layers.0.bias"] = torch.zeros(V1)
        _SPOT_ENGINES[V1] = gigaam.load_model("v2_ctc", fp16_encoder=False, device=_dev(), checkpoint=ck)._get_engine()
    return _SPOT_ENGINES[V1]


@pytest.mark.gpu
def test_results_do_not_depend_on_batch_keyword_order_or_warps():
    rng = np.random.default_rng(8)
    V1, B, T = 34, 8, 300
    lp, keywords = _random_case(rng, V1, B, T)
    enc_len = [T, 280, 0, T, 150, 299, 7, T]
    eng = _engine_for(V1)
    base = _run(eng, lp, enc_len, keywords, 0.2, 16)
    b = 3
    alone = _run(eng, lp[b:b + 1], enc_len[b:b + 1], keywords, 0.2, 16)
    for g, w in zip(alone, base):
        assert np.array_equal(g.view(np.int32), w[b:b + 1].view(np.int32))
    perm = list(rng.permutation(len(keywords)))
    extra = [[int(i) for i in rng.integers(0, V1 - 1, 9)] for _ in range(21)]
    order = perm[:3] + [None] * 5 + perm[3:] + [None] * 16           # permuted, padded by 21 other keywords
    it = iter(extra)
    kws = [keywords[i] if i is not None else next(it) for i in order]
    for warps in (None, 1, 4, 16):
        got = _run(eng, lp, enc_len, kws, 0.2, 16, warps)
        for j, i in enumerate(order):
            if i is None:
                continue
            for g, w in zip(got, base):
                assert np.array_equal(g[:, j].view(np.int32), w[:, i].view(np.int32)), (warps, i)


@pytest.mark.gpu
def test_planted_greedy_paths_have_confidence_one():
    V1, T = 34, 400
    rng = np.random.default_rng(3)
    logits = rng.normal(0, 1.0, (T, V1))
    logits[:, V1 - 1] += 8.0                                         # greedy: blank everywhere ...
    plants = [(20, [5, 6, 7]), (100, [9, 9, 2]), (250, [4])]
    want = {}
    for t0, y in plants:                                            # ... except the planted runs
        t = t0
        runs = []
        for i, tok in enumerate(y):
            if i and tok == y[i - 1]:
                t += 1                                               # a blank between repeated tokens
            runs.append(t)
            logits[t:t + 2, tok] += 20.0
            t += 2
        want[tuple(y)] = (t0, runs[-1] + 1)
    lp = torch.tensor(logits).float().log_softmax(-1).numpy()[None]
    eng = _engine_for(V1)
    kws = [list(y) for y in want]
    st, en, sc, cnt = _run(eng, lp, [T], kws, 1.0, 4)
    for k, y in enumerate(kws):
        assert cnt[0, k] == 1, (y, cnt[0, k])
        assert (st[0, k, 0], en[0, k, 0]) == want[tuple(y)]
        assert sc[0, k, 0] == 0.0 and math.exp(sc[0, k, 0] / len(y)) == 1.0


# ------------------------------------------------------------------------------------------ GPU: the public path
def _words_with_ids(tok, ids, frames):
    """(first token index, token ids) of every word of a greedy hypothesis (timestamps_utils.frames_to_words' split)."""
    out, cur = [], []
    for i, t in enumerate(ids):
        piece = tok.id_to_str(t)
        if piece == " " or piece.startswith("▁"):
            if cur:
                out.append(cur)
            cur = []
            if piece == " ":
                continue
        cur.append(i)
    if cur:
        out.append(cur)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,seconds", [("v2_ctc", 6.0), ("v3_e2e_ctc", 1.5)])
def test_every_greedy_word_is_found_where_transcribe_puts_it(name, seconds):
    model = _model(name)
    tok = model.decoding.tokenizer
    wav, _ = synthetic.synthetic_audio(1, seconds, seed=5)
    wav = wav[0]
    res = model.transcribe(wav, word_timestamps=True)
    w_d, l_d = model.prepare_wav(wav)
    with torch.inference_mode():
        enc, enc_len = model(w_d, l_d)
        _, ids, frames = model.decoding.decode(model.head, enc, enc_len)[0]
    # the greedy labels are the argmax of the log-probs spot searches (so the greedy path scores exactly 0)
    lab = model.head(enc)[0, :int(enc_len[0])].argmax(-1).tolist()
    blank = len(tok)
    runs = [(t, x) for t, x in enumerate(lab) if x != blank and (t == 0 or lab[t - 1] != x)]
    assert [x for _, x in runs] == ids and [t for t, _ in runs] == frames
    words = _words_with_ids(tok, ids, frames)
    assert len(words) == len(res.words) and len(words) > 0
    keywords, checks = [], []
    for w, word in zip(words, res.words):
        y = [ids[i] for i in w]
        if len(y) > 64:
            continue
        spans = [(frames[i], frames[i + len(y) - 1] + 1) for i in range(len(ids) - len(y) + 1) if ids[i:i + len(y)] == y]
        if any(a < d and c < b for (a, b), (c, d) in itertools.combinations(spans, 2)):
            continue                                                 # occurrences that overlap: not checked
        checks.append((len(keywords), word, spans))
        keywords.append(y)
    assert checks
    dets = model.spot(wav, keywords, threshold=0.5)
    for k, word, spans in checks:
        mine = [d for d in dets if d.keyword_index == k and d.score == 0.0]
        assert len(mine) >= len(spans)
        assert any(d.start == word.start and d.end == word.end and d.confidence == 1.0 for d in mine), (k, word, mine[:3])
    assert dets == sorted(dets, key=lambda d: (d.start, d.keyword_index))


@pytest.mark.gpu
def test_long_recording_equals_spotting_the_stitched_log_probs():
    model = _model("v2_ctc")
    eng = model._get_engine()
    tok = model.decoding.tokenizer
    wav, _ = synthetic.synthetic_audio(1, 300.0, seed=4)
    wav = wav[0][: 300 * 16000 - 4321]
    # every symbol, a word with its spaces given as ids, and a few short keywords, at a low threshold: many detections
    keywords = list(tok.vocab) + [[tok.vocab.index(" "), tok.vocab.index("и"), tok.vocab.index(" ")], "но", "при"]
    keywords[0] = [tok.vocab.index(" ")]                                # " " normalises to nothing: pass it as an id
    names, ids = model._keyword_ids(keywords, 0.05)
    dets = model.spot(wav, keywords, threshold=0.05, batch_size=4)
    windows, T = plan_windows(wav.numel(), 30.0, 4.0, model._encoded_length, 768)
    assert len(windows) > 5
    with torch.inference_mode():
        w_d, length = model.prepare_wav(wav)
        lp = stitch_ctc_log_probs(model, w_d[0], windows, T, 4)
        kw, kw_len = _pad(ids)
        out = eng.ctc_spot(lp, torch.tensor([T]), kw, kw_len, 0.05, T)
    from gigaam_b200.timestamps_utils import compute_frame_shift
    start, end, score, count = (t[0].cpu() for t in out)
    stored = [list(zip(start[k, :c].tolist(), end[k, :c].tolist(), score[k, :c].tolist())) for k, c in enumerate(count.tolist())]
    want = model._detections(names, ids, stored, compute_frame_shift(int(length[0]), T))
    print(f"\n{len(dets)} detections over {T} frames")
    assert dets == want and len(dets) >= 10
    # one window: the same as spot_batch
    short = wav[:20 * 16000]
    one = model.spot(short, keywords, threshold=0.05)
    batch = model.spot_batch(short[None].to(_dev()), torch.tensor([short.numel()], device=_dev()), keywords, threshold=0.05,
                             max_det=1000)
    assert one == batch[0] and len(one) > 0


@pytest.mark.gpu
def test_device_memory_stays_within_the_stitched_log_probs():
    model = _model("v2_ctc")
    V1 = model._get_engine().num_classes
    peaks, frames = {}, {}
    for minutes in (2, 20, 2, 20):
        wav, _ = synthetic.synthetic_audio(1, 60.0 * minutes, seed=minutes)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        model.spot(wav[0], ["а", "то", "при"], threshold=0.3, batch_size=4)
        torch.cuda.synchronize()
        peaks[minutes] = torch.cuda.max_memory_allocated() - base
        frames[minutes] = model._encoded_length(wav.shape[1])
    grow = (frames[20] - frames[2]) * V1 * 4
    print(f"\npeak above baseline: 2 min {peaks[2] / 2**20:.1f} MiB, 20 min {peaks[20] / 2**20:.1f} MiB, "
          f"stitched log-probs grow by {grow / 2**20:.1f} MiB")
    assert peaks[20] - peaks[2] < grow + 16 * 2**20


@pytest.mark.gpu
def test_refusals_and_graph_capture():
    eng = _engine_for(34)
    lp = torch.randn(2, 50, 34, device=_dev()).log_softmax(-1)
    enc_len = torch.tensor([50, 30], dtype=torch.int32, device=_dev())
    kw, kw_len = (t.to(_dev()) for t in _pad([[1, 2], [3]]))
    outs = [torch.empty((2, 2, 4), dtype=torch.int32, device=_dev()), torch.empty((2, 2, 4), dtype=torch.int32, device=_dev()),
            torch.empty((2, 2, 4), device=_dev()), torch.empty((2, 2), dtype=torch.int32, device=_dev())]
    ptrs = [t.data_ptr() for t in outs]

    def call(K=2, Umax=2, theta=0.5, max_det=4):
        return eng.lib.gam_ctc_spot(eng.handle, lp.data_ptr(), enc_len.data_ptr(), 2, 50, kw.data_ptr(), kw_len.data_ptr(), K, Umax,
                                    theta, max_det, *ptrs, eng._stream())
    for kwargs, msg in (({"K": 0}, "K=0"), ({"Umax": 65}, "Umax=65"), ({"theta": 0.0}, "threshold"), ({"theta": 1.01}, "threshold"),
                        ({"max_det": 0}, "max_det")):
        assert call(**kwargs) != 0
        assert msg in eng.lib.gam_last_error(eng.handle).decode()
    assert call() == 0
    rnnt = _model("v2_rnnt")
    with pytest.raises(NotImplementedError):
        decoding.spot(rnnt.head, torch.zeros(1, 768, 10, device=_dev()), torch.tensor([10]), kw, kw_len, 0.5, 4)
    with pytest.raises(NotImplementedError):
        rnnt.spot(np.zeros(16000, np.float32), ["а"])
    # one capture, replayed: the same bits as the eager call
    want = [t.clone() for t in eng.ctc_spot(lp, enc_len, kw, kw_len, 0.05, 4)]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        eng.ctc_spot(lp, enc_len, kw, kw_len, 0.05, 4)               # warm up on the capture stream
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            got = eng.ctc_spot(lp, enc_len, kw, kw_len, 0.05, 4)
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(got, want):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
