"""Long-form alignment of texts that only partly match the recording: gam_ctc_align_long_gaps (include/gigaam_b200.h has the
definition) and `GigaAMASR.align_longform(..., gap_threshold=theta)` (INTEGRATION.md §7e).

The Viterbi recursion with gaps is still a fixed sequence of fp32 adds, maxes and strict compares, so the numpy float32
oracle below (`gap_replay`) reproduces frames, token log-probs, the path score and the three gap outputs bit for bit; the
forward score is compared with a float64 recursion within test_align.py's bound.

CPU: the oracle against a float64 brute force over every path, a planted case where the graph without gaps misplaces a
token, line_edges, refusals, and that gap_threshold=None runs exactly the calls it ran before.  GPU: bit identity with the
oracle (three vocabularies, a ragged batch with empty, NaN and bad-id recordings, forced cluster sizes, alone and in a batch),
log theta = -inf against gam_ctc_align_long, a planted hour, the public call end to end, a CUDA-graph replay and the memory.
"""
import math

import numpy as np
import pytest
import torch

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, longform, synthetic
from gigaam_b200.longform import line_edges, line_segments, plan_windows, unmatched_intervals
from gigaam_b200.timestamps_utils import compute_frame_shift, gap_confidence
from gigaam_b200.types import LongformAlignment, Segment

from test_align import F32, INF, NAN, _log_probs, ctc_forward_bound

_CPU_MODELS = {}


def _cpu_model(name):
    if name not in _CPU_MODELS:
        _CPU_MODELS[name] = gigaam.load_model(name, device="cpu", checkpoint=synthetic.synthetic_checkpoint(name, n_layers=1))
    return _CPU_MODELS[name]


# ------------------------------------------------------------------------------------------ the oracle
def _graph(V1, y, edges):
    """Labels, skip flags and boundary flags of the S = 2U + 1 states."""
    blank, n = V1 - 1, len(y)
    S = 2 * n + 1
    lab = np.full(S, blank, np.int64)
    lab[1::2] = y
    skip = np.zeros(S, bool)
    skip[3::2] = np.asarray(y[1:], np.int64) != np.asarray(y[:-1], np.int64)
    bound = np.zeros(S, bool)
    for s in range(0, S, 2):
        j = s // 2
        bound[s] = s == 0 or j == n or bool(edges[j] & 1) or bool(edges[j - 1] & 2)
    return lab, skip, bound


def _emissions(lp, Tb, lab, bound, log_theta):
    """e [Tb, S] f32: lp[t, l'_s], and max(lp[t, blank], m[t] + log theta) at boundary states; g [Tb] = m[t] + log theta."""
    m = lp[:Tb].max(axis=1) + F32(0.0)
    with np.errstate(invalid="ignore"):
        g = (m + F32(log_theta)).astype(F32)
        e = lp[:Tb][:, lab].copy()
        e[:, bound] = np.fmax(e[:, bound], g[:, None])
    return e, g


def gap_replay(lp, Tb, y, edges, log_theta, U=None):
    """gam_ctc_align_long_gaps for one recording in numpy float32.  lp [T, V+1] f32, y its ids, edges its line_edges.
    -> (frames [U], token_logp [U], viterbi, path_rows, unmatched [T] u8, unmatched_rows, unmatched_logp)."""
    lp = np.asarray(lp, F32)
    T, V1 = lp.shape
    blank, n = V1 - 1, len(y)
    U = n if U is None else U
    frames, tok = np.full(U, -1, np.int32), np.full(U, -INF, F32)
    flags = np.zeros(T, np.uint8)
    if any(not 0 <= i < blank for i in y) or (Tb > 0 and np.isnan(lp[:Tb]).any()):
        tok[:n] = NAN
        return frames, tok, F32(NAN), Tb, flags, 0, F32(NAN)
    if Tb == 0:
        return frames, tok, F32(-INF), Tb, flags, 0, F32(0.0)
    lab, skip, bound = _graph(V1, y, edges)
    S = len(lab)
    e, g = _emissions(lp, Tb, lab, bound, log_theta)
    v = np.full(S, -INF, F32)
    v[:2] = e[0, :2]
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
            v = e[t] + best
    s = S - 1
    if S >= 2 and v[S - 2] > v[S - 1]:
        s = S - 2
    vit = v[s]
    if vit == -INF:
        return frames, tok, vit, Tb, flags, 0, F32(0.0)
    for t in range(Tb - 1, -1, -1):
        if s & 1:
            frames[s >> 1] = t
        elif bound[s] and g[t] > lp[t, blank]:
            flags[t] = 1
        if t > 0:
            s -= int(code[t, s])
    tok[:n] = lp[frames[:n], y]
    total = F32(0.0)
    for t in np.flatnonzero(flags):
        total = F32(total + g[t])
    return frames, tok, vit, Tb, flags, int(flags.sum()), total


def gap_forward64(lp, Tb, y, edges, log_theta):
    """The forward score of the graph with gaps in float64 over the fp32 emissions, and the largest finite |f| per frame."""
    lp = np.asarray(lp, F32)
    lab, skip, bound = _graph(lp.shape[1], y, edges)
    S = len(lab)
    e, _ = _emissions(lp, Tb, lab, bound, log_theta)
    e = e.astype(np.float64)
    f = np.full(S, -INF)
    f[:2] = e[0, :2]
    mags = [np.abs(f[np.isfinite(f)]).max(initial=0.0)]
    with np.errstate(invalid="ignore", divide="ignore"):
        for t in range(1, Tb):
            a = np.concatenate([[-INF], f[:-1]])
            b = np.where(skip, np.concatenate([[-INF, -INF], f[:-2]])[:S], -INF)
            f = np.logaddexp(np.logaddexp(f, a), b) + e[t]
            mags.append(np.abs(f[np.isfinite(f)]).max(initial=0.0))
    ll = np.logaddexp(f[S - 1], f[S - 2]) if S >= 2 else f[0]
    return float(ll), mags


def _brute_force(lp, Tb, y, edges, log_theta):
    """Every path of the graph with gaps in float64: (best score, runner-up score, best path's states, forward score)."""
    lp = np.asarray(lp, F32)
    lab, skip, bound = _graph(lp.shape[1], y, edges)
    S = len(lab)
    e, _ = _emissions(lp, Tb, lab, bound, log_theta)
    e = e.astype(np.float64)
    scores, paths = [], []

    def walk(t, s, acc, path):
        acc = acc + e[t, s]
        path = path + [s]
        if t == Tb - 1:
            if s >= S - 2:
                scores.append(acc)
                paths.append(path)
            return
        for nxt in (s, s + 1, s + 2):
            if nxt < S and (nxt <= s + 1 or skip[nxt]):
                walk(t + 1, nxt, acc, path)
    for s0 in range(min(2, S)):
        walk(0, s0, 0.0, [])
    if not scores:
        return -INF, -INF, None, -INF
    order = np.argsort(scores)[::-1]
    best = scores[order[0]]
    second = scores[order[1]] if len(order) > 1 else -INF
    return best, second, paths[order[0]], float(np.logaddexp.reduce(scores))


def _random_edges(rng, n):
    """Random line edges of n tokens: random cuts into lines, so bit 0 on every line start and bit 1 on every line end."""
    cuts = sorted(set(rng.integers(1, n, rng.integers(0, n)).tolist())) if n > 1 else []
    bounds = [0] + cuts + [n]
    return line_edges(list(zip(bounds[:-1], bounds[1:])), n)


# ------------------------------------------------------------------------------------------ CPU
def test_oracle_matches_a_float64_brute_force_over_every_path():
    rng = np.random.default_rng(0)
    checked = flagged = 0
    for case in range(400):
        V1 = int(rng.integers(3, 6))
        Tb = int(rng.integers(1, 9))
        n = int(rng.integers(0, 4))
        y = rng.integers(0, V1 - 1, n).tolist()
        edges = _random_edges(rng, n)
        theta = float(rng.uniform(1e-3, 1.0)) if case % 5 else 1.0
        log_theta = float(F32(math.log(theta)))
        lp = _log_probs(rng, (Tb, V1))
        fr, tok, vit, rows, flags, urows, ulogp = gap_replay(lp, Tb, y, edges, log_theta)
        assert rows == Tb and urows == int(flags.sum())
        best, second, path, fwd = _brute_force(lp, Tb, y, edges, log_theta)
        if best == -INF:
            assert vit == -INF and (fr == -1).all() and urows == 0
            continue
        assert abs(float(vit) - best) <= 1e-5 * (1 + abs(best)), (case, vit, best)
        want_fwd, mags = gap_forward64(lp, Tb, y, edges, log_theta)
        assert abs(want_fwd - fwd) <= 1e-9 * (1 + abs(fwd))
        if best - second < 1e-4:
            continue                                                # near-tie: the path is not determined by the scores
        lab, _, bound = _graph(V1, y, edges)
        want_fr = np.full(n, -1, np.int32)
        for t in range(Tb - 1, -1, -1):
            if path[t] & 1:
                want_fr[path[t] >> 1] = t
        assert np.array_equal(fr, want_fr), case
        m = lp.max(axis=1) + F32(0.0)
        g = (m + F32(log_theta)).astype(F32)
        want_flags = np.array([bound[s] and g[t] > lp[t, V1 - 1] for t, s in enumerate(path)], np.uint8)
        assert np.array_equal(flags, want_flags), case
        checked += 1
        flagged += int(want_flags.any())
    assert checked > 200 and flagged > 30


def _planted_case():
    """Two lines "ab" and "cd" (V + 1 = 6, blank 5) with four frames of foreign speech between them whose sounds resemble
    "c": the graph without gaps emits c inside the foreign speech, the graph with gaps leaves the speech unmatched."""
    V1, T = 6, 14
    lp = np.full((T, V1), -12.0, F32)
    plan = [(0, 0), (1, 5), (2, 1), (3, 5)]                         # a, blank, b, blank
    plan += [(4, 4), (5, 4)]                                       # foreign: class 4 peaked
    plan += [(8, 5), (9, 2), (10, 5), (11, 3), (12, 5), (13, 5)]   # blank, c, blank, d, blank, blank
    for t, c in plan:
        lp[t, c] = -0.05
    lp[6:8, 2] = -0.5                                              # foreign frames that sound like "c"
    lp[6:8, 4] = -0.6
    y, edges = [0, 1, 2, 3], line_edges([(0, 2), (2, 4)], 4)
    return lp, y, edges


def test_planted_foreign_speech_moves_a_token_without_gaps_only():
    lp, y, edges = _planted_case()
    T = lp.shape[0]
    plain = gap_replay(lp, T, y, edges, -INF)
    gaps = gap_replay(lp, T, y, edges, float(F32(math.log(0.5))))
    fr = plain[0].tolist()
    assert fr[:2] == [0, 2] and 4 <= fr[2] <= 7 and fr[3] == 11    # "c" pulled into the foreign speech
    assert not plain[4].any()
    assert gaps[0].tolist() == [0, 2, 9, 11]                       # every token at its planted frame
    assert np.flatnonzero(gaps[4]).tolist() == [4, 5, 6, 7] and gaps[5] == 4


def test_reduction_to_the_graph_without_gaps():
    from test_align import ctc_replay
    rng = np.random.default_rng(3)
    for _ in range(100):
        V1, Tb, n = 5, int(rng.integers(1, 12)), int(rng.integers(0, 5))
        y = rng.integers(0, V1 - 1, n).tolist()
        lp = _log_probs(rng, (Tb, V1), ties=True)
        got = gap_replay(lp, Tb, y, _random_edges(rng, n), -INF)
        want = ctc_replay(lp, Tb, y)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
        assert F32(got[2]).view(np.uint32) == F32(want[2]).view(np.uint32) and not got[4].any() and got[5] == 0


class _SentencePieceLike:
    charwise = False
    vocab = ["▁при", "вет", "▁как", "▁де", "ла"]
    _pieces = {"привет": [0, 1], "как дела": [2, 3, 4], "как": [2]}

    def normalize(self, text):
        return " ".join(text.lower().split())

    def encode(self, text):
        return list(self._pieces.get(self.normalize(text), []))


def test_line_edges_from_line_tokens():
    model = _cpu_model("v2_ctc")
    tok = model.decoding.tokenizer
    sp = tok.vocab.index(" ")
    _, ids, ranges = model._line_tokens(["аб", "", "в", "гд е"])
    assert ids == tok.encode("аб") + [sp] + tok.encode("в") + [sp] + tok.encode("гд е")
    edges = line_edges(ranges, len(ids))
    assert edges == [1, 2, 0, 3, 0, 1, 0, 0, 2]                    # the joining spaces and the space inside a line: 0
    bound = _graph(len(tok.vocab) + 1, ids, edges)[2]
    assert np.flatnonzero(bound).tolist() == [0, 4, 6, 8, 10, 18]  # both sides of each joining space, the two ends
    _, ids, ranges = model._line_tokens(["", "", ""])
    assert ids == [] and line_edges(ranges, 0) == []
    assert np.flatnonzero(_graph(34, [], [])[2]).tolist() == [0]   # U = 0: the single state is a boundary state
    saved = model.decoding.tokenizer
    try:
        model.decoding.tokenizer = _SentencePieceLike()
        _, ids, ranges = model._line_tokens(["Привет", "", "как дела", "как"])
        assert ids == [0, 1, 2, 3, 4, 2] and ranges == [(0, 2), (2, 2), (2, 5), (5, 6)]
        assert line_edges(ranges, len(ids)) == [1, 2, 1, 0, 2, 3]
    finally:
        model.decoding.tokenizer = saved


def test_unmatched_intervals_and_record():
    flags = torch.tensor([1, 1, 0, 0, 1, 0, 1, 1, 1], dtype=torch.uint8)
    assert unmatched_intervals(flags, 0.04) == [(0.0, 0.08), (0.16, 0.2), (0.24, 0.36)]
    assert unmatched_intervals(torch.zeros(5, dtype=torch.uint8), 0.04) == []
    seg = Segment("аб", 0.0, 0.08, None, 0.5)
    plain = LongformAlignment([seg], -3.5, 0.7)
    assert plain.unmatched is None and "unmatched" not in repr(plain)
    gapped = LongformAlignment([seg], -3.5, 0.7, [(1.0, 2.0)])
    assert gapped.unmatched == [(1.0, 2.0)] and repr(gapped).endswith("unmatched=[(1.0, 2.0)])") and gapped != plain
    assert gap_confidence(-4.0, -1.0, 3) == math.exp(-1.0) and math.isnan(gap_confidence(-4.0, -4.0, 0))
    assert gap_confidence(-INF, 0.0, 5) == 0.0


def test_gap_threshold_refusals_before_device_work():
    model = _cpu_model("v2_ctc")
    wav = np.zeros(16000, np.float32)
    for theta in (0.0, -0.5, 1.5, NAN, INF, 1e-46, 1.0000001):     # 1e-46 is 0 in float32, 1.0000001 is 1 + 2^-23 after rounding
        with pytest.raises(ValueError, match="gap_threshold"):
            model.align_longform(wav, "а", gap_threshold=theta)
    with pytest.raises(TypeError):
        model.align_longform(wav, "а", True, 30.0, 4.0, 16, 0.5)   # keyword-only
    for name in ("v2_rnnt", "v3_e2e_rnnt"):
        with pytest.raises(NotImplementedError, match="CTC"):
            _cpu_model(name).align_longform(wav, "а", gap_threshold=0.5)


def test_exports():
    lib = _lib.load()
    for name in ("gam_ctc_align_long_gaps", "gam_ctc_align_long_gaps_workspace_bytes", "gam_test_ctc_align_long_gaps"):
        assert name in _lib.EXPORTS and hasattr(lib, name)


class _Recorder:
    """Stands in for the engine: records the ctc_align_long calls."""

    def __init__(self):
        self.calls = []
        self.device = torch.device("cpu")
        self.num_classes = 34

    def ctc_align_long(self, lp, enc_len, targets, target_len, **kw):
        self.calls.append((4, tuple(sorted(kw))))
        U = targets.shape[1]
        outs = (torch.zeros((1, U), dtype=torch.int32), torch.zeros((1, U)), torch.tensor([-1.0]), torch.tensor([-2.0]),
                torch.tensor([int(enc_len[0])], dtype=torch.int32))
        if "gaps" in kw:
            outs += (torch.zeros((1, lp.shape[1]), dtype=torch.uint8), torch.tensor([0], dtype=torch.int32), torch.tensor([0.0]))
        return outs

    def __getattr__(self, name):
        raise AssertionError(f"unexpected engine call {name}")


def test_gap_threshold_none_calls_what_it_called_before(monkeypatch):
    model = _cpu_model("v2_ctc")
    eng = _Recorder()
    monkeypatch.setattr(model, "_get_engine", lambda: eng)
    monkeypatch.setattr(longform, "stitch_ctc_log_probs", lambda m, wav, windows, T, bs: torch.zeros((1, T, 34)))
    wav = np.zeros(16000, np.float32)
    for kwargs in ({}, {"gap_threshold": None}):
        eng.calls.clear()
        res = model.align_longform(wav, ["аб", "в"], word_timestamps=False, **kwargs)
        assert eng.calls == [(4, ())] and res.unmatched is None
    eng.calls.clear()
    res = model.align_longform(wav, ["аб", "в"], word_timestamps=False, gap_threshold=0.5)
    assert eng.calls == [(4, ("gaps",))] and res.unmatched == []


# ------------------------------------------------------------------------------------------ GPU helpers
def _dev():
    return torch.device("cuda", 0)


def _engine(V1):
    from test_keyword_spotting import _engine_for
    return _engine_for(V1)


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _run(eng, lp, enc_len, targets, target_len, edges, log_theta, cluster_ctas=None):
    out = eng.ctc_align_long(torch.from_numpy(lp).to(_dev()), torch.tensor(enc_len), torch.from_numpy(targets),
                             torch.tensor(target_len), cluster_ctas=cluster_ctas,
                             gaps=(torch.from_numpy(edges).to(_dev()), log_theta))
    return [t.cpu().numpy() for t in out]


def _check_oracle(got, lp, enc_len, targets, target_len, edges, log_theta):
    fr, tok, vit, ll, rows, flags, urows, ulogp = got
    T = lp.shape[1]
    for b in range(lp.shape[0]):
        Tb, Ub = min(max(enc_len[b], 0), T), target_len[b]
        y = targets[b, :Ub].tolist()
        w = gap_replay(lp[b], Tb, y, edges[b, :Ub], log_theta, targets.shape[1])
        assert np.array_equal(fr[b], w[0]), b
        assert np.array_equal(tok[b].view(np.uint32), w[1].view(np.uint32)), b
        assert F32(vit[b]).view(np.uint32) == F32(w[2]).view(np.uint32), (b, vit[b], w[2])
        assert rows[b] == w[3] and np.array_equal(flags[b], w[4]) and urows[b] == w[5], b
        assert F32(ulogp[b]).view(np.uint32) == F32(w[6]).view(np.uint32), (b, ulogp[b], w[6])
        if math.isfinite(vit[b]):
            want, mags = gap_forward64(lp[b], Tb, y, edges[b, :Ub], log_theta)
            assert abs(ll[b] - want) <= ctc_forward_bound(mags, want), (b, ll[b], want)
        else:
            assert F32(ll[b]).view(np.uint32) == F32(vit[b]).view(np.uint32), b


def _ragged_batch(rng, V1):
    """Ragged lengths, enc_len 0, U = 0, NaN rows inside and past a recording, a NaN in a class no target uses, a bad id;
    the lines of each recording are random, and the foreign frames planted before, between and after them."""
    B, T, U = 10, 260, 120
    lp = _log_probs(rng, (B, T, V1))
    targets = rng.integers(0, V1 - 1, (B, U)).astype(np.int32)
    enc_len = [260, 240, 0, 200, 260, 150, 260, 230, 260, 300]
    target_len = [120, 90, 10, 0, 120, 60, 40, 100, 120, 70]
    edges = np.zeros((B, U), np.uint8)
    for b in range(B):
        edges[b, :target_len[b]] = _random_edges(rng, target_len[b])
    for b in range(B):                                             # foreign speech: a peaked non-blank class
        for t in list(range(0, 15)) + list(range(100, 115)) + list(range(T - 12, T)):
            lp[b, t] = F32(-8.0)
            lp[b, t, int(rng.integers(0, V1 - 1))] = F32(-0.02)
    lp[5, 70, :] = NAN                                             # inside the recording: poisoned
    lp[7, 235, :] = NAN                                            # past the recording: not read
    unused = sorted(set(range(V1 - 1)) - set(targets[6, :40].tolist()))[0]
    lp[6, 30, unused] = NAN                                        # a class no target uses: poisoned in gap mode
    targets[8, 3] = -4
    return lp, enc_len, targets, target_len, edges


# ------------------------------------------------------------------------------------------ GPU: kernel
@pytest.mark.gpu
@pytest.mark.parametrize("V1", [34, 257, 1025])
def test_bit_identical_to_the_oracle_on_a_ragged_batch(V1):
    eng = _engine(V1)
    assert eng.num_classes == V1
    rng = np.random.default_rng(V1)
    lp, enc_len, targets, target_len, edges = _ragged_batch(rng, V1)
    saw_flag = False
    for theta in (0.02, 0.3, 1.0):
        log_theta = float(F32(math.log(theta)))
        base = None
        for c in (None, 1, 2, 3, 16):
            got = _run(eng, lp, enc_len, targets, target_len, edges, log_theta, c)
            if c is not None:
                assert eng.last_align_long_plan[0] == c
            if base is None:
                _check_oracle(got, lp, enc_len, targets, target_len, edges, log_theta)
                base = got
                saw_flag |= bool(got[6].sum() > 0)
            else:
                assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(got, base)), c
        for b in (0, 4, 6, 9):                                     # alone: the same bits as in the batch
            alone = _run(eng, lp[b:b + 1], enc_len[b:b + 1], targets[b:b + 1], target_len[b:b + 1], edges[b:b + 1], log_theta)
            assert all(np.array_equal(x.view(np.uint8), y[b:b + 1].view(np.uint8)) for x, y in zip(alone, base)), b
    assert saw_flag


@pytest.mark.gpu
def test_log_theta_minus_inf_equals_ctc_align_long():
    eng = _engine(34)
    rng = np.random.default_rng(4)
    lp, enc_len, targets, target_len, edges = _ragged_batch(rng, 34)
    lp = np.nan_to_num(lp, nan=-3.0)
    targets[8, 3] = 1
    lp[1, :, 5] = 0.0                                              # ties, and -inf entries
    lp[4, 10, :] = -INF
    for c in (None, 2):
        args = (torch.from_numpy(lp).to(_dev()), torch.tensor(enc_len), torch.from_numpy(targets), torch.tensor(target_len))
        want = eng.ctc_align_long(*args, cluster_ctas=c)
        got = eng.ctc_align_long(*args, cluster_ctas=c, gaps=(torch.from_numpy(edges), -INF))
        assert all(torch.equal(_bits(x), _bits(y)) for x, y in zip(got[:5], want))
        assert not got[5].any() and not got[6].any() and not got[7].any()


@pytest.mark.gpu
def test_refusals_of_the_c_level():
    eng = _engine(34)
    lp = torch.zeros(1, 4, 34, device=_dev())
    args = (lp, torch.tensor([4]), torch.zeros(1, 2, dtype=torch.int32), torch.tensor([2]))
    for bad in (NAN, 0.5, INF):
        with pytest.raises(_lib.GamError, match="log_theta"):
            eng.ctc_align_long(*args, gaps=(torch.zeros(1, 2, dtype=torch.uint8), bad))
    eng.ctc_align_long(*args, gaps=(torch.zeros(1, 2, dtype=torch.uint8), 0.0))
    with pytest.raises(ValueError):
        eng.ctc_align_long(lp, torch.tensor([4]), torch.zeros(1, 65537, dtype=torch.int32), torch.tensor([1]),
                           gaps=(torch.zeros(1, 65537, dtype=torch.uint8), -1.0))
    with pytest.raises(_lib.GamError, match="without states"):
        eng.ctc_align_long(*args, cluster_ctas=16, gaps=(torch.zeros(1, 2, dtype=torch.uint8), -1.0))


@pytest.mark.gpu
@pytest.mark.parametrize("V1", [34, 257])
def test_planted_hour_with_foreign_speech(V1):
    """T' = 90 000 frames, U = 65 536 tokens in 120 lines.  Token i is peaked at frame f_i, blank on the other frames of
    the lines, and foreign speech (a class no token uses, peaked) fills stretches before the first line, between lines and
    after the last one.  Every token must land at f_i and exactly the foreign frames must be flagged."""
    eng = _engine(V1)
    T, U, L = 90000, 65536, 120
    g = torch.Generator().manual_seed(V1)
    foreign = V1 - 2                                               # no token uses it
    steps = torch.randint(1, V1 - 2, (U,), generator=g)
    y = (torch.cumsum(steps, 0) % (V1 - 2)).to(torch.int32)        # no label repeats its neighbour
    cuts = torch.sort(torch.randperm(U - 1, generator=g)[:L - 1] + 1).values.tolist()
    bounds = [0] + cuts + [U]
    ranges = list(zip(bounds[:-1], bounds[1:]))
    stretch = [int(x) for x in torch.randint(0, 150, (L + 1,), generator=g)]
    stretch[0], stretch[-1] = 800, 700
    extra = T - U - sum(stretch)
    gaps_in = torch.zeros(U, dtype=torch.int64)
    gaps_in[torch.randperm(U, generator=g)[:extra // 2]] = 1       # blank frames inside lines
    f = torch.empty(U, dtype=torch.int64)
    is_foreign = torch.zeros(T, dtype=torch.bool)
    t = 0
    for li, (a, b) in enumerate(ranges):
        is_foreign[t:t + stretch[li]] = True
        t += stretch[li]
        for i in range(a, b):
            t += int(gaps_in[i])
            f[i] = t
            t += 1
    is_foreign[t:t + stretch[-1]] = True
    t += stretch[-1]
    assert t <= T
    lp = torch.full((1, T, V1), -30.0, device=_dev())
    lp[0, :, V1 - 1] = 0.0
    fd, ff = f.to(_dev()), torch.nonzero(is_foreign).reshape(-1).to(_dev())
    lp[0, fd, y.long().to(_dev())] = 0.0
    lp[0, fd, V1 - 1] = -30.0
    lp[0, f[::7].to(_dev()), y[::7].long().to(_dev())] = -0.25
    lp[0, ff, V1 - 1] = -30.0
    lp[0, ff, foreign] = -0.125
    edges = torch.tensor(line_edges(ranges, U), dtype=torch.uint8)
    log_theta = float(F32(math.log(0.5)))
    out = eng.ctc_align_long(lp, torch.tensor([T]), y[None], torch.tensor([U]), gaps=(edges[None], log_theta))
    frames, _, vit, ll, rows, flags, urows, ulogp = (x.cpu() for x in out)
    assert torch.equal(frames[0].long(), f)
    assert torch.equal(flags[0].bool(), is_foreign) and int(urows[0]) == int(is_foreign.sum())
    gt = F32(F32(-0.125) + F32(log_theta))
    s = F32(0.0)
    for _ in range(int(is_foreign.sum())):
        s = F32(s + gt)
    assert F32(ulogp[0]) == s
    path = np.zeros(T, F32)
    path[f.numpy()] = np.where(np.arange(U) % 7 == 0, F32(-0.25), F32(0.0))
    path[is_foreign.numpy()] = gt
    v = F32(0.0)
    for x in path:
        v = F32(v + x)
    assert F32(vit[0]) == v and int(rows[0]) == T and math.isfinite(float(ll[0]))


@pytest.mark.gpu
def test_graph_capture_and_memory():
    eng = _engine(34)
    rng = np.random.default_rng(2)
    B, T, U = 2, 3000, 1200
    lp = torch.from_numpy(_log_probs(rng, (B, T, 34))).to(_dev())
    targets = torch.from_numpy(rng.integers(0, 33, (B, U)).astype(np.int32)).to(_dev())
    enc_len = torch.tensor([3000, 2500], dtype=torch.int32, device=_dev())
    tlen = torch.tensor([1200, 700], dtype=torch.int32, device=_dev())
    edges = torch.from_numpy(np.stack([_random_edges(rng, U) for _ in range(B)]).astype(np.uint8)).to(_dev())
    gaps = (edges, float(F32(math.log(0.2))))

    def peak(**kw):
        eng._ws_align._d.clear()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = eng.ctc_align_long(lp, enc_len, targets, tlen, **kw)
        torch.cuda.synchronize()
        del out
        return torch.cuda.max_memory_allocated() - base
    plain, gapped = peak(), peak(gaps=gaps)
    m_bytes = -(-B * T * 4 // 1024) * 1024
    flags = -(-B * T // 512) * 512
    assert 0 < gapped - plain <= m_bytes + flags + 2 * 512, (plain, gapped)
    want = [t.clone() for t in eng.ctc_align_long(lp, enc_len, targets, tlen, gaps=gaps)]
    assert int(want[6].sum()) > 0
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        eng.ctc_align_long(lp, enc_len, targets, tlen, gaps=gaps)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            captured = eng.ctc_align_long(lp, enc_len, targets, tlen, gaps=gaps)
    torch.cuda.current_stream().wait_stream(stream)
    for t in captured:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(_bits(x), _bits(y)) for x, y in zip(captured, want))


# ------------------------------------------------------------------------------------------ GPU: end to end
_MODELS = {}


def _model(name):
    """A synthetic model whose blank bias is lowered by 5, so that its greedy transcripts of synthetic audio have text."""
    if name not in _MODELS:
        ck = synthetic.synthetic_checkpoint(name, seed=0, n_layers=1)
        ck["state_dict"]["head.decoder_layers.0.bias"][-1] -= 5.0
        _MODELS[name] = gigaam.load_model(name, fp16_encoder=False, device=_dev(), checkpoint=ck)
    return _MODELS[name]


class _IdTokenizer:
    """The e2e model's vocabulary as SentencePiece-like pieces "▁<i>" (every token a word), with lines written as ids."""
    charwise = False

    def __init__(self, V):
        self.vocab = [f"\u2581<{i}>" for i in range(V)]

    def __len__(self):
        return len(self.vocab)

    def id_to_str(self, i):
        return self.vocab[i]

    def normalize(self, text):
        return " ".join(text.split())

    def encode(self, text):
        return [int(x) for x in text.split()]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v3_e2e_ctc"])
def test_align_longform_with_gaps_end_to_end(name):
    import re
    model = _model(name)
    wav, _ = synthetic.synthetic_audio(1, 100.0, seed=21)
    wav = wav[0]
    lines = []
    for k in range(0, wav.numel(), 20 * 16000):
        text = model.transcribe(wav[k:k + 20 * 16000]).text
        if name == "v2_ctc":
            lines.append(text[: len(text) // 3])                    # a third of each piece: the rest is left to the gaps
        else:
            ids = re.findall(r"<(\d+)>", text)
            lines.append(" ".join(ids[: len(ids) // 3]))
    lines.insert(2, "")
    saved = model.decoding.tokenizer
    if name != "v2_ctc":
        model.decoding.tokenizer = _IdTokenizer(len(saved))
        model.__dict__.pop("_token_flags", None)
    try:
        _check_end_to_end(model, wav, lines)
    finally:
        model.decoding.tokenizer = saved
        model.__dict__.pop("_token_flags", None)


def _check_end_to_end(model, wav, lines):
    theta = 0.7
    res = model.align_longform(wav, lines, gap_threshold=theta)
    assert len(res.segments) == len(lines) and res.unmatched, lines
    dur = wav.numel() / 16000
    for (a, b), (c, d) in zip(res.unmatched, res.unmatched[1:]):
        assert b < c
    words = res.words
    for a, b in res.unmatched:
        assert 0.0 <= a < b <= dur + 1e-9
        assert all(w.end <= a or b <= w.start for w in words), (a, b)
    # the oracle over one encoder pass: the stitched log-probs align_longform aligned
    windows, T = plan_windows(wav.numel(), 30.0, 4.0, model._encoded_length, 768)
    assert len(windows) > 2
    wav_d, length = model.prepare_wav(wav)
    with torch.inference_mode():
        lp = longform.stitch_ctc_log_probs(model, wav_d[0], windows, T, 16)[0].cpu().numpy()
    norm, ids, ranges = model._line_tokens(lines)
    edges = np.array(line_edges(ranges, len(ids)), np.uint8)
    log_theta = float(F32(math.log(theta)))
    fr, tok, vit, rows, flags, urows, ulogp = gap_replay(lp, T, ids, edges, log_theta)
    shift = compute_frame_shift(int(length[0]), T)
    assert res.unmatched == unmatched_intervals(torch.from_numpy(flags), shift)
    assert res.confidence == gap_confidence(float(vit), float(ulogp), T - urows)
    want = line_segments(norm, ranges, fr.tolist(), tok.tolist(), shift, float(vit))
    assert [(s.start, s.end, s.confidence) for s in res.segments] == [(s.start, s.end, s.confidence) for s in want]
    ll, mags = gap_forward64(lp, T, ids, edges, log_theta)
    assert abs(res.log_likelihood - ll) <= ctc_forward_bound(mags, ll)
    plain = model.align_longform(wav, lines)
    assert plain.unmatched is None and "unmatched" not in repr(plain)
