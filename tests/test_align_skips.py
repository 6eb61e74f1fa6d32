"""Long-form alignment that skips text lines the recording does not contain: gam_ctc_align_long_skips (include/gigaam_b200.h
has the definition) and `GigaAMASR.align_longform(..., skip_threshold=psi)` (INTEGRATION.md §7e).

The graph is gam_ctc_align_long_gaps' plus one edge per line, from the exit blank of the line end before it to its own exit
blank, at fp32(n_i) * log psi.  The recursion is still a fixed sequence of fp32 adds, maxes and strict compares, so the
numpy float32 oracle below (`skip_replay`) reproduces every output bit for bit except the forward score, which is compared
with a float64 recursion within test_align.py's bound.

CPU: the oracle against a float64 brute force over every path (ties built on purpose), its reduction to `gap_replay` at
log psi = -inf, planted missing lines, the skip sources, skipped segments, the record, the confidence rule, refusals and the
engine calls.  GPU: bit identity with the oracle on ragged batches at forced cluster sizes, the reductions to
gam_ctc_align_long_gaps and gam_ctc_align_long, planted missing lines (and a planted hour), NaN poisoning, refusals,
CUDA-graph capture, memory, and the public call end to end.
"""
import math

import numpy as np
import pytest
import torch

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, longform, synthetic
from gigaam_b200.longform import line_edges, line_segments, plan_windows, skip_edges, skipped_lines, unmatched_intervals
from gigaam_b200.timestamps_utils import compute_frame_shift, gap_confidence
from gigaam_b200.types import LongformAlignment, Segment

from test_align import F32, INF, NAN, _log_probs, ctc_forward_bound
from test_align_gaps import (_SentencePieceLike, _bits, _cpu_model, _dev, _emissions, _engine, _graph, _IdTokenizer, _model,
                             _random_edges, gap_replay)


# ------------------------------------------------------------------------------------------ the oracle
def _skips(edges, log_psi):
    """{x_i: (e_i, pen_i)} of the skip edges, pen_i = fp32(n_i) * log psi."""
    with np.errstate(invalid="ignore"):
        return {x: (e, F32(F32((x - e) // 2) * F32(log_psi))) for e, x in skip_edges(edges)}


def skip_replay(lp, Tb, y, edges, log_theta, log_psi, U=None):
    """gam_ctc_align_long_skips for one recording in numpy float32.  -> (frames [U], token_logp [U], viterbi, path_rows,
    unmatched [T] u8, unmatched_rows, unmatched_logp, skipped_rows, skip_logp)."""
    lp = np.asarray(lp, F32)
    T, V1 = lp.shape
    blank, n = V1 - 1, len(y)
    U = n if U is None else U
    frames, tok = np.full(U, -1, np.int32), np.full(U, -INF, F32)
    flags = np.zeros(T, np.uint8)
    if any(not 0 <= i < blank for i in y) or (Tb > 0 and np.isnan(lp[:Tb]).any()):
        tok[:n] = NAN
        return frames, tok, F32(NAN), Tb, flags, 0, F32(NAN), 0, F32(NAN)
    if Tb == 0:
        return frames, tok, F32(-INF), Tb, flags, 0, F32(0.0), 0, F32(0.0)
    lab, skip, bound = _graph(V1, y, edges)
    S = len(lab)
    e, g = _emissions(lp, Tb, lab, bound, log_theta)
    sk = _skips(edges, log_psi)
    xs = np.array(sorted(sk), np.int64)
    es = np.array([sk[x][0] for x in xs], np.int64)
    pens = np.array([sk[x][1] for x in xs], F32)
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
            if len(xs):
                c3 = (v[es] + pens).astype(F32)
                m3 = c3 > best[xs]
                best[xs[m3]] = c3[m3]
                code[t, xs[m3]] = 3
            v = (e[t] + best).astype(F32)
    s = S - 1
    if S >= 2 and v[S - 2] > v[S - 1]:
        s = S - 2
    vit = v[s]
    if vit == -INF:
        return frames, tok, vit, Tb, flags, 0, F32(0.0), 0, F32(0.0)
    taken = []                                                     # (frame, pen) of the skip edges on the path
    for t in range(Tb - 1, -1, -1):
        if s & 1:
            frames[s >> 1] = t
        elif bound[s] and g[t] > lp[t, blank]:
            flags[t] = 1
        if t > 0:
            c = int(code[t, s])
            if c == 3:
                taken.append((t, sk[s][1]))
                s = sk[s][0]
            else:
                s -= c
    on = frames[:n] >= 0
    tok[:n][on] = lp[frames[:n][on], np.asarray(y, np.int64)[on]]
    total = F32(0.0)
    for t in np.flatnonzero(flags):
        total = F32(total + g[t])
    pen_sum = F32(0.0)
    for _, pen in sorted(taken):                                   # in frame order
        pen_sum = F32(pen_sum + pen)
    return frames, tok, vit, Tb, flags, int(flags.sum()), total, len(taken), pen_sum


def _successors(S, skip, sk):
    """Every edge of the graph with skips: succ[s] = [(s', weight)]."""
    src = {e: (x, float(pen)) for x, (e, pen) in sk.items()}
    succ = []
    for s in range(S):
        out = [(s, 0.0)]
        if s + 1 < S:
            out.append((s + 1, 0.0))
        if s + 2 < S and skip[s + 2]:
            out.append((s + 2, 0.0))
        if s in src and src[s][1] != -INF:
            out.append(src[s])
        succ.append(out)
    return succ


def skip_forward64(lp, Tb, y, edges, log_theta, log_psi):
    """The forward score of the graph with skips in float64 over the fp32 emissions and penalties, and the largest finite
    |f| per frame."""
    lp = np.asarray(lp, F32)
    lab, skip, bound = _graph(lp.shape[1], y, edges)
    S = len(lab)
    e, _ = _emissions(lp, Tb, lab, bound, log_theta)
    e = e.astype(np.float64)
    sk = _skips(edges, log_psi)
    f = np.full(S, -INF)
    f[:2] = e[0, :2]
    mags = [np.abs(f[np.isfinite(f)]).max(initial=0.0)]
    with np.errstate(invalid="ignore", divide="ignore"):
        for t in range(1, Tb):
            a = np.concatenate([[-INF], f[:-1]])
            b = np.where(skip, np.concatenate([[-INF, -INF], f[:-2]])[:S], -INF)
            for x, (src, pen) in sk.items():
                b[x] = f[src] + float(pen)
            f = np.logaddexp(np.logaddexp(f, a), b) + e[t]
            mags.append(np.abs(f[np.isfinite(f)]).max(initial=0.0))
    ll = np.logaddexp(f[S - 1], f[S - 2]) if S >= 2 else f[0]
    return float(ll), mags


def _brute_force(lp, Tb, y, edges, log_theta, log_psi):
    """Every path of the graph with skips in float64: (best score, runner-up score, the best path's states, forward score).
    Among paths of equal best score the path is the one the tie rules pick: read backwards, the larger state first (the
    final state S - 1 before S - 2, then stay before s - 1 before s - 2 before the skip source)."""
    lp = np.asarray(lp, F32)
    lab, skip, bound = _graph(lp.shape[1], y, edges)
    S = len(lab)
    e, _ = _emissions(lp, Tb, lab, bound, log_theta)
    e = e.astype(np.float64)
    succ = _successors(S, skip, _skips(edges, log_psi))
    scores, paths = [], []

    def walk(t, s, acc, path):
        acc = acc + e[t, s]
        path = path + [s]
        if t == Tb - 1:
            if s >= S - 2:
                scores.append(acc)
                paths.append(path)
            return
        for nxt, w in succ[s]:
            walk(t + 1, nxt, acc + w, path)
    for s0 in range(min(2, S)):
        walk(0, s0, 0.0, [])
    if not scores:
        return -INF, -INF, None, -INF
    best = max(scores)
    tied = [p for sc, p in zip(scores, paths) if sc == best]
    pick = max(tied, key=lambda p: p[::-1])
    second = max([sc for sc in scores if sc != best], default=-INF)
    return best, second if len(tied) == 1 else best, pick, float(np.logaddexp.reduce(scores))


def _frames_of(path, n):
    fr = np.full(n, -1, np.int32)
    for t in range(len(path) - 1, -1, -1):
        if path[t] & 1:
            fr[path[t] >> 1] = t
    return fr


# ------------------------------------------------------------------------------------------ CPU: the oracle
def test_oracle_matches_a_float64_brute_force_over_every_path():
    rng = np.random.default_rng(0)
    checked = skipped = tie_checked = 0
    for case in range(500):
        ties = case % 2 == 1
        V1 = int(rng.integers(3, 6))
        Tb = int(rng.integers(1, 8))
        n = int(rng.integers(0, 6))
        y = rng.integers(0, V1 - 1, n).tolist()
        edges = _random_edges(rng, n)
        if ties:                                                   # quarter steps: every sum is exact in fp32 and float64
            lp = _log_probs(rng, (Tb, V1), ties=True)
            log_theta = [-INF, -1.0, -0.25][case % 3]
            log_psi = [-0.5, -1.0, -0.25, 0.0][case % 4]
        else:
            lp = _log_probs(rng, (Tb, V1))
            log_theta = -INF if case % 3 == 0 else float(F32(math.log(rng.uniform(1e-3, 1.0))))
            log_psi = float(F32(math.log(rng.uniform(1e-2, 1.0)))) if case % 7 else 0.0
        fr, tok, vit, rows, flags, urows, ulogp, srows, slogp = skip_replay(lp, Tb, y, edges, log_theta, log_psi)
        assert rows == Tb and urows == int(flags.sum())
        best, second, path, fwd = _brute_force(lp, Tb, y, edges, log_theta, log_psi)
        if best == -INF:
            assert vit == -INF and (fr == -1).all() and urows == 0 and srows == 0 and slogp == 0.0
            continue
        assert abs(float(vit) - best) <= 1e-5 * (1 + abs(best)), (case, vit, best)
        want_fwd, _ = skip_forward64(lp, Tb, y, edges, log_theta, log_psi)
        assert abs(want_fwd - fwd) <= 1e-9 * (1 + abs(fwd)), case
        if not ties and best - second < 1e-4:
            continue                                               # near-tie without exact sums: the path is not determined
        if ties:
            assert float(vit) == best, case                         # exact arithmetic: the same score, and the same path
            tie_checked += best == second
        assert np.array_equal(fr, _frames_of(path, n)), (case, fr, path)
        sk = _skips(edges, log_psi)
        jumps = [(t, sk[path[t]][1]) for t in range(1, Tb)   # only the skip edge enters a blank from further left
                 if path[t] in sk and path[t - 1] == sk[path[t]][0]]
        assert srows == len(jumps), (case, path)
        want = F32(0.0)
        for _, pen in jumps:
            want = F32(want + pen)
        assert F32(slogp).view(np.uint32) == want.view(np.uint32), case
        assert np.isneginf(tok[fr < 0]).all() and np.isfinite(tok[fr >= 0]).all()
        checked += 1
        skipped += srows > 0
    assert checked > 250 and skipped > 40 and tie_checked > 20, (checked, skipped, tie_checked)


def test_log_psi_minus_inf_is_gap_replay():
    rng = np.random.default_rng(3)
    for case in range(150):
        V1, Tb, n = 5, int(rng.integers(1, 14)), int(rng.integers(0, 7))
        y = rng.integers(0, V1 - 1, n).tolist()
        lp = _log_probs(rng, (Tb, V1), ties=case % 2 == 0)
        edges = _random_edges(rng, n)
        log_theta = -INF if case % 3 == 0 else -0.5
        got = skip_replay(lp, Tb, y, edges, log_theta, -INF)
        want = gap_replay(lp, Tb, y, edges, log_theta)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
        assert F32(got[2]).view(np.uint32) == F32(want[2]).view(np.uint32) and got[3] == want[3]
        assert np.array_equal(got[4], want[4]) and got[5] == want[5] and F32(got[6]).view(np.uint32) == F32(want[6]).view(np.uint32)
        assert got[7] == 0 and (got[8] == 0.0 or math.isnan(want[2]))


# ------------------------------------------------------------------------------------------ planted missing lines
_SPACE = 0                                                         # the joining token of the planted texts


def _planted_text(V1, n_lines, rng, line_len=(8, 12)):
    """Lines of letters (ids 1 .. V1 - 2, no id equal to its neighbour) joined by the space token 0, as a charwise text."""
    lines, prev = [], -1
    for _ in range(n_lines):
        row = []
        for _ in range(int(rng.integers(*line_len))):
            c = int(rng.integers(1, V1 - 1))
            while c == prev:
                c = int(rng.integers(1, V1 - 1))
            row.append(c)
            prev = c
        lines.append(row)
    ids, ranges = [], []
    for row in lines:
        if ids:
            ids.append(_SPACE)
        ranges.append((len(ids), len(ids) + len(row)))
        ids.extend(row)
    return ids, ranges


def _planted_audio(V1, ids, ranges, missing, lead=3, between=3, tail=3, spare=64):
    """Log-probs that spell the text without the missing lines: the tokens a skip of those lines leaves (each line's tokens
    on consecutive frames, `between` blank frames before each kept joining space, `spare` instead before the first space
    between two kept lines, and one after it) and blank elsewhere.  The blank stretches next to a missing line are too
    short for it, so a path without skips must move its neighbours; the spare frames make sure it has a path.
    -> lp [T, V1] f32, the planted frame of every kept token (-1 for the jumped ones), line_edges."""
    jumped = np.zeros(len(ids), bool)
    edges = line_edges(ranges, len(ids))
    for li, (e, x) in enumerate(skip_edges(edges)):
        if li in missing:
            jumped[e // 2:x // 2] = True
    plan, t = [], lead
    want = np.full(len(ids), -1, np.int32)
    for i, c in enumerate(ids):
        if jumped[i]:
            continue
        if c == _SPACE:
            li = next(k for k, (a, _) in enumerate(ranges) if a == i + 1)   # the space joins lines li - 1 and li
            if spare and li - 1 not in missing and li not in missing:
                t += spare
                spare = 0
            else:
                t += between
            want[i] = t
            t += 2
        else:
            want[i] = t
            t += 1
    T = t + tail
    lp = np.full((T, V1), F32(-30.0), F32)
    lp[:, V1 - 1] = 0.0
    for i in np.flatnonzero(want >= 0):
        lp[want[i], V1 - 1] = -30.0
        lp[want[i], ids[i]] = 0.0 if i % 3 else F32(-0.25)
    return lp, want, np.array(edges, np.uint8)


_MISSING = [[2], [0], [4], [1, 2], [0, 1, 4]]                      # a middle line, the first, the last, two consecutive, ...


def test_planted_missing_lines_are_skipped_in_the_replay():
    rng = np.random.default_rng(5)
    V1, log_psi = 12, float(F32(math.log(0.5)))
    for missing in _MISSING:
        ids, ranges = _planted_text(V1, 5, rng)
        lp, want, edges = _planted_audio(V1, ids, ranges, missing)
        T = lp.shape[0]
        out = skip_replay(lp, T, ids, edges, -INF, log_psi)
        assert skipped_lines(ranges, out[0].tolist()) == missing
        assert np.array_equal(out[0], want), missing
        assert out[7] == len(missing) and math.isfinite(out[2])
        plain = gap_replay(lp, T, ids, edges, -INF)
        kept = want >= 0
        assert not np.array_equal(plain[0][kept], want[kept]), missing    # the missing lines pull their neighbours
        assert (plain[0] >= 0).all()


def test_skip_sources_of_charwise_and_sentencepiece_texts():
    model = _cpu_model("v2_ctc")
    tok = model.decoding.tokenizer
    sp = tok.vocab.index(" ")
    _, ids, ranges = model._line_tokens(["аб", "", "в", "гд е"])
    assert ids == tok.encode("аб") + [sp] + tok.encode("в") + [sp] + tok.encode("гд е")
    edges = line_edges(ranges, len(ids))
    # lines end at tokens 1, 3 and 8: exits 4, 8, 18; the second and third edges also jump the joining space
    assert skip_edges(edges) == [(0, 4), (4, 8), (8, 18)]
    assert [(x - e) // 2 for e, x in skip_edges(edges)] == [2, 2, 5]
    assert skip_edges([]) == []
    saved = model.decoding.tokenizer
    try:
        model.decoding.tokenizer = _SentencePieceLike()
        _, ids, ranges = model._line_tokens(["Привет", "", "как дела", "как"])
        assert skip_edges(line_edges(ranges, len(ids))) == [(0, 4), (4, 10), (10, 12)]   # no joining tokens: n_i = len
    finally:
        model.decoding.tokenizer = saved
    frames = [0, 1, -1, -1, -1, 5, 6, 7, -1]
    assert skipped_lines([(0, 2), (2, 2), (3, 5), (5, 8)], frames) == [2]
    assert skipped_lines([(0, 2), (3, 5)], [-1, -1, 2, -1, -1]) == [0, 1]


def test_skipped_segments_record_and_confidence():
    ranges = [(0, 2), (3, 5), (6, 8), (9, 11)]
    frames = [0, 1, -1, -1, -1, 7, 8, 9, 10, 11, 12]
    logp = [-0.1] * 11
    norm = ["аб", "вг", "де", "жз"]
    segs = line_segments(norm, ranges, frames, logp, 0.04, -5.0, [], [], skipped=[1])
    assert segs[1].text == "вг" and segs[1].start == segs[1].end == segs[0].end and math.isnan(segs[1].confidence)
    assert segs[1].words == [] and segs[2].start == 8 * 0.04
    segs = line_segments(norm, [(0, 2)] + ranges[1:], [-1, -1] + frames[2:], logp, 0.04, -5.0, None, None, skipped=[0, 1])
    assert segs[0].start == segs[0].end == 0.0 and segs[1].start == 0.0 and segs[0].words is None
    seg = Segment("аб", 0.0, 0.08, None, 0.5)
    plain = LongformAlignment([seg], -3.5, 0.7)
    assert plain.skipped is None and "skipped" not in repr(plain)
    gapped = LongformAlignment([seg], -3.5, 0.7, [(1.0, 2.0)])     # positional construction as before
    assert gapped.skipped is None and repr(gapped).endswith("unmatched=[(1.0, 2.0)])")
    skipping = LongformAlignment([seg], -3.5, 0.7, None, [0, 2])
    assert repr(skipping).endswith("confidence=0.7, skipped=[0, 2])") and "unmatched" not in repr(skipping)
    assert skipping != plain and skipping == LongformAlignment([seg], -3.5, 0.7, skipped=[0, 2])
    assert LongformAlignment([seg], -3.5, 0.7, skipped=[]) != plain
    assert gap_confidence(-6.0, -1.0, 4, -1.0) == math.exp(-1.0)
    assert gap_confidence(-6.0, -1.0, 4) == math.exp(-5.0 / 4) and math.isnan(gap_confidence(-6.0, 0.0, 0, -2.0))


def test_skip_threshold_refusals_before_device_work():
    model = _cpu_model("v2_ctc")
    wav = np.zeros(16000, np.float32)
    for psi in (0.0, -0.5, 1.5, NAN, INF, 1e-46, 1.0000001):
        with pytest.raises(ValueError, match="skip_threshold"):
            model.align_longform(wav, "а", skip_threshold=psi)
        with pytest.raises(ValueError, match="skip_threshold"):
            model.align_longform(wav, "а", gap_threshold=0.5, skip_threshold=psi)
    with pytest.raises(ValueError, match="gap_threshold"):
        model.align_longform(wav, "а", gap_threshold=2.0, skip_threshold=0.5)
    for name in ("v2_rnnt", "v3_e2e_rnnt"):
        with pytest.raises(NotImplementedError, match="CTC"):
            _cpu_model(name).align_longform(wav, "а", skip_threshold=NAN)   # before the threshold check


def test_exports():
    lib = _lib.load()
    for name in ("gam_ctc_align_long_skips", "gam_ctc_align_long_skips_workspace_bytes", "gam_test_ctc_align_long_skips"):
        assert name in _lib.EXPORTS and hasattr(lib, name)


class _Recorder:
    """Stands in for the engine: records the ctc_align_long calls and returns frames that skip line `skip`."""

    def __init__(self, skip=None):
        self.calls = []
        self.device = torch.device("cpu")
        self.num_classes = 34
        self.skip = skip

    def ctc_align_long(self, lp, enc_len, targets, target_len, **kw):
        self.calls.append((4, tuple(sorted(kw)), kw.get("gaps", (None, None))[1], kw.get("skips")))
        U, T = targets.shape[1], lp.shape[1]
        frames = torch.arange(U, dtype=torch.int32)[None]
        if self.skip is not None:
            frames[0, self.skip[0]:self.skip[1]] = -1
        outs = (frames, torch.zeros((1, U)), torch.tensor([-10.0]), torch.tensor([-2.0]), torch.tensor([T], dtype=torch.int32))
        if "gaps" in kw:
            outs += (torch.zeros((1, T), dtype=torch.uint8), torch.tensor([2], dtype=torch.int32), torch.tensor([-3.0]))
        if "skips" in kw:
            outs += (torch.tensor([1], dtype=torch.int32), torch.tensor([-4.0]))
        return outs

    def __getattr__(self, name):
        raise AssertionError(f"unexpected engine call {name}")


def test_engine_calls_with_and_without_skip_threshold(monkeypatch):
    model = _cpu_model("v2_ctc")
    monkeypatch.setattr(longform, "stitch_ctc_log_probs", lambda m, wav, windows, T, bs: torch.zeros((1, T, 34)))
    wav = np.zeros(16000, np.float32)
    lines = ["аб", "в", "гд"]                                      # tokens: а б _ в _ г д
    eng = _Recorder()
    monkeypatch.setattr(model, "_get_engine", lambda: eng)
    for kwargs in ({}, {"skip_threshold": None}, {"gap_threshold": None, "skip_threshold": None}):
        eng.calls.clear()
        res = model.align_longform(wav, lines, word_timestamps=False, **kwargs)
        assert eng.calls == [(4, (), None, None)] and res.skipped is None and res.unmatched is None
    eng.calls.clear()
    res = model.align_longform(wav, lines, word_timestamps=False, gap_threshold=0.5)
    assert eng.calls == [(4, ("gaps",), float(F32(math.log(0.5))), None)] and res.skipped is None
    eng.skip = (2, 4)                                              # the joining space and "в": line 1 skipped
    eng.calls.clear()
    res = model.align_longform(wav, lines, word_timestamps=False, skip_threshold=0.25)
    log_psi = float(F32(math.log(0.25)))
    assert eng.calls == [(4, ("gaps", "skips"), -INF, log_psi)]
    assert res.skipped == [1] and res.unmatched is None
    assert res.segments[1].start == res.segments[1].end == res.segments[0].end and math.isnan(res.segments[1].confidence)
    T = model._encoded_length(16000)
    assert res.confidence == math.exp((-10.0 - -3.0 - -4.0) / (T - 2))
    eng.calls.clear()
    res = model.align_longform(wav, lines, word_timestamps=False, gap_threshold=0.5, skip_threshold=0.25)
    assert eng.calls == [(4, ("gaps", "skips"), float(F32(math.log(0.5))), log_psi)]
    assert res.skipped == [1] and res.unmatched == []


class _WordRecorder(_Recorder):
    """_Recorder that also takes group_words calls: it records the tokens and frames it is given and finds no words."""

    def group_words(self, targets, frames, target_len, flags):
        self.calls.append(("words", targets[0, :int(target_len[0])].tolist(), frames[0, :int(target_len[0])].tolist()))
        z = torch.zeros((1, 1), dtype=torch.int32)
        return z, z, z, z, torch.zeros(1, dtype=torch.int32)


def test_word_timestamps_when_lines_are_skipped(monkeypatch):
    model = _cpu_model("v2_ctc")
    monkeypatch.setattr(longform, "stitch_ctc_log_probs", lambda m, wav, windows, T, bs: torch.zeros((1, T, 34)))
    wav = np.zeros(16000, np.float32)
    lines = ["аб", "в", "гд"]                                      # tokens: а б _ в _ г д
    _, ids, _ = model._line_tokens(lines)
    eng = _WordRecorder(skip=(0, len(ids)))                        # the path skips every line
    monkeypatch.setattr(model, "_get_engine", lambda: eng)
    res = model.align_longform(wav, lines, skip_threshold=0.5)     # word_timestamps=True: no grouping of nothing
    assert [c[0] for c in eng.calls] == [4] and res.skipped == [0, 1, 2] and res.words == []
    assert all(seg.start == seg.end == 0.0 and seg.words == [] and math.isnan(seg.confidence) for seg in res.segments)
    res = model.align_longform(wav, lines, word_timestamps=False, skip_threshold=0.5)
    assert res.skipped == [0, 1, 2] and all(seg.words is None for seg in res.segments)
    eng.skip = (2, 4)                                              # line 1 skipped: only the aligned tokens are grouped
    eng.calls.clear()
    res = model.align_longform(wav, lines, skip_threshold=0.5)
    assert res.skipped == [1]
    assert eng.calls[1] == ("words", ids[:2] + ids[4:], [0, 1, 4, 5, 6])


# ------------------------------------------------------------------------------------------ GPU helpers
def _run(eng, lp, enc_len, targets, target_len, edges, log_theta, log_psi, cluster_ctas=None):
    out = eng.ctc_align_long(torch.from_numpy(lp).to(_dev()), torch.tensor(enc_len), torch.from_numpy(targets),
                             torch.tensor(target_len), cluster_ctas=cluster_ctas,
                             gaps=(torch.from_numpy(edges).to(_dev()), log_theta), skips=log_psi)
    return [t.cpu().numpy() for t in out]


def _check_oracle(got, lp, enc_len, targets, target_len, edges, log_theta, log_psi):
    fr, tok, vit, ll, rows, flags, urows, ulogp, srows, slogp = got
    T = lp.shape[1]
    for b in range(lp.shape[0]):
        Tb, Ub = min(max(enc_len[b], 0), T), target_len[b]
        y = targets[b, :Ub].tolist()
        w = skip_replay(lp[b], Tb, y, edges[b, :Ub], log_theta, log_psi, targets.shape[1])
        assert np.array_equal(fr[b], w[0]), b
        assert np.array_equal(tok[b].view(np.uint32), w[1].view(np.uint32)), b
        assert F32(vit[b]).view(np.uint32) == F32(w[2]).view(np.uint32), (b, vit[b], w[2])
        assert rows[b] == w[3] and np.array_equal(flags[b], w[4]) and urows[b] == w[5], b
        assert F32(ulogp[b]).view(np.uint32) == F32(w[6]).view(np.uint32), (b, ulogp[b], w[6])
        assert srows[b] == w[7] and F32(slogp[b]).view(np.uint32) == F32(w[8]).view(np.uint32), (b, srows[b], slogp[b], w[7:])
        if math.isfinite(vit[b]):
            want, mags = skip_forward64(lp[b], Tb, y, edges[b, :Ub], log_theta, log_psi)
            assert abs(ll[b] - want) <= ctc_forward_bound(mags, want), (b, ll[b], want)
        else:
            assert F32(ll[b]).view(np.uint32) == F32(vit[b]).view(np.uint32), b


def _edges_of(lengths, U):
    bounds = np.cumsum([0] + list(lengths)).tolist()
    return line_edges(list(zip(bounds[:-1], bounds[1:])), U)


def _ragged_batch(rng, V1):
    """Ragged lengths, enc_len 0, U = 0, a NaN row inside and one past a recording, a bad id.  Lines of 1 to 80 tokens: at
    16 states per CTA every line of more than 8 tokens has its skip source in another CTA, and the 70- and 80-token lines
    are longer than a CTA's share at 2 CTAs.  Recordings 1 and 6 have planted missing lines."""
    B, T, U = 9, 300, 120
    lp = _log_probs(rng, (B, T, V1))
    targets = rng.integers(0, V1 - 1, (B, U)).astype(np.int32)
    enc_len = [300, 280, 0, 200, 300, 150, 260, 300, 300]
    target_len = [120, 104, 10, 0, 120, 60, 0, 100, 120]
    lines = {0: [3, 80, 5, 20, 12], 1: None, 2: [10], 4: [1, 2, 1, 30, 70, 4, 12], 5: [60], 7: [25, 25, 25, 25],
             8: [40, 40, 40]}
    edges = np.zeros((B, U), np.uint8)
    for b, ls in lines.items():
        if ls is not None:
            edges[b, :target_len[b]] = _edges_of(ls, target_len[b])
    # recording 1: a charwise-like text whose line 2 and lines 5, 6 are missing from its planted audio
    ids, ranges = _planted_text(V1, 8, rng, (8, 16))
    ids, ranges = ids[:104], [(a, min(b, 104)) for a, b in ranges if a < 104]
    plp, _, pedges = _planted_audio(V1, ids, ranges, [2, 5, 6], between=2)
    n = min(plp.shape[0], T)
    lp[1, :n] = plp[:n]
    enc_len[1] = n
    targets[1, :len(ids)] = ids
    target_len[1] = len(ids)
    edges[1, :len(ids)] = pedges
    lp[5, 70, :] = NAN                                             # inside the recording: poisoned
    lp[7, 300 - 1, :] = NAN
    enc_len[7] = 290                                               # past the recording: not read
    targets[8, 3] = -4
    return lp, enc_len, targets, target_len, edges


# ------------------------------------------------------------------------------------------ GPU: kernel
@pytest.mark.gpu
@pytest.mark.parametrize("V1", [34, 257])
def test_bit_identical_to_the_oracle_on_a_ragged_batch(V1):
    eng = _engine(V1)
    assert eng.num_classes == V1
    rng = np.random.default_rng(V1)
    lp, enc_len, targets, target_len, edges = _ragged_batch(rng, V1)
    skipped = 0
    for log_theta, psi in ((-INF, 0.5), (float(F32(math.log(0.3))), 0.9), (float(F32(math.log(0.05))), 0.02)):
        log_psi = float(F32(math.log(psi)))
        base = None
        for c in (None, 1, 2, 3, 4, 8, 16):
            got = _run(eng, lp, enc_len, targets, target_len, edges, log_theta, log_psi, c)
            if c is not None:
                assert eng.last_align_long_plan[0] == c
            if base is None:
                _check_oracle(got, lp, enc_len, targets, target_len, edges, log_theta, log_psi)
                base = got
                skipped += int(got[8].sum())
            else:
                assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(got, base)), c
        assert base[8][1] >= 3 and (base[0][1] == -1).sum() > 0
        for b in (0, 1, 4, 8):                                     # alone: the same bits as in the batch
            alone = _run(eng, lp[b:b + 1], enc_len[b:b + 1], targets[b:b + 1], target_len[b:b + 1], edges[b:b + 1],
                         log_theta, log_psi)
            assert all(np.array_equal(x.view(np.uint8), y[b:b + 1].view(np.uint8)) for x, y in zip(alone, base)), b
        assert base[8][5] == 0 and math.isnan(base[9][5]) and math.isnan(base[9][8])   # poisoned, bad id
    assert skipped > 6


@pytest.mark.gpu
def test_log_psi_minus_inf_equals_the_gaps_and_plain_calls():
    eng = _engine(34)
    rng = np.random.default_rng(4)
    lp, enc_len, targets, target_len, edges = _ragged_batch(rng, 34)
    lp[4, :, 5] = 0.0                                              # ties, and -inf entries
    lp[0, 10, :] = -INF
    args = (torch.from_numpy(lp).to(_dev()), torch.tensor(enc_len), torch.from_numpy(targets), torch.tensor(target_len))
    for c in (None, 16):
        for log_theta in (float(F32(math.log(0.2))), -INF):
            gaps = (torch.from_numpy(edges), log_theta)
            want = eng.ctc_align_long(*args, cluster_ctas=c, gaps=gaps)
            got = eng.ctc_align_long(*args, cluster_ctas=c, gaps=gaps, skips=-INF)
            assert all(torch.equal(_bits(x), _bits(y)) for x, y in zip(got[:8], want))
            assert not got[8].any()
            assert torch.equal(got[9].isnan(), want[7].isnan()) and not got[9].nan_to_num().any()
    clean = np.nan_to_num(lp, nan=-3.0)
    clean_targets = targets.copy()
    clean_targets[8, 3] = 1
    args = (torch.from_numpy(clean).to(_dev()), torch.tensor(enc_len), torch.from_numpy(clean_targets), torch.tensor(target_len))
    want = eng.ctc_align_long(*args)
    got = eng.ctc_align_long(*args, gaps=(torch.from_numpy(edges), -INF), skips=-INF)
    assert all(torch.equal(_bits(x), _bits(y)) for x, y in zip(got[:5], want))


def _most_ctas(U):
    """The largest forced cluster size in (16, 8, 4, 2) that leaves no CTA without states."""
    S = 2 * U + 1
    return next(c for c in (16, 8, 4, 2) if (c - 1) * (-(-(-(-S // c)) // 16) * 16) < S)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [None, 3, "most"])
def test_planted_missing_lines(c):
    eng = _engine(34)
    rng = np.random.default_rng(11)
    log_psi = float(F32(math.log(0.7)))
    for missing in _MISSING:
        ids, ranges = _planted_text(34, 5, rng, (6, 20))
        lp, want, edges = _planted_audio(34, ids, ranges, missing)
        T, U = lp.shape[0], len(ids)
        cc = _most_ctas(U) if c == "most" else c
        targets = np.array([ids], np.int32)
        got = _run(eng, lp[None], [T], targets, [U], edges[None], -INF, log_psi, cc)
        _check_oracle(got, lp[None], [T], targets, [U], edges[None], -INF, log_psi)
        assert np.array_equal(got[0][0], want) and skipped_lines(ranges, got[0][0].tolist()) == missing
        plain = eng.ctc_align_long(torch.from_numpy(lp[None]).to(_dev()), torch.tensor([T]), torch.from_numpy(targets),
                                   torch.tensor([U]), cluster_ctas=cc)[0][0].cpu().numpy()
        kept = want >= 0
        assert (plain >= 0).all() and not np.array_equal(plain[kept], want[kept]), missing


@pytest.mark.gpu
def test_planted_hour_with_missing_lines():
    """T' = 90 000 frames, U = 65 536 tokens in 128 lines of 512 (SentencePiece-like: no joining tokens).  Every line but
    the first, line 40, lines 70-71 and the last is spelled: its tokens peaked on consecutive frames, blank on the frames
    between lines.  The library's cluster size; exactly those lines must be skipped, every other token land on its frame,
    and the path score and skip score equal their fp32 sums in frame order."""
    eng = _engine(34)
    V1, T, U, L = 34, 90000, 65536, 128
    missing = [0, 40, 70, 71, L - 1]
    g = torch.Generator().manual_seed(7)
    steps = torch.randint(1, V1 - 2, (U,), generator=g)
    y = (torch.cumsum(steps, 0) % (V1 - 1)).to(torch.int32)       # no label repeats its neighbour
    ranges = [(i * 512, (i + 1) * 512) for i in range(L)]
    want = torch.full((U,), -1, dtype=torch.int64)
    t = 20
    for li, (a, b) in enumerate(ranges):
        if li in missing:
            continue
        want[a:b] = torch.arange(t, t + 512)
        t += 512 + 30
    assert t + 20 <= T
    lp = torch.full((1, T, V1), -30.0, device=_dev())
    lp[0, :, V1 - 1] = 0.0
    kept = torch.nonzero(want >= 0).reshape(-1)
    fd = want[kept].to(_dev())
    lp[0, fd, V1 - 1] = -30.0
    lp[0, fd, y[kept].long().to(_dev())] = 0.0
    sevens = kept[kept % 7 == 0]
    lp[0, want[sevens].to(_dev()), y[sevens].long().to(_dev())] = -0.25
    edges = torch.tensor(line_edges(ranges, U), dtype=torch.uint8)
    log_psi = float(F32(math.log(0.5)))
    out = eng.ctc_align_long(lp, torch.tensor([T]), y[None], torch.tensor([U]), gaps=(edges[None], -INF), skips=log_psi)
    frames, tok, vit, ll, rows, flags, urows, ulogp, srows, slogp = (x.cpu() for x in out)
    assert torch.equal(frames[0].long(), want)
    assert skipped_lines(ranges, frames[0].tolist()) == missing and int(srows[0]) == len(missing)
    assert torch.isneginf(tok[0][want < 0]).all() and int(urows[0]) == 0
    pen = F32(F32(512) * F32(log_psi))
    s = F32(0.0)
    for _ in missing:
        s = F32(s + pen)
    assert F32(slogp[0]) == s
    v = F32(0.0)                                                   # blank frames add +0: where the skips land is immaterial
    per_frame = np.zeros(T, F32)
    per_frame[want[sevens].numpy()] = F32(-0.25)
    first_kept = int(want[kept[0]])
    skips_at = {}                                                  # each skip before the frame of the next kept line
    for li in missing:
        nxt = next((want[a].item() for a, _ in ranges[li + 1:] if want[a] >= 0), T)
        skips_at.setdefault(nxt - 1, 0)
        skips_at[nxt - 1] += 1
    for t in range(T):
        for _ in range(skips_at.get(t, 0)):
            v = F32(v + pen)
        v = F32(v + per_frame[t])
    assert first_kept > 0 and F32(vit[0]) == v and int(rows[0]) == T and math.isfinite(float(ll[0]))


@pytest.mark.gpu
def test_refusals_of_the_c_level():
    eng = _engine(34)
    lp = torch.zeros(1, 4, 34, device=_dev())
    args = (lp, torch.tensor([4]), torch.zeros(1, 2, dtype=torch.int32), torch.tensor([2]))
    gaps = (torch.tensor([[1, 2]], dtype=torch.uint8), -INF)
    for bad in (NAN, 0.5, INF):
        with pytest.raises(_lib.GamError, match="log_psi"):
            eng.ctc_align_long(*args, gaps=gaps, skips=bad)
    with pytest.raises(_lib.GamError, match="log_theta"):
        eng.ctc_align_long(*args, gaps=(gaps[0], NAN), skips=-1.0)
    with pytest.raises(ValueError, match="needs gaps"):
        eng.ctc_align_long(*args, skips=-1.0)
    eng.ctc_align_long(*args, gaps=gaps, skips=0.0)
    with pytest.raises(ValueError):
        eng.ctc_align_long(lp, torch.tensor([4]), torch.zeros(1, 65537, dtype=torch.int32), torch.tensor([1]),
                           gaps=(torch.zeros(1, 65537, dtype=torch.uint8), -1.0), skips=-1.0)
    with pytest.raises(_lib.GamError, match="without states"):
        eng.ctc_align_long(*args, cluster_ctas=16, gaps=gaps, skips=-1.0)
    lib, h = eng.lib, eng.handle
    enc_d, tgt_d, tlen_d = args[1].to(_dev()).int(), args[2].to(_dev()), args[3].to(_dev()).int()
    outs = [torch.zeros(1, 2, dtype=torch.int32, device=_dev())] + [torch.zeros(2, device=_dev()) for _ in range(9)]
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=_dev())
    e = gaps[0].to(_dev())
    ptrs = [o.data_ptr() for o in outs]
    # skipped_rows is checked by gam_ctc_align_long_skips itself, skip_logp by the shared run: one NULL each
    for null in (8, 9):
        with pytest.raises(_lib.GamError, match="NULL"):
            rc = lib.gam_ctc_align_long_skips(h, lp.data_ptr(), enc_d.data_ptr(), tgt_d.data_ptr(), tlen_d.data_ptr(), e.data_ptr(),
                                              1, 4, 2, -INF, -1.0, ws.data_ptr(), ws.numel(),
                                              *[None if k == null else p for k, p in enumerate(ptrs)], None)
            _lib.check(lib, h, rc, "gam_ctc_align_long_skips")
    rc = lib.gam_ctc_align_long_skips(h, lp.data_ptr(), enc_d.data_ptr(), tgt_d.data_ptr(), tlen_d.data_ptr(), e.data_ptr(), 1, 4, 2,
                                      -INF, -1.0, ws.data_ptr(), ws.numel(), *ptrs, None)
    _lib.check(lib, h, rc, "gam_ctc_align_long_skips")              # the same call with every pointer is accepted


@pytest.mark.gpu
def test_graph_capture_and_memory():
    eng = _engine(34)
    rng = np.random.default_rng(2)
    B, T, U = 2, 3000, 1200
    lp = torch.from_numpy(_log_probs(rng, (B, T, 34))).to(_dev())
    targets = torch.from_numpy(rng.integers(0, 33, (B, U)).astype(np.int32)).to(_dev())
    enc_len = torch.tensor([3000, 2500], dtype=torch.int32, device=_dev())
    tlen = torch.tensor([1200, 700], dtype=torch.int32, device=_dev())
    edges = torch.from_numpy(np.stack([_edges_of([5, 300, 20, 8] * 3 + [201], U)] * B).astype(np.uint8)).to(_dev())
    gaps = (edges, float(F32(math.log(0.2))))
    log_psi = float(F32(math.log(0.9)))

    def peak(**kw):
        eng._ws_align._d.clear()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = eng.ctc_align_long(lp, enc_len, targets, tlen, **kw)
        torch.cuda.synchronize()
        del out
        return torch.cuda.max_memory_allocated() - base
    gapped, skipping = peak(gaps=gaps), peak(gaps=gaps, skips=log_psi)
    assert 0 < skipping - gapped <= 2 * 512, (gapped, skipping)    # two [B] outputs, no table
    want = [t.clone() for t in eng.ctc_align_long(lp, enc_len, targets, tlen, gaps=gaps, skips=log_psi)]
    assert int(want[8].sum()) > 0
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        eng.ctc_align_long(lp, enc_len, targets, tlen, gaps=gaps, skips=log_psi)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            captured = eng.ctc_align_long(lp, enc_len, targets, tlen, gaps=gaps, skips=log_psi)
    torch.cuda.current_stream().wait_stream(stream)
    for t in captured:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(_bits(x), _bits(y)) for x, y in zip(captured, want))


# ------------------------------------------------------------------------------------------ GPU: end to end
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v1_ctc", "v2_ctc", "v3_e2e_ctc"])
def test_align_longform_with_skips_end_to_end(name):
    import re
    model = _model(name)
    wav, _ = synthetic.synthetic_audio(1, 70.0, seed=23)
    wav = wav[0]
    e2e = name == "v3_e2e_ctc"
    lines = []
    for k in range(0, wav.numel(), 20 * 16000):
        text = model.transcribe(wav[k:k + 20 * 16000]).text
        lines.append(" ".join(re.findall(r"<(\d+)>", text)) if e2e else text)
    saved = model.decoding.tokenizer
    if e2e:
        model.decoding.tokenizer = _IdTokenizer(len(saved))
        model.__dict__.pop("_token_flags", None)
        said = {int(x) for line in lines for x in line.split()}
        junk = " ".join(str(i) for i in [i for i in range(len(saved)) if i not in said][:40])
    else:
        said = set("".join(lines))
        letters = [ch for ch in saved.vocab if ch != " " and ch not in said] or ["ё"]
        junk = "".join(letters[i % len(letters)] for i in range(40))
    lines.insert(2, junk)                                          # a line the recording does not contain
    lines.insert(0, "")
    try:
        _check_end_to_end(model, wav, lines)
    finally:
        model.decoding.tokenizer = saved
        model.__dict__.pop("_token_flags", None)


def _check_end_to_end(model, wav, lines):
    theta, psi = 0.7, 0.5
    res = model.align_longform(wav, lines, gap_threshold=theta, skip_threshold=psi)
    assert len(res.segments) == len(lines) and 3 in res.skipped, res.skipped
    for i in res.skipped:
        seg = res.segments[i]
        assert seg.start == seg.end and seg.words == [] and math.isnan(seg.confidence)
    windows, T = plan_windows(wav.numel(), 30.0, 4.0, model._encoded_length, 768)
    wav_d, length = model.prepare_wav(wav)
    with torch.inference_mode():
        lp = longform.stitch_ctc_log_probs(model, wav_d[0], windows, T, 16)[0].cpu().numpy()
    norm, ids, ranges = model._line_tokens(lines)
    edges = np.array(line_edges(ranges, len(ids)), np.uint8)
    log_theta, log_psi = (float(F32(math.log(float(F32(x))))) for x in (theta, psi))   # the public call's rounding
    fr, tok, vit, rows, flags, urows, ulogp, srows, slogp = skip_replay(lp, T, ids, edges, log_theta, log_psi)
    shift = compute_frame_shift(int(length[0]), T)
    assert res.skipped == skipped_lines(ranges, fr.tolist()) and srows == len(res.skipped)
    assert res.unmatched == unmatched_intervals(torch.from_numpy(flags), shift)
    assert res.confidence == gap_confidence(float(vit), float(ulogp), T - urows, float(slogp))
    want = line_segments(norm, ranges, fr.tolist(), tok.tolist(), shift, float(vit), skipped=res.skipped)
    assert [(s.start, s.end) for s in res.segments] == [(s.start, s.end) for s in want]
    assert all(s.confidence == w.confidence or (math.isnan(s.confidence) and math.isnan(w.confidence))
               for s, w in zip(res.segments, want))
    kept_frames = sorted(int(f) for f in fr if f >= 0)
    for w in res.words:                                            # words of the aligned tokens only
        assert any(w.start <= f * shift + 1e-9 and f * shift < w.end for f in kept_frames)
    ll, mags = skip_forward64(lp, T, ids, edges, log_theta, log_psi)
    assert abs(res.log_likelihood - ll) <= ctc_forward_bound(mags, ll)
    only = model.align_longform(wav, lines, skip_threshold=psi)
    assert only.unmatched is None and 3 in only.skipped
    # the wrong recording for its text, a single line nobody said: with gaps the speech is left unmatched and the line is
    # skipped, so the path skips every line and has no words (these synthetic models' low blank bias make the all-blank
    # path too dear without gaps)
    alone = model.align_longform(wav, lines[3], gap_threshold=theta, skip_threshold=0.9)
    _, a_ids, a_ranges = model._line_tokens([lines[3]])
    a_fr = skip_replay(lp, T, a_ids, np.array(line_edges(a_ranges, len(a_ids)), np.uint8), log_theta,
                       float(F32(math.log(float(F32(0.9))))))[0]
    assert alone.skipped == skipped_lines(a_ranges, a_fr.tolist()) == [0]
    assert alone.words == [] and alone.segments[0].words == [] and math.isfinite(alone.log_likelihood)
    assert alone.segments[0].start == alone.segments[0].end == 0.0 and alone.unmatched
    plain = model.align_longform(wav, lines, gap_threshold=theta)
    assert plain.skipped is None and "skipped" not in repr(plain)
