"""CTC hotwords: gam_ctc_bias (include/gigaam_b200.h has the definition), `Engine.ctc_bias` and the `hotwords=` argument of
`GigaAMASR.transcribe` / `transcribe_windowed` (INTEGRATION.md §7h).

CPU: a float32 / float64 oracle of the definition's steps 1-7, written line by line on top of the spot oracle of
test_keyword_spotting; hand-built cases for every rule; the refusals, all before device work; hotwords=None calls what the
methods called before.
GPU: bit identity with the oracle at three vocabularies; invariance to the batch and the keyword order; traced paths score
their detections; planted misspellings; hotwords that confirm greedy words change nothing; the windowed path over one
encoder pass; graph capture; device memory.
"""
import numpy as np
import pytest
import torch

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, synthetic
from gigaam_b200.engine import DecodeBuffers
from gigaam_b200.longform import plan_windows, stitch_ctc_log_probs
from test_keyword_spotting import _engine_for, _pad, spot_oracle, tau_of

F32 = np.float32
NEG = F32(-np.inf)


# ------------------------------------------------------------------------------------------ the oracle
def frame_max(row):
    """m[t]: the row's max (+0 for a zero max), NaN when the row holds a NaN."""
    return F32(np.nan) if np.isnan(row).any() else F32(row.max() + F32(0))


def replaced_range(ids, frames, flags, s, e):
    """Steps 2 and 3: the trimmed range [i0, i1) of span [s, e), or None when it is empty or not on word boundaries."""
    V = len(flags)
    fl = [int(flags[i]) if 0 <= i < V else 0 for i in ids]
    n = len(ids)
    i0, i1 = int(np.searchsorted(frames, s, "left")), int(np.searchsorted(frames, e, "left"))
    while i0 < i1 and fl[i0] & 1:
        i0 += 1
    while i1 > i0 and fl[i1 - 1] & 1:
        i1 -= 1
    if i1 <= i0:
        return None

    def boundary(p):
        return p == 0 or p == n or bool(fl[p - 1] & 1) or bool(fl[p] & 3)
    return (i0, i1) if boundary(i0) and boundary(i1) else None


def trace(lp, s0, e0, y):
    """Step 6: the keyword's best path over [s0, e0) from state 0 at s0 to state S - 1 at e0 - 1 (spot's recursion and ties, no
    fresh start) -> (label per frame, [(token id, first frame of its run)])."""
    V1 = lp.shape[1]
    U = len(y)
    S = 2 * U - 1
    lab = np.array([y[s // 2] if s % 2 == 0 else V1 - 1 for s in range(S)])
    skip = np.array([s % 2 == 0 and s >= 2 and y[s // 2] != y[s // 2 - 1] for s in range(S)])
    codes = {}
    v = np.full(S, NEG, F32)
    for t in range(s0, e0):
        row = lp[t]
        m = frame_max(row)
        if t == s0:
            v = np.full(S, NEG, F32)
            v[0] = F32(F32(row[lab[0]] - m) + F32(0))
            continue
        best, code = v.copy(), np.zeros(S, np.int64)
        c1 = np.concatenate([[NEG], v[:-1]]).astype(F32)
        take = c1 > best
        best, code = np.where(take, c1, best), np.where(take, 1, code)
        c2 = np.concatenate([[NEG, NEG], v[:-2]])[:S].astype(F32)
        take = skip & (c2 > best)
        best, code = np.where(take, c2, best), np.where(take, 2, code)
        v = ((row[lab] - m).astype(F32) + best).astype(F32)
        codes[t] = code
    labels, tokens = {}, []
    st = S - 1
    for t in range(e0 - 1, s0 - 1, -1):
        labels[t] = int(lab[st])
        prev = st if t == s0 else st - int(codes[t][st])
        if st % 2 == 0 and (t == s0 or prev != st):
            tokens.append((y[st // 2], t))
        st = max(prev, 0)
    return labels, tokens[::-1]


def bias_oracle(lp, enc_len, keywords, threshold, spotted, flags, ids, frames, counts, token_logp=None, path_logp=None,
                frame_logp=None):
    """gam_ctc_bias on host arrays: spotted = gam_ctc_spot's (start, end, score, count).  -> dict of out_ids, out_frames,
    out_counts, out_source (lists per recording), out_token_logp (list per recording, or None), out_path_logp (f32 [B] or
    None), frame_logp (an adjusted copy, or None) and `accepted`: per recording [(s, e, k, identity)] in start order."""
    st, en, sc, cnt = spotted
    B, T, V1 = lp.shape
    max_det = st.shape[2]
    out = {k: [] for k in ("ids", "frames", "source", "token_logp", "accepted")}
    path = None if path_logp is None else np.zeros(B, F32)
    fl_out = None if frame_logp is None else frame_logp.astype(np.float64).copy()
    for b in range(B):
        n = min(max(int(counts[b]), 0), ids.shape[1])
        g_ids, g_fr = [int(i) for i in ids[b, :n]], [int(f) for f in frames[b, :n]]
        Tb = min(max(int(enc_len[b]), 0), T)
        cands = []
        for k, y in enumerate(keywords):
            tau = tau_of(len(y), threshold)
            for j in range(min(int(cnt[b, k]), max_det)):
                s, e, E = int(st[b, k, j]), int(en[b, k, j]), F32(sc[b, k, j])
                G = F32(F32(E - tau) + F32(0))                               # step 1
                if not G >= 0 or not 0 <= s < e <= Tb:
                    continue
                r = replaced_range(g_ids, g_fr, flags, s, e)                 # steps 2 and 3
                if r is None:
                    continue
                cands.append(((-float(G), s, -len(y), tuple(y), k), s, e, E, k, r))
        cands.sort(key=lambda c: c[0])                                      # step 4
        busy = np.zeros(T, bool)
        acc = []
        for _, s, e, E, k, r in cands:
            if not busy[s:e].any():
                busy[s:e] = True
                acc.append((s, e, E, k, r))
        acc.sort(key=lambda c: c[0])
        # output items (frame, group, order, id, source, token_logp): group 0 = greedy tokens written before the frame's
        # spliced token, 1 = the spliced token, 2 = greedy tokens written after it
        place = {i: (f, 0) for i, f in enumerate(g_fr)}
        src = [-1] * n
        items = []
        total = None if path_logp is None else np.float64(path_logp[b])
        accepted = []
        for s, e, E, k, (i0, i1) in acc:
            y = keywords[k]
            same = g_ids[i0:i1] == list(y)                                   # step 5
            accepted.append((s, e, k, same))
            if same:
                for i in range(i0, i1):
                    src[i] = k
                continue
            for i in range(i0, i1):                                          # step 6
                del place[i]
            labels, tokens = trace(lp[b], s, e, y)
            for u, (tok, f) in enumerate(tokens):
                items.append((f, 1, u, tok, k, F32(lp[b, f, tok])))
            last = tokens[-1][1]
            r0, r1 = int(np.searchsorted(g_fr, s, "left")), int(np.searchsorted(g_fr, e, "left"))
            for i in range(r0, i0):                                          # left-edge spaces: before the keyword, at s
                place[i] = (s, 0)
            for i in range(i1, r1):                                          # right-edge spaces up to its last token: after it
                if g_fr[i] <= last:
                    place[i] = (last, 2)
            if total is not None:                                            # step 7
                total = total + np.float64(E)
            if fl_out is not None:
                for t, l in labels.items():
                    fl_out[b, t] = fl_out[b, t] + (np.float64(lp[b, t, l]) - np.float64(frame_max(lp[b, t])))
        for i, (f, grp) in place.items():
            items.append((f, grp, i, g_ids[i], src[i], None if token_logp is None else F32(token_logp[b, i])))
        items.sort(key=lambda x: x[:3])
        o_ids, o_fr, o_src, o_lp = [x[3] for x in items], [x[0] for x in items], [x[4] for x in items], [x[5] for x in items]
        m = ids.shape[1]
        out["ids"].append(o_ids[:m]); out["frames"].append(o_fr[:m]); out["source"].append(o_src[:m])
        out["token_logp"].append(None if token_logp is None else o_lp[:m])
        out["accepted"].append(accepted)
        if path is not None:
            path[b] = F32(total)
    out["path_logp"] = path
    out["frame_logp"] = fl_out
    return out


# ------------------------------------------------------------------------------------------ CPU: hand-built cases
TOY_V1 = 9                      # toy vocabulary: 0 = " ", 1..6 letters, 7 = a U+2581 piece, blank = 8
FLAGS = np.array([1, 0, 0, 0, 0, 0, 0, 2], np.uint8)


def rows(labels, second=None, gap=F32(-0.5)):
    """log-prob-like rows: label l scores 0 and the rest -6; second = {t: c or (c, score)} gives class c `gap` (or that
    score) at frame t."""
    lp = np.full((len(labels), TOY_V1), F32(-6), F32)
    for t, l in enumerate(labels):
        lp[t, l] = 0
    for t, c in (second or {}).items():
        c, x = c if isinstance(c, tuple) else (c, gap)
        lp[t, c] = x
    return lp


def greedy_of(lp):
    """CTC greedy on the rows (argmax, first index on ties, collapse, drop blanks): ids and first frames."""
    lab = lp.argmax(-1)
    blank = lp.shape[1] - 1
    ids, frames = [], []
    for t, x in enumerate(lab):
        if x != blank and (t == 0 or lab[t - 1] != x):
            ids.append(int(x))
            frames.append(t)
    return ids, frames


def run_oracle(lp, keywords, threshold, flags=FLAGS, spotted=None, **scores):
    lp = lp[None]
    T = lp.shape[1]
    ids, frames = greedy_of(lp[0])
    g_ids = np.zeros((1, T), np.int32)
    g_fr = np.zeros((1, T), np.int32)
    g_ids[0, :len(ids)], g_fr[0, :len(ids)] = ids, frames
    if spotted is None:
        spotted = spot_oracle(lp, [T], keywords, threshold, T, lp.shape[2] - 1)
    return bias_oracle(lp, [T], keywords, threshold, spotted, flags, g_ids, g_fr, [len(ids)], **scores), ids, frames


B8 = TOY_V1 - 1                 # the blank label


def test_identity_changes_nothing():
    # " 12 34 " : the greedy word (3, 4) given as a hotword is confirmed in place
    lp = rows([0, B8, 1, 2, B8, 0, 3, 3, 4, B8, 0])
    fl = np.zeros((1, 11))
    got, ids, frames = run_oracle(lp, [[3, 4]], 1.0, token_logp=np.zeros((1, 11), F32), path_logp=[F32(-1.5)], frame_logp=fl)
    assert got["ids"][0] == ids and got["frames"][0] == frames
    assert got["source"][0] == [-1, -1, -1, -1, 0, 0, -1]
    assert got["accepted"][0] == [(6, 9, 0, True)]
    assert got["path_logp"][0] == F32(-1.5) and (got["frame_logp"] == 0).all()


def test_misspelling_is_replaced_at_the_traced_frames():
    # greedy writes " 12 35 " where (3, 4) scores close behind at frames 8..9
    lp = rows([0, B8, 1, 2, B8, 0, 3, 3, 5, 5, B8, 0], second={8: 4, 9: 4})
    fl = np.zeros((1, 12))
    got, ids, frames = run_oracle(lp, [[3, 4]], 0.5, token_logp=np.zeros((1, 12), F32), path_logp=[F32(-2.0)], frame_logp=fl)
    assert ids == [0, 1, 2, 0, 3, 5, 0]
    assert got["ids"][0] == [0, 1, 2, 0, 3, 4, 0] and got["frames"][0] == [0, 2, 3, 5, 6, 8, 11]
    assert got["source"][0] == [-1, -1, -1, -1, 0, 0, -1]
    E = F32(-0.5)                                                        # the path ends on 4's first frame
    assert got["accepted"][0] == [(6, 9, 0, False)]
    assert got["path_logp"][0] == F32(np.float64(-2.0) + np.float64(E))
    assert got["frame_logp"][0, 6:9].sum() == float(E) and got["frame_logp"][0, 8] == -0.5
    assert got["token_logp"][0][5] == F32(-0.5)


def test_keyword_inside_a_longer_word_is_refused():
    # " 3456 ": the greedy word contains (4, 5) but neither edge is a word boundary; (3, 4) lacks its right edge
    lp = rows([0, 3, 4, 5, 6, B8, 0])
    for kw in ([4, 5], [3, 4], [5, 6]):
        got, ids, _ = run_oracle(lp, [kw], 1.0)
        assert got["accepted"][0] == [] and got["ids"][0] == ids


def test_a_span_over_blanks_only_is_not_applied():
    # the keyword (3) scores close behind greedy blanks at frames 2..3: its span holds no greedy token
    lp = rows([1, B8, B8, B8, 0, 2], second={2: 3, 3: 3})
    got, ids, _ = run_oracle(lp, [[3]], 0.5)
    assert got["accepted"][0] == [] and got["ids"][0] == ids


def test_charwise_spaces_at_the_edges_stay():
    # greedy " 1 56 2"; (4, 6) ties with the space at frame 2 and scores close behind 5 at frame 3, so its span [2, 5) starts on
    # the space: the space stays, 5 becomes 4 and 6 is confirmed
    lp = rows([0, 1, 0, 5, 6, B8, 0, 2], second={2: (4, F32(0)), 3: 4})
    got, ids, frames = run_oracle(lp, [[4, 6]], 0.5)
    assert ids == [0, 1, 0, 5, 6, 0, 2]
    assert got["accepted"][0] == [(2, 5, 0, False)]
    # the kept space and the keyword's first token share frame 2, the space first
    assert got["ids"][0] == [0, 1, 0, 4, 6, 0, 2] and got["frames"][0] == [0, 1, 2, 2, 4, 6, 7]
    assert got["source"][0] == [-1, -1, -1, 0, 0, -1, -1]
    # a span that holds nothing but a space is not applied
    got, _, _ = run_oracle(lp, [[4]], 0.5, spotted=hand_spotted([(0, 2, 3, F32(0))], 1))
    assert got["accepted"][0] == []


def test_edge_spaces_inside_the_span_stay_outside_the_keyword():
    # greedy " 1 56" at frames 0, 1, 3, 4, 5 dropped the 3 that was said at frame 2, before the space: (3, 5, 6) spans [2, 6)
    # and the space, kept, is written before the whole keyword (at frame 2), not between its tokens
    lp = rows([0, 1, B8, 0, 5, 6, B8], second={2: (3, F32(-0.3)), 3: (B8, F32(-0.3))})
    got, ids, frames = run_oracle(lp, [[3, 5, 6]], 0.3)
    assert (ids, frames) == ([0, 1, 0, 5, 6], [0, 1, 3, 4, 5])
    assert got["accepted"][0] == [(2, 6, 0, False)]
    assert got["ids"][0] == [0, 1, 0, 3, 5, 6] and got["frames"][0] == [0, 1, 2, 2, 4, 5]
    assert got["source"][0] == [-1, -1, -1, 0, 0, 0]
    # the right edge: greedy " 5 " then "1" lost the 3 said after the space; (5, 3) spans [1, 4) and the space is written
    # after the keyword's last token, at its frame
    lp = rows([0, 5, 0, B8, B8, 1], second={2: (B8, F32(-0.3)), 3: (3, F32(-0.3))})
    got, ids, frames = run_oracle(lp, [[5, 3]], 0.3)
    assert (ids, frames) == ([0, 5, 0, 1], [0, 1, 2, 5])
    assert got["accepted"][0] == [(1, 4, 0, False)]
    assert got["ids"][0] == [0, 5, 3, 0, 1] and got["frames"][0] == [0, 1, 3, 3, 5]
    assert got["source"][0] == [-1, 0, 0, -1, -1]


def test_sentencepiece_word_edges():
    # no space token: piece 7 opens a word.  "7 1 2 | 7 3 5": (7, 3, 4) may replace the second word, (3, 4) may not (its left
    # edge is inside a word)
    lp = rows([7, 1, 2, 7, 3, 5, 5], second={5: 4, 6: 4})
    got, ids, _ = run_oracle(lp, [[7, 3, 4]], 0.3)
    assert got["ids"][0] == [7, 1, 2, 7, 3, 4]
    got, ids, _ = run_oracle(lp, [[3, 4]], 0.3)
    assert got["accepted"][0] == [] and got["ids"][0] == ids


def hand_spotted(dets, K, max_det=4):
    """gam_ctc_spot outputs for one recording from [(k, s, e, E)]."""
    st = np.full((1, K, max_det), -1, np.int32)
    en = np.full((1, K, max_det), -1, np.int32)
    sc = np.full((1, K, max_det), NEG, F32)
    cnt = np.zeros((1, K), np.int32)
    for k, s, e, E in dets:
        j = cnt[0, k]
        st[0, k, j], en[0, k, j], sc[0, k, j] = s, e, E
        cnt[0, k] += 1
    return st, en, sc, cnt


def test_overlaps_and_every_tie_break():
    lp = rows([0, 1, 2, B8, 0, 3, 4, B8, 0])                          # " 12 34 ": words at frames 1..2 and 5..6
    tau1, tau2 = tau_of(1, 0.5), tau_of(2, 0.5)

    def winner(keywords, dets):
        got, _, _ = run_oracle(lp, keywords, 0.5, spotted=hand_spotted(dets, len(keywords)))
        return [(s, e, k) for s, e, k, _ in got["accepted"][0]]
    # the higher gain wins an overlap, whatever the keyword order
    kws = [[5, 6], [6, 5]]
    assert winner(kws, [(0, 1, 3, tau2 + F32(0.25)), (1, 1, 3, tau2 + F32(0.5))]) == [(1, 3, 1)]
    assert winner(kws[::-1], [(1, 1, 3, tau2 + F32(0.25)), (0, 1, 3, tau2 + F32(0.5))]) == [(1, 3, 0)]
    # equal gains: the earlier start
    assert winner(kws, [(0, 2, 5, tau2), (1, 1, 3, tau2)]) == [(1, 3, 1)]
    # equal gains and starts: the longer keyword (its tau is lower, so its score is too)
    kws = [[5], [5, 6]]
    assert winner(kws, [(0, 1, 3, tau1), (1, 1, 3, tau2)]) == [(1, 3, 1)]
    # equal gains, starts and lengths: the smaller ids
    kws = [[6, 5], [5, 6]]
    assert winner(kws, [(0, 1, 3, tau2), (1, 1, 3, tau2)]) == [(1, 3, 1)]
    assert winner(kws[::-1], [(1, 1, 3, tau2), (0, 1, 3, tau2)]) == [(1, 3, 0)]
    # exact duplicates: the smaller index, with the same tokens either way
    kws = [[5, 6], [5, 6]]
    assert winner(kws, [(0, 1, 3, tau2), (1, 1, 3, tau2)]) == [(1, 3, 0)]
    # disjoint spans are all accepted, in start order
    assert winner([[5, 6], [6, 5]], [(1, 1, 3, tau2), (0, 5, 7, tau2)]) == [(1, 3, 1), (5, 7, 0)]


def test_duplicate_hotwords_give_the_same_output():
    lp = rows([0, 1, 2, B8, 0, 3, 3, 5, 5, B8, 0], second={7: 4, 8: 4})
    one, _, _ = run_oracle(lp, [[3, 4]], 0.5)
    two, _, _ = run_oracle(lp, [[3, 4], [3, 4]], 0.5)
    assert one["ids"] == two["ids"] and one["frames"] == two["frames"] and one["source"] == two["source"]


# ------------------------------------------------------------------------------------------ CPU: refusals and surface
_CPU_MODELS = {}


def _cpu_model(name):
    if name not in _CPU_MODELS:
        _CPU_MODELS[name] = gigaam.load_model(name, device="cpu", checkpoint=synthetic.synthetic_checkpoint(name, n_layers=1))
    return _CPU_MODELS[name]


def test_refusals_come_before_device_work():
    model = _cpu_model("v2_ctc")
    tok = model.decoding.tokenizer
    V, sp = len(tok), tok.vocab.index(" ")
    wav = np.zeros(16000, np.float32)
    bad = [([], "no keywords"), (["123"], "no tokens"), ([[]], "without tokens"), (["а" * 65], "65 tokens"), ([[0, V]], "outside"),
           ([[sp, 3]], "space token"), ([[3, sp]], "space token"), ([[sp]], "space token")]
    for kws, match in bad:
        with pytest.raises(ValueError, match=match):
            model.transcribe(wav, hotwords=kws)
        with pytest.raises(ValueError, match=match):
            model.transcribe_windowed(wav, hotwords=kws)
    for theta in (0.0, 1.5, float("nan")):
        with pytest.raises(ValueError, match="threshold"):
            model.transcribe(wav, hotwords=["да"], hotword_threshold=theta)
        with pytest.raises(ValueError, match="threshold"):
            model.transcribe_windowed(wav, hotwords=["да"], hotword_threshold=theta)
    model._hotword_ids([[3, sp, 4], "да нет"], 0.5, "transcribe")      # a space inside a hotword is fine
    for name in ("v2_rnnt", "v3_e2e_rnnt"):
        rnnt = _cpu_model(name)
        with pytest.raises(NotImplementedError, match="_ctc"):
            rnnt.transcribe(wav, hotwords=["а"])
        with pytest.raises(NotImplementedError, match="_ctc"):
            rnnt.transcribe_windowed(wav, hotwords=["а"])


def test_exports():
    lib = _lib.load()
    for name in ("gam_ctc_bias", "gam_ctc_bias_workspace_bytes"):
        assert name in _lib.EXPORTS and hasattr(lib, name)


class _Recorder:
    """Stands in for the engine: records the calls, and fails on any hotword call."""

    def __init__(self):
        self.calls = []
        self.device = torch.device("cpu")
        self.num_classes = 34

    def group_words(self, ids, frames, counts, flags):
        self.calls.append("group_words")
        B, m = ids.shape
        return [torch.zeros((B, m), dtype=torch.int32) for _ in range(4)] + [torch.zeros(B, dtype=torch.int32)]

    def __getattr__(self, name):
        raise AssertionError(f"unexpected engine call {name}")


def test_hotwords_none_runs_the_plain_path(monkeypatch):
    import gigaam_b200.longform as longform
    model = _cpu_model("v2_ctc")
    log = []
    enc = torch.zeros((1, 768, 25))
    monkeypatch.setattr(model, "forward", lambda wav, length: (log.append("forward"), (enc, torch.tensor([25])))[1])
    monkeypatch.setattr(model, "_decode", lambda *a: (log.append(("decode",) + tuple(a[3:])), [("txt", None, None)])[1])
    eng = _Recorder()                     # fails on ctc_log_probs, ctc_spot, ctc_bias and any other engine call
    monkeypatch.setattr(model, "_get_engine", lambda: eng)
    wav = np.zeros(16000, np.float32)
    for kwargs in ({}, {"hotwords": None}):
        log.clear()
        assert model.transcribe(wav, word_timestamps=True, **kwargs).text == "txt"
        assert log == ["forward", ("decode", True, False)] and eng.calls == []
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)

    def fake_decode(m, host, windows, T, batch_size, scores, *extra, **kw):
        log.append(("decode_windows", len(extra), tuple(kw)))
        i32 = dict(dtype=torch.int32)
        return DecodeBuffers(torch.zeros((1, T), **i32), torch.zeros((1, T), **i32), torch.zeros(1, **i32))
    monkeypatch.setattr(longform, "decode_windows", fake_decode)
    for kwargs in ({}, {"hotwords": None}):
        log.clear()
        eng.calls.clear()
        model.transcribe_windowed(wav, **kwargs)
        assert log == [("decode_windows", 0, ())] and eng.calls == ["group_words"]


# ------------------------------------------------------------------------------------------ GPU helpers
def _dev():
    return torch.device("cuda", 0)


_MODELS = {}


def _model(name):
    if name not in _MODELS:
        _MODELS[name] = gigaam.load_model(name, fp16_encoder=False, device=_dev(),
                                          checkpoint=synthetic.synthetic_checkpoint(name, seed=0, n_layers=1))
    return _MODELS[name]


def _flags_for(V, sp):
    """A flag table: charwise (token 0 is the space) or SentencePiece (tokens >= V / 2 open a word)."""
    flags = np.zeros(V, np.uint8)
    if sp:
        flags[V // 2:] = 2
    else:
        flags[0] = 1
    return flags


def _planted_case(rng, V1, B, T, sp):
    """Recordings of words (a space token between them, or SentencePiece word openers) with hotwords planted: as they are, or
    misspelled with the right token close behind; plus random keywords, a duplicate, one inside another and one that
    extends another.  -> lp [B, T, V1] f32, keywords, flags."""
    V = V1 - 1
    letters = list(range(1, V // 2)) if sp else list(range(1, min(V, 30)))
    openers = list(range(V // 2, V)) if sp else None

    def word(n):
        w = [int(rng.choice(letters)) for _ in range(n)]
        if sp:
            w[0] = int(rng.choice(openers))
        return w
    hot = [word(int(rng.integers(1, 6))) for _ in range(6)]
    keywords = hot + [hot[0], hot[1][:max(1, len(hot[1]) - 1)], hot[2] + [int(rng.choice(letters))], word(3), word(2)]
    logits = rng.normal(0, 1.0, (B, T, V1))
    logits[..., V] += 2.0
    for b in range(B):
        t = int(rng.integers(0, 3))
        while t < T - 12:
            w = list(hot[int(rng.integers(0, len(hot)))]) if rng.random() < 0.6 else word(int(rng.integers(1, 6)))
            right = list(w)
            if rng.random() < 0.6:
                i = int(rng.integers(0, len(w)))
                w[i] = int(rng.choice(openers if sp and i == 0 else letters))
            for tok, good in zip(w, right):
                for _ in range(int(rng.integers(1, 3))):
                    if t < T:
                        logits[b, t, tok] += 7.0
                        if good != tok:
                            logits[b, t, good] += rng.choice([6.0, 6.6, 7.4])
                        t += 1
                if rng.random() < 0.5:
                    t += 1
            if not sp and t < T:
                logits[b, t, 0] += 7.0
                t += 1
            t += int(rng.integers(0, 3))
    lp = torch.tensor(logits).float().log_softmax(-1).numpy()
    return lp, keywords, _flags_for(V, sp)


def _greedy_batch(lp, enc_len):
    B, T, _ = lp.shape
    ids = np.zeros((B, T), np.int32)
    frames = np.zeros((B, T), np.int32)
    counts = np.zeros(B, np.int32)
    for b in range(B):
        Tb = min(max(int(enc_len[b]), 0), T)
        i, f = greedy_of(lp[b, :Tb])
        ids[b, :len(i)], frames[b, :len(i)], counts[b] = i, f, len(i)
    return ids, frames, counts


def _run_bias(eng, lp, enc_len, keywords, threshold, flags, greedy, scores=None, max_det=None):
    """Engine.ctc_spot + Engine.ctc_bias on host arrays -> (spot outputs, bias outputs, adjusted frame_logp) on the host."""
    dev = _dev()
    kw, kw_len = (t.to(dev) for t in _pad(keywords))
    lp_d = torch.as_tensor(lp).to(dev).contiguous()
    enc = torch.as_tensor(np.asarray(enc_len, np.int32)).to(dev)
    spotted = eng.ctc_spot(lp_d, enc, kw, kw_len, threshold, max_det or lp.shape[1])
    ids, frames, counts = (torch.as_tensor(x).to(dev) for x in greedy)
    tl, pl, fl = (None, None, None) if scores is None else (torch.as_tensor(x).to(dev) for x in scores)
    out = eng.ctc_bias(lp_d, enc, kw, kw_len, spotted, threshold, torch.as_tensor(flags), ids, frames, counts, tl, pl, fl)
    host = lambda t: None if t is None else t.cpu().numpy()
    return [host(t) for t in spotted], [host(t) for t in out], host(fl)


def _scores(rng, lp, greedy):
    ids, frames, counts = greedy
    B, T, _ = lp.shape
    tl = rng.normal(-0.1, 0.05, ids.shape).astype(F32)
    pl = rng.normal(-3, 1, B).astype(F32)
    fl = rng.normal(-0.01, 0.01, (B, T + 3))
    return tl, pl, fl


def _rows(got):
    """Per recording: (ids, frames, source, token_logp bits) up to its count (entries past it are not written)."""
    ids, frames, counts, source, tl, _ = got
    return [(ids[b, :n].tolist(), frames[b, :n].tolist(), source[b, :n].tolist(),
             None if tl is None else tl[b, :n].view(np.int32).tolist()) for b, n in enumerate(counts.tolist())]


def _check(got, want, fl_got=None):
    ids, frames, counts, source, tl, pl = got
    for b in range(ids.shape[0]):
        n = int(counts[b])
        assert n == len(want["ids"][b]), (b, n, len(want["ids"][b]))
        assert ids[b, :n].tolist() == want["ids"][b]
        assert frames[b, :n].tolist() == want["frames"][b]
        assert source[b, :n].tolist() == want["source"][b]
        if tl is not None:
            assert np.array_equal(tl[b, :n].view(np.int32), np.array(want["token_logp"][b], F32).view(np.int32))
    if pl is not None:
        np.testing.assert_allclose(pl, want["path_logp"], rtol=1e-6)
    if fl_got is not None:
        np.testing.assert_allclose(fl_got, want["frame_logp"], rtol=0, atol=1e-9)


# ------------------------------------------------------------------------------------------ GPU: the kernel against the oracle
@pytest.mark.gpu
@pytest.mark.parametrize("V1", [34, 257, 1025])
def test_bit_identical_to_the_oracle(V1):
    rng = np.random.default_rng(V1)
    B, T = 4, 400
    sp = V1 == 257
    lp, keywords, flags = _planted_case(rng, V1, B, T, sp)
    enc_len = [T, 301, 0, T - 1]
    eng = _engine_for(V1)
    greedy = _greedy_batch(lp, enc_len)
    splices = identities = 0
    for theta in (0.2, 0.6):
        scores = _scores(rng, lp, greedy)
        spotted, got, fl = _run_bias(eng, lp, enc_len, keywords, theta, flags, greedy, scores)
        want = bias_oracle(lp, enc_len, keywords, theta, spotted, flags, *greedy, *scores)
        _check(got, want, fl)
        acc = [a for r in want["accepted"] for a in r]
        splices += sum(not a[3] for a in acc)
        identities += sum(a[3] for a in acc)
        # unscored: the same tokens
        _, got2, _ = _run_bias(eng, lp, enc_len, keywords, theta, flags, greedy)
        assert got2[4] is None and got2[5] is None
        assert [r[:3] for r in _rows(got2)] == [r[:3] for r in _rows(got)]
        # the traced paths score their detections: a float64 sum of lp[t, l(t)] - m[t] over the oracle's traced labels is E
        # to fp32 rounding
        for b, r in enumerate(want["accepted"]):
            for s, e, k, same in r:
                if same:
                    continue
                j = int(np.nonzero(spotted[0][b, k] == s)[0][0])
                labels, _ = trace(lp[b], s, e, keywords[k])
                lp64 = lp[b].astype(np.float64)
                path = sum(lp64[t, l] - lp64[t].max() for t, l in labels.items())
                assert abs(path - float(spotted[2][b, k, j])) <= 1e-6 * (e - s) * max(1.0, abs(path)), (b, s, e, k)
    print(f"\n{splices} splices, {identities} identities")
    assert splices >= 5 and identities >= 2


@pytest.mark.gpu
def test_output_does_not_depend_on_batch_or_keyword_order():
    rng = np.random.default_rng(5)
    V1, B, T = 34, 5, 500
    lp, keywords, flags = _planted_case(rng, V1, B, T, False)
    enc_len = [T, 480, T, 333, 20]
    eng = _engine_for(V1)
    greedy = _greedy_batch(lp, enc_len)
    scores = _scores(rng, lp, greedy)
    _, base, fl = _run_bias(eng, lp, enc_len, keywords, 0.3, flags, greedy, scores)
    b = 3
    _, alone, fl1 = _run_bias(eng, lp[b:b + 1], enc_len[b:b + 1], keywords, 0.3, flags, tuple(x[b:b + 1] for x in greedy),
                              tuple(x[b:b + 1] for x in scores))
    assert _rows(alone) == _rows(base)[b:b + 1] and alone[5][0] == base[5][b]
    assert np.array_equal(fl1, fl[b:b + 1])
    perm = [int(i) for i in rng.permutation(len(keywords))]
    _, moved, fl2 = _run_bias(eng, lp, enc_len, [keywords[i] for i in perm], 0.3, flags, greedy, scores)
    assert [r[:2] + r[3:] for r in _rows(moved)] == [r[:2] + r[3:] for r in _rows(base)] and np.array_equal(moved[5], base[5])
    assert np.array_equal(fl2, fl)
    # sources name the same keywords (duplicates, keyword 0 and 6, are interchangeable)
    same = {k: {k} for k in range(len(keywords))}
    same[0] = same[6] = {0, 6}
    for r in range(B):
        n = int(base[2][r])
        for x, y in zip(moved[3][r, :n], base[3][r, :n]):
            assert (x == -1 and y == -1) or (x >= 0 and perm[x] in same[int(y)])


@pytest.mark.gpu
def test_planted_misspelling_is_written_at_the_traced_frames():
    V1, T = 34, 60
    rng = np.random.default_rng(1)
    logits = rng.normal(0, 0.02, (T, V1))
    logits[:, V1 - 1] += 9.0
    heard = [(5, 0), (6, 4), (8, 5), (10, 0), (12, 7), (13, 9), (15, 9), (16, 2), (18, 0), (20, 6)]
    for t, tok in heard:                                                # " 45 7 9 2 6": greedy hears 9 where 8 was said
        logits[t, tok] += 14.0
    logits[13, 8] += 13.5
    logits[14, 8] += 8.7
    lp = torch.tensor(logits).float().log_softmax(-1).numpy()[None]
    flags = _flags_for(V1 - 1, False)
    greedy = _greedy_batch(lp, [T])
    assert greedy[0][0, :greedy[2][0]].tolist() == [0, 4, 5, 0, 7, 9, 9, 2, 0, 6]
    keyword = [7, 8, 9, 2]
    pl = np.array([-4.0], F32)
    spotted, got, _ = _run_bias(_engine_for(V1), lp, [T], [keyword], 0.5, flags, greedy,
                                (np.zeros((1, T), F32), pl, np.zeros((1, T))))
    assert spotted[3][0, 0] == 1 and spotted[0][0, 0, 0] == 12 and spotted[1][0, 0, 0] == 17
    n = int(got[2][0])
    assert got[0][0, :n].tolist() == [0, 4, 5, 0, 7, 8, 9, 2, 0, 6]
    assert got[1][0, :n].tolist() == [5, 6, 8, 10, 12, 13, 15, 16, 18, 20]
    assert got[3][0, :n].tolist() == [-1] * 4 + [0] * 4 + [-1] * 2
    E = spotted[2][0, 0, 0]
    assert got[5][0] == F32(np.float64(pl[0]) + np.float64(E)) and E < 0


@pytest.mark.gpu
def test_edge_spaces_inside_the_span_on_the_device():
    V1 = 34                                                             # the toy rows in the v2_ctc vocabulary: 0 is " "
    eng = _engine_for(V1)
    flags = _flags_for(V1 - 1, False)
    cases = [(rows([0, 1, B8, 0, 5, 6, B8], second={2: (3, F32(-0.3)), 3: (B8, F32(-0.3))}), [3, 5, 6], [0, 1, 0, 3, 5, 6],
              [0, 1, 2, 2, 4, 5]),
             (rows([0, 5, 0, B8, B8, 1], second={2: (B8, F32(-0.3)), 3: (3, F32(-0.3))}), [5, 3], [0, 5, 3, 0, 1], [0, 1, 3, 3, 5])]
    for toy, kw, want_ids, want_frames in cases:
        lp = np.full((1, toy.shape[0], V1), F32(-6), F32)
        lp[0, :, :B8] = toy[:, :B8]
        lp[0, :, V1 - 1] = toy[:, B8]
        greedy = _greedy_batch(lp, [lp.shape[1]])
        scores = _scores(np.random.default_rng(0), lp, greedy)
        spotted, got, fl = _run_bias(eng, lp, [lp.shape[1]], [kw], 0.3, flags, greedy, scores)
        want = bias_oracle(lp, [lp.shape[1]], [kw], 0.3, spotted, flags, *greedy, *scores)
        _check(got, want, fl)
        assert want["ids"][0] == want_ids and want["frames"][0] == want_frames


@pytest.mark.gpu
@pytest.mark.parametrize("name,seconds", [("v2_ctc", 6.0), ("v3_e2e_ctc", 1.5)])
def test_own_words_at_threshold_one_change_nothing(name, seconds):
    model = _model(name)
    tok = model.decoding.tokenizer
    wav, _ = synthetic.synthetic_audio(1, seconds, seed=5)
    wav = wav[0]
    w_d, l_d = model.prepare_wav(wav)
    with torch.inference_mode():
        enc, enc_len = model(w_d, l_d)
        _, ids, frames = model.decoding.decode(model.head, enc, enc_len)[0]
        lab = model.head(enc)[0, :int(enc_len[0])].argmax(-1).tolist()
    blank = len(tok)
    runs = [(t, x) for t, x in enumerate(lab) if x != blank and (t == 0 or lab[t - 1] != x)]
    assert [x for _, x in runs] == ids and [t for t, _ in runs] == frames   # logits and log-probs pick the same labels
    # its own words, as the greedy decoder wrote them (spaces are word edges, not part of a word)
    words, cur = [], []
    for i in ids + [None]:
        if i is None or tok.id_to_str(i) == " " or tok.id_to_str(i).startswith("▁"):
            if cur and len(cur) <= 64:
                words.append(cur)
            cur = []
        if i is not None and tok.id_to_str(i) != " ":
            cur.append(i)
    assert words
    plain = model.transcribe(wav, word_timestamps=True, confidence=True)
    hot = model.transcribe(wav, word_timestamps=True, confidence=True, hotwords=words, hotword_threshold=1.0)
    assert hot == plain and len(plain.words) > 0


@pytest.mark.gpu
def test_windowed_equals_the_oracle_over_one_encoder_pass(monkeypatch):
    model = _model("v2_ctc")
    eng = model._get_engine()
    tok = model.decoding.tokenizer
    wav, _ = synthetic.synthetic_audio(1, 150.0, seed=9)
    wav = wav[0][: 150 * 16000 - 777]
    plain = model.transcribe_windowed(wav, word_timestamps=True, confidence=True, batch_size=2)
    words = sorted({w.text for s in plain.segments for w in s.words if 2 <= len(w.text) <= 64})[:25]
    letters = "аеиорст"
    hot = [w[:i] + c + w[i + 1:] for w in words for i in (0, len(w) // 2, len(w) - 1) for c in letters if c != w[i]]   # near misses
    hot = sorted(set(hot))
    assert hot, [w.text for s in plain.segments for w in s.words][:20]
    forwards = []
    real_forward = type(model).forward
    monkeypatch.setattr(type(model), "forward", lambda self, *a: (forwards.append(1), real_forward(self, *a))[1])
    res = model.transcribe_windowed(wav, word_timestamps=True, confidence=True, batch_size=2, hotwords=hot, hotword_threshold=0.1)
    windows, T = plan_windows(wav.numel(), 30.0, 4.0, model._encoded_length, 768)
    groups = []                                                     # longform.window_batches' batches of up to 2 windows
    for w in windows:
        if w.keep_end <= w.keep_start:
            continue
        if groups and len(groups[-1]) < 2 and groups[-1][0].end - groups[-1][0].start == w.end - w.start:
            groups[-1].append(w)
        else:
            groups.append([w])
    assert len(windows) > 4 and len(forwards) == len(groups)
    monkeypatch.undo()
    # the oracle over the stitched log-probs and the windowed greedy output
    from gigaam_b200.longform import decode_windows
    with torch.inference_mode():
        host = wav.to(model._dtype).pin_memory()
        lp = torch.empty((1, T, eng.num_classes), device=_dev())
        out = decode_windows(model, host, windows, T, 2, True, log_probs=lp)
        w_d, _ = model.prepare_wav(wav)
        assert torch.equal(lp, stitch_ctc_log_probs(model, w_d[0], windows, T, 2))
        names, ids = model._keyword_ids(hot, 0.1)
        spotted = model._spot_all(lp, torch.tensor([T], dtype=torch.int32, device=_dev()), *(t.to(_dev()) for t in _pad(ids)), ids,
                                  0.1)
    lp_h = lp.cpu().numpy()
    want = bias_oracle(lp_h, [T], ids, 0.1, [t.cpu().numpy() for t in spotted], model._word_flags().cpu().numpy(),
                       out.ids.cpu().numpy(), out.frames.cpu().numpy(), out.counts.cpu().numpy(), out.token_logp.cpu().numpy(),
                       out.path_logp.cpu().numpy(), out.frame_logp.cpu().numpy())
    assert "".join(s.text for s in res.segments).replace(" ", "") == tok.decode(want["ids"][0]).replace(" ", "")
    got_words = [w for s in res.segments for w in s.words]
    from gigaam_b200.timestamps_utils import frames_to_words
    shift = (wav.numel() / 16000) / T
    ref = frames_to_words(tok, want["ids"][0], want["frames"][0], shift)
    assert [(w.text, w.start, w.end) for w in got_words] == [(w.text, w.start, w.end) for w in ref]
    splices = sum(not a[3] for a in want["accepted"][0])
    print(f"\n{len(hot)} hotwords, {splices} splices over {T} frames")
    assert splices > 0
    conf = [s.confidence for s in res.segments]
    assert all(0 < c <= 1 for c in conf)


@pytest.mark.gpu
def test_graph_capture_replays_with_other_inputs():
    rng = np.random.default_rng(2)
    V1, B, T = 34, 3, 300
    eng = _engine_for(V1)
    dev = _dev()
    cases = []
    for _ in range(2):
        lp, keywords, flags = _planted_case(rng, V1, B, T, False)
        greedy = _greedy_batch(lp, [T] * B)
        cases.append((lp, keywords[:6], flags, greedy, _scores(rng, lp, greedy)))
    K, Umax, max_det = 6, max(len(y) for c in cases for y in c[1]), 40

    def load(case):
        lp, keywords, flags, greedy, scores = case
        kw = torch.zeros((K, Umax), dtype=torch.int32)
        kw_len = torch.tensor([len(y) for y in keywords], dtype=torch.int32)
        for k, y in enumerate(keywords):
            kw[k, :len(y)] = torch.tensor(y)
        return [torch.as_tensor(lp), kw, kw_len, *(torch.as_tensor(x) for x in greedy), *(torch.as_tensor(x) for x in scores)]
    bufs = [x.to(dev) for x in load(cases[0])]
    enc = torch.full((B,), T, dtype=torch.int32, device=dev)
    flags = torch.as_tensor(cases[0][2]).to(dev)

    def step():
        lp, kw, kw_len, ids, frames, counts, tl, pl, fl = bufs
        spotted = eng.ctc_spot(lp, enc, kw, kw_len, 0.3, max_det)
        return eng.ctc_bias(lp, enc, kw, kw_len, spotted, 0.3, flags, ids, frames, counts, tl, pl, fl)
    fl0 = bufs[8].clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            got = step()
    torch.cuda.synchronize()
    for case in cases[::-1]:
        for buf, x in zip(bufs, load(case)):
            buf.copy_(x)
        g.replay()
        torch.cuda.synchronize()
        lp, keywords, fl_, greedy, scores = case
        spotted = [t.cpu().numpy() for t in eng.ctc_spot(bufs[0], enc, bufs[1], bufs[2], 0.3, max_det)]
        want = bias_oracle(lp, [T] * B, keywords, 0.3, spotted, fl_, *greedy, *scores)
        _check([t.cpu().numpy() for t in got], want, bufs[8].cpu().numpy())
    assert not torch.equal(fl0, bufs[8])


@pytest.mark.gpu
def test_device_memory_stays_within_workspace_and_stitched_log_probs():
    model = _model("v2_ctc")
    eng = model._get_engine()
    V1 = eng.num_classes
    peaks, frames = {}, {}
    for minutes in (2, 12, 2, 12):
        wav, _ = synthetic.synthetic_audio(1, 60.0 * minutes, seed=minutes)
        model.transcribe_windowed(wav[0], batch_size=4, hotwords=["при", "кот"], hotword_threshold=0.3)   # caches warm
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        model.transcribe_windowed(wav[0], batch_size=4, hotwords=["при", "кот"], hotword_threshold=0.3)
        torch.cuda.synchronize()
        peaks[minutes] = torch.cuda.max_memory_allocated() - base
        frames[minutes] = model._encoded_length(wav.shape[1])
    T2, T12 = frames[2], frames[12]
    ws = int(eng.lib.gam_ctc_bias_workspace_bytes(eng.handle, 1, T12, 2, 256))
    grow = (T12 - T2) * V1 * 4
    print(f"\npeak above baseline: 2 min {peaks[2] / 2**20:.1f} MiB, 12 min {peaks[12] / 2**20:.1f} MiB; stitched log-probs grow "
          f"by {grow / 2**20:.1f} MiB, bias workspace {ws / 2**20:.1f} MiB")
    assert peaks[12] - peaks[2] < grow + ws + 16 * 2**20
