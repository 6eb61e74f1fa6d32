"""Hotwords in live streams: gam_ctc_bias_resume (include/gigaam_b200.h has the rule), `Engine.ctc_bias_resume` and the
`hotwords=` argument of `GigaAMASR.streaming` (INTEGRATION.md §7i).

CPU: a Python reference of the resumable rule -- a streaming spot oracle (spot's recursion, scan and early emission), the
horizon, the decided components and the release frame, with test_hotwords.bias_oracle applied to the held span -- run over
random consecutive splits of planted cases; every split's released tokens concatenate to bias_oracle over the whole
recording.  The refusals, all before device work; the exported symbols.
GPU: the kernel equals the reference call by call and one gam_ctc_bias call over the whole stream; batch and keyword order
do not change a stream's bits; closed streams equal transcribe_windowed with hotwords; hotwords=None launches nothing new;
device memory; refusals and graph capture.
"""
import random

import numpy as np
import pytest
import torch

from gigaam_b200 import _lib, synthetic
from test_hotwords import (F32, NEG, _cpu_model, _greedy_batch, _planted_case, bias_oracle, greedy_of, hand_spotted,
                           rows, FLAGS, B8)
from test_keyword_spotting import _engine_for, _pad, tau_of


# ------------------------------------------------------------------------------------------ the reference
class SpotStream:
    """One keyword's gam_ctc_spot_resume over consecutive calls: the recursion, the detection scan and the early emission of
    the pending detection, one fp32 operation at a time."""

    def __init__(self, y, V1, threshold):
        U = len(y)
        self.S = S = 2 * U - 1
        self.lab = np.array([y[s // 2] if s % 2 == 0 else V1 - 1 for s in range(S)])
        self.skip = np.array([s % 2 == 0 and s >= 2 and y[s // 2] != y[s // 2 - 1] for s in range(S)])
        self.tau = tau_of(U, threshold)
        self.v = np.full(S, NEG, F32)
        self.a = np.zeros(S, np.int64)
        self.pending = None

    def walk(self, lp, t0, t1, finish):
        """Frames [t0, t1) of lp [T, V1] (stream frames) -> the detections emitted by the call."""
        out = []
        S = self.S
        for t in range(t0, t1):
            row = lp[t]
            if np.isnan(row).any():
                self.v, self.a = np.full(S, NEG, F32), np.full(S, t, np.int64)
            else:
                m = F32(row.max() + F32(0))
                c = (row[self.lab] - m).astype(F32)
                v, a = self.v, self.a
                best, start = v.copy(), a.copy()
                c1 = np.concatenate([[NEG], v[:-1]]).astype(F32)
                a1 = np.concatenate([[0], a[:-1]])
                take = c1 > best
                best, start = np.where(take, c1, best), np.where(take, a1, start)
                c2 = np.concatenate([[NEG, NEG], v[:-2]])[:S].astype(F32)
                a2 = np.concatenate([[0, 0], a[:-2]])[:S]
                take = self.skip & (c2 > best)
                best, start = np.where(take, c2, best), np.where(take, a2, start)
                if F32(0) > best[0]:
                    best[0], start[0] = F32(0), t
                self.v, self.a = (c + best).astype(F32), start
            E, Es = self.v[S - 1], int(self.a[S - 1])
            if E >= self.tau:
                p = self.pending
                if p is not None and Es < p[1]:
                    if E > p[2]:
                        self.pending = (Es, t + 1, E)
                else:
                    if p is not None:
                        out.append(p)
                    self.pending = (Es, t + 1, E)
        p = self.pending
        if p is not None and (finish or not any(self.v[s] > NEG and self.a[s] < p[1] for s in range(S))):
            out.append(p)
            self.pending = None
        return out

    def horizon(self):
        """The earliest start of a path that can still end as a detection: the pending one's, or a state's with v >= tau."""
        starts = [int(self.a[s]) for s in range(self.S) if self.v[s] >= self.tau]
        return min(starts + ([self.pending[0]] if self.pending is not None else []), default=None)


def release_frame(known, C, h, last_greedy, finish):
    """(D, R): the first undecided component's start and the release frame, from the known detections [(s, e)]."""
    if finish:
        return C, C
    L = min(h, last_greedy)
    D = C
    c0, c1 = 0, -1
    for s, e in sorted(known):
        if s >= c1:
            if c1 > L:
                D = c0
                break
            c0, c1 = s, e
        else:
            c1 = max(c1, e)
    else:
        if c1 > L:
            D = c0
    return D, min(h, D)


class ResumeReference:
    """The resumable rule over one stream: lp [T, V1], the greedy tokens of the whole stream, the hotwords.  call(C, finish)
    walks frames [C_prev, C) and returns (ids, frames, source, token_logp, R, frame_logp of the released frames)."""

    def __init__(self, lp, keywords, threshold, flags, g_ids, g_frames, token_logp=None, frame_logp=None):
        self.lp, self.keywords, self.threshold, self.flags = lp, keywords, threshold, flags
        self.g_ids, self.g_frames, self.tl, self.fl = list(g_ids), list(g_frames), token_logp, frame_logp
        self.spots = [SpotStream(y, lp.shape[1], threshold) for y in keywords]
        self.C = self.R = 0
        self.left = True
        self.carry = [[] for _ in keywords]
        self.released_greedy = 0

    def call(self, C, finish):
        new = [sp.walk(self.lp, self.C, C, finish) for sp in self.spots]
        self.C = C
        dets = [self.carry[k] + new[k] for k in range(len(self.keywords))]
        held = [i for i, f in enumerate(self.g_frames) if self.R <= f < C]
        starts = [sp.horizon() for sp in self.spots]
        h = min([C] + [s for s in starts if s is not None])
        last = self.g_frames[held[-1]] if held else -1
        D, R = release_frame([(s, e) for d in dets for s, e, _ in d], C, h, last, finish)
        out = self._release(dets, held, D, R, C, finish)
        self.carry = [[x for x in d if x[0] >= D] for d in dets]
        gone = [i for i in held if self.g_frames[i] < R]
        if gone:
            self.left = bool(self.flags[self.g_ids[gone[-1]]] & 1)
        self.R = R
        return out + (R,)

    def _release(self, dets, held, D, R, C, finish):
        """bias_oracle over the held span [R_prev, C) with the decided detections: the frames move one up behind a sentinel
        row and token that stands for what precedes the span (a space when it starts on a word boundary, a letter if not), and
        a span that does not finish ends past its greedy tokens."""
        base, V = self.R - 1, len(self.flags)
        flags = np.concatenate([self.flags, np.array([1, 0], np.uint8)])
        T = C - base
        lp = np.concatenate([self.lp[base + 1:base + 2], self.lp[base + 1:C]])[None]
        ids = [V if self.left else V + 1] + [self.g_ids[i] for i in held]
        frames = [0] + [self.g_frames[i] - base for i in held]
        n = len(ids)
        K = len(self.keywords)
        decided = [[x for x in d if x[0] < D] for d in dets]
        spotted = hand_spotted([(k, s - base, e - base, E) for k, d in enumerate(decided) for s, e, E in d], K,
                               max(1, max(len(d) for d in decided)))
        g = (np.array([ids + [0] * (T - n)], np.int32), np.array([frames + [0] * (T - n)], np.int32), [n])
        tl = None if self.tl is None else np.array([[F32(0)] + [self.tl[i] for i in held] + [F32(0)] * (T - n)], F32)
        fl = None if self.fl is None else np.concatenate([[0.0], self.fl[base + 1:C]])[None]
        got = bias_oracle(lp, [T], self.keywords, self.threshold, spotted, flags, *g, token_logp=tl, frame_logp=fl)
        keep = [i for i, f in enumerate(got["frames"][0]) if 1 <= f < R - base]
        o_ids = [got["ids"][0][i] for i in keep]
        o_fr = [got["frames"][0][i] + base for i in keep]
        o_src = [got["source"][0][i] for i in keep]
        o_tl = None if tl is None else [got["token_logp"][0][i] for i in keep]
        o_fl = None if fl is None else got["frame_logp"][0, 1:R - base]
        return o_ids, o_fr, o_src, o_tl, o_fl


def _splits(rng, T, spans=()):
    """Consecutive cut points ending at T: random steps, single frames, and cuts at span edges."""
    cuts = set()
    t = 0
    while t < T:
        t += int(rng.choice([1, 1, 2, 5, 17, 40]))
        cuts.add(min(t, T))
    for s, e in spans:
        if rng.random() < 0.5:
            cuts.update(x for x in (s, e) if 0 < x <= T)
    return sorted(cuts | {T})


def _stream_equals_whole(lp, keywords, theta, flags, rng, scored):
    T = lp.shape[0]
    ids, frames = greedy_of(lp)
    tl = rng.normal(-0.1, 0.05, max(1, len(ids))).astype(F32) if scored else None
    fl = rng.normal(-0.01, 0.01, T) if scored else None
    g = (np.array([ids + [0] * (T - len(ids))], np.int32), np.array([frames + [0] * (T - len(ids))], np.int32), [len(ids)])
    from test_keyword_spotting import spot_oracle
    spotted = spot_oracle(lp[None], [T], keywords, theta, T, lp.shape[1] - 1)
    want = bias_oracle(lp[None], [T], keywords, theta, spotted, flags, *g,
                       token_logp=None if tl is None else np.concatenate([tl, np.zeros(T, F32)])[None, :T],
                       frame_logp=None if fl is None else fl[None])
    spans = [(int(spotted[0][0, k, j]), int(spotted[1][0, k, j])) for k in range(len(keywords))
             for j in range(min(int(spotted[3][0, k]), spotted[0].shape[2]))]
    ref = ResumeReference(lp, keywords, theta, flags, ids, frames, tl, fl)
    got = [[], [], [], [], []]
    Rs = []
    for C in _splits(rng, T, spans):
        o = ref.call(C, C == T)
        for i in range(4):
            if o[i] is not None:
                got[i] += o[i]
        if o[4] is not None:
            got[4].append(o[4])
        Rs.append(o[5])
    assert Rs == sorted(Rs) and Rs[-1] == T
    assert got[0] == want["ids"][0] and got[1] == want["frames"][0] and got[2] == want["source"][0]
    if scored:
        assert np.array_equal(np.array(got[3], F32).view(np.int32), np.array(want["token_logp"][0], F32).view(np.int32))
        assert np.array_equal(np.concatenate(got[4]), want["frame_logp"][0])
    return want


# ------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("sp", [False, True])
def test_reference_splits_equal_the_whole_recording(sp):
    rng = np.random.default_rng(11 + sp)
    splices = 0
    for case in range(6):
        V1 = [34, 257][sp] if case % 2 else 34 + 2 * sp
        lp, keywords, flags = _planted_case(rng, V1, 1, 160, sp)
        for theta in (0.2, 0.6):
            want = _stream_equals_whole(lp[0], keywords, theta, flags, rng, scored=case % 3 == 0)
            splices += sum(not a[3] for a in want["accepted"][0])
    assert splices >= 10


def test_reference_hand_cases():
    rng = np.random.default_rng(3)
    # a misspelling replaced, an identity, edge spaces on both sides, and SentencePiece openers
    cases = [(rows([0, B8, 1, 2, B8, 0, 3, 3, 5, 5, B8, 0], second={8: 4, 9: 4}), [[3, 4]], 0.5, FLAGS),
             (rows([0, B8, 1, 2, B8, 0, 3, 3, 4, B8, 0]), [[3, 4]], 1.0, FLAGS),
             (rows([0, 1, B8, 0, 5, 6, B8], second={2: (3, F32(-0.3)), 3: (B8, F32(-0.3))}), [[3, 5, 6]], 0.3, FLAGS),
             (rows([0, 5, 0, B8, B8, 1], second={2: (B8, F32(-0.3)), 3: (3, F32(-0.3))}), [[5, 3]], 0.3, FLAGS),
             (rows([7, 1, 2, 7, 3, 5, 5], second={5: 4, 6: 4}), [[7, 3, 4], [3, 4]], 0.3, FLAGS),
             # overlapping candidates of different hotwords
             (rows([0, 1, 2, B8, 0, 3, 4, B8, 0], second={1: 5, 2: 6, 5: 6, 6: 5}), [[5, 6], [6, 5], [1, 2, 0, 3]], 0.4, FLAGS)]
    for lp, kws, theta, flags in cases:
        for _ in range(8):
            _stream_equals_whole(lp, kws, theta, flags, rng, scored=True)


def test_a_silent_tail_keeps_a_candidate_undecided():
    # "12 3" then a long silence: the greedy 3 at frame 5 is followed by no greedy token, so the candidate (3, 4) over it is
    # not decided (its right boundary is unknown) until the stream finishes
    lp = rows([0, 1, 2, B8, 0, 3, 3] + [B8] * 30, second={6: 4})
    ids, frames = greedy_of(lp)
    ref = ResumeReference(lp, [[3, 4]], 0.5, FLAGS, ids, frames)
    Rs = [ref.call(C, False)[5] for C in range(8, lp.shape[0])]
    assert all(R <= 5 for R in Rs) and (any(ref.carry) or ref.spots[0].pending is not None)
    o = ref.call(lp.shape[0], True)
    assert o[0][-2:] == [3, 4] and o[5] == lp.shape[0]


def test_refusals_come_before_device_work():
    model = _cpu_model("v2_ctc")
    tok = model.decoding.tokenizer
    V, sp = len(tok), tok.vocab.index(" ")
    for kws, match in [([], "no keywords"), ([[]], "without tokens"), ([[0, V]], "outside"), ([[sp, 3]], "space token"),
                       ([[3, sp]], "space token")]:
        with pytest.raises(ValueError, match=match):
            model.streaming(hotwords=kws)
    for theta in (0.0, 1.5, float("nan")):
        with pytest.raises(ValueError, match="threshold"):
            model.streaming(hotwords=["да"], hotword_threshold=theta)
    for name in ("v2_rnnt", "v3_e2e_rnnt"):
        with pytest.raises(NotImplementedError, match="_ctc"):
            _cpu_model(name).streaming(hotwords=["а"])
    srv = model.streaming(hotwords=["да"], keywords=["нет"])
    assert srv.hw_ids and srv._eng is None


def test_exports():
    lib = _lib.load()
    for name in ("gam_ctc_bias_resume", "gam_ctc_bias_resume_workspace_bytes"):
        assert name in _lib.EXPORTS and hasattr(lib, name)


# ------------------------------------------------------------------------------------------ GPU
def _dev():
    return torch.device("cuda", 0)


class KernelStreams:
    """A batch of streams over host log-probs lp [B, T, V1] driven through Engine.ctc_spot_resume and
    Engine.ctc_bias_resume, the caller's hold kept on the host: call(Cs, finish) advances stream b to frame Cs[b]."""

    def __init__(self, eng, lp, keywords, theta, flags, greedy, scores=None):
        self.eng, self.lp, self.keywords, self.theta = eng, lp, keywords, theta
        self.B = lp.shape[0]
        self.flags = torch.as_tensor(flags).to(_dev())
        self.flags_host = flags
        self.kw, self.kw_len = (t.to(_dev()) for t in _pad(keywords))
        self.state = eng.spot_state(self.B, len(keywords), self.kw.shape[1])
        self.g_ids, self.g_frames = greedy
        self.tl, self.fl = scores if scores is not None else (None, None)
        self.C = [0] * self.B
        self.R = [0] * self.B
        self.left = [True] * self.B
        self.carry = [[[] for _ in keywords] for _ in range(self.B)]

    def call(self, Cs, finish):
        eng, dev, B, K = self.eng, _dev(), self.B, len(self.keywords)
        i32 = dict(dtype=torch.int32, device=dev)
        Tn = max(1, max(c - c0 for c, c0 in zip(Cs, self.C)))
        new = np.zeros((B, Tn, self.lp.shape[2]), F32)
        for b in range(B):
            new[b, :Cs[b] - self.C[b]] = self.lp[b, self.C[b]:Cs[b]]
        rng = torch.tensor([[0] * B, [c - c0 for c, c0 in zip(Cs, self.C)], self.C, [int(finish)] * B], dtype=torch.int32).to(dev)
        md = Tn // min(len(y) for y in self.keywords) + 2
        det = (torch.empty((B, K, md), **i32), torch.empty((B, K, md), **i32), torch.empty((B, K, md), dtype=torch.float32, device=dev),
               torch.zeros((B, K), **i32))
        eng.ctc_spot_resume(torch.as_tensor(new).to(dev), rng[0], rng[1], rng[2], rng[3], self.kw, self.kw_len, self.theta,
                            self.state, det)
        st, en, sc, cnt = (t.cpu().numpy() for t in det)
        for b in range(B):
            for k in range(K):
                self.carry[b][k] += [(int(st[b, k, j]), int(en[b, k, j]), F32(sc[b, k, j])) for j in range(int(cnt[b, k]))]
        T = max(1, max(c - r for c, r in zip(Cs, self.R)))
        lp = np.zeros((B, T, self.lp.shape[2]), F32)
        held = []
        for b in range(B):
            lp[b, :Cs[b] - self.R[b]] = self.lp[b, self.R[b]:Cs[b]]
            held.append([i for i in range(len(self.g_frames[b])) if self.R[b] <= self.g_frames[b][i] < Cs[b]])
        m = max(T, max(len(h) for h in held))
        ids = np.zeros((B, m), np.int32)
        frames = np.zeros((B, m), np.int32)
        tl = None if self.tl is None else np.zeros((B, m), F32)
        fl = None if self.fl is None else np.zeros((B, T))
        for b, h in enumerate(held):
            ids[b, :len(h)] = [self.g_ids[b][i] for i in h]
            frames[b, :len(h)] = [self.g_frames[b][i] for i in h]
            if tl is not None:
                tl[b, :len(h)] = [self.tl[b][i] for i in h]
                fl[b, :Cs[b] - self.R[b]] = self.fl[b, self.R[b]:Cs[b]]
        mdet = max(1, max(len(d) for c in self.carry for d in c))
        dd = (np.full((B, K, mdet), -1, np.int32), np.full((B, K, mdet), -1, np.int32), np.zeros((B, K, mdet), F32),
              np.zeros((B, K), np.int32))
        for b in range(B):
            for k, d in enumerate(self.carry[b]):
                for j, (a, e, x) in enumerate(d):
                    dd[0][b, k, j], dd[1][b, k, j], dd[2][b, k, j] = a, e, x
                dd[3][b, k] = len(d)
        fl_d = None if fl is None else torch.as_tensor(fl).to(dev)
        hr = torch.tensor([[c - r for c, r in zip(Cs, self.R)], self.R, [int(finish)] * B, [int(x) for x in self.left],
                           [len(h) for h in held]], dtype=torch.int32).to(dev)
        out = eng.ctc_bias_resume(torch.as_tensor(lp).to(dev), hr[0], hr[1], hr[2], self.kw, self.kw_len, self.theta, self.state,
                                  tuple(torch.as_tensor(x).to(dev) for x in dd), self.flags, torch.as_tensor(ids).to(dev),
                                  torch.as_tensor(frames).to(dev), hr[4], hr[3], None if tl is None else torch.as_tensor(tl).to(dev),
                                  fl_d)
        o = [None if t is None else t.cpu().numpy() for t in out]
        res = []
        for b in range(B):
            n, R = int(o[2][b]), int(o[5][b])
            res.append((o[0][b, :n].tolist(), o[1][b, :n].tolist(), o[3][b, :n].tolist(),
                        None if o[4] is None else o[4][b, :n].view(np.int32).tolist(), R,
                        None if fl_d is None else fl_d[b, :R - self.R[b]].cpu().numpy()))
            gone = [i for i in held[b] if self.g_frames[b][i] < R]
            if gone:
                self.left[b] = bool(self.flags_host[self.g_ids[b][gone[-1]]] & 1)
            self.carry[b] = [[(int(o[6][b, k, j]), int(o[7][b, k, j]), F32(o[8][b, k, j])) for j in range(int(o[9][b, k]))]
                             for k in range(K)]
            self.R[b] = R
        self.C = list(Cs)
        return res


def _cut_lists(rng, B, T, n):
    """n increasing cut points per stream, the last at T; some one frame apart."""
    out = []
    for _ in range(B):
        pts = sorted(set(int(x) for x in rng.integers(1, T, 3 * n)))
        while len(pts) < n - 1:
            pts = sorted(set(pts) | {int(rng.integers(1, T))})
        pick = sorted(rng.choice(pts, n - 1, replace=False).tolist()) + [T]
        out.append(pick)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("V1", [34, 257, 1025])
def test_kernel_equals_the_reference_and_one_shot_bias(V1):
    rng = np.random.default_rng(V1 + 1)
    B, T, n_calls = 3, 240, 12
    sp = V1 == 257
    lp, keywords, flags = _planted_case(rng, V1, B, T, sp)
    eng = _engine_for(V1)
    g_ids, g_frames = zip(*[greedy_of(lp[b]) for b in range(B)])
    tl = [rng.normal(-0.1, 0.05, max(1, len(x))).astype(F32) for x in g_ids]
    fl = rng.normal(-0.01, 0.01, (B, T))
    splices = 0
    for theta in (0.25, 0.6):
        drv = KernelStreams(eng, lp, keywords, theta, flags, (g_ids, g_frames), (tl, fl))
        refs = [ResumeReference(lp[b], keywords, theta, flags, g_ids[b], g_frames[b], tl[b], fl[b]) for b in range(B)]
        cuts = _cut_lists(rng, B, T, n_calls)
        whole = [[[], [], [], [], []] for _ in range(B)]
        for i in range(n_calls):
            got = drv.call([c[i] for c in cuts], i == n_calls - 1)
            for b in range(B):
                want = refs[b].call(cuts[b][i], i == n_calls - 1)
                assert got[b][4] == want[5], (theta, i, b)
                assert got[b][:3] == tuple(want[:3]), (theta, i, b)
                assert got[b][3] == np.array(want[3], F32).view(np.int32).tolist()
                assert np.array_equal(got[b][5], want[4])
                for j in range(4):
                    whole[b][j] += got[b][j]
                whole[b][4].append(got[b][5])
        # one gam_ctc_bias call over the whole streams
        dev = _dev()
        kw, kw_len = (t.to(dev) for t in _pad(keywords))
        lp_d = torch.as_tensor(lp).to(dev)
        enc = torch.full((B,), T, dtype=torch.int32, device=dev)
        spotted = eng.ctc_spot(lp_d, enc, kw, kw_len, theta, T)
        gi, gf, gc = _greedy_batch(lp, [T] * B)
        tl_b = np.zeros((B, T), F32)
        for b in range(B):
            tl_b[b, :len(g_ids[b])] = tl[b][:len(g_ids[b])]
        fl_d = torch.as_tensor(fl).to(dev)
        one = eng.ctc_bias(lp_d, enc, kw, kw_len, spotted, theta, torch.as_tensor(flags), *(torch.as_tensor(x).to(dev) for x in (gi, gf, gc)),
                           torch.as_tensor(tl_b).to(dev), torch.zeros(B, device=dev), fl_d)
        one = [None if t is None else t.cpu().numpy() for t in one]
        for b in range(B):
            n = int(one[2][b])
            assert whole[b][0] == one[0][b, :n].tolist() and whole[b][1] == one[1][b, :n].tolist()
            assert whole[b][2] == one[3][b, :n].tolist() and whole[b][3] == one[4][b, :n].view(np.int32).tolist()
            assert np.array_equal(np.concatenate(whole[b][4]), fl_d[b].cpu().numpy())
            splices += sum(1 for x, y in zip(whole[b][0], gi[b, :int(gc[b])].tolist()) if x != y)
    print(f"\n{splices} changed token positions")
    assert splices > 0


@pytest.mark.gpu
def test_a_stream_does_not_depend_on_its_batch_or_the_hotword_order():
    rng = np.random.default_rng(8)
    V1, B, T, n_calls = 34, 4, 200, 9
    lp, keywords, flags = _planted_case(rng, V1, B, T, False)
    eng = _engine_for(V1)
    greedy = tuple(zip(*[greedy_of(lp[b]) for b in range(B)]))
    cuts = _cut_lists(rng, B, T, n_calls)
    perm = list(range(len(keywords)))[::-1]
    batch = KernelStreams(eng, lp, keywords, 0.3, flags, greedy)
    flipped = KernelStreams(eng, lp, [keywords[k] for k in perm], 0.3, flags, greedy)
    alone = [KernelStreams(eng, lp[b:b + 1], keywords, 0.3, flags, ([greedy[0][b]], [greedy[1][b]])) for b in range(B)]
    for i in range(n_calls):
        fin = i == n_calls - 1
        got = batch.call([c[i] for c in cuts], fin)
        got_f = flipped.call([c[i] for c in cuts], fin)
        for b in range(B):
            a = alone[b].call([cuts[b][i]], fin)[0]
            assert got[b][:2] == a[:2] and got[b][2] == a[2] and got[b][4] == a[4]
            assert got_f[b][:2] == a[:2] and got_f[b][4] == a[4]
            assert got_f[b][2] == [-1 if k < 0 else perm[k] for k in a[2]] or all(
                keywords[perm[x]] == keywords[y] for x, y in zip(got_f[b][2], a[2]) if x >= 0)


@pytest.mark.gpu
def test_refusals_and_graph_capture():
    eng = _engine_for(34)
    lib, h, dev = eng.lib, eng.handle, _dev()
    rng = np.random.default_rng(4)
    lp, keywords, flags = _planted_case(rng, 34, 2, 120, False)
    greedy = tuple(zip(*[greedy_of(lp[b]) for b in range(2)]))
    drv = KernelStreams(eng, lp, keywords, 0.3, flags, greedy)
    drv.call([50, 70], False)
    bad_state = drv.state[:, :, :-4].contiguous()
    with pytest.raises(_lib.GamError, match="record_bytes"):
        eng.ctc_bias_resume(torch.zeros((2, 8, 34), device=dev), *(torch.zeros(2, dtype=torch.int32, device=dev) for _ in range(3)),
                            drv.kw, drv.kw_len, 0.3, bad_state, tuple(torch.zeros((2, len(keywords), 2), dtype=d, device=dev)
                                                                      for d in (torch.int32, torch.int32, torch.float32)) +
                            (torch.zeros((2, len(keywords)), dtype=torch.int32, device=dev),), drv.flags,
                            torch.zeros((2, 8), dtype=torch.int32, device=dev), torch.zeros((2, 8), dtype=torch.int32, device=dev),
                            torch.zeros(2, dtype=torch.int32, device=dev), torch.ones(2, dtype=torch.int32, device=dev))
    z = torch.zeros(64, dtype=torch.int32, device=dev)
    p = z.data_ptr()
    args = lambda **kw: [kw.get(n, p) for n in ("lp", "hi", "base", "fin", "kw", "kwl")]
    for nulls in ("hi", "base", "fin"):
        a = args(**{nulls: None})
        rc = lib.gam_ctc_bias_resume(h, a[0], 1, 4, a[1], a[2], a[3], a[4], a[5], 1, 1, p, 0, p, p, p, p, 1, 0.5, p, 33, p, p, p, p, 4,
                                     None, None, 0, p, 1 << 20, p, p, p, p, None, p, p, p, p, p, None)
        assert rc != 0 and b"required" in lib.gam_last_error(h)
    rc = lib.gam_ctc_bias_resume(h, p, 1, 4, p, p, p, p, p, 1, 1, p, int(eng.lib.gam_ctc_spot_state_bytes(h, 1)), p, p, p, p, 1, 0.5, p,
                                 33, p, p, p, p, 4, None, None, 0, p, 16, p, p, p, p, None, p, p, p, p, p, None)
    assert rc != 0 and b"workspace" in lib.gam_last_error(h).lower()
    # graph capture of one launch, replayed with other inputs
    B, T = 2, 120
    state = drv.state
    bufs = [torch.as_tensor(lp).to(dev), torch.tensor([T, T], dtype=torch.int32, device=dev)]
    g_ids = np.zeros((B, T), np.int32)
    g_fr = np.zeros((B, T), np.int32)
    for b in range(B):
        g_ids[b, :len(greedy[0][b])], g_fr[b, :len(greedy[1][b])] = greedy[0][b], greedy[1][b]
    ids, frs = torch.as_tensor(g_ids).to(dev), torch.as_tensor(g_fr).to(dev)
    cnt = torch.tensor([len(x) for x in greedy[0]], dtype=torch.int32, device=dev)
    zero = torch.zeros(B, dtype=torch.int32, device=dev)
    one_ = torch.ones(B, dtype=torch.int32, device=dev)
    spotted = eng.ctc_spot(bufs[0], bufs[1], drv.kw, drv.kw_len, 0.3, T)

    def step():
        return eng.ctc_bias_resume(bufs[0], bufs[1], zero, one_, drv.kw, drv.kw_len, 0.3, state, spotted, drv.flags, ids, frs, cnt, one_)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            got = step()
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    want = eng.ctc_bias(bufs[0], bufs[1], drv.kw, drv.kw_len, spotted, 0.3, drv.flags, ids, frs, cnt)
    for x, y in ((got[0], want[0]), (got[1], want[1]), (got[3], want[3])):
        for b in range(B):
            n = int(want[2][b])
            assert int(got[2][b]) == n and torch.equal(x[b, :n], y[b, :n])
    assert got[5].tolist() == [T, T] and int(got[9].sum()) == 0


_MODELS = {}


def _model(name):
    if name not in _MODELS:
        import gigaam_b200 as gigaam
        _MODELS[name] = gigaam.load_model(name, fp16_encoder=False, device=_dev(),
                                          checkpoint=synthetic.synthetic_checkpoint(name, seed=0, n_layers=1))
    return _MODELS[name]


def _near_misses(model, wavs, per_wav=6):
    """Hotwords (token ids) one token away from the model's own greedy words in the recordings: the middle token of a word
    becomes the runner-up class at its frame, so the hotword scores close behind greedy and splices happen.  -> (hotwords,
    greedy words)."""
    from gigaam_b200.longform import plan_windows, stitch_ctc_log_probs
    from gigaam_b200.timestamps_utils import token_flag_table
    flags = token_flag_table(model.decoding.tokenizer).numpy()
    V = len(flags)
    words, hot = [], []
    for wav in wavs:
        windows, T = plan_windows(wav.numel(), 8.0, 4.0, model._encoded_length, model._max_frames)
        w_d, _ = model.prepare_wav(wav)
        lp = stitch_ctc_log_probs(model, w_d[0], windows, T, 4)[0].cpu().numpy()
        ids, frames = greedy_of(lp)
        found, cur = [], []
        for tok, f in list(zip(ids, frames)) + [(None, None)]:
            if tok is None or flags[tok] & 1 or (flags[tok] & 2 and cur):
                if 2 <= len(cur) <= 8:
                    found.append(cur)
                elif len(cur) > 8:   # a run without word boundaries: its hotwords are spotted but never eligible
                    found.append(cur[:4])
                cur = []
            if tok is not None and not flags[tok] & 1:
                cur.append((tok, f))
        for word in found[:per_wav]:
            i = len(word) // 2
            tok, f = word[i]
            alt = next((int(c) for c in np.argsort(-lp[f]) if c < V and c != tok and not flags[c] & 1
                        and flags[c] & 2 == flags[tok] & 2), None)
            if alt is not None:
                hot.append([t for t, _ in word[:i]] + [alt] + [t for t, _ in word[i + 1:]])
                words.append([t for t, _ in word])
    return hot, words


@pytest.mark.gpu
@pytest.mark.parametrize("confidence", [False, True])
@pytest.mark.parametrize("name", ["v2_ctc", "v3_e2e_ctc"])
def test_closed_streams_equal_transcribe_windowed_with_hotwords(name, confidence):
    from test_streaming import _drive, _recordings
    model = _model(name)
    wavs = _recordings(5 + confidence, n=7)
    hot, words = _near_misses(model, wavs)
    keywords = words[:2]
    assert hot
    changed = 0
    with torch.inference_mode():
        for seed in (1, 2):
            srv = model.streaming(window=8.0, overlap=4.0, batch_size=3, confidence=confidence, keywords=keywords,
                                  hotwords=hot, hotword_threshold=0.1)
            results, updates = _drive(srv, wavs, random.Random(seed))
            tok = model.decoding.tokenizer
            for i, w in enumerate(wavs):
                want = model.transcribe_windowed(w, word_timestamps=True, confidence=confidence, window=8.0, overlap=4.0, pause=0.3,
                                                  max_segment=6.0, hotwords=hot, hotword_threshold=0.1)
                assert repr(results[i].transcript) == repr(want), (seed, i)
                assert repr(results[i].detections) == repr(model.spot(w, keywords, window=8.0, overlap=4.0))
                committed = [t for u in updates[i] for t in u.new_tokens]
                assert "".join(u.new_text for u in updates[i]) == tok.decode(committed)
                times = [u.committed_until for u in updates[i]]
                assert times == sorted(times)
                if seed == 1:
                    plain = model.transcribe_windowed(w, window=8.0, overlap=4.0)
                    changed += want.text != plain.text
    print(f"\n{len(hot)} hotwords, {changed} of {len(wavs)} transcripts changed by them")
    if name == "v2_ctc":   # the synthetic v3_e2e_ctc writes no word openers, so nothing is eligible there
        assert changed > 0


@pytest.mark.gpu
@pytest.mark.parametrize("batch_size", [64, 1])
def test_hotwords_none_runs_only_the_plain_launches(monkeypatch, batch_size):
    """Without hotwords a step makes exactly the launches of its encoder batches and greedy rounds (no head, spot or bias
    launch), and the closed stream is transcribe_windowed's.  batch_size 1 puts the stream's older windows in groups that
    hold no stream's newest window, which have no tentative decode."""
    import gigaam_b200.streaming as streaming
    model = _model("v2_ctc")
    eng = model._get_engine()
    wav, _ = synthetic.synthetic_audio(1, 30.0, seed=12)
    wav = wav[0]
    inside = []

    def counted(fn, what):
        def run(*a, **kw):
            n0 = eng.launch_count()
            out = fn(*a, **kw)
            inside.append((what, eng.launch_count() - n0))
            return out
        return run
    monkeypatch.setattr(streaming, "encode_rows", counted(streaming.encode_rows, "encode"))
    monkeypatch.setattr(eng, "greedy_resume", counted(eng.greedy_resume, "greedy"))
    for name in ("ctc_spot_resume", "ctc_bias_resume", "ctc_log_probs"):
        monkeypatch.setattr(eng, name, lambda *a, _n=name, **kw: pytest.fail(f"{_n} called without hotwords or keywords"))
    with torch.inference_mode():
        srv = model.streaming(window=8.0, overlap=4.0, batch_size=batch_size)
        a = srv.open()
        srv.push(a, wav[:20 * 16000].numpy())            # three ready windows in one step
        inside.clear()
        n0 = eng.launch_count()
        updates = srv.step()
        total = eng.launch_count() - n0
        what = [w for w, _ in inside]
        assert total == sum(n for _, n in inside) > 0
        groups = 1 if batch_size == 64 else 3
        assert what.count("encode") == groups and what.count("greedy") == 3 + 1   # three rounds and one tentative decode
        srv.push(a, wav[20 * 16000:].numpy())
        res = srv.close(a, word_timestamps=True)
    monkeypatch.undo()
    want = model.transcribe_windowed(wav, word_timestamps=True, window=8.0, overlap=4.0)
    assert repr(res.transcript) == repr(want)
    assert len(updates) == 1 and updates[0].committed_until > 0


@pytest.mark.gpu
def test_stream_device_memory_stays_flat_with_hotwords():
    model = _model("v2_ctc")
    wav, _ = synthetic.synthetic_audio(1, 240.0, seed=21)
    hot = [[1, 2], [2, 3, 4], [5, 1], [3, 3]]
    with torch.inference_mode():
        srv = model.streaming(window=8.0, overlap=4.0, hotwords=hot, hotword_threshold=0.1)
        a = srv.open()
        mem, held = [], []
        for i in range(0, wav.shape[1], 4 * 16000):
            srv.push(a, wav[0, i:i + 4 * 16000].numpy())
            srv.step()
            torch.cuda.synchronize()
            s = srv._streams[a]
            held.append(0 if s.hw_rows is None else s.hw_rows.shape[0])
            mem.append(torch.cuda.memory_allocated() - (0 if s.hw_rows is None else s.hw_rows.untyped_storage().nbytes()))
        srv.close(a)
    print(f"\nheld rows: max {max(held)}, memory spread {(max(mem[5:]) - min(mem[5:])) / 2**20:.2f} MiB")
    assert max(mem[5:]) - min(mem[5:]) < 8 * 2**20
