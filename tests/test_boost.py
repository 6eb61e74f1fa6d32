"""Phrase boosting in the RNN-T greedy decoder (include/gigaam_b200.h, gam_rnnt_greedy_boost; INTEGRATION.md §7j).

CPU: the boost graph builder (decoding.boost_graph) against a brute-force restatement of the phrase rule, walks of random
token sequences, every refusal, `boost=None` taking exactly the paths it took before, and the exports.

GPU: every decision of gam_test_rnnt_greedy_boost against a float64 replay of the boosted rule (q and the bonus carried
along the trace) on both sides of the boosted shared-memory / L2 boundary; exact ties; non-finite rows; zero bonuses against
gam_rnnt_greedy_resume bit for bit; scores against float64; chunking, batch invariance and CUDA-graph replay of the engine
call; and the public calls (transcribe, transcribe_windowed, streaming) on the synthetic v2_rnnt and v3_e2e_rnnt models."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, synthetic
from gigaam_b200.decoding import BOOST_MAX_STATES, boost_graph
from test_greedy_decisions import (H, JOINT_TIE, T_SWEEP, _call, _dev_weights, _tie_weights, dev, eng, geometry,  # noqa: F401
                                   make_encproj, make_lens, make_weights)

_CPU_MODELS = {}


def _cpu_model(name):
    if name not in _CPU_MODELS:
        _CPU_MODELS[name] = gigaam.load_model(name, device="cpu", checkpoint=synthetic.synthetic_checkpoint(name, n_layers=1))
    return _CPU_MODELS[name]


# ------------------------------------------------------------------------------------------ CPU: the phrase rule
def _prefixes(phrases, anchor):
    pats = {tuple(([] if anchor is None else [anchor]) + list(p)) for p in phrases}
    return {p[:k] for p in pats for k in range(len(p) + 1)}


def _longest_suffix(s, Pi):
    return next(s[k:] for k in range(len(s) + 1) if s[k:] in Pi)


def _state_names(nxt, Pi, anchor):
    """Each state id's prefix: a nonempty prefix is the walk of its tokens from state 0 (the anchor's state, whose own token
    the walk skips); the one id no walk reaches is the empty prefix."""
    name = {}
    for s in Pi:
        if s:
            q = 0
            for t in (s[1:] if anchor is not None else s):
                q = int(nxt[q, t])
            assert q not in name, (s, name.get(q))
            name[q] = s
    rest = set(range(nxt.shape[0])) - set(name)
    assert len(rest) == 1
    name[rest.pop()] = ()
    return name


def _random_sets(seed):
    rng = random.Random(seed)
    V = rng.choice([4, 6, 33, 257])
    anchor = rng.choice([None, 0])
    lo = 1 if anchor == 0 else 0
    ph = [[rng.randrange(lo, V) for _ in range(rng.randint(1, 6))] for _ in range(rng.randint(1, 6))]
    ph.append(ph[0] + [rng.randrange(lo, V) for _ in range(3)])     # a shared prefix ("газ" / "газпром")
    if len(ph[1]) > 1:
        ph.append(ph[1][1:])                                            # a suffix of another phrase
    ph.append([ph[0][0]] * 3)                                           # repeated tokens
    ph.append(list(ph[0]))                                              # a duplicate
    return V, anchor, ph


@pytest.mark.parametrize("seed", range(40))
def test_builder_equals_the_brute_force_rule(seed):
    V, anchor, ph = _random_sets(seed)
    V1, blank, lam = V + 1, V, 1.75
    nxt, bonus = (t.numpy() for t in boost_graph(ph, lam, anchor, V1, blank))
    Pi = _prefixes(ph, anchor)
    start = () if anchor is None else (anchor,)
    assert nxt.shape == bonus.shape == (len(Pi), V1) and nxt.dtype == np.int32 and bonus.dtype == np.float32
    name = _state_names(nxt, Pi, anchor)
    assert name[0] == start
    for q, s in name.items():
        for v in range(V):
            t = _longest_suffix(s + (v,), Pi)
            assert name[int(nxt[q, v])] == t, (s, v)
            assert bonus[q, v] == (np.float32(lam) if t not in ((), start) else 0), (s, v, t)
        assert nxt[q, blank] == q and bonus[q, blank] == 0


@pytest.mark.parametrize("seed", range(10))
def test_walks_end_in_the_longest_suffix(seed):
    V, anchor, ph = _random_sets(100 + seed)
    nxt, _ = (t.numpy() for t in boost_graph(ph, 1.0, anchor, V + 1, V))
    Pi = _prefixes(ph, anchor)
    name = _state_names(nxt, Pi, anchor)
    rng = random.Random(seed)
    words = [t for p in ph for t in p] + ([anchor] if anchor is not None else [])
    q, hist = 0, () if anchor is None else (anchor,)   # the transcript's start is a word start
    for _ in range(400):
        v = rng.choice(words) if rng.random() < 0.7 else rng.randrange(V + 1)
        q = int(nxt[q, v])
        if v != V:
            hist += (v,)
        assert name[q] == _longest_suffix(hist, Pi)


def test_charwise_phrases_are_anchored_at_word_starts():
    tok = _cpu_model("v2_rnnt").decoding.tokenizer
    sp = tok.vocab.index(" ")
    gas, gazprom = tok.encode("газ"), tok.encode("газпром")
    nxt, bonus = (t.numpy() for t in boost_graph([gas, gazprom], 2.0, sp, len(tok) + 1, len(tok)))

    def walk(text):
        q, got = 0, []
        for t in tok.encode(text):
            got.append(float(bonus[q, t]))
            q = int(nxt[q, t])
        return got
    assert walk("газпром") == [2.0] * 7                                  # the start of the transcript is a word start
    assert walk("да газпром") == [0, 0, 0] + [2.0] * 7
    assert walk("эгаз") == [0, 0, 0, 0]                                 # never inside a word
    assert walk("газ газ") == [2.0] * 3 + [0] + [2.0] * 3


def test_refusals_come_before_device_work():
    model = _cpu_model("v2_rnnt")
    tok = model.decoding.tokenizer
    V, sp = len(tok), tok.vocab.index(" ")
    wav = np.zeros(16000, np.float32)
    bad = [([], "no phrases"), (["123"], "no tokens"), ([[]], "without tokens"), (["а" * 65], "65 tokens"), ([[0, V]], "outside"),
           ([[sp, 3]], "space token"), ([[3, sp]], "space token"), ([[sp]], "space token")]
    for phrases, match in bad:
        with pytest.raises(ValueError, match=match):
            model.transcribe(wav, boost=phrases)
        with pytest.raises(ValueError, match=match):
            model.transcribe_windowed(wav, boost=phrases)
        with pytest.raises(ValueError, match=match):
            model.streaming(boost=phrases)
    for w in (0.0, -1.0, float("nan"), float("inf"), 1e-50, 1e39):
        with pytest.raises(ValueError, match="weight"):
            model.transcribe(wav, boost=["да"], boost_weight=w)
        with pytest.raises(ValueError, match="weight"):
            model.streaming(boost=["да"], boost_weight=w)
    model._boost_tables([[3, sp, 4], "да нет"], 1.0, "transcribe")      # a space inside a phrase is fine
    rng = np.random.default_rng(0)
    many = [rng.integers(0, 30, size=64).tolist() for _ in range(BOOST_MAX_STATES // 60)]
    with pytest.raises(ValueError, match="states"):
        boost_graph(many, 1.0, None, 31, 30)
    ctc = _cpu_model("v2_ctc")
    for call in (lambda: ctc.transcribe(wav, boost=["да"]), lambda: ctc.transcribe_windowed(wav, boost=["да"]),
                 lambda: ctc.streaming(boost=["да"])):
        with pytest.raises(NotImplementedError, match="hotwords="):
            call()
    with pytest.raises(NotImplementedError, match="_ctc"):             # hotwords keep their own refusal on RNN-T
        model.transcribe(wav, hotwords=["да"])


def test_boost_none_runs_the_plain_path(monkeypatch):
    import gigaam_b200.longform as longform
    from gigaam_b200.engine import DecodeBuffers
    model = _cpu_model("v2_rnnt")
    log = []
    enc = torch.zeros((1, 768, 25))
    monkeypatch.setattr(model, "forward", lambda wav, length: (log.append("forward"), (enc, torch.tensor([25])))[1])
    monkeypatch.setattr(model, "_decode", lambda *a: (log.append(("decode",) + tuple(a[3:])), [("txt", None, None)])[1])

    class Recorder:
        device = torch.device("cpu")
        num_classes = 35

        def group_words(self, ids, frames, counts, flags):
            B, m = ids.shape
            return [torch.zeros((B, m), dtype=torch.int32) for _ in range(4)] + [torch.zeros(B, dtype=torch.int32)]

        def __getattr__(self, name):      # greedy_resume with tables, decode_state and any other engine call
            raise AssertionError(f"unexpected engine call {name}")
    monkeypatch.setattr(model, "_get_engine", lambda: Recorder())
    wav = np.zeros(16000, np.float32)
    for kwargs in ({}, {"boost": None}, {"boost": None, "boost_weight": 3.0}):
        log.clear()
        assert model.transcribe(wav, word_timestamps=True, **kwargs).text == "txt"
        assert log == ["forward", ("decode", True, False)]
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)

    def fake_decode(m, host, windows, T, batch_size, scores, *extra, **kw):
        log.append(("decode_windows", len(extra), tuple(kw)))
        i32 = dict(dtype=torch.int32)
        return DecodeBuffers(torch.zeros((1, T), **i32), torch.zeros((1, T), **i32), torch.zeros(1, **i32))
    monkeypatch.setattr(longform, "decode_windows", fake_decode)
    for kwargs in ({}, {"boost": None}):
        log.clear()
        model.transcribe_windowed(wav, **kwargs)
        assert log == [("decode_windows", 0, ())]
    log.clear()
    model.transcribe_windowed(wav, boost=["да"])
    assert log == [("decode_windows", 0, ("boost",))]
    assert model.streaming().boost is None


def test_engine_boost_none_makes_the_resume_call(monkeypatch):
    """Engine.greedy_resume with boost=None calls gam_rnnt_greedy_resume with the arguments it passed before; with tables
    it calls gam_rnnt_greedy_boost with the same arguments plus the tables and S."""
    from gigaam_b200.engine import DecodeBuffers, Engine
    calls = []

    class Stub:
        device = torch.device("cpu")
        head_type = 2
        num_classes = 5

        class lib:
            @staticmethod
            def gam_decode_state_bytes(h):
                return 4128

            @staticmethod
            def gam_decode_resume_workspace_bytes(h, B, T):
                return 64
        handle = None

        class _ws_dec:
            @staticmethod
            def get(key, n, device):
                return torch.zeros(n, dtype=torch.uint8)

        def _call(self, name, *args):
            calls.append((name, len(args)))
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    i32 = dict(dtype=torch.int32)
    enc = torch.zeros((2, 3, 4))
    r = torch.zeros(2, **i32)
    out = DecodeBuffers(torch.zeros((2, 6), **i32), torch.zeros((2, 6), **i32), torch.zeros(2, **i32))
    state = torch.zeros((2, 4128), dtype=torch.uint8)
    Engine.greedy_resume(Stub(), enc, r, r, r, state, out)
    Engine.greedy_resume(Stub(), enc, r, r, r, state, out, boost=None)
    Engine.greedy_resume(Stub(), enc, r, r, r, state, out, boost=(torch.zeros((3, 5), **i32), torch.zeros((3, 5))))
    assert calls == [("gam_rnnt_greedy_resume", 19), ("gam_rnnt_greedy_resume", 19), ("gam_rnnt_greedy_boost", 22)]


def test_exports():
    lib = _lib.load()
    for name in ("gam_rnnt_greedy_boost", "gam_test_rnnt_greedy_boost"):
        assert name in _lib.EXPORTS and hasattr(lib, name)


# ------------------------------------------------------------------------------------------ the float64 replay
def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def replay_boost(W, encproj, L, max_symbols, ids, frames, nxt, bonus, eps=JOINT_TIE, token_logp=None):
    """test_greedy_decisions.replay with the boost graph: the label of a row in state q is within eps of the maximum of
    z + bonus[q] (blank: + 0; non-finite rows: torch's label of z), q follows next on emission (out of range: 0).  With
    token_logp, also checks each emitted token's l against float64 log_softmax(z)[label].  Returns statistics, among them
    `steered`: decisions whose label is not within eps of the unboosted maximum."""
    emb_gates, whhT, wpT, bp, wo, bo = (np.asarray(W[k], dtype=np.float64) for k in ("emb_gates", "whhT", "wpT", "bp", "wo", "bo"))
    V1 = wo.shape[0]
    blank = V1 - 1
    S = nxt.shape[0]
    n = len(ids)
    assert len(frames) == n and all(0 <= k < V1 for k in ids)

    def lstm(label, h, c):
        g = emb_gates[label] + h @ whhT
        i, f, gg, o = np.split(g, 4)
        c2 = _sig(f) * c + _sig(i) * np.tanh(gg)
        return _sig(o) * np.tanh(c2), c2

    st = dict(decisions=0, steered=0, nonfinite=0, worst_l=0.0, rows=0)
    hn, cn = lstm(blank, np.zeros(H), np.zeros(H))
    pg = hn @ wpT + bp
    pos, q, path = 0, 0, 0.0
    with np.errstate(invalid="ignore", over="ignore"):
        for t in range(L):
            e = np.asarray(encproj[t], dtype=np.float64)
            for _ in range(max_symbols):
                z = e + pg
                z = wo @ np.where(z < 0, 0.0, z) + bo
                b = bonus[q].astype(np.float64).copy()
                b[blank] = 0.0
                zb = z + b
                k = ids[pos] if pos < n and frames[pos] == t else blank
                st["decisions"] += 1
                if np.isfinite(z).all():
                    margin = float(zb.max() - zb[k])
                    assert margin <= eps, f"frame {t}: label {k} is {margin:.3g} below the boosted maximum (class {int(zb.argmax())})"
                    st["steered"] += int(z.max() - z[k] > eps)
                    lz = float(z[k] - z.max() - np.log(np.exp(z - z.max()).sum()))
                    path += lz
                    if token_logp is not None and k != blank:
                        err = abs(float(token_logp[pos]) - lz)
                        bound = 2 * JOINT_TIE + 1e-5 * (1 + abs(lz))
                        assert err <= bound, f"frame {t}: token_logp {token_logp[pos]} vs float64 {lz} (bound {bound:.3g})"
                        st["worst_l"] = max(st["worst_l"], err)
                else:
                    want = int(torch.log_softmax(torch.from_numpy(z), -1).argmax())
                    assert k == want, f"frame {t}: non-finite row decoded as {k}, torch gives {want}"
                    st["nonfinite"] += 1
                    path = float("nan")
                st["rows"] += 1
                if k == blank:
                    break
                pos += 1
                qn = int(nxt[q, k])
                q = qn if 0 <= qn < S else 0
                hn, cn = lstm(k, hn, cn)
                pg = hn @ wpT + bp
    assert pos == n, f"trace not used up: {n - pos} of {n} tokens left"
    st["path"] = path
    return st


# ------------------------------------------------------------------------------------------ GPU: the kernel
def run_boost(eng, Wd, V1, encproj, lens, max_symbols, graph, scored=False):
    """gam_test_rnnt_greedy_boost -> ([(ids, frames[, token_logp, path_logp, path_rows])] per utterance, plan dict)."""
    dev = eng.device
    B, T, _ = encproj.shape
    max_out = T * max_symbols
    ids = torch.full((B, max_out), -7, dtype=torch.int32, device=dev)
    frames = torch.full((B, max_out), -7, dtype=torch.int32, device=dev)
    counts = torch.full((B,), -7, dtype=torch.int32, device=dev)
    tl = torch.full((B, max_out), 7.0, device=dev) if scored else None
    pl = torch.full((B,), 7.0, device=dev) if scored else None
    pr = torch.full((B,), -7, dtype=torch.int32, device=dev) if scored else None
    plan = (C.c_int32 * 7)()
    e = torch.from_numpy(np.ascontiguousarray(encproj, dtype=np.float32)).to(dev)
    ln = torch.from_numpy(np.asarray(lens, dtype=np.int32)).to(dev)
    nxt, bonus = (torch.as_tensor(np.ascontiguousarray(a)).to(dev) for a in graph)
    _call(eng, "gam_test_rnnt_greedy_boost", e, ln, *Wd, B, T, V1, max_symbols, max_out, ids, frames, counts, tl, pl, pr, nxt, bonus,
          nxt.shape[0], C.cast(plan, C.c_void_p))
    ids, frames, counts = ids.cpu().numpy(), frames.cpu().numpy(), counts.cpu().numpy()
    hyps = []
    for b in range(B):
        h = (ids[b, :counts[b]].tolist(), frames[b, :counts[b]].tolist())
        if scored:
            h += (tl[b, :counts[b]].cpu().numpy(), float(pl[b]), int(pr[b]))
        hyps.append(h)
    return hyps, dict(zip(("NH", "GLOB", "rows_smem", "cls_per", "nu", "groups", "clusters"), list(plan)))


def _graph(V1, seed, lam=3.0, n=40):
    """A graph of n random unanchored phrases of 1-4 tokens (numpy next, bonus)."""
    rng = np.random.default_rng(seed)
    ph = [rng.integers(0, V1 - 1, size=rng.integers(1, 5)).tolist() for _ in range(n)]
    return tuple(t.numpy() for t in boost_graph(ph, lam, None, V1, V1 - 1))


@pytest.fixture(scope="module")
def boost_geometry(eng, dev, geometry):
    """Per NH, the largest V1 whose class rows all fit in shared memory next to the bonus slices."""
    Vmax = 8192
    Wz = {k: np.zeros_like(v) for k, v in make_weights(2, 0).items()}
    Wz["emb_gates"] = np.zeros((Vmax, 4 * H), np.float32)
    Wz["wo"] = np.zeros((Vmax, H), np.float32)
    Wz["bo"] = np.zeros(Vmax, np.float32)
    Wd = _dev_weights(Wz, dev)
    out = dict(geometry)
    for (nh, B), scored in ((n, sc) for n in ((1, 1), (2, geometry["b_switch"] + 1)) for sc in (False, True)):
        def plan(V1):
            g = (np.zeros((1, V1), np.int32), np.zeros((1, V1), np.float32))
            return run_boost(eng, Wd, V1, np.zeros((B, 1, H), np.float32), np.zeros(B, np.int32), 1, g, scored)[1]
        lo, hi = 2, Vmax
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if plan(mid)["GLOB"]:
                hi = mid
            else:
                lo = mid
        assert plan(lo)["NH"] == nh
        out[f"boost_last_smem_{nh}_{int(scored)}"] = lo
        # the bonus slices take shared memory: the boundary moves down, never up
        assert lo <= geometry[f"last_smem_{nh}"], (lo, geometry)
    print("boost geometry (NH, scored):", {k: v for k, v in out.items() if k.startswith("boost")}, "unboosted, unscored:",
          geometry["last_smem_1"], geometry["last_smem_2"])
    return out


@pytest.mark.gpu
def test_every_boosted_decision_against_float64(eng, dev, boost_geometry):
    g = boost_geometry
    bs = g["b_switch"]
    b_ragged = 8 * g["clusters"] + 3
    vs = sorted({2, 3, 34, 257, 1025, 4097} | {g[k] + d for k in g if k.startswith("boost_last_smem") for d in (0, 1)})
    cases = []
    for i, V1 in enumerate(vs):
        cases.append((V1, [1, bs - 1, bs][i % 3], (1, 2, 10)[i % 3], 1))
        cases.append((V1, [bs + 1, b_ragged][i % 2], (10, 1, 2)[i % 3], 2))
    steered, decisions, paths = 0, 0, set()
    for ci, (V1, B, ms, nh) in enumerate(cases):
        W = make_weights(V1, V1)
        Wd = _dev_weights(W, dev)
        graph = _graph(V1, ci)
        enc, lens = make_encproj(B, T_SWEEP, 3000 + ci), make_lens(B, T_SWEEP, 3000 + ci)
        scored = (ci // 2) % 2 == 1
        hyps, plan = run_boost(eng, Wd, V1, enc, lens, ms, graph, scored)
        assert plan["NH"] == nh and plan["GLOB"] == int(V1 > g[f"boost_last_smem_{nh}_{int(scored)}"]), (V1, B, plan)
        paths.add((plan["NH"], plan["GLOB"]))
        for b in range(B):
            try:
                st = replay_boost(W, enc[b], int(lens[b]), ms, hyps[b][0], hyps[b][1], *graph,
                                  token_logp=hyps[b][2] if scored else None)
            except AssertionError as e:
                raise AssertionError(f"V1={V1} B={B} max_symbols={ms} plan={plan} utterance {b}: {e}") from None
            steered += st["steered"]
            decisions += st["decisions"]
            if scored:
                assert hyps[b][4] == st["rows"], (V1, b)
                bound = st["rows"] * (2 * JOINT_TIE + 1e-5) + 1e-5 * abs(st["path"])
                assert abs(hyps[b][3] - st["path"]) <= bound, (V1, b, hyps[b][3], st["path"])
        alone, _ = run_boost(eng, Wd, V1, enc[B - 1:B], lens[B - 1:B], ms, graph, scored)
        assert [list(map(lambda x: x if not isinstance(x, np.ndarray) else x.tolist(), h)) for h in alone] == \
               [list(map(lambda x: x if not isinstance(x, np.ndarray) else x.tolist(), hyps[B - 1]))]
    print(f"boosted sweep: {decisions} decisions, {steered} steered away from the unboosted maximum; paths {sorted(paths)}")
    assert steered > 0, "no decision differs from the unboosted argmax: the sweep is vacuous"
    assert {(1, 0), (1, 1), (2, 0), (2, 1)} <= paths


@pytest.mark.gpu
@pytest.mark.parametrize("nh", [1, 2])
def test_ties_keep_the_lower_index_and_a_bonus_breaks_them(eng, dev, geometry, nh):
    B = 3 if nh == 1 else geometry["b_switch"] + 2
    V1 = geometry[f"l2_gt32_{nh}"]
    lo, hi = 4, 9 * (-(-V1 // 16)) + 1
    W = _tie_weights(V1, [(lo, hi)], 60)
    Wd = _dev_weights(W, dev)
    enc, lens = make_encproj(B, T_SWEEP, 61), make_lens(B, T_SWEEP, 61)
    nxt = np.zeros((1, V1), np.int32)
    both = np.zeros((1, V1), np.float32)
    both[0, lo] = both[0, hi] = 0.5
    hyps, _ = run_boost(eng, Wd, V1, enc, lens, 10, (nxt, both))
    assert sum(h[0].count(lo) for h in hyps) > 0 and all(hi not in h[0] for h in hyps)
    only_hi = np.zeros((1, V1), np.float32)
    only_hi[0, hi] = 2.0 ** -20
    hyps, _ = run_boost(eng, Wd, V1, enc, lens, 10, (nxt, only_hi))
    assert sum(h[0].count(hi) for h in hyps) > 0 and all(lo not in h[0] for h in hyps)
    for b, h in enumerate(hyps):
        replay_boost(W, enc[b], int(lens[b]), 10, *h, nxt, only_hi)


@pytest.mark.gpu
@pytest.mark.parametrize("V1,nh", [(34, 1), (1025, 2)])
def test_nonfinite_rows_decode_as_unboosted(eng, dev, geometry, V1, nh):
    W = make_weights(V1, 7)
    cls = np.arange(V1)
    W["wo"][:, 1] = np.where(cls % 2 == 0, 0.3, -0.3)
    W["wo"][:, 2] = np.where(cls % 3 == 0, -0.2, 0.2)
    W["wo"][:, 3] = -np.abs(W["wo"][:, 3]) - 1e-3
    W["wo"][:, 4] = np.abs(W["wo"][:, 4]) + 1e-3
    B = 5 if nh == 1 else geometry["b_switch"] + 3
    bad = make_encproj(B, T_SWEEP, 90 + V1)
    lens = np.full(B, T_SWEEP, np.int32)
    bad[0, 2, :] = np.nan
    bad[1, 3, 1] = bad[1, 3, 2] = np.inf
    bad[2, 1, 3] = np.inf
    bad[3, 5, 4] = np.inf
    graph = _graph(V1, 5, lam=5.0)
    hyps, plan = run_boost(eng, _dev_weights(W, dev), V1, bad, lens, 10, graph, scored=True)
    assert plan["NH"] == nh
    nonfinite = sum(replay_boost(W, bad[b], T_SWEEP, 10, hyps[b][0], hyps[b][1], *graph)["nonfinite"] for b in range(B))
    assert nonfinite >= 4
    assert [k for k, f in zip(hyps[0][0], hyps[0][1]) if f == 2] == [0] * 10
    assert all(np.isnan(hyps[b][3]) for b in range(4))


# ------------------------------------------------------------------------------------------ GPU: the engine call
def _dev():
    return torch.device("cuda", 0)


_MODELS = {}


def _model(name):
    if name not in _MODELS:
        ck = synthetic.synthetic_checkpoint(name, seed=0, n_layers=1)
        _MODELS[name] = gigaam.load_model(name, fp16_encoder=False, device=_dev(), checkpoint=ck)
    return _MODELS[name]


def _engine_run(eng, enc, lo, hi, state, out_width, T, scores, boost, fb=None):
    B = enc.shape[0]
    i32 = dict(dtype=torch.int32, device=eng.device)
    out = eng.decode_buffers(B, out_width, T, scores=scores)
    fb = torch.zeros(B, **i32) if fb is None else fb
    eng.greedy_resume(enc, torch.as_tensor(lo, **i32), torch.as_tensor(hi, **i32), fb, state, out, scores, boost)
    return out


def _bits(out):
    """The written part of DecodeBuffers as integer tensors: ids, frames and token_logp up to each row's count, the rest whole."""
    n = out.counts.tolist()
    got = []
    for i, t in enumerate(out):
        if t is None:
            continue
        t = t.view(torch.int32) if t.dtype == torch.float32 else (t.view(torch.int64) if t.dtype == torch.float64 else t)
        got.append(torch.cat([t[b, :n[b]] for b in range(len(n))]) if i in (0, 1, 3) else t)
    return got


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(_bits(a), _bits(b)))


def _model_graph(model, seed, lam=2.0, n=30):
    eng = model._get_engine()
    V = eng.num_classes - 1
    rng = np.random.default_rng(seed)
    ph = [rng.integers(0, V, size=rng.integers(1, 5)).tolist() for _ in range(n)]
    return tuple(t.to(eng.device) for t in boost_graph(ph, lam, None, V + 1, V))


@pytest.mark.gpu
@pytest.mark.parametrize("scores", [False, True])
def test_zero_bonuses_are_the_resume_call_bit_for_bit(scores):
    model = _model("v2_rnnt")
    eng = model._get_engine()
    B, T = 6, 40
    enc = torch.randn(B, T, eng.d_model, device=eng.device, generator=torch.Generator(eng.device).manual_seed(3))
    V1 = eng.num_classes
    g = torch.Generator().manual_seed(4)
    nxt = torch.randint(-3, 12, (9, V1), generator=g, dtype=torch.int32).to(eng.device)   # arbitrary, some out of range
    zero = (nxt, torch.zeros((9, V1), device=eng.device))
    lens = [T, 0, 1, 17, T, 33]
    st_a, st_b = eng.decode_state(B), eng.decode_state(B)
    assert st_a.shape[1] == 4128
    for lo, hi in (([0] * B, [min(10, x) for x in lens]), ([min(10, x) for x in lens], lens)):
        a = _engine_run(eng, enc, lo, hi, st_a, eng.hyp_width(T), T, scores, None)
        b = _engine_run(eng, enc, lo, hi, st_b, eng.hyp_width(T), T, scores, zero)
        assert _same(a, b)
    diff = (st_a != st_b).any(0).nonzero().reshape(-1).tolist()
    assert set(diff) <= set(range(32, 36)), diff          # only the q slot (the first int of part[])


@pytest.mark.gpu
def test_chunks_batches_and_graph_replay_give_the_bits_of_one_call():
    model = _model("v2_rnnt")
    eng = model._get_engine()
    T = 60
    V1 = eng.num_classes
    boost = _model_graph(model, 1)
    enc = torch.randn(61, T, eng.d_model, device=eng.device, generator=torch.Generator(eng.device).manual_seed(8))
    width = eng.hyp_width(T)
    one = _engine_run(eng, enc[:1], [0], [T], eng.decode_state(1), width, T, True, boost)
    plain = _engine_run(eng, enc[:1], [0], [T], eng.decode_state(1), width, T, True, None)
    assert not torch.equal(one.ids[0, :int(one.counts[0])], plain.ids[0, :int(plain.counts[0])]), "the graph changes nothing"
    rng = random.Random(2)
    for cuts in ([1] * T, [2] * (T // 2), [7] * 8 + [4], [0, 5, 0, 55], None):
        if cuts is None:
            cuts = []
            while sum(cuts) < T:
                cuts.append(min(rng.randint(0, 9), T - sum(cuts)))
        state, out = eng.decode_state(1), eng.decode_buffers(1, width, T, scores=True)
        pos = 0
        for c in cuts:
            i32 = dict(dtype=torch.int32, device=eng.device)
            eng.greedy_resume(enc[:1], torch.tensor([pos], **i32), torch.tensor([pos + c], **i32), torch.zeros(1, **i32), state, out,
                              True, boost)
            pos += c
        assert _same(out, one), cuts
    # an out-of-range next entry sends the stream to state 0, as a 0 entry does
    nxt, bonus = boost
    wild = nxt.clone()
    wild[wild == 0] = -5
    wild[:, :3] = torch.where(wild[:, :3] == -5, torch.tensor(nxt.shape[0] + 3, dtype=torch.int32, device=eng.device), wild[:, :3])
    assert _same(_engine_run(eng, enc[:1], [0], [T], eng.decode_state(1), width, T, True, (wild, bonus)), one)
    # batches of 8, 40 and 61: row 0 keeps its bits
    for B in (8, 40, 61):
        out = _engine_run(eng, enc[:B], [0] * B, [T] * B, eng.decode_state(B), width, T, True, boost)
        assert _same(type(out)(*[None if t is None else t[:1] for t in out]), one), B
    # CUDA-graph capture and replay
    state = eng.decode_state(1)
    fresh = state.clone()
    out = eng.decode_buffers(1, width, T, scores=True)
    i32 = dict(dtype=torch.int32, device=eng.device)
    lo, hi, fb = torch.zeros(1, **i32), torch.tensor([T], **i32), torch.zeros(1, **i32)
    eng.greedy_resume(enc[:1], lo, hi, fb, state, out, True, boost)      # warm the workspace cache
    s = torch.cuda.Stream(eng.device)
    s.wait_stream(torch.cuda.current_stream(eng.device))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        eng.greedy_resume(enc[:1], lo, hi, fb, state, out, True, boost)
    torch.cuda.current_stream(eng.device).wait_stream(s)
    for t in out[2:]:
        if t is not None:
            t.zero_()
    state.copy_(fresh)
    graph.replay()
    torch.cuda.synchronize()
    assert _same(out, one)


@pytest.mark.gpu
def test_planted_near_miss_comes_out_as_the_phrase(eng, dev):
    """Decision 0 of an utterance: the greedy token k beats the runner-up r by m; the phrase [r] at weight m + 0.01 turns it
    into r, at weight m - 0.01 it stays k."""
    V1, T = 34, 6
    W = make_weights(V1, 11)
    Wd = _dev_weights(W, dev)
    enc = make_encproj(1, T, 12)
    enc[0, 0, 0] = -30.0                                              # a burst frame: tokens win
    hyps, _ = run_boost(eng, Wd, V1, enc, [T], 2, (np.zeros((1, V1), np.int32), np.zeros((1, V1), np.float32)))
    emb_gates, whhT, wpT, bp, wo, bo = (np.asarray(W[k], np.float64) for k in ("emb_gates", "whhT", "wpT", "bp", "wo", "bo"))
    g = emb_gates[V1 - 1]
    i, f, gg, o = np.split(g, 4)
    c = _sig(i) * np.tanh(gg)
    h = _sig(o) * np.tanh(c)
    z = wo @ np.maximum(enc[0, 0].astype(np.float64) + h @ wpT + bp, 0) + bo
    k = int(np.argmax(z))
    assert hyps[0][0][0] == k
    zs = z.copy()
    zs[k] = -np.inf
    r = int(np.argmax(zs[:V1 - 1]))
    m = float(z[k] - z[r])
    for lam, want in ((m + 0.01, r), (max(m - 0.01, 1e-3), k)):
        graph = tuple(t.numpy() for t in boost_graph([[r]], lam, None, V1, V1 - 1))
        got, _ = run_boost(eng, Wd, V1, enc, [T], 2, graph)
        assert got[0][0][0] == want, (lam, m, k, r, got[0][0][:3])


# ------------------------------------------------------------------------------------------ GPU: the public calls
def _phrases_from(model, text, n=3):
    tok = model.decoding.tokenizer
    # the first tokens of a greedy word with the last of them changed
    out = []
    for w in text.split():
        ids = tok.encode(w)[:6]
        if len(ids) >= 2:
            out.append(ids[:-1] + [(ids[-1] + 1) % len(tok)])
    out = [p for p in out if tok.id_to_str(p[0]) != " " and tok.id_to_str(p[-1]) != " "][:n]
    return out or [[1, 2]]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_rnnt", "v3_e2e_rnnt"])
def test_public_calls_equal_the_engine_call(name):
    from gigaam_b200.decoding import _as_btd
    model = _model(name)
    eng = model._get_engine()
    wav, _ = synthetic.synthetic_audio(1, 6.0, seed=31)
    w = wav[0]
    with torch.inference_mode():
        plain = model.transcribe(w)
        phrases = _phrases_from(model, plain.text)
        for weight in (0.5, 4.0):
            got = model.transcribe(w, boost=phrases, boost_weight=weight, confidence=True, word_timestamps=True)
            wv, length = model.prepare_wav(w)
            encoded, enc_len = model.forward(wv, length)
            enc = _as_btd(encoded.to(dtype=torch.float32))
            T = enc.shape[1]
            tables = tuple(t.to(eng.device) for t in model._boost_tables(phrases, weight, "transcribe"))
            out = _engine_run(eng, enc, [0], enc_len.tolist(), eng.decode_state(1), eng.hyp_width(T), T, True, tables)
            n = int(out.counts[0])
            assert got.text == model.decoding.tokenizer.decode(out.ids[0, :n].tolist())
            one = model.transcribe_windowed(w, boost=phrases, boost_weight=weight, window=30.0)
            assert " ".join(s.text for s in one.segments if s.text) == got.text
        # many windows: one boosted call over the stitched encoder output
        long_wav, _ = synthetic.synthetic_audio(1, 70.0, seed=32)
        got = model.transcribe_windowed(long_wav[0], boost=phrases, boost_weight=4.0, window=8.0, overlap=4.0, confidence=True)
        from gigaam_b200.longform import decode_windows, plan_windows
        windows, T = plan_windows(long_wav[0].numel(), 8.0, 4.0, model._encoded_length, 5000)
        host = long_wav[0].to(model._dtype)
        tables = tuple(t.to(eng.device) for t in model._boost_tables(phrases, 4.0, "x"))
        out = decode_windows(model, host, windows, T, 16, True, boost=tables)
        n = int(out.counts[0])
        assert "".join(s.text + " " for s in got.segments).split() == model.decoding.tokenizer.decode(out.ids[0, :n].tolist()).split()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_rnnt", "v3_e2e_rnnt"])
def test_closed_boosted_streams_equal_transcribe_windowed(name):
    from test_streaming import _drive, _recordings
    model = _model(name)
    wavs = _recordings(40 + len(name), n=8)
    phrases = _phrases_from(model, model.transcribe_windowed(wavs[-1], window=8.0, overlap=4.0).text)
    rng = random.Random(41)
    with torch.inference_mode():
        srv = model.streaming(window=8.0, overlap=4.0, batch_size=5, confidence=True, boost=phrases, boost_weight=3.0)
        results, _ = _drive(srv, wavs, rng)
        for i, w in enumerate(wavs):
            want = model.transcribe_windowed(w, word_timestamps=True, confidence=True, window=8.0, overlap=4.0, pause=0.3,
                                              max_segment=6.0, boost=phrases, boost_weight=3.0)
            assert repr(results[i].transcript) == repr(want), i
