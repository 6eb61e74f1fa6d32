"""Every greedy decision of the RNN-T cluster kernel (csrc/rnnt_cluster.cu) and of the CTC argmax (csrc/ctc.cu) against
float64, and the decision contract on non-finite joint rows.

The contract (DESIGN §4): the label of a row is torch's log_softmax(row).argmax(-1) -- the first maximal index of a row
whose maximum is finite, and 0 when any logit is NaN or +inf or no logit exceeds -inf (log_softmax makes such a row
all-NaN).

CPU: a float64 replay checker that walks the reference's greedy rule (gigaam/decoding.py:184-205) along a kernel trace and
accepts it only if every chosen label is within JOINT_TIE of its row's maximum (non-finite rows: exactly torch's label)
and the trace is used up exactly; negative controls show it rejects the oracle's own traces replayed on faulty weights;
and the oracle's rnnt_greedy equals the reference's decoder on rows of every non-finite kind.

GPU: gam_test_rnnt_greedy over vocabularies on both sides of every shared-memory / L2 boundary, both group widths,
ragged group counts, lengths 0, 1 and T and max_symbols 1, 2 and 10, in ascending and then descending V1 in one process;
exact ties across class-ownership boundaries; non-finite rows; the CTC argmax through an engine with custom head weights;
and non-finite encoder frames through a whole v2_rnnt model."""
import ctypes as C
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, synthetic
from gigaam_b200.engine import Engine
from oracle import gigaam_oracle as orc
from oracle import ref_loader

H = 320
JOINT_TIE = 1e-4        # a chosen label's float64 logit may be this far below its row's maximum (fp32 joint and state)
NEAR_MAX = 0.01         # non-vacuity: at most this fraction of decisions may have a top-2 gap inside the JOINT_TIE band
CTC_TIE = 1e-4          # CTC: the same band for the 768-long fp32 dot products
T_SWEEP = 9
INF, NAN = float("inf"), float("nan")


# ------------------------------------------------------------------------------------------ weights and inputs
def make_weights(V1, seed):
    """Joint and prediction weights in the kernel's layout (float32, numpy).  Unit 0 of the joint's hidden layer is the
    blank switch: blank's W_o row has 1 there and every token row 0, and blank's bias is -5, so that an encoder frame
    with encproj[0] = +30 is a blank frame, -30 a burst frame (relu zeroes the switch; tokens win every decision) and
    4..16 a frame where blank and tokens compete."""
    rng = np.random.default_rng(seed)
    blank = V1 - 1
    emb = rng.standard_normal((V1, H)) * 0.5
    emb[blank] = 0.0                                   # predict(None): the zero embedding
    w_ih = rng.standard_normal((4 * H, H)) * 0.1
    w_hh = rng.standard_normal((4 * H, H)) * 0.1
    bias = rng.standard_normal(4 * H) * 0.1
    wo = rng.standard_normal((V1, H)) * 0.1
    wo[:, 0] = 0.0
    wo[blank, 0] = 1.0
    bo = rng.standard_normal(V1) * 0.1
    bo[blank] = -5.0
    wpT = rng.standard_normal((H, H)) * 0.3
    wpT[:, 0] *= 4                                     # the prediction state moves the blank switch: bursts end early
    W = dict(emb_gates=emb @ w_ih.T + bias, whhT=w_hh.T, wpT=wpT,
             bp=rng.standard_normal(H) * 0.1, wo=wo, bo=bo)
    return {k: np.ascontiguousarray(v, dtype=np.float32) for k, v in W.items()}


def make_encproj(B, T, seed):
    """[B, T, H] float32 with a frame kind per (b, t) on unit 0: blank (+30), burst (-30) or contested (4..16)."""
    rng = np.random.default_rng(seed)
    e = rng.standard_normal((B, T, H))
    kind = rng.choice(3, size=(B, T), p=[0.3, 0.3, 0.4])
    e[..., 0] = np.where(kind == 0, 30.0, np.where(kind == 1, -30.0, rng.uniform(4.0, 16.0, size=(B, T))))
    return e.astype(np.float32)


def make_lens(B, T, seed):
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, T + 1, size=B)
    for i, v in enumerate((T, 0, 1, T)):
        if i < B:
            lens[i] = v
    return lens.astype(np.int32)


# ------------------------------------------------------------------------------------------ the float64 replay
def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def replay(W, encproj, L, max_symbols, ids, frames, eps=JOINT_TIE):
    """Walk the reference's greedy rule for one utterance in float64, forced along the trace (ids, frames).  Raises
    AssertionError on the first decision the trace gets wrong; returns statistics of the walk."""
    emb_gates, whhT, wpT, bp, wo, bo = (np.asarray(W[k], dtype=np.float64)
                                        for k in ("emb_gates", "whhT", "wpT", "bp", "wo", "bo"))
    V1 = wo.shape[0]
    blank = V1 - 1
    ids, frames = [int(x) for x in ids], [int(x) for x in frames]
    n = len(ids)
    assert len(frames) == n
    assert all(0 <= k < V1 for k in ids), f"label outside [0, {V1}): {ids}"
    assert all(a <= b for a, b in zip(frames, frames[1:])), f"frames decrease: {frames}"
    assert all(0 <= f < L for f in frames), f"frame outside [0, {L}): {frames}"
    per_frame = np.bincount(np.asarray(frames, dtype=np.int64), minlength=L) if L else np.zeros(0, np.int64)
    assert (per_frame <= max_symbols).all(), f"more than {max_symbols} tokens on a frame"

    def lstm(label, h, c):
        g = emb_gates[label] + h @ whhT
        i, f, gg, o = np.split(g, 4)
        c2 = _sig(f) * c + _sig(i) * np.tanh(gg)
        return _sig(o) * np.tanh(c2), c2

    st = dict(decisions=0, near=0, worst=0.0, nonfinite=0, blank_frames=0, singles=0, bursts=0)
    hn, cn = lstm(blank, np.zeros(H), np.zeros(H))
    pg = hn @ wpT + bp
    pos = 0
    with np.errstate(invalid="ignore", over="ignore"):
        for t in range(L):
            e = np.asarray(encproj[t], dtype=np.float64)
            for _ in range(max_symbols):
                z = e + pg
                z = wo @ np.where(z < 0, 0.0, z) + bo          # relu keeps NaN
                k = ids[pos] if pos < n and frames[pos] == t else blank
                st["decisions"] += 1
                if np.isfinite(z).all():
                    margin = float(z.max() - z[k])
                    assert margin <= eps, f"frame {t}, decision {st['decisions']}: label {k} is {margin:.3g} below the maximum " \
                                          f"{float(z.max()):.6g} (class {int(z.argmax())})"
                    top2 = np.partition(z, -2)[-2:]
                    st["near"] += int(top2[1] - top2[0] < eps)
                    st["worst"] = max(st["worst"], margin)
                else:
                    want = int(torch.log_softmax(torch.from_numpy(z), -1).argmax())
                    assert k == want, f"frame {t}: non-finite row decoded as {k}, torch gives {want}"
                    st["nonfinite"] += 1
                if k == blank:
                    break
                pos += 1
                hn, cn = lstm(k, hn, cn)
                pg = hn @ wpT + bp
    assert pos == n, f"trace not used up: {n - pos} of {n} tokens left after the last frame"
    st["blank_frames"] = int((per_frame == 0).sum())
    st["singles"] = int((per_frame == 1).sum())
    st["bursts"] = int((per_frame == max_symbols).sum())
    return st


def _merge(total, st):
    for k, v in st.items():
        total[k] = max(total.get(k, 0.0), v) if k == "worst" else total.get(k, 0) + v


def _assert_non_vacuous(total, what):
    print(f"{what}: {total['decisions']} decisions, worst margin {total['worst']:.3g}, {total['near']} inside the band")
    assert total["decisions"] > 0 and total["near"] < NEAR_MAX * total["decisions"], (what, total)
    assert total["blank_frames"] > 0 and total["singles"] > 0 and total["bursts"] > 0, (what, total)


# ------------------------------------------------------------------------------------------ CPU: the replay on oracle traces
def _oracle_setup(V1=34, B=8, T=16, seed=5):
    """A v2_rnnt state_dict whose joint follows make_weights' design, its kernel-layout weights (float64 packing of
    engine._pack_rnnt, rounded to fp32), an encoder output and its projection."""
    ck = synthetic.synthetic_checkpoint("v2_rnnt", seed=seed, n_layers=1)
    sd = {k: v.clone() for k, v in ck["state_dict"].items()}
    W = make_weights(V1, seed)
    rng = np.random.default_rng(seed + 1)
    w_ih = rng.standard_normal((4 * H, H)) * 0.1
    emb = rng.standard_normal((V1, H)) * 0.5
    emb[V1 - 1] = 0
    b_ih = rng.standard_normal(4 * H) * 0.05
    b_hh = rng.standard_normal(4 * H) * 0.05
    t32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))   # noqa: E731
    sd["head.decoder.embed.weight"] = t32(emb)
    sd["head.decoder.lstm.weight_ih_l0"], sd["head.decoder.lstm.bias_ih_l0"] = t32(w_ih), t32(b_ih)
    sd["head.decoder.lstm.weight_hh_l0"], sd["head.decoder.lstm.bias_hh_l0"] = t32(W["whhT"].T), t32(b_hh)
    sd["head.joint.pred.weight"], sd["head.joint.pred.bias"] = t32(W["wpT"].T), t32(W["bp"])
    sd["head.joint.joint_net.1.weight"], sd["head.joint.joint_net.1.bias"] = t32(W["wo"]), t32(W["bo"])
    # joint.enc: unit-variance projections, and unit 0 reads feature 0 alone, so that the frame kind of make_encproj
    # can be set on the encoder side
    we = t32(rng.standard_normal((H, 768)) / np.sqrt(768))
    we[0] = 0
    we[:, 0] = 0
    we[0, 0] = 1.0
    sd["head.joint.enc.weight"], sd["head.joint.enc.bias"] = we, torch.zeros(H)
    W = dict(W)
    W["emb_gates"] = (emb.astype(np.float32).astype(np.float64) @ w_ih.astype(np.float32).astype(np.float64).T
                      + b_ih.astype(np.float32).astype(np.float64) + b_hh.astype(np.float32).astype(np.float64))
    enc = torch.randn(B, 768, T, generator=torch.Generator().manual_seed(seed))
    kind = make_encproj(B, T, seed)[..., 0]
    enc[:, 0, :] = torch.from_numpy(kind)
    encproj = (F.linear(enc.transpose(1, 2).double(), sd["head.joint.enc.weight"].double(),
                        sd["head.joint.enc.bias"].double())).numpy()
    lens = make_lens(B, T, seed)
    return sd, W, enc, encproj, lens


def _faulty(W, fault):
    W = {k: np.array(v, dtype=np.float64) for k, v in W.items()}
    if fault == "i_f_swapped":
        for k in ("emb_gates", "whhT"):
            a = W[k]
            a[..., :H], a[..., H:2 * H] = a[..., H:2 * H].copy(), a[..., :H].copy()
    elif fault == "wo_shifted":
        W["wo"], W["bo"] = np.roll(W["wo"], 1, axis=0), np.roll(W["bo"], 1)
    elif fault == "last_row_dropped":
        W["wo"], W["bo"] = W["wo"][:-1], W["bo"][:-1]
        W["emb_gates"] = W["emb_gates"][:-1]
    return W


@pytest.mark.parametrize("max_symbols", [1, 2, 10])
def test_replay_accepts_oracle_traces_and_rejects_faulty_weights(max_symbols):
    sd, W, enc, encproj, lens = _oracle_setup(seed=5 + max_symbols)
    hyps = orc.rnnt_greedy(enc, torch.from_numpy(lens), sd, max_symbols=max_symbols)
    total = {}
    for b, (ids, frames) in enumerate(hyps):
        _merge(total, replay(W, encproj[b], int(lens[b]), max_symbols, ids, frames))
    _assert_non_vacuous(total, f"oracle, max_symbols={max_symbols}")
    faults = [("i_f_swapped", max_symbols), ("wo_shifted", max_symbols), ("last_row_dropped", max_symbols),
              ("none", max_symbols + 1)] + ([("none", max_symbols - 1)] if max_symbols > 1 else [])
    for fault, ms in faults:
        Wf = _faulty(W, fault)
        rejected = 0
        for b, (ids, frames) in enumerate(hyps):
            try:
                replay(Wf, encproj[b], int(lens[b]), ms, ids, frames)
            except AssertionError:
                rejected += 1
        assert rejected > 0, f"the replay accepts every trace with fault {fault}, max_symbols {ms}"


# ------------------------------------------------------------------------------------------ CPU: oracle == reference
def _imported_reference():
    before, path = set(sys.modules), list(sys.path)
    try:
        return ref_loader.import_reference()
    finally:
        for k in set(sys.modules) - before:
            if k.split(".")[0] in ("gigaam", "hydra", "omegaconf", "soundfile"):
                del sys.modules[k]
        sys.path[:] = path


def _nonfinite_setup():
    """A v2_rnnt head and an encoder output with one joint row of each non-finite kind: a NaN frame (utterance 0), +inf
    on a feature that drives unit 1 whose W_o column has both signs and zeros (partial NaN, utterance 1), unit 2 whose
    column is negative below class 5 and positive from it (+inf from class 5 on, utterance 2), and unit 3 whose column is
    negative (all -inf, utterance 3)."""
    sd, W, enc, encproj, lens = _oracle_setup(seed=21)
    V1 = W["wo"].shape[0]
    we, wo = sd["head.joint.enc.weight"], sd["head.joint.joint_net.1.weight"]
    for unit, feat in ((1, 1), (2, 2), (3, 3)):
        we[:, feat] = -we[:, feat].abs() - 1e-3
        we[unit, feat] = 0.5
    col1 = torch.where(torch.arange(V1) % 2 == 0, 0.3, -0.3)
    col1[7] = 0.0
    wo[:, 1] = col1
    wo[:, 2] = torch.where(torch.arange(V1) < 5, -0.3, 0.3)
    wo[:, 3] = -0.3
    enc = enc.clone()
    enc[0, :, 2] = NAN
    enc[1, 1, 3], enc[2, 2, 4], enc[3, 3, 1] = INF, INF, INF
    lens = np.array([6, 7, 8, 9, 10, 10, 12, 16], dtype=np.int32)
    return sd, enc, lens


def test_oracle_equals_reference_on_nonfinite_rows():
    if ref_loader.reference_root() is None:
        pytest.skip("the reference is neither in its source tree nor compiled into oracle/_ref")
    _, _, rd, ref_decoding = _imported_reference()
    sd, enc, lens = _nonfinite_setup()
    ck = synthetic.synthetic_checkpoint("v2_rnnt", n_layers=1)
    head = ck["cfg"]["head"]
    ref = rd.RNNTHead(head["decoder"], head["joint"])
    ref.load_state_dict({k[len("head."):]: v for k, v in sd.items() if k.startswith("head.")}, strict=True)
    ref.eval()
    # the rows really are of the four kinds
    x = enc.transpose(1, 2)
    with torch.no_grad():
        g, _ = ref.decoder.predict(None, None, batch_size=1)
        rows = [ref.joint.joint(x[b:b + 1, t:t + 1], g)[0, 0, 0] for b, t in ((0, 2), (1, 3), (2, 4), (3, 1))]
        raw = [F.linear(F.relu(F.linear(x[b, t], sd["head.joint.enc.weight"], sd["head.joint.enc.bias"]) + ref.joint.pred(g[0, 0])),
                        sd["head.joint.joint_net.1.weight"], sd["head.joint.joint_net.1.bias"])
               for b, t in ((0, 2), (1, 3), (2, 4), (3, 1))]
    assert bool(raw[0].isnan().all())
    assert bool(raw[1].isnan().any()) and not bool(raw[1].isnan().all())
    assert not bool(raw[2].isnan().any()) and bool(raw[2].isposinf().any()) and int(raw[2].isposinf().int().argmax()) == 5
    assert bool(raw[3].isneginf().all())
    assert [int(r.argmax()) for r in rows] == [0, 0, 0, 0]     # all four rows are all-NaN after log_softmax
    assert all(bool(r.isnan().all()) for r in rows)
    dec = ref_decoding.RNNTGreedyDecoding(ck["cfg"]["decoding"]["vocabulary"], None, 10)
    with torch.no_grad():
        theirs = dec.decode(ref, enc, torch.from_numpy(lens))
    ours = orc.rnnt_greedy(enc, torch.from_numpy(lens), sd, max_symbols=10)
    for b, (o, r) in enumerate(zip(ours, theirs)):
        assert (o[0], o[1]) == (r[1], r[2]), b


# ------------------------------------------------------------------------------------------ GPU plumbing
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (there is no CPU fallback to test instead)"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def eng(dev):
    ck = synthetic.synthetic_checkpoint("v2_rnnt", seed=0, n_layers=1)
    return Engine(ck["cfg"], ck["state_dict"], dev)


def _call(eng, fn, *args):
    ptrs = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    rc = getattr(eng.lib, fn)(eng.handle, *ptrs, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    _lib.check(eng.lib, eng.handle, rc, fn)


_KEYS = ("emb_gates", "whhT", "wpT", "bp", "wo", "bo")


def _dev_weights(W, dev):
    return [torch.from_numpy(np.ascontiguousarray(W[k], dtype=np.float32)).to(dev) for k in _KEYS]


def run_greedy(eng, Wd, V1, encproj, lens, max_symbols):
    """gam_test_rnnt_greedy -> ([(ids, frames)] per utterance, plan dict)."""
    dev = eng.device
    B, T, _ = encproj.shape
    max_out = T * max_symbols
    ids = torch.full((B, max_out), -7, dtype=torch.int32, device=dev)
    frames = torch.full((B, max_out), -7, dtype=torch.int32, device=dev)
    counts = torch.full((B,), -7, dtype=torch.int32, device=dev)
    plan = (C.c_int32 * 7)()
    e = torch.from_numpy(np.ascontiguousarray(encproj, dtype=np.float32)).to(dev)
    ln = torch.from_numpy(np.asarray(lens, dtype=np.int32)).to(dev)
    _call(eng, "gam_test_rnnt_greedy", e, ln, *Wd, B, T, V1, max_symbols, max_out, ids, frames, counts, C.cast(plan, C.c_void_p))
    ids, frames, counts = ids.cpu().numpy(), frames.cpu().numpy(), counts.cpu().numpy()
    assert ((counts >= 0) & (counts <= max_out)).all(), counts
    hyps = [(ids[b, :counts[b]].tolist(), frames[b, :counts[b]].tolist()) for b in range(B)]
    return hyps, dict(zip(("NH", "GLOB", "rows_smem", "cls_per", "nu", "groups", "clusters"), list(plan)))


def _l2_rows(plan):
    return plan["cls_per"] - plan["rows_smem"]


@pytest.fixture(scope="module")
def geometry(eng, dev):
    """Probed on the device with all lengths 0: the NH = 1 / 2 batch switch, resident clusters, and per NH the largest
    V1 whose class rows all fit in shared memory."""
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    b_switch = 4 * max(1, sms // 16 - 2)
    Vmax = 8192
    Wz = {k: np.zeros_like(v) for k, v in make_weights(2, 0).items()}
    Wz["emb_gates"] = np.zeros((Vmax, 4 * H), np.float32)
    Wz["wo"] = np.zeros((Vmax, H), np.float32)
    Wz["bo"] = np.zeros(Vmax, np.float32)
    Wd = _dev_weights(Wz, dev)

    def plan(V1, B):
        return run_greedy(eng, Wd, V1, np.zeros((B, 1, H), np.float32), np.zeros(B, np.int32), 1)[1]

    out = dict(b_switch=b_switch, clusters=plan(2, 400)["clusters"])
    for nh, B in ((1, 1), (2, b_switch + 1)):
        assert plan(2, B)["NH"] == nh and plan(2, B)["GLOB"] == 0 and plan(Vmax, B)["GLOB"] == 1
        lo, hi = 2, Vmax            # GLOB(lo) == 0, GLOB(hi) == 1
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if plan(mid, B)["GLOB"]:
                hi = mid
            else:
                lo = mid
        out[f"last_smem_{nh}"] = lo
        rs = plan(lo + 1, B)["rows_smem"]
        out[f"l2_16_32_{nh}"] = 16 * (rs + 24)          # cls_per = rs + 24 -> 24 L2 rows (rows_smem barely moves)
        out[f"l2_gt32_{nh}"] = 16 * (rs + 40) + 1       # 41 classes per CTA, the last CTA owns fewer
    print("geometry:", out)
    return out


# ------------------------------------------------------------------------------------------ GPU: the sweep
@pytest.mark.gpu
def test_rnnt_sweep_every_decision_against_float64(eng, dev, geometry):
    g = geometry
    vs = sorted({2, 3, 15, 17, 34, 257, 1025, 4097, g["last_smem_1"], g["last_smem_1"] + 1, g["last_smem_2"], g["last_smem_2"] + 1,
                 g["l2_16_32_1"], g["l2_gt32_1"], g["l2_16_32_2"], g["l2_gt32_2"]})
    bs = g["b_switch"]
    b_ragged = 8 * g["clusters"] + 3                   # more groups of 8 than resident clusters, a ragged last group
    nh1_B, nh2_B = [1, bs - 1, bs], [bs + 1, b_ragged]
    cases = []
    for i, V1 in enumerate(vs):
        cases.append((V1, nh1_B[i % 3], (1, 2, 10)[i % 3], 1))
        cases.append((V1, nh2_B[i % 2], (10, 1, 2)[i % 3], 2))
    cases.append((vs[-1], b_ragged, 10, 2))
    weights = {V1: make_weights(V1, V1) for V1 in vs}
    dweights = {V1: _dev_weights(W, dev) for V1, W in weights.items()}
    totals, paths, results = {}, set(), {}
    for ci, (V1, B, ms, nh) in enumerate(cases):
        enc, lens = make_encproj(B, T_SWEEP, 1000 + ci), make_lens(B, T_SWEEP, 1000 + ci)
        hyps, plan = run_greedy(eng, dweights[V1], V1, enc, lens, ms)
        assert plan["NH"] == nh, (V1, B, plan)
        expect_glob = V1 > g[f"last_smem_{nh}"]
        assert plan["GLOB"] == int(expect_glob), (V1, B, plan)
        assert plan["cls_per"] == -(-V1 // 16)
        if V1 == g[f"l2_16_32_{nh}"]:
            assert 16 <= _l2_rows(plan) <= 32, plan
        if V1 == g[f"l2_gt32_{nh}"]:
            assert _l2_rows(plan) > 32, plan
        paths.add((plan["NH"], plan["GLOB"], "L2>32" if _l2_rows(plan) > 32 else ("L2>0" if _l2_rows(plan) > 0 else "smem")))
        if plan["groups"] > plan["clusters"] and B % plan["nu"] != 0:
            paths.add("ragged")
        for b in range(B):
            try:
                _merge(totals.setdefault(ms, {}), replay(weights[V1], enc[b], int(lens[b]), ms, *hyps[b]))
            except AssertionError as e:
                raise AssertionError(f"V1={V1} B={B} max_symbols={ms} plan={plan} utterance {b}: {e}") from None
        # each utterance decoded alone gives the same bits
        for b in range(B):
            alone, _ = run_greedy(eng, dweights[V1], V1, enc[b:b + 1], lens[b:b + 1], ms)
            assert alone[0] == hyps[b], (V1, B, ms, b)
        results[ci] = (enc, lens, hyps)
    # descending V1 in the same process: cached launch attributes must not change a bit
    for ci in sorted(range(len(cases)), key=lambda i: -cases[i][0]):
        V1, B, ms, nh = cases[ci]
        enc, lens, hyps = results[ci]
        again, plan = run_greedy(eng, dweights[V1], V1, enc, lens, ms)
        assert plan["NH"] == nh and again == hyps, (V1, B, ms)
    print("paths:", sorted(map(str, paths)))
    for want in ((1, 0, "smem"), (1, 1, "L2>0"), (1, 1, "L2>32"), (2, 0, "smem"), (2, 1, "L2>0"), (2, 1, "L2>32"), "ragged"):
        assert want in paths, want
    for ms, total in sorted(totals.items()):
        _assert_non_vacuous(total, f"sweep, max_symbols={ms}")


# ------------------------------------------------------------------------------------------ GPU: exact ties
def _tie_weights(V1, pairs, seed):
    """make_weights with each (lo, hi) pair given one strong W_o row and bias, so that the pair wins most token decisions
    with bit-identical logits; (k, blank) pairs copy blank's row into k."""
    W = make_weights(V1, seed)
    blank = V1 - 1
    strong = np.full(H, 0.05, np.float32)
    strong[0] = 0.0
    for lo, hi in pairs:
        if hi == blank:
            W["wo"][lo], W["bo"][lo] = W["wo"][blank], W["bo"][blank]
        else:
            W["wo"][lo] = W["wo"][hi] = strong
            W["bo"][lo] = W["bo"][hi] = 1.0
    return W


@pytest.mark.gpu
@pytest.mark.parametrize("nh", [1, 2])
def test_rnnt_exact_ties_lower_index_wins(eng, dev, geometry, nh):
    g = geometry
    B = 3 if nh == 1 else g["b_switch"] + 2
    V1 = g[f"l2_gt32_{nh}"]                           # smem rows, prefetched L2 rows and remainder-loop rows in every CTA
    probe = make_weights(V1, 0)
    _, plan = run_greedy(eng, _dev_weights(probe, dev), V1, np.zeros((B, 1, H), np.float32), np.zeros(B, np.int32), 1)
    cp, rs = plan["cls_per"], plan["rows_smem"]
    assert plan["NH"] == nh and plan["GLOB"] == 1 and cp - rs > 32, plan
    cases = {
        "smem row vs L2 prefetch row": (3 * cp + rs - 1, 3 * cp + rs),
        "CTA 0 vs CTA 15": (0, 15 * cp),
        "remainder row vs a later CTA's smem row": (2 * cp + rs + 35, 9 * cp + 1),
        "earlier smem row vs remainder row": (4, 5 * cp + rs + 33),
        "token vs blank": (11, V1 - 1),
    }
    for ci, (what, (lo, hi)) in enumerate(cases.items()):
        W = _tie_weights(V1, [(lo, hi)], 50 + ci)
        ms = 2 if ci % 2 else 10
        enc, lens = make_encproj(B, T_SWEEP, 70 + ci), make_lens(B, T_SWEEP, 70 + ci)
        hyps, _ = run_greedy(eng, _dev_weights(W, dev), V1, enc, lens, ms)
        ties = sum(h[0].count(lo) for h in hyps)
        for b, h in enumerate(hyps):
            replay(W, enc[b], int(lens[b]), ms, *h)
            if hi == V1 - 1:   # blank's logit always equals token lo's: the kernel must never choose blank
                assert len(h[0]) == int(lens[b]) * ms, (what, b)
            else:
                assert hi not in h[0], (what, b, lo, hi)
        assert ties > 0, f"{what}: the tied classes never won, the test is vacuous"


# ------------------------------------------------------------------------------------------ GPU: non-finite rows
@pytest.mark.gpu
@pytest.mark.parametrize("V1,nh", [(34, 1), (34, 2), (1025, 1), (4097, 2)])
def test_rnnt_nonfinite_rows_decode_as_torch(eng, dev, geometry, V1, nh):
    W = make_weights(V1, 7)
    wo = W["wo"]
    cls = np.arange(V1)
    wo[:, 1] = np.where(cls % 2 == 0, 0.3, -0.3)               # units 1 + 2 at +inf: opposite signs -> NaN logits
    wo[:, 2] = np.where(cls % 3 == 0, -0.2, 0.2)
    wo[:, 3] = -np.abs(wo[:, 3]) - 1e-3                          # all -inf
    wo[:, 4] = np.abs(wo[:, 4]) + 1e-3                           # all +inf
    wo[:, 5] = np.where(cls < 5, -0.3, 0.3)                      # +inf from class 5 on
    B = 5 if nh == 1 else geometry["b_switch"] + 3
    T = T_SWEEP
    clean = make_encproj(B, T, 90 + V1)
    lens = np.full(B, T, np.int32)
    lens[B - 1] = 4
    bad = clean.copy()
    bad[0, 2, :] = NAN
    bad[1, 3, 1] = bad[1, 3, 2] = INF
    bad[2, 1, 3] = INF
    bad[3, 5, 4] = INF
    bad[4, 0, 5] = INF
    Wd = _dev_weights(W, dev)
    hyps, plan = run_greedy(eng, Wd, V1, bad, lens, 10)
    assert plan["NH"] == nh
    nonfinite = 0
    for b in range(B):
        assert all(0 <= k < V1 for k in hyps[b][0])
        st = replay(W, bad[b], int(lens[b]), 10, *hyps[b])
        nonfinite += st["nonfinite"]
    assert nonfinite >= 5
    # a NaN frame emits token 0 max_symbols times, as the reference's argmax of an all-NaN row
    assert [k for k, f in zip(*hyps[0]) if f == 2] == [0] * 10
    ref, _ = run_greedy(eng, Wd, V1, clean, lens, 10)
    for b in range(5, B):
        assert hyps[b] == ref[b], b
    again, _ = run_greedy(eng, Wd, V1, clean, lens, 10)        # the device is healthy afterwards
    assert again == ref


# ------------------------------------------------------------------------------------------ GPU: CTC
_CTC = {}


def _ctc_model(V1, dev):
    if V1 not in _CTC:
        ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1)
        ck["cfg"]["head"]["num_classes"] = V1
        ck["cfg"]["decoding"]["vocabulary"] = [f"<{i}>" for i in range(V1 - 1)]
        rng = np.random.default_rng(V1)
        w = rng.standard_normal((V1, 768)) * 0.05
        b = rng.standard_normal(V1) * 0.5
        # exact ties across class groups (9 classes) and tiles (36): identical rows give bit-identical logits
        # columns for the non-finite rows: +inf on feature 700 meets both signs and a zero (partial NaN), on 701 a
        # column negative for class 0 and positive after it (+inf from class 1 on), on 702 a negative column (-inf)
        cls = np.arange(V1)
        w[:, 700] = np.where(cls % 2 == 0, 0.01, -0.01)
        w[V1 // 2, 700] = 0.0
        w[:, 701] = np.where(cls < 1, -0.01, 0.01)
        w[:, 702] = -np.abs(w[:, 702]) - 1e-4
        pairs, used = [], set()
        for lo, hi in ((0, 10), (8, 9), (3, 40), (30, 71), (20, V1 - 1)):     # (20, blank): a token against blank
            if lo < hi < V1 and not {lo, hi} & used:
                pairs.append((lo, hi))
                used |= {lo, hi}
        dirs = rng.choice([-1.0, 1.0], size=(max(len(pairs), 1), 768))
        for i, (lo, hi) in enumerate(pairs):
            w[lo] = w[hi] = 0.02 * dirs[i]
            b[lo] = b[hi] = 1.0
        sd = ck["state_dict"]
        sd["head.decoder_layers.0.weight"] = torch.from_numpy(w.astype(np.float32)).unsqueeze(-1)
        sd["head.decoder_layers.0.bias"] = torch.from_numpy(b.astype(np.float32))
        model = gigaam.load_model("v2_ctc", fp16_encoder=False, device=dev, checkpoint=ck)
        _CTC[V1] = (model, sd, pairs, torch.from_numpy(dirs).float())
    return _CTC[V1]


@pytest.mark.gpu
@pytest.mark.parametrize("V1", [2, 35, 36, 37, 72, 73, 1025])
def test_ctc_argmax_against_float64_and_torch(dev, V1):
    model, sd, pairs, dirs = _ctc_model(V1, dev)
    B, T = 5, 64
    g = torch.Generator().manual_seed(V1)
    x = torch.randn(B, T, 768, generator=g) * 0.05
    # every other frame points at one tied pair's row: that pair is the row's maximum, with bit-identical logits
    for t in range(0, T, 2):
        x[:, t] += 0.5 * dirs[(t // 2) % len(dirs)]
    W, bias = sd["head.decoder_layers.0.weight"][..., 0], sd["head.decoder_layers.0.bias"]
    # non-finite rows: a NaN frame, partial NaN, +inf from class 1 on and all -inf: label 0 for each
    n_bad = 4
    x[0, 5] = NAN
    x[1, 7, 700] = INF
    x[2, 9, 701] = INF
    x[3, 11, 702] = INF
    lens = torch.tensor([T, T, T, T, 33], dtype=torch.int32)
    encoded = x.to(dev).transpose(1, 2)
    with torch.inference_mode():
        model.decoding.decode(model.head, encoded, lens.to(dev))
        labels = model._get_engine()._ws_dec.peek((B, T))[: B * T * 4].view(torch.int32).view(B, T).cpu().long()
    z = F.linear(x.double(), W.double(), bias.double())
    want = torch.log_softmax(z, -1).argmax(-1)
    finite = torch.isfinite(z).all(-1)
    assert ((labels >= 0) & (labels < V1)).all()
    assert torch.equal(labels[~finite], want[~finite])
    assert int((~finite).sum()) == n_bad
    assert want[1, 7] == want[2, 9] == want[3, 11] == 0 and bool(z[1, 7].isnan().any()) and bool(z[2, 9].isposinf().any())
    zf = z[finite]
    lf = labels[finite]
    margin = zf.max(-1).values - zf.gather(1, lf[:, None])[:, 0]
    top2 = zf.topk(min(2, V1), -1).values
    near = (top2[:, 0] - top2[:, 1]) < CTC_TIE
    exact_ties = 0
    for lo, hi in pairs:
        assert not bool((lf == hi).any()), (lo, hi)
        exact_ties += int((lf == lo).sum())
    print(f"V1={V1}: worst margin {float(margin.max()):.3g}, {int(near.sum())} near ties, {exact_ties} exact ties won")
    assert float(margin.max()) <= CTC_TIE
    assert int(near.sum()) - exact_ties < NEAR_MAX * len(lf)
    if pairs:
        assert exact_ties > 0


# ------------------------------------------------------------------------------------------ GPU: model level
@pytest.mark.gpu
def test_nonfinite_encoder_frames_decode_as_oracle_and_leave_neighbours_alone(dev):
    """A whole v2_rnnt model: a NaN frame in one utterance of a ragged batch and +inf on one feature of a frame in another
    reach model.decoding.decode; both hypotheses equal the oracle's, the other utterances do not move, and
    head.joint.joint has NaN exactly where the oracle has it."""
    ck = synthetic.synthetic_checkpoint("v2_rnnt", seed=0, n_layers=2)
    sd = ck["state_dict"]
    model = gigaam.load_model("v2_rnnt", fp16_encoder=False, device=dev, checkpoint=ck)
    wav, wav_len = gigaam.synthetic_audio(4, 1.5, seed=3, ragged=True)
    with torch.inference_mode():
        enc, enc_len = model(wav.to(dev), wav_len.to(dev))
        hyp_c = model.decoding.decode(model.head, enc, enc_len)
        bad = enc.clone()
        bad[2, :, 3] = NAN
        bad[1, 5, 4] = INF
        hyp_b = model.decoding.decode(model.head, bad, enc_len)
    for b in (0, 3):
        assert hyp_b[b][1:] == hyp_c[b][1:], b
    want = orc.rnnt_greedy(bad.float().cpu(), enc_len.cpu(), sd, max_symbols=ck["cfg"]["decoding"]["max_symbols_per_step"])
    for b in (1, 2):
        assert (hyp_b[b][1], hyp_b[b][2]) == want[b], b
        assert all(0 <= k < ck["cfg"]["head"]["joint"]["num_classes"] for k in hyp_b[b][1])
    assert [k for k, f in zip(hyp_b[2][1], hyp_b[2][2]) if f == 3] == [0] * 10     # the NaN frame: token 0, max_symbols times
    # head.joint.joint keeps NaN where the oracle has it
    dec = torch.rand(4, 3, 320, generator=torch.Generator().manual_seed(1)) * 2 - 1
    with torch.inference_mode():
        got = model.head.joint.joint(bad.transpose(1, 2), dec.to(dev)).cpu()
    e = F.linear(bad.transpose(1, 2).float().cpu(), sd["head.joint.enc.weight"], sd["head.joint.enc.bias"]).unsqueeze(2)
    p = F.linear(dec, sd["head.joint.pred.weight"], sd["head.joint.pred.bias"]).unsqueeze(1)
    ref = F.linear(F.relu(e + p), sd["head.joint.joint_net.1.weight"], sd["head.joint.joint_net.1.bias"]).log_softmax(-1)
    assert bool(ref[2, 3].isnan().all())
    assert torch.equal(got.isnan(), ref.isnan())
    fin = ~ref.isnan()
    assert float((got[fin] - ref[fin]).abs().max()) <= 2.5e-4
