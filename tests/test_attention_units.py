"""The rotary and rel_pos attention kernels held to float64 element by element, at every head width a model loads with
(rotary n_heads 48 / 24 / 16 = d_k 16 / 32 / 48; rel_pos also 12 = d_k 64), through gam_test_attention,
gam_test_attention_relpos and gam_test_attention_varlen.  The Frobenius tests of test_gpu_parity.py and
test_long_utterances.py hold a whole [B*T, 768] output at once, which dilutes an error confined to one warp's rows, one
query row or one head; here every element is held to a worst-case bound, and containment is checked bit for bit.

The bound is a contract any correct implementation meets, not a replay of today's kernels: fp16 q / k / v, scores
accumulated in fp32 and scaled by c = fp32(log2 e / sqrt(d_k)) into the exponent of ex2.approx, an online softmax whose
reference point may move once per key block (lazily or not), P rounded to fp16 with the row sum taken over those same
fp16 values, P.V accumulated in fp32, one division and one fp16 store.  Terms (u = 2^-24, U16 = 2^-11):

  * score error ds_ij: fp16 products are exact, the fp32 sum of d_k of them is within d_k u sum_k |q_ik||k_jk|.  rel_pos
    adds two such dot products, (q+u).k_j and (q+v).p_{i-j}: d_k u (sum |q+u||k| + sum |q+v||p|) + u (|ac| + |bd|).
  * exponent: x_ij = s_ij c - m_i, evaluated as fmaf(s, c, -m) in fp32.  Its error, in log2 units, is
        dx_ij = c ds_ij + 3 u c |s_ij| + u (c |s_ij| + L_i),      L_i = c max_j (|s_ij| + ds_ij)
    (c carries 3 roundings: log2 e, sqrtf and the division; the fma one rounding of a value of size <= c |s| + |m|).
    A shift common to a row cancels in the ratio, so only these per-key parts count.
  * ex2.approx.ftz.f32: the PTX ISA gives at most 2 ulp from the correctly rounded result; EX2_REL rounds that up to
    2^-21.5, as TANH_REL does for tanh.  Results flushed to zero are below the fp16 absolute term.
  * P -> fp16: U16 relative, plus F16_ABS = 2^-25 absolute below the normal range.  The denominator sums those same fp16
    values, so the rounding is an error of the weights, not of the ratio.
  * each move of the reference point multiplies every earlier weight by ex2(old - new): EX2_REL plus the rounding of the
    argument, 3 u L_i in log2 units.  The number of moves is bounded by the number of key blocks nb = ceil(n / 128), so
    the bound does not depend on the lazy rule: every weight carries nb - 1 moves.
  Together key j of row i carries a relative weight error
        delta_ij = (1 + expm1(ln2 dx_ij)) (1 + EX2_REL) (1 + U16) (1 + EX2_REL + 3 ln2 u L_i)^(nb - 1) - 1
  and an absolute one of F16_ABS in the scale of the final reference point, where the row sum is >= D_MIN (the key that
  set the reference point has P = fp16(ex2(~0)) = 1).  With e_j the error of key j's weight, o~ - o = sum_j e_j (v_j - o)
  / sum, so, with w_ij the exact softmax weights and |v_j - o| <= |v_j| + |o|:
        weights = [sum_j w_ij delta_ij |v_jd| + |o_id| sum_j w_ij delta_ij + F16_ABS / D_MIN (sum_j |v_jd| + n |o_id|)]
                  / (1 - max_j delta_ij - n F16_ABS / D_MIN)
  * P.V and the row sum accumulated in fp32 at depth n, plus one multiply per move and the two shuffles of the sum:
        acc = (n + nb + 2) u (sum_j w_ij |v_jd| + |o_id|) (1 + max delta) / (1 - max delta)
  * 1 / sum and the multiply: 2 u; then one fp16 store: U16 |value| + F16_ABS.

A row with no valid key is exactly zero.  The worst err / bound of every (kernel, n_heads, case) is printed; a tight
aggregate check (relative Frobenius error against float64) is added as test_kernel_units.py does.

Containment is exact: NaN in one head's columns, in key / value rows at or past an utterance's length, in a neighbouring
utterance's rows or behind the stream changes no bit anywhere else, rows that belong to no utterance keep their
sentinel, and an utterance gives the same bits at every batch position and in every layout that stores it.

Negative controls (CPU): a float64 emulation of one (utterance, head) built as that contract describes, with five faults
planted one at a time, each of which the per-element checker must reject, next to what the whole-batch Frobenius bar of
the older tests would have said.  Model tests at the new widths run a 2-layer encoder against the oracle, and refusals
of heads wider than a kernel runs are checked at load time."""
import ctypes as C
import math

import pytest
import torch

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, synthetic
from gigaam_b200.engine import Engine, rotary_half_tables

U = 2.0 ** -24                 # fp32 unit roundoff
U16 = 2.0 ** -11               # fp16 rounding, relative
F16_ABS = 2.0 ** -25           # fp16 rounding below the normal range, absolute
EX2_REL = 2.0 ** -21.5         # ex2.approx.ftz.f32, relative (PTX ISA: 2 ulp)
D_MIN = 1.0 - 2.0 ** -10       # the row sum in the scale of the final reference point
LOG2E = 1.4426950408889634
LN2 = math.log(2.0)
D = 768
F16_FRO = 1e-3                 # aggregate: relative Frobenius error of the fp16 outputs against float64
SENT16 = -4096.0
NAN = float("nan")
ROTARY_HEADS = [48, 24, 16]
RELPOS_HEADS = [48, 24, 16, 12]
WIDTHS = [("rotary", h) for h in ROTARY_HEADS] + [("rel_pos", h) for h in RELPOS_HEADS]
_WORST = {}                    # (kernel, n_heads, case) -> worst err / bound


# ------------------------------------------------------------------------------------------ the float64 reference and bound
def softmax_bound(s, ds, v, dk):
    """Exact softmax(s / sqrt(dk)) @ v and the per-element bound of the module docstring.  s, ds [..., Tq, n] float64
    scores and their worst-case error, v [..., n, dk] float64 (of fp16 values), n >= 1 -> (o, bound) [..., Tq, dk]."""
    n = s.shape[-1]
    nb = (n + 127) // 128
    c = LOG2E / math.sqrt(dk)
    w = torch.softmax(s / math.sqrt(dk), -1)
    o = w @ v
    sa = s.abs()
    L = c * (sa + ds).amax(-1, keepdim=True)
    dx = c * ds + 3 * U * c * sa + U * (c * sa + L)
    mv = EX2_REL + 3 * LN2 * U * L
    delta = (1 + torch.expm1(LN2 * dx)) * ((1 + EX2_REL) * (1 + U16)) * (1 + mv) ** (nb - 1) - 1
    dmax = delta.amax(-1, keepdim=True)
    wd = w * delta
    va, oa = v.abs(), o.abs()
    a_abs = F16_ABS / D_MIN
    weights = (wd @ va + oa * wd.sum(-1, keepdim=True) + a_abs * (va.sum(-2, keepdim=True) + n * oa)) / (1 - dmax - n * a_abs)
    acc = (n + nb + 2) * U * (w @ va + oa) * (1 + dmax) / (1 - dmax)
    pre = weights + acc
    pre = pre + 2 * U * (oa + pre)
    return o, pre + U16 * (oa + pre) + F16_ABS


def _head_chunk(T, n, H):
    return max(1, min(H, (1 << 25) // max(1, T * (T + n))))


def utterance_ref(kind, x, n, H, pos=None, max_t=None, count_moves=False):
    """float64 (want, bound) [T, 768] of one utterance: x [T, parts * 768] its rows (every row a query, the first n
    keys).  rel_pos scores read the position table directly at row max_t - 1 - (i - j).  count_moves: also the number of
    moves of the rotary kernel's lazy reference point per (head, row) at key blocks >= 6 (after the ring wraps)."""
    T = x.shape[0]
    dk = D // H
    parts = 4 if kind == "rel_pos" else 3
    xv = x.double().view(T, parts, H, dk).permute(1, 2, 0, 3)          # [parts, H, T, dk]
    want = torch.zeros((T, D), dtype=torch.float64, device=x.device)
    tol = torch.zeros_like(want)
    late = torch.zeros((H, T), dtype=torch.float64, device=x.device) if count_moves else None
    if n == 0:
        return want, tol, late
    hc = _head_chunk(T, n, H)
    for h0 in range(0, H, hc):
        hs = slice(h0, min(H, h0 + hc))
        if kind == "rel_pos":
            qu, qv, k, v = xv[0, hs], xv[1, hs], xv[2, hs, :n], xv[3, hs, :n]
            pm = pos[max_t - T: max_t - 1 + n].double().view(T + n - 1, H, dk)[:, hs].transpose(0, 1)   # r = T-1 ... -(n-1)
            idx = (T - 1 - torch.arange(T, device=x.device)[:, None] + torch.arange(n, device=x.device)[None, :])
            idx = idx.expand(qv.shape[0], T, n)
            ac = qu @ k.transpose(-1, -2)
            bd = torch.gather(qv @ pm.transpose(-1, -2), -1, idx)
            dacc = torch.gather(qv.abs() @ pm.abs().transpose(-1, -2), -1, idx) + qu.abs() @ k.abs().transpose(-1, -2)
            s = ac + bd
            ds = dk * U * dacc + U * (ac.abs() + bd.abs())
        else:
            q, k, v = xv[0, hs], xv[1, hs, :n], xv[2, hs, :n]
            s = q @ k.transpose(-1, -2)
            ds = dk * U * (q.abs() @ k.abs().transpose(-1, -2))
        o, b = softmax_bound(s, ds, v, dk)
        want.view(T, H, dk)[:, hs] = o.transpose(0, 1)
        tol.view(T, H, dk)[:, hs] = b.transpose(0, 1)
        if count_moves:
            nb = (n + 127) // 128
            l2 = torch.nn.functional.pad(s * (LOG2E / math.sqrt(dk)), (0, nb * 128 - n), value=-math.inf)
            bmax = l2.view(s.shape[0], T, nb, 128).amax(-1)
            mc = bmax[..., 0].clone()
            for j in range(1, nb):
                move = bmax[..., j] > mc + 8.0
                late[hs] += move * (j >= 6)
                mc = torch.where(move, bmax[..., j], mc)
    return want, tol, late


def worst_element(got, want, tol, dk):
    """(err / bound, description) of the worst element of one utterance's [T, 768] rows; NaN counts as infinite."""
    r = (got.double() - want).abs() / tol
    r = torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)
    i = int(r.argmax())
    row, col = divmod(i, r.shape[1])
    return float(r.view(-1)[i]), (f"row {row} (query tile {row // 128}), head {col // dk}, column {col % dk}: got "
                                  f"{float(got[row, col])!r}, want {float(want[row, col])!r}, bound {float(tol[row, col]):.3e}")


def _check_case(key, outs, refs, dk, fro_bar=F16_FRO):
    """outs / refs: per utterance (klen, got [T, 768], (want, tol)).  Every element within its bound, rows of an
    utterance without keys exactly zero, and the aggregate Frobenius error small; records the worst ratio."""
    worst, where = 0.0, ""
    g_all, w_all = [], []
    for b, (n, got, (want, tol)) in enumerate(zip(outs[0], outs[1], refs)):
        if n == 0:
            assert bool((got == 0).all()), f"{key}: utterance {b} has no key but a non-zero output"
            continue
        r, desc = worst_element(got, want, tol, dk)
        if r > worst:
            worst, where = r, f"utterance {b} (klen {n}, {(n + 127) // 128} key blocks), {desc}"
        g_all.append(got.double().reshape(-1))
        w_all.append(want.reshape(-1))
    _WORST[key] = worst
    print(f"{key}: worst err / bound {worst:.3f} at {where}")
    assert worst <= 1.0, f"{key}: element outside its bound: {where} (err / bound {worst:.2f})"
    if g_all:
        g, w = torch.cat(g_all), torch.cat(w_all)
        rel = float((g - w).norm() / w.norm())
        assert rel < fro_bar, f"{key}: relative Frobenius error {rel:.2e}"


# ------------------------------------------------------------------------------------------ negative controls (CPU)
def emulate(q, k, v, n, *, pos_scores=None, lazy=8.0, fault=None, rows=slice(80, 96)):
    """float64 emulation of one (utterance, head) as the kernels' contract describes: 128-key blocks, block maximum as
    reference point on the first block and moved (rescaling O and the row sum) when a block maximum exceeds it by more
    than `lazy` (0: a running maximum), P = fp16(2^(s c - m)) over the valid keys, the row sum over the same fp16 P,
    O = sum P v, then O / sum stored in fp16.  q [T, dk], k / v [Tk >= n, dk]; pos_scores(i, j) -> the positional term
    of score (i, j) for rel_pos.  `fault` plants one error in the query rows `rows` (one warp's, unless it is one move
    of one row)."""
    T, dk = q.shape
    c = LOG2E / math.sqrt(dk)
    O = torch.zeros((T, dk), dtype=torch.float64)
    S = torch.zeros(T, dtype=torch.float64)
    mc = None
    moved = 0
    qi = torch.arange(T)
    nb = (n + 127) // 128
    for kb in range(nb):
        keys = torch.arange(kb * 128, min(n, kb * 128 + 128))
        s = q @ k[keys].t()
        if pos_scores is not None:
            s = s + pos_scores(qi[:, None], keys[None, :])
            if fault == "rel_shift" and kb == nb - 2:          # chunk 3 of the last full block reads the next diagonal
                ch = slice(48, 64)
                s[rows, ch] = (q[rows] @ k[keys[ch]].t()) + pos_scores(qi[rows, None], keys[None, ch] + 1)
        x = s * c
        bm = x.amax(1)
        if mc is None:
            mc = bm
        else:
            move = bm > mc + lazy
            corr = torch.where(move, torch.exp2(mc - bm), torch.ones_like(mc))
            if fault == "skip_rescale" and bool(move.any()) and moved == 0:
                r0 = int(move.nonzero()[0])                      # one row keeps its old O scale at one move
                keep = O[r0].clone()
                O *= corr[:, None]
                O[r0] = keep
            else:
                O *= corr[:, None]
            moved += int(move.sum())
            S *= corr
            mc = torch.where(move, bm, mc)
        p = torch.exp2(x - mc[:, None]).half().double()
        if fault == "drop_last" and kb == nb - 1:
            p[rows, -1] = 0.0
        S += p.sum(1)
        O += p @ v[keys]
        if fault == "masked_in_sum" and kb == nb - 1:          # key n counted in the denominator only
            S[rows] += torch.exp2((q[rows] @ k[n]) * c - mc[rows]).half().double()
    return (O / S[:, None]).half(), moved


def _control_data(T, n, dk, peaked, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((T, 3, 2 * dk), generator=g, dtype=torch.float64)   # this head and the next one
    if peaked:                                                             # the inputs of the peaked-rows tests
        x[:, 0] *= 6.0
        x[:, 1] *= (0.1 + 2.4 * torch.arange(T, dtype=torch.float64) / T)[:, None]
    return x.half().double()


@pytest.mark.parametrize("fault", ["none", "drop_last", "masked_in_sum", "rel_shift", "skip_rescale", "next_head_column"])
def test_checker_rejects_planted_faults(fault):
    """One (utterance, head) of d_k = 48, T = 256 query rows, n = 200 valid keys (last block: 72 keys, a partial 16-key
    chunk).  The clean emulation passes the per-element checker; each planted fault fails it: the last valid key
    dropped, key n counted in the row sum but not in P.V, the rel_pos diagonal read one off in one 16-key chunk (each
    in one warp's 16 query rows), O not rescaled at one move of one row (peaked rows), and q / k column 47 read from the
    next head's column 0 in one query tile.  The whole-batch Frobenius
    bar of the older tests is evaluated as at (B, T) = (2, 751) with 16 heads: the other 31 (utterance, head) pairs
    exact, each with the norm of this one per row."""
    T, n, dk = 256, 200, 48
    relpos = fault == "rel_shift"
    x = _control_data(T, n, dk, fault == "skip_rescale", 1 + len(fault))
    q, k, v = x[:, 0, :dk], x[:, 1, :dk], x[:, 2, :dk]
    pos_scores = None
    if relpos:
        g = torch.Generator().manual_seed(5)
        qv = torch.randn((T, dk), generator=g, dtype=torch.float64).half().double()
        table = torch.randn((2 * T + 1, dk), generator=g, dtype=torch.float64).half().double()   # row T + r: position r
        pos_scores = lambda i, j: (qv[i] * table[T + i - j]).sum(-1)                          # noqa: E731
    got, moved = emulate(q, k, v, n, pos_scores=pos_scores, lazy=0.0 if relpos else 8.0, fault=fault)
    if fault == "next_head_column":        # query tile 1 (one CTA) reads column 0 of the next head for q and k column 47
        qq, kk = q.clone(), k.clone()
        qq[:, dk - 1], kk[:, dk - 1] = x[:, 0, dk], x[:, 1, dk]
        got[128:] = emulate(qq, kk, v, n)[0][128:]
    s = q @ k[:n].t()
    ds = dk * U * (q.abs() @ k[:n].abs().t())
    if relpos:
        bd = pos_scores(torch.arange(T)[:, None], torch.arange(n)[None, :])
        s = s + bd
        ds = ds + dk * U * (qv.abs()[:, None, :] * table[T + torch.arange(T)[:, None] - torch.arange(n)[None, :]].abs()).sum(-1)
    want, tol = softmax_bound(s, ds, v[:n], dk)
    r, desc = worst_element(got, want, tol, dk)
    fro = float((got.double() - want).norm() / (want.norm() * math.sqrt(2 * 751 * 16 / T)))
    print(f"fault {fault}: per-element worst err / bound {r:.3g} ({desc}); whole-batch Frobenius {fro:.2e} "
          f"-> {'passes' if fro < 1e-3 else 'fails'} the 1e-3 bar")
    if fault == "skip_rescale":
        assert moved > 0, "the peaked rows must move the reference point"
    if fault == "none":
        assert r <= 1.0 and fro < 1e-3
    else:
        assert r > 1.0, f"the per-element checker did not see fault {fault}"


# ------------------------------------------------------------------------------------------ GPU plumbing
def _i32(x, dev):
    return torch.as_tensor(x, dtype=torch.int32).to(dev)


def _call(eng, fn, *args):
    ptrs = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    rc = getattr(eng.lib, fn)(eng.handle, *ptrs, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    _lib.check(eng.lib, eng.handle, rc, fn)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (there is no CPU fallback to test instead)"
    return torch.device("cuda", 0)


def _ckpt(kind, heads, n_layers=1):
    cfg = synthetic.model_cfg("v1_ctc" if kind == "rel_pos" else "v2_ctc", n_layers)
    cfg["encoder"]["n_heads"] = heads
    return {"cfg": cfg, "state_dict": synthetic.synthetic_state_dict(cfg, seed=0)}


_ENGINES = {}


def _engine(dev, kind, heads, max_t=5000):
    key = (kind, heads, max_t)
    if key not in _ENGINES:
        ck = _ckpt(kind, heads)
        _ENGINES[key] = Engine(ck["cfg"], ck["state_dict"], dev, max_encoded_frames=max_t)
    return _ENGINES[key]


def _inputs(kind, rows, max_t, dev, seed, peaked=False, T=None):
    g = torch.Generator(device=dev).manual_seed(seed)
    parts = 4 if kind == "rel_pos" else 3
    x = torch.randn((rows, parts, D), generator=g, device=dev)
    if peaked:
        x[:, 0] *= 6.0
        t = torch.arange(rows, device=dev) % T
        x[:, 1] *= (0.1 + 2.4 * t / T)[:, None]
    pos = torch.randn((2 * max_t - 1, D), generator=g, device=dev).half() if kind == "rel_pos" else None
    return x.reshape(rows, parts * D).half(), pos


def _padded(eng, kind, qkv, pos, lens, B, T):
    out = torch.full((B * T, D), SENT16, dtype=torch.float16, device=qkv.device)
    klen = _i32(lens, qkv.device) if lens is not None else None
    if kind == "rel_pos":
        _call(eng, "gam_test_attention_relpos", qkv, pos, klen, out, B, T)
    else:
        _call(eng, "gam_test_attention", qkv, klen, out, B, T)
    return out


def _varlen(eng, kind, qkv, pos, lens, cu, B, T):
    rows = qkv.shape[0]
    out = torch.full((rows, D), SENT16, dtype=torch.float16, device=qkv.device)
    _call(eng, "gam_test_attention_varlen", qkv, pos if kind == "rel_pos" else None, _i32(lens, qkv.device),
          _i32(cu + [cu[-1] + lens[-1]], qkv.device), out, B, T, rows)
    return out


_LAST_BLOCK = [r + 128 * (i % 6) for i, r in enumerate(list(range(1, 17)) + list(range(113, 129)))] + [0, 1, 127, 128, 129, 768]
PADDED_CASES = {
    # klen = 1 ... 16 and 113 ... 128 (mod 128) and the edges, one ragged batch: the partial 16-key chunk and V zeroing
    "last_block": (768, _LAST_BLOCK, 5000),
    # the rotary K / V ring past 768 keys, ragged
    "ring_769": (769, [769, 1], 5000),
    "ring_1537": (1537, [1537, 768, 1300], 5000),
    "ring_5000": (5000, [5000, 3001], 5000),
    # rel_pos with a 2 * 1000 - 1 row table: the last query tile's window starts before the table
    "table_1000": (1000, [1000, 871], 1000),
    "table_999": (999, [999, 500], 1000),
}


@pytest.mark.gpu
@pytest.mark.parametrize("kind,heads,case", [(k, h, c) for k, h in WIDTHS for c in PADDED_CASES
                                             if k == "rel_pos" or not c.startswith("table")])
def test_attention_padded_within_float64_bound(dev, kind, heads, case):
    T, lens, max_t = PADDED_CASES[case]
    eng = _engine(dev, kind, heads, max_t)
    B = len(lens)
    qkv, pos = _inputs(kind, B * T, max_t, dev, 100 + heads + T)
    out = _padded(eng, kind, qkv, pos, lens, B, T)
    refs, got = [], []
    for b, n in enumerate(lens):
        want, tol, _ = utterance_ref(kind, qkv[b * T:(b + 1) * T], n, heads, pos, max_t)
        refs.append((want, tol))
        got.append(out[b * T:(b + 1) * T])
    _check_case(f"{kind} n_heads={heads} {case}", (lens, got), refs, D // heads)


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,lens", [(1, 1537, None), (2, 2000, [2000, 1300])])
@pytest.mark.parametrize("heads", ROTARY_HEADS)
def test_rotary_peaked_rows_within_float64_bound(dev, heads, B, T, lens):
    """Score rows whose spread grows along the key axis move the lazy reference point again and again after the ring
    wraps; the moves past block 6 are counted from the float64 scores so the case is not vacuous."""
    eng = _engine(dev, "rotary", heads)
    qkv, _ = _inputs("rotary", B * T, 5000, dev, 7 + heads + T, peaked=True, T=T)
    out = _padded(eng, "rotary", qkv, None, lens, B, T)
    refs, got, ns = [], [], lens or [T]
    for b, n in enumerate(ns):
        want, tol, late = utterance_ref("rotary", qkv[b * T:(b + 1) * T], n, heads, count_moves=True)
        print(f"n_heads={heads} utterance {b}: {float(late.mean()):.2f} late moves per row, "
              f"{float((late > 0).double().mean()):.2f} of the rows moving past block 6")
        assert float(late.mean()) >= 1.0 and float((late > 0).double().mean()) > 0.5
        refs.append((want, tol))
        got.append(out[b * T:(b + 1) * T])
    _check_case(f"rotary n_heads={heads} peaked T={T}", (ns, got), refs, D // heads, fro_bar=2e-3)


def _packing(lens, gap, tail):
    cu, r = [], 0
    for n in lens:
        cu.append(r)
        r += n + gap
    return cu, r - gap + tail


VARLEN_CASES = {"short": (768, [300, 0, 1, 129, 768, 5]), "long": (1537, [1537, 200, 769])}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(VARLEN_CASES))
@pytest.mark.parametrize("kind,heads", WIDTHS)
def test_attention_varlen_within_bound_and_contained(dev, kind, heads, case):
    """Packed rows with 9 unused rows between utterances and 300 behind the last: every utterance within its float64
    bound; then each utterance again with every other row NaN (its neighbours', the gaps', the tail's) gives the same
    bits; rows that belong to no utterance keep their sentinel in every run."""
    T, lens = VARLEN_CASES[case]
    B = len(lens)
    eng = _engine(dev, kind, heads)
    cu, rows = _packing(lens, 9, 300)
    qkv, pos = _inputs(kind, rows, 5000, dev, 300 + heads + T)
    out = _varlen(eng, kind, qkv, pos, lens, cu, B, T)
    owned = torch.zeros(rows, dtype=torch.bool, device=dev)
    refs, got = [], []
    for b, n in enumerate(lens):
        owned[cu[b]:cu[b] + n] = True
        refs.append(utterance_ref(kind, qkv[cu[b]:cu[b] + n], n, heads, pos, 5000)[:2])
        got.append(out[cu[b]:cu[b] + n])
    assert bool((out[~owned] == SENT16).all()), "rows outside every utterance were written"
    _check_case(f"{kind} n_heads={heads} varlen {case}", (lens, got), refs, D // heads)
    for b, n in enumerate(lens):
        alone = torch.full_like(qkv, NAN)
        alone[cu[b]:cu[b] + n] = qkv[cu[b]:cu[b] + n]
        o2 = _varlen(eng, kind, alone, pos, lens, cu, B, T)
        assert torch.equal(o2[cu[b]:cu[b] + n].view(torch.int16), out[cu[b]:cu[b] + n].view(torch.int16)), \
            f"utterance {b}: NaN in other rows changed its output"
        assert bool((o2[~owned] == SENT16).all())


@pytest.mark.gpu
@pytest.mark.parametrize("kind,heads", WIDTHS)
def test_attention_heads_are_contained(dev, kind, heads):
    """NaN in the q, k and v columns (and the position-table columns) of heads 1, H/2 and H-1 leaves every other head's
    output bit-identical.  The 64-column TMA box of a head of 48 also loads 16 columns of the next head, of 16 the next
    three heads."""
    T, lens = 300, [300, 211]
    B = len(lens)
    eng = _engine(dev, kind, heads)
    dk = D // heads
    qkv, pos = _inputs(kind, B * T, 5000, dev, 11 + heads)
    clean = _padded(eng, kind, qkv, pos, lens, B, T)
    bad = sorted({1, heads // 2, heads - 1})
    poisoned, ppos = qkv.clone(), pos.clone() if pos is not None else None
    parts = poisoned.view(B * T, -1, D)
    keep = torch.ones(D, dtype=torch.bool, device=dev)
    for h in bad:
        parts[:, :, h * dk:(h + 1) * dk] = NAN
        if ppos is not None:
            ppos[:, h * dk:(h + 1) * dk] = NAN
        keep[h * dk:(h + 1) * dk] = False
    out = _padded(eng, kind, poisoned, ppos, lens, B, T)
    assert torch.equal(out[:, keep].view(torch.int16), clean[:, keep].view(torch.int16)), f"NaN in heads {bad} leaked"


@pytest.mark.gpu
@pytest.mark.parametrize("fill", [NAN, 65504.0, -65504.0])
@pytest.mark.parametrize("kind,heads", WIDTHS)
def test_attention_keys_past_klen_are_contained(dev, kind, heads, fill):
    """Padded layout: the key and value rows at or past each klen filled with NaN or +-65504 leave every stored row
    bit-identical to a finite fill.  Lengths end inside a 16-key chunk, on a chunk and block boundary, and at 0."""
    T, lens = 900, [900, 263, 128, 0, 769]
    B = len(lens)
    eng = _engine(dev, kind, heads)
    qkv, pos = _inputs(kind, B * T, 5000, dev, 21 + heads)
    clean = _padded(eng, kind, qkv, pos, lens, B, T)
    filled = qkv.clone().view(B, T, -1, D)
    for b, n in enumerate(lens):
        filled[b, n:, -2:] = fill                   # k and v are the last two parts in both layouts
    out = _padded(eng, kind, filled.view(B * T, -1), pos, lens, B, T)
    assert torch.equal(out.view(torch.int16), clean.view(torch.int16)), f"keys past klen filled with {fill} changed the output"


@pytest.mark.gpu
@pytest.mark.parametrize("kind,heads", WIDTHS)
def test_attention_same_bits_in_every_layout(dev, kind, heads):
    """One utterance of 333 frames: padded alone (T = 333, no klen), padded at each position of a batch of three with
    T = 500, and packed between two neighbours, all give the same bits."""
    n, T = 333, 500
    eng = _engine(dev, kind, heads)
    utt, pos = _inputs(kind, n, 5000, dev, 31 + heads)
    other, _ = _inputs(kind, 2 * T, 5000, dev, 41 + heads)
    alone = _padded(eng, kind, utt, pos, None, 1, n)
    for at in range(3):
        batch = torch.empty((3, T, utt.shape[1]), dtype=torch.float16, device=dev)
        batch[[i for i in range(3) if i != at]] = other.view(2, T, -1)
        batch[at, :n] = utt
        batch[at, n:] = NAN
        out = _padded(eng, kind, batch.view(3 * T, -1), pos, [T, T, T][:at] + [n] + [T, T][at:], 3, T)
        assert torch.equal(out.view(3, T, D)[at, :n].view(torch.int16), alone.view(torch.int16)), f"batch position {at}"
    lens = [200, n, 457]
    cu, rows = _packing(lens, 0, 40)
    packed = torch.cat([other[:200], utt, other[T:T + 457], torch.full((40, utt.shape[1]), NAN, dtype=torch.float16, device=dev)])
    out = _varlen(eng, kind, packed, pos, lens, cu, 3, T)
    assert torch.equal(out[200:200 + n].view(torch.int16), alone.view(torch.int16)), "packed layout"


@pytest.mark.gpu
def test_bounds_are_not_vacuous():
    """At least one case per kernel comes within 1 % of its bound; a bound no case approaches is too loose."""
    if not _WORST:
        pytest.skip("no bounded case ran in this session")
    for kind in ("rotary", "rel_pos"):
        r = [v for k, v in _WORST.items() if k.startswith(kind + " ")]
        if r:
            print(f"{kind}: worst err / bound over {len(r)} cases {max(r):.3f}, least {min(r):.3f}")
            assert max(r) > 0.01, f"{kind}: no case comes within 1 % of its bound"


# ------------------------------------------------------------------------------------------ LN + RoPE at the new half-widths
@pytest.mark.gpu
@pytest.mark.parametrize("heads", [48, 24])
def test_ln_rope_half_widths_to_position_4999(dev, heads):
    """ln_rope_f16_kernel at half-widths 8 and 16 with the engine's fp32 tables of a 5000-frame model, positions
    0 ... 4999 from row_t, held to test_kernel_units.test_ln_rope's bound."""
    from test_kernel_units import _f16_store, _ln_ref, _ln_rows, _assert_within, rope_ref
    eng = _engine(dev, "rotary", heads)
    dk, base, R = D // heads, 5000, 5003
    cos, sin = (t.to(dev).contiguous() for t in rotary_half_tables(dk, base, base))
    t = (torch.arange(R, device=dev) * 7919) % 5000                     # every position, in scrambled order
    t[:3] = torch.tensor([0, 4999, 4998], device=dev)
    x, gamma, beta = _ln_rows(R, dev, 40 + heads)
    ou = torch.full((R, D), SENT16, dtype=torch.float16, device=dev)
    orr = torch.full((R, D), SENT16, dtype=torch.float16, device=dev)
    _call(eng, "gam_test_ln_rope", x, gamma, beta, cos, sin, cos.shape[0], dk // 2, ou, orr, R, None,
          t.to(torch.int32), 5000, 1)
    y, dy = _ln_ref(x, gamma, beta)
    _assert_within(ou, y, dy + _f16_store(y), f"out_u half-width {dk // 2}")
    want, tol = rope_ref(y, dy, t, dk, base)
    _assert_within(orr, want, tol + _f16_store(want), f"out_r half-width {dk // 2}")


# ------------------------------------------------------------------------------------------ the whole path at the new widths
@pytest.mark.gpu
@pytest.mark.parametrize("kind,heads", [("rotary", 24), ("rotary", 48), ("rel_pos", 12)])
def test_encoder_at_other_head_widths_against_oracle(dev, kind, heads):
    """A 2-layer encoder through load_model on a ragged batch against the oracle, with the bars of
    test_varlen_ragged_batch_against_oracle: ln_rope at half-widths 8 / 16, rotary_half_tables and pack_rel_pos_qkv at
    other d_k, and both kernels inside gam_encode."""
    from test_gpu_parity import _encoder_parity
    ck = _ckpt(kind, heads, n_layers=2)
    model = gigaam.load_model("v1_ctc" if kind == "rel_pos" else "v2_ctc", device=dev, checkpoint=ck)
    secs = [10.0, 0.06, 3.3, 7.77, 0.5, 1.29]
    wav, _ = synthetic.synthetic_audio(len(secs), 10.0, seed=4321)
    wav_len = torch.tensor([int(s * 16000) for s in secs])
    for b, n in enumerate(wav_len.tolist()):
        wav[b, n:] = 0.0
    enc, enc_len, _, len_o, _ = _encoder_parity(model, ck, wav, wav_len, dev)
    pad = torch.arange(enc.shape[2], device=dev)[None, :] >= enc_len[:, None]
    assert float(enc.transpose(1, 2)[pad].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------ refusal at load time
def _refused(kind, heads):
    return (kind == "rotary" and D // heads > _lib.ROTARY_MAX_DK) or (kind == "rel_pos" and D // heads > _lib.REL_POS_MAX_DK)


@pytest.mark.parametrize("kind,heads", [("rotary", 8), ("rotary", 12), ("rel_pos", 8)])
def test_load_model_refuses_heads_wider_than_the_kernel(kind, heads):
    """Before any device work, so on any machine: the message names d_k, n_heads and the kernel's limit."""
    assert _refused(kind, heads)
    limit = _lib.REL_POS_MAX_DK if kind == "rel_pos" else _lib.ROTARY_MAX_DK
    with pytest.raises(ValueError, match=rf"{kind} attention runs heads of d_k <= {limit}, but d_model 768 / "
                                         rf"n_heads {heads} gives d_k = {D // heads}"):
        gigaam.load_model("v1_ctc" if kind == "rel_pos" else "v2_ctc", device="cpu", checkpoint=_ckpt(kind, heads))


def test_head_limits_come_from_the_header():
    assert (_lib.ROTARY_MAX_DK, _lib.REL_POS_MAX_DK) == (48, 64)
    assert not any(_refused(k, h) for k, h in WIDTHS)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,heads", [("rotary", 8), ("rotary", 12), ("rel_pos", 8)])
def test_engine_and_gam_create_refuse_heads_wider_than_the_kernel(dev, kind, heads):
    """Engine(...) raises before it uploads anything (device memory unchanged), and gam_create refuses the same
    configuration with -10 for C callers."""
    ck = _ckpt(kind, heads)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(dev)
    with pytest.raises(ValueError, match=rf"n_heads {heads} gives d_k = {D // heads}"):
        Engine(ck["cfg"], ck["state_dict"], dev)
    assert torch.cuda.memory_allocated(dev) == before
    lib = _lib.load()
    gc = _lib.GamConfig()
    gc.sample_rate, gc.n_mels, gc.n_fft, gc.win_length, gc.hop_length, gc.center = 16000, 64, 400, 400, 160, 1
    gc.feat_in, gc.n_layers, gc.d_model, gc.n_heads, gc.d_ff = 64, 1, D, heads, 3072
    gc.subsampling, gc.subs_kernel_size, gc.conv_kernel_size = 0, 3, 31
    gc.self_attention, gc.pos_emb_max_len = int(kind == "rel_pos"), 5000
    gw = _lib.GamWeights()
    h = C.c_void_p()
    rc = lib.gam_create(C.byref(gc), C.byref(gw), dev.index, C.byref(h))
    try:
        msg = lib.gam_last_error(h).decode()
        assert rc == -10, msg
        limit = _lib.REL_POS_MAX_DK if kind == "rel_pos" else _lib.ROTARY_MAX_DK
        assert f"d_k <= {limit}" in msg and f"n_heads {heads}" in msg and f"d_k = {D // heads}" in msg, msg
    finally:
        lib.gam_destroy(h)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,heads", WIDTHS)
def test_every_accepted_width_loads_and_encodes(dev, kind, heads):
    ck = _ckpt(kind, heads)
    model = gigaam.load_model("v1_ctc" if kind == "rel_pos" else "v2_ctc", device=dev, checkpoint=ck)
    wav, wav_len = synthetic.synthetic_audio(2, 1.0, seed=3, ragged=True)
    enc, enc_len = model(wav.to(dev), wav_len.to(dev))
    assert enc.shape[:2] == (2, D) and bool(torch.isfinite(enc).all())
