"""The fused RNN-T loss (decoding.rnnt_loss; include/gigaam_b200.h, gam_rnnt_loss / gam_rnnt_loss_backward).

CPU: a float64 restatement of the loss (the joint in float64, alpha by logaddexp, gradients by autograd) is itself checked
against torchaudio's rnnt_loss, and the refusals happen before any device work.  GPU: the loss equals -log_likelihood of
decoding.align bit for bit; the eight outputs of the backward are held element by element to a float64 restatement driven
by the kernels' own fp32 operands (kernel_reference, bounds from the arithmetic in kernel_bounds), and those operands -- the
projections, the saved row lse and the occupancies -- to float64 under the walk argument (check_operands); the prediction
network's gradients follow through the chained predict check; realistic shapes agree with the lattice route (joint.joint +
torchaudio); the edge cases, batch invariance, determinism, reductions, the memory formula, training steps and CUDA graph
capture.

The bounds are functions of the widths (d_model, pred_hidden H, joint_hidden J, V+1) and of the launch plan,
which loss_plan restates from rnnt_loss_plan and every GPU case pins to the library through the backward's workspace
size (backward_workspace_bytes).  A CPU emulation of the node and class kernels' partitioning (strips, frame ranges, node
slices and their reductions) shows that the per-element checker passes the correct partitioning and rejects planted
faults in each of them."""
import math

import pytest
import torch

from gigaam_b200 import decoding, synthetic
import gigaam_b200 as gigaam

U32 = 2.0 ** -24     # unit roundoff of fp32


# ------------------------------------------------------------------------------------------ float64 restatement
def lattice64(enc, dec, sd):
    """enc [B, T, d], dec [B, U+1, H] -> (log-probs [B, T, U+1, V+1], hidden rows) of the joint in float64"""
    E = enc @ sd["head.joint.enc.weight"].t() + sd["head.joint.enc.bias"]
    P = dec @ sd["head.joint.pred.weight"].t() + sd["head.joint.pred.bias"]
    hid = (E[:, :, None, :] + P[:, None, :, :]).clamp_min(0)
    z = hid @ sd["head.joint.joint_net.1.weight"].t() + sd["head.joint.joint_net.1.bias"]
    return z.log_softmax(-1), hid


def scores64(lp, y):
    """lp [B, T, U+1, V+1], y [B, U] (ids in [0, V) where used) -> blank, label [B, T, U+1] (label -inf at u = U)"""
    B, T, U1, V1 = lp.shape
    blank = lp[..., V1 - 1]
    yy = y.clamp(0, V1 - 2).long()[:, None, :, None].expand(B, T, U1 - 1, 1)
    label = torch.cat([lp[:, :, :-1].gather(-1, yy)[..., 0], torch.full_like(blank[:, :, :1], float("-inf"))], 2)
    return blank, label


def alpha_beta64(blank, label, enc_len, tlen):
    """-> (loss [B], alpha, beta [B, T, U+1] (-inf outside the lattice)) by logaddexp, differentiable through loss"""
    B, T, U1 = blank.shape
    ninf = torch.tensor(float("-inf"), dtype=blank.dtype, device=blank.device)
    losses, alphas, betas = [], [], []
    for b in range(B):
        Tb, Ub = int(enc_len[b]), int(tlen[b])
        a = [[ninf] * U1 for _ in range(T)]
        be = [[ninf] * U1 for _ in range(T)]
        if Tb == 0:
            losses.append(-ninf)
        else:
            for t in range(Tb):
                for u in range(Ub + 1):
                    if t == 0 and u == 0:
                        a[t][u] = blank.new_zeros(())
                        continue
                    cb = a[t - 1][u] + blank[b, t - 1, u] if t > 0 else ninf
                    cl = a[t][u - 1] + label[b, t, u - 1] if u > 0 else ninf
                    a[t][u] = torch.logaddexp(cb, cl)
            for t in reversed(range(Tb)):
                for u in reversed(range(Ub + 1)):
                    nb = be[t + 1][u] if t + 1 < Tb else (blank.new_zeros(()) if u == Ub else ninf)
                    nl = label[b, t, u] + be[t][u + 1] if u < Ub else ninf
                    be[t][u] = torch.logaddexp(blank[b, t, u] + nb, nl)
            losses.append(-(a[Tb - 1][Ub] + blank[b, Tb - 1, Ub]))
        alphas.append(torch.stack([torch.stack(r) for r in a]).detach())
        betas.append(torch.stack([torch.stack(r) for r in be]).detach())
    return torch.stack(losses), torch.stack(alphas), torch.stack(betas)


def alpha_beta_diag64(blank, label, enc_len, tlen):
    """alpha_beta64's recursions one anti-diagonal at a time, vectorised over u (not differentiable) -> (loss, alpha, beta),
    cheap enough for U = 4096"""
    B, T, U1 = blank.shape
    inf = float("inf")
    alpha = torch.full_like(blank, -inf)
    beta = torch.full_like(blank, -inf)
    loss = torch.full((B,), inf, dtype=blank.dtype, device=blank.device)
    ninf = torch.tensor(-inf, dtype=blank.dtype, device=blank.device)
    for b in range(B):
        Tb, Ub = int(enc_len[b]), int(tlen[b])
        if Tb == 0:
            continue
        a, be, bl, lb = alpha[b], beta[b], blank[b], label[b]
        a[0, 0] = 0
        for d in range(1, Tb + Ub):
            u = torch.arange(max(0, d - (Tb - 1)), min(Ub, d) + 1, device=blank.device)
            t = d - u
            tp, um = (t - 1).clamp_min(0), (u - 1).clamp_min(0)
            cb = torch.where(t > 0, a[tp, u] + bl[tp, u], ninf)
            cl = torch.where(u > 0, a[t, um] + lb[t, um], ninf)
            a[t, u] = torch.logaddexp(cb, cl)
        loss[b] = -(a[Tb - 1, Ub] + bl[Tb - 1, Ub])
        for d in range(Tb - 1 + Ub, -1, -1):
            u = torch.arange(max(0, d - (Tb - 1)), min(Ub, d) + 1, device=blank.device)
            t = d - u
            tn, un = (t + 1).clamp_max(T - 1), (u + 1).clamp_max(U1 - 1)
            nb = torch.where(t + 1 < Tb, be[tn, u], torch.where(u == Ub, torch.zeros_like(ninf), ninf))
            nl = torch.where(u < Ub, lb[t, u] + be[t, un], ninf)
            be[t, u] = torch.logaddexp(bl[t, u] + nb, nl)
    return loss, alpha, beta


def occupancies64(blank, label, alpha, beta, enc_len, tlen, loss):
    """-> (e_blank, e_label) [B, T, U+1] of the header's definition, 0 outside the lattice and for an utterance without a path"""
    B, T, U1 = blank.shape
    eb, el = torch.zeros_like(blank), torch.zeros_like(blank)
    for b in range(B):
        Tb, Ub = int(enc_len[b]), int(tlen[b])
        if Tb == 0 or not math.isfinite(float(loss[b])):
            continue
        a, be, ll = alpha[b, :Tb, :Ub + 1], beta[b, :Tb, :Ub + 1], -loss[b]
        nxt = torch.cat([be[1:], torch.full_like(be[:1], float("-inf"))], 0)
        nxt[Tb - 1, Ub] = 0
        eb[b, :Tb, :Ub + 1] = (a + blank[b, :Tb, :Ub + 1] + nxt - ll).exp()
        el[b, :Tb, :Ub] = (a[:, :Ub] + label[b, :Tb, :Ub] + be[:, 1:] - ll).exp()
    return eb, el


def upstream64(eb, el, y, w, V1):
    """dL/dlog-probs [B, T, U+1, V+1] of sum_b w_b loss_b: -w e_blank on the blank class, -w e_label on class y_{u+1}"""
    B, T, U1 = eb.shape
    G = torch.zeros(B, T, U1, V1, dtype=eb.dtype, device=eb.device)
    G[..., V1 - 1] = -w[:, None, None] * eb
    if U1 > 1:
        idx = y.clamp(0, V1 - 2).long()[:, None, :, None].expand(B, T, U1 - 1, 1)
        G[:, :, :-1].scatter_add_(-1, idx, (-w[:, None, None] * el[:, :, :-1])[..., None])
    return G


def loss_plan(B, T, U, V1, J):
    """rnnt_loss_plan (csrc/rnnt_loss.cu) restated, with the derived sizes the kernels use: a strip of tU columns (the
    smallest power of two >= U+1, at most 64) and tT = 64 / tU frames per node tile; NS strips; ST frame ranges of `chunk`
    tiles each (ranges past the last tile own none); S node slices of s_chunk nodes (a multiple of 64); NC = ceil(J / 64)."""
    U1 = U + 1
    tU = 1
    while tU < U1 and tU < 64:
        tU *= 2
    tT, NS = 64 // tU, -(-U1 // tU)
    n_tiles = -(-T // tT)
    ST = min(min(max(-(-528 // (B * NS)), 1), 64), n_tiles)
    chunk = -(-n_tiles // ST)
    nodes = B * T * U1
    S = min(min(max(-(-528 // -(-V1 // 64)), 1), 64), -(-nodes // 64))
    s_chunk = -(-(-(-nodes // S)) // 64) * 64
    return dict(tU=tU, tT=tT, NS=NS, ST=ST, chunk=chunk, n_tiles=n_tiles, empty=ST - -(-n_tiles // chunk), S=S, s_chunk=s_chunk,
                NC=-(-J // 64), nodes=nodes)


def backward_workspace_bytes(B, T, U, V1, J, d, H):
    """gam_rnnt_loss_backward_workspace_bytes restated from loss_bwd_layout (gam_api.cu): 1 KiB-aligned pieces E, P, dE, dP,
    dE_part (NS B T J), dP_part (ST B (U+1) J) and the larger of the slices' partials and the projection sums' partials"""
    from test_head_training import outer_splits
    p = loss_plan(B, T, U, V1, J)
    BT, BU1 = B * T, B * (U + 1)

    def osw(rows, K):
        S = outer_splits(rows, J, K + 1)
        return S * J * (K + 1) if S > 1 else 0
    pieces = [BT * J, BU1 * J, BT * J, BU1 * J, p["NS"] * BT * J, p["ST"] * BU1 * J,
              max(p["S"] * V1 * (J + 1) if p["S"] > 1 else 0, osw(BT, d), osw(BU1, H))]
    return sum(-(-4 * n // 1024) * 1024 for n in pieces) + 1024


def _ragged(B, T, U, V1, seed, zero_u=True):
    g = torch.Generator().manual_seed(seed)
    enc_len = torch.tensor([T - (3 * b) % max(1, T // 2) for b in range(B)], dtype=torch.int32)
    tlen = torch.tensor([U - (2 * b) % max(1, U) for b in range(B)], dtype=torch.int32)
    if zero_u and B > 1:
        tlen[-1] = 0
    y = torch.randint(0, V1 - 1, (B, U), generator=g)
    for b in range(B):   # garbage past the transcript must never be read
        y[b, int(tlen[b]):] = 10 ** 6 if b % 2 else -7
    return enc_len, y, tlen


# ------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("B,T,U,V1", [(3, 9, 4, 6), (4, 13, 6, 11), (2, 5, 1, 3)])
def test_float64_restatement_equals_torchaudio(B, T, U, V1):
    """The oracle is itself checked: loss and d(logits) of the float64 restatement against torchaudio's fp32 rnnt_loss.
    torchaudio's fp32 errors are bounded by (T + U + V1) steps of relative rounding on O(1 + |loss|) magnitudes; the bound
    below is 16 times that."""
    ta = pytest.importorskip("torchaudio.functional")
    g = torch.Generator().manual_seed(B * 100 + T)
    logits = torch.randn(B, T, U + 1, V1, generator=g, dtype=torch.float64) * 2
    enc_len, y, tlen = _ragged(B, T, U, V1, seed=T)
    l64 = logits.clone().requires_grad_(True)
    blank, label = scores64(l64.log_softmax(-1), y)
    loss64, _, _ = alpha_beta64(blank, label, enc_len, tlen)
    loss64.sum().backward()
    l32 = logits.float().requires_grad_(True)
    yt = torch.where(torch.arange(U)[None] < tlen[:, None].long(), y, torch.zeros_like(y)).int()
    loss32 = ta.rnnt_loss(l32, yt, enc_len, tlen, blank=V1 - 1, reduction="none")
    loss32.sum().backward()
    c = 16 * (T + U + V1) * U32
    assert bool(((loss32.double() - loss64.detach()).abs() <= c * (1 + loss64.detach().abs())).all())
    for b in range(B):   # torchaudio leaves padded nodes' gradient unspecified; compare inside the lattice
        Tb, Ub = int(enc_len[b]), int(tlen[b])
        err = (l32.grad[b, :Tb, :Ub + 1].double() - l64.grad[b, :Tb, :Ub + 1]).abs()
        assert bool((err <= c).all()), float(err.max())
        assert float(l64.grad[b, Tb:].abs().sum() + l64.grad[b, :, Ub + 1:].abs().sum()) == 0.0


@pytest.mark.parametrize("B,T,U", [(3, 9, 4), (2, 5, 0), (4, 13, 6), (2, 4, 9)])
def test_diagonal_alpha_beta_equals_the_scalar_walk(B, T, U):
    """alpha_beta_diag64 (one diagonal at a time) against alpha_beta64, and the occupancy upstream (upstream64) against
    autograd through alpha_beta64's loss."""
    V1 = 7
    g = torch.Generator().manual_seed(B * 10 + U)
    lp = torch.randn(B, T, U + 1, V1, generator=g, dtype=torch.float64).log_softmax(-1).requires_grad_(True)
    enc_len, y, tlen = _ragged(B, T, U, V1, seed=U)
    enc_len[0] = 0 if B > 2 else enc_len[0]
    blank, label = scores64(lp, y)
    loss_s, alpha_s, beta_s = alpha_beta64(blank, label, enc_len, tlen)
    loss_d, alpha_d, beta_d = alpha_beta_diag64(blank.detach(), label.detach(), enc_len, tlen)
    assert torch.allclose(loss_d, loss_s.detach(), rtol=1e-12, atol=0, equal_nan=False) or torch.equal(loss_d, loss_s.detach())
    for a, b in ((alpha_d, alpha_s), (beta_d, beta_s)):
        fin = torch.isfinite(b)
        assert torch.equal(fin, torch.isfinite(a)) and torch.allclose(a[fin], b[fin], rtol=1e-12, atol=1e-12)
    w = torch.rand(B, generator=g, dtype=torch.float64) + 0.5
    fin = torch.isfinite(loss_s)
    (w[fin] * loss_s[fin]).sum().backward()
    eb, el = occupancies64(blank.detach(), label.detach(), alpha_d, beta_d, enc_len, tlen, loss_d)
    G = upstream64(eb, el, torch.where(torch.arange(U)[None] < tlen[:, None].long(), y, torch.full_like(y, V1 - 1)), w, V1)
    assert torch.allclose(G, lp.grad, rtol=1e-10, atol=1e-12), float((G - lp.grad).abs().max())


# ------------------------------------------------------------------------------------------ CPU: the checker's negative controls
def _emulate(E, P, Wo, bo, lse, eb, el, g, y, enc_len, tlen, plan, fault=None):
    """float32 emulation of rnnt_loss_node_grad_kernel and rnnt_loss_class_grad_kernel's partitioning and of the two
    reductions: dE summed per strip of tU columns, then over the NS strips in order; dP summed per frame range of `chunk`
    tiles of tT frames, then over the ST ranges in order; dW_out / db_out per slice of s_chunk nodes, then over the S slices.
    `fault` plants one mistake -> (dE [B, T, J], dP [B, U+1, J], dW_out, db_out)."""
    B, T, J = E.shape
    U1, V1 = P.shape[1], Wo.shape[0]
    t = torch.arange(T)[None, :, None]
    u = torch.arange(U1)[None, None, :]
    live = (t < enc_len[:, None, None]) & (u <= tlen[:, None, None])
    hid = (E[:, :, None, :] + P[:, None, :, :]).clamp_min(0)
    p = ((hid @ Wo.t() + bo) - lse[..., None]).exp()
    ebm, elm = eb * live, el * live
    d = p * (ebm + elm)[..., None]
    d[..., V1 - 1] -= ebm
    lab = elm.clone()
    if fault == "e_label":            # the label term missing at u = U_b - 1
        for b in range(B):
            if int(tlen[b]) > 0:
                lab[b, :, int(tlen[b]) - 1] = 0
    if U1 > 1:
        d[:, :, :-1].scatter_add_(-1, y.clamp(0, V1 - 2).long()[:, None, :, None].expand(B, T, U1 - 1, 1), -lab[:, :, :-1, None])
    dz = g[:, None, None, None] * d
    dhid = (dz @ Wo) * (hid > 0)
    if fault == "j_tail":             # the last 64-unit column chunk of the hidden row dropped
        dhid[..., 64 * (plan["NC"] - 1):] = 0
    tU, tT = plan["tU"], plan["tT"]
    strips = [dhid[:, :, s * tU:(s + 1) * tU].sum(2) for s in range(plan["NS"])]
    if fault == "strip":              # the last strip's dE partial dropped
        strips = strips[:-1]
    dE = torch.zeros(B, T, J)
    for part in strips:
        dE = dE + part
    src = dhid.clone()
    if fault == "neighbour":          # utterance 0's dP summed over utterance 1's columns
        src[0] = dhid[1]
    dP = torch.zeros(B, U1, J)
    for r in range(plan["ST"]):
        t0, t1 = r * plan["chunk"] * tT, min(T, (r + 1) * plan["chunk"] * tT)
        if fault == "range" and r == 0:   # the first range stops one tile short
            t1 -= tT
        dP = dP + src[:, t0:max(t0, t1)].sum(1)
    rows = B * T * U1
    h2, dz2 = hid.reshape(rows, J), dz.reshape(rows, V1)
    dWo, dbo = torch.zeros(V1, J), torch.zeros(V1)
    for sl in range(plan["S"]):
        r0, r1 = sl * plan["s_chunk"], min(rows, (sl + 1) * plan["s_chunk"])
        if fault == "slice_tile" and sl == plan["S"] - 1:   # the slice's last (partial) node tile skipped
            r1 = r0 + (r1 - r0 - 1) // 64 * 64
        dWo = dWo + dz2[r0:r1].t() @ h2[r0:r1]
        dbo = dbo + dz2[r0:r1].sum(0)
    return dE, dP, dWo, dbo


# fault, B, T, U, V+1, joint_hidden: the shapes of test_gradients_against_float64's cases for each regime (NS = 2, 20 empty
# frame ranges, 65 nodes in two slices, NC = 2, and the default widths)
FAULTS = [("strip", 2, 9, 64, 34, 196), ("range", 1, 700, 7, 34, 20), ("slice_tile", 1, 13, 4, 65, 64), ("j_tail", 2, 30, 31, 65, 68),
          ("e_label", 4, 23, 6, 34, 320), ("neighbour", 4, 23, 6, 34, 320)]


@pytest.mark.parametrize("fault,B,T,U,V1,J", FAULTS)
def test_checker_rejects_planted_partition_faults(fault, B, T, U, V1, J):
    """The per-element checker (kernel_reference within kernel_bounds) on the float32 emulation of the gradient kernels, at
    the GPU cases' shapes and lengths and four input seeds: the correct partitioning stays under its bound, each planted fault
    goes over it by at least a factor 10.  Also printed: whether the relative-Frobenius comparison of
    test_realistic_shape_agrees_with_the_lattice_route (tolerance 4 sqrt(T + U) u max|loss|) would have caught it."""
    from test_head_training import _head_ckpt
    sd32 = {k: v.float() for k, v in _head_ckpt("v2_rnnt", V1=V1, J=J)["state_dict"].items() if k.startswith("head.")}
    sd = {k: v.double() for k, v in sd32.items()}
    We, Wp = sd32["head.joint.enc.weight"], sd32["head.joint.pred.weight"]
    Wo, bo = sd32["head.joint.joint_net.1.weight"], sd32["head.joint.joint_net.1.bias"]
    enc_len, y, tlen = _ragged(B, T, U, V1, seed=V1 + T)
    y_used = torch.where(torch.arange(U)[None] < tlen[:, None].long(), y, torch.full_like(y, V1 - 1))
    plan = loss_plan(B, T, U, V1, J)
    assert {"strip": plan["NS"] == 2, "range": plan["empty"] > 0, "slice_tile": plan["S"] > 1 and plan["nodes"] % 64 != 0,
            "j_tail": plan["NC"] == 2}.get(fault, True), plan
    worst_ok, least_bad = 0.0, float("inf")
    for seed in range(4):
        g = torch.Generator().manual_seed(seed)
        enc = torch.randn(B, T, 768, generator=g)
        dec = torch.rand(B, U + 1, 320, generator=g) * 2 - 1
        w = torch.rand(B, generator=g) + 0.5
        # the kernels' fp32 operands: the projections, the row lse, and the occupancies of the float64 walk rounded to fp32
        E = enc @ We.t() + sd32["head.joint.enc.bias"]
        P = dec @ Wp.t() + sd32["head.joint.pred.bias"]
        logits = (E[:, :, None, :] + P[:, None, :, :]).clamp_min(0) @ Wo.t() + bo
        lse = logits.logsumexp(-1)
        lp64 = logits.double().log_softmax(-1)
        blank, label = scores64(lp64, y_used)
        l64, alpha, beta = alpha_beta_diag64(blank, label, enc_len, tlen)
        eb, el = (t.float() for t in occupancies64(blank, label, alpha, beta, enc_len, tlen, l64))
        want, pieces = kernel_reference(E.double(), P.double(), lse.double(), eb.double(), el.double(), w.double(), y_used, enc_len,
                                        tlen, sd, enc.double(), dec.double())
        bounds = kernel_bounds(pieces, sd, enc.double(), dec.double(), plan, w.double())
        tol = 4 * (T + U) ** 0.5 * U32 * float(l64[torch.isfinite(l64)].abs().max())
        for f in (None, fault):
            dE, dP, dWo, dbo = _emulate(E, P, Wo, bo, lse, eb, el, w, y_used, enc_len, tlen, plan, f)
            E2, P2 = dE.reshape(-1, J), dP.reshape(-1, J)
            got = (dE @ We, dP @ Wp, E2.t() @ enc.flatten(0, 1), E2.sum(0), P2.t() @ dec.flatten(0, 1), P2.sum(0), dWo, dbo)
            ratio = max(float(((a.double() - wt).abs() / bd.clamp_min(1e-300)).max()) for a, wt, bd in zip(got, want, bounds))
            fro = max(float((a.double() - wt).norm() / wt.norm().clamp_min(1e-30)) for a, wt in zip(got, want))
            print(f"emulation {f or 'correct'} seed {seed} B={B} T={T} U={U} V1={V1} J={J} (tU={plan['tU']} NS={plan['NS']} "
                  f"ST={plan['ST']} empty={plan['empty']} S={plan['S']} NC={plan['NC']}): worst err/bound {ratio:.3g}; relative "
                  f"Frobenius {fro:.3g} vs {tol:.3g}: {'caught' if fro >= tol else 'missed'} by it")
            if f is None:
                worst_ok = max(worst_ok, ratio)
            else:
                least_bad = min(least_bad, ratio)
    assert worst_ok < 1, worst_ok
    assert least_bad > 10, f"{fault}: a planted fault within 10 times the bound (worst err/bound {least_bad:.3g})"


def _cpu_rnnt(J=None, H=None):
    from test_head_forward_units import _cfg
    return gigaam.GigaAMASR(_cfg("v2_rnnt", J=J, H=H))


@pytest.mark.parametrize("J", [348, 346])
def test_joint_width_refused_before_device_work(J):
    """A joint the fused loss cannot run is refused by rnnt_loss before the head's engine is ever asked for (this model has
    none: it was never placed on a device), with or without gradients; the message names the width and the limit."""
    rnnt = _cpu_rnnt(J=J)
    enc, n = torch.zeros(1, 768, 4), torch.tensor([4])
    y, yl = torch.zeros(1, 2, dtype=torch.long), torch.tensor([2])
    with pytest.raises(ValueError, match=f"joint_hidden {J} .*<= 344"):
        decoding.rnnt_loss(rnnt.head, enc, n, y, yl)
    with torch.no_grad(), pytest.raises(ValueError, match=f"joint_hidden {J} .*<= 344"):
        decoding.rnnt_loss(rnnt.head, enc, n, y, yl)


def test_pred_hidden_the_loss_cannot_project_refused_before_device_work():
    """The loss's projections run pred_hidden in k-steps of 16 (sgemm_bias_kernel): pred_hidden 72 is refused by rnnt_loss
    before any device work, with or without gradients."""
    rnnt = _cpu_rnnt(H=72)
    enc, n = torch.zeros(1, 768, 4), torch.tensor([4])
    y, yl = torch.zeros(1, 2, dtype=torch.long), torch.tensor([2])
    with torch.no_grad(), pytest.raises(ValueError, match="pred_hidden 72 .*multiple of 16"):
        decoding.rnnt_loss(rnnt.head, enc, n, y, yl)


def test_untrainable_pred_hidden_refused_before_device_work():
    """pred_hidden 640 > GAM_PREDICT_BACKWARD_MAX_HIDDEN: the first rnnt_loss / predict that needs its gradient raises
    ValueError naming 640 and 614 before any launch."""
    from gigaam_b200 import _lib
    assert (_lib.RNNT_LOSS_MAX_JOINT_HIDDEN, _lib.PREDICT_BACKWARD_MAX_HIDDEN) == (344, 614)
    rnnt = _cpu_rnnt(H=640)
    rnnt.head.requires_grad_(True)
    enc, n = torch.zeros(1, 768, 4), torch.tensor([4])
    y, yl = torch.zeros(1, 2, dtype=torch.long), torch.tensor([2])
    with pytest.raises(ValueError, match="pred_hidden 640 .*<= 614"):
        decoding.rnnt_loss(rnnt.head, enc, n, y, yl)
    with pytest.raises(ValueError, match="pred_hidden 640 .*<= 614"):
        rnnt.head.decoder.predict(y, None)
    rnnt.head.requires_grad_(False)
    h = torch.zeros(1, 1, 640, requires_grad=True)
    with pytest.raises(ValueError, match="pred_hidden 640 .*<= 614"):
        rnnt.head.decoder.predict(y[:1], (h, torch.zeros(1, 1, 640)))


def test_refusals_happen_before_device_work():
    ck = synthetic.synthetic_checkpoint("v2_ctc", n_layers=1)
    ctc = gigaam.GigaAMASR(ck["cfg"])
    enc, n = torch.zeros(1, 768, 4), torch.tensor([4])
    y, yl = torch.zeros(1, 2, dtype=torch.long), torch.tensor([2])
    with pytest.raises(NotImplementedError, match="ctc_loss"):
        decoding.rnnt_loss(ctc.head, enc, n, y, yl)
    ck = synthetic.synthetic_checkpoint("v2_rnnt", n_layers=1)
    rnnt = gigaam.GigaAMASR(ck["cfg"])
    with pytest.raises(ValueError, match="reduction"):
        decoding.rnnt_loss(rnnt.head, enc, n, y, yl, reduction="batchmean")


# ------------------------------------------------------------------------------------------ GPU
def _dev():
    return torch.device("cuda", 0)


def _model(name, V1, seed=0, J=None, H=None):
    from test_head_training import _model as model_for
    return model_for(name, V1=V1, seed=seed, J=J, H=H)[0]


def _inputs(B, T, U, V1, seed, dev, zero_u=True):
    g = torch.Generator(device=dev).manual_seed(seed)
    enc = torch.randn(B, 768, T, generator=g, device=dev)
    enc_len, y, tlen = _ragged(B, T, U, V1, seed, zero_u)
    return enc, enc_len.to(dev), y.to(dev), tlen.to(dev)


def _grads(model):
    return {k: p.grad.clone() for k, p in model.head.named_parameters()}


BIT_CASES =[("v2_rnnt", 34, 7, 61, 13, None), ("v2_rnnt", 257, 7, 61, 13, None), ("v3_e2e_rnnt", 1025, 7, 61, 13, None),
             ("v2_rnnt", 34, 3, 9, 0, 4), ("v2_rnnt", 65, 3, 30, 31, 68), ("v2_rnnt", 2, 2, 20, 63, 132), ("v2_rnnt", 34, 3, 9, 64, 196),
             ("v2_rnnt", 34, 2, 12, 40, 344), ("v2_rnnt", 34, 1, 700, 7, 20), ("v2_rnnt", 34, 2, 3, 1500, 64),
             ("v2_rnnt", 34, 1, 2, 4096, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,V1,B,T,U,J", BIT_CASES,
                         ids=[f"{c[0]}-{c[1]}" + (f"-{c[2]}-{c[3]}-{c[4]}-J{c[5]}" if c[5] else "") for c in BIT_CASES])
def test_loss_is_minus_align_log_likelihood_bit_for_bit(name, V1, B, T, U, J):
    model = _model(name, V1, J=J)
    enc, enc_len, y, tlen = _inputs(B, T, U, V1, seed=V1, dev=_dev())
    with torch.no_grad():
        ll = decoding.align(model.head, enc, enc_len, y, tlen)[3]
        loss = decoding.rnnt_loss(model.head, enc, enc_len, y, tlen, reduction="none")
    assert torch.isfinite(ll).all()
    assert torch.equal(loss, -ll), (loss, -ll)


def lattice_mask(enc_len, tlen, T, U1, device):
    """[B, T, U+1] True at the nodes of each utterance's lattice, t < T_b and u <= U_b"""
    t = torch.arange(T, device=device)[None, :, None]
    u = torch.arange(U1, device=device)[None, None, :]
    return (t < enc_len.to(device)[:, None, None]) & (u <= tlen.to(device)[:, None, None])


def kernel_reference(E, P, lse, eb, el, g, y, enc_len, tlen, sd, enc, dec):
    """The eight outputs of gam_rnnt_loss_backward (d_enc, d_dec, dW_enc, db_enc, dW_pred, db_pred, dW_out, db_out) in float64
    from the operands its gradient kernels read in fp32: E [B, T, J] and P [B, U+1, J] (the backward's own projections), the
    forward's saved lse / e_blank / e_label [B, T, U+1], g = dL/dloss [B] and the targets y [B, U] as used; enc / dec feed the
    projection gradients.  -> (outputs, the intermediate values kernel_bounds needs)"""
    Wo, bo = sd["head.joint.joint_net.1.weight"], sd["head.joint.joint_net.1.bias"]
    We, Wp = sd["head.joint.enc.weight"], sd["head.joint.pred.weight"]
    B, T, J = E.shape
    U1, V1, d, H = P.shape[1], Wo.shape[0], We.shape[1], Wp.shape[1]
    live = lattice_mask(enc_len, tlen, T, U1, E.device)
    z = E[:, :, None, :] + P[:, None, :, :]
    hid = z.clamp_min(0)
    logits = hid @ Wo.t() + bo
    p = torch.where(live[..., None], (logits - lse[..., None]).exp(), torch.zeros_like(logits))
    G = upstream64(eb.masked_fill(~live, 0), el.masked_fill(~live, 0), y, g, V1)
    dz = G + p * (-G).sum(-1, keepdim=True)
    dhid = (dz @ Wo) * (hid > 0)
    dE, dP = dhid.sum(2), dhid.sum(1)
    E2, P2 = dE.reshape(-1, J), dP.reshape(-1, J)
    out = [dE @ We, dP @ Wp, E2.t() @ enc.reshape(-1, d), E2.sum(0), P2.t() @ dec.reshape(-1, H), P2.sum(0),
           dz.reshape(-1, V1).t() @ hid.reshape(-1, J), dz.sum((0, 1, 2))]
    return out, dict(live=live, z=z, hid=hid, logits=logits, lse=lse, p=p, G=G)


def kernel_bounds(pieces, sd, enc, dec, plan, g):
    """Per-element bounds of kernel_reference's outputs for the fp32 kernels at the launch plan `plan` (loss_plan).  Their
    operands are kernel_reference's inputs, so only the kernels' own rounding enters; a sum evaluated at depth k is within
    k u sum|terms| (test_kernel_units.py's rule).  The depths, from the code:
      hidden rows: the fp32 add E + P, one rounding (which never changes the sign, so no ReLU mask flips);
      logits: logit_tile's fma chain over J (K chunks of 16, ascending k) plus the bias, depth J + 1, and the hidden rows'
        rounding through |W_o|;
      dz = g (exp(z - lse) gamma - [blank] e_blank - [y] e_label): exp's argument carries the logit error and one rounding,
        expf 4 u, then the products and differences; an fp32 value below the normal range underflows by at most 2^-126;
      dhid = dz W_o: one fma chain over V1 (64-class tiles, 16-row chunks), dhid_bounds;
      dE: tU columns inside a strip, then NS strips in segment_sum: depth tU + NS;
      dP: chunk tT frames accumulated in dP_s over a range's tiles, then ST ranges: depth chunk tT + ST;
      dW_out / db_out: the slice's s_chunk nodes, then S slices (a direct write when S = 1), with the hidden entries'
        rounding;
      d_enc, d_dec and the projection gradients: joint_input_bounds."""
    from test_head_training import dhid_bounds, joint_input_bounds
    Wo, bo = sd["head.joint.joint_net.1.weight"], sd["head.joint.joint_net.1.bias"]
    J, V1 = Wo.shape[1], Wo.shape[0]
    live, z, hid, logits, lse, p, G = (pieces[k] for k in ("live", "z", "hid", "logits", "lse", "p", "G"))
    zerr = U32 * z.abs()
    lerr = (J + 1) * U32 * (hid @ Wo.abs().t() + bo.abs()) + zerr @ Wo.abs().t()
    dp = torch.where(live[..., None], lerr + U32 * (logits - lse[..., None]).abs() + 4 * U32, torch.zeros_like(lerr))
    Ga = G.abs()
    Gs = Ga.sum(-1, keepdim=True)
    dz = Ga + p * Gs
    dz_err = (dp + 4 * U32) * p * Gs + 2 * U32 * Ga + 2.0 ** -126 * (2 * p + 2) * g.abs()[:, None, None, None] * live[..., None]
    dh, dh_err = dhid_bounds(dz, dz_err, z, zerr, Wo)
    kE, kP = plan["tU"] + plan["NS"], plan["chunk"] * plan["tT"] + plan["ST"]
    dE, dE_err = dh.sum(2), dh_err.sum(2) + kE * U32 * dh.sum(2)
    dP, dP_err = dh.sum(1), dh_err.sum(1) + kP * U32 * dh.sum(1)
    kO = plan["s_chunk"] + (plan["S"] if plan["S"] > 1 else 0)
    h2, dz2, dze2 = hid.reshape(-1, J), dz.reshape(-1, V1), dz_err.reshape(-1, V1)
    dWo = dze2.t() @ h2 + dz2.t() @ zerr.reshape(-1, J) + kO * U32 * (dz2.t() @ h2)
    dbo = dze2.sum(0) + kO * U32 * dz2.sum(0)
    return joint_input_bounds(enc, dec, sd, dE, dE_err, dP, dP_err) + [dWo, dbo]


def check_operands(E, P, saved, loss, e64, d64, sd, y_used, enc_len, tlen):
    """The gradient kernels' fp32 operands against float64, each within its own derived bound: E / P within the projections'
    depth (d + 1 and H + 1); the saved row lse within the logits' error (depth J + 1 plus the hidden rows' error) and the
    running log-sum-exp's (4 u per class, the rounding of m + log s); each saved occupancy within eps_b e + 2^-126, where
    eps_b is the walk argument: the T_b + U_b + 2 lse2 steps of each walk add a rounding of 4 u (M + 1), M the largest
    |alpha| + |beta| + |ll| of the utterance, and every score read carries its logit and lse error; the loss within the
    forward walk's half of that.  -> (loss64, worst err/bound)"""
    from test_head_training import _check_bound, hidden_rows
    We, be = sd["head.joint.enc.weight"], sd["head.joint.enc.bias"]
    Wp, bp = sd["head.joint.pred.weight"], sd["head.joint.pred.bias"]
    Wo, bo = sd["head.joint.joint_net.1.weight"], sd["head.joint.joint_net.1.bias"]
    d, H, J, V1 = We.shape[1], Wp.shape[1], Wo.shape[1], Wo.shape[0]
    B = E.shape[0]
    mE, mP = e64.abs() @ We.abs().t() + be.abs(), d64.abs() @ Wp.abs().t() + bp.abs()
    worst = max(_check_bound("E", E, e64 @ We.t() + be, (d + 1) * U32 * mE), _check_bound("P", P, d64 @ Wp.t() + bp, (H + 1) * U32 * mP))
    z, zerr = hidden_rows(e64, d64, sd)
    hid = z.clamp_min(0)
    logits = hid @ Wo.t() + bo
    lerr = (J + 1) * U32 * (hid @ Wo.abs().t() + bo.abs()) + zerr @ Wo.abs().t()
    lse = logits.logsumexp(-1)
    lse_err = lerr.amax(-1) + U32 * (4 * V1 + 2 * lse.abs() + 2)
    worst = max(worst, _check_bound("lse", saved[0], lse, lse_err))
    lp64 = logits - lse[..., None]
    blank, label = scores64(lp64, y_used)
    el_c, tl_c = enc_len.cpu(), tlen.cpu()
    loss64, alpha, beta = alpha_beta_diag64(blank, label, el_c, tl_c)
    eb, el = occupancies64(blank, label, alpha, beta, el_c, tl_c, loss64)
    serr = lerr.amax(-1) + lse_err + U32 * lp64.abs().amax(-1)
    eps = torch.zeros(B, dtype=torch.float64, device=E.device)
    lb = torch.zeros(B, dtype=torch.float64, device=E.device)
    for b in range(B):
        Tb, Ub = int(el_c[b]), int(tl_c[b])
        if Tb == 0 or not math.isfinite(float(loss64[b])):
            continue
        a, be_ = alpha[b, :Tb, :Ub + 1], beta[b, :Tb, :Ub + 1]
        fin = torch.isfinite(a) & torch.isfinite(be_)
        M = float((a.abs() + be_.abs())[fin].max()) + abs(float(loss64[b]))
        se = float(serr[b, :Tb, :Ub + 1].max())
        lb[b] = (Tb + Ub + 2) * (2 * U32 * (M + 1) + se)
        eps[b] = (Tb + Ub + 2) * (4 * U32 * (M + 1) + 2 * se)
    _check_loss(loss, loss64, lb)
    for nm, got, want in (("e_blank", saved[1], eb), ("e_label", saved[2], el)):
        worst = max(worst, _check_bound(nm, got, want, eps[:, None, None] * want + 2.0 ** -126))
    return loss64, worst


def _check_loss(loss, loss64, lb):
    inf = torch.isinf(loss64)
    assert torch.equal(torch.isinf(loss.cpu()), inf.cpu()), (loss, loss64)
    err = (loss.double() - loss64.to(loss.device)).abs()[~inf.to(loss.device)]
    assert bool((err <= lb.to(loss.device)[~inf.to(loss.device)]).all()), (loss, loss64, lb)


def _call(eng, fn, *args):
    import ctypes as C
    from gigaam_b200 import _lib
    ptrs = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    rc = getattr(eng.lib, fn)(eng.handle, *ptrs, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    _lib.check(eng.lib, eng.handle, rc, fn)


def _backward(eng, enc, dec, y_used, enc_len, tlen, saved, g, fill=0):
    """gam_rnnt_loss_backward called directly, its workspace and outputs filled with the byte `fill` / NaN -> (the eight
    outputs, E [B, T, J], P [B, U+1, J]: the projections it computed, read back from the workspace (loss_bwd_layout carves E
    at the first 1 KiB boundary and P at the next one past it))"""
    B, T, d = enc.shape
    U1, H = dec.shape[1], dec.shape[2]
    U, J, V1 = U1 - 1, eng.gam_config.joint_hidden, eng.num_classes
    nb = int(eng.lib.gam_rnnt_loss_backward_workspace_bytes(eng.handle, B, T, U))
    assert nb == backward_workspace_bytes(B, T, U, V1, J, d, H)
    ws = torch.full((nb,), fill, dtype=torch.uint8, device=enc.device)
    outs = [torch.full(sh, float("nan"), device=enc.device) for sh in [(B, T, d), (B, U1, H), (J, d), (J,), (J, H), (J,), (V1, J), (V1,)]]
    i32 = [t.to(torch.int32).contiguous() for t in (y_used, enc_len, tlen)]
    _call(eng, "gam_rnnt_loss_backward", enc, dec, *i32, B, T, U, saved, g, ws, nb, *outs)
    off = -ws.data_ptr() % 1024
    e_bytes = B * T * J * 4
    p_off = off + -(-e_bytes // 1024) * 1024
    E = ws[off:off + e_bytes].view(torch.float32).view(B, T, J).clone()
    P = ws[p_off:p_off + B * U1 * J * 4].view(torch.float32).view(B, U1, J).clone()
    return outs, E, P


def _gpu_case(model, enc, enc_len, y, tlen, w, fill=0):
    """One GPU case: the forward and a direct backward at the kernels' own prediction-network outputs; their operands
    checked against float64 (check_operands), the outputs against kernel_reference within kernel_bounds.  -> (outputs,
    kernel_reference's outputs, bounds, plan, worst ratios of the operands and of the outputs)"""
    from test_head_training import _check_bound
    eng = model._get_engine()
    y_used, x = decoding._rnnt_inputs(eng, y, tlen)
    e = enc.detach().transpose(1, 2).contiguous()
    with torch.no_grad():
        dec, _ = model.head.decoder.predict(x, None)
        loss, saved = eng.rnnt_loss(e, dec, y_used, enc_len, tlen)
    outs, E, P = _backward(eng, e, dec, y_used, enc_len, tlen, saved, w, fill)
    sd = {f"head.{k}": v.detach().double().to(enc.device) for k, v in model.head.state_dict().items()}
    e64, d64 = e.double(), dec.double()
    _, worst_ops = check_operands(E, P, saved, loss, e64, d64, sd, y_used, enc_len, tlen)
    want, pieces = kernel_reference(E.double(), P.double(), *(t.double() for t in saved), w.double(), y_used, enc_len, tlen, sd, e64, d64)
    B, T, _ = e.shape
    plan = loss_plan(B, T, y.shape[1], eng.num_classes, eng.gam_config.joint_hidden)
    bounds = kernel_bounds(pieces, sd, e64, d64, plan, w.double())
    names = ("d_enc", "d_dec", "dW_enc", "db_enc", "dW_pred", "db_pred", "dW_out", "db_out")
    worst = max(_check_bound(nm, a, wt, bd) for nm, a, wt, bd in zip(names, outs, want, bounds))
    return dict(outs=outs, want=want, bounds=bounds, plan=plan, loss=loss, x=x, sd=sd, worst_ops=worst_ops, worst=worst)


# name, V+1, B, T, U, joint_hidden (None: the model's 320), pred_hidden (None: 320), the plan regime the case is chosen for,
# lengths (None: _ragged)
GRAD_CASES = [
    ("v2_rnnt", 34, 4, 23, 6, None, None, dict(tU=8, NS=1, NC=5), None),
    ("v2_rnnt", 257, 3, 17, 9, None, None, dict(tU=16, NS=1), None),
    ("v3_e2e_rnnt", 1025, 3, 13, 5, None, None, dict(tU=8), None),
    ("v2_rnnt", 34, 2, 9, 0, 4, None, dict(tU=1, tT=64, NC=1, S=1), None),
    ("v2_rnnt", 63, 3, 11, 1, 20, None, dict(tU=2, NC=1), None),
    ("v2_rnnt", 64, 2, 40, 3, 64, 16, dict(tU=4, NC=1), None),
    ("v2_rnnt", 65, 2, 30, 31, 68, None, dict(tU=32, NC=2), None),
    ("v2_rnnt", 2, 2, 20, 63, 132, None, dict(tU=64, NS=1, NC=3), None),
    ("v2_rnnt", 34, 2, 9, 64, 196, None, dict(tU=64, NS=2, NC=4), None),
    ("v2_rnnt", 34, 2, 12, 40, 344, None, dict(tU=64, NC=6), None),
    ("v2_rnnt", 34, 2, 5, 200, 64, None, dict(NS=4), None),
    ("v2_rnnt", 34, 1, 700, 7, 20, None, dict(tT=8, ST=64, chunk=2, empty=20), None),
    ("v2_rnnt", 65, 1, 13, 4, 64, None, dict(S=2, nodes=65), None),
    ("v2_rnnt", 34, 5, 30, 9, 64, None, dict(tT=4, chunk=1), ([30, 0, 1, 17, 30], [9, 4, 0, 9, 3])),
    ("v3_e2e_rnnt", 1025, 2, 60, 2, None, None, {}, None),      # blank-heavy: many more frames than tokens
    ("v3_e2e_rnnt", 1025, 2, 8, 20, None, None, {}, None),      # label-heavy: more tokens than frames
    ("v2_rnnt", 34, 1, 3, 1023, 64, None, dict(NS=16), None),   # alpha / beta: U+1 = 1024 threads, one node each
    ("v2_rnnt", 34, 1, 3, 1500, 64, None, {}, None),            # 1024 threads looping over each diagonal
    ("v2_rnnt", 34, 1, 2, 4096, 64, None, {}, None),            # the longest transcript (kAlignMaxTokens)
    ("v2_rnnt", 34, 3, 11, 5, 64, 80, {}, None),                # predict backward: a 64-unit block and a 16-unit tail
    ("v2_rnnt", 34, 3, 11, 5, 64, 608, {}, None),               # the widest pred_hidden the loss and the predict backward share
]


def _case_id(c):
    name, V1, B, T, U, J, H, _, lens = c
    return f"{name}-{V1}-{B}-{T}-{U}" + (f"-J{J}" if J else "") + (f"-H{H}" if H else "") + ("-lengths" if lens else "")


def test_plan_restatement_covers_every_regime():
    """The cases of test_gradients_against_float64 reach, by loss_plan: NC 1-6, tU 1-64, NS 1, 2 and >= 4, an empty frame
    range, S = 1 and S > 1, and alpha / beta with more lattice columns than threads; each its own regime."""
    plans = []
    for name, V1, B, T, U, J, H, regime, _ in GRAD_CASES:
        p = loss_plan(B, T, U, V1, J or 320)
        assert all(p[k] == v for k, v in regime.items()), (name, B, T, U, J, regime, p)
        plans.append((p, U))
    assert {p["NC"] for p, _ in plans} == set(range(1, 7))
    assert {p["tU"] for p, _ in plans} == {1, 2, 4, 8, 16, 32, 64}
    assert {1, 2} <= {p["NS"] for p, _ in plans} and max(p["NS"] for p, _ in plans) >= 4
    assert any(p["empty"] > 0 for p, _ in plans) and any(p["S"] == 1 for p, _ in plans) and any(p["S"] > 1 for p, _ in plans)
    assert max(U + 1 for _, U in plans) > 1024
    # the plan's own arithmetic at the edges: the first range holds chunk tiles, the last non-empty range at least one
    p = loss_plan(1, 700, 7, 34, 20)
    assert (p["n_tiles"], p["ST"], p["chunk"], p["empty"]) == (88, 64, 2, 20)


@pytest.mark.gpu
@pytest.mark.parametrize("case", GRAD_CASES, ids=[_case_id(c) for c in GRAD_CASES])
def test_gradients_against_float64(case):
    """decoding.rnnt_loss's gradients equal, bit for bit, a direct gam_rnnt_loss_backward on the same forward; its eight
    outputs are held to kernel_reference within kernel_bounds, its operands to float64 (check_operands), and the prediction
    network's gradients to predict_grads of kernel_reference's d_dec, whose bound is carried."""
    from test_head_training import _check_bound, _predict_bounds, predict_grads
    name, V1, B, T, U, J, H, regime, lens = case
    dev = _dev()
    model = _model(name, V1, J=J, H=H)
    model.head.requires_grad_(True)
    enc, enc_len, y, tlen = _inputs(B, T, U, V1, seed=V1 + T, dev=dev)
    if lens is not None:           # valid ids up to each new length, garbage past it
        enc_len = torch.tensor(lens[0], dtype=torch.int32, device=dev)
        tlen = torch.tensor(lens[1], dtype=torch.int32, device=dev)
        y = y.clamp(0, V1 - 2)
        for b in range(B):
            y[b, lens[1][b]:] = 10 ** 6 if b % 2 else -7
    enc.requires_grad_(True)
    w = torch.rand(B, generator=torch.Generator(device=dev).manual_seed(3), device=dev) + 0.5
    w[enc_len == 0] = 1e6          # an utterance without a path: its upstream weight must not matter
    loss = decoding.rnnt_loss(model.head, enc, enc_len, y, tlen, reduction="none")
    loss.backward(w)
    c = _gpu_case(model, enc, enc_len, y, tlen, w)
    plan = c["plan"]
    assert all(plan[k] == v for k, v in regime.items()), (regime, plan)
    assert torch.equal(c["loss"], loss.detach())
    j = model.head.joint
    auto = (enc.grad.transpose(1, 2), None, j.enc.weight.grad, j.enc.bias.grad, j.pred.weight.grad, j.pred.bias.grad,
            j.joint_net._modules["1"].weight.grad, j.joint_net._modules["1"].bias.grad)
    for i, (a, o) in enumerate(zip(auto, c["outs"])):
        assert a is None or torch.equal(a, o), f"output {i}: autograd and the direct call differ"
    # the prediction network: its backward (gam_rnnt_predict_backward) from the reference d_dec, whose own bound is carried
    Hm, sd, x = model.head.decoder.pred_hidden, c["sd"], c["x"]
    z = torch.zeros(B, Hm, dtype=torch.float64, device=dev)
    want_p = predict_grads(x, z, z, sd, c["want"][1], z, z)
    carried = predict_grads(x, z, z, sd, c["bounds"][1], z, z, absm=True)
    pb = [p + q for p, q in zip(_predict_bounds(x, z, z, sd, c["want"][1], z, z), carried)]
    dcd = model.head.decoder
    got_p = (dcd.embed.weight.grad, dcd.lstm.weight_ih_l0.grad, dcd.lstm.weight_hh_l0.grad, dcd.lstm.bias_ih_l0.grad)
    worst_p = max(_check_bound(nm, a, want_p[i], pb[i]) for nm, a, i in zip(("d_embed", "dW_ih", "dW_hh", "d_bias"), got_p, (2, 3, 4, 5)))
    print(f"rnnt_loss {name} V1={V1} J={j.joint_net._modules['1'].weight.shape[1]} H={Hm} B={B} T={T} U={U} plan tU={plan['tU']} "
          f"NS={plan['NS']} ST={plan['ST']} (empty {plan['empty']}) S={plan['S']} NC={plan['NC']}: worst err/bound gradients "
          f"{c['worst']:.3g}, operands {c['worst_ops']:.3g}, predict {worst_p:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,U,J", [(2, 9, 64, 196), (1, 700, 7, 20), (2, 9, 0, 4)])
def test_backward_overwrites_every_partial_it_reads(B, T, U, J):
    """gam_rnnt_loss_backward with its workspace and outputs filled with NaN, at plans with two strips (NS = 2), 20 empty
    frame ranges, and S = 1 (the class kernel writes dW / db itself) next to S > 1: every output is finite, within the bound,
    and the same bits as with a zeroed workspace."""
    dev = _dev()
    V1 = 34
    model = _model("v2_rnnt", V1, J=J)
    enc, enc_len, y, tlen = _inputs(B, T, U, V1, seed=B + T + U, dev=dev)
    w = torch.rand(B, generator=torch.Generator(device=dev).manual_seed(5), device=dev) + 0.5
    nan = _gpu_case(model, enc, enc_len, y, tlen, w, fill=0xFF)    # 0xFFFFFFFF is a NaN in every float of the workspace
    zero = _gpu_case(model, enc, enc_len, y, tlen, w, fill=0)
    for a, b in zip(nan["outs"], zero["outs"]):
        assert bool(a.isfinite().all()) and torch.equal(a, b)
    plan = nan["plan"]
    print(f"NaN workspace B={B} T={T} U={U} J={J}: plan NS={plan['NS']} ST={plan['ST']} (empty {plan['empty']}) S={plan['S']}; "
          f"worst err/bound {nan['worst']:.3g}")


@pytest.mark.gpu
def test_untrainable_pred_hidden_keeps_inference():
    """A pred_hidden 640 model runs the prediction network, the joint and the loss without gradients, and refuses a
    gradient through the prediction network before any launch (training only the joint still works)."""
    dev = _dev()
    V1 = 34
    model = _model("v2_rnnt", V1, H=640)
    enc, enc_len, y, tlen = _inputs(2, 9, 3, V1, seed=1, dev=dev)
    with torch.no_grad():
        loss = decoding.rnnt_loss(model.head, enc, enc_len, y, tlen, reduction="none")
        dec, _ = model.head.decoder.predict(y.clamp(0, V1 - 2), None)
        lp = model.head.joint.joint(enc.transpose(1, 2), dec)
    assert bool(loss.isfinite().all()) and bool(lp.isfinite().all()) and dec.shape[-1] == 640
    model.head.requires_grad_(True)
    with pytest.raises(ValueError, match="pred_hidden 640 .*<= 614"):
        decoding.rnnt_loss(model.head, enc, enc_len, y, tlen)
    # greedy transcription is the cluster kernel's, which runs pred_hidden = joint_hidden = 320 only: it refuses this model
    # with its own message, as it did before the training limit existed
    from gigaam_b200._lib import GamError
    with torch.no_grad(), pytest.raises(GamError, match="pred_hidden != joint_hidden"):
        model.decoding.decode(model.head, enc, enc_len)
    model.head.decoder.requires_grad_(False)
    again = decoding.rnnt_loss(model.head, enc, enc_len, y, tlen, reduction="none")
    again.sum().backward()
    assert torch.equal(again.detach(), loss) and bool(model.head.joint.enc.weight.grad.isfinite().all())


def _lattice_route(model, enc, enc_len, y, tlen, w):
    ta = pytest.importorskip("torchaudio.functional")
    V1 = model._get_engine().num_classes
    y_used, x = decoding._rnnt_inputs(model._get_engine(), y, tlen)
    dec, _ = model.head.decoder.predict(x, None)
    lp = model.head.joint.joint(enc.transpose(1, 2), dec)
    yt = torch.where(y_used == V1 - 1, torch.zeros_like(y_used), y_used).int()
    loss = ta.rnnt_loss(lp, yt, enc_len.int(), tlen.int(), blank=V1 - 1, reduction="none", fused_log_softmax=False)
    return loss, (w * loss).sum()


@pytest.mark.gpu
def test_realistic_shape_agrees_with_the_lattice_route():
    """8 x 251 x U 60, V+1 = 1025.  Both routes are fp32 with different summation orders and different lse / occupancy
    arithmetic.  Each occupancy exp(alpha + score + beta - ll) carries the rounding of two T + U step walks over values as
    large as |ll| (thousands of nats for this untrained head), so the two routes' gradients are compared by relative
    Frobenius norm against the random-walk scale of that error, 4 sqrt(T + U) u max|ll|."""
    dev = _dev()
    model = _model("v3_e2e_rnnt", 1025)
    model.head.requires_grad_(True)
    # torchaudio's CUDA loss does not handle a zero-length target, so every utterance here has one (U_b = 0 is held to
    # float64 in test_gradients_against_float64)
    enc, enc_len, y, tlen = _inputs(8, 251, 60, 1025, seed=5, dev=dev, zero_u=False)
    w = torch.ones(8, device=dev)
    runs = []
    for fused in (True, False):
        model.head.zero_grad(set_to_none=True)
        e = enc.clone().requires_grad_(True)
        if fused:
            loss = decoding.rnnt_loss(model.head, e, enc_len, y, tlen, reduction="none")
            (w * loss).sum().backward()
        else:
            loss, total = _lattice_route(model, e, enc_len, y, tlen, w)
            total.backward()
        runs.append((loss.detach(), e.grad, _grads(model)))
    (lf, ef, gf), (ll_, el, gl) = runs
    assert bool(((lf - ll_).abs() <= 1e-4 * (1 + ll_.abs())).all()), (lf, ll_)
    tol = 4 * (251 + 60) ** 0.5 * U32 * float(ll_.abs().max())
    rel = float((ef - el).norm() / el.norm())
    assert rel < tol, f"d_encoded: relative difference {rel:.3g} >= {tol:.3g}"
    for k in gl:
        rel = float((gf[k] - gl[k]).norm() / gl[k].norm().clamp_min(1e-30))
        assert rel < tol, f"{k}: relative difference {rel:.3g} >= {tol:.3g}"
    print(f"lattice route: tolerance {tol:.3g}, largest |loss| {float(ll_.abs().max()):.0f}")


@pytest.mark.gpu
def test_edge_cases():
    dev = _dev()
    V1 = 257
    model = _model("v2_rnnt", V1)
    model.head.requires_grad_(True)
    enc, enc_len, y, tlen = _inputs(5, 40, 8, V1, seed=9, dev=dev)
    enc_len[1] = 0                       # T_b = 0
    enc.requires_grad_(True)

    def run(yy, w):
        model.head.zero_grad(set_to_none=True)
        enc.grad = None
        loss = decoding.rnnt_loss(model.head, enc, enc_len, yy, tlen, reduction="none")
        (w * torch.where(torch.isinf(loss), torch.zeros_like(loss), loss)).sum().backward()
        return loss.detach(), enc.grad.clone(), _grads(model)

    w = torch.ones(5, device=dev)
    loss, ge, gp = run(y, w)
    assert torch.isinf(loss[1]) and loss[1] > 0 and torch.isfinite(loss[[0, 2, 3, 4]]).all()
    assert tlen[-1] == 0 and torch.isfinite(loss[-1])
    assert float(ge[1].abs().sum()) == 0.0
    # +inf contributes nothing: the gradients do not depend on its upstream weight
    w2 = w.clone()
    w2[1] = 3.0
    model.head.zero_grad(set_to_none=True)
    enc.grad = None
    l2 = decoding.rnnt_loss(model.head, enc, enc_len, y, tlen, reduction="none")
    l2.backward(w2)
    assert torch.equal(enc.grad, ge) and all(torch.equal(p.grad, gp[k]) for k, p in model.head.named_parameters())
    # garbage past target_lengths changes nothing
    y2 = y.clone()
    for b in range(5):
        y2[b, int(tlen[b]):] = 3 + b
    loss2, ge2, gp2 = run(y2, w)
    assert torch.equal(loss2, loss) and torch.equal(ge2, ge) and all(torch.equal(gp2[k], gp[k]) for k in gp)
    # a bad id is NaN in its own utterance's loss only
    y3 = y.clone()
    y3[2, 0] = V1 + 5
    with torch.no_grad():
        l3 = decoding.rnnt_loss(model.head, enc, enc_len, y3, tlen, reduction="none")
    assert torch.isnan(l3[2]) and torch.equal(l3[[0, 1, 3, 4]], loss[[0, 1, 3, 4]])


@pytest.mark.gpu
def test_batch_invariance_determinism_and_reductions():
    dev = _dev()
    V1 = 1025
    model = _model("v3_e2e_rnnt", V1)
    enc, enc_len, y, tlen = _inputs(4, 47, 11, V1, seed=2, dev=dev)
    with torch.no_grad():
        full = decoding.rnnt_loss(model.head, enc, enc_len, y, tlen, reduction="none")
        for b in range(4):
            n = int(enc_len[b])
            alone = decoding.rnnt_loss(model.head, enc[b:b + 1, :, :n], enc_len[b:b + 1], y[b:b + 1, :int(tlen[b])],
                                       tlen[b:b + 1], reduction="none")
            assert torch.equal(alone, full[b:b + 1]), (b, alone, full[b])
        assert torch.equal(decoding.rnnt_loss(model.head, enc, enc_len, y, tlen, reduction="sum"), full.sum())
        assert torch.equal(decoding.rnnt_loss(model.head, enc, enc_len, y, tlen, reduction="mean"), full.mean())
    model.head.requires_grad_(True)
    runs = []
    for red in ("sum", "sum", "mean", "none"):
        model.head.zero_grad(set_to_none=True)
        e = enc.clone().requires_grad_(True)
        loss = decoding.rnnt_loss(model.head, e, enc_len, y, tlen, reduction=red)
        (loss if red != "none" else (0.5 * loss).sum()).backward()
        runs.append((e.grad, _grads(model)))
    (e0, g0), (e1, g1), (em, gm), (eh, gh) = runs
    assert torch.equal(e0, e1) and all(torch.equal(g0[k], g1[k]) for k in g0)     # bit-identical on a second call
    # B = 4 and the weight 0.5 are powers of two: the scaled upstream scales every dz exactly, except where a product or a
    # partial sum is subnormal (below 2^-126), whose rounding does not scale
    tiny = 1e-30
    assert float((em - e0 / 4).abs().max()) <= tiny and float((eh - e0 / 2).abs().max()) <= tiny
    for k in g0:
        assert float((gm[k] - g0[k] / 4).abs().max()) <= tiny and float((gh[k] - g0[k] / 2).abs().max()) <= tiny, k


@pytest.mark.gpu
def test_memory_stays_within_the_header_formula():
    """16 x 750 x U 200 on v3_e2e_rnnt: the lattice would be 9.9 GB.  Peak allocation above the inputs must stay within
    saved + the larger workspace + the gradients' own tensors (header formula) plus 256 MiB of slack for the prediction
    network's training buffers, the torch-side prologue and the allocator's rounding."""
    dev = _dev()
    V1, B, T, U = 1025, 16, 750, 200
    model = _model("v3_e2e_rnnt", V1)
    model.head.requires_grad_(True)
    enc, enc_len, _, tlen = _inputs(B, T, U, V1, seed=4, dev=dev)
    enc_len[:] = T
    tlen[:] = U
    y = torch.randint(0, V1 - 1, (B, U), generator=torch.Generator(device=dev).manual_seed(4), device=dev)
    eng = model._get_engine()
    lib, h = eng.lib, eng.handle
    saved = int(lib.gam_rnnt_loss_saved_bytes(h, B, T, U))
    fwd = int(lib.gam_rnnt_loss_workspace_bytes(h, B, T, U))
    bwd = int(lib.gam_rnnt_loss_backward_workspace_bytes(h, B, T, U))
    N, J = B * T * (U + 1), 320
    assert saved + fwd <= 24 * N + 4 * (B * T + B * (U + 1)) * J + 8 * 1024
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    loss = decoding.rnnt_loss(model.head, enc, enc_len, y, tlen)
    loss.backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    allowed = saved + max(fwd, bwd) + 2 * 4 * B * T * 768 + 256 * 2 ** 20
    print(f"rnnt_loss memory: N = {N} nodes, peak {peak / 2 ** 20:.0f} MiB (saved {saved / 2 ** 20:.0f}, forward ws "
          f"{fwd / 2 ** 20:.0f}, backward ws {bwd / 2 ** 20:.0f} MiB); lattice would be {N * V1 * 4 / 1e9:.1f} GB")
    assert peak <= allowed, (peak, allowed)
    assert torch.isfinite(loss)


@pytest.mark.gpu
def test_adamw_steps_match_the_lattice_route_and_greedy_follows():
    dev = _dev()
    from test_head_training import _batch
    models = [_model("v2_rnnt", None, seed=1) for _ in range(2)]
    eng = models[0]._get_engine()
    V1 = eng.num_classes
    enc, enc_len = _batch(models[0], 4, 1.5, seed=3)
    g = torch.Generator().manual_seed(8)
    y = torch.randint(0, V1 - 1, (4, 6), generator=g).to(dev)
    tlen = torch.tensor([6, 5, 6, 3], dtype=torch.int32, device=dev)
    lr = 1e-3
    p0 = {k: p.detach().clone() for k, p in models[0].head.named_parameters()}
    for i, m in enumerate(models):
        m.head.requires_grad_(True)
        opt = torch.optim.AdamW([p for p in m.parameters() if p.requires_grad], lr=lr)
        for _ in range(3):
            opt.zero_grad()
            if i == 0:
                decoding.rnnt_loss(m.head, enc, enc_len, y, tlen).backward()
            else:
                loss, _ = _lattice_route(m, enc, enc_len, y, tlen, torch.ones(4, device=dev))
                loss.mean().backward()
            opt.step()
    for (k, a), (_, b) in zip(models[0].head.named_parameters(), models[1].head.named_parameters()):
        da, db = a.detach() - p0[k], b.detach() - p0[k]
        assert float(db.norm()) > 0, k
        rel = float((da - db).norm() / db.norm())
        # an Adam step normalises each gradient entry: where |g| is near its own rounding the two routes may step apart by
        # up to 2 lr, but over the whole tensor the steps must agree
        assert rel < 0.05, f"{k}: parameter change differs by {rel:.3g}"
        assert float((da - db).abs().max()) <= 6 * lr, k
    with torch.no_grad():
        hyps = [m.decoding.decode(m.head, enc, enc_len) for m in models]
    assert [h[1] for h in hyps[0]] == [h[1] for h in hyps[1]]


@pytest.mark.gpu
def test_engine_forward_and_backward_capture_in_a_cuda_graph():
    dev = _dev()
    V1 = 257
    model = _model("v2_rnnt", V1)
    eng = model._get_engine()
    B, T, U = 3, 30, 7
    enc, enc_len, y, tlen = _inputs(B, T, U, V1, seed=6, dev=dev)
    enc = enc.transpose(1, 2).contiguous()
    y_used, x = decoding._rnnt_inputs(eng, y, tlen)
    with torch.no_grad():
        dec, _ = model.head.decoder.predict(x, None)
    y32, el, tl = y_used.int(), enc_len.int(), tlen.int()
    grad = torch.rand(B, device=dev)

    def step():
        loss, saved = eng.rnnt_loss(enc, dec, y32, el, tl)
        return (loss,) + eng.rnnt_loss_backward(enc, dec, y32, el, tl, saved, grad, True, True, True)

    eager = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(out, eager):
        assert torch.equal(a, b)
