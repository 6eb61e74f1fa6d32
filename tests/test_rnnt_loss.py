"""The fused RNN-T loss (decoding.rnnt_loss; include/gigaam_b200.h, gam_rnnt_loss / gam_rnnt_loss_backward).

CPU: a float64 restatement of the loss (the joint in float64, alpha by logaddexp, gradients by autograd) is itself checked
against torchaudio's rnnt_loss, and the refusals happen before any device work.  GPU: the loss equals -log_likelihood of
decoding.align bit for bit; every head gradient and d_encoded is held to the float64 restatement element by element, with
bounds derived from the arithmetic (see _loss_bounds); realistic shapes agree with the lattice route (joint.joint +
torchaudio); the edge cases, batch invariance, determinism, reductions, the memory formula, training steps and CUDA graph
capture."""
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


def _model(name, V1, seed=0):
    from test_head_training import _model as model_for
    return model_for(name, V1=V1, seed=seed)[0]


def _inputs(B, T, U, V1, seed, dev, zero_u=True):
    g = torch.Generator(device=dev).manual_seed(seed)
    enc = torch.randn(B, 768, T, generator=g, device=dev)
    enc_len, y, tlen = _ragged(B, T, U, V1, seed, zero_u)
    return enc, enc_len.to(dev), y.to(dev), tlen.to(dev)


def _grads(model):
    return {k: p.grad.clone() for k, p in model.head.named_parameters()}


@pytest.mark.gpu
@pytest.mark.parametrize("name,V1", [("v2_rnnt", 34), ("v2_rnnt", 257), ("v3_e2e_rnnt", 1025)])
def test_loss_is_minus_align_log_likelihood_bit_for_bit(name, V1):
    model = _model(name, V1)
    enc, enc_len, y, tlen = _inputs(7, 61, 13, V1, seed=V1, dev=_dev())
    with torch.no_grad():
        ll = decoding.align(model.head, enc, enc_len, y, tlen)[3]
        loss = decoding.rnnt_loss(model.head, enc, enc_len, y, tlen, reduction="none")
    assert torch.isfinite(ll).all()
    assert torch.equal(loss, -ll), (loss, -ll)


def _loss_bounds(e64, d64, sd, lp64, G64, blank, label, alpha, beta, enc_len, tlen, ll):
    """Per-element bounds of (d_enc, d_dec, dW_enc, db_enc, dW_pred, db_pred, dW_out, db_out) of the fused kernels.
    The fused dz equals the lattice route's dlogit for the upstream G = dL/dlog-probs, except that e_blank / e_label come
    from the fp32 alpha / beta walks.  So: _joint_bounds (the joint backward's rounding for that G, test_head_training.py)
    plus the occupancy error carried through the same sums.  Each occupancy exp(alpha + score + beta - ll) has relative
    error at most eps_b: the T_b + U_b + 2 lse2 steps of each walk add a rounding of 4 u times the largest |alpha| + |beta|
    + |ll| of the utterance, and each score read carries its own error (the logit's J-term dot product, the rebuilt hidden
    row and the row lse), summed along the walk."""
    from test_head_training import _joint_bounds, joint_grads
    B, T, U1, V1 = lp64.shape
    J = 320
    Wo, bo = sd["head.joint.joint_net.1.weight"], sd["head.joint.joint_net.1.bias"]
    We, Wp = sd["head.joint.enc.weight"], sd["head.joint.pred.weight"]
    mE = e64.abs() @ We.abs().t() + sd["head.joint.enc.bias"].abs()
    mP = d64.abs() @ Wp.abs().t() + sd["head.joint.pred.bias"].abs()
    hmag = mE[:, :, None, :] + mP[:, None, :, :]
    zmag = hmag @ Wo.abs().t() + bo.abs()
    zerr = (2 * (J + 800) * U32 * zmag + 4 * U32 * (lp64.abs() + 1)).amax(-1)   # [B, T, U1]
    eps = torch.zeros(B, dtype=torch.float64, device=lp64.device)
    for b in range(B):
        Tb, Ub = int(enc_len[b]), int(tlen[b])
        if Tb == 0:
            continue
        a, be = alpha[b, :Tb, :Ub + 1], beta[b, :Tb, :Ub + 1]
        fin = torch.isfinite(a) & torch.isfinite(be)
        M = float((a.abs() + be.abs())[fin].max()) + abs(float(ll[b]))
        eps[b] = (Tb + Ub + 2) * (4 * U32 * M + 2 * float(zerr[b, :Tb, :Ub + 1].max()))
    base = _joint_bounds(e64, d64, sd, lp64, G64)
    occ = joint_grads(e64, d64, sd, lp64, 2 * eps[:, None, None, None] * G64.abs(), absm=True)
    return [x + o for x, o in zip(base, occ)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,V1,B,T,U", [("v2_rnnt", 34, 4, 23, 6), ("v2_rnnt", 257, 3, 17, 9), ("v3_e2e_rnnt", 1025, 3, 13, 5)])
def test_gradients_against_float64(name, V1, B, T, U):
    from test_head_training import _check_bound, _predict_bounds, predict_grads
    dev = _dev()
    model = _model(name, V1)
    model.head.requires_grad_(True)
    enc, enc_len, y, tlen = _inputs(B, T, U, V1, seed=V1 + T, dev=dev)
    enc.requires_grad_(True)
    w = torch.rand(B, generator=torch.Generator(device=dev).manual_seed(3), device=dev) + 0.5
    loss = decoding.rnnt_loss(model.head, enc, enc_len, y, tlen, reduction="none")
    (w * loss).sum().backward()
    # float64 at the GPU's own prediction-network outputs (the same bits rnnt_loss used)
    y_used, x = decoding._rnnt_inputs(model._get_engine(), y, tlen)
    with torch.no_grad():
        dec, _ = model.head.decoder.predict(x, None)
    sd = {f"head.{k}": v.detach().double().to(dev).requires_grad_(True) for k, v in model.head.state_dict().items()}
    e64 = enc.detach().double().transpose(1, 2).contiguous().requires_grad_(True)
    d64 = dec.double().requires_grad_(True)
    lp64, _ = lattice64(e64, d64, sd)
    lp64.retain_grad()
    blank, label = scores64(lp64, y_used)
    loss64, alpha, beta = alpha_beta64(blank, label, enc_len.cpu(), tlen.cpu())
    assert bool(((loss.double() - loss64.detach()).abs() <= 1e-3 * (1 + loss64.detach().abs())).all())
    (w.double() * loss64).sum().backward()
    G64 = lp64.grad.detach()
    bounds = _loss_bounds(e64.detach(), d64.detach(), {k: v.detach() for k, v in sd.items()}, lp64.detach(), G64, blank, label,
                          alpha, beta, enc_len, tlen, -loss64.detach())
    j = model.head.joint
    got = (enc.grad.transpose(1, 2), j.enc.weight.grad, j.enc.bias.grad, j.pred.weight.grad, j.pred.bias.grad,
           j.joint_net._modules["1"].weight.grad, j.joint_net._modules["1"].bias.grad)
    want = (e64.grad, sd["head.joint.enc.weight"].grad, sd["head.joint.enc.bias"].grad, sd["head.joint.pred.weight"].grad,
            sd["head.joint.pred.bias"].grad, sd["head.joint.joint_net.1.weight"].grad, sd["head.joint.joint_net.1.bias"].grad)
    worst = 0.0
    for nm, a, wt, bd in zip(("d_enc", "dW_enc", "db_enc", "dW_pred", "db_pred", "dW_out", "db_out"), got, want,
                             [bounds[0]] + bounds[2:]):
        worst = max(worst, _check_bound(nm, a, wt, bd))
    # the prediction network: its backward (gam_rnnt_predict_backward) from the float64 d_dec, whose own bound is carried
    z = torch.zeros(B, 320, dtype=torch.float64, device=dev)
    sdd = {k: v.detach() for k, v in sd.items()}
    want_p = predict_grads(x, z, z, sdd, d64.grad, z, z)
    carried = predict_grads(x, z, z, sdd, bounds[1], z, z, absm=True)
    pb = [p + c for p, c in zip(_predict_bounds(x, z, z, sdd, d64.grad, z, z), carried)]
    dcd = model.head.decoder
    got_p = (dcd.embed.weight.grad, dcd.lstm.weight_ih_l0.grad, dcd.lstm.weight_hh_l0.grad, dcd.lstm.bias_ih_l0.grad)
    for nm, a, i in zip(("d_embed", "dW_ih", "dW_hh", "d_bias"), got_p, (2, 3, 4, 5)):
        worst = max(worst, _check_bound(nm, a, want_p[i], pb[i]))
    print(f"rnnt_loss {name} V1={V1} B={B} T={T} U={U}: worst err/bound {worst:.3g}")


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
