"""Training the CTC and RNN-T heads on a frozen encoder: the backward passes of csrc/head_grads.cu behind CTCHead.forward,
RNNTJoint.joint and RNNTDecoder.predict, the in-place head repack after optimizer steps, and the refusals.

CPU: this file's float64 gradient restatements equal autograd through the reference's heads, and the RNN-T recipe (zero
embedding start, unfused loss on log-probs) equals the reference fine-tuner's arithmetic.  GPU: each backward against the
float64 restatements with per-element bounds derived from the float64 sum of |terms|, determinism, the forward-only path
left untouched, SGD / AdamW steps against the reference heads, greedy decoding after the repack, and a fine-tuned
checkpoint round trip through the on-disk pack cache."""
import math
import sys

import pytest
import torch
import torch.nn.functional as F

import gigaam_b200 as gigaam
from gigaam_b200 import synthetic
from oracle import ref_loader

U32 = 2.0 ** -24     # unit roundoff of fp32


# ------------------------------------------------------------------------------------------ float64 restatements
# Each returns the gradients and, with absm=True, the same sums over |terms| (the magnitude every fp32 error bound scales with).
def _a(t, absm):
    return t.abs() if absm else t


def softmax_grad(G, logp, absm=False):
    """log_softmax backward: dlogit = G - exp(logp) * sum(G) per row"""
    p = logp.exp()
    if absm:
        return G.abs() + p * G.abs().sum(-1, keepdim=True)
    return G - p * G.sum(-1, keepdim=True)


def ctc_grads(enc, W, b, logp, G, absm=False):
    """enc [B, T, d], W [V1, d], logp / G [B, T, V1] -> (d_enc, dW, db)"""
    dl = softmax_grad(G, logp, absm).reshape(-1, W.shape[0])
    e = _a(enc.reshape(-1, W.shape[1]), absm)
    return (dl @ _a(W, absm)).reshape(enc.shape), dl.t() @ e, dl.sum(0)


def joint_grads(enc, dec, sd, logp, G, absm=False):
    """RNNTJoint.joint backward: enc [B, T, d], dec [B, U, H] -> (d_enc, d_dec, dWe, dbe, dWp, dbp, dWo, dbo)"""
    We, be = sd["head.joint.enc.weight"], sd["head.joint.enc.bias"]
    Wp, bp = sd["head.joint.pred.weight"], sd["head.joint.pred.bias"]
    Wo = sd["head.joint.joint_net.1.weight"]
    E = enc @ We.t() + be
    P = dec @ Wp.t() + bp
    z = E[:, :, None, :] + P[:, None, :, :]
    hid = z.clamp_min(0)
    dl = softmax_grad(G, logp, absm)
    dhid = (dl @ _a(Wo, absm)) * (hid > 0)
    dE, dP = dhid.sum(2), dhid.sum(1)
    J = Wo.shape[1]
    dWo = dl.reshape(-1, Wo.shape[0]).t() @ hid.reshape(-1, J)
    dWe = dE.reshape(-1, J).t() @ _a(enc.reshape(-1, enc.shape[-1]), absm)
    dWp = dP.reshape(-1, J).t() @ _a(dec.reshape(-1, dec.shape[-1]), absm)
    return (dE @ _a(We, absm), dP @ _a(Wp, absm), dWe, dE.sum((0, 1)), dWp, dP.sum((0, 1)), dWo, dl.sum((0, 1, 2)))


def predict_grads(x, h0, c0, sd, gG, gh1, gc1, absm=False):
    """BPTT through RNNTDecoder.predict (1-layer LSTM, blank row of the embedding zero) -> (dh0, dc0, d_embed, dW_ih,
    dW_hh, d_bias)"""
    emb_w = sd["head.decoder.embed.weight"].clone()
    V1, H = emb_w.shape
    emb_w[V1 - 1] = 0
    W_ih, W_hh = sd["head.decoder.lstm.weight_ih_l0"], sd["head.decoder.lstm.weight_hh_l0"]
    bias = sd["head.decoder.lstm.bias_ih_l0"] + sd["head.decoder.lstm.bias_hh_l0"]
    B, U = gG.shape[:2]
    xx = x if x is not None else torch.full((B, 1), V1 - 1, dtype=torch.long, device=gG.device)
    emb = emb_w[xx]
    h, c = h0, c0
    hs, cs, acts = [h0], [c0], []
    for u in range(U):
        gates = emb[:, u] @ W_ih.t() + h @ W_hh.t() + bias
        i, f, g, o = gates.chunk(4, -1)
        i, f, g, o = i.sigmoid(), f.sigmoid(), g.tanh(), o.sigmoid()
        c = f * c + i * g
        h = o * c.tanh()
        hs.append(h)
        cs.append(c)
        acts.append((i, f, g, o))
    m = (lambda t: t.abs()) if absm else (lambda t: t)
    dh_n, dc_n = m(gh1), m(gc1)
    da = [None] * U
    for u in range(U - 1, -1, -1):
        i, f, g, o = acts[u]
        tc = cs[u + 1].tanh()
        dh = m(gG[:, u]) + dh_n
        dc = dc_n + dh * o * (1 - tc * tc)
        da[u] = torch.cat([dc * m(g) * i * (1 - i), dc * m(cs[u]) * f * (1 - f), dc * i * (1 - g * g), dh * m(tc) * o * (1 - o)], -1)
        dh_n = da[u] @ m(W_hh)
        dc_n = dc * f
    A = torch.stack(da, 1).reshape(B * U, 4 * H)
    hp = torch.stack(hs[:-1], 1).reshape(B * U, H)
    dW_hh = A.t() @ m(hp)
    dW_ih = A.t() @ m(emb.reshape(B * U, H))
    cls = torch.zeros(V1, 4 * H, dtype=A.dtype, device=A.device).index_add_(0, xx.reshape(-1), A)
    cls[V1 - 1] = 0
    return dh_n, dc_n, cls @ m(W_ih), dW_ih, dW_hh, A.sum(0)


# ------------------------------------------------------------------------------------------ reference heads (CPU)
def _imported_reference():
    before, path = set(sys.modules), list(sys.path)
    try:
        return ref_loader.import_reference()
    finally:
        for k in set(sys.modules) - before:
            if k.split(".")[0] in ("gigaam", "hydra", "omegaconf", "soundfile"):
                del sys.modules[k]
        sys.path[:] = path


@pytest.fixture(scope="module")
def reference():
    if ref_loader.reference_root() is None:
        pytest.skip("the reference is neither in its source tree nor compiled into oracle/_ref")
    return _imported_reference()


def _head_sd(ck, scale=None, seed=0):
    """Head weights of a synthetic checkpoint, the embedding's blank row zero (nn.Embedding's padding_idx).  `scale`
    rescales the output layer so that rows are far from one-hot (the synthetic joint's logits are 150-250)."""
    sd = {k: v.clone() for k, v in ck["state_dict"].items() if k.startswith("head.")}
    if "head.decoder.embed.weight" in sd:
        sd["head.decoder.embed.weight"][-1] = 0
    if scale is not None:
        g = torch.Generator().manual_seed(seed)
        for k in ("head.joint.joint_net.1.weight", "head.decoder_layers.0.weight"):
            if k in sd:
                sd[k] = torch.randn(sd[k].shape, generator=g) * scale
    return sd


def _ref_head(reference, ck, sd):
    _, _, rd, _ = reference
    head = ck["cfg"]["head"]
    m = rd.CTCHead(head["feat_in"], head["num_classes"]) if head["type"] == "ctc" else rd.RNNTHead(head["decoder"], head["joint"])
    m.load_state_dict({k[len("head."):]: v for k, v in sd.items()}, strict=True)
    return m.double()


def _close(got, want, tol=1e-9):
    scale = max(1.0, float(want.abs().max()))
    return float((got - want).abs().max()) <= tol * scale


def test_ctc_grad_restatement_equals_reference_autograd(reference):
    ck = synthetic.synthetic_checkpoint("v2_ctc", seed=3, n_layers=1)
    sd = {k: v.double() for k, v in _head_sd(ck, scale=0.05).items()}
    ref = _ref_head(reference, ck, sd)
    g = torch.Generator().manual_seed(1)
    enc = torch.randn(3, 768, 17, generator=g, dtype=torch.float64, requires_grad=True)
    lp = ref(enc)
    G = torch.randn(lp.shape, generator=g, dtype=torch.float64)
    lp.backward(G)
    W = sd["head.decoder_layers.0.weight"][..., 0]
    d_enc, dW, db = ctc_grads(enc.detach().transpose(1, 2), W, sd["head.decoder_layers.0.bias"], lp.detach(), G)
    assert _close(d_enc.transpose(1, 2), enc.grad)
    assert _close(dW, ref.decoder_layers[0].weight.grad[..., 0]) and _close(db, ref.decoder_layers[0].bias.grad)


@pytest.mark.parametrize("with_state", [False, True])
def test_rnnt_grad_restatements_equal_reference_autograd(reference, with_state):
    ck = synthetic.synthetic_checkpoint("v2_rnnt", seed=3, n_layers=1)
    sd = {k: v.double() for k, v in _head_sd(ck, scale=0.05).items()}
    ref = _ref_head(reference, ck, sd)
    g = torch.Generator().manual_seed(2)
    B, T, U, V1 = 3, 5, 4, 34
    enc = torch.randn(B, T, 768, generator=g, dtype=torch.float64, requires_grad=True)
    dec = (torch.rand(B, U, 320, generator=g, dtype=torch.float64) * 2 - 1).requires_grad_(True)
    lp = ref.joint.joint(enc, dec)
    G = torch.randn(lp.shape, generator=g, dtype=torch.float64)
    lp.backward(G)
    got = joint_grads(enc.detach(), dec.detach(), sd, lp.detach(), G)
    j = ref.joint
    want = (enc.grad, dec.grad, j.enc.weight.grad, j.enc.bias.grad, j.pred.weight.grad, j.pred.bias.grad,
            j.joint_net[1].weight.grad, j.joint_net[1].bias.grad)
    for a, b in zip(got, want):
        assert _close(a, b)
    # predict: x with blank ids in it, optional state
    x = torch.randint(0, V1, (B, U), generator=g)
    x[0, 1] = V1 - 1
    h0 = torch.randn(1, B, 320, generator=g, dtype=torch.float64, requires_grad=True) if with_state else None
    c0 = torch.randn(1, B, 320, generator=g, dtype=torch.float64, requires_grad=True) if with_state else None
    ref.zero_grad()
    gs, (h1, c1) = ref.decoder.predict(x, (h0, c0) if with_state else None)
    gG, gh, gc = (torch.randn(t.shape, generator=g, dtype=torch.float64) for t in (gs, h1, c1))
    torch.autograd.backward([gs, h1, c1], [gG, gh, gc])
    z = torch.zeros(B, 320, dtype=torch.float64)
    dh0, dc0, d_emb, dW_ih, dW_hh, d_b = predict_grads(x, h0[0].detach() if with_state else z, c0[0].detach() if with_state else z,
                                                       sd, gG, gh[0], gc[0])
    d = ref.decoder
    assert _close(d_emb, d.embed.weight.grad) and _close(dW_ih, d.lstm.weight_ih_l0.grad)
    assert _close(dW_hh, d.lstm.weight_hh_l0.grad) and _close(d_b, d.lstm.bias_ih_l0.grad) and _close(d_b, d.lstm.bias_hh_l0.grad)
    if with_state:
        assert _close(dh0, h0.grad[0]) and _close(dc0, c0.grad[0])


def test_rnnt_recipe_equals_reference_finetuner_arithmetic(reference):
    """predict(cat([blank, tokens])) reproduces lstm(cat[zeros, embed(tokens)]), and rnnt_loss on log-probs with
    fused_log_softmax=False equals the fused call on raw logits (the reference fine-tuner's _rnnt_joint + _rnnt_loss)."""
    ta = pytest.importorskip("torchaudio.functional")
    ck = synthetic.synthetic_checkpoint("v2_rnnt", seed=3, n_layers=1)
    sd = _head_sd(ck, scale=0.05)
    ref = _ref_head(reference, ck, sd).float()
    g = torch.Generator().manual_seed(4)
    B, T, V1 = 2, 9, 34
    tokens = torch.randint(0, V1 - 1, (B, 4), generator=g)
    enc = torch.randn(B, T, 768, generator=g)
    # the reference fine-tuner: LSTM over [zeros ; embed(tokens)], joint on raw logits, fused loss
    emb = torch.cat([torch.zeros(B, 1, 320), ref.decoder.embed(tokens)], 1)
    dec_ref, _ = ref.decoder.lstm(emb.transpose(0, 1))
    dec_ref = dec_ref.transpose(0, 1)
    j = ref.joint
    logits = j.joint_net(j.enc(enc).unsqueeze(2) + j.pred(dec_ref).unsqueeze(1))
    args = (tokens.int(), torch.full((B,), T, dtype=torch.int32), torch.full((B,), 4, dtype=torch.int32))
    loss_ref = ta.rnnt_loss(logits, *args, blank=V1 - 1, reduction="mean")
    # the recipe: predict from a blank first id, joint log-probs, unfused loss
    blank = torch.full((B, 1), V1 - 1, dtype=torch.long)
    dec, _ = ref.decoder.predict(torch.cat([blank, tokens], 1), None)
    assert float((dec - dec_ref).abs().max()) <= 1e-6
    lp = ref.joint.joint(enc, dec)
    loss = ta.rnnt_loss(lp, *args, blank=V1 - 1, reduction="mean", fused_log_softmax=False)
    assert abs(float(loss - loss_ref)) <= 1e-5 * max(1.0, abs(float(loss_ref)))
    # and the two give the same gradient on the logits: unfused loss on log_softmax(logits) vs the fused loss on logits
    z1 = logits.detach().clone().requires_grad_(True)
    ta.rnnt_loss(z1, *args, blank=V1 - 1, reduction="mean").backward()
    z2 = logits.detach().clone().requires_grad_(True)
    ta.rnnt_loss(z2.log_softmax(-1), *args, blank=V1 - 1, reduction="mean", fused_log_softmax=False).backward()
    # both sides evaluate log_softmax in fp32 once (explicitly, or inside the fused kernel): each log-prob is off by at most
    # ~2u (max|z| + log V) of its row.  A lattice gradient is a sum of probability-weighted terms whose exponents are
    # alpha + beta - loss, log-sums along paths of T + U + 1 log-probs, so a row's entries differ by at most a small
    # multiple of (T + U + 1) log-prob errors times the row's sum of |grad|
    lerr = 2 * U32 * (z1.detach().abs().amax(-1, keepdim=True) + math.log(V1))
    bound = 8 * (T + tokens.shape[1] + 1) * lerr * z1.grad.abs().sum(-1, keepdim=True)
    diff = (z1.grad - z2.grad).abs()
    assert bool((diff <= bound).all()), float((diff / bound).max())


def test_encoder_with_grad_is_refused():
    ck = synthetic.synthetic_checkpoint("v2_ctc", n_layers=1)
    model = gigaam.GigaAMASR(ck["cfg"])
    model.load_state_dict(ck["state_dict"])
    model.encoder.requires_grad_(True)
    wav = torch.zeros(1, 16000)
    with pytest.raises(NotImplementedError, match="inference-only"):
        model(wav, torch.tensor([16000]))
    with pytest.raises(NotImplementedError, match="inference-only"):
        model.encoder(torch.zeros(1, 64, 100), torch.tensor([100]))


def test_parameters_stay_frozen_by_default_and_load_state_dict_drops_the_pack_cache_key():
    ck = synthetic.synthetic_checkpoint("v2_rnnt", n_layers=1)
    model = gigaam.GigaAMASR(ck["cfg"])
    assert not any(p.requires_grad for p in model.parameters())
    model.__dict__["_pack_cache_base"] = "/nonexistent/base"
    model.load_state_dict(ck["state_dict"])
    assert model._pack_cache_path() is None


# ------------------------------------------------------------------------------------------ GPU
def _dev():
    return torch.device("cuda", 0)


def _head_ckpt(name, V1=None, J=None, H=None, scale=0.05, seed=0):
    """A 2-layer synthetic checkpoint (V+1 classes, joint_hidden J, pred_hidden H) with a head that is not saturated."""
    from test_head_forward_units import _cfg
    cfg = _cfg(name, V1=V1, J=J, H=H, n_layers=2)
    sd = synthetic.synthetic_state_dict(cfg, seed=seed)
    ck = {"cfg": cfg, "state_dict": sd}
    sd.update(_head_sd(ck, scale=scale, seed=seed))
    return ck


def _model(name, V1=None, scale=0.05, seed=0, J=None, H=None):
    """_head_ckpt's model on the GPU."""
    ck = _head_ckpt(name, V1=V1, J=J, H=H, scale=scale, seed=seed)
    model = gigaam.load_model(name, device=_dev(), checkpoint=ck, fp16_encoder=False)
    return model, ck


def _entropy_min(lp):
    return float(-(lp.double().exp() * lp.double()).sum(-1).min())


def _check(name, got, want, mag, extra=0.0, c=None):
    """|got - want| <= c * u * mag + extra, element by element (mag = float64 sum of |terms|)"""
    bound = c * U32 * mag + extra
    err = (got.double() - want).abs()
    bad = err > bound
    assert not bool(bad.any()), (f"{name}: {int(bad.sum())} elements outside the bound, worst err/bound "
                                 f"{float((err / bound.clamp_min(1e-300)).max()):.3g}")
    return float((err / bound.clamp_min(1e-300)).max())


def _check_bound(name, got, want, bound):
    err = (got.double() - want.to(got.device)).abs()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=got.device)
    bad = err > bound
    ratio = float((err / bound.clamp_min(1e-300)).max())
    assert not bool(bad.any()), f"{name}: {int(bad.sum())} elements outside the bound, worst err/bound {ratio:.3g}"
    return ratio


def _ctc_bounds(e64, W, lp64, G64):
    """Per-element error bounds of (d_enc, dW, db) computed in fp32 from (enc [B, T, d], W, saved log-probs, G)."""
    B, T, V1 = lp64.shape
    d = W.shape[1]
    mag = ctc_grads(e64, W, None, lp64, G64, absm=True)
    # the saved log-probs carry fp32 error: |d exp(logp)| <= p * (|logp error|), logp error <= 2^-22 (|logit| + 1) per row
    pe = (4 * U32 * (lp64.abs().amax(-1, keepdim=True) + 1) * lp64.exp() * G64.abs().sum(-1, keepdim=True)).reshape(-1, V1)
    ext = ((pe @ W.abs()).reshape(B, T, d), pe.t() @ e64.abs().reshape(-1, d), pe.sum(0))
    return [2 * (n + 4) * U32 * m + x for n, m, x in zip((V1, B * T, B * T), mag, ext)]


def _predict_bounds(x, h0, c0, sd, gG, gh1, gc1):
    """Per-element error bounds of the six predict gradients computed in fp32 (BPTT over U steps of H units)."""
    B, U, H = gG.shape
    mag = predict_grads(x, h0, c0, sd, gG, gh1, gc1, absm=True)
    return [(4 * H + 40 * U + B * U) * U32 * m for m in mag]


def _ragged_grad(B, T, U, V1, lens, g, dev):
    """upstream gradient, zero past each utterance's length (T frames and, for the joint, U+1 label positions)"""
    shape = (B, T, V1) if U is None else (B, T, U, V1)
    G = torch.randn(shape, generator=g, device=dev)
    for b, n in enumerate(lens):
        G[b, n:] = 0
    return G


@pytest.mark.gpu
@pytest.mark.parametrize("V1,B,T", [(34, 32, 251), (257, 5, 40), (1025, 3, 17), (34, 1, 5000)])
def test_ctc_backward_against_float64(V1, B, T):
    dev = _dev()
    model, ck = _model("v2_ctc", V1=V1)
    g = torch.Generator(device=dev).manual_seed(V1 + T)
    enc = torch.randn(B, 768, T, generator=g, device=dev).requires_grad_(True)
    model.head.requires_grad_(True)
    lp = model.head(enc)
    lens = [T - (7 * b) % max(1, T // 2) for b in range(B)]
    G = _ragged_grad(B, T, None, V1, lens, g, dev)
    lp.backward(G)
    sd = {k: v.double().to(dev) for k, v in model.head.state_dict().items()}
    W, bb = sd["decoder_layers.0.weight"][..., 0], sd["decoder_layers.0.bias"]
    e64 = enc.detach().double().transpose(1, 2)
    want = ctc_grads(e64, W, bb, lp.detach().double(), G.double())
    bounds = _ctc_bounds(e64, W, lp.detach().double(), G.double())
    got = (enc.grad.transpose(1, 2), model.head.decoder_layers._modules["0"].weight.grad[..., 0], model.head.decoder_layers._modules["0"].bias.grad)
    worst = [_check_bound(nm, a, w, bd) for nm, a, w, bd in zip(("d_enc", "dW", "db"), got, want, bounds)]
    print(f"ctc V1={V1} B={B} T={T}: min row entropy {_entropy_min(lp.detach()):.3f} nats, worst err/bound {max(worst):.3g}")


def _joint_case(model, B, T, U, g, dev):
    enc = torch.randn(B, T, model.head.joint.enc_hidden, generator=g, device=dev).requires_grad_(True)
    dec = (torch.rand(B, U, model.head.joint.pred_hidden, generator=g, device=dev) * 2 - 1).requires_grad_(True)
    lp = model.head.joint.joint(enc, dec)
    return enc, dec, lp


JOINT_CASES = [("v2_rnnt", 34, 32, 251, 7, None), ("v2_rnnt", 257, 4, 60, 100, None), ("v3_e2e_rnnt", 1025, 3, 33, 1, None),
               ("v3_e2e_rnnt", 1025, 2, 19, 100, None), ("v2_rnnt", 34, 3, 21, 5, 4), ("v2_rnnt", 65, 2, 17, 9, 68),
               ("v3_e2e_rnnt", 257, 2, 13, 40, 344)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,V1,B,T,U,J", JOINT_CASES, ids=["-".join(map(str, c[:5])) + (f"-J{c[5]}" if c[5] else "") for c in JOINT_CASES])
def test_joint_backward_against_float64(name, V1, B, T, U, J):
    dev = _dev()
    model, ck = _model(name, V1=V1, J=J)
    model.head.requires_grad_(True)
    g = torch.Generator(device=dev).manual_seed(V1 + T + U)
    enc, dec, lp = _joint_case(model, B, T, U, g, dev)
    lens = [T - (5 * b) % max(1, T // 2) for b in range(B)]
    G = _ragged_grad(B, T, U, V1, lens, g, dev)
    for b in range(B):
        G[b, :, max(1, U - b):] = 0     # label positions past each utterance's transcript
    lp.backward(G)
    sd = {f"head.{k}": v.double().to(dev) for k, v in model.head.state_dict().items()}
    l64, G64 = lp.detach().double(), G.double()
    want = joint_grads(enc.detach().double(), dec.detach().double(), sd, l64, G64)
    j = model.head.joint
    got = (enc.grad, dec.grad, j.enc.weight.grad, j.enc.bias.grad, j.pred.weight.grad, j.pred.bias.grad,
           j.joint_net._modules["1"].weight.grad, j.joint_net._modules["1"].bias.grad)
    bounds = _joint_bounds(enc.detach().double(), dec.detach().double(), sd, l64, G64)
    worst = 0.0
    for i, (a, w, bd) in enumerate(zip(got, want, bounds)):
        worst = max(worst, _check_bound(f"joint grad {i}", a, w, bd))
    print(f"joint V1={V1} J={model.head.joint_cfg['joint_hidden']} B={B} T={T} U={U}: min row entropy {_entropy_min(l64):.3f} nats, "
          f"worst err/bound {worst:.3g}")


def hidden_rows(e64, d64, sd):
    """-> (z, zerr) [B, T, U, J]: the joint's pre-activation E + P in float64 and the bound of its fp32 error.  E and P are
    sgemm_bias_kernel's sums (one fma chain over ascending k, then the bias: depth d + 1 and H + 1); the add is one more
    rounding."""
    We, be = sd["head.joint.enc.weight"], sd["head.joint.enc.bias"]
    Wp, bp = sd["head.joint.pred.weight"], sd["head.joint.pred.bias"]
    d, H = We.shape[1], Wp.shape[1]
    zE, zP = e64 @ We.t() + be, d64 @ Wp.t() + bp
    mE, mP = e64.abs() @ We.abs().t() + be.abs(), d64.abs() @ Wp.abs().t() + bp.abs()
    z = zE[:, :, None, :] + zP[:, None, :, :]
    return z, U32 * ((d + 1) * mE[:, :, None, :] + (H + 1) * mP[:, None, :, :] + z.abs())


def outer_splits(rows, N, Kc):
    """outer_splits of csrc/head_grads.cu: the number of row slices of an outer sum"""
    tiles = -(-N // 64) * -(-Kc // 64)
    S = min(max(-(-264 // tiles), 1), 64)
    return min(S, max(-(-rows // 256), 1))


def outer_depth(rows, N, K):
    """rounding depth of outer_sum_kernel's sums over `rows` (with the bias column): one fma chain over the rows of a slice
    (chunk rows, a multiple of 16), then outer_sum_reduce_kernel's sum of the S slices in order when S > 1"""
    S = outer_splits(rows, N, K + 1)
    chunk = -(-(-(-rows // S)) // 16) * 16
    return min(chunk, rows) + (S if S > 1 else 0)


def dhid_bounds(dl, dl_err, z, zerr, Wo):
    """dhid = (dl W_o) [z > 0] over V1 classes in one fma chain (depth V1): -> (magnitude, error bound) [..., J].  A hidden
    entry whose fp32 pre-activation may sit on the other side of 0 than the float64 one (|z| <= zerr) may flip its ReLU
    mask: its whole |dl| . |W_o| term may be present on one side only."""
    V1 = Wo.shape[0]
    full = dl @ Wo.abs()
    mask, amb = z > 0, z.abs() <= zerr
    err = ((dl_err + V1 * U32 * dl) @ Wo.abs()) * mask + full * amb
    print(f"joint: {int(amb.sum())} of {amb.numel()} hidden entries within fp32 rounding of 0")
    return full * (mask | amb), err


def joint_input_bounds(e64, d64, sd, dE, dE_err, dP, dP_err):
    """Bounds of (d_enc, d_dec, dW_enc, db_enc, dW_pred, db_pred) as joint_input_grads (gam_api.cu) forms them from dE
    [B, T, J] / dP [B, U, J] given as their float64 sums of |terms| and the bounds of their own errors: d_enc = dE W_e and
    d_dec = dP W_p are matmul_kernel's J-deep fma chains, the weight gradients outer sums over B T and B U rows."""
    We, Wp = sd["head.joint.enc.weight"], sd["head.joint.pred.weight"]
    J, d, H = We.shape[0], We.shape[1], Wp.shape[1]
    e, x = e64.abs().reshape(-1, d), d64.abs().reshape(-1, H)
    E, Ee, P, Pe = dE.reshape(-1, J), dE_err.reshape(-1, J), dP.reshape(-1, J), dP_err.reshape(-1, J)
    kE, kP = outer_depth(E.shape[0], J, d), outer_depth(P.shape[0], J, H)
    return [dE_err @ We.abs() + J * U32 * (dE @ We.abs()), dP_err @ Wp.abs() + J * U32 * (dP @ Wp.abs()),
            Ee.t() @ e + kE * U32 * (E.t() @ e), Ee.sum(0) + kE * U32 * E.sum(0),
            Pe.t() @ x + kP * U32 * (P.t() @ x), Pe.sum(0) + kP * U32 * P.sum(0)]


def _joint_bounds(e64, d64, sd, l64, G64):
    """Per-element bounds of the eight joint gradients computed in fp32 from (enc, dec, saved log-probs, G) by
    gam_rnnt_joint_backward, each a sum evaluated at depth k within k u sum|terms| (test_kernel_units.py's rule):
      dl = G - exp(logp) sum(G): the warp-strided row sum (depth <= V1), expf (2 ulp = 4 u), the product and the difference;
      dhid = dl W_o: depth V1 (dhid_bounds, with the ReLU flips);
      dE = sum over U label positions, dP = sum over T frames: segment_sum_kernel, depth U and T;
      dW_out / db_out: outer_sum_joint over B T U rows, whose rebuilt hidden entries carry hidden_rows' error;
      the rest: joint_input_bounds."""
    B, T, U, V1 = l64.shape
    Wo = sd["head.joint.joint_net.1.weight"]
    J = Wo.shape[1]
    z, zerr = hidden_rows(e64, d64, sd)
    dl = softmax_grad(G64, l64, True)
    dl_err = (V1 + 6) * U32 * dl
    dh, dh_err = dhid_bounds(dl, dl_err, z, zerr, Wo)
    dE, dE_err = dh.sum(2), dh_err.sum(2) + U * U32 * dh.sum(2)
    dP, dP_err = dh.sum(1), dh_err.sum(1) + T * U32 * dh.sum(1)
    hid = z.clamp_min(0).reshape(-1, J)
    kO = outer_depth(B * T * U, V1, J)
    dl2, dle2 = dl.reshape(-1, V1), dl_err.reshape(-1, V1)
    dWo = dle2.t() @ hid + dl2.t() @ zerr.reshape(-1, J) + kO * U32 * (dl2.t() @ hid)
    dbo = dle2.sum(0) + kO * U32 * dl2.sum(0)
    ins = joint_input_bounds(e64, d64, sd, dE, dE_err, dP, dP_err)
    return ins + [dWo, dbo]


@pytest.mark.gpu
def test_joint_backward_past_2_31_lattice_elements():
    dev = _dev()
    model, _ = _model("v3_e2e_rnnt")
    model.head.requires_grad_(True)
    B, T, U, V1 = 2, 1100, 960, 1025       # 2 * 1100 * 960 * 1025 = 2.16e9 > 2^31 elements
    assert B * T * U * V1 > 2 ** 31
    g = torch.Generator(device=dev).manual_seed(5)
    enc = torch.randn(B, T, 768, generator=g, device=dev)
    dec = (torch.rand(B, U, 320, generator=g, device=dev) * 2 - 1)
    lp = model.head.joint.joint(enc, dec.requires_grad_(True))
    G = torch.zeros_like(lp)
    G[-1, -1, -1] = torch.randn(V1, generator=g, device=dev)      # one upstream row, at the far end of the lattice
    g_row = G[-1, -1, -1].clone()
    lp.backward(G)
    del G
    # only lattice row (B-1, T-1, U-1) has an upstream gradient: its d_dec row is the float64 restatement of that one row
    sd = {f"head.{k}": v.double().to(dev) for k, v in model.head.state_dict().items()}
    lp_row = lp.detach()[-1:, -1:, -1:].double()
    args = (enc[-1:, -1:].double(), dec.detach()[-1:, -1:].double(), sd, lp_row, g_row.double().view(1, 1, 1, V1))
    del lp
    want, mag = joint_grads(*args)[1], joint_grads(*args, absm=True)[1]
    nz = dec.grad.abs().sum(-1) > 0
    assert bool(nz[-1, -1]) and int(nz.sum()) == 1
    # depths: dl (V1 + 6, as _joint_bounds), dhid (V1), dP over the T frames, d_dec = dP W_p (J)
    J = model.head.joint_cfg["joint_hidden"]
    _check("d_dec past 2^31", dec.grad[-1:, -1:], want, mag, c=2 * V1 + 6 + T + J, extra=4 * U32 * mag.abs().amax())


PREDICT_CASES = [(1, False, False, 320), (1, True, True, 320), (7, True, True, 320), (100, False, True, 320), (100, True, True, 320),
                 (9, True, True, 16), (9, True, True, 72), (9, True, True, 614)]


@pytest.mark.gpu
@pytest.mark.parametrize("U,with_state,with_x,H", PREDICT_CASES,
                         ids=["-".join(map(str, c[:3])) + (f"-H{c[3]}" if c[3] != 320 else "") for c in PREDICT_CASES])
def test_predict_backward_against_float64(U, with_state, with_x, H):
    """H = 72 is one 64-unit block with an 8-unit tail; H = 614 is the widest the backward runs
    (GAM_PREDICT_BACKWARD_MAX_HIDDEN: 49 120 of the 49 152 bytes of shared memory)."""
    dev = _dev()
    model, ck = _model("v2_rnnt", H=None if H == 320 else H)
    model.head.requires_grad_(True)
    B, V1 = 13, 34
    g = torch.Generator(device=dev).manual_seed(U + 2 * with_state)
    x = torch.randint(0, V1, (B, U), generator=g, device=dev) if with_x else None
    if with_x:
        x[0, 0] = V1 - 1        # blank ids: zero embedding, no embedding gradient
        x[1, U // 2] = V1 - 1
    h0 = (torch.randn(1, B, H, generator=g, device=dev) * 0.5).requires_grad_(True) if with_state else None
    c0 = (torch.randn(1, B, H, generator=g, device=dev) * 0.5).requires_grad_(True) if with_state else None
    gs, (h1, c1) = model.head.decoder.predict(x, (h0, c0) if with_state else None, batch_size=B)
    gG, gh, gc = (torch.randn(t.shape, generator=g, device=dev) for t in (gs, h1, c1))
    torch.autograd.backward([gs, h1, c1], [gG, gh, gc])
    sd = {f"head.{k}": v.double().to(dev) for k, v in model.head.state_dict().items()}
    z = torch.zeros(B, H, dtype=torch.float64, device=dev)
    hh = h0[0].detach().double() if with_state else z
    cc = c0[0].detach().double() if with_state else z
    args = (x, hh, cc, sd, gG.double(), gh[0].double(), gc[0].double())
    want, bounds = predict_grads(*args), _predict_bounds(*args)
    d = model.head.decoder
    got = [h0.grad[0] if with_state else None, c0.grad[0] if with_state else None, d.embed.weight.grad, d.lstm.weight_ih_l0.grad,
           d.lstm.weight_hh_l0.grad, d.lstm.bias_ih_l0.grad]
    assert torch.equal(d.lstm.bias_ih_l0.grad, d.lstm.bias_hh_l0.grad)
    assert not bool(d.embed.weight.grad[V1 - 1].any())
    worst = 0.0
    for i, (a, w, bd) in enumerate(zip(got, want, bounds)):
        if a is not None:
            worst = max(worst, _check_bound(f"predict grad {i}", a, w, bd))
    print(f"predict H={H} U={U} state={with_state} x={with_x}: worst err/bound {worst:.3g}")


@pytest.mark.gpu
def test_predict_backward_out_of_range_id_stays_in_its_utterance():
    dev = _dev()
    model, _ = _model("v2_rnnt")
    B, U, H = 4, 5, 320
    g = torch.Generator(device=dev).manual_seed(9)
    x = torch.randint(0, 33, (B, U), generator=g, device=dev)
    x[2, 3] = 99
    h0 = torch.randn(1, B, H, generator=g, device=dev).requires_grad_(True)
    c0 = torch.randn(1, B, H, generator=g, device=dev).requires_grad_(True)
    gs, (h1, c1) = model.head.decoder.predict(x, (h0, c0))
    gs.sum().backward()
    bad = torch.zeros(B, dtype=torch.bool)
    bad[2] = True
    for t in (h0.grad[0], c0.grad[0]):
        assert bool(t[2].isnan().all()) and bool(t[~bad.to(dev)].isfinite().all())


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v2_rnnt"])
def test_backward_is_deterministic_and_forward_only_path_is_untouched(name):
    dev = _dev()
    model, _ = _model(name)
    g = torch.Generator(device=dev).manual_seed(3)
    enc = torch.randn(4, 768, 30, generator=g, device=dev)
    x = torch.randint(0, 33, (4, 6), generator=g, device=dev)

    def run():
        if name == "v2_ctc":
            return model.head(enc)
        dec, _ = model.head.decoder.predict(x, None)
        return model.head.joint(enc, dec.transpose(1, 2))
    with torch.inference_mode():
        ref_out = run()
    with torch.no_grad():
        assert torch.equal(run(), ref_out)
    out = run()                      # grad enabled, nothing requires grad: forward-only path
    assert out.grad_fn is None and torch.equal(out, ref_out)
    model.head.requires_grad_(True)
    grads = []
    for _ in range(2):
        model.head.zero_grad(set_to_none=True)
        out = run()
        assert out.grad_fn is not None and torch.equal(out.detach(), ref_out)
        (out * torch.linspace(-1, 1, out.shape[-1], device=dev)).sum().backward()
        grads.append([p.grad.clone() for p in model.head.parameters()])
    for a, b in zip(*grads):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------ GPU: training
def _batch(model, B, seconds, seed):
    wav, wav_len = synthetic.synthetic_audio(B, seconds, seed=seed, ragged=True)
    with torch.no_grad():
        enc, enc_len = model(wav.to(_dev()), wav_len.to(_dev()))
    return enc.detach(), enc_len


def _targets(B, V1, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, V1 - 1, (B, n), generator=g)


def _ctc_loss(lp, enc_len, tgt, V1):
    n = torch.full((tgt.shape[0],), tgt.shape[1], dtype=torch.long)
    return F.ctc_loss(lp.transpose(0, 1), tgt, enc_len.long().cpu(), n, blank=V1 - 1, reduction="none", zero_infinity=True).mean()


def _rnnt_loss(head, enc, enc_len, tgt, V1, ta):
    B = tgt.shape[0]
    blank = torch.full((B, 1), V1 - 1, dtype=torch.long, device=tgt.device)
    dec, _ = head.decoder.predict(torch.cat([blank, tgt], 1), None)
    lp = head.joint.joint(enc, dec).float()      # torchaudio's loss takes fp32 log-probs (the float64 reference casts here)
    n = torch.full((B,), tgt.shape[1], dtype=torch.int32, device=tgt.device)
    return ta.rnnt_loss(lp, tgt.int(), enc_len.int().to(tgt.device), n, blank=V1 - 1, reduction="mean", fused_log_softmax=False)


def _sync(ref, model):
    """the float64 reference head takes the GPU head's current parameters"""
    with torch.no_grad():
        for (k, p), (kr, pr) in zip(model.head.named_parameters(), ref.named_parameters()):
            assert k == kr
            pr.copy_(p.detach().cpu().double())


def _reference_greedy(reference, ck, ref, enc, enc_len, V1, name):
    """The reference's greedy decode (CTC: argmax + collapse of CTCHead's log-probs; RNN-T: its RNNTGreedyDecoding) with
    the reference head in fp32 on the CPU -> token ids per utterance"""
    with torch.no_grad():
        if "ctc" in name:
            lab = ref.float()(enc.cpu().float()).argmax(-1)
            out = []
            for b in range(lab.shape[0]):
                seq, prev = [], None
                for t in range(int(enc_len[b])):
                    k = int(lab[b, t])
                    if k != V1 - 1 and k != prev:
                        seq.append(k)
                    prev = k
                out.append(seq)
            return out
        _, _, _, rdec = reference
        rd = rdec.RNNTGreedyDecoding(ck["cfg"]["decoding"]["vocabulary"])
        return [h[1] for h in rd.decode(ref.float(), enc.cpu().float(), enc_len.cpu())]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v2_rnnt", "v3_e2e_rnnt"])
def test_sgd_steps_track_the_reference_head_in_float64(reference, name):
    """Five SGD steps.  At every step the float64 reference head (the reference's own module) holds the GPU head's
    parameters and receives the same upstream gradients (dL/dlog-probs, and for RNN-T dL/d(prediction outputs)), so each
    parameter after the step must equal p - lr * g_ref within lr * (the gradient's derived per-element bound) plus the
    rounding of the fp32 update."""
    ta = pytest.importorskip("torchaudio.functional")
    dev = _dev()
    model, ck = _model(name)
    V1 = ck["cfg"]["head"]["num_classes"] if "ctc" in name else ck["cfg"]["head"]["joint"]["num_classes"]
    B = 3
    enc, enc_len = _batch(model, B, 1.5, seed=11)
    tgt = _targets(B, V1, 5, seed=1)
    ref = _ref_head(reference, ck, {f"head.{k}": v.detach().cpu() for k, v in model.head.state_dict().items()})
    model.head.requires_grad_(True)
    lr = 1e-3
    opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=lr)
    e64 = enc.detach().double().cpu()
    worst = 0.0
    for step in range(5):
        _sync(ref, model)
        ref.zero_grad()
        opt.zero_grad()
        sd = {f"head.{k}": v.detach().double() for k, v in ref.state_dict().items()}
        if "ctc" in name:
            lp = model.head(enc)
            lp.retain_grad()
            _ctc_loss(lp.cpu(), enc_len, tgt, V1).backward()
            G = lp.grad.double().cpu()
            ref(e64).backward(G)
            W = sd["head.decoder_layers.0.weight"][..., 0]
            _, bW, bb = _ctc_bounds(e64.transpose(1, 2), W, lp.detach().double().cpu(), G)
            bounds = {"decoder_layers.0.weight": bW[..., None], "decoder_layers.0.bias": bb}
        else:
            blank = torch.full((B, 1), V1 - 1, dtype=torch.long)
            x = torch.cat([blank, tgt], 1)
            dec, _ = model.head.decoder.predict(x.to(dev), None)
            dec.retain_grad()
            lp = model.head.joint.joint(enc.transpose(1, 2), dec)
            lp.retain_grad()
            n = torch.full((B,), tgt.shape[1], dtype=torch.int32, device=dev)
            ta.rnnt_loss(lp, tgt.int().to(dev), enc_len.int(), n, blank=V1 - 1, reduction="mean",
                         fused_log_softmax=False).backward()
            G, gdec = lp.grad.double().cpu(), dec.grad.double().cpu()
            d64 = dec.detach().double().cpu()
            ref.joint.joint(e64.transpose(1, 2), d64).backward(G)           # the reference joint at the GPU's inputs
            g_ref, _ = ref.decoder.predict(x, None)
            g_ref.backward(gdec)                                               # the reference LSTM, same upstream gradient
            jb = _joint_bounds(e64.transpose(1, 2), d64, sd, lp.detach().double().cpu(), G)
            z = torch.zeros(B, 320, dtype=torch.float64)
            pb = _predict_bounds(x, z, z, sd, gdec, z, z)
            bounds = {"joint.enc.weight": jb[2], "joint.enc.bias": jb[3], "joint.pred.weight": jb[4], "joint.pred.bias": jb[5],
                      "joint.joint_net.1.weight": jb[6], "joint.joint_net.1.bias": jb[7], "decoder.embed.weight": pb[2],
                      "decoder.lstm.weight_ih_l0": pb[3], "decoder.lstm.weight_hh_l0": pb[4], "decoder.lstm.bias_ih_l0": pb[5],
                      "decoder.lstm.bias_hh_l0": pb[5]}
        old = {k: p.detach().cpu().double().clone() for k, p in model.head.named_parameters()}
        opt.step()
        for (k, p), (_, pr) in zip(model.head.named_parameters(), ref.named_parameters()):
            want = old[k] - lr * pr.grad
            new = p.detach().cpu().double()
            # the gradient's bound, and the fp32 rounding of p - lr * g (one product, one sum)
            bound = lr * (bounds[k] + 2 * U32 * pr.grad.abs()) + U32 * new.abs()
            worst = max(worst, _check_bound(f"step {step}: {k}", new, want, bound))
    print(f"{name}: 5 SGD steps, worst err/bound {worst:.3g}")
    # greedy decoding with the trained head (the repacked device weights) equals the reference greedy loop
    _sync(ref, model)
    hyps = model.decoding.decode(model.head, enc, enc_len)
    assert [h[1] for h in hyps] == _reference_greedy(reference, ck, ref, enc, enc_len, V1, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v2_rnnt"])
def test_greedy_decoding_follows_the_trained_head(reference, name):
    """Steps large enough to change the hypotheses: the greedy kernels (which read the packed head) must move with the
    parameters and agree with the reference's greedy decode of the trained reference head."""
    ta = pytest.importorskip("torchaudio.functional")
    dev = _dev()
    model, ck = _model(name)
    V1 = ck["cfg"]["head"]["num_classes"] if "ctc" in name else ck["cfg"]["head"]["joint"]["num_classes"]
    enc, enc_len = _batch(model, 3, 1.5, seed=14)
    tgt = _targets(3, V1, 6, seed=5)
    before = [h[1] for h in model.decoding.decode(model.head, enc, enc_len)]
    model.head.requires_grad_(True)
    opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=0.05)
    for _ in range(10):
        opt.zero_grad()
        if "ctc" in name:
            loss = _ctc_loss(model.head(enc).cpu(), enc_len, tgt, V1)
        else:
            loss = _rnnt_loss(model.head, enc.transpose(1, 2), enc_len, tgt.to(dev), V1, ta)
        loss.backward()
        opt.step()
    after = [h[1] for h in model.decoding.decode(model.head, enc, enc_len)]
    assert after != before, "training did not change the hypotheses: the test would not see a stale head"
    ref = _ref_head(reference, ck, {f"head.{k}": v.detach().cpu() for k, v in model.head.state_dict().items()})
    assert after == _reference_greedy(reference, ck, ref, enc, enc_len, V1, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v2_rnnt"])
def test_adamw_with_reference_settings_lowers_the_loss(name):
    ta = pytest.importorskip("torchaudio.functional")
    dev = _dev()
    model, ck = _model(name)
    V1 = ck["cfg"]["head"]["num_classes"] if "ctc" in name else ck["cfg"]["head"]["joint"]["num_classes"]
    enc, enc_len = _batch(model, 4, 1.5, seed=12)
    tgt = _targets(4, V1, 5, seed=2)
    model.head.requires_grad_(True)
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4, weight_decay=1e-3)
    losses = []
    for _ in range(20):
        opt.zero_grad()
        if "ctc" in name:
            loss = _ctc_loss(model.head(enc).cpu(), enc_len, tgt, V1)
        else:
            loss = _rnnt_loss(model.head, enc.transpose(1, 2), enc_len, tgt.to(dev), V1, ta)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < losses[0], losses


@pytest.mark.gpu
def test_finetuned_checkpoint_round_trip_ignores_the_base_pack_cache(tmp_path):
    dev = _dev()
    ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=2)
    torch.save(ck, tmp_path / "v2_ctc.ckpt")
    base = gigaam.load_model("v2_ctc", device=dev, download_root=str(tmp_path))
    enc, enc_len = _batch(base, 2, 1.5, seed=13)
    assert len(list(tmp_path.glob("v2_ctc.*.b200pack"))) == 1      # the base model's pack cache exists
    base.head.requires_grad_(True)
    opt = torch.optim.SGD(base.head.parameters(), lr=5.0)
    tgt = _targets(2, 34, 6, seed=3)
    for _ in range(3):
        opt.zero_grad()
        _ctc_loss(base.head(enc).cpu(), enc_len, tgt, 34).backward()
        opt.step()
    trained = base.decoding.decode(base.head, enc, enc_len)
    path = tmp_path / "finetuned.ckpt"
    torch.save({"hyper_parameters": {"model_name": "v2_ctc"}, "state_dict": {k: v.detach().cpu() for k, v in base.state_dict().items()}},
               path)
    loaded = gigaam.load_model(str(path), device=dev, download_root=str(tmp_path))
    assert loaded.decoding.decode(loaded.head, enc, enc_len) == trained
    for k, v in loaded.head.state_dict().items():
        assert torch.equal(v.cpu(), base.head.state_dict()[k].detach().cpu())


def _train(model, name, enc, enc_len, tgt, V1, lr, steps):
    ta = pytest.importorskip("torchaudio.functional")
    model.head.requires_grad_(True)
    opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=lr)
    for _ in range(steps):
        opt.zero_grad()
        if "ctc" in name:
            loss = _ctc_loss(model.head(enc).cpu(), enc_len, tgt, V1)
        else:
            loss = _rnnt_loss(model.head, enc.transpose(1, 2), enc_len, tgt.to(_dev()), V1, ta)
        loss.backward()
        opt.step()
    model.head.requires_grad_(False)


@pytest.mark.gpu
@pytest.mark.parametrize("name,lr,steps", [("v2_ctc", 5.0, 3), ("v2_rnnt", 0.05, 10)])
def test_rebuilt_engine_keeps_the_trained_head_and_the_pack_cache_never_holds_it(tmp_path, name, lr, steps):
    """A model loaded from a checkpoint file (so with a pack cache) is trained, then its engine is rebuilt by `.to()`
    (cache hit) and `.float()` (cache miss, a new cache file is written).  Decoding keeps the trained head every time, the
    existing cache files do not change, and a fresh load from the cache decodes as the untrained checkpoint.  A head
    changed in place before the first engine build is used as well."""
    dev = _dev()
    ck = synthetic.synthetic_checkpoint(name, seed=0, n_layers=2)
    V1 = ck["cfg"]["head"]["num_classes"] if "ctc" in name else ck["cfg"]["head"]["joint"]["num_classes"]
    torch.save(ck, tmp_path / f"{name}.ckpt")
    model = gigaam.load_model(name, device=dev, download_root=str(tmp_path))
    enc, enc_len = _batch(model, 3, 1.5, seed=15)
    untrained = model.decoding.decode(model.head, enc, enc_len)
    files = {p: p.read_bytes() for p in tmp_path.glob("*.b200pack")}
    assert len(files) == 1
    _train(model, name, enc, enc_len, _targets(3, V1, 6, seed=6), V1, lr, steps)
    trained = model.decoding.decode(model.head, enc, enc_len)
    assert trained != untrained
    model.to(dev)                                       # engine rebuilt from the cache
    assert model.decoding.decode(model.head, enc, enc_len) == trained and model._get_engine().pack_cache_hit
    model.float()                                       # another dtype: a cache miss, a new file is written
    assert model.decoding.decode(model.head, enc, enc_len) == trained and not model._get_engine().pack_cache_hit
    assert all(p.read_bytes() == b for p, b in files.items())
    assert len(list(tmp_path.glob("*.b200pack"))) == 2
    fresh = gigaam.load_model(name, device=dev, download_root=str(tmp_path), fp16_encoder=False)
    assert fresh.decoding.decode(fresh.head, enc, enc_len) == untrained and fresh._get_engine().pack_cache_hit
    # a head changed in place before the first engine build of a model loaded from the cache
    again = gigaam.load_model(name, device=dev, download_root=str(tmp_path))
    with torch.no_grad():
        for p, q in zip(again.head.parameters(), model.head.parameters()):
            p.copy_(q)
    assert again.decoding.decode(again.head, enc, enc_len) == trained and again._get_engine().pack_cache_hit
