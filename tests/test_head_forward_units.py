"""The heads' forward kernels one at a time against float64: ctc_log_probs_kernel and rnnt_joint_kernel (lattice and
gather) of csrc/heads.cu, sgemm_bias_kernel of csrc/rnnt.cu (the joint's two projections and the greedy path's encoder
projection) and lstm_step_kernel (predict).  test_head_forward.py compares them with an fp32 restatement at the shipped
shapes under absolute tolerances; here every element is held to a worst-case bound derived from the arithmetic, at the
tile edges of each kernel, and the non-finite rows follow torch.

Each reference is computed in float64 from the kernel's own fp32 operands: the packed head buffers the library reads
(Engine._head_bufs), the projections E / P the lattice kernel read (the joint's workspace), the previous step's h and c
of the LSTM.  Bounds use u = 2^-24 (fp32 unit roundoff) and gamma(n) = n u / (1 - n u):
  * logit (CTC, joint) and projection: a K-step fp32 FMA chain plus the bias add, |v - z| <= gamma(K + 1) (sum |w x| + |b|).
    The joint's hidden entry is relu(fl(E + P)), one more rounding of every term: gamma(J + 2) (sum |W_o| hid + |b_o|).
  * log-sum-exp lse = m + logf(s), s = sum exp(v - m) kept as a running (max, sum) per thread and merged across threads:
      - the largest logit error of the row (the log-sum-exp is 1-Lipschitz in the max norm);
      - s: each term leaves its push through one expf (2 ulp = 4u, CUDA Math API; the build has no --use_fast_math) of a
        rounded difference, then goes through at most k + g more rescales (expf and a product) and adds, k = classes per
        thread, g = merges.  Its relative error is <= u (M - v) + 6u (k + g + 1); weighted by the terms, sum p (M - v) <=
        log(V+1), so |log s~ - log s| <= u (log(V+1) + 6 (k + g + 1));
      - logf at 1 ulp: 2u log(V+1); the add m + log s: u |lse|.
  * the final subtraction v - lse: u |out|.
  * LSTM step: gate = fl(acc + emb_gates[id]), gamma(H + 1) (sum |W_hh h| + |emb_gates|); sigmoid 1 / (1 + expf(-x)) with
    |sigmoid'| <= 1/4 and 6u relative (expf, add, div); tanhf at 2 ulp (4u relative) with |tanh'| <= 1; c' and h' add
    their products' errors plus 2u and u of rounding.
All bounds are first order; a factor 1.001 covers the second-order terms.  A worst-case bound cannot fail by chance on a
correct kernel, so a relative Frobenius check (F32_FRO) is added over every output to catch small systematic errors.
Each case prints its worst err/bound and, for log-probs, the minimum row entropy: the synthetic heads' joint logits are
150-250 (near one-hot rows), the unsaturated heads (_head_sd(scale=0.05)) give rows far from one-hot.

Non-finite rows: torch.log_softmax gives -inf at a -inf logit and finite log-probs elsewhere, and all NaN for a row with a
NaN or +inf logit (or with every logit -inf).  The kernels must put NaN and +-inf at exactly the positions of float64
torch.log_softmax of the float64 logits, and keep the other entries within their bound.

The CPU tests at the end are negative controls: float64 emulations of plausible kernel faults, and float32 emulations of
the running log-sum-exp with the kernels' tiling, must be rejected by the same checkers."""
import math

import numpy as np
import pytest
import torch

import gigaam_b200 as gigaam
from gigaam_b200 import synthetic
from test_head_training import _head_sd
from test_kernel_units import F32_FRO, U, _assert_within, _rel_fro

INF, NAN = float("inf"), float("nan")
JOINT_MAX_HIDDEN = 736   # rnnt_joint_max_hidden(): the largest J % 16 == 0 with (J + 16) * 68 * 4 bytes <= 200 KiB
UNSAT = 0.05             # _head_sd scale of the unsaturated head
# (threads per row, classes per thread per tile, merges) of the two log-softmax kernels
CTC_TILING = (4, 9, 3)
JOINT_TILING = (16, 4, 4)


def gamma(n):
    return n * U / (1 - n * U)


def _per_thread(V1, tiling):
    threads, width, _ = tiling
    return width * -(-V1 // (threads * width))


# ------------------------------------------------------------------------------------------ checkers
def _nonfinite_equal(name, got, want):
    for what, f in (("NaN", torch.isnan), ("+inf", lambda t: t == INF), ("-inf", lambda t: t == -INF)):
        mg, mw = f(got), f(want)
        if not torch.equal(mg, mw):
            idx = tuple((mg != mw).nonzero()[0].tolist())
            raise AssertionError(f"{name}: {int((mg != mw).sum())} entries differ from float64 log_softmax in where {what} "
                                 f"sits; first at {idx}: got {float(got[idx])!r}, want {float(want[idx])!r}")


def check_log_probs(name, got, z, e, tiling):
    """got: a kernel's fp32 log-probs [..., V+1]; z: float64 logits from the kernel's fp32 operands; e: the bound of the
    kernel's fp32 logit error (read only where z is finite).  Returns (worst err/bound, relative Frobenius error, minimum
    row entropy in nats)."""
    V1 = z.shape[-1]
    got = got.to(z.device).double()
    want = torch.log_softmax(z, -1)
    _nonfinite_equal(name, got, want)
    ec = torch.where(torch.isfinite(z), e, torch.zeros_like(e))
    emax = ec.amax(-1, keepdim=True)
    k, g = _per_thread(V1, tiling), tiling[2]
    lse = torch.logsumexp(torch.nan_to_num(z, nan=0.0, posinf=0.0), -1, keepdim=True)
    dl = emax + U * (3 * math.log(V1) + 6 * (k + g + 1)) + U * lse.abs()
    bound = 1.001 * (ec + dl + U * (want.abs() + ec + dl))
    fin = torch.isfinite(want)
    if not bool(fin.any()):
        return 0.0, 0.0, float("nan")
    _assert_within(got[fin], want[fin], bound[fin], name)
    worst = float(((got - want).abs()[fin] / bound[fin]).max())
    fro = _rel_fro(got[fin], want[fin])
    assert fro <= F32_FRO, f"{name}: relative Frobenius error {fro:.3g} > {F32_FRO}"
    rows = fin.all(-1)
    ent = -(want.exp() * want).sum(-1)[rows]
    return worst, fro, float(ent.min()) if ent.numel() else float("nan")


def ctc_logits(enc, W, b):
    """enc [R, d], W [V+1, d], b [V+1] fp32 -> float64 logits and the bound of the kernel's logit error"""
    x, w, bb = enc.double(), W.double(), b.double()
    return x @ w.t() + bb, gamma(x.shape[-1] + 1) * (x.abs() @ w.abs().t() + bb.abs())


def joint_logits(E, P, Wo, bo, B, T, U_):
    """E [B*T, J], P [B*U, J] (the kernel's projections), W_o [V+1, J], b_o -> float64 logits [B, T, U, V+1] and bounds"""
    J = E.shape[-1]
    hid = torch.relu(E.double().view(B, T, 1, J) + P.double().view(B, 1, U_, J))
    w, bb = Wo.double(), bo.double()
    return hid @ w.t() + bb, gamma(J + 2) * (hid @ w.abs().t() + bb.abs())


def check_projection(name, got, A, W, b):
    """sgemm_bias_kernel: got [M, N] = A [M, K] W [N, K]^T + b, element by element.  Returns worst err/bound."""
    a, w, bb = A.double(), W.double(), b.double()
    want = a @ w.t() + bb
    bound = 1.001 * gamma(a.shape[-1] + 1) * (a.abs() @ w.abs().t() + bb.abs())
    _assert_within(got, want, bound, name)
    assert _rel_fro(got, want) <= F32_FRO, name
    return float(((got.double() - want).abs() / bound.clamp_min(1e-300)).max())


def lstm_step(ids, h, c, emb_gates, whh_t):
    """one lstm_step_kernel step in float64 from its fp32 operands: ids [B], h / c [B, H], emb_gates [V+1, 4H],
    whh_t [H, 4H] -> (h', c', bound of h', bound of c')"""
    H = h.shape[-1]
    gx = emb_gates.double()[ids]
    hd, w = h.double(), whh_t.double()
    gates = gx + hd @ w
    err = gamma(H + 1) * (hd.abs() @ w.abs() + gx.abs())
    (i, f, g, o), (ei, ef, eg, eo) = gates.chunk(4, -1), err.chunk(4, -1)
    si, sf, so, tg = i.sigmoid(), f.sigmoid(), o.sigmoid(), g.tanh()
    esi, esf, eso = (0.25 * e + 6 * U * s for e, s in ((ei, si), (ef, sf), (eo, so)))
    etg = eg + 4 * U * tg.abs()
    cd = c.double()
    cn = sf * cd + si * tg
    ec = cd.abs() * esf + tg.abs() * esi + si * etg + 2 * U * (sf * cd.abs() + si * tg.abs())
    tc = cn.tanh()
    hn = so * tc
    eh = tc.abs() * eso + so * (ec + 4 * U * tc.abs()) + U * hn.abs()
    return hn, cn, 1.001 * eh, 1.001 * ec


def check_lstm(name, g, c_seq, x, h0, c0, emb_gates, whh_t, V1):
    """g [B, U, H] and c_seq [U, B, H] of rnnt_predict_train: every step against one float64 step from the kernel's
    previous h (g[:, u-1]) and c (c_seq[u-1]).  Returns worst err/bound."""
    B, U_, H = g.shape
    worst = 0.0
    for u in range(U_):
        hp = (h0 if h0 is not None else torch.zeros(B, H, device=g.device)) if u == 0 else g[:, u - 1]
        cp = (c0 if c0 is not None else torch.zeros(B, H, device=g.device)) if u == 0 else c_seq[u - 1]
        ids = x[:, u] if x is not None else torch.full((B,), V1 - 1, dtype=torch.long, device=g.device)
        hn, cn, eh, ec = lstm_step(ids, hp, cp, emb_gates, whh_t)
        for what, got, want, bd in (("h", g[:, u], hn, eh), ("c", c_seq[u], cn, ec)):
            _assert_within(got, want, bd, f"{name} step {u} {what}")
            assert _rel_fro(got, want) <= F32_FRO, f"{name} step {u} {what}"
            worst = max(worst, float(((got.double() - want).abs() / bd.clamp_min(1e-300)).max()))
    return worst


def _bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def check_gather(name, lat, blank, label, targets):
    """rnnt_align_scores against the lattice of the same inputs: bit-identical entries, NaN for a target outside
    [0, V), -inf in the last column."""
    B, T, U1, V1 = lat.shape
    Uy = U1 - 1
    assert _bits(blank, lat[..., V1 - 1]), f"{name}: blank scores differ from the lattice"
    if Uy:
        tg = targets.long().to(lat.device)
        valid = ((tg >= 0) & (tg < V1 - 1))[:, None, :].expand(B, T, Uy)
        ref = lat[:, :, :Uy].gather(-1, tg.clamp(0, V1 - 1)[:, None, :, None].expand(B, T, Uy, 1))[..., 0]
        lab = label[:, :, :Uy]
        assert _bits(lab[valid], ref[valid]), f"{name}: label scores differ from the lattice"
        assert bool(lab[~valid].isnan().all()), f"{name}: a target outside [0, V) did not give NaN"
    assert bool((label[:, :, Uy] == -INF).all()), f"{name}: the last column is not -inf"


# ------------------------------------------------------------------------------------------ GPU plumbing
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (there is no CPU fallback to test instead)"
    return torch.device("cuda", 0)


def _cfg(name, V1=None, J=None, H=None, n_layers=1):
    """synthetic.model_cfg with n_layers encoder layers, V+1 classes, joint_hidden J and pred_hidden H"""
    cfg = synthetic.model_cfg(name, n_layers=n_layers)
    h = cfg["head"]
    if V1 is not None:
        cfg["decoding"]["vocabulary"] = [f"<{i}>" for i in range(V1 - 1)]
        cfg["decoding"].pop("model_path", None)
        if h["type"] == "ctc":
            h["num_classes"] = V1
        else:
            h["decoder"]["num_classes"] = h["joint"]["num_classes"] = V1
    if J is not None:
        h["joint"]["joint_hidden"] = J
    if H is not None:
        h["decoder"]["pred_hidden"] = h["joint"]["pred_hidden"] = H
    return cfg


def _model(dev, name, **kw):
    cfg = _cfg(name, **kw)
    ck = {"cfg": cfg, "state_dict": synthetic.synthetic_state_dict(cfg, seed=0)}
    return gigaam.load_model(name, fp16_encoder=False, device=dev, checkpoint=ck), ck


def _set_params(model, values):
    """copy values {"head.*": tensor} into the live parameters (the engine repacks the head on its next call)"""
    params = dict(model.named_parameters())
    with torch.no_grad():
        for k, v in values.items():
            params[k].copy_(v)


def _unsaturate(model, ck):
    sd = _head_sd(ck, scale=UNSAT, seed=1)
    _set_params(model, {k: sd[k] for k in ("head.joint.joint_net.1.weight", "head.decoder_layers.0.weight") if k in sd})


def _heads(model, ck):
    """run the caller's cases once with the synthetic head, then once with the unsaturated one"""
    yield "synthetic"
    _unsaturate(model, ck)
    yield f"unsaturated({UNSAT})"


def _bufs(model):
    return model._get_engine()._head_bufs


def _ctc(model, enc_btd):
    with torch.inference_mode():
        lp = model.head(enc_btd.transpose(1, 2))
    torch.cuda.synchronize()
    return lp


def _joint_ws(model, B, T, U_, J):
    """E [B*T, J] and P [B*U, J] as the last rnnt_joint call left them in its workspace (gam_rnnt_joint carves E at the
    first 1 KiB boundary, P at the next one past E)"""
    ws = model._get_engine()._ws_joint.peek((B, T, U_))
    off = -ws.data_ptr() % 1024
    e_bytes = B * T * J * 4
    p_off = off + -(-e_bytes // 1024) * 1024
    E = ws[off:off + e_bytes].view(torch.float32).view(B * T, J)
    P = ws[p_off:p_off + B * U_ * J * 4].view(torch.float32).view(B * U_, J)
    return E.clone(), P.clone()


def _joint(model, enc, dec):
    with torch.inference_mode():
        lat = model.head.joint.joint(enc, dec)
    torch.cuda.synchronize()
    return lat


def _scores(model, enc, dec, targets):
    with torch.inference_mode():
        blank, label = model._get_engine().rnnt_align_scores(enc, dec, targets)
    torch.cuda.synchronize()
    return blank, label


def _targets(B, Uy, V1, g):
    """ids in [0, V) with, where there is room, one -1, one V (the blank id) and one V + 3: ids the gather maps to NaN"""
    t = torch.randint(0, V1 - 1, (B, Uy), generator=g)
    if Uy:
        t[0, 0] = -1
        t[-1, -1] = V1 - 1
        if Uy > 2:
            t[B // 2, 1] = V1 + 3
    return t


# ------------------------------------------------------------------------------------------ GPU: CTC log-probs
CTC_ROWS = [(1, 1), (1, 31), (1, 32), (1, 33), (64, 251)]


@pytest.mark.gpu
@pytest.mark.parametrize("V1", [2, 9, 10, 35, 36, 37, 72, 73, 257, 1025])
def test_ctc_log_probs_against_float64(dev, V1):
    model, ck = _model(dev, "v2_ctc", V1=V1)
    g = torch.Generator().manual_seed(V1)
    for head in _heads(model, ck):
        for B, T in CTC_ROWS:
            enc = torch.randn(B, T, 768, generator=g).to(dev)
            lp = _ctc(model, enc)
            assert lp.shape == (B, T, V1)
            bufs = _bufs(model)
            z, e = ctc_logits(enc.view(-1, 768), bufs["ctc_w"], bufs["ctc_b"])
            worst, fro, ent = check_log_probs(f"ctc V1={V1} {head} {B}x{T}", lp.view(-1, V1), z, e, CTC_TILING)
            print(f"ctc V1={V1} {head} rows {B}x{T}: worst err/bound {worst:.3g}, rel fro {fro:.2g}, "
                  f"min row entropy {ent:.3f} nats")


# ------------------------------------------------------------------------------------------ GPU: projections
def _check_joint_projections(model, name, enc, dec, E, P):
    bufs = _bufs(model)
    we = check_projection(f"{name} E", E, enc.reshape(E.shape[0], -1), bufs["rnnt_enc_w"], bufs["rnnt_enc_b"])
    wp = check_projection(f"{name} P", P, dec.reshape(P.shape[0], -1), bufs["rnnt_wp_t"].t(), bufs["rnnt_bp"])
    return max(we, wp)


@pytest.mark.gpu
@pytest.mark.parametrize("J,H", [(60, 320), (64, 320), (68, 320), (64, 16), (68, 48)])
def test_joint_projections_against_float64(dev, J, H):
    """sgemm_bias_kernel in both layouts (W [N, K] for E, W^T [K, N] for P) at row counts and J around its 64 x 64 tile"""
    model, _ = _model(dev, "v2_rnnt", J=J, H=H)
    g = torch.Generator().manual_seed(J + H)
    for B, T, U_ in [(1, 63, 65), (1, 64, 64), (1, 65, 63), (2, 32, 33)]:
        enc, dec = torch.randn(B, T, 768, generator=g).to(dev), (torch.rand(B, U_, H, generator=g) * 2 - 1).to(dev)
        _joint(model, enc, dec)
        E, P = _joint_ws(model, B, T, U_, J)
        worst = _check_joint_projections(model, f"J={J} H={H} {B}x{T}x{U_}", enc, dec, E, P)
        print(f"projections J={J} H={H} rows E {B * T}, P {B * U_}: worst err/bound {worst:.3g}")


@pytest.mark.gpu
def test_greedy_encoder_projection_against_float64(dev):
    """the encoder projection the RNN-T greedy path runs over all 64 x 251 rows (the decode workspace's first buffer)"""
    model, _ = _model(dev, "v2_rnnt")
    B, T, J = 64, 251, 320
    enc = torch.randn(B, T, 768, generator=torch.Generator().manual_seed(5)).to(dev)
    with torch.inference_mode():
        model.decoding.decode(model.head, enc.transpose(1, 2), torch.full((B,), T, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()
    ws = model._get_engine()._ws_dec.peek((B, T))
    encproj = ws[:B * T * J * 4].view(torch.float32).view(B * T, J)
    bufs = _bufs(model)
    worst = check_projection("greedy encproj", encproj, enc.view(-1, 768), bufs["rnnt_enc_w"], bufs["rnnt_enc_b"])
    print(f"greedy encoder projection {B}x{T}: worst err/bound {worst:.3g}")


# ------------------------------------------------------------------------------------------ GPU: joint lattice and gather
JOINT_SHAPES = [(1, 1, 1), (3, 3, 7), (2, 4, 8), (1, 5, 13), (3, 251, 17)]   # B*T*U = 1, 63, 64, 65 and 12801


@pytest.mark.gpu
@pytest.mark.parametrize("J", [4, 20, 320, 324, JOINT_MAX_HIDDEN])
@pytest.mark.parametrize("V1", [2, 34, 63, 64, 65, 129, 1025])
def test_joint_lattice_and_gather_against_float64(dev, V1, J):
    model, ck = _model(dev, "v2_rnnt", V1=V1, J=J)
    g = torch.Generator().manual_seed(V1 * 1000 + J)
    for head in _heads(model, ck):
        for B, T, U_ in JOINT_SHAPES:
            name = f"joint V1={V1} J={J} {head} {B}x{T}x{U_}"
            enc, dec = torch.randn(B, T, 768, generator=g).to(dev), (torch.rand(B, U_, 320, generator=g) * 2 - 1).to(dev)
            lat = _joint(model, enc, dec)
            assert lat.shape == (B, T, U_, V1)
            E, P = _joint_ws(model, B, T, U_, J)
            wproj = _check_joint_projections(model, name, enc, dec, E, P)
            bufs = _bufs(model)
            z, e = joint_logits(E, P, bufs["rnnt_wo"], bufs["rnnt_bo"], B, T, U_)
            worst, fro, ent = check_log_probs(name, lat, z, e, JOINT_TILING)
            targets = _targets(B, U_ - 1, V1, g)
            check_gather(name, lat, *_scores(model, enc, dec, targets), targets)
            print(f"{name}: worst err/bound {worst:.3g} (projections {wproj:.3g}), rel fro {fro:.2g}, "
                  f"min row entropy {ent:.3f} nats")


@pytest.mark.gpu
def test_joint_refuses_hidden_sizes_past_its_limit(dev):
    """load and engine creation take any joint_hidden; the lattice takes J % 4 == 0 up to the shared-memory limit and
    refuses the next multiple of 4 and a J that is not one, naming the limit"""
    enc, dec = torch.randn(1, 2, 768, device=dev), torch.rand(1, 3, 320, device=dev)
    for J in (JOINT_MAX_HIDDEN + 4, 18):
        model, _ = _model(dev, "v2_rnnt", J=J)
        with pytest.raises(RuntimeError, match=f"joint_hidden % 4 == 0 and <= {JOINT_MAX_HIDDEN}"):
            _joint(model, enc, dec)


# ------------------------------------------------------------------------------------------ GPU: LSTM step
@pytest.mark.gpu
@pytest.mark.parametrize("H", [16, 64, 72, 320, 1024])
def test_lstm_steps_against_float64(dev, H):
    model, _ = _model(dev, "v2_rnnt", H=H)
    V1 = 34
    eng = model._get_engine()
    bufs = _bufs(model)
    g = torch.Generator().manual_seed(H)
    worst = 0.0
    for B in (1, 7, 8, 9, 40):
        for U_, with_x in ((1, True), (3, True), (1, False)):
            for with_state in (False, True):
                x = torch.randint(0, V1, (B, U_), generator=g).to(dev) if with_x else None
                if with_x:
                    x[B // 2, U_ - 1] = V1 - 1          # the blank id: the zero-embedding row
                h0, c0 = ((torch.randn(B, H, generator=g).to(dev), torch.randn(B, H, generator=g).to(dev)) if with_state
                          else (None, None))
                with torch.inference_mode():
                    gg, h1, c1, c_seq = eng.rnnt_predict_train(x, h0, c0, B)
                    g2, h2, c2 = eng.rnnt_predict(x, h0, c0, B)
                torch.cuda.synchronize()
                name = f"lstm H={H} B={B} U={U_} x={with_x} state={with_state}"
                assert _bits(gg, g2) and _bits(h1, h2) and _bits(c1, c2), f"{name}: predict and predict_train differ"
                assert _bits(h1, gg[:, -1]) and _bits(c1, c_seq[-1]), name
                worst = max(worst, check_lstm(name, gg, c_seq, x, h0, c0, bufs["rnnt_emb_gates"], bufs["rnnt_whh_t"], V1))
    print(f"lstm H={H}: 30 cases, worst err/bound {worst:.3g}")


# ------------------------------------------------------------------------------------------ GPU: non-finite rows
def _ctc_bias_cases(V1):
    V = V1 - 1
    group_firsts = [c for c in (0, 9, 18, 27, 35, 36, V) if c < V1]
    cases = [(f"bias[{c}] = -inf", {c: -INF}) for c in group_firsts]
    cases.append((f"bias{group_firsts} = -inf", {c: -INF for c in group_firsts}))
    cases.append(("bias[5] = NaN", {5: NAN}))
    # class group 0 all -inf and group 1 NaN / -inf only: the NaN must survive the merge of two groups without a finite logit
    cases.append(("groups 0 and 1 without a finite logit, one NaN", {**{c: -INF for c in range(18)}, 9: NAN}))
    cases.append(("every bias -inf", {c: -INF for c in range(V1)}))
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("V1", [34, 73])
def test_ctc_nonfinite_rows_follow_torch(dev, V1):
    model, _ = _model(dev, "v2_ctc", V1=V1)
    key = "head.decoder_layers.0.bias"
    b0 = dict(model.named_parameters())[key].detach().clone()
    g = torch.Generator().manual_seed(V1)
    B, T = 2, 40
    enc = torch.randn(B, T, 768, generator=g).to(dev)
    enc[0, 3, 100] = INF        # one +inf and one NaN encoder component: those two rows are all NaN
    enc[1, 17, 5] = NAN
    for what, edits in _ctc_bias_cases(V1):
        b = b0.clone()
        for c, v in edits.items():
            b[c] = v
        _set_params(model, {key: b})
        lp = _ctc(model, enc)
        bufs = _bufs(model)
        assert _bits(bufs["ctc_b"], b), "the edited bias did not reach the kernel"
        z, e = ctc_logits(enc.view(-1, 768), bufs["ctc_w"], bufs["ctc_b"])
        worst, _, _ = check_log_probs(f"ctc V1={V1} {what}", lp.view(-1, V1), z, e, CTC_TILING)
        print(f"ctc V1={V1} {what}: non-finite entries as torch, worst err/bound {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("V1", [34, 1025])
def test_joint_nonfinite_rows_follow_torch(dev, V1):
    model, _ = _model(dev, "v2_rnnt", V1=V1)
    key = "head.joint.joint_net.1.bias"
    b0 = dict(model.named_parameters())[key].detach().clone()
    V = V1 - 1
    banned = [c for c in (0, 4, 60, 64, V) if c < V1]
    cases = [(f"b_o[{c}] = -inf", {c: -INF}) for c in banned] + [(f"b_o{banned} = -inf", {c: -INF for c in banned})]
    # lanes 0 and 8 of a row group (classes 0-3 and 32-35) without a finite logit, a NaN among them
    cases.append(("lanes 0 and 8 without a finite logit, one NaN", {**{c: -INF for c in (0, 1, 2, 3, 33)}, 32: NAN}))
    g = torch.Generator().manual_seed(V1)
    B, T, U_ = 2, 9, 6
    enc, dec = torch.randn(B, T, 768, generator=g).to(dev), (torch.rand(B, U_, 320, generator=g) * 2 - 1).to(dev)
    enc[1, 4, 7] = NAN          # every lattice row (1, 4, :) is NaN
    dec[0, 2, 11] = NAN         # and every row (0, :, 2)
    # labels at banned classes (-inf scores) and the last non-blank id
    targets = torch.tensor([[0] * (U_ - 1), [V - 1, 4, 60 % V, 0, 64 % V]], dtype=torch.int64)
    for what, edits in cases:
        b = b0.clone()
        for c, v in edits.items():
            b[c] = v
        _set_params(model, {key: b})
        lat = _joint(model, enc, dec)
        E, P = _joint_ws(model, B, T, U_, 320)
        bufs = _bufs(model)
        assert _bits(bufs["rnnt_bo"], b), "the edited bias did not reach the kernel"
        z, e = joint_logits(E, P, bufs["rnnt_wo"], bufs["rnnt_bo"], B, T, U_)
        name = f"joint V1={V1} {what}"
        worst, _, _ = check_log_probs(name, lat, z, e, JOINT_TILING)
        check_gather(name, lat, *_scores(model, enc, dec, targets), targets)
        print(f"{name}: non-finite entries as torch, gather bit-identical, worst err/bound {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v2_rnnt"])
def test_head_edit_reaches_the_kernels_in_any_grad_mode(dev, name):
    """An engine built under torch.inference_mode(), then a head edit: calls inside and outside inference mode both use
    the edited head, and the repack leaves nothing pending (the packed buffers are not views of the parameters)."""
    model, ck = _model(dev, name)
    enc = torch.randn(2, 5, 768, device=dev)
    dec = torch.rand(2, 3, 320, device=dev)

    def run():
        return model.head(enc.transpose(1, 2)) if name == "v2_ctc" else model.head.joint.joint(enc, dec)
    with torch.inference_mode():
        before = run()
    _unsaturate(model, ck)
    with torch.inference_mode():
        inside = run()
    assert model._get_engine().head_signature == model._head_signature(), "the repack changed the parameters it read"
    with torch.no_grad():
        outside = run()
    assert torch.equal(inside, outside) and not torch.equal(before, inside)


@pytest.mark.gpu
def test_align_with_a_banned_class_is_finite(dev):
    """A -inf bias bans a token: alignment of a transcript without it still has a finite log-likelihood."""
    model, _ = _model(dev, "v2_ctc")
    key = "head.decoder_layers.0.bias"
    b = dict(model.named_parameters())[key].detach().clone()
    b[0] = -INF
    _set_params(model, {key: b})
    wav, wav_len = gigaam.synthetic_audio(2, 2.0, seed=3, ragged=True)
    out = model.align_batch(wav.to(dev), wav_len.to(dev), [[1, 2, 3, 4, 5], [7, 7, 12]])
    for a in out:
        assert math.isfinite(a.log_likelihood) and a.log_likelihood <= 0, a.log_likelihood
    with torch.inference_mode():
        enc, _ = model(wav.to(dev), wav_len.to(dev))
        lp = model.head(enc)
    assert bool((lp[..., 0] == -INF).all()) and bool(lp[..., 1:].isfinite().all())


# ------------------------------------------------------------------------------------------ CPU: negative controls
def _raises(fn, *args):
    with pytest.raises(AssertionError):
        fn(*args)


def _cpu_joint(B, T, U_, J, V1, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B * T, J, generator=g), torch.randn(B * U_, J, generator=g), torch.randn(V1, J, generator=g) * 0.3,
            torch.randn(V1, generator=g))


def _fp32_lattice(E, P, Wo, bo, B, T, U_):
    J = E.shape[-1]
    return (torch.relu(E.view(B, T, 1, J) + P.view(B, 1, U_, J)) @ Wo.t() + bo).log_softmax(-1)


def test_joint_checker_rejects_a_dropped_last_k_chunk():
    B, T, U_, J, V1 = 2, 3, 4, 20, 34
    E, P, Wo, bo = _cpu_joint(B, T, U_, J, V1, 0)
    z, e = joint_logits(E, P, Wo, bo, B, T, U_)
    check_log_probs("fp32 lattice", _fp32_lattice(E, P, Wo, bo, B, T, U_), z, e, JOINT_TILING)
    # J % 16 != 0: a kernel whose K loop stops at the last full 16-wide chunk
    dropped = torch.relu(E.double().view(B, T, 1, J) + P.double().view(B, 1, U_, J))[..., :J // 16 * 16]
    bad = (dropped @ Wo.double()[:, :J // 16 * 16].t() + bo.double()).log_softmax(-1).float()
    _raises(check_log_probs, "dropped k chunk", bad, z, e, JOINT_TILING)


def test_joint_checker_rejects_p_of_the_wrong_utterance():
    B, T, U_, J, V1 = 2, 3, 4, 20, 34
    E, P, Wo, bo = _cpu_joint(B, T, U_, J, V1, 1)
    z, e = joint_logits(E, P, Wo, bo, B, T, U_)
    P_swapped = P.view(B, U_, J).roll(1, 0).reshape(B * U_, J)
    bad = _fp32_lattice(E, P_swapped, Wo, bo, B, T, U_)
    _raises(check_log_probs, "P of utterance b+1", bad, z, e, JOINT_TILING)


def test_ctc_checker_rejects_a_class_tile_missing_from_the_log_sum_exp():
    R, D, V1 = 5, 64, 73
    g = torch.Generator().manual_seed(2)
    enc, W, b = torch.randn(R, D, generator=g), torch.randn(V1, D, generator=g) * 0.2, torch.randn(V1, generator=g)
    z, e = ctc_logits(enc, W, b)
    check_log_probs("fp32 log-probs", (enc @ W.t() + b).log_softmax(-1), z, e, CTC_TILING)
    keep = torch.ones(V1, dtype=torch.bool)
    keep[36:72] = False                                          # the second 36-class tile left out of the statistics
    bad = (z - torch.logsumexp(z[:, keep], -1, keepdim=True)).float()
    _raises(check_log_probs, "tile missing", bad, z, e, CTC_TILING)


def test_lstm_checker_rejects_swapped_f_and_g_gates():
    B, H, V1 = 3, 16, 5
    g = torch.Generator().manual_seed(3)
    emb_gates, whh_t = torch.randn(V1, 4 * H, generator=g), torch.randn(H, 4 * H, generator=g) * 0.3
    x = torch.randint(0, V1, (B, 2), generator=g)
    h0, c0 = torch.randn(B, H, generator=g), torch.randn(B, H, generator=g)

    def run(perm):
        gs, cs, h, c = [], [], h0, c0
        for u in range(2):
            i, f, gg, o = (emb_gates[x[:, u]] + h @ whh_t).chunk(4, -1)
            i, f, gg, o = (i, f, gg, o) if not perm else (i, gg, f, o)
            c = f.sigmoid() * c + i.sigmoid() * gg.tanh()
            h = o.sigmoid() * c.tanh()
            gs.append(h)
            cs.append(c)
        return torch.stack(gs, 1), torch.stack(cs, 0)
    check_lstm("fp32 lstm", *run(False), x, h0, c0, emb_gates, whh_t, V1)
    _raises(check_lstm, "f and g swapped", *run(True), x, h0, c0, emb_gates, whh_t, V1)


# float32 emulation of lse_push / lse_merge over the kernels' tiling.  push_guard: which logits the else branch of
# lse_push adds ("none": all, as at first; "finite": v > -inf, which also drops NaN; "not -inf": v != -inf).
# keep_nan_on_empty_merge: lse_merge of two sides without a logit above -inf adds their sums (0, or NaN) instead of
# returning.
def _lse_emulated(logits, tiling, push_guard, keep_nan_on_empty_merge):
    threads, width, _ = tiling
    f32 = np.float32
    out = np.empty_like(logits)
    with np.errstate(all="ignore"):
        for r, row in enumerate(logits):
            V1 = row.shape[0]
            m = [f32(-np.inf)] * threads
            s = [f32(0)] * threads
            for t in range(threads):
                for c0 in range(0, V1, threads * width):
                    for c in range(width):
                        n = c0 + t * width + c
                        if n >= V1:
                            continue
                        v = row[n]
                        if v > m[t]:
                            s[t] = f32(s[t] * np.exp(f32(m[t] - v)) + f32(1))
                            m[t] = v
                        elif (push_guard == "none" or (push_guard == "finite" and v > -np.inf)
                              or (push_guard == "not -inf" and v != -np.inf)):
                            s[t] = f32(s[t] + np.exp(f32(v - m[t])))

            def merge(a, b):
                M = np.fmax(a[0], b[0])
                if M == -np.inf:
                    return (a[0], f32(a[1] + b[1])) if keep_nan_on_empty_merge else a
                return M, f32(a[1] * np.exp(f32(a[0] - M)) + b[1] * np.exp(f32(b[0] - M)))
            st = list(zip(m, s))
            if threads == 4:                       # ctc_log_probs_kernel: group 0 merges groups 1, 2, 3 in turn
                for t in range(1, 4):
                    st[0] = merge(st[0], st[t])
            else:                                  # rnnt_joint_kernel: xor butterfly over the 16 lanes of a row
                for off in (8, 4, 2, 1):
                    st = [merge(st[t], st[t ^ off]) for t in range(threads)]
            lse = f32(st[0][0] + np.log(st[0][1]))
            out[r] = row - lse
    return torch.from_numpy(out)


def _nonfinite_rows(V1, tiling, seed):
    """rows with -inf at the first class of every thread, at several classes, NaN and +inf logits, every logit -inf,
    and the merge case of two threads without a finite logit and one NaN between them"""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(V1, generator=g) * 3
    threads, width, _ = tiling
    firsts = sorted({t * width for t in range(threads) if t * width < V1} | {V1 - 1})
    rows = []
    for c in firsts:
        rows.append(base.clone().index_fill_(0, torch.tensor([c]), -INF))
    rows.append(base.clone().index_fill_(0, torch.tensor(firsts), -INF))
    for v in (NAN, INF):
        rows.append(base.clone().index_fill_(0, torch.tensor([1]), v))
    rows.append(torch.full((V1,), -INF))
    other = 1 if threads == 4 else 8            # CTC: group 0 then group 1; joint: lane 0 and its first partner, lane 8
    empty = [c for t in (0, other) for c0 in range(0, V1, threads * width) for c in range(c0 + t * width, c0 + (t + 1) * width)
             if c < V1]
    r = base.clone().index_fill_(0, torch.tensor(empty), -INF)
    r[empty[-1]] = NAN
    rows.append(r)
    return torch.stack(rows)


@pytest.mark.parametrize("tiling,V1", [(CTC_TILING, 34), (CTC_TILING, 73), (JOINT_TILING, 65), (JOINT_TILING, 130)])
def test_lse_rules_against_float64_log_softmax(tiling, V1):
    """The running log-sum-exp rule of heads.cu (skip -inf; NaN and +inf poison the row; a merge of two sides without a
    finite logit keeps a NaN) gives torch's non-finite rows.  The rule without a -inf case gives all-NaN rows for a -inf
    first logit of a thread; the guard v > -inf drops NaN and leaves a NaN row finite; a merge that returns on two empty
    sides loses a NaN: the checker rejects each."""
    z = _nonfinite_rows(V1, tiling, V1).double()
    e = torch.zeros_like(z)
    logits = z.float().numpy()
    check_log_probs("fixed rule", _lse_emulated(logits, tiling, "not -inf", True), z, e, tiling)
    _raises(check_log_probs, "no -inf case", _lse_emulated(logits, tiling, "none", True), z, e, tiling)
    _raises(check_log_probs, "guard v > -inf", _lse_emulated(logits, tiling, "finite", True), z, e, tiling)
    _raises(check_log_probs, "merge drops NaN", _lse_emulated(logits, tiling, "not -inf", False), z, e, tiling)
