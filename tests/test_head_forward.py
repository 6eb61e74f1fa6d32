"""The heads' own forward passes: CTCHead.forward, RNNTJoint.joint / forward, RNNTDecoder.predict / forward and
GigaAMASR.forward_for_export (gigaam/decoder.py, gigaam/model.py:142-149).

CPU: this file's fp32 restatements of the three forward passes equal the reference modules on seeded weights, and the RNN-T head keeps the reference's
module tree (state_dict keys, attributes).  GPU: the kernels of csrc/heads.cu against the oracle, the greedy path and
the reference's own greedy loop driven through our head."""
import sys

import pytest
import torch
import torch.nn.functional as F

import gigaam_b200 as gigaam
from gigaam_b200 import synthetic
from gigaam_b200.decoder import CTCHead, RNNTDecoder, RNNTHead, RNNTJoint
from oracle import gigaam_oracle as orc
from oracle import ref_loader

LP_TOL = 1e-4        # log-probs vs the fp32 CPU oracle (different summation order only)
# The synthetic joint weights give lattice logits of magnitude 150-250 for any input, and every log-prob of a row goes
# through that row's log-sum-exp.  At that magnitude fp32 rounding alone moves entries by about 1e-4: the fp32 CPU oracle
# itself is up to 1.8e-4 away from an fp64 evaluation of the same formula.  The kernel and the oracle, two fp32
# evaluations, are compared at 2.5e-4; an indexing or normalisation error shows up as O(1).
JOINT_TOL = 2.5e-4
STATE_TOL = 1e-5     # prediction-network outputs
MARGIN = 1e-5        # CTC: frames whose oracle top-2 margin is below this may flip between summation orders
JOINT_TIE = 1e-4     # RNN-T: a token may differ from the cluster kernel's only on a near-tie of the joint


# ------------------------------------------------------------------------------------------ CPU fp32 restatements
# The heads' forward passes in plain PyTorch, state_dict-driven, on top of the oracle's `ctc_logits` and `_lstm_step`
# (paths relative to the reference repository).  The CPU tests below pin them to the reference modules.
def ctc_log_probs(enc, sd):
    """gigaam/decoder.py:18-21 (CTCHead.forward).  enc [B, d, T] -> [B, T, V+1]"""
    return torch.log_softmax(orc.ctc_logits(enc, sd), dim=-1)


def rnnt_joint(enc, dec, sd):
    """gigaam/decoder.py:41-47 (RNNTJoint.joint).  enc [B, T, d], dec [B, U, H] -> [B, T, U, V+1]"""
    e = F.linear(enc, sd["head.joint.enc.weight"], sd["head.joint.enc.bias"]).unsqueeze(2)
    p = F.linear(dec, sd["head.joint.pred.weight"], sd["head.joint.pred.bias"]).unsqueeze(1)
    return F.linear(F.relu(e + p), sd["head.joint.joint_net.1.weight"], sd["head.joint.joint_net.1.bias"]).log_softmax(-1)


def rnnt_predict(x, state, sd, batch_size=1):
    """gigaam/decoder.py:85-102 (RNNTDecoder.predict; :131-137 forward is the same with a state): x [B, U] ids or None
    (one step from the zero embedding), state ([1, B, H], [1, B, H]) or None (zeros) -> (g [B, U, H], (h, c) [1, B, H])."""
    emb_w = sd["head.decoder.embed.weight"]
    H = emb_w.shape[1]
    emb = emb_w[x] if x is not None else torch.zeros(batch_size, 1, H)
    B = emb.shape[0]
    h, c = (state[0][0], state[1][0]) if state is not None else (torch.zeros(B, H), torch.zeros(B, H))
    gs = []
    for u in range(emb.shape[1]):
        h, c = orc._lstm_step(emb[:, u], h, c, sd)
        gs.append(h)
    return torch.stack(gs, 1), (h.unsqueeze(0), c.unsqueeze(0))


def _imported_reference():
    """Import the reference package (source tree or compiled archive), run the caller, then drop the stub and reference
    modules again so that later tests see the interpreter as it was."""
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


def _ref_modules(reference, ck):
    _, _, rd, _ = reference
    head = ck["cfg"]["head"]
    if head["type"] == "ctc":
        m = rd.CTCHead(head["feat_in"], head["num_classes"])
    else:
        m = rd.RNNTHead(head["decoder"], head["joint"])
    m.load_state_dict({k[len("head."):]: v for k, v in ck["state_dict"].items() if k.startswith("head.")}, strict=True)
    return m.eval()


def _ckpt(name):
    return synthetic.synthetic_checkpoint(name, seed=3, n_layers=1)


# ------------------------------------------------------------------------------------------ CPU: oracle == reference
@pytest.mark.parametrize("name", ["v2_ctc", "v3_e2e_ctc"])
def test_oracle_ctc_log_probs_equal_reference(reference, name):
    ck = _ckpt(name)
    ref = _ref_modules(reference, ck)
    enc = torch.randn(3, 768, 29, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want = ref(enc)
    got = ctc_log_probs(enc, ck["state_dict"])
    assert got.shape == want.shape == (3, 29, ck["cfg"]["head"]["num_classes"])
    assert float((got - want).abs().max()) <= 1e-6


@pytest.mark.parametrize("name", ["v2_rnnt", "v3_e2e_rnnt"])
@pytest.mark.parametrize("U", [1, 7])
def test_oracle_rnnt_joint_equals_reference(reference, name, U):
    ck = _ckpt(name)
    ref = _ref_modules(reference, ck)
    g = torch.Generator().manual_seed(U)
    enc, dec = torch.randn(2, 11, 768, generator=g), torch.rand(2, U, 320, generator=g) * 2 - 1
    with torch.no_grad():
        want = ref.joint.joint(enc, dec)
        want_fwd = ref.joint(enc.transpose(1, 2), dec.transpose(1, 2))
    got = rnnt_joint(enc, dec, ck["state_dict"])
    assert got.shape == want.shape == (2, 11, U, ck["cfg"]["head"]["joint"]["num_classes"])
    assert float((got - want).abs().max()) <= 1e-6
    assert float((got - want_fwd).abs().max()) <= 1e-6


@pytest.mark.parametrize("name", ["v2_rnnt", "v3_e2e_rnnt"])
@pytest.mark.parametrize("U,with_x", [(1, True), (7, True), (1, False)])    # predict(None, ...) is one step
@pytest.mark.parametrize("with_state", [True, False])
def test_oracle_rnnt_predict_equals_reference(reference, name, U, with_x, with_state):
    ck = _ckpt(name)
    ref = _ref_modules(reference, ck)
    V1 = ck["cfg"]["head"]["decoder"]["num_classes"]
    g = torch.Generator().manual_seed(10 * U + 2 * with_x + with_state)
    B = 4
    x = torch.randint(0, V1, (B, U), generator=g) if with_x else None
    state = (torch.randn(1, B, 320, generator=g), torch.randn(1, B, 320, generator=g)) if with_state else None
    with torch.no_grad():
        gw, (hw, cw) = ref.decoder.predict(x, state, batch_size=B)
    go, (ho, co) = rnnt_predict(x, state, ck["state_dict"], batch_size=B)
    assert go.shape == gw.shape == (B, U, 320) and ho.shape == hw.shape == (1, B, 320)
    for a, b in ((go, gw), (ho, hw), (co, cw)):
        assert float((a - b).abs().max()) <= 1e-6
    if with_x and with_state:     # the ONNX form
        with torch.no_grad():
            gf, hf, cf = ref.decoder(x, *state)
        assert float((go - gf).abs().max()) <= 1e-6 and float((ho - hf).abs().max()) <= 1e-6


# ------------------------------------------------------------------------------------------ CPU: module tree
@pytest.mark.parametrize("name", ["v2_rnnt", "v3_e2e_rnnt"])
def test_rnnt_head_tree_keeps_reference_keys_and_attributes(name):
    ck = synthetic.synthetic_checkpoint(name, n_layers=1)
    model = gigaam.GigaAMASR(ck["cfg"])
    model.load_state_dict(ck["state_dict"], strict=True)
    assert list(model.state_dict().keys()) == list(ck["state_dict"].keys())
    head = model.head
    assert type(head) is RNNTHead and type(head.decoder) is RNNTDecoder and type(head.joint) is RNNTJoint
    dc, jt = ck["cfg"]["head"]["decoder"], ck["cfg"]["head"]["joint"]
    assert head.decoder.blank_id == dc["num_classes"] - 1 and head.decoder.pred_hidden == dc["pred_hidden"]
    assert head.joint.enc_hidden == jt["enc_hidden"] and head.joint.pred_hidden == jt["pred_hidden"]
    assert [k for k, _ in head.named_parameters()] == [k[len("head."):] for k in ck["state_dict"] if k.startswith("head.")]


@pytest.mark.parametrize("name", ["v2_rnnt", "v3_e2e_rnnt"])
def test_rnnt_head_attributes_match_reference(reference, name):
    ck = _ckpt(name)
    ref = _ref_modules(reference, ck)
    ours = gigaam.GigaAMASR(ck["cfg"]).head
    for a in ("blank_id", "pred_hidden"):
        assert getattr(ours.decoder, a) == getattr(ref.decoder, a), a
    for a in ("enc_hidden", "pred_hidden"):
        assert getattr(ours.joint, a) == getattr(ref.joint, a), a
    assert list(ours.state_dict()) == list(ref.state_dict())


def test_head_calls_on_a_cpu_model_raise_no_cpu_path():
    ctc = gigaam.load_model("v2_ctc", device="cpu", checkpoint=synthetic.synthetic_checkpoint("v2_ctc", n_layers=1))
    with pytest.raises(RuntimeError, match="no CPU"):
        ctc.head(torch.zeros(1, 768, 4))
    with pytest.raises(RuntimeError, match="no CPU"):
        ctc.forward_for_export(torch.zeros(1, 64, 100), torch.tensor([100]))
    rnnt = gigaam.load_model("v2_rnnt", device="cpu", checkpoint=synthetic.synthetic_checkpoint("v2_rnnt", n_layers=1))
    with pytest.raises(RuntimeError, match="no CPU"):
        rnnt.head.decoder.predict(None, None, batch_size=2)
    with pytest.raises(RuntimeError, match="no CPU"):
        rnnt.head.joint.joint(torch.zeros(1, 3, 768), torch.zeros(1, 2, 320))
    with pytest.raises(NotImplementedError):       # RNNTHead has no forward, as in the reference
        rnnt.head(torch.zeros(1, 768, 4))
    assert isinstance(CTCHead(768, 34), torch.nn.Module)


# ------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (there is no CPU fallback to test instead)"
    return torch.device("cuda", 0)


_MODELS = {}


def _model(name, dev, n_layers=2):
    key = (name, n_layers)
    if key not in _MODELS:
        ck = synthetic.synthetic_checkpoint(name, seed=0, n_layers=n_layers)
        _MODELS[key] = (gigaam.load_model(name, fp16_encoder=False, device=dev, checkpoint=ck), ck)
    return _MODELS[key]


def _ragged_encoded(B, T, lens, seed, dev):
    """A stand-in for the encoder's output: [B, d, T] transposed view of a [B, T, d] buffer, zeros past each length."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, 768, generator=g)
    x[torch.arange(T)[None, :] >= torch.tensor(lens)[:, None]] = 0
    return x.to(dev).transpose(1, 2), torch.tensor(lens, dtype=torch.int32, device=dev)


def _collapse(labels, L, blank):
    ids, frames = [], []
    for t in range(L):
        l = int(labels[t])
        if l != blank and (t == 0 or l != int(labels[t - 1])):
            ids.append(l)
            frames.append(t)
    return ids, frames


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v3_e2e_ctc"])
def test_ctc_log_probs_against_oracle_and_greedy(dev, name):
    model, ck = _model(name, dev)
    sd = ck["state_dict"]
    V1 = ck["cfg"]["head"]["num_classes"]
    lens = [70, 1, 43, 12, 69, 2]
    B, T = len(lens), 70
    encoded, enc_len = _ragged_encoded(B, T, lens, seed=V1, dev=dev)
    with torch.inference_mode():
        lp = model.head(encoded)
        torch.cuda.synchronize()
    assert lp.shape == (B, T, V1) and lp.dtype == torch.float32 and lp.is_cuda
    want = ctc_log_probs(encoded.cpu(), sd)
    valid = torch.arange(T)[None, :] < torch.tensor(lens)[:, None]
    lpc = lp.cpu()
    assert float((lpc[valid] - want[valid]).abs().max()) <= LP_TOL
    assert float((lpc.double().exp().sum(-1) - 1).abs().max()) <= 1e-5      # every row, padded frames included

    # frame labels of the greedy kernel (its decode workspace starts with labels [B*T] i32)
    eng = model._get_engine()
    hyps = model.decoding.decode(model.head, encoded, enc_len)
    ws = eng._ws_dec.peek((B, T))
    greedy_labels = ws[: B * T * 4].view(torch.int32).view(B, T).cpu()
    top2 = orc.ctc_logits(encoded.cpu(), sd).topk(2, dim=-1).values
    safe = (top2[..., 0] - top2[..., 1]) > MARGIN
    ours = lpc.argmax(-1)
    assert torch.equal(ours[valid & safe], greedy_labels[valid & safe].long())
    checked = 0
    for b, L in enumerate(lens):
        if not bool(safe[b, :L].all()):
            continue
        checked += 1
        ids, frames = _collapse(ours[b], L, V1 - 1)
        assert (ids, frames) == (hyps[b][1], hyps[b][2]), b
    assert checked >= len(lens) - 1


@pytest.mark.gpu
def test_forward_for_export_is_head_of_encoder(dev):
    model, _ = _model("v2_ctc", dev)
    wav, wav_len = gigaam.synthetic_audio(3, 1.5, seed=5, ragged=True)
    with torch.inference_mode():
        mel, mel_len = model.preprocessor(wav.to(dev), wav_len.to(dev))
        lp, lp_len = model.forward_for_export(mel, mel_len)
        enc, enc_len = model.encoder(mel, mel_len)
        want = model.head(enc)
    assert torch.equal(lp, want) and torch.equal(lp_len, enc_len)
    rnnt, _ = _model("v2_rnnt", dev)
    with pytest.raises(NotImplementedError):
        rnnt.forward_for_export(mel, mel_len)


def _assert_lattice_close(got, want):
    assert float((got - want).abs().max()) <= JOINT_TOL


def _joint_inputs(B, T, U, seed, dev):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, T, 768, generator=g).to(dev), (torch.rand(B, U, 320, generator=g) * 2 - 1).to(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_rnnt", "v3_e2e_rnnt"])
@pytest.mark.parametrize("B,T,U", [(1, 1, 1), (3, 251, 17), (8, 40, 33)])
def test_joint_lattice_against_oracle(dev, name, B, T, U):
    model, ck = _model(name, dev)
    enc, dec = _joint_inputs(B, T, U, B * T + U, dev)
    with torch.inference_mode():
        out = model.head.joint.joint(enc, dec)
        fwd = model.head.joint(enc.transpose(1, 2), dec.transpose(1, 2))
        torch.cuda.synchronize()
    V1 = ck["cfg"]["head"]["joint"]["num_classes"]
    assert out.shape == (B, T, U, V1)
    want = rnnt_joint(enc.cpu(), dec.cpu(), ck["state_dict"])
    _assert_lattice_close(out.cpu(), want)
    assert torch.equal(fwd, out)


@pytest.mark.gpu
def test_joint_lattice_past_2_pow_31_elements(dev):
    """B*T*U*(V+1) = 4*376*1400*1025 > 2^31 (8.6 GB of fp32): sampled rows, the last ones and those around element 2^31,
    against the oracle."""
    model, ck = _model("v3_e2e_rnnt", dev)
    sd = ck["state_dict"]
    B, T, U, V1 = 4, 376, 1400, 1025
    assert B * T * U * V1 > 2 ** 31
    enc, dec = _joint_inputs(B, T, U, 31, dev)
    with torch.inference_mode():
        out = model.head.joint.joint(enc, dec)
        rows = out.view(-1, V1)
        n = rows.shape[0]
        g = torch.Generator().manual_seed(0)
        pick = torch.cat([torch.randint(0, n, (48,), generator=g), torch.arange(n - 8, n),
                          torch.arange(2 ** 31 // V1 - 4, 2 ** 31 // V1 + 4)])
        got = rows[pick.to(dev)].cpu()
        torch.cuda.synchronize()
    del out, rows
    torch.cuda.empty_cache()
    b, t, u = pick // (T * U), (pick // U) % T, pick % U
    e = F.linear(enc.cpu()[b, t], sd["head.joint.enc.weight"], sd["head.joint.enc.bias"])
    p = F.linear(dec.cpu()[b, u], sd["head.joint.pred.weight"], sd["head.joint.pred.bias"])
    want = F.linear(F.relu(e + p), sd["head.joint.joint_net.1.weight"], sd["head.joint.joint_net.1.bias"]).log_softmax(-1)
    _assert_lattice_close(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 8, 40])
@pytest.mark.parametrize("U,with_x", [(1, True), (5, True), (1, False)])    # predict(None, ...) is one step
@pytest.mark.parametrize("with_state", [True, False])
def test_predict_against_oracle(dev, B, U, with_x, with_state):
    model, ck = _model("v2_rnnt", dev)
    V1 = ck["cfg"]["head"]["decoder"]["num_classes"]
    g = torch.Generator().manual_seed(B * 10 + U)
    x = torch.randint(0, V1, (B, U), generator=g) if with_x else None
    state = None
    if with_state:     # strided [1, B, H] views, as the reference's greedy loop slices its states
        h, c = torch.randn(1, 2 * B, 320, generator=g), torch.randn(1, 2 * B, 320, generator=g)
        state = (h[:, ::2], c[:, 1::2])
    with torch.inference_mode():
        gg, (hh, cc) = model.head.decoder.predict(None if x is None else x.to(dev),
                                                  None if state is None else tuple(s.to(dev) for s in state), batch_size=B)
        torch.cuda.synchronize()
    assert gg.shape == (B, U, 320) and hh.shape == cc.shape == (1, B, 320)
    gw, (hw, cw) = rnnt_predict(x, None if state is None else tuple(s.contiguous() for s in state), ck["state_dict"],
                                    batch_size=B)
    for a, w in ((gg, gw), (hh, hw), (cc, cw)):
        assert float((a.cpu() - w).abs().max()) <= STATE_TOL
    if with_x and with_state:
        with torch.inference_mode():
            gf, hf, cf = model.head.decoder(x.to(dev), *(s.to(dev) for s in state))
        assert torch.equal(gf, gg) and torch.equal(hf, hh) and torch.equal(cf, cc)


@pytest.mark.gpu
def test_predict_out_of_range_id_gives_nan_for_that_utterance_only(dev):
    model, ck = _model("v2_rnnt", dev)
    V1 = ck["cfg"]["head"]["decoder"]["num_classes"]
    B, U = 8, 5
    g = torch.Generator().manual_seed(4)
    x = torch.randint(0, V1, (B, U), generator=g)
    state = (torch.randn(1, B, 320, generator=g), torch.randn(1, B, 320, generator=g))
    bad = x.clone()
    bad[3, 2] = V1
    bad[5, 0] = -1
    with torch.inference_mode():
        gg, (hh, cc) = model.head.decoder.predict(bad.to(dev), tuple(s.to(dev) for s in state))
        torch.cuda.synchronize()
    gw, (hw, cw) = rnnt_predict(x, state, ck["state_dict"])
    ok = torch.tensor([b not in (3, 5) for b in range(B)])
    for a, w in ((gg.cpu(), gw), (hh.cpu()[0], hw[0]), (cc.cpu()[0], cw[0])):
        assert bool(a[~ok].isnan().all())
        assert float((a[ok] - w[ok]).abs().max()) <= STATE_TOL
    with torch.inference_mode():     # the device is still healthy
        g2, _ = model.head.decoder.predict(x.to(dev), tuple(s.to(dev) for s in state))
    assert float((g2.cpu() - gw).abs().max()) <= STATE_TOL


def _ref_decisions(head, encoded, L, max_symbols, blank):
    """The reference's greedy rule for ONE utterance through our head (batch-independent, decoding.py:128-207), with the
    top-2 joint margin of every decision: [(t, token or blank, margin)]."""
    x = encoded.transpose(1, 2)
    state, label, out = None, None, []
    for t in range(L):
        for _ in range(max_symbols):
            if state is None:
                gp, hid = head.decoder.predict(None, None, batch_size=1)
            else:
                gp, hid = head.decoder.predict(label, state, batch_size=1)
            lp = head.joint.joint(x[:, t:t + 1], gp)[0, 0, 0]
            top = lp.topk(2).values
            k = int(lp.argmax())
            out.append((t, k, float(top[0] - top[1])))
            if k == blank:
                break
            state, label = hid, torch.tensor([[k]], device=lp.device)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_rnnt", "v3_e2e_rnnt"])
def test_reference_greedy_loop_on_our_head_is_a_drop_in(dev, name):
    """The reference's own RNNTGreedyDecoding.decode (from the compiled archive that travels with the tree) driving our
    model.head gives the cluster kernel's hypotheses; a token may differ only on a joint near-tie."""
    assert ref_loader.ARCHIVE.is_file() or ref_loader.reference_root() is not None, \
        "oracle/_ref/gigaam_ref.zip is missing: build() compiles it from the reference"
    _, _, _, ref_decoding = _imported_reference()
    model, ck = _model(name, dev, n_layers=None)
    cfg = ck["cfg"]
    wav, wav_len = gigaam.synthetic_audio(4, 2.0, seed=11, ragged=True)
    with torch.inference_mode():
        encoded, enc_len = model(wav.to(dev), wav_len.to(dev))
        ours = model.decoding.decode(model.head, encoded, enc_len)
        ref_dec = ref_decoding.RNNTGreedyDecoding(cfg["decoding"]["vocabulary"], None, cfg["decoding"]["max_symbols_per_step"])
        theirs = ref_dec.decode(model.head, encoded, enc_len)
    assert sum(len(h[1]) for h in ours) > 0, "no tokens emitted: the comparison would be vacuous"
    blank = cfg["head"]["joint"]["num_classes"] - 1
    for b, (o, r) in enumerate(zip(ours, theirs)):
        if (o[1], o[2]) == (r[1], r[2]):
            continue
        # find the decision where the reference path leaves the kernel's path and show it is a near-tie
        with torch.inference_mode():
            steps = _ref_decisions(model.head, encoded[b:b + 1], int(enc_len[b]), ref_dec.max_symbols, blank)
        want = list(zip(o[2], o[1]))
        i = 0
        for t, k, margin in steps:
            expect = want[i] if i < len(want) else None
            if k != blank:
                if expect != (t, k):
                    assert margin < JOINT_TIE, (b, t, k, margin)
                    break
                i += 1
            elif expect is not None and expect[0] == t:
                assert margin < JOINT_TIE, (b, t, "blank", margin)
                break
        else:
            pytest.fail(f"utterance {b}: hypotheses differ but no diverging decision was found")


@pytest.mark.gpu
def test_graph_capture_replays_bit_exact(dev):
    ctc, _ = _model("v2_ctc", dev)
    encoded, _ = _ragged_encoded(4, 50, [50, 1, 33, 7], seed=9, dev=dev)
    with torch.inference_mode():
        eager = ctc.head(encoded)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ctc.head(encoded)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = ctc.head(encoded)
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(out, eager)

    rnnt, ck = _model("v2_rnnt", dev)
    V1 = ck["cfg"]["head"]["decoder"]["num_classes"]
    B = 16
    g = torch.Generator().manual_seed(2)
    x = torch.randint(0, V1, (B, 1), generator=g).to(dev)
    h, c = torch.randn(1, B, 320, generator=g).to(dev), torch.randn(1, B, 320, generator=g).to(dev)
    f = torch.randn(B, 1, 768, generator=g).to(dev)

    def step():
        gp, (h1, c1) = rnnt.head.decoder.predict(x, (h, c))
        return rnnt.head.joint.joint(f, gp), h1, c1

    with torch.inference_mode():
        want = step()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()
        torch.cuda.current_stream().wait_stream(s)
        graph2 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph2):
            got = step()
        graph2.replay()
        torch.cuda.synchronize()
    for a, w in zip(got, want):
        assert torch.equal(a, w)
