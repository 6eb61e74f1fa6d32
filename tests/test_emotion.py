"""GigaAM-Emo: `load_model("emo")`, `GigaAMEmo.get_probs` / `forward_for_export`, the `Linear` head and `gam_emo_head`
(gigaam/model.py:262-293).

Frames pooled for utterance b: n_b = encoded_len[b], except that a batch of ONE pools all T' frames (DESIGN §3.1's rule).
That reproduces the reference's get_probs exactly and makes each utterance's probabilities independent of its batch; it
differs from the reference's forward_for_export only on ragged batches of more than one utterance, where the reference
averages over padding.

CPU: this file's restatement of that rule (`emo_probs`) against a real reference GigaAMEmo, the state_dict schema, the
load-time refusals of unsupported heads and the missing CPU path.  GPU: the kernel against float64 with derived bounds,
bit-identity under batching, the full model against the oracle, `model.head`, CUDA-graph replay and an opportunistic
known-answer test."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

import gigaam_b200 as gigaam
from gigaam_b200 import synthetic
from oracle import gigaam_oracle as orc
from oracle import ref_loader

D = 768
U = 2.0 ** -24        # unit roundoff of fp32
CHUNK = 32            # kPoolChunk of csrc/kernels.h: frames summed per CTA of the first kernel


def gamma(k):
    """gamma_k = k u / (1 - k u): relative bound of k consecutive fp32 roundings (Higham, Accuracy and Stability, §3.1)."""
    return k * U / (1 - k * U)


# ------------------------------------------------------------------------------------------ CPU restatement (the oracle)
def emo_pool(enc, enc_len, batch_of_one=None):
    """Decision 1 on the reference's layout: enc [B, d, T] -> [B, d], the mean over n_b = enc_len[b] frames, or over all T
    frames for a batch of one (gigaam/model.py:278-280 pools every frame of get_probs' one utterance)."""
    B, _, T = enc.shape
    if batch_of_one is None:
        batch_of_one = B == 1
    n = [T] * B if (enc_len is None or batch_of_one) else [int(v) for v in enc_len]
    return torch.stack([enc[b, :, : n[b]].mean(-1) for b in range(B)])


def emo_probs(enc, enc_len, sd, batch_of_one=None):
    """gigaam/model.py:272-293 with Decision 1's pooling: softmax(head(mean)) -> [B, C]"""
    return F.softmax(F.linear(emo_pool(enc, enc_len, batch_of_one), sd["head.weight"], sd["head.bias"]), dim=-1)


def _emo_ckpt(n_layers=None, num_classes=None, seed=0):
    cfg = synthetic.emo_cfg(n_layers, num_classes)
    return {"cfg": cfg, "state_dict": synthetic.synthetic_state_dict(cfg, seed)}


# ------------------------------------------------------------------------------------------ CPU: against the reference
@pytest.fixture(scope="module")
def ref_emo():
    """A real gigaam.model.GigaAMEmo built without hydra: the reference's preprocessor and 2-layer v1 encoder, a
    torch.nn.Linear head loaded from the synthetic state_dict and an in-memory prepare_wav."""
    if ref_loader.reference_root() is None:
        pytest.skip("the reference is neither in its source tree nor compiled into oracle/_ref")
    before, path = set(sys.modules), list(sys.path)
    try:
        ref_loader.import_reference()
        import gigaam.model as ref_model
        ck = _emo_ckpt(n_layers=2, seed=5)
        cfg, sd = ck["cfg"], ck["state_dict"]
        body, _ = ref_loader.build_reference({k: v for k, v in cfg.items() if k != "head"},
                                             {k: v for k, v in sd.items() if not k.startswith("head.")})
        m = ref_model.GigaAMEmo.__new__(ref_model.GigaAMEmo)
        torch.nn.Module.__init__(m)
        m.cfg = cfg
        m.preprocessor, m.encoder = body.preprocessor, body.encoder
        m.head = torch.nn.Linear(D, len(cfg["id2name"]))
        m.head.load_state_dict({"weight": sd["head.weight"], "bias": sd["head.bias"]}, strict=True)
        m.id2name = cfg["id2name"]
        m.prepare_wav = lambda wav: (wav[None].float(), torch.tensor([wav.numel()]))
        return m.eval(), ck
    finally:
        for k in set(sys.modules) - before:
            if k.split(".")[0] in ("gigaam", "hydra", "omegaconf", "soundfile"):
                del sys.modules[k]
        sys.path[:] = path


def _ragged_wavs(secs, seed):
    wavs = [synthetic.synthetic_audio(1, s, seed=seed + i)[0][0] for i, s in enumerate(secs)]
    n = max(w.numel() for w in wavs)
    batch = torch.zeros(len(wavs), n)
    for b, w in enumerate(wavs):
        batch[b, : w.numel()] = w
    return wavs, batch, torch.tensor([w.numel() for w in wavs])


def test_oracle_equals_reference_get_probs_and_export(ref_emo):
    ref, ck = ref_emo
    sd = ck["state_dict"]
    wavs, batch, lens = _ragged_wavs([3.0, 2.2, 1.4], seed=40)
    with torch.inference_mode():
        # get_probs: the dict in id2name order, equal to the oracle on the reference's own encoder output
        for w in wavs:
            got = ref.get_probs(w)
            assert list(got) == ck["cfg"]["id2name"]
            enc, enc_len = ref.forward(w[None], torch.tensor([w.numel()]))
            want = emo_probs(enc, enc_len, sd)[0]
            assert max(abs(got[k] - float(want[i])) for i, k in enumerate(got)) <= 1e-6
        # forward_for_export on a full-length batch and on a padded batch of one: pools every frame, as the oracle does
        full = torch.stack([w[: wavs[2].numel()] for w in wavs])
        full_len = torch.full((3,), wavs[2].numel())
        for wv, wl in ((full, full_len), (batch[1:2], lens[1:2])):
            mel, mel_len = ref.preprocessor(wv, wl)
            got = ref.forward_for_export(mel, mel_len)
            enc, enc_len = ref.encoder(mel, mel_len)
            assert float((got - emo_probs(enc, enc_len, sd)).abs().max()) <= 1e-6
        assert int(enc_len[0]) < enc.shape[-1], "the batch of one must be padded"
        # ragged batch: the reference's rows move with the padding; the oracle's equal each utterance alone
        alone = torch.stack([torch.tensor(list(ref.get_probs(w).values())) for w in wavs])
        mel, mel_len = ref.preprocessor(batch, lens)
        theirs = ref.forward_for_export(mel, mel_len)
        enc, enc_len = ref.encoder(mel, mel_len)
        ours = emo_probs(enc, enc_len, sd)
    # the reference's valid frames near a padded end are not quite those of the utterance alone (its subsampling convs
    # read the padded log-mel): 3.2e-4 measured, against 0.30 and 0.53 for the reference's padded rows
    assert float((ours - alone).abs().max()) <= 1e-3
    assert float((theirs[1:] - alone[1:]).abs().max(1).values.min()) > 0.05, "padding no longer moves the reference's rows"
    assert float((theirs[0] - alone[0]).abs().max()) <= 1e-4      # the full-length utterance has no padding


def test_synthetic_emo_checkpoint_loads_strictly_with_the_reference_keys(ref_emo):
    ref, _ = ref_emo
    ck = synthetic.synthetic_checkpoint("emo", n_layers=2, seed=5)
    assert ck["cfg"]["head"] == {"_target_": "torch.nn.Linear", "in_features": 768, "out_features": 4, "bias": True}
    assert ck["cfg"]["id2name"] == ["angry", "sad", "neutral", "positive"]
    assert ck["cfg"]["encoder"]["self_attention_model"] == "rel_pos" and ck["cfg"]["encoder"]["subsampling"] == "conv2d"
    model = gigaam.GigaAMEmo(ck["cfg"])
    model.load_state_dict(ck["state_dict"], strict=True)
    assert set(model.state_dict()) == set(ref.state_dict()) == set(ck["state_dict"])   # registration orders differ
    assert list(model.state_dict())[-2:] == list(ref.state_dict())[-2:] == ["head.weight", "head.bias"]
    assert model.id2name == ck["cfg"]["id2name"]
    assert [k for k, _ in model.head.named_parameters()] == ["weight", "bias"]


# ------------------------------------------------------------------------------------------ CPU: refusals, no CPU path
def _refused(monkeypatch, ck, *needles):
    def no_device_work(*a, **k):
        raise AssertionError("device work before the head was checked")
    monkeypatch.setattr(torch.nn.Module, "to", no_device_work)
    monkeypatch.setattr(gigaam.model.Engine, "__init__", no_device_work)
    with pytest.raises(NotImplementedError) as e:
        gigaam.load_model("emo", device="cpu", checkpoint=ck)
    for s in needles:
        assert s in str(e.value), (s, str(e.value))


def test_unknown_emo_head_is_refused_with_its_target_and_keys(monkeypatch):
    ck = _emo_ckpt(n_layers=1)
    ck["cfg"]["head"] = {"_target_": "mypkg.heads.MLPHead", "hidden": 256}
    sd = {k: v for k, v in ck["state_dict"].items() if not k.startswith("head.")}
    sd["head.fc1.weight"], sd["head.fc2.weight"] = torch.zeros(256, 768), torch.zeros(4, 256)
    ck["state_dict"] = sd
    _refused(monkeypatch, ck, "mypkg.heads.MLPHead", "Linear", "head.fc1.weight", "head.fc2.weight")


@pytest.mark.parametrize("change,needle", [
    (dict(out_features=5), "len(id2name)"),
    (dict(in_features=512), "in_features 512"),
    (dict(bias=False), "without bias"),
])
def test_mismatched_linear_head_is_refused(monkeypatch, change, needle):
    ck = _emo_ckpt(n_layers=1)
    ck["cfg"]["head"].update(change)
    _refused(monkeypatch, ck, needle, "head.weight", "head.bias")


def test_more_than_256_classes_are_refused(monkeypatch):
    _refused(monkeypatch, _emo_ckpt(n_layers=1, num_classes=257), "257 classes outside [1, 256]")
    monkeypatch.undo()
    assert gigaam.load_model("emo", device="cpu", checkpoint=_emo_ckpt(n_layers=1, num_classes=256)).head.out_features == 256


def test_emo_model_on_cpu_has_no_compute_path():
    model = gigaam.load_model("emo", device="cpu", synthetic=True)
    assert type(model) is gigaam.GigaAMEmo and model.id2name == synthetic.EMO_CLASSES
    assert model.head.weight.dtype == torch.float32
    with pytest.raises(RuntimeError, match="no CPU"):
        model.get_probs(torch.zeros(16000))
    with pytest.raises(RuntimeError, match="no CPU"):
        model.forward_for_export(torch.zeros(1, 64, 100), torch.tensor([100]))
    with pytest.raises(RuntimeError, match="no CPU"):
        model.head(torch.zeros(2, 768))
    assert "GigaAMEmo" in gigaam.__all__


# ------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (there is no CPU fallback to test instead)"
    return torch.device("cuda", 0)


_MODELS = {}


def _head_model(C, dev):
    """A 1-layer emo model with C classes: only its head is used by the kernel tests."""
    if C not in _MODELS:
        ck = _emo_ckpt(n_layers=1, num_classes=None if C == 4 else C, seed=C)
        _MODELS[C] = (gigaam.load_model("emo", device=dev, checkpoint=ck), ck)
    return _MODELS[C]


def _kernel_inputs(B, T, lens, seed, dev):
    """[B, T, 768] f32 with per-utterance offsets and scales; frames t >= n_b and a whole utterance's worth of rows behind
    the buffer are NaN (a batch of one keeps every frame: it pools all T)."""
    g = torch.Generator().manual_seed(seed)
    off = torch.randn(B, 1, 1, generator=g) * 20
    scale = torch.rand(B, 1, 1, generator=g) * 4 + 0.1
    buf = torch.full(((B + 1) * T * D,), float("nan"))
    x = buf[: B * T * D].view(B, T, D)
    x.copy_(torch.randn(B, T, D, generator=g) * scale + off)
    if lens is not None and B > 1:
        x[torch.arange(T)[None, :] >= torch.tensor(lens)[:, None]] = float("nan")
    return buf.to(dev)[: B * T * D].view(B, T, D), x


def _check_kernel_outputs(x, lens, sd, pooled, logits, probs):
    """Each element against float64 within the bound of the fp32 arithmetic the kernels perform."""
    B, T, _ = x.shape
    n = [T] * B if (lens is None or B == 1) else list(lens)
    W, b = sd["head.weight"].double(), sd["head.bias"].double()
    C = W.shape[0]
    pooled, logits, probs = pooled.cpu(), logits.cpu(), probs.cpu()
    for i in range(B):
        if n[i] == 0:
            assert bool(pooled[i].isnan().all() and logits[i].isnan().all() and probs[i].isnan().all()), i
            continue
        xs = x[i, : n[i]].double()
        want = xs.mean(0)
        # pooled: kPoolChunk-frame sums in ascending t (<= 31 roundings each; the first frame is taken as it is), then the
        # nc chunk sums from 0.0 in ascending order (nc roundings), then one division.  Every term meets at most
        # k = 31 + nc roundings, so |sum_hat - sum| <= gamma_k sum|x| and |mean_hat - mean| <= gamma_k (1 + u) mean|x| + u |mean|.
        k = 31 + math.ceil(n[i] / CHUNK)
        tol = gamma(k) * (1 + U) * xs.abs().mean(0) + U * want.abs()
        assert bool(((pooled[i].double() - want).abs() <= tol).all()), (i, float((pooled[i].double() - want).abs().max()))
        # logits from the kernel's own pooled vector: per lane 24 fmaf (one rounding each), 5 xor-shuffle adds, + bias:
        # at most 30 roundings per term, |err| <= gamma_30 (sum_k |W_ck p_k| + |b_c|)
        p = pooled[i].double()
        want_l = W @ p + b
        tol_l = gamma(30) * (W.abs() @ p.abs() + b.abs())
        assert bool(((logits[i].double() - want_l).abs() <= tol_l).all()), i
        # probs from the kernel's own logits v: m = max v is exact; d = fl(v - m) moves e = exp(d) by a factor
        # exp(u |d|); expf adds <= 2 ulp (4u, CUDA C Programming Guide, maximum ulp error of expf), so
        # r_c = (1 + 4u) exp(u |d_c|) - 1.  The sum S >= 1 (exp(0) = 1 exactly) takes <= 12 roundings (5 in the warp tree, 7
        # across the 8 warps) and sum_c e_c u |d_c| <= C u / e (x exp(-x) <= 1/e), so S's relative error is
        # rho <= (C u / e + 4u)(1 + gamma_12) + gamma_12; the division adds u.  Underflowed terms (d < -87) get 2^-126 absolute.
        v = logits[i].double()
        d = v - v.max()
        want_p = torch.softmax(v, 0)
        r = (1 + 4 * U) * torch.exp(U * d.abs()) - 1
        rho = (C * U / math.e + 4 * U) * (1 + gamma(12)) + gamma(12)
        tol_p = want_p * ((1 + r) * (1 + U) / (1 - rho) - 1) + 2.0 ** -126
        assert bool(((probs[i].double() - want_p).abs() <= tol_p).all()), (i, float((probs[i].double() - want_p).abs().max()))


_KERNEL_CASES = [
    # (B, T, lengths): 0, 1, chunk - 1, chunk, chunk + 1 and T in one batch, up to T = 5000 and B = 64
    (6, 5000, [0, 1, CHUNK - 1, CHUNK, CHUNK + 1, 5000]),
    (64, 251, None),
    (1, 77, [40]),              # a batch of one pools all T frames, whatever its length says
    (3, 40, "none"),            # enc_len = NULL: all T frames
]


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 4, 33, 256])
@pytest.mark.parametrize("case", range(len(_KERNEL_CASES)))
def test_emo_head_kernel_against_float64(dev, C, case):
    model, ck = _head_model(C, dev)
    B, T, lens = _KERNEL_CASES[case]
    if lens is None:
        g = torch.Generator().manual_seed(C)
        lens = [0, 1, CHUNK - 1, CHUNK, CHUNK + 1, T] + torch.randint(0, T + 1, (B - 6,), generator=g).tolist()
    no_len = lens == "none"
    xd, x = _kernel_inputs(B, T, None if no_len else lens, seed=100 * C + case, dev=dev)
    eng = model._get_engine()
    with torch.inference_mode():
        enc_len = None if no_len else torch.tensor(lens, dtype=torch.int32, device=dev)
        pooled, logits, probs = eng.emo_head(xd, enc_len)
        torch.cuda.synchronize()
    assert pooled.shape == (B, D) and logits.shape == probs.shape == (B, C)
    _check_kernel_outputs(x, None if no_len else lens, ck["state_dict"], pooled, logits, probs)


@pytest.mark.gpu
def test_emo_head_is_bit_identical_under_batching(dev):
    """One utterance of 300 frames in batches with other neighbours, B and T' widths (and alone, where T = its length)."""
    model, _ = _head_model(33, dev)
    eng = model._get_engine()
    g = torch.Generator().manual_seed(8)
    utt = torch.randn(300, D, generator=g) * 3 + 1
    outs = []
    for B, T, pos in ((5, 300, 2), (17, 700, 11), (2, 350, 0), (64, 301, 63), (1, 300, 0)):
        x = torch.randn(B, T, D, generator=g) * 5 - 2
        lens = torch.randint(0, T + 1, (B,), generator=g)
        x[pos, :300], lens[pos] = utt, 300
        with torch.inference_mode():
            outs.append([t[pos].cpu() for t in eng.emo_head(x.to(dev), lens.to(dev))])
    for o in outs[1:]:
        for a, w in zip(o, outs[0]):
            assert torch.equal(a, w)


_FULL = {}


def _full_model(dev, max_encoded_frames=None):
    if max_encoded_frames not in _FULL:
        model = gigaam.load_model("emo", device=dev, synthetic=True, max_encoded_frames=max_encoded_frames)
        ck = synthetic.synthetic_checkpoint("emo")
        sd16 = {k: (v.half().float() if k.startswith("encoder.") and v.is_floating_point() else v) for k, v in ck["state_dict"].items()}
        _FULL[max_encoded_frames] = (model, ck["cfg"], sd16)
    return _FULL[max_encoded_frames]


def _probs_tol(enc_o, enc_len, sd, batch_of_one):
    """Probability tolerance per utterance from the encoder's 1e-3 relative-Frobenius bar (DESIGN §2): if the encoder output
    E_b of n frames moves by ||dE||_F <= 1e-3 ||E_b||_F, the mean moves by <= ||dE||_F / sqrt(n) (Cauchy-Schwarz), the
    logits by <= ||W||_2 times that, and the probabilities by <= 1/2 of the logits' move (||diag(p) - p p^T||_2 <= 1/2)."""
    B, _, T = enc_o.shape
    w2 = float(torch.linalg.matrix_norm(sd["head.weight"].double(), ord=2))
    tol = []
    for b in range(B):
        n = T if batch_of_one else int(enc_len[b])
        tol.append(0.5 * w2 * 1e-3 * float(enc_o[b, :, :n].norm()) / math.sqrt(n))
    return torch.tensor(tol)


@pytest.mark.gpu
@pytest.mark.parametrize("secs", [1.0, 10.0, 30.0])
def test_get_probs_against_oracle(dev, secs):
    model, cfg, sd16 = _full_model(dev)
    wav = synthetic.synthetic_audio(1, secs, seed=int(secs) + 3)[0][0]
    got = model.get_probs(wav)
    assert list(got) == synthetic.EMO_CLASSES and all(isinstance(v, float) for v in got.values())
    with torch.inference_mode():
        enc_o, len_o = orc.model_forward(wav[None].half().float(), torch.tensor([wav.numel()]), sd16, cfg)
    want = emo_probs(enc_o, len_o, sd16)[0]
    tol = float(_probs_tol(enc_o, len_o, sd16, True)[0])
    assert max(abs(got[k] - float(want[i])) for i, k in enumerate(got)) <= tol
    assert abs(sum(got.values()) - 1.0) <= 1e-5


@pytest.mark.gpu
def test_forward_for_export_ragged_batch_against_oracle_and_get_probs(dev):
    model, cfg, sd16 = _full_model(dev)
    wav, wav_len = synthetic.synthetic_audio(16, 4.0, seed=77, ragged=True)
    with torch.inference_mode():
        mel, mel_len = model.preprocessor(wav.to(dev), wav_len.to(dev))
        probs = model.forward_for_export(mel, mel_len).cpu()
        rev = model.forward_for_export(mel.flip(0), mel_len.flip(0)).flip(0).cpu()
        enc_o, len_o = orc.model_forward(wav, wav_len, sd16, cfg)
    assert probs.shape == (16, 4)
    want = emo_probs(enc_o, len_o, sd16)
    tol = _probs_tol(enc_o, len_o, sd16, False)
    assert bool(((probs - want).abs().max(1).values <= tol).all())
    assert torch.equal(rev, probs), "an utterance's row changed with its position in a batch of the same width"
    alone = torch.stack([torch.tensor(list(model.get_probs(wav[b, : int(wav_len[b])]).values())) for b in range(16)])
    # both sides within `tol` of their oracle rows, which agree to fp32 round-off; get_probs also rounds the wav to fp16
    alone_o = torch.stack([emo_probs(*orc.model_forward(wav[b:b + 1, : int(wav_len[b])].half().float(), wav_len[b:b + 1], sd16, cfg),
                                     sd16)[0] for b in range(16)])
    assert bool(((alone - alone_o).abs().max(1).values <= tol).all())
    assert bool(((alone - probs).abs().max(1).values <= 2 * tol + (alone_o - want).abs().max(1).values).all())


@pytest.mark.gpu
def test_get_probs_60s_on_a_long_model(dev):
    model, cfg, sd16 = _full_model(dev, max_encoded_frames=5000)
    wav = synthetic.synthetic_audio(1, 60.0, seed=60)[0][0]
    got = torch.tensor(list(model.get_probs(wav).values()))
    with torch.inference_mode():
        enc_o, len_o = orc.model_forward(wav[None].half().float(), torch.tensor([wav.numel()]), sd16, cfg)
    assert enc_o.shape[-1] > 768
    want = emo_probs(enc_o, len_o, sd16)[0]
    assert float((got - want).abs().max()) <= float(_probs_tol(enc_o, len_o, sd16, True)[0])


@pytest.mark.gpu
def test_head_forward_against_float64_linear(dev):
    model, ck = _head_model(33, dev)
    sd = ck["state_dict"]
    g = torch.Generator().manual_seed(3)
    for shape in ((5, D), (2, 3, D), (D,)):
        x = torch.randn(*shape, generator=g) * 4 + 1
        with torch.inference_mode():
            got = model.head(x.to(dev)).cpu()
        assert got.shape == (*shape[:-1], 33)
        xs = x.reshape(-1, D).double()
        want = F.linear(xs, sd["head.weight"].double(), sd["head.bias"].double())
        # a mean over one frame is the frame itself (no rounding), so the logits bound of the kernel test applies
        tol = gamma(30) * (xs.abs() @ sd["head.weight"].double().abs().t() + sd["head.bias"].double().abs())
        assert bool(((got.reshape(-1, 33).double() - want).abs() <= tol).all())
    with pytest.raises(RuntimeError, match="no CPU"):
        model.head(torch.zeros(2, D))


@pytest.mark.gpu
def test_graph_capture_of_wav_to_probs_replays_bit_exact(dev):
    model, _, _ = _full_model(dev)
    wav, wav_len = synthetic.synthetic_audio(4, 3.0, seed=19, ragged=True)
    wav, wav_len = wav.to(dev), wav_len.to(dev)

    def step():
        return model.forward_for_export(*model.preprocessor(wav, wav_len))

    with torch.inference_mode():
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
    assert torch.equal(out, eager)


_KNOWN = {"angry": 7.70451661082916e-05, "sad": 0.002205904107540846, "neutral": 0.9233596324920654,
          "positive": 0.07435736805200577}    # the reference's tests/test_loading.py:13-18


@pytest.mark.gpu
def test_known_answer_when_the_real_checkpoint_is_present(dev):
    """The only check of the RECALLED head class (torch.nn.Linear(768, 4) under `head.weight` / `head.bias`): with the
    real emo checkpoint and the reference's example.wav, get_probs must give the reference's values within 1e-3."""
    ckpt = os.path.expanduser("~/.cache/gigaam/emo.ckpt")
    wav = next((p for p in ("example.wav", os.path.expanduser("~/.cache/gigaam/example.wav")) if os.path.isfile(p)), None)
    if not os.path.isfile(ckpt) or wav is None:
        pytest.skip("needs ~/.cache/gigaam/emo.ckpt and example.wav (not available offline)")
    got = gigaam.load_model("emo", device=dev).get_probs(wav)
    assert list(got) == list(_KNOWN)
    assert all(abs(got[k] - _KNOWN[k]) < 1e-3 for k in _KNOWN), got
