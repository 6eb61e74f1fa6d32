"""Synthetic checkpoints and audio (there are no real checkpoints or network in the build/bench boxes).

`synthetic_checkpoint(name)` returns the same `{"cfg": ..., "state_dict": ...}` structure the reference
loads from `<name>.ckpt` (gigaam/__init__.py:167): a plain-dict cfg whose sections mirror the Hydra cfg
(`preprocessor`, `encoder`, `head`, `decoding`) and a state_dict with the reference's key names
(SURVEY Appendix B).  Weights are seeded, finite and well-scaled; eval-BatchNorm statistics are
randomised so that BN folding is actually exercised.

`synthetic_audio(batch, seconds)` is the reference's own test signal (tests/test_batching.py:15-25).
"""
from __future__ import annotations

import math
from pathlib import Path
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

SAMPLE_RATE = 16000

_CHAR_VOCAB = [" "] + [chr(c) for c in range(ord("а"), ord("я") + 1)]  # 33 symbols -> V+1 = 34
assert len(_CHAR_VOCAB) == 33

# Per-model calibration of the synthetic RNN-T joint network, written by oracle/calibrate_rnnt.py (random weights
# otherwise emit max_symbols tokens on every frame or none at all, SURVEY 8d): the mean encoder frame that
# `head.joint.enc.bias` cancels, the utterance-to-utterance directions `head.joint.enc.weight` is made blind to, and the
# blank-logit bias that lands the token rate on BASELINE.md's target.
RNNT_CALIBRATION_FILE = Path(__file__).with_name("rnnt_calibration.npz")


def _rnnt_calibration(model_name: str) -> Dict:
    if not RNNT_CALIBRATION_FILE.exists():
        return {}
    with np.load(RNNT_CALIBRATION_FILE) as z:
        return {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(model_name + "/")}


def _encoder_cfg(version: str) -> Dict:
    if version == "v3":  # RECALLED shape (SURVEY Appendix C); a real checkpoint's cfg overrides it
        return dict(feat_in=64, n_layers=16, d_model=768, subsampling="conv1d", subs_kernel_size=5,
                    subsampling_factor=4, ff_expansion_factor=4, self_attention_model="rotary", n_heads=16,
                    pos_emb_max_len=5000, conv_norm_type="layer_norm", conv_kernel_size=5, flash_attn=False)
    # v1: the Transformer-XL relative-position attention of gigaam/encoder.py:191-228 (RECALLED to be the v1_* setting)
    return dict(feat_in=64, n_layers=16, d_model=768, subsampling="conv2d", subs_kernel_size=3,
                subsampling_factor=4, ff_expansion_factor=4, self_attention_model="rel_pos" if version == "v1" else "rotary",
                n_heads=16, pos_emb_max_len=5000, conv_norm_type="batch_norm", conv_kernel_size=31, flash_attn=False)


def model_cfg(model_name: str, n_layers: int | None = None) -> Dict:
    """Plain-dict cfg for a model name of the reference's registry (gigaam/__init__.py:28-41)."""
    if model_name == "emo":
        return emo_cfg(n_layers)
    version = model_name.split("_")[0]
    if version not in ("v1", "v2", "v3"):
        raise ValueError(f"unknown synthetic model {model_name!r}")
    enc = _encoder_cfg(version)
    if n_layers is not None:
        enc["n_layers"] = n_layers
    pre = dict(sample_rate=SAMPLE_RATE, features=64)
    if version == "v3":
        pre.update(win_length=320, n_fft=320, hop_length=160, center=False)
    cfg: Dict = dict(model_name=model_name, sample_rate=SAMPLE_RATE, preprocessor=pre, encoder=enc)
    kind = model_name.split("_", 1)[1]
    if kind == "ssl":
        return cfg
    e2e = "e2e" in kind
    vocab = [f"<{i}>" for i in range(256 if "ctc" in kind else 1024)] if e2e else list(_CHAR_VOCAB)
    ncls = len(vocab) + 1
    if "ctc" in kind:
        cfg["head"] = dict(type="ctc", feat_in=enc["d_model"], num_classes=ncls)
        cfg["decoding"] = dict(type="ctc", vocabulary=vocab)
    elif "rnnt" in kind:
        cfg["head"] = dict(type="rnnt",
                           decoder=dict(pred_hidden=320, pred_rnn_layers=1, num_classes=ncls),
                           joint=dict(enc_hidden=enc["d_model"], pred_hidden=320, joint_hidden=320, num_classes=ncls))
        cfg["decoding"] = dict(type="rnnt", vocabulary=vocab, max_symbols_per_step=10)
    else:
        raise ValueError(f"unknown synthetic model {model_name!r}")
    return cfg


EMO_CLASSES = ["angry", "sad", "neutral", "positive"]   # order of the reference's expected values (tests/test_loading.py:13-18)


def emo_cfg(n_layers: int | None = None, num_classes: int | None = None) -> Dict:
    """GigaAM-Emo: a v1 encoder (README.md:56) and a Linear(768, C) head over the mean of the encoder frames
    (gigaam/model.py:262-293).  The head's `_target_` is RECALLED to be torch.nn.Linear: the reference instantiates a class
    outside `gigaam` that maps [B, 768] -> [B, C].  `num_classes` (default 4) replaces the class list by C generic names."""
    enc = _encoder_cfg("v1")
    if n_layers is not None:
        enc["n_layers"] = n_layers
    names = list(EMO_CLASSES) if num_classes is None else [f"class_{i}" for i in range(num_classes)]
    return dict(model_name="emo", sample_rate=SAMPLE_RATE, preprocessor=dict(sample_rate=SAMPLE_RATE, features=64), encoder=enc,
                head={"_target_": "torch.nn.Linear", "in_features": enc["d_model"], "out_features": len(names), "bias": True},
                id2name=names)


def head_kind(head) -> Optional[str]:
    """"ctc" | "rnnt" | "emo" for a head section (a normalized cfg carries `type`; the emo head is named by its
    `_target_`), None without a head."""
    if not head:
        return None
    if "type" in head:
        return head["type"]
    return "emo" if str(head.get("_target_", "")).rsplit(".", 1)[-1] == "Linear" else None


# ------------------------------------------------------------------------------------------ front-end buffers
def hann_window(n: int) -> torch.Tensor:
    """Periodic Hann window (torch.hann_window default, used by torchaudio Spectrogram)."""
    k = torch.arange(n, dtype=torch.float64)
    return (0.5 - 0.5 * torch.cos(2.0 * math.pi * k / n)).to(torch.float32)


def mel_filterbank(n_freqs: int, n_mels: int, sample_rate: int) -> torch.Tensor:
    """HTK mel triangles, f_min=0, f_max=sr/2, norm=None -> [n_freqs, n_mels] (torchaudio melscale_fbanks)."""
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs)
    m_min = 2595.0 * math.log10(1.0 + 0.0 / 700.0)
    m_max = 2595.0 * math.log10(1.0 + (sample_rate / 2.0) / 700.0)
    m_pts = torch.linspace(m_min, m_max, n_mels + 2)
    f_pts = 700.0 * (10 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    down = (-1.0 * slopes[:, :-2]) / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    return torch.clamp(torch.min(down, up), min=0.0).to(torch.float32)


# ------------------------------------------------------------------------------------------ weights
# Random heads are nearly input-independent (every frame gives the same argmax); these gains make the joint
# network's logits depend on the frame and on the prediction-network state so that greedy decoding is not a
# degenerate all-or-nothing function of the blank bias.
_GAIN = {"head.joint.joint_net.1.weight": 6.0, "head.joint.enc.weight": 20.0, "head.joint.pred.weight": 10.0,
         "head.decoder_layers.0.weight": 4.0, "head.weight": 4.0}

def _param_list(cfg: Dict) -> List[Tuple[str, Tuple[int, ...], str, float]]:
    """(key, shape, kind, fan_in) in a fixed order.  kind: w|b|ln_w|ln_b|bn_mean|bn_var|int|emb"""
    return encoder_param_list(cfg["encoder"]) + head_param_list(cfg.get("head"))


def encoder_param_list(enc: Dict) -> List[Tuple[str, Tuple[int, ...], str, float]]:
    """state_dict entries of gigaam.encoder.ConformerEncoder (keys carry the "encoder." prefix)."""
    d, L = enc["d_model"], enc["n_layers"]
    ff = d * enc["ff_expansion_factor"]
    k = enc["subs_kernel_size"]
    out: List[Tuple[str, Tuple[int, ...], str, float]] = []

    def lin(prefix: str, o: int, i: int, bias: bool = True):
        out.append((prefix + ".weight", (o, i), "w", i))
        if bias:
            out.append((prefix + ".bias", (o,), "b", i))

    def ln(prefix: str):
        out.append((prefix + ".weight", (d,), "ln_w", 0))
        out.append((prefix + ".bias", (d,), "ln_b", 0))

    p = "encoder.pre_encode."
    if enc["subsampling"] == "conv2d":
        out.append((p + "conv.0.weight", (d, 1, k, k), "w", k * k))
        out.append((p + "conv.0.bias", (d,), "b", k * k))
        out.append((p + "conv.2.weight", (d, d, k, k), "w", d * k * k))
        out.append((p + "conv.2.bias", (d,), "b", d * k * k))
        f = enc["feat_in"]
        for _ in range(2):
            f = (f + 2 * ((k - 1) // 2) - k) // 2 + 1
        lin(p + "out", d, d * f)
    else:
        out.append((p + "conv.0.weight", (d, enc["feat_in"], k), "w", enc["feat_in"] * k))
        out.append((p + "conv.0.bias", (d,), "b", enc["feat_in"] * k))
        out.append((p + "conv.2.weight", (d, d, k), "w", d * k))
        out.append((p + "conv.2.bias", (d,), "b", d * k))
    ck = enc["conv_kernel_size"]
    for l in range(L):
        q = f"encoder.layers.{l}."
        ln(q + "norm_feed_forward1")
        lin(q + "feed_forward1.linear1", ff, d)
        lin(q + "feed_forward1.linear2", d, ff)
        ln(q + "norm_conv")
        out.append((q + "conv.pointwise_conv1.weight", (2 * d, d, 1), "w", d))
        out.append((q + "conv.pointwise_conv1.bias", (2 * d,), "b", d))
        out.append((q + "conv.depthwise_conv.weight", (d, 1, ck), "w", ck))
        out.append((q + "conv.depthwise_conv.bias", (d,), "b", ck))
        out.append((q + "conv.batch_norm.weight", (d,), "ln_w", 0))
        out.append((q + "conv.batch_norm.bias", (d,), "ln_b", 0))
        if enc["conv_norm_type"] == "batch_norm":
            out.append((q + "conv.batch_norm.running_mean", (d,), "bn_mean", 0))
            out.append((q + "conv.batch_norm.running_var", (d,), "bn_var", 0))
            out.append((q + "conv.batch_norm.num_batches_tracked", (), "int", 0))
        out.append((q + "conv.pointwise_conv2.weight", (d, d, 1), "w", d))
        out.append((q + "conv.pointwise_conv2.bias", (d,), "b", d))
        ln(q + "norm_self_att")
        for nm in ("linear_q", "linear_k", "linear_v", "linear_out"):
            lin(q + "self_attn." + nm, d, d)
        if enc["self_attention_model"] == "rel_pos":
            # the reference leaves pos_bias_u / pos_bias_v uninitialised (torch.FloatTensor, encoder.py:199-200); a
            # checkpoint always overwrites them, so the synthetic one draws them like biases
            dk = d // enc["n_heads"]
            lin(q + "self_attn.linear_pos", d, d, bias=False)
            out.append((q + "self_attn.pos_bias_u", (enc["n_heads"], dk), "b", dk))
            out.append((q + "self_attn.pos_bias_v", (enc["n_heads"], dk), "b", dk))
        ln(q + "norm_feed_forward2")
        lin(q + "feed_forward2.linear1", ff, d)
        lin(q + "feed_forward2.linear2", d, ff)
        ln(q + "norm_out")
    return out


def head_param_list(head) -> List[Tuple[str, Tuple[int, ...], str, float]]:
    """state_dict entries of gigaam.decoder.CTCHead / RNNTHead and of the emo model's torch.nn.Linear head (keys carry
    the "head." prefix)."""
    out: List[Tuple[str, Tuple[int, ...], str, float]] = []

    def lin(prefix: str, o: int, i: int):
        out.append((prefix + ".weight", (o, i), "w", i))
        out.append((prefix + ".bias", (o,), "b", i))

    kind = head_kind(head)
    if kind == "emo":
        out.append(("head.weight", (head["out_features"], head["in_features"]), "w", head["in_features"]))
        if head.get("bias", True):
            out.append(("head.bias", (head["out_features"],), "b", head["in_features"]))
    elif kind == "ctc":
        out.append(("head.decoder_layers.0.weight", (head["num_classes"], head["feat_in"], 1), "w", head["feat_in"]))
        out.append(("head.decoder_layers.0.bias", (head["num_classes"],), "b", head["feat_in"]))
    elif kind == "rnnt":
        dc, jt = head["decoder"], head["joint"]
        H = dc["pred_hidden"]
        out.append(("head.decoder.embed.weight", (dc["num_classes"], H), "emb", 0))
        for l in range(dc["pred_rnn_layers"]):
            out.append((f"head.decoder.lstm.weight_ih_l{l}", (4 * H, H), "w", H))
            out.append((f"head.decoder.lstm.weight_hh_l{l}", (4 * H, H), "w", H))
            out.append((f"head.decoder.lstm.bias_ih_l{l}", (4 * H,), "b", H))
            out.append((f"head.decoder.lstm.bias_hh_l{l}", (4 * H,), "b", H))
        lin("head.joint.pred", jt["joint_hidden"], jt["pred_hidden"])
        lin("head.joint.enc", jt["joint_hidden"], jt["enc_hidden"])
        lin("head.joint.joint_net.1", jt["num_classes"], jt["joint_hidden"])
    return out


def synthetic_state_dict(cfg: Dict, seed: int = 0, rnnt_calibration: Optional[Dict] = None) -> Dict[str, torch.Tensor]:
    """Seeded fp32 state_dict with the reference's key names and shapes.  `rnnt_calibration` overrides the stored
    calibration of an RNN-T head (`{}` = none: what oracle/calibrate_rnnt.py starts from)."""
    gen = torch.Generator(device="cpu")
    gen.manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    pre = cfg["preprocessor"]
    n_fft = pre.get("n_fft", pre["sample_rate"] // 40)
    sd["preprocessor.featurizer.0.spectrogram.window"] = hann_window(pre.get("win_length", n_fft))
    sd["preprocessor.featurizer.0.mel_scale.fb"] = mel_filterbank(n_fft // 2 + 1, pre["features"], pre["sample_rate"])
    for key, shape, kind, fan_in in _param_list(cfg):
        if kind == "w":
            bound = 1.0 / math.sqrt(fan_in)
            t = (torch.rand(shape, generator=gen) * 2 - 1) * bound
        elif kind == "b":
            bound = 1.0 / math.sqrt(fan_in)
            t = (torch.rand(shape, generator=gen) * 2 - 1) * bound
        elif kind == "ln_w":
            t = 1.0 + 0.1 * torch.randn(shape, generator=gen)
        elif kind == "ln_b":
            t = 0.05 * torch.randn(shape, generator=gen)
        elif kind == "bn_mean":
            t = 0.1 * torch.randn(shape, generator=gen)
        elif kind == "bn_var":
            t = 0.05 + 0.2 * torch.rand(shape, generator=gen)
        elif kind == "emb":
            t = torch.randn(shape, generator=gen)
            t[-1].zero_()  # padding_idx = blank row (gigaam/decoder.py:81)
        elif kind == "int":
            t = torch.tensor(0, dtype=torch.long)
        else:
            raise AssertionError(kind)
        sd[key] = t * _GAIN.get(key, 1.0)
    head = cfg.get("head")
    if head_kind(head) == "rnnt":
        cal = _rnnt_calibration(cfg["model_name"]) if rnnt_calibration is None else rnnt_calibration
        if "enc_null" in cal:       # rows orthogonal to the directions in which utterance means differ (oracle/calibrate_rnnt.py)
            null = torch.as_tensor(cal["enc_null"])
            w = sd["head.joint.enc.weight"]
            sd["head.joint.enc.weight"] = w - (w @ null.t()) @ null
        if "enc_mean" in cal:
            sd["head.joint.enc.bias"] = -(sd["head.joint.enc.weight"] @ torch.as_tensor(cal["enc_mean"]))
        sd["head.joint.joint_net.1.bias"][-1] += float(cal.get("blank_bias", 0.0))
    return sd


def synthetic_checkpoint(model_name: str, seed: int = 0, n_layers: int | None = None,
                         rnnt_calibration: Optional[Dict] = None) -> Dict:
    cfg = model_cfg(model_name, n_layers)
    return {"cfg": cfg, "state_dict": synthetic_state_dict(cfg, seed, rnnt_calibration)}


# ------------------------------------------------------------------------------------------ audio
def synthetic_audio(batch: int, seconds: float, seed: int = 1234, ragged: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """[B, N] float32 in [-1, 1] and int64 lengths.  Recipe of the reference's tests/test_batching.py:15-25:
    0.5 sin(2 pi 220 t) + 0.3 sin(2 pi 440 t) + 0.2 sin(2 pi 660 t) + 0.01 N(0,1), Tukey(alpha=0.1) envelope.
    Every utterance gets its own noise and a small per-utterance detune so that batches are not degenerate."""
    rng = np.random.default_rng(seed)
    n = int(round(seconds * SAMPLE_RATE))
    t = np.arange(n, dtype=np.float64) / SAMPLE_RATE
    wav = np.zeros((batch, n), dtype=np.float32)
    lengths = np.full((batch,), n, dtype=np.int64)
    for b in range(batch):
        det = 1.0 + 0.03 * rng.standard_normal()
        sig = (0.5 * np.sin(2 * np.pi * 220 * det * t) + 0.3 * np.sin(2 * np.pi * 440 * det * t)
               + 0.2 * np.sin(2 * np.pi * 660 * det * t) + 0.01 * rng.standard_normal(n))
        nb = n
        if ragged and b > 0:
            nb = int(n * rng.uniform(0.5, 1.0))
        alpha = 0.1
        w = np.ones(nb)
        edge = int(alpha * (nb - 1) / 2.0)
        if edge > 0:
            k = np.arange(edge + 1)
            ramp = 0.5 * (1 + np.cos(np.pi * (2.0 * k / (alpha * (nb - 1)) - 1.0)))
            w[: edge + 1] = ramp
            w[nb - edge - 1:] = ramp[::-1]
        wav[b, :nb] = (sig[:nb] * w).astype(np.float32)
        lengths[b] = nb
    return torch.from_numpy(wav), torch.from_numpy(lengths)
