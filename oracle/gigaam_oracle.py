"""ORACLE -- test infrastructure only.  Never imported by the product (gigaam_b200/).

CPU fp32 restatement (plain PyTorch, functional, state_dict-driven) of the reference's hot path:
log-mel -> Conformer encoder -> CTC / RNN-T greedy decode.  Every function cites the reference
file:line it restates (paths relative to salute-developers/GigaAM @ 85558932).

Pinning: `oracle/make_golden.py` imports the real reference modules from /root/reference (with hydra /
omegaconf / soundfile stubbed), loads the SAME seeded state_dict into them, runs them on the same
synthetic audio and (a) asserts this restatement agrees with them, (b) writes tests/golden/*.npz, which
`tests/test_oracle_golden.py` re-checks on every box (the reference itself cannot travel).  The
reference's own known-answer tests (tests/test_loading.py:19-21 transcripts etc.) need downloaded
checkpoints that do not exist offline, so parity is pinned to reference *outputs generated here*, not to
those strings.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / --impl reference leg may import
this module.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
SD = Dict[str, Tensor]


# ------------------------------------------------------------------------------------------ front end
def logmel_out_len(n: Tensor, hop: int, win: int, center: bool) -> Tensor:
    """gigaam/preprocess.py:78-92"""
    if center:
        return n.div(hop, rounding_mode="floor").add(1).long()
    return (n - win).div(hop, rounding_mode="floor").add(1).long()


def log_mel(wav: Tensor, sd: SD, pre: Dict) -> Tensor:
    """gigaam/preprocess.py:43-50,67-74,98 (torchaudio MelSpectrogram: Spectrogram(power=2, center,
    pad_mode='reflect', periodic Hann, onesided, not normalized) -> MelScale(fb) -> log(clamp(1e-9, 1e9)))."""
    sr = pre["sample_rate"]
    n_fft = pre.get("n_fft", sr // 40)
    hop = pre.get("hop_length", sr // 100)
    center = pre.get("center", True)
    window = sd["preprocessor.featurizer.0.spectrogram.window"].float()
    fb = sd["preprocessor.featurizer.0.mel_scale.fb"].float()
    x = wav.float()
    if center:
        x = F.pad(x.unsqueeze(1), (n_fft // 2, n_fft // 2), mode="reflect").squeeze(1)
    frames = x.unfold(-1, n_fft, hop)                       # [B, M, n_fft]
    spec = torch.fft.rfft(frames * window, dim=-1)          # [B, M, n_fft/2+1]
    power = spec.real ** 2 + spec.imag ** 2
    mel = torch.matmul(power, fb).transpose(1, 2)           # [B, n_mels, M]
    return torch.log(mel.clamp(1e-9, 1e9))


# ------------------------------------------------------------------------------------------ subsampling
def sub_out_len(lengths: Tensor, k: int, stages: int = 2) -> Tensor:
    """gigaam/encoder.py:77-90 (float arithmetic, floor, cast to int32)."""
    pad = (k - 1) // 2
    add_pad = 2 * pad - k
    l = lengths.to(torch.float)
    for _ in range(stages):
        l = torch.floor((l + add_pad) / 2 + 1.0)
    return l.to(torch.int)


def _mask_time(x: Tensor, lengths: Tensor) -> Tensor:
    """gigaam/encoder.py:92-109"""
    t = torch.arange(x.size(2))
    pad = (t[None, :] >= lengths[:, None])[:, None]
    if x.dim() == 4:
        pad = pad[..., None]
    return x.masked_fill(pad, 0.0)


def pre_encode(mel: Tensor, lengths: Tensor, sd: SD, enc: Dict) -> Tuple[Tensor, Tensor]:
    """gigaam/encoder.py:111-130 (StridingSubsampling.forward); mel is [B, F, M]."""
    k = enc["subs_kernel_size"]
    pad = (k - 1) // 2
    p = "encoder.pre_encode."
    x = mel.transpose(1, 2)                                  # encoder.py:609-611
    if enc["subsampling"] == "conv2d":
        x = x.unsqueeze(1)
        conv = F.conv2d
    else:
        x = x.transpose(1, 2)
        conv = F.conv1d
    cur = lengths
    x = _mask_time(x, cur)
    for i in (0, 2):
        x = conv(x, sd[f"{p}conv.{i}.weight"], sd[f"{p}conv.{i}.bias"], stride=2, padding=pad)
        cur = sub_out_len(cur, k, 1)
        x = _mask_time(x, cur)
        x = F.relu(x)
    if enc["subsampling"] == "conv2d":
        b, _, t, _ = x.shape
        x = F.linear(x.transpose(1, 2).reshape(b, t, -1), sd[p + "out.weight"], sd[p + "out.bias"])
    else:
        x = x.transpose(1, 2)
    return x, sub_out_len(lengths, k, 2)


# ------------------------------------------------------------------------------------------ conformer layer
def rotary_tables(length: int, dim: int, base: int) -> Tuple[Tensor, Tensor]:
    """gigaam/encoder.py:342-355: cos/sin of t * base^(-2i/dim), duplicated over the two halves. [T, dim]"""
    inv_freq = 1.0 / (base ** (torch.arange(0, dim, 2).float() / dim))
    t = torch.arange(length).float()
    freqs = torch.einsum("i,j->ij", t, inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos(), emb.sin()


def _rtt_half(x: Tensor) -> Tensor:
    """gigaam/utils.py:83-85"""
    x1, x2 = x[..., : x.shape[-1] // 2], x[..., x.shape[-1] // 2:]
    return torch.cat([-x2, x1], dim=-1)


def rotary_mhsa(u: Tensor, sd: SD, q: str, n_heads: int, cos: Tensor, sin: Tensor, key_valid: Optional[Tensor]) -> Tensor:
    """gigaam/encoder.py:236-277 + utils.py:88-100: RoPE on the (LayerNorm-ed) input *before* the q/k
    projections, v from the un-rotated input, softmax(q k^T / sqrt(d_k)) with padded keys at -inf."""
    b, t, d = u.shape
    dk = d // n_heads
    uh = u.view(b, t, n_heads, dk)
    c, s = cos[:t].view(1, t, 1, dk), sin[:t].view(1, t, 1, dk)
    ur = (uh * c + _rtt_half(uh) * s).reshape(b, t, d)
    qh = F.linear(ur, sd[q + "linear_q.weight"], sd[q + "linear_q.bias"]).view(b, t, n_heads, dk).transpose(1, 2)
    kh = F.linear(ur, sd[q + "linear_k.weight"], sd[q + "linear_k.bias"]).view(b, t, n_heads, dk).transpose(1, 2)
    vh = F.linear(u, sd[q + "linear_v.weight"], sd[q + "linear_v.bias"]).view(b, t, n_heads, dk).transpose(1, 2)
    scores = torch.matmul(qh, kh.transpose(-2, -1)) / math.sqrt(dk)
    if key_valid is not None:
        # reference mask is ~(valid_i & valid_j); rows of padded queries are don't-care, so masking keys only is
        # identical on every valid frame (encoder.py:620-624)
        scores = scores.masked_fill(~key_valid[:, None, None, :], float("-inf"))
    o = torch.matmul(torch.softmax(scores, dim=-1), vh)
    o = o.transpose(1, 2).reshape(b, t, d)
    return F.linear(o, sd[q + "linear_out.weight"], sd[q + "linear_out.bias"])


def rel_pos_table(t: int, d: int) -> Tensor:
    """gigaam/encoder.py:312-334: sinusoids of the relative positions t-1 ... -(t-1) (the slice forward() cuts out of
    the pos_emb_max_len table), sin on even / cos on odd columns, frequencies 10000^(-2i/d).  [2t-1, d]"""
    pos = torch.arange(t - 1, -t, -1, dtype=torch.float32).unsqueeze(1)
    div = torch.exp(torch.arange(0, d, 2, dtype=torch.float32) * -(math.log(10000.0) / d))
    pe = torch.zeros(2 * t - 1, d)
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe


def rel_pos_mhsa(u: Tensor, sd: SD, q: str, n_heads: int, pos_emb: Tensor, key_valid: Optional[Tensor]) -> Tensor:
    """gigaam/encoder.py:208-228 (+ :159-188): Transformer-XL scores
        s[i, j] = ((q_i + u) . k_j + (q_i + v) . p_{i-j}) / sqrt(d_k),   p_r = W_pos pe(r),
    written with the explicit index the reference's pad/view `rel_shift` (:202-206) produces: row i of the
    [T, 2T-1] position scores is read at column T-1-i+j.  Padded keys are excluded (the reference fills them with
    -10000 before the softmax and zeroes them after it, :182-183, which is the same on every valid query row)."""
    b, t, d = u.shape
    dk = d // n_heads
    qh = F.linear(u, sd[q + "linear_q.weight"], sd[q + "linear_q.bias"]).view(b, t, n_heads, dk)
    kh = F.linear(u, sd[q + "linear_k.weight"], sd[q + "linear_k.bias"]).view(b, t, n_heads, dk).transpose(1, 2)
    vh = F.linear(u, sd[q + "linear_v.weight"], sd[q + "linear_v.bias"]).view(b, t, n_heads, dk).transpose(1, 2)
    p = F.linear(pos_emb, sd[q + "linear_pos.weight"]).view(2 * t - 1, n_heads, dk).transpose(0, 1)   # [h, 2t-1, dk]
    qu = (qh + sd[q + "pos_bias_u"]).transpose(1, 2)                                                   # [b, h, t, dk]
    qv = (qh + sd[q + "pos_bias_v"]).transpose(1, 2)
    ac = torch.matmul(qu, kh.transpose(-2, -1))
    bd_raw = torch.matmul(qv, p.transpose(-2, -1))                                                      # [b, h, t, 2t-1]
    idx = (t - 1) - torch.arange(t)[:, None] + torch.arange(t)[None, :]                                 # [t, t]
    bd = torch.gather(bd_raw, 3, idx.expand(b, n_heads, t, t))
    scores = (ac + bd) / math.sqrt(dk)
    if key_valid is not None:
        scores = scores.masked_fill(~key_valid[:, None, None, :], float("-inf"))
    o = torch.matmul(torch.softmax(scores, dim=-1), vh)
    o = o.transpose(1, 2).reshape(b, t, d)
    return F.linear(o, sd[q + "linear_out.weight"], sd[q + "linear_out.bias"])


def conv_module(u: Tensor, sd: SD, q: str, enc: Dict, pad_mask: Tensor) -> Tensor:
    """gigaam/encoder.py:396-409"""
    x = u.transpose(1, 2)
    x = F.conv1d(x, sd[q + "pointwise_conv1.weight"], sd[q + "pointwise_conv1.bias"])
    x = F.glu(x, dim=1)
    x = x.masked_fill(pad_mask.unsqueeze(1), 0.0)
    k = enc["conv_kernel_size"]
    x = F.conv1d(x, sd[q + "depthwise_conv.weight"], sd[q + "depthwise_conv.bias"], padding=(k - 1) // 2, groups=x.shape[1])
    if enc["conv_norm_type"] == "batch_norm":
        x = F.batch_norm(x, sd[q + "batch_norm.running_mean"], sd[q + "batch_norm.running_var"],
                         sd[q + "batch_norm.weight"], sd[q + "batch_norm.bias"], training=False, eps=1e-5)
    else:
        x = F.layer_norm(x.transpose(1, 2), (x.shape[1],), sd[q + "batch_norm.weight"], sd[q + "batch_norm.bias"], 1e-5).transpose(1, 2)
    x = F.silu(x)
    x = F.conv1d(x, sd[q + "pointwise_conv2.weight"], sd[q + "pointwise_conv2.bias"])
    return x.transpose(1, 2)


def _ln(x: Tensor, sd: SD, name: str) -> Tensor:
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], 1e-5)


def _ff(x: Tensor, sd: SD, name: str) -> Tensor:
    """gigaam/encoder.py:412-424"""
    return F.linear(F.silu(F.linear(x, sd[name + ".linear1.weight"], sd[name + ".linear1.bias"])),
                    sd[name + ".linear2.weight"], sd[name + ".linear2.bias"])


def conformer_layer(x: Tensor, sd: SD, l: int, enc: Dict, cos: Tensor, sin: Tensor, key_valid: Optional[Tensor],
                    pad_mask: Tensor) -> Tensor:
    """gigaam/encoder.py:473-498"""
    q = f"encoder.layers.{l}."
    r = x + 0.5 * _ff(_ln(x, sd, q + "norm_feed_forward1"), sd, q + "feed_forward1")
    if enc["self_attention_model"] == "rotary":
        r = r + rotary_mhsa(_ln(r, sd, q + "norm_self_att"), sd, q + "self_attn.", enc["n_heads"], cos, sin, key_valid)
    else:   # rel_pos: `cos` carries the [2T-1, d] position table
        r = r + rel_pos_mhsa(_ln(r, sd, q + "norm_self_att"), sd, q + "self_attn.", enc["n_heads"], cos, key_valid)
    r = r + conv_module(_ln(r, sd, q + "norm_conv"), sd, q + "conv.", enc, pad_mask)
    r = r + 0.5 * _ff(_ln(r, sd, q + "norm_feed_forward2"), sd, q + "feed_forward2")
    return _ln(r, sd, q + "norm_out")


def encoder_forward(mel: Tensor, mel_len: Tensor, sd: SD, enc: Dict, n_layers_run: Optional[int] = None,
                    return_all: bool = False):
    """gigaam/encoder.py:605-647.  Returns ([B, d, T'], len int32) (+ list of [B, T', d] per stage)."""
    x, length = pre_encode(mel, mel_len, sd, enc)
    stages = [x]
    t = x.size(1)
    if enc["self_attention_model"] == "rotary":
        cos, sin = rotary_tables(enc["pos_emb_max_len"], enc["d_model"] // enc["n_heads"], enc["pos_emb_max_len"])
    else:
        cos, sin = rel_pos_table(t, enc["d_model"]), None
    valid = torch.arange(t)[None, :] < length[:, None]
    key_valid = valid if x.shape[0] > 1 else None
    pad_mask = ~valid
    L = enc["n_layers"] if n_layers_run is None else n_layers_run
    for l in range(L):
        x = conformer_layer(x, sd, l, enc, cos, sin, key_valid, pad_mask)
        stages.append(x)
    out = (x.transpose(1, 2), length)
    return (*out, stages) if return_all else out


def model_forward(wav: Tensor, wav_len: Tensor, sd: SD, cfg: Dict):
    """gigaam/model.py:27-37 on CPU (no autocast)."""
    pre = cfg["preprocessor"]
    sr = pre["sample_rate"]
    mel = log_mel(wav, sd, pre)
    mel_len = logmel_out_len(wav_len, pre.get("hop_length", sr // 100), pre.get("win_length", sr // 40), pre.get("center", True))
    return encoder_forward(mel, mel_len, sd, cfg["encoder"])


# ------------------------------------------------------------------------------------------ CTC
def ctc_logits(enc: Tensor, sd: SD) -> Tensor:
    """gigaam/decoder.py:14-21 without the (argmax-invariant) log_softmax.  enc [B, d, T] -> [B, T, V+1]"""
    return F.conv1d(enc, sd["head.decoder_layers.0.weight"], sd["head.decoder_layers.0.bias"]).transpose(1, 2)


def ctc_greedy(enc: Tensor, enc_len: Tensor, sd: SD) -> List[Tuple[List[int], List[int]]]:
    """gigaam/decoding.py:56-96 -> per utterance (token ids, frames)."""
    logits = ctc_logits(enc, sd)
    blank = logits.shape[-1] - 1
    labels = torch.log_softmax(logits, dim=-1).argmax(dim=-1)
    out = []
    for b in range(labels.shape[0]):
        ids, frames = [], []
        L = int(min(max(int(enc_len[b]), 0), labels.shape[1]))
        prev = None
        for t in range(labels.shape[1]):
            l = int(labels[b, t])
            if t < L and l != blank and (t == 0 or l != prev):
                ids.append(l)
                frames.append(t)
            prev = l
        out.append((ids, frames))
    return out


# ------------------------------------------------------------------------------------------ RNN-T
def _lstm_step(emb: Tensor, h: Tensor, c: Tensor, sd: SD) -> Tuple[Tensor, Tensor]:
    """One step of nn.LSTM(H, H, 1), gate order i,f,g,o (gigaam/decoder.py:82,95-102)."""
    g = (F.linear(emb, sd["head.decoder.lstm.weight_ih_l0"], sd["head.decoder.lstm.bias_ih_l0"])
         + F.linear(h, sd["head.decoder.lstm.weight_hh_l0"], sd["head.decoder.lstm.bias_hh_l0"]))
    i, f, gg, o = g.chunk(4, dim=-1)
    c2 = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
    h2 = torch.sigmoid(o) * torch.tanh(c2)
    return h2, c2


def rnnt_greedy(enc: Tensor, enc_len: Tensor, sd: SD, max_symbols: int = 10) -> List[Tuple[List[int], List[int]]]:
    """gigaam/decoding.py:128-207 restated per utterance (the batched loop is batch-independent,
    SURVEY 3.4): state commits only on a non-blank emission; at most max_symbols tokens per frame."""
    x = enc.transpose(1, 2)
    W_e, b_e = sd["head.joint.enc.weight"], sd["head.joint.enc.bias"]
    W_p, b_p = sd["head.joint.pred.weight"], sd["head.joint.pred.bias"]
    W_o, b_o = sd["head.joint.joint_net.1.weight"], sd["head.joint.joint_net.1.bias"]
    emb_w = sd["head.decoder.embed.weight"]
    H = emb_w.shape[1]
    blank = W_o.shape[0] - 1
    out = []
    for b in range(x.shape[0]):
        ids, frames = [], []
        h = torch.zeros(1, H)
        c = torch.zeros(1, H)
        emb = torch.zeros(1, H)                      # predict(None, None): zero embedding, zero state
        hn, cn = _lstm_step(emb, h, c, sd)
        pg = F.linear(hn, W_p, b_p)
        L = int(min(max(int(enc_len[b]), 0), x.shape[1]))
        for t in range(L):
            f = F.linear(x[b, t:t + 1], W_e, b_e)
            for _ in range(max_symbols):
                # argmax after log_softmax, as gigaam/decoder.py:47 + decoding.py:162: a row with a NaN gives 0
                k = int(torch.log_softmax(F.linear(F.relu(f + pg), W_o, b_o), dim=-1).argmax(dim=-1))
                if k == blank:
                    break
                ids.append(k)
                frames.append(t)
                h, c = hn, cn
                hn, cn = _lstm_step(emb_w[k:k + 1], h, c, sd)
                pg = F.linear(hn, W_p, b_p)
        out.append((ids, frames))
    return out
