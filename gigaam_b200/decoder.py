"""CTC / RNN-T heads with the reference's interface and state_dict keys (gigaam/decoder.py).  The greedy decoders use
the heads' parameters inside their own fused kernels (`gam_ctc_greedy`, `gam_rnnt_greedy`); the heads' public
methods -- `CTCHead.forward`, `RNNTDecoder.predict` / `forward`, `RNNTJoint.joint` / `forward` -- run the head
kernels of csrc/heads.cu (`gam_ctc_log_probs`, `gam_rnnt_predict`, `gam_rnnt_joint`) for callers that do their own
search.  `Linear` is the emo model's head (a torch.nn.Linear in the reference's checkpoint); it runs `gam_emo_head`.  All
head arithmetic is fp32, as in the reference (gigaam/__init__.py:188-189)."""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
from torch import Tensor

from . import synthetic
from ._params import Bound, build_tree
from .decoding import _as_btd


def _zeros(entries):
    return [(k, torch.zeros(shape, dtype=torch.float32)) for k, shape, kind, _ in entries]


def _on_device(t: Tensor, eng, dtype: torch.dtype) -> Tensor:
    if not t.is_cuda:
        raise RuntimeError("gigaam_b200 has no CPU path: pass CUDA tensors to the head (the model runs on "
                           f"{eng.device})")
    return t.to(device=eng.device, dtype=dtype)


class CTCHead(Bound):
    """gigaam/decoder.py:7-21 -- Conv1d(feat_in, num_classes, k=1) under `decoder_layers.0`."""

    def __init__(self, feat_in: int, num_classes: int):
        super().__init__()
        self.feat_in, self.num_classes = feat_in, num_classes
        build_tree(self, _zeros(synthetic.head_param_list(dict(type="ctc", feat_in=feat_in, num_classes=num_classes))), "head.")

    def forward(self, encoder_output: Tensor) -> Tensor:
        """[B, feat_in, T] -> log-probs [B, T, num_classes] (gigaam/decoder.py:18-21).  The encoder's output is a
        transposed view of a [B, T, d] buffer, which the kernel reads as it is."""
        eng = self._engine()
        return eng.ctc_log_probs(_as_btd(_on_device(encoder_output, eng, torch.float32)))


class RNNTJoint(Bound):
    """gigaam/decoder.py:24-69 -- `enc` / `pred` / `joint_net.1` parameters; the lattice runs in `gam_rnnt_joint`."""

    def __init__(self, enc_hidden: int, pred_hidden: int, joint_hidden: int, num_classes: int):
        super().__init__()
        self.enc_hidden = enc_hidden
        self.pred_hidden = pred_hidden

    def joint(self, encoder_out: Tensor, decoder_out: Tensor) -> Tensor:
        """[B, T, enc_hidden], [B, U, pred_hidden] -> log-probs [B, T, U, num_classes] (gigaam/decoder.py:41-47)"""
        eng = self._engine()
        enc = _on_device(encoder_out, eng, torch.float32).contiguous()
        dec = _on_device(decoder_out, eng, torch.float32).contiguous()
        return eng.rnnt_joint(enc, dec)

    def forward(self, enc: Tensor, dec: Tensor) -> Tensor:
        """[B, enc_hidden, T], [B, pred_hidden, U] -> [B, T, U, num_classes] (gigaam/decoder.py:68-69)"""
        return self.joint(enc.transpose(1, 2), dec.transpose(1, 2))


class RNNTDecoder(Bound):
    """gigaam/decoder.py:72-137 -- `embed` + 1-layer `lstm` parameters; the steps run in `gam_rnnt_predict`."""

    def __init__(self, pred_hidden: int, pred_rnn_layers: int, num_classes: int):
        super().__init__()
        self.blank_id = num_classes - 1
        self.pred_hidden = pred_hidden

    def predict(self, x: Optional[Tensor], state: Optional[Tuple[Tensor, Tensor]], batch_size: int = 1
                ) -> Tuple[Tensor, Tuple[Tensor, Tensor]]:
        """x [B, U] label ids or None (one step from the zero embedding, `batch_size` rows); state (h, c), each
        [1, B, pred_hidden] (strided views are fine), or None (zeros) -> (g [B, U, pred_hidden], (h, c) [1, B, pred_hidden])
        (gigaam/decoder.py:85-102).  A row with an id outside [0, num_classes) comes back as NaN."""
        eng = self._engine()
        if x is not None:
            x = _on_device(x, eng, torch.int64).contiguous()
        h = c = None
        if state is not None:
            h, c = (_on_device(s, eng, torch.float32) for s in state)
            if h.dim() != 3 or h.shape[0] != 1 or c.shape != h.shape:
                raise ValueError(f"predict: state must be two [1, B, {self.pred_hidden}] tensors (one LSTM layer), got "
                                 f"{tuple(h.shape)} and {tuple(c.shape)}")
            h, c = h[0].contiguous(), c[0].contiguous()
        g, h1, c1 = eng.rnnt_predict(x, h, c, batch_size)
        return g, (h1.unsqueeze(0), c1.unsqueeze(0))

    def forward(self, x: Tensor, h: Tensor, c: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
        """ONNX form of predict: (x, h, c) -> (g, h, c) (gigaam/decoder.py:131-137)"""
        g, (h, c) = self.predict(x, (h, c))
        return g, h, c


class RNNTHead(Bound):
    """gigaam/decoder.py:140-149 -- `decoder` (RNNTDecoder) and `joint` (RNNTJoint)."""

    def __init__(self, decoder: Dict[str, int], joint: Dict[str, int]):
        super().__init__()
        self.decoder_cfg, self.joint_cfg = dict(decoder), dict(joint)
        self.decoder = RNNTDecoder(**self.decoder_cfg)
        self.joint = RNNTJoint(**self.joint_cfg)
        build_tree(self, _zeros(synthetic.head_param_list(dict(type="rnnt", decoder=self.decoder_cfg, joint=self.joint_cfg))), "head.")

    def _bind(self, owner) -> None:
        super()._bind(owner)
        self.decoder._bind(owner)
        self.joint._bind(owner)


class Linear(Bound):
    """The emo model's head: torch.nn.Linear(in_features, out_features) with keys `head.weight` [C, d] and `head.bias` [C]
    (gigaam/model.py:269, instantiated from the checkpoint's `head._target_`).  Only in_features = d_model with a bias is
    supported; the model refuses other heads at load time."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        build_tree(self, _zeros(synthetic.head_param_list(dict(type="emo", in_features=in_features, out_features=out_features,
                                                               bias=bias))), "head.")

    def forward(self, x: Tensor) -> Tensor:
        """x [..., in_features] -> logits [..., out_features] (x W^T + b, fp32).  Runs the pooled-head kernel with one frame
        per row, whose mean is the row itself."""
        eng = self._engine()
        x = _on_device(x, eng, torch.float32)
        if x.shape[-1] != self.in_features:
            raise ValueError(f"Linear: last dimension {x.shape[-1]} != in_features {self.in_features}")
        rows = x.reshape(-1, 1, self.in_features).contiguous()
        if rows.shape[0] == 0:
            return torch.empty((*x.shape[:-1], self.out_features), dtype=torch.float32, device=eng.device)
        _, logits, _ = eng.emo_head(rows, None)
        return logits.reshape(*x.shape[:-1], self.out_features)
