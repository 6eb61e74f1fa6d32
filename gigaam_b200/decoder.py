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

from . import _lib, synthetic
from ._params import Bound, build_tree
from .decoding import _as_btd


def _zeros(entries):
    return [(k, torch.zeros(shape, dtype=torch.float32)) for k, shape, kind, _ in entries]


def _trains(module, *inputs) -> bool:
    """The autograd path engages only when grad mode is on and a parameter of the head module or an input tensor requires
    grad; otherwise the forward-only path runs (same kernels, same bits, nothing saved)."""
    if not torch.is_grad_enabled():
        return False
    return any(p.requires_grad for p in module.parameters()) or any(t is not None and t.requires_grad for t in inputs)


def _param_versions(module) -> Tuple:
    return tuple(p._version for p in module.parameters())


def _check_versions(ctx) -> None:
    if _param_versions(ctx.module) != ctx.versions:
        raise RuntimeError(f"{type(ctx.module).__name__}: a head parameter was modified between forward and backward")


def _f32(t: Optional[Tensor]) -> Optional[Tensor]:
    return None if t is None else t.detach().float().contiguous()


class _CTCLogProbs(torch.autograd.Function):
    """CTCHead.forward with gam_ctc_log_probs_backward behind it (dL/d encoder output, decoder_layers.0.weight / bias)."""

    @staticmethod
    def forward(ctx, module, enc, weight, bias):
        eng = module._engine()
        out = eng.ctc_log_probs(enc.detach())
        ctx.module, ctx.versions = module, _param_versions(module)
        ctx.save_for_backward(enc, out)
        return out

    @staticmethod
    def backward(ctx, grad):
        _check_versions(ctx)
        enc, out = ctx.saved_tensors
        eng = ctx.module._engine()
        need_w = ctx.needs_input_grad[2] or ctx.needs_input_grad[3]
        d_enc, dW, db = eng.ctc_log_probs_backward(enc.detach(), out, _f32(grad), ctx.needs_input_grad[1], need_w)
        w = ctx.module.decoder_layers._modules["0"].weight
        return (None, d_enc, None if dW is None else dW.view(w.shape).to(w.dtype),
                None if db is None else db.to(w.dtype))


class _RNNTJointFn(torch.autograd.Function):
    """RNNTJoint.joint with gam_rnnt_joint_backward behind it (enc / dec inputs, joint.enc, joint.pred, joint_net.1)."""

    @staticmethod
    def forward(ctx, module, enc, dec, *params):
        eng = module._engine()
        out = eng.rnnt_joint(enc.detach(), dec.detach())
        ctx.module, ctx.versions = module, _param_versions(module)
        ctx.save_for_backward(enc, dec, out)
        return out

    @staticmethod
    def backward(ctx, grad):
        _check_versions(ctx)
        enc, dec, out = ctx.saved_tensors
        eng = ctx.module._engine()
        need_w = any(ctx.needs_input_grad[3:])
        d_enc, d_dec, *dw = eng.rnnt_joint_backward(enc.detach(), dec.detach(), out, _f32(grad), ctx.needs_input_grad[1],
                                                    ctx.needs_input_grad[2], need_w)
        return (None, d_enc, d_dec, *dw)


class _RNNTLossFn(torch.autograd.Function):
    """The fused RNN-T loss (decoding.rnnt_loss) with gam_rnnt_loss_backward behind it (enc / dec inputs, joint.enc, joint.pred,
    joint_net.1).  Saves the loss call's per-node [3, B, T, U+1] operands, never a lattice."""

    @staticmethod
    def forward(ctx, module, enc, dec, targets, enc_len, target_len, *params):
        eng = module._engine()
        loss, saved = eng.rnnt_loss(enc.detach(), dec.detach(), targets, enc_len, target_len)
        ctx.module, ctx.versions = module, _param_versions(module)
        ctx.save_for_backward(enc, dec, targets, enc_len, target_len, saved)
        return loss

    @staticmethod
    def backward(ctx, grad):
        _check_versions(ctx)
        enc, dec, targets, enc_len, target_len, saved = ctx.saved_tensors
        eng = ctx.module._engine()
        need_w = any(ctx.needs_input_grad[6:])
        d_enc, d_dec, *dw = eng.rnnt_loss_backward(enc.detach(), dec.detach(), targets, enc_len, target_len, saved, _f32(grad),
                                                   ctx.needs_input_grad[1], ctx.needs_input_grad[2], need_w)
        return (None, d_enc, d_dec, None, None, None, *dw)


class _RNNTPredictFn(torch.autograd.Function):
    """RNNTDecoder.predict with gam_rnnt_predict_backward behind it (h0 / c0, embed, lstm weights and biases)."""

    @staticmethod
    def forward(ctx, module, x, h, c, batch_size, embed, w_ih, w_hh, b_ih, b_hh):
        eng = module._engine()
        h_d, c_d = _f32(h), _f32(c)
        g, h1, c1, c_seq = eng.rnnt_predict_train(x, h_d, c_d, batch_size)
        ctx.module, ctx.versions = module, _param_versions(module)
        ctx.save_for_backward(x, h_d, c_d, g, c_seq)
        return g, h1, c1

    @staticmethod
    def backward(ctx, grad_g, grad_h1, grad_c1):
        _check_versions(ctx)
        x, h, c, g, c_seq = ctx.saved_tensors
        eng = ctx.module._engine()
        lstm = ctx.module.lstm
        need_state = ctx.needs_input_grad[2] or ctx.needs_input_grad[3]
        need_w = any(ctx.needs_input_grad[5:])
        d_h, d_c, d_emb, dW_ih, dW_hh, d_b = eng.rnnt_predict_backward(
            x, h, c, g, c_seq, _f32(grad_g), _f32(grad_h1), _f32(grad_c1), _f32(ctx.module.embed.weight),
            _f32(lstm.weight_ih_l0), _f32(lstm.weight_hh_l0), need_state, need_w)
        return None, None, d_h, d_c, None, d_emb, dW_ih, dW_hh, d_b, None if d_b is None else d_b.clone()


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
        enc = _as_btd(_on_device(encoder_output, eng, torch.float32))
        if _trains(self, enc):
            layer = self.decoder_layers._modules["0"]
            return _CTCLogProbs.apply(self, enc, layer.weight, layer.bias)
        return eng.ctc_log_probs(enc)


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
        if _trains(self, enc, dec):
            out = self.joint_net._modules["1"]
            return _RNNTJointFn.apply(self, enc, dec, self.enc.weight, self.enc.bias, self.pred.weight, self.pred.bias,
                                      out.weight, out.bias)
        return eng.rnnt_joint(enc, dec)

    def forward(self, enc: Tensor, dec: Tensor) -> Tensor:
        """[B, enc_hidden, T], [B, pred_hidden, U] -> [B, T, U, num_classes] (gigaam/decoder.py:68-69)"""
        return self.joint(enc.transpose(1, 2), dec.transpose(1, 2))

    def _loss(self, enc: Tensor, dec: Tensor, targets: Tensor, enc_len: Tensor, target_len: Tensor) -> Tensor:
        """enc [B, T, enc_hidden], dec [B, U+1, pred_hidden] f32 on the device, targets [B, U] (blank where unused), enc_len /
        target_len [B] -> the per-utterance loss [B] (gam_rnnt_loss), differentiable when a joint parameter, enc or dec
        requires grad.  decoding.rnnt_loss is the public entry point."""
        eng = self._engine()
        enc, dec = enc.contiguous(), dec.contiguous()
        if _trains(self, enc, dec):
            out = self.joint_net._modules["1"]
            return _RNNTLossFn.apply(self, enc, dec, targets, enc_len, target_len, self.enc.weight, self.enc.bias, self.pred.weight,
                                     self.pred.bias, out.weight, out.bias)
        return eng.rnnt_loss(enc, dec, targets, enc_len, target_len)[0]


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
        (gigaam/decoder.py:85-102).  A row with an id outside [0, num_classes) comes back as NaN.  With a gradient to
        compute, pred_hidden above the backward's limit raises ValueError before any launch."""
        self._check_trainable(*(state if state is not None else ()))
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
        if _trains(self, h, c):
            lstm = self.lstm
            g, h1, c1 = _RNNTPredictFn.apply(self, x, h, c, batch_size, self.embed.weight, lstm.weight_ih_l0, lstm.weight_hh_l0,
                                             lstm.bias_ih_l0, lstm.bias_hh_l0)
        else:
            g, h1, c1 = eng.rnnt_predict(x, h, c, batch_size)
        return g, (h1.unsqueeze(0), c1.unsqueeze(0))

    def _check_trainable(self, *state: Tensor) -> None:
        """A call that would need gam_rnnt_predict_backward at a pred_hidden it cannot run is refused here, before its
        forward launches; without a gradient every width up to the forward's runs."""
        limit = _lib.PREDICT_BACKWARD_MAX_HIDDEN
        if self.pred_hidden > limit and _trains(self, *state):
            raise ValueError(f"predict: pred_hidden {self.pred_hidden} cannot be trained: the prediction network's backward "
                             f"runs pred_hidden <= {limit}; call it without gradients or freeze head.decoder")

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
