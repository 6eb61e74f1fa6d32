"""Conformer encoder with the reference's interface (gigaam/encoder.py:501-647).  Parameters live in holder
modules under the reference's state_dict names; `forward` / `pre_encode` run the CUDA path (`gam_encode`)."""
from __future__ import annotations

from typing import Tuple

import torch
from torch import Tensor

from . import synthetic
from ._params import Bound, build_tree


class StridingSubsampling(Bound):
    """Holder + entry point for encoder.pre_encode (gigaam/encoder.py:32-130)."""

    def __init__(self, subsampling: str, kernel_size: int):
        super().__init__()
        self.subsampling_type = subsampling
        self._kernel_size = kernel_size
        self._padding = (kernel_size - 1) // 2
        self._stride = 2
        self._sampling_num = 2

    def calc_output_length(self, lengths: Tensor, num_stages=None) -> Tensor:
        """gigaam/encoder.py:77-90"""
        if num_stages is None:
            num_stages = self._sampling_num
        add_pad = 2 * self._padding - self._kernel_size
        lengths = lengths.to(torch.float)
        for _ in range(num_stages):
            lengths = torch.floor((lengths + add_pad) / self._stride + 1.0)
        return lengths.to(dtype=torch.int)

    def forward(self, x: Tensor, lengths: Tensor) -> Tuple[Tensor, Tensor]:
        """x: [B, M, F] (the reference passes the transposed log-mel, encoder.py:609-611) -> ([B, T', d], len)"""
        eng = self._engine()
        mel = x.to(device=eng.device, dtype=torch.float32).transpose(1, 2)
        enc, enc_len = eng.encode(mel, lengths, n_layers_run=0)
        return enc, enc_len


class ConformerEncoder(Bound):
    """Drop-in for gigaam.encoder.ConformerEncoder: same ctor kwargs (encoder.py:510-526), same state_dict keys."""

    def __init__(self, feat_in: int = 64, n_layers: int = 16, d_model: int = 768, subsampling: str = "conv2d",
                 subs_kernel_size: int = 3, subsampling_factor: int = 4, ff_expansion_factor: int = 4,
                 self_attention_model: str = "rotary", n_heads: int = 16, pos_emb_max_len: int = 5000,
                 conv_norm_type: str = "batch_norm", conv_kernel_size: int = 31, flash_attn: bool = False,
                 activation_checkpointing: bool = False):
        super().__init__()
        assert self_attention_model in ["rotary", "rel_pos"], f"Not supported attn = {self_attention_model}"
        self.feat_in = feat_in
        self.cfg = dict(feat_in=feat_in, n_layers=n_layers, d_model=d_model, subsampling=subsampling,
                        subs_kernel_size=subs_kernel_size, subsampling_factor=subsampling_factor,
                        ff_expansion_factor=ff_expansion_factor, self_attention_model=self_attention_model,
                        n_heads=n_heads, pos_emb_max_len=pos_emb_max_len, conv_norm_type=conv_norm_type,
                        conv_kernel_size=conv_kernel_size, flash_attn=flash_attn)
        self.pos_emb_max_len = pos_emb_max_len
        self.pre_encode = StridingSubsampling(subsampling, subs_kernel_size)
        entries = [(k, torch.zeros(shape, dtype=torch.long if kind == "int" else torch.float32))
                   for k, shape, kind, _ in synthetic.encoder_param_list(self.cfg)]
        build_tree(self, entries, "encoder.")

    def _bind(self, owner) -> None:
        super()._bind(owner)
        self.pre_encode._bind(owner)

    def forward(self, audio_signal: Tensor, length: Tensor) -> Tuple[Tensor, Tensor]:
        """[B, F, M] log-mel, [B] lengths -> ([B, d_model, T'], [B] int32)  (gigaam/encoder.py:605-647).  Inference-only:
        with grad enabled and a parameter of this encoder requiring grad this raises NotImplementedError."""
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("the encoder is inference-only; freeze it (requires_grad_(False)) and train the head on "
                                      "its output")
        eng = self._engine()
        mel = audio_signal.to(device=eng.device, dtype=torch.float32)
        enc, enc_len = eng.encode(mel, length)
        return enc.transpose(1, 2), enc_len
