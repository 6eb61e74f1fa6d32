"""Host side of the C ABI: packs a reference state_dict into the device layout the kernels want, owns the
gam_handle and the scratch workspace, and turns torch tensors into raw pointers.  No arithmetic of the path is
done here -- only one-off weight re-layout at load time (BatchNorm folding, q/k concatenation, GLU row pairing,
conv weight permutation, fp16 casts, DFT / rotary tables)."""
from __future__ import annotations

import collections
import ctypes as C
import hashlib
import json
import math
import os
from typing import Dict, List, NamedTuple, Optional, Tuple

import torch

from . import _lib

Tensor = torch.Tensor


class DecodeBuffers(NamedTuple):
    """Outputs that Engine.greedy_resume appends to across calls (Engine.decode_buffers); the score fields are None for
    unscored decoding."""
    ids: Tensor
    frames: Tensor
    counts: Tensor
    token_logp: Optional[Tensor] = None
    path_logp: Optional[Tensor] = None
    path_rows: Optional[Tensor] = None
    frame_logp: Optional[Tensor] = None
    frame_rows: Optional[Tensor] = None


def _cfg_get(section, key, default=None):
    if isinstance(section, dict):
        return section.get(key, default)
    return getattr(section, key, default) if hasattr(section, key) else (section.get(key, default) if hasattr(section, "get") else default)


# ---------------------------------------------------------------------------------- pure weight re-layout (CPU-testable)
def glu_row_permutation(d: int, half: int = 128) -> Tensor:
    """Row order of pointwise_conv1 so that accumulator tile j (2*half columns) = [value rows j*half.. | gate rows d+j*half..]:
    the GEMM epilogue then computes value * sigmoid(gate) thread-locally (gigaam/encoder.py:398-399 GLU over channels)."""
    return torch.cat([torch.cat([torch.arange(j * half, (j + 1) * half), d + torch.arange(j * half, (j + 1) * half)])
                      for j in range(d // half)])


def fold_batchnorm(dw_w: Tensor, dw_b: Tensor, gamma: Tensor, beta: Tensor, mean: Tensor, var: Tensor, eps: float = 1e-5):
    """Eval-mode BatchNorm1d after the depthwise conv folded into its weights (gigaam/encoder.py:402-405)."""
    s = gamma / torch.sqrt(var + eps)
    return dw_w * s[:, None], (dw_b - mean) * s + beta


def pack_conv2_weight(w2: Tensor) -> Tensor:
    """[C_out, C_in, kt, kf] -> [C_out, (kt, kf, C_in)]: K order of the implicit GEMM (tap-major, channel-minor)."""
    return w2.permute(0, 2, 3, 1).reshape(w2.shape[0], -1)


def pack_conv1d_weight(w: Tensor) -> Tensor:
    """Conv1d weight [C_out, C_in, k] -> [C_out, (k, C_in)]: K order (tap, channel) of the implicit conv1d GEMM."""
    return w.permute(0, 2, 1).reshape(w.shape[0], -1)


def pack_sub_out_weight(wo: Tensor, channels: int) -> Tensor:
    """pre_encode.out.weight [d, C*F2] with K index c*F2+f (gigaam/encoder.py:125-127) -> K index f*C+c, the order in
    which the stage-2 conv epilogue writes its [B, T', F2, C] output."""
    f2 = wo.shape[1] // channels
    return wo.reshape(wo.shape[0], channels, f2).permute(0, 2, 1).reshape(wo.shape[0], f2 * channels)


DFT_BASIS_SCALE = 8.0      # must match kBasisScale / kFrameScale in csrc/gam_api.cu, frontend.cu
DFT_FRAME_SCALE = 2048.0


def split_dft_basis(n_fft: int) -> Tensor:
    """fp16 [512, 3*Kp] basis of the real DFT for the K-concatenated split-precision GEMM (Kp = n_fft rounded up to 64).
    Rows: two 256-row tiles, tile t = [128 cos rows | 128 sin rows] of bins t*128 + j (bins >= n_fft/2+1 are zero rows);
    columns: [d_hi | d_hi | d_lo] with d = cos / sin(2 pi k i / n_fft), d_hi = fp16(d), d_lo = fp16(d - d_hi)."""
    kp = (n_fft + 63) // 64 * 64
    nb = n_fft // 2 + 1
    k = torch.arange(256, dtype=torch.float64)[:, None]
    i = torch.arange(kp, dtype=torch.float64)[None, :]
    ang = 2.0 * math.pi * k * i / n_fft
    valid = ((k < nb) & (i < n_fft)).double()
    # x 8: keeps the fp16 `lo` halves of small basis values out of the subnormal range (the frames are scaled by
    # 2^11 for the same reason; the power epilogue multiplies by 2^-28)
    basis = torch.stack([torch.cos(ang) * valid, torch.sin(ang) * valid], 1) * DFT_BASIS_SCALE   # [256 bins, 2, kp]
    rows = basis.view(2, 128, 2, kp).permute(0, 2, 1, 3).reshape(512, kp)          # tile, (cos|sin), bin-in-tile
    hi = rows.to(torch.float16)
    lo = (rows - hi.double()).to(torch.float16)
    return torch.cat([hi, hi, lo], dim=1).contiguous()


def rel_pos_embedding(max_t: int, d: int) -> Tensor:
    """Sinusoids of the relative positions max_t-1 ... -(max_t-1), row max_t-1-r for position r, sin on even / cos on
    odd columns (gigaam/encoder.py:318-326).  The reference slices the same rows out of its pos_emb_max_len table
    (:329-334), so the projected table below serves every T' <= max_t."""
    pos = torch.arange(max_t - 1, -max_t, -1, dtype=torch.float32).unsqueeze(1)
    div = torch.exp(torch.arange(0, d, 2, dtype=torch.float32) * -(math.log(10000.0) / d))
    pe = torch.zeros(2 * max_t - 1, d)
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe


def pack_rel_pos_qkv(wq: Tensor, bq: Tensor, wk: Tensor, bk: Tensor, wv: Tensor, bv: Tensor, bias_u: Tensor, bias_v: Tensor):
    """One projection for the rel_pos attention: rows [q ; q ; k ; v] with pos_bias_u / pos_bias_v (gigaam/encoder.py:
    221-222, [h, d_k] = the d_model axis split by head) folded into the two q biases -> ([4d, d], [4d])."""
    w = torch.cat([wq, wq, wk, wv], 0)
    b = torch.cat([bq + bias_u.reshape(-1), bq + bias_v.reshape(-1), bk, bv], 0)
    return w, b


def max_encoded_frames_config(max_encoded_frames: Optional[int], pos_emb_max_len: int) -> int:
    """gam_config.max_encoded_frames for a requested limit on T': 0 (the library's default of _lib.REL_POS_MAX_T frames)
    for None, else the value, which must lie in [REL_POS_MAX_T, pos_emb_max_len] -- the rotary and relative-position
    tables of the reference have pos_emb_max_len rows (gigaam/encoder.py:312-361)."""
    if max_encoded_frames is None:
        return 0
    if isinstance(max_encoded_frames, bool) or int(max_encoded_frames) != max_encoded_frames:
        raise ValueError(f"max_encoded_frames must be an integer, got {max_encoded_frames!r}")
    if not _lib.REL_POS_MAX_T <= max_encoded_frames <= pos_emb_max_len:
        raise ValueError(f"max_encoded_frames={max_encoded_frames} outside [{_lib.REL_POS_MAX_T}, {pos_emb_max_len}] "
                         f"(pos_emb_max_len of this encoder)")
    return int(max_encoded_frames)


def check_attention_heads(enc: Dict) -> None:
    """Refuse, before any device work, a head width d_k = d_model / n_heads wider than the attention kernel of this
    encoder runs (_lib.ROTARY_MAX_DK / REL_POS_MAX_DK, the header's limits, which gam_create also enforces).  The other
    shape limits (d_model 768, d_k % 16 == 0) are gam_create's."""
    d, h = enc["d_model"], enc["n_heads"]
    if h <= 0 or d % h != 0:
        return
    kind = enc["self_attention_model"]
    dk_max = _lib.REL_POS_MAX_DK if kind == "rel_pos" else _lib.ROTARY_MAX_DK
    if d // h > dk_max:
        raise ValueError(f"{kind} attention runs heads of d_k <= {dk_max}, but d_model {d} / n_heads {h} gives "
                         f"d_k = {d // h}")


def rotary_half_tables(dk: int, base: float, max_len: int):
    """cos/sin [max_len, dk/2] of t * base^(-2i/dk) (gigaam/encoder.py:342-355; base = pos_emb_max_len)."""
    inv_freq = 1.0 / (base ** (torch.arange(0, dk, 2).float() / dk))
    freqs = torch.einsum("i,j->ij", torch.arange(max_len).float(), inv_freq)
    return freqs.cos(), freqs.sin()


RNNT_HEAD_FIELDS = ("rnnt_emb_gates", "rnnt_whh_t", "rnnt_wp_t", "rnnt_bp", "rnnt_enc_w", "rnnt_enc_b", "rnnt_wo", "rnnt_bo")


def rnnt_head_packing(sd: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """The RNN-T head's device layout (gam_weights fields), fp32, computed on the tensors' device: the embedding table is
    folded through the LSTM's input weights and both biases, W_hh and W_p are transposed."""
    emb = sd["head.decoder.embed.weight"].double().clone()
    # predict(None, None) starts from an all-zero embedding (gigaam/decoder.py:92-95) and nn.Embedding's padding_idx
    # row is zero by construction but not enforced by load_state_dict: the table's blank row carries the biases only
    emb[emb.shape[0] - 1].zero_()
    w_ih, w_hh = sd["head.decoder.lstm.weight_ih_l0"].double(), sd["head.decoder.lstm.weight_hh_l0"].float()
    bias = sd["head.decoder.lstm.bias_ih_l0"].double() + sd["head.decoder.lstm.bias_hh_l0"].double()
    return {"rnnt_emb_gates": (emb @ w_ih.t() + bias).float(), "rnnt_whh_t": w_hh.t(),
            "rnnt_wp_t": sd["head.joint.pred.weight"].float().t(), "rnnt_bp": sd["head.joint.pred.bias"].float(),
            "rnnt_enc_w": sd["head.joint.enc.weight"].float(), "rnnt_enc_b": sd["head.joint.enc.bias"].float(),
            "rnnt_wo": sd["head.joint.joint_net.1.weight"].float(), "rnnt_bo": sd["head.joint.joint_net.1.bias"].float()}


class _WorkspaceCache:
    """Bounded LRU of scratch tensors of ONE kind (encode / log-mel / decode).  Eviction only drops this cache's
    reference: a CUDA graph that baked a workspace pointer keeps the tensor alive through `Engine.held_workspaces`."""

    def __init__(self, cap: int):
        self.cap = cap
        self._d: "collections.OrderedDict[Tuple, Tensor]" = collections.OrderedDict()

    def get(self, key, nbytes: int, device) -> Tensor:
        ws = self._d.get(key)
        if ws is not None and ws.numel() >= nbytes:
            self._d.move_to_end(key)
            return ws
        while len(self._d) >= self.cap:
            self._d.popitem(last=False)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self._d[key] = ws
        return ws

    def peek(self, key) -> Optional[Tensor]:
        return self._d.get(key)

    def tensors(self) -> List[Tensor]:
        return list(self._d.values())

    def __len__(self):
        return len(self._d)


class Engine:
    """One model replica on one CUDA device."""

    WS_CACHE = 4      # workspaces kept per kind (distinct batch shapes)

    PACK_FORMAT = 4   # bump when the packing order / layouts below change (4: the head is no longer cached)

    def __init__(self, cfg: Dict, state_dict: Dict[str, Tensor], device: torch.device, pack_cache: Optional[str] = None, *,
                 max_encoded_frames: Optional[int] = None):
        """`pack_cache`: path of an on-disk cache of the re-laid-out weights (SURVEY 8f-4).  When it exists and matches
        this cfg the load-time re-layout (BN folding, concatenations, permutations, fp16 casts, tables) is skipped and the
        packed tensors are uploaded as stored; otherwise it is written after packing.  Callers key the path by the
        checkpoint's md5 (load_model does).  The cache holds the front end and the encoder only: the head is packed from
        `state_dict` on every build, because head weights are trainable (a model's head may no longer be its checkpoint's)
        and re-laying it out costs one small matmul.

        `max_encoded_frames`: longest T' (encoder frames, 40 ms each) this engine encodes; None = _lib.REL_POS_MAX_T (768,
        30.7 s), at most the encoder's pos_emb_max_len (5000 for the shipped checkpoints, just under 200 s).  A rel_pos
        (v1) model's projected position tables grow with it: 16 x (2 * max - 1) x 768 fp16."""
        if device.type != "cuda":
            raise RuntimeError("gigaam_b200 runs on CUDA (sm_90a, H100) devices only; there is no CPU path")
        if device.index is None:      # an index-less "cuda" means the CURRENT device, not GPU 0
            device = torch.device("cuda", torch.cuda.current_device())
        self.lib = _lib.load()
        self.device = device
        self.cfg = cfg
        self._keep: List[Tensor] = []
        enc = cfg["encoder"]
        check_attention_heads(enc)
        gc_max = max_encoded_frames_config(max_encoded_frames, enc["pos_emb_max_len"])
        self.max_encoded_frames = gc_max or _lib.REL_POS_MAX_T
        # the limit sizes the rel_pos position tables that go through _dev(): a cache written for one limit must not be
        # replayed for another
        self._pack_sig = hashlib.sha256(json.dumps([self.PACK_FORMAT, cfg, self.max_encoded_frames], sort_keys=True,
                                                   default=str).encode()).hexdigest()
        self._pack_in: Optional[List[Tensor]] = None      # tensors replayed from the cache, in _dev() call order
        self._pack_out: Optional[List[Tensor]] = None     # tensors recorded for the cache
        if pack_cache is not None:
            self._pack_in = self._read_pack_cache(pack_cache)
            if self._pack_in is None:
                self._pack_out = []
        self._ws_enc = _WorkspaceCache(self.WS_CACHE)
        self._ws_mel = _WorkspaceCache(self.WS_CACHE)
        self._ws_dec = _WorkspaceCache(self.WS_CACHE)
        self._ws_joint = _WorkspaceCache(self.WS_CACHE)
        self._ws_align = _WorkspaceCache(self.WS_CACHE)
        self._ws_emo = _WorkspaceCache(self.WS_CACHE)
        self._resample_plans: Dict[int, Tuple[Tensor, int, int, int]] = {}
        self.handle = C.c_void_p()
        pre = cfg["preprocessor"]
        head = cfg.get("head") if isinstance(cfg, dict) else None
        sr = _cfg_get(pre, "sample_rate")
        self.n_fft = _cfg_get(pre, "n_fft", sr // 40)
        self.win = _cfg_get(pre, "win_length", sr // 40)
        self.hop = _cfg_get(pre, "hop_length", sr // 100)
        self.center = bool(_cfg_get(pre, "center", True))
        self.n_mels = _cfg_get(pre, "features")
        self.d_model = enc["d_model"]
        self.n_layers = enc["n_layers"]
        self.n_heads = enc["n_heads"]
        self.d_ff = self.d_model * enc["ff_expansion_factor"]
        if enc["self_attention_model"] not in ("rotary", "rel_pos"):
            raise ValueError(f"unknown self_attention_model {enc['self_attention_model']!r}")
        self.rel_pos = enc["self_attention_model"] == "rel_pos"
        self._pos_emb = rel_pos_embedding(self.max_encoded_frames, self.d_model).to(device) if self.rel_pos else None
        self.head_type = 0
        self.num_classes = 0
        self._head_bufs: Dict[str, Tensor] = {}     # packed head tensors the handle points at, by gam_weights field
        self.head_signature = None                  # set by the owning model: the head parameters this pack reflects
        self.max_symbols = 10
        gc = _lib.GamConfig()
        gc.sample_rate, gc.n_mels, gc.n_fft, gc.win_length, gc.hop_length, gc.center = sr, self.n_mels, self.n_fft, self.win, self.hop, int(self.center)
        gc.feat_in, gc.n_layers, gc.d_model, gc.n_heads, gc.d_ff = enc["feat_in"], self.n_layers, self.d_model, self.n_heads, self.d_ff
        gc.subsampling = 0 if enc["subsampling"] == "conv2d" else 1
        gc.subs_kernel_size = enc["subs_kernel_size"]
        gc.conv_kernel_size = enc["conv_kernel_size"]
        gc.conv_norm = 0 if enc["conv_norm_type"] == "batch_norm" else 1
        gc.self_attention = 1 if self.rel_pos else 0
        gc.pos_emb_max_len = enc["pos_emb_max_len"]
        gc.max_encoded_frames = gc_max
        gw = _lib.GamWeights()
        sd = state_dict
        self._pack_frontend(gw, sd)
        self._pack_subsampling(gw, sd, enc)
        self._pack_rope(gw, enc)
        self._layers = (_lib.GamLayerWeights * self.n_layers)()
        for l in range(self.n_layers):
            self._pack_layer(self._layers[l], sd, l, enc)
        gw.layers = C.cast(self._layers, C.POINTER(_lib.GamLayerWeights))
        if head is not None:
            if head["type"] == "ctc":
                self.head_type, self.num_classes = 1, head["num_classes"]
                gw.ctc_w = self._dev_head("ctc_w", sd["head.decoder_layers.0.weight"].reshape(self.num_classes, -1))
                gw.ctc_b = self._dev_head("ctc_b", sd["head.decoder_layers.0.bias"])
            elif head["type"] == "emo":
                # Linear(d, C) over the mean of the encoder frames (gigaam/model.py:272-293), fp32 like the reference's head
                self.head_type, self.num_classes = 3, head["out_features"]
                gw.emo_w = self._dev_head("emo_w", sd["head.weight"])
                gw.emo_b = self._dev_head("emo_b", sd["head.bias"])
            else:
                self._pack_rnnt(gw, gc, sd, head)
                self.max_symbols = int(_cfg_get(cfg.get("decoding", {}), "max_symbols_per_step", 10))
        gc.head, gc.num_classes, gc.max_symbols = self.head_type, self.num_classes, self.max_symbols
        self.gam_config = gc
        with torch.cuda.device(device):
            rc = self.lib.gam_create(C.byref(gc), C.byref(gw), device.index, C.byref(self.handle))
        _lib.check(self.lib, self.handle, rc, "gam_create")
        if self._pack_out is not None:
            self._write_pack_cache(pack_cache)
        self.pack_cache_hit = self._pack_in is not None
        self._pack_in = self._pack_out = None

    # ------------------------------------------------------------------ packing helpers
    def _dev(self, t, dtype: Optional[torch.dtype] = None) -> int:
        """Upload one packed tensor (or, given a callable, the tensor it computes) and keep it alive; returns the device
        pointer.  With a cache hit the stored tensor of this call position is uploaded and `t` is never evaluated."""
        if self._pack_in is not None:
            t = self._pack_in[len(self._keep)]
        else:
            t = (t() if callable(t) else t).detach()
            if dtype is not None:
                t = t.to(dtype)
            if self._pack_out is not None:
                self._pack_out.append(t.cpu().contiguous())
        t = t.to(self.device).contiguous()
        self._keep.append(t)
        return t.data_ptr()

    def _dev_head(self, name: str, t: Tensor) -> int:
        """Upload one packed head tensor (fp32) outside the pack cache: it is neither replayed from nor written to it.
        repack_head() later rewrites it in place.  The buffer is always a copy, never a view of the parameter (a repack
        would bump the parameter's version counter and so repack again on every later call), and a normal tensor even
        when the engine is built under torch.inference_mode() (a repack outside it could not write an inference tensor)."""
        with torch.inference_mode(False):
            buf = torch.empty(t.shape, dtype=torch.float32, device=self.device)
            buf.copy_(t.detach())
        self._head_bufs[name] = buf
        return buf.data_ptr()

    def _read_pack_cache(self, path: str) -> Optional[List[Tensor]]:
        if not os.path.isfile(path):
            return None
        try:
            blob = torch.load(path, map_location="cpu", weights_only=True)
            if blob.get("signature") == self._pack_sig and isinstance(blob.get("tensors"), list):
                return blob["tensors"]
        except Exception:
            pass
        return None          # stale or unreadable: repack and overwrite

    def _write_pack_cache(self, path: str) -> None:
        try:
            tmp = f"{path}.tmp{os.getpid()}"
            torch.save({"signature": self._pack_sig, "tensors": self._pack_out}, tmp)
            os.replace(tmp, path)
        except OSError:
            pass             # a read-only cache directory must not break loading

    def _pack_frontend(self, gw, sd):
        n = self.n_fft
        K = n // 2 + 1
        window = sd["preprocessor.featurizer.0.spectrogram.window"].float()
        if window.numel() != n:
            raise NotImplementedError("win_length != n_fft")
        idx = torch.arange(K, dtype=torch.float64)
        ang = 2.0 * math.pi * torch.outer(idx, idx) / n  # [n, k]
        gw.window = self._dev(window)
        gw.dft_cos = self._dev(torch.cos(ang).float())
        gw.dft_sin = self._dev(torch.sin(ang).float())
        fb = sd["preprocessor.featurizer.0.mel_scale.fb"].float().cpu()
        gw.mel_fb = self._dev(fb)
        # tensor-core front end: split-precision DFT basis + bin range of every mel filter
        if K <= 256:
            gw.dft_w = self._dev(lambda: split_dft_basis(n))
            nz = fb != 0
            lo = torch.where(nz.any(0), nz.float().argmax(0), torch.zeros(fb.shape[1], dtype=torch.long))
            hi = torch.where(nz.any(0), fb.shape[0] - nz.flip(0).float().argmax(0), torch.zeros(fb.shape[1], dtype=torch.long))
            gw.mel_lo = self._dev(lo.to(torch.int32))
            gw.mel_hi = self._dev(hi.to(torch.int32))
            self._logmel_tc = True
        else:
            self._logmel_tc = False

    def _pack_subsampling(self, gw, sd, enc):
        p = "encoder.pre_encode."
        d = self.d_model
        if enc["subsampling"] == "conv1d":
            # Conv1d weights [out, in, k] -> (out, k, in): K order (tap, channel) of the implicit GEMM
            for i, name in ((0, "c1d_w1"), (2, "c1d_w2")):
                setattr(gw, name, self._dev(pack_conv1d_weight(sd[f"{p}conv.{i}.weight"].float()), torch.float16))
            gw.c1d_b1 = self._dev(sd[p + "conv.0.bias"].float())
            gw.c1d_b2 = self._dev(sd[p + "conv.2.bias"].float())
            return
        w1 = sd[p + "conv.0.weight"].float()                     # [C, 1, 3, 3]
        gw.sub1_w = self._dev(w1.reshape(d, 9))
        gw.sub1_b = self._dev(sd[p + "conv.0.bias"].float())
        w2 = sd[p + "conv.2.weight"].float()                     # [C_out, C_in, kt, kf]
        gw.sub2_w = self._dev(lambda: pack_conv2_weight(w2), torch.float16)
        gw.sub2_b = self._dev(sd[p + "conv.2.bias"].float())
        wo = sd[p + "out.weight"].float()                        # [d, C*F2] with K index c*F2 + f
        gw.sub_out_w = self._dev(lambda: pack_sub_out_weight(wo, d), torch.float16)
        gw.sub_out_b = self._dev(sd[p + "out.bias"].float())

    def _pack_rope(self, gw, enc):
        dk = self.d_model // self.n_heads
        base = enc["pos_emb_max_len"]  # the reference passes pos_emb_max_len as the rotary base (encoder.py:546-548)
        cos, sin = rotary_half_tables(dk, base, enc["pos_emb_max_len"])
        gw.rope_cos = self._dev(cos)
        gw.rope_sin = self._dev(sin)

    def _pack_layer(self, lw, sd, l: int, enc):
        q = f"encoder.layers.{l}."
        d = self.d_model
        h16 = torch.float16

        def f(name):
            return sd[q + name].float()

        lw.ln_ff1_g, lw.ln_ff1_b = self._dev(f("norm_feed_forward1.weight")), self._dev(f("norm_feed_forward1.bias"))
        lw.ff1_w1, lw.ff1_b1 = self._dev(f("feed_forward1.linear1.weight"), h16), self._dev(f("feed_forward1.linear1.bias"))
        lw.ff1_w2, lw.ff1_b2 = self._dev(f("feed_forward1.linear2.weight"), h16), self._dev(f("feed_forward1.linear2.bias"))
        lw.ln_att_g, lw.ln_att_b = self._dev(f("norm_self_att.weight")), self._dev(f("norm_self_att.bias"))
        if self.rel_pos:
            w4, b4 = pack_rel_pos_qkv(f("self_attn.linear_q.weight"), f("self_attn.linear_q.bias"),
                                      f("self_attn.linear_k.weight"), f("self_attn.linear_k.bias"),
                                      f("self_attn.linear_v.weight"), f("self_attn.linear_v.bias"),
                                      f("self_attn.pos_bias_u"), f("self_attn.pos_bias_v"))
            lw.w_qkv_rel, lw.b_qkv_rel = self._dev(w4, h16), self._dev(b4)
            # linear_pos (no bias, encoder.py:198,219) of a constant table is a constant: projected once at load time
            lw.pos_proj = self._dev(lambda: self._pos_emb @ f("self_attn.linear_pos.weight").to(self.device).t(), h16)
            lw.w_qk = lw.b_qk = lw.w_v = lw.b_v = None
        else:
            # [W_q ; W_k ; W_v] and their biases in ONE allocation each: w_v / b_v point behind w_qk / b_qk, which lets the
            # library run the three projections as a single launch (two A operands: rope(u) for q, k and u for v)
            w_qkv = self._dev(torch.cat([f("self_attn.linear_q.weight"), f("self_attn.linear_k.weight"),
                                         f("self_attn.linear_v.weight")], 0), h16)
            b_qkv = self._dev(torch.cat([f("self_attn.linear_q.bias"), f("self_attn.linear_k.bias"), f("self_attn.linear_v.bias")], 0))
            lw.w_qk, lw.w_v = w_qkv, w_qkv + 2 * d * d * 2
            lw.b_qk, lw.b_v = b_qkv, b_qkv + 2 * d * 4
            lw.w_qkv_rel = lw.b_qkv_rel = lw.pos_proj = None
        lw.w_o, lw.b_o = self._dev(f("self_attn.linear_out.weight"), h16), self._dev(f("self_attn.linear_out.bias"))
        lw.ln_conv_g, lw.ln_conv_b = self._dev(f("norm_conv.weight")), self._dev(f("norm_conv.bias"))
        # GLU pairing: accumulator tile j (256 columns) = [value rows j*128.. | gate rows d + j*128..]
        perm = glu_row_permutation(d)
        w1 = f("conv.pointwise_conv1.weight").reshape(2 * d, d)
        lw.pw1_w, lw.pw1_b = self._dev(w1[perm], h16), self._dev(f("conv.pointwise_conv1.bias")[perm])
        dw = f("conv.depthwise_conv.weight").reshape(d, -1)
        db = f("conv.depthwise_conv.bias")
        if enc["conv_norm_type"] == "batch_norm":
            dw, db = fold_batchnorm(dw, db, f("conv.batch_norm.weight"), f("conv.batch_norm.bias"),
                                    f("conv.batch_norm.running_mean"), f("conv.batch_norm.running_var"))
            lw.cn_g, lw.cn_b = None, None
        else:
            lw.cn_g, lw.cn_b = self._dev(f("conv.batch_norm.weight")), self._dev(f("conv.batch_norm.bias"))
        lw.dw_w, lw.dw_b = self._dev(dw.t()), self._dev(db)     # taps transposed to [k, d]: coalesced per-tap loads
        lw.pw2_w = self._dev(f("conv.pointwise_conv2.weight").reshape(d, d), h16)
        lw.pw2_b = self._dev(f("conv.pointwise_conv2.bias"))
        lw.ln_ff2_g, lw.ln_ff2_b = self._dev(f("norm_feed_forward2.weight")), self._dev(f("norm_feed_forward2.bias"))
        lw.ff2_w1, lw.ff2_b1 = self._dev(f("feed_forward2.linear1.weight"), h16), self._dev(f("feed_forward2.linear1.bias"))
        lw.ff2_w2, lw.ff2_b2 = self._dev(f("feed_forward2.linear2.weight"), h16), self._dev(f("feed_forward2.linear2.bias"))
        lw.ln_out_g, lw.ln_out_b = self._dev(f("norm_out.weight")), self._dev(f("norm_out.bias"))

    def _pack_rnnt(self, gw, gc, sd, head):
        dc, jt = head["decoder"], head["joint"]
        if dc["pred_rnn_layers"] != 1:
            raise NotImplementedError("multi-layer prediction LSTM")
        self.head_type, self.num_classes = 2, jt["num_classes"]
        self.pred_hidden = dc["pred_hidden"]
        gc.pred_hidden, gc.joint_hidden = dc["pred_hidden"], jt["joint_hidden"]
        packed = rnnt_head_packing(sd)
        for name in RNNT_HEAD_FIELDS:
            setattr(gw, name, self._dev_head(name, packed[name]))

    def repack_head(self, sd: Dict[str, Tensor]) -> None:
        """Re-lay the head weights out from `sd` (the model's current head parameters, key "head.*") into the device
        buffers the handle already points at, on the current stream.  The encoder is untouched, the handle and any captured
        CUDA graph stay valid, and nothing is written to the pack cache."""
        if self.head_type == 1:
            packed = {"ctc_w": sd["head.decoder_layers.0.weight"].reshape(self.num_classes, -1), "ctc_b": sd["head.decoder_layers.0.bias"]}
        elif self.head_type == 2:
            packed = rnnt_head_packing({k: v.to(self.device) for k, v in sd.items()})
        elif self.head_type == 3:
            packed = {"emo_w": sd["head.weight"], "emo_b": sd["head.bias"]}
        else:
            return
        with torch.no_grad(), torch.cuda.device(self.device):
            for name, t in packed.items():
                self._head_bufs[name].copy_(t.detach().reshape(self._head_bufs[name].shape))

    # ------------------------------------------------------------------ calls
    def _stream(self) -> C.c_void_p:
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _call(self, name: str, *args) -> None:
        """Run entry point `name` on this engine's handle and current stream: a tensor passes its data pointer, None passes
        NULL.  A nonzero return raises GamError with the library's message."""
        args = [a.data_ptr() if isinstance(a, Tensor) else a for a in args]
        with torch.cuda.device(self.device):
            rc = getattr(self.lib, name)(self.handle, *args, self._stream())
        _lib.check(self.lib, self.handle, rc, name)

    def _ws(self, cache: Optional["_WorkspaceCache"], key, query: str, *sizes, what: str) -> Tensor:
        """The workspace entry point `query` sizes for `sizes`, from `cache` (None: a fresh one).  A negative size, which the
        library returns for sizes it refuses, raises ValueError(what)."""
        nbytes = int(getattr(self.lib, query)(self.handle, *sizes))
        if nbytes < 0:
            raise ValueError(what)
        if cache is None:
            return torch.empty(max(nbytes, 1), dtype=torch.uint8, device=self.device)
        return cache.get(key, nbytes, self.device)

    def logmel_frames(self, n: int) -> int:
        return int(self.lib.gam_logmel_frames(self.handle, int(n)))

    def encoded_frames(self, m: int) -> int:
        return int(self.lib.gam_encoded_frames(self.handle, int(m)))

    def workspace(self, B: int, M: int) -> Tensor:
        return self._ws_enc.get((B, M), int(self.lib.gam_workspace_bytes(self.handle, B, M)), self.device)

    def held_workspaces(self, B: int, N: int) -> List[Tensor]:
        """The scratch tensors a step over a [B, N] waveform batch touches.  A captured CUDA graph stores this list: the
        pointers it baked stay valid however many other shapes pass through the engine afterwards."""
        M = self.logmel_frames(N)
        T = self.encoded_frames(M)
        held = [self._ws_mel.peek((B, N)), self._ws_enc.peek((B, M)), self._ws_dec.peek((B, T)), self._ws_emo.peek((B, T))]
        return [t for t in held if t is not None]

    def logmel(self, wav: Tensor, fused: bool = False) -> Tensor:
        """[B, N] f32 on device -> [B, n_mels, M] f32 (FeatureExtractor.forward, gigaam/preprocess.py:94-98).
        `fused=True` selects the single CUDA-core kernel (no workspace) instead of the tensor-core DFT."""
        assert wav.is_cuda and wav.dtype == torch.float32 and wav.dim() == 2
        wav = wav.contiguous()
        B, N = wav.shape
        M = self.logmel_frames(N)
        mel = torch.empty((B, self.n_mels, M), dtype=torch.float32, device=self.device)
        if self._logmel_tc and not fused:
            ws = self._ws_mel.get((B, N), int(self.lib.gam_logmel_workspace_bytes(self.handle, B, N)), self.device)
            self._call("gam_logmel_tc", wav, B, N, mel, ws, ws.numel())
        else:
            self._call("gam_logmel", wav, B, N, mel)
        return mel

    # ------------------------------------------------------------------ resampling to 16 kHz (INTEGRATION.md §7k)
    def resample_plan(self, sample_rate: int) -> Tuple[Tensor, int, int, int]:
        """(table, o, n, w) of gam_resample from `sample_rate`: the device table is preprocess.resample_table transposed to
        [2 w + o, n], built once per rate.  ValueError for the rates preprocess.resample_ratio refuses and for 16 kHz, which
        is not resampled."""
        from .preprocess import SAMPLE_RATE, resample_ratio, resample_table
        if sample_rate == SAMPLE_RATE:
            raise ValueError("16 kHz audio is not resampled")
        plan = self._resample_plans.get(sample_rate)
        if plan is None:
            o, n, w = resample_ratio(sample_rate)
            plan = (resample_table(sample_rate).t().contiguous().to(self.device), o, n, w)
            self._resample_plans[int(sample_rate)] = plan
        return plan

    def resample_spans(self, x: Tensor, spans: Tensor, sample_rate: int, out: Tensor) -> Tensor:
        """gam_resample, the span form: row b of x (device f32 [B, P]) holds samples [in_begin[b], in_end[b]) of its signal,
        and row b of out (device f32 [B, C]) gets its outputs [out_begin[b], out_end[b]) from column 0; spans = int64
        [in_begin, in_end, out_begin, out_end] x [B].  Other columns of out are not written.  Host spans are checked first
        (ValueError for an inverted range, a negative out_begin, or more samples or outputs than the rows hold); device spans
        are passed as they are (a CUDA graph can capture the call)."""
        table, o, n, w = self.resample_plan(sample_rate)
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and out.is_cuda and out.dtype == torch.float32
        B = x.shape[0]
        if spans.shape != (4, B) or out.shape[0] != B:
            raise ValueError(f"resample: spans of shape {tuple(spans.shape)} and {out.shape[0]} output rows for {B} input rows")
        if spans.device.type == "cpu":
            in_lo, in_hi, out_lo, out_hi = spans.tolist()
            for b in range(B):
                if in_hi[b] < in_lo[b] or out_hi[b] < out_lo[b] or out_lo[b] < 0:
                    raise ValueError(f"resample: row {b} has an inverted span (in [{in_lo[b]}, {in_hi[b]}), out "
                                     f"[{out_lo[b]}, {out_hi[b]}))")
                if in_hi[b] - in_lo[b] > x.shape[1] or out_hi[b] - out_lo[b] > out.shape[1]:
                    raise ValueError(f"resample: row {b} spans more samples or outputs than its row holds")
            spans = spans.to(device=self.device, dtype=torch.int64)
        if not out.is_contiguous():
            raise ValueError("resample: out must be contiguous")
        if out.shape[1] == 0:
            return out
        x = x.contiguous()
        if x.shape[1] == 0:
            x = torch.zeros((B, 1), dtype=torch.float32, device=self.device)
        self._call("gam_resample", x, x.shape[1], B, spans.contiguous(), table, table.shape[0], table.shape[1], o, n, out, out.shape[1])
        return out

    def resample(self, x: Tensor, lengths: Tensor, sample_rate: int) -> Tuple[Tensor, Tensor]:
        """Resample the batch x [B, L] (row b: lengths[b] samples at `sample_rate`) to 16 kHz in one launch: -> (y device f32
        [B, max length], zero past each row's length; int64 lengths ceil(n lengths / o) on lengths' device).  16 kHz input is returned as it is, with no launch."""
        from .preprocess import SAMPLE_RATE, resampled_length
        if sample_rate == SAMPLE_RATE:
            return x, lengths
        self.resample_plan(sample_rate)
        lens = [int(v) for v in lengths.reshape(-1).tolist()]
        if x.dim() != 2 or len(lens) != x.shape[0] or any(not 0 <= v <= x.shape[1] for v in lens):
            raise ValueError(f"resample: lengths {lens} do not fit a batch of shape {tuple(x.shape)}")
        out_len = [resampled_length(v, sample_rate) for v in lens]
        spans = torch.tensor([[0] * len(lens), lens, [0] * len(lens), out_len], dtype=torch.int64)
        y = torch.zeros((len(lens), max(out_len, default=0)), dtype=torch.float32, device=self.device)
        self.resample_spans(x.to(device=self.device, dtype=torch.float32), spans, sample_rate, y)
        return y, torch.tensor(out_len, dtype=torch.int64, device=lengths.device)

    def encode(self, mel: Tensor, mel_len: Tensor, n_layers_run: int = -1) -> Tuple[Tensor, Tensor]:
        """[B, F, M] f32, [B] i64 -> ([B, T', d] f32 row-major, [B] i32)"""
        assert mel.is_cuda and mel.dtype == torch.float32 and mel.dim() == 3
        mel = mel.contiguous()
        mel_len = mel_len.to(device=self.device, dtype=torch.int64).contiguous()
        B, _, M = mel.shape
        T = self.encoded_frames(M)
        ws = self.workspace(B, M)
        enc = torch.empty((B, T, self.d_model), dtype=torch.float32, device=self.device)
        enc_len = torch.empty((B,), dtype=torch.int32, device=self.device)
        self._call("gam_encode", mel, mel_len, B, M, ws, ws.numel(), enc, enc_len, n_layers_run)
        return enc, enc_len

    def hyp_width(self, T: int) -> int:
        """Row pitch of the id / frame matrices for T encoder frames."""
        return T if self.head_type == 1 else T * self.max_symbols

    def packed_hypotheses(self, rows: int, T: int) -> Tensor:
        """Zeroed int32 buffer [ids rows x W | frames rows x W | counts rows] (the layout gam_gather_hyps all-gathers)."""
        w = self.hyp_width(T)
        return torch.zeros(2 * rows * w + rows, dtype=torch.int32, device=self.device)

    def greedy(self, enc_btd: Tensor, enc_len: Tensor, packed: Optional[Tensor] = None, scores: bool = False) -> Tuple[Tensor, ...]:
        """enc [B, T, d] f32 contiguous, len [B] -> (ids [B, max_out] i32, frames, counts [B] i32) on device.
        `packed` (from packed_hypotheses, rows >= B): the results are written into that buffer and returned as views of it.
        `scores=True` decodes with gam_*_greedy_scored (the same ids / frames / counts) and also returns token_logp
        [B, max_out] f32, path_logp [B] f32 and path_rows [B] i32 (include/gigaam_b200.h has the definitions)."""
        assert enc_btd.is_cuda and enc_btd.dtype == torch.float32 and enc_btd.is_contiguous()
        if self.head_type == 0:
            raise RuntimeError("model has no head to decode with")
        if scores and packed is not None:
            raise ValueError("scores are not part of the packed hypothesis layout")
        B, T, _ = enc_btd.shape
        enc_len = enc_len.to(device=self.device, dtype=torch.int32).contiguous()
        max_out = self.hyp_width(T)
        if packed is not None:
            rows = packed.numel() // (2 * max_out + 1)
            assert rows >= B and packed.numel() == rows * (2 * max_out + 1) and packed.dtype == torch.int32
            ids = packed[: rows * max_out].view(rows, max_out)[:B]
            frames = packed[rows * max_out: 2 * rows * max_out].view(rows, max_out)[:B]
            counts = packed[2 * rows * max_out: 2 * rows * max_out + B]
        else:
            ids = torch.empty((B, max_out), dtype=torch.int32, device=self.device)
            frames = torch.empty((B, max_out), dtype=torch.int32, device=self.device)
            counts = torch.empty((B,), dtype=torch.int32, device=self.device)
        if scores:
            token_logp = torch.empty((B, max_out), dtype=torch.float32, device=self.device)
            path_logp = torch.empty((B,), dtype=torch.float32, device=self.device)
            path_rows = torch.empty((B,), dtype=torch.int32, device=self.device)
            ws = self._ws_dec.get((B, T), int(self.lib.gam_decode_scored_workspace_bytes(self.handle, B, T)), self.device)
            self._call("gam_ctc_greedy_scored" if self.head_type == 1 else "gam_rnnt_greedy_scored", enc_btd, enc_len, B, T, ws,
                       ws.numel(), ids, frames, counts, max_out, token_logp, path_logp, path_rows)
            return ids, frames, counts, token_logp, path_logp, path_rows
        ws = self._ws_dec.get((B, T), int(self.lib.gam_decode_workspace_bytes(self.handle, B, T)), self.device)
        self._call("gam_ctc_greedy" if self.head_type == 1 else "gam_rnnt_greedy", enc_btd, enc_len, B, T, ws, ws.numel(), ids, frames,
                   counts, max_out)
        return ids, frames, counts

    # ------------------------------------------------------------------ resumable greedy decoding (gam_*_greedy_resume)
    def decode_state(self, n: int = 1) -> Tensor:
        """n fresh decoding streams (gam_decode_state_init): uint8 [n, gam_decode_state_bytes] on the device."""
        nbytes = int(self.lib.gam_decode_state_bytes(self.handle))
        if nbytes < 0:
            raise RuntimeError("model has no head to decode with")
        state = torch.empty((n, nbytes), dtype=torch.uint8, device=self.device)
        self._call("gam_decode_state_init", state, n)
        return state

    def decode_buffers(self, B: int, max_out: int, n_frames: int = 0, scores: bool = False) -> "DecodeBuffers":
        """The outputs greedy_resume appends to, for B streams: ids / frames [B, max_out], counts [B] = 0 and, with `scores`,
        token_logp [B, max_out], the running path_logp / path_rows [B] and frame_logp (f64) / frame_rows [B, n_frames] = 0."""
        i32 = dict(dtype=torch.int32, device=self.device)
        out = DecodeBuffers(torch.empty((B, max_out), **i32), torch.empty((B, max_out), **i32), torch.zeros((B,), **i32))
        if not scores:
            return out
        return out._replace(token_logp=torch.empty((B, max_out), dtype=torch.float32, device=self.device),
                            path_logp=torch.zeros((B,), dtype=torch.float32, device=self.device), path_rows=torch.zeros((B,), **i32),
                            frame_logp=torch.zeros((B, n_frames), dtype=torch.float64, device=self.device),
                            frame_rows=torch.zeros((B, n_frames), **i32))

    def greedy_resume(self, enc_btd: Tensor, lo: Tensor, hi: Tensor, frame_base: Tensor, state: Tensor, out: "DecodeBuffers",
                      scores: bool = False, boost: Optional[Tuple[Tensor, Tensor]] = None) -> None:
        """Decode frames [lo[b], hi[b]) of enc [B, T, d] (f32 contiguous) continuing stream b of `state` (decode_state) and
        append to `out` (decode_buffers, emitted frames frame_base[b] + t).  lo / hi / frame_base: device int32 [B].  Decoding
        an utterance in consecutive ranges gives `greedy`'s bits (include/gigaam_b200.h, gam_ctc_greedy_resume).  `boost`:
        a boost graph's device tables (next int32 [S, V+1], bonus f32 [S, V+1], decoding.boost_graph) steer an RNN-T decoder
        (gam_rnnt_greedy_boost); None runs gam_*_greedy_resume."""
        assert enc_btd.is_cuda and enc_btd.dtype == torch.float32 and enc_btd.is_contiguous() and enc_btd.dim() == 3
        B, T, _ = enc_btd.shape
        for t in (lo, hi, frame_base):
            assert t.device == self.device and t.dtype == torch.int32 and t.is_contiguous() and t.numel() == B
        assert state.dtype == torch.uint8 and state.is_contiguous() and state.shape[0] >= B
        assert state.shape[1] == int(self.lib.gam_decode_state_bytes(self.handle))
        assert out.ids.shape[0] >= B and out.ids.is_contiguous() and out.frames.is_contiguous()
        if scores and out.token_logp is None:
            raise ValueError("greedy_resume: scores need buffers from decode_buffers(..., scores=True)")
        ws = self._ws_dec.get(("resume", B, T), int(self.lib.gam_decode_resume_workspace_bytes(self.handle, B, T)), self.device)
        sc = [out.token_logp, out.path_logp, out.path_rows, out.frame_logp, out.frame_rows] if scores else [None] * 5
        pitch = out.frame_logp.shape[1] if scores else 0
        args = (enc_btd, B, T, lo, hi, frame_base, state, ws, ws.numel(), out.ids, out.frames, out.counts, out.ids.shape[1], *sc, pitch)
        if boost is not None:
            nxt, bonus = boost
            assert nxt.shape == bonus.shape and nxt.dim() == 2 and nxt.shape[1] == self.num_classes
            assert nxt.dtype == torch.int32 and bonus.dtype == torch.float32 and nxt.is_contiguous() and bonus.is_contiguous()
            assert nxt.device == bonus.device == self.device
            self._call("gam_rnnt_greedy_boost", *args, nxt, bonus, nxt.shape[0])
            return
        self._call("gam_ctc_greedy_resume" if self.head_type == 1 else "gam_rnnt_greedy_resume", *args)

    def ctc_log_probs(self, enc_btd: Tensor) -> Tensor:
        """enc [B, T, d] f32 contiguous -> log_probs [B, T, V+1] f32 (CTCHead.forward, gigaam/decoder.py:18-21)."""
        assert enc_btd.is_cuda and enc_btd.dtype == torch.float32 and enc_btd.is_contiguous() and enc_btd.dim() == 3
        if self.head_type != 1:
            raise RuntimeError("model has no CTC head")
        B, T, _ = enc_btd.shape
        out = torch.empty((B, T, self.num_classes), dtype=torch.float32, device=self.device)
        self._call("gam_ctc_log_probs", enc_btd, B, T, out)
        return out

    def rnnt_joint(self, enc: Tensor, dec: Tensor) -> Tensor:
        """enc [B, T, d], dec [B, U, pred_hidden] f32 contiguous -> [B, T, U, V+1] log-probs (RNNTJoint.joint,
        gigaam/decoder.py:41-47).  The projection workspace is cached per (B, T, U) like the decode workspace."""
        assert enc.is_cuda and dec.is_cuda and enc.dtype == dec.dtype == torch.float32
        assert enc.is_contiguous() and dec.is_contiguous() and enc.dim() == dec.dim() == 3
        if self.head_type != 2:
            raise RuntimeError("model has no RNN-T head")
        B, T, _ = enc.shape
        U = dec.shape[1]
        if dec.shape[0] != B:
            raise ValueError(f"joint: encoder batch {B} != decoder batch {dec.shape[0]}")
        out = torch.empty((B, T, U, self.num_classes), dtype=torch.float32, device=self.device)
        ws = self._ws(self._ws_joint, (B, T, U), "gam_rnnt_joint_workspace_bytes", B, T, U, what=f"joint: bad sizes B={B}, T={T}, U={U}")
        self._call("gam_rnnt_joint", enc, dec, B, T, U, ws, ws.numel(), out)
        return out

    def _predict_sizes(self, x: Optional[Tensor], batch_size: int) -> Tuple[int, int, int]:
        """(B, U, H) of a prediction-network call, after the checks rnnt_predict and rnnt_predict_train share."""
        if self.head_type != 2:
            raise RuntimeError("model has no RNN-T head")
        if x is not None:
            assert x.is_cuda and x.dtype == torch.int64 and x.is_contiguous() and x.dim() == 2
        B, U = (x.shape[0], x.shape[1]) if x is not None else (int(batch_size), 1)
        return B, U, self.pred_hidden

    def rnnt_predict(self, x: Optional[Tensor], h: Optional[Tensor], c: Optional[Tensor], batch_size: int = 1
                     ) -> Tuple[Tensor, Tensor, Tensor]:
        """x [B, U] i64 or None (one step from the zero embedding), h / c [B, H] f32 contiguous or None (zeros)
        -> (g [B, U, H], h1 [B, H], c1 [B, H]) (RNNTDecoder.predict, gigaam/decoder.py:85-102)."""
        B, U, H = self._predict_sizes(x, batch_size)
        for name, t in (("h", h), ("c", c)):
            if t is not None:
                assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
                if tuple(t.shape) != (B, H):
                    raise ValueError(f"predict: state {name} has shape {tuple(t.shape)}, expected ({B}, {H})")
        g, h1, c1 = self._empty(B, U, H), self._empty(B, H), self._empty(B, H)
        self._call("gam_rnnt_predict", x, h, c, B, U, g, h1, c1)
        return g, h1, c1

    # ------------------------------------------------------------------ alignment of known transcripts (align.cu)
    def _align_outputs(self, B: int, U: int) -> Tuple[Tensor, ...]:
        i32 = dict(dtype=torch.int32, device=self.device)
        f32 = dict(dtype=torch.float32, device=self.device)
        return (torch.empty((B, U), **i32), torch.empty((B, U), **f32), torch.empty((B,), **f32), torch.empty((B,), **f32),
                torch.empty((B,), **i32))

    @staticmethod
    def _i32(t: Tensor, device) -> Tensor:
        return t.to(device=device, dtype=torch.int32).contiguous()

    def ctc_align(self, log_probs: Tensor, enc_len: Tensor, targets: Tensor, target_len: Tensor) -> Tuple[Tensor, ...]:
        """log_probs [B, T, V+1] f32 contiguous (ctc_log_probs), enc_len [B], targets [B, U], target_len [B] -> (frames [B, U] i32,
        token_logp [B, U] f32, viterbi_logp [B] f32, log_likelihood [B] f32, path_rows [B] i32) on the device (gam_ctc_align)."""
        assert log_probs.is_cuda and log_probs.dtype == torch.float32 and log_probs.is_contiguous() and log_probs.dim() == 3
        if self.head_type != 1:
            raise RuntimeError("model has no CTC head")
        B, T, _ = log_probs.shape
        U = targets.shape[1]
        ws = self._ws(self._ws_align, ("ctc", B, T, U), "gam_ctc_align_workspace_bytes", B, T, U,
                      what=f"ctc_align: bad sizes B={B}, T={T}, U={U}")
        enc_len, targets, target_len = (self._i32(t, self.device) for t in (enc_len, targets, target_len))
        outs = self._align_outputs(B, U)
        self._call("gam_ctc_align", log_probs, enc_len, targets, target_len, B, T, U, ws, ws.numel(), *outs)
        return outs

    def ctc_align_long(self, log_probs: Tensor, enc_len: Tensor, targets: Tensor, target_len: Tensor,
                       cluster_ctas: Optional[int] = None, gaps: Optional[Tuple[Tensor, float]] = None,
                       skips: Optional[float] = None) -> Tuple[Tensor, ...]:
        """ctc_align for recordings of any length and up to 65 536 tokens (gam_ctc_align_long): the same arguments and
        outputs, and the same bits on every input ctc_align accepts.  `cluster_ctas` forces the number of CTAs per utterance
        (gam_test_ctc_align_long*); the plan used, (CTAs, states per CTA), is then kept in `last_align_long_plan`.
        `gaps` = (line_edges [B, U] u8, log_theta) runs gam_ctc_align_long_gaps instead and appends its three outputs
        (unmatched [B, T] u8, unmatched_rows [B] i32, unmatched_logp [B] f32).  `skips` = log_psi (with `gaps`; log_theta
        = -inf for skips without gaps) runs gam_ctc_align_long_skips and appends (skipped_rows [B] i32, skip_logp [B] f32)."""
        assert log_probs.is_cuda and log_probs.dtype == torch.float32 and log_probs.is_contiguous() and log_probs.dim() == 3
        if self.head_type != 1:
            raise RuntimeError("model has no CTC head")
        if skips is not None and gaps is None:
            raise ValueError("ctc_align_long: skips needs gaps=(line_edges, log_theta); pass log_theta=-inf for skips alone")
        B, T, _ = log_probs.shape
        U = targets.shape[1]
        if skips is not None:
            name, kind = "gam_ctc_align_long_skips", "ctc_long_skips"
        elif gaps is not None:
            name, kind = "gam_ctc_align_long_gaps", "ctc_long_gaps"
        else:
            name, kind = "gam_ctc_align_long", "ctc_long"
        ws = self._ws(self._ws_align, (kind, B, T, U), name + "_workspace_bytes", B, T, U,
                      what=f"ctc_align_long: bad sizes B={B}, T={T}, U={U}")
        enc_len, targets, target_len = (self._i32(t, self.device) for t in (enc_len, targets, target_len))
        outs = self._align_outputs(B, U)
        head = [log_probs, enc_len, targets, target_len]
        if gaps is not None:
            line_edges, log_theta = gaps
            line_edges = line_edges.to(device=self.device, dtype=torch.uint8).contiguous()
            if tuple(line_edges.shape) != (B, U):
                raise ValueError(f"ctc_align_long: line_edges has shape {tuple(line_edges.shape)}, expected ({B}, {U})")
            outs = outs + (torch.empty((B, T), dtype=torch.uint8, device=self.device),
                           torch.empty((B,), dtype=torch.int32, device=self.device),
                           torch.empty((B,), dtype=torch.float32, device=self.device))
            head += [line_edges]
        if skips is not None:
            outs = outs + (torch.empty((B,), dtype=torch.int32, device=self.device),
                           torch.empty((B,), dtype=torch.float32, device=self.device))
        sizes = [B, T, U] + ([] if gaps is None else [float(log_theta)]) + ([] if skips is None else [float(skips)])
        args = head + sizes + [ws, ws.numel(), *outs]
        if cluster_ctas is None:
            self._call(name, *args)
        else:
            plan = (C.c_int32 * 2)()
            test_name = {"gam_ctc_align_long": "gam_test_ctc_align_long", "gam_ctc_align_long_gaps": "gam_test_ctc_align_long_gaps",
                         "gam_ctc_align_long_skips": "gam_test_ctc_align_long_skips"}[name]
            self._call(test_name, *args, int(cluster_ctas), plan)
            self.last_align_long_plan = (int(plan[0]), int(plan[1]))
        return outs

    def ctc_spot(self, log_probs: Tensor, enc_len: Tensor, keywords: Tensor, keyword_len: Tensor, threshold: float, max_det: int,
                 warps_per_cta: Optional[int] = None) -> Tuple[Tensor, ...]:
        """log_probs [B, T, V+1] f32 contiguous (ctc_log_probs, or stitched windows), enc_len [B], keywords [K, Umax] token ids,
        keyword_len [K] -> (start [B, K, max_det] i32, end [B, K, max_det] i32, score [B, K, max_det] f32, count [B, K] i32) on
        the device (gam_ctc_spot).  `warps_per_cta` forces the keyword warps per CTA (gam_test_ctc_spot)."""
        assert log_probs.is_cuda and log_probs.dtype == torch.float32 and log_probs.is_contiguous() and log_probs.dim() == 3
        if self.head_type != 1:
            raise RuntimeError("model has no CTC head")
        B, T, _ = log_probs.shape
        K, Umax = keywords.shape
        enc_len, keywords, keyword_len = (self._i32(t, self.device) for t in (enc_len, keywords, keyword_len))
        i32 = dict(dtype=torch.int32, device=self.device)
        outs = (torch.empty((B, K, max_det), **i32), torch.empty((B, K, max_det), **i32),
                torch.empty((B, K, max_det), dtype=torch.float32, device=self.device), torch.empty((B, K), **i32))
        args = [log_probs, enc_len, B, T, keywords, keyword_len, K, Umax, float(threshold), int(max_det), *outs]
        if warps_per_cta is None:
            self._call("gam_ctc_spot", *args)
        else:
            self._call("gam_test_ctc_spot", *args, int(warps_per_cta))
        return outs

    def spot_state(self, n: int, K: int, Umax: int) -> Tensor:
        """n x K fresh keyword-spotting records (gam_ctc_spot_state_init): uint8 [n, K, gam_ctc_spot_state_bytes(Umax)] on the
        device."""
        nbytes = int(self.lib.gam_ctc_spot_state_bytes(self.handle, int(Umax)))
        if nbytes < 0:
            raise ValueError(f"spot_state: no CTC head, or Umax={Umax} outside [1, 64]")
        state = torch.empty((n, K, nbytes), dtype=torch.uint8, device=self.device)
        self._call("gam_ctc_spot_state_init", state, n, K, int(Umax))
        return state

    def ctc_spot_resume(self, log_probs: Tensor, lo: Tensor, hi: Tensor, frame_base: Tensor, finish: Tensor, keywords: Tensor,
                        keyword_len: Tensor, threshold: float, state: Tensor, det: Tuple[Tensor, ...],
                        pending: Optional[Tuple[Tensor, ...]] = None) -> None:
        """Spot over local frames [lo[b], hi[b]) of log_probs [B, T, V+1] as stream frames frame_base[b] + t, continuing the
        records state [B, K, bytes] (spot_state) (gam_ctc_spot_resume).  lo / hi / frame_base / finish: device int32 [B].
        det = (start, end, score [B, K, max_det], count [B, K]) on the device: detections are appended at count.  `pending` =
        (start, end, score [B, K]) receives the pending detections."""
        assert log_probs.is_cuda and log_probs.dtype == torch.float32 and log_probs.is_contiguous() and log_probs.dim() == 3
        B, T, _ = log_probs.shape
        K, Umax = keywords.shape
        for t in (lo, hi, frame_base, finish, keywords, keyword_len):
            assert t.device == self.device and t.dtype == torch.int32 and t.is_contiguous()
        assert state.dtype == torch.uint8 and state.is_contiguous() and tuple(state.shape[:2]) == (B, K)
        assert all(t.is_contiguous() and t.shape[:2] == (B, K) for t in det)
        max_det = det[0].shape[2]
        pend = [None] * 3 if pending is None else pending
        self._call("gam_ctc_spot_resume", log_probs, B, T, lo, hi, frame_base, finish, keywords, keyword_len, K, Umax, float(threshold),
                   int(max_det), state, state.shape[2], *det, *pend)

    def ctc_bias(self, log_probs: Tensor, enc_len: Tensor, keywords: Tensor, keyword_len: Tensor, spotted: Tuple[Tensor, ...],
                 threshold: float, token_flags: Tensor, ids: Tensor, frames: Tensor, counts: Tensor,
                 token_logp: Optional[Tensor] = None, path_logp: Optional[Tensor] = None, frame_logp: Optional[Tensor] = None
                 ) -> Tuple[Tensor, ...]:
        """Hotwords (gam_ctc_bias): the detections `spotted` = ctc_spot(log_probs, enc_len, keywords, keyword_len, threshold,
        max_det) replace the greedy words they outscore in ids / frames [B, max_out], counts [B] (greedy).  -> (ids, frames
        [B, max_out] i32, counts [B] i32, source [B, max_out] i32, token_logp [B, max_out] f32 or None, path_logp [B] f32 or
        None); the scores are returned when token_logp / path_logp are given.  frame_logp (f64 [B, pitch], greedy_resume's
        per-frame sums) is adjusted in place."""
        assert log_probs.is_cuda and log_probs.dtype == torch.float32 and log_probs.is_contiguous() and log_probs.dim() == 3
        if self.head_type != 1:
            raise RuntimeError("model has no CTC head")
        B, T, _ = log_probs.shape
        K, Umax = keywords.shape
        max_out = ids.shape[1]
        max_det = spotted[0].shape[2]
        ws = self._ws(self._ws_align, ("bias", B, T, K, max_det), "gam_ctc_bias_workspace_bytes", B, T, K, max_det,
                      what=f"ctc_bias: bad sizes B={B}, T={T}, K={K}, max_det={max_det}")
        enc_len, keywords, keyword_len, ids, frames, counts = (self._i32(t, self.device)
                                                               for t in (enc_len, keywords, keyword_len, ids, frames, counts))
        flags = token_flags.to(device=self.device, dtype=torch.uint8).contiguous()
        for t in spotted:
            assert t.is_cuda and t.is_contiguous()
        for t in (token_logp, path_logp):
            assert t is None or (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous())
        assert frame_logp is None or (frame_logp.dtype == torch.float64 and frame_logp.is_contiguous() and frame_logp.dim() == 2)
        i32 = dict(dtype=torch.int32, device=self.device)
        out = [torch.empty((B, max_out), **i32), torch.empty((B, max_out), **i32), torch.empty((B,), **i32),
               torch.empty((B, max_out), **i32),
               None if token_logp is None else torch.empty((B, max_out), dtype=torch.float32, device=self.device),
               None if path_logp is None else torch.empty((B,), dtype=torch.float32, device=self.device)]
        self._call("gam_ctc_bias", log_probs, enc_len, B, T, keywords, keyword_len, K, Umax, *spotted, max_det, float(threshold), flags,
                   flags.numel(), ids, frames, counts, max_out, token_logp, path_logp, frame_logp,
                   0 if frame_logp is None else frame_logp.shape[1], ws, ws.numel(), *out)
        return tuple(out)

    def ctc_bias_resume(self, log_probs: Tensor, hi: Tensor, frame_base: Tensor, finish: Tensor, keywords: Tensor,
                        keyword_len: Tensor, threshold: float, state: Tensor, det: Tuple[Tensor, ...], token_flags: Tensor,
                        ids: Tensor, frames: Tensor, counts: Tensor, left_boundary: Tensor, token_logp: Optional[Tensor] = None,
                        frame_logp: Optional[Tensor] = None) -> Tuple[Tensor, ...]:
        """Resumable hotwords (gam_ctc_bias_resume) over held stream frames frame_base[b] + t, t < hi[b], of log_probs
        [B, T, V+1]: `state` the spot records [B, K, bytes] after this step's ctc_spot_resume, det = (start, end, score
        [B, K, max_det], count [B, K]) the undecided detections in stream frames, ids / frames [B, max_out] and counts [B] the
        held greedy tokens (frames in stream frames).  hi / frame_base / finish / left_boundary: device int32 [B].  -> (ids,
        frames [B, max_out] i32, counts [B] i32, source [B, max_out] i32, token_logp [B, max_out] f32 or None, released_until
        [B] i32, carry_start, carry_end [B, K, max_det] i32, carry_score [B, K, max_det] f32, carry_count [B, K] i32);
        frame_logp (f64 [B, pitch], the held frames' per-frame sums) is adjusted in place."""
        assert log_probs.is_cuda and log_probs.dtype == torch.float32 and log_probs.is_contiguous() and log_probs.dim() == 3
        if self.head_type != 1:
            raise RuntimeError("model has no CTC head")
        B, T, _ = log_probs.shape
        K, Umax = keywords.shape
        max_out = ids.shape[1]
        max_det = det[0].shape[2]
        ws = self._ws(self._ws_align, ("bias", B, T, K, max_det), "gam_ctc_bias_resume_workspace_bytes", B, T, K, max_det,
                      what=f"ctc_bias_resume: bad sizes B={B}, T={T}, K={K}, max_det={max_det}")
        hi, frame_base, finish, left_boundary, keywords, keyword_len, ids, frames, counts = (
            self._i32(t, self.device) for t in (hi, frame_base, finish, left_boundary, keywords, keyword_len, ids, frames, counts))
        flags = token_flags.to(device=self.device, dtype=torch.uint8).contiguous()
        assert state.dtype == torch.uint8 and state.is_contiguous() and tuple(state.shape[:2]) == (B, K)
        assert all(t.is_cuda and t.is_contiguous() and t.shape[:2] == (B, K) for t in det)
        assert token_logp is None or (token_logp.is_cuda and token_logp.dtype == torch.float32 and token_logp.is_contiguous())
        assert frame_logp is None or (frame_logp.dtype == torch.float64 and frame_logp.is_contiguous() and frame_logp.dim() == 2)
        i32 = dict(dtype=torch.int32, device=self.device)
        out = [torch.empty((B, max_out), **i32), torch.empty((B, max_out), **i32), torch.empty((B,), **i32),
               torch.empty((B, max_out), **i32),
               None if token_logp is None else torch.empty((B, max_out), dtype=torch.float32, device=self.device),
               torch.empty((B,), **i32), torch.empty((B, K, max_det), **i32), torch.empty((B, K, max_det), **i32),
               torch.empty((B, K, max_det), dtype=torch.float32, device=self.device), torch.empty((B, K), **i32)]
        self._call("gam_ctc_bias_resume", log_probs, B, T, hi, frame_base, finish, keywords, keyword_len, K, Umax, state,
                   state.shape[2], *det, max_det, float(threshold), flags, flags.numel(), ids, frames, counts, left_boundary,
                   max_out, token_logp, frame_logp, 0 if frame_logp is None else frame_logp.shape[1], ws, ws.numel(), *out)
        return tuple(out)

    def rnnt_align_scores(self, enc: Tensor, dec: Tensor, targets: Tensor) -> Tuple[Tensor, Tensor]:
        """enc [B, T, d], dec [B, U+1, pred_hidden] f32 contiguous, targets [B, U] -> (blank, label) [B, T, U+1] f32: the
        entries of rnnt_joint's lattice that alignment reads (gam_rnnt_align_scores)."""
        assert enc.is_cuda and dec.is_cuda and enc.dtype == dec.dtype == torch.float32
        assert enc.is_contiguous() and dec.is_contiguous() and enc.dim() == dec.dim() == 3
        if self.head_type != 2:
            raise RuntimeError("model has no RNN-T head")
        B, T, _ = enc.shape
        U = targets.shape[1]
        if dec.shape[0] != B or dec.shape[1] != U + 1:
            raise ValueError(f"align scores: dec has shape {tuple(dec.shape)}, expected ({B}, {U + 1}, H)")
        ws = self._ws(self._ws_joint, (B, T, U + 1), "gam_rnnt_align_scores_workspace_bytes", B, T, U,
                      what=f"align scores: bad sizes B={B}, T={T}, U={U}")
        targets = self._i32(targets, self.device)
        blank = torch.empty((B, T, U + 1), dtype=torch.float32, device=self.device)
        label = torch.empty((B, T, U + 1), dtype=torch.float32, device=self.device)
        self._call("gam_rnnt_align_scores", enc, dec, targets, B, T, U, ws, ws.numel(), blank, label)
        return blank, label

    def rnnt_align(self, blank: Tensor, label: Tensor, enc_len: Tensor, target_len: Tensor) -> Tuple[Tensor, ...]:
        """blank / label [B, T, U+1] f32 contiguous, enc_len [B], target_len [B] -> the outputs of ctc_align (gam_rnnt_align)."""
        assert blank.is_cuda and label.is_cuda and blank.dtype == label.dtype == torch.float32
        assert blank.is_contiguous() and label.is_contiguous() and blank.dim() == 3 and blank.shape == label.shape
        if self.head_type != 2:
            raise RuntimeError("model has no RNN-T head")
        B, T, U1 = blank.shape
        U = U1 - 1
        ws = self._ws(self._ws_align, ("rnnt", B, T, U), "gam_rnnt_align_workspace_bytes", B, T, U,
                      what=f"rnnt_align: bad sizes B={B}, T={T}, U={U}")
        enc_len, target_len = self._i32(enc_len, self.device), self._i32(target_len, self.device)
        outs = self._align_outputs(B, U)
        self._call("gam_rnnt_align", blank, label, enc_len, target_len, B, T, U, ws, ws.numel(), *outs)
        return outs

    # ------------------------------------------------------------------ fused RNN-T loss (rnnt_loss.cu)
    def _loss_args(self, enc: Tensor, dec: Tensor, targets: Tensor, enc_len: Tensor, target_len: Tensor, what: str):
        assert enc.is_cuda and dec.is_cuda and enc.dtype == dec.dtype == torch.float32
        assert enc.is_contiguous() and dec.is_contiguous() and enc.dim() == dec.dim() == 3
        if self.head_type != 2:
            raise RuntimeError("model has no RNN-T head")
        B, T, _ = enc.shape
        U = targets.shape[1]
        if dec.shape[0] != B or dec.shape[1] != U + 1 or targets.shape[0] != B:
            raise ValueError(f"{what}: dec has shape {tuple(dec.shape)} and targets {tuple(targets.shape)}, expected ({B}, {U + 1}, H) "
                             f"and ({B}, U)")
        return B, T, U, self._i32(targets, self.device), self._i32(enc_len, self.device), self._i32(target_len, self.device)

    def rnnt_loss(self, enc: Tensor, dec: Tensor, targets: Tensor, enc_len: Tensor, target_len: Tensor) -> Tuple[Tensor, Tensor]:
        """enc [B, T, d], dec [B, U+1, pred_hidden] f32 contiguous, targets [B, U], enc_len [B], target_len [B] -> (loss [B] f32,
        saved [3, B, T, U+1] f32: the per-node lse, e_blank and e_label that rnnt_loss_backward reads) (gam_rnnt_loss)."""
        B, T, U, targets, enc_len, target_len = self._loss_args(enc, dec, targets, enc_len, target_len, "rnnt_loss")
        ws = self._ws(None, None, "gam_rnnt_loss_workspace_bytes", B, T, U,
                      what=f"rnnt_loss: unsupported sizes B={B}, T={T}, U={U} (limits: T <= the model's max_encoded_frames, "
                           f"U <= 4096 tokens, joint_hidden <= {_lib.RNNT_LOSS_MAX_JOINT_HIDDEN})")
        saved = self._empty(3, B, T, U + 1)
        loss = self._empty(B)
        self._call("gam_rnnt_loss", enc, dec, targets, enc_len, target_len, B, T, U, ws, ws.numel(), saved, loss)
        return loss, saved

    def rnnt_loss_backward(self, enc: Tensor, dec: Tensor, targets: Tensor, enc_len: Tensor, target_len: Tensor, saved: Tensor,
                           grad: Tensor, need_enc: bool, need_dec: bool, need_weights: bool):
        """-> (d_enc [B, T, d], d_dec [B, U+1, H], dW_enc, db_enc, dW_pred, db_pred, dW_out, db_out); None where not needed.
        grad: dL/dloss [B] f32 (gam_rnnt_loss_backward)."""
        B, T, U, targets, enc_len, target_len = self._loss_args(enc, dec, targets, enc_len, target_len, "rnnt_loss_backward")
        assert saved.is_contiguous() and tuple(saved.shape) == (3, B, T, U + 1)
        grad = grad.to(device=self.device, dtype=torch.float32).contiguous()
        d, H = enc.shape[2], dec.shape[2]
        J, V1 = self.gam_config.joint_hidden, self.num_classes
        outs = [self._empty(B, T, d) if need_enc else None, self._empty(B, U + 1, H) if need_dec else None]
        if need_weights:
            outs += [self._empty(J, d), self._empty(J), self._empty(J, H), self._empty(J), self._empty(V1, J), self._empty(V1)]
        else:
            outs += [None] * 6
        ws = self._ws(None, None, "gam_rnnt_loss_backward_workspace_bytes", B, T, U, what="rnnt_loss_backward: bad sizes")
        self._call("gam_rnnt_loss_backward", enc, dec, targets, enc_len, target_len, B, T, U, saved, grad, ws, ws.numel(), *outs)
        return tuple(outs)

    # ------------------------------------------------------------------ backward passes of the head calls (head_grads.cu)
    def _empty(self, *shape) -> Tensor:
        return torch.empty(shape, dtype=torch.float32, device=self.device)

    def rnnt_predict_train(self, x: Optional[Tensor], h: Optional[Tensor], c: Optional[Tensor], batch_size: int = 1
                           ) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
        """rnnt_predict (same bits) that also returns the cell state of every step, c_seq [U, B, H]."""
        B, U, H = self._predict_sizes(x, batch_size)
        for name, t in (("h", h), ("c", c)):
            if t is not None and (tuple(t.shape) != (B, H) or not t.is_contiguous()):
                raise ValueError(f"predict: state {name} has shape {tuple(t.shape)}, expected ({B}, {H})")
        g, h1, c1, c_seq = self._empty(B, U, H), self._empty(B, H), self._empty(B, H), self._empty(U, B, H)
        self._call("gam_rnnt_predict_train", x, h, c, B, U, g, h1, c1, c_seq)
        return g, h1, c1, c_seq

    def ctc_log_probs_backward(self, enc: Tensor, log_probs: Tensor, grad: Tensor, need_enc: bool, need_weights: bool):
        """-> (d_enc [B, T, d] or None, dW [V+1, d] or None, db [V+1] or None); every tensor f32 contiguous on the device."""
        B, T, d = enc.shape
        d_enc = self._empty(B, T, d) if need_enc else None
        dW, db = (self._empty(self.num_classes, d), self._empty(self.num_classes)) if need_weights else (None, None)
        ws = self._ws(None, None, "gam_ctc_log_probs_backward_workspace_bytes", B, T, what="ctc backward: bad sizes")
        self._call("gam_ctc_log_probs_backward", enc, B, T, log_probs, grad, ws, ws.numel(), d_enc, dW, db)
        return d_enc, dW, db

    def rnnt_joint_backward(self, enc: Tensor, dec: Tensor, log_probs: Tensor, grad: Tensor, need_enc: bool, need_dec: bool,
                            need_weights: bool):
        """-> (d_enc [B, T, d], d_dec [B, U, H], dW_enc, db_enc, dW_pred, db_pred, dW_out, db_out); None where not needed."""
        B, T, d = enc.shape
        U, H = dec.shape[1], dec.shape[2]
        J, V1 = self.gam_config.joint_hidden, self.num_classes
        outs = [self._empty(B, T, d) if need_enc else None, self._empty(B, U, H) if need_dec else None]
        if need_weights:
            outs += [self._empty(J, d), self._empty(J), self._empty(J, H), self._empty(J), self._empty(V1, J), self._empty(V1)]
        else:
            outs += [None] * 6
        ws = self._ws(None, None, "gam_rnnt_joint_backward_workspace_bytes", B, T, U, what="joint backward: bad sizes")
        self._call("gam_rnnt_joint_backward", enc, dec, B, T, U, log_probs, grad, ws, ws.numel(), *outs)
        return tuple(outs)

    def rnnt_predict_backward(self, x: Optional[Tensor], h: Optional[Tensor], c: Optional[Tensor], g: Tensor, c_seq: Tensor,
                              grad_g: Tensor, grad_h1: Optional[Tensor], grad_c1: Optional[Tensor], embed: Tensor, w_ih: Tensor,
                              w_hh: Tensor, need_state: bool, need_weights: bool):
        """BPTT through rnnt_predict_train -> (d_h0, d_c0 [B, H], d_embed [V+1, H], dW_ih, dW_hh [4H, H], d_bias [4H]); None
        where not needed.  embed / w_ih / w_hh: the module's weights, f32 contiguous on the device."""
        B, U, H = g.shape
        V1 = self.num_classes
        outs = [self._empty(B, H), self._empty(B, H)] if need_state else [None, None]
        outs += ([self._empty(V1, H), self._empty(4 * H, H), self._empty(4 * H, H), self._empty(4 * H)] if need_weights
                 else [None] * 4)
        ws = self._ws(None, None, "gam_rnnt_predict_backward_workspace_bytes", B, U, what="predict backward: bad sizes")
        self._call("gam_rnnt_predict_backward", x, h, c, B, U, g, c_seq, grad_g, grad_h1, grad_c1, embed, w_ih, w_hh, ws, ws.numel(),
                   *outs)
        return tuple(outs)

    def emo_head(self, enc_btd: Tensor, enc_len: Optional[Tensor]) -> Tuple[Tensor, Tensor, Tensor]:
        """enc [B, T, d] f32 contiguous, len [B] or None (all T frames) -> (pooled [B, d], logits [B, C], probs [B, C]) f32
        (gam_emo_head: GigaAMEmo's mean + head + softmax, gigaam/model.py:272-293).  Utterance b pools len[b] frames, except
        that a batch of ONE pools all T.  The workspace is cached per (B, T) like the decode workspace."""
        assert enc_btd.is_cuda and enc_btd.dtype == torch.float32 and enc_btd.is_contiguous() and enc_btd.dim() == 3
        if self.head_type != 3:
            raise RuntimeError("model has no emo head")
        B, T, _ = enc_btd.shape
        ws = self._ws(self._ws_emo, (B, T), "gam_emo_workspace_bytes", B, T, what=f"emo_head: bad sizes B={B}, T={T}")
        if enc_len is not None:
            enc_len = enc_len.to(device=self.device, dtype=torch.int32).contiguous()
        pooled = torch.empty((B, self.d_model), dtype=torch.float32, device=self.device)
        logits = torch.empty((B, self.num_classes), dtype=torch.float32, device=self.device)
        probs = torch.empty((B, self.num_classes), dtype=torch.float32, device=self.device)
        self._call("gam_emo_head", enc_btd, enc_len, B, T, ws, ws.numel(), pooled, logits, probs)
        return pooled, logits, probs

    def emo_frame_logits(self, enc_btd: Tensor, lo: Tensor, hi: Tensor, dst: Tensor, frame_logits: Tensor) -> Tensor:
        """gam_emo_frame_logits: enc [B, T, d] f32 contiguous; lo / hi / dst device i32 [B] -> row b's local frames [lo, hi)
        get their logits W f + b written to rows dst[b] + t - lo[b] of frame_logits (f32 [n_frames, C] on the device, filled in
        place and returned).  Rows outside [0, n_frames) are dropped."""
        assert enc_btd.is_cuda and enc_btd.dtype == torch.float32 and enc_btd.is_contiguous() and enc_btd.dim() == 3
        assert frame_logits.dtype == torch.float32 and frame_logits.is_contiguous() and frame_logits.shape[-1] == self.num_classes
        if self.head_type != 3:
            raise RuntimeError("model has no emo head")
        B, T, _ = enc_btd.shape
        self._call("gam_emo_frame_logits", enc_btd, B, T, lo, hi, dst, frame_logits, frame_logits.shape[0])
        return frame_logits

    def emo_spans(self, frame_logits: Tensor, start: Tensor, end: Tensor, logits: bool = True) -> Tuple[Optional[Tensor], Tensor]:
        """gam_emo_spans: frame_logits f32 [n_frames, C]; start / end device i32 [S] -> (logits [S, C], the mean of the frame
        logits over each span [start, end), or None without `logits`; probs [S, C], its softmax).  An empty span gives NaN."""
        assert frame_logits.dtype == torch.float32 and frame_logits.is_contiguous() and frame_logits.shape[-1] == self.num_classes
        if self.head_type != 3:
            raise RuntimeError("model has no emo head")
        S = start.numel()
        out_l = self._empty(S, self.num_classes) if logits else None
        probs = self._empty(S, self.num_classes)
        self._call("gam_emo_spans", frame_logits, frame_logits.shape[0], start, end, S, out_l, probs)
        return out_l, probs

    def group_words(self, ids: Tensor, frames: Tensor, counts: Tensor, token_flags: Tensor):
        """Device word grouping (gam_group_words): -> (word_start, word_end, word_first, word_ntok [B, max_out] i32, n_words [B] i32)."""
        B, max_out = ids.shape
        flags = token_flags.to(device=self.device, dtype=torch.uint8).contiguous()
        outs = [torch.empty((B, max_out), dtype=torch.int32, device=self.device) for _ in range(4)]
        n_words = torch.empty((B,), dtype=torch.int32, device=self.device)
        self._call("gam_group_words", ids, frames, counts, B, max_out, flags, flags.numel(), max_out, *outs, n_words)
        return (*outs, n_words)

    def profile_begin(self) -> None:
        _lib.check(self.lib, self.handle, self.lib.gam_profile_begin(self.handle), "gam_profile_begin")

    def profile_end(self) -> Dict[str, Tuple[float, int]]:
        """{kernel class: (total ms, launches)} measured with CUDA events since profile_begin()."""
        n = int(self.lib.gam_profile_class_count())
        ms = (C.c_double * n)()
        cnt = (C.c_int64 * n)()
        _lib.check(self.lib, self.handle, self.lib.gam_profile_end(self.handle, ms, cnt, n), "gam_profile_end")
        return {self.lib.gam_profile_class_name(i).decode(): (float(ms[i]), int(cnt[i])) for i in range(n) if cnt[i] > 0}

    def launch_count(self) -> int:
        return int(self.lib.gam_launch_count(self.handle))

    def __del__(self):
        try:
            if getattr(self, "handle", None) and self.handle.value:
                self.lib.gam_destroy(self.handle)
                self.handle = C.c_void_p()
        except Exception:
            pass
