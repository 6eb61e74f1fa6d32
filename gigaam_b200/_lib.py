"""ctypes binding of libgigaam_b200.so, with the prototypes parsed from include/gigaam_b200.h.  There is no CPU fallback:
if the library is missing it is built with nvcc, and if that is impossible the import of any compute class fails loudly."""
from __future__ import annotations

import ctypes as C
import os
import re
from pathlib import Path
from typing import Any, Dict, List, Optional, Tuple

_PKG = Path(__file__).resolve().parent
_HEADER_PATH = _PKG.parent / "include" / "gigaam_b200.h"
_LIB: Optional[C.CDLL] = None


class GamConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "sample_rate", "n_mels", "n_fft", "win_length", "hop_length", "center",
        "feat_in", "n_layers", "d_model", "n_heads", "d_ff",
        "subsampling", "subs_kernel_size", "conv_kernel_size", "conv_norm", "self_attention", "pos_emb_max_len",
        "head", "num_classes", "pred_hidden", "joint_hidden", "max_symbols", "max_encoded_frames")]


LAYER_FIELDS = (
    "ln_ff1_g", "ln_ff1_b", "ff1_w1", "ff1_b1", "ff1_w2", "ff1_b2",
    "ln_att_g", "ln_att_b", "w_qk", "b_qk", "w_v", "b_v", "w_o", "b_o",
    "ln_conv_g", "ln_conv_b", "pw1_w", "pw1_b", "dw_w", "dw_b", "cn_g", "cn_b", "pw2_w", "pw2_b",
    "ln_ff2_g", "ln_ff2_b", "ff2_w1", "ff2_b1", "ff2_w2", "ff2_b2", "ln_out_g", "ln_out_b",
    "w_qkv_rel", "b_qkv_rel", "pos_proj")


class GamLayerWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in LAYER_FIELDS]


WEIGHT_FIELDS_HEAD = ("window", "dft_cos", "dft_sin", "mel_fb", "sub1_w", "sub1_b", "sub2_w", "sub2_b",
                      "sub_out_w", "sub_out_b", "rope_cos", "rope_sin")
WEIGHT_FIELDS_TAIL = ("ctc_w", "ctc_b", "rnnt_enc_w", "rnnt_enc_b", "rnnt_emb_gates", "rnnt_whh_t", "rnnt_wp_t",
                      "rnnt_bp", "rnnt_wo", "rnnt_bo", "c1d_w1", "c1d_b1", "c1d_w2", "c1d_b2", "dft_w", "mel_lo", "mel_hi",
                      "emo_w", "emo_b")


class GamWeights(C.Structure):
    _fields_ = ([(n, C.c_void_p) for n in WEIGHT_FIELDS_HEAD] + [("layers", C.POINTER(GamLayerWeights))]
                + [(n, C.c_void_p) for n in WEIGHT_FIELDS_TAIL])


_SCALARS = {"int": C.c_int32, "int32_t": C.c_int32, "int64_t": C.c_int64, "float": C.c_float}
_DECL = re.compile(r"^[ \t]*((?:const[ \t]+)?\w+[ \t]*\**)[ \t]*(gam_\w+)\s*\(([^()]*)\)\s*;", re.M)


def _ctype(decl: str, what: str, ret: bool = False):
    """ctypes type of one C type (a return type, or a parameter with its name): every pointer is c_void_p, except a
    `const char*` return (c_char_p); `void` is None."""
    if "*" in decl:
        return C.c_char_p if ret and decl.replace(" ", "") == "constchar*" else C.c_void_p
    words = [w for w in decl.split() if w != "const"]
    if words[:1] == ["void"] and len(words) == 1 and ret:
        return None
    if len(words) != (1 if ret else 2) or words[0] not in _SCALARS:
        raise ValueError(f"{what}: no ctypes mapping for {decl.strip()!r}")
    return _SCALARS[words[0]]


def parse_prototypes(text: str) -> Dict[str, Tuple[Any, List[Any]]]:
    """{name: (restype, argtypes)} of every `gam_*` function declared in the header text.  A type outside the table of
    _ctype, or a declaration this parser cannot read, raises: a header change must not bind silently wrong."""
    code = re.sub(r"//[^\n]*", "", re.sub(r"/\*.*?\*/", "", text, flags=re.S))
    protos = {}
    for ret, name, params in _DECL.findall(code):
        params = params.strip()
        args = [] if params == "void" else [_ctype(p, name) for p in params.split(",")]
        protos[name] = (_ctype(ret, name, ret=True), args)
    unread = set(re.findall(r"\b(gam_\w+)\s*\(", code)) - set(protos)
    if unread:
        raise ValueError(f"declarations not understood: {sorted(unread)}")
    return protos


_HEADER = _HEADER_PATH.read_text()
PROTOTYPES = parse_prototypes(_HEADER)
EXPORTS = tuple(PROTOTYPES)
# the default longest T' (GamConfig.max_encoded_frames = 0)
REL_POS_MAX_T = int(re.search(r"#define\s+GAM_REL_POS_MAX_T\s+(\d+)", _HEADER).group(1))
# the widest head d_k each attention kernel runs (gam_create refuses wider ones)
ROTARY_MAX_DK = int(re.search(r"#define\s+GAM_ROTARY_MAX_DK\s+(\d+)", _HEADER).group(1))
REL_POS_MAX_DK = int(re.search(r"#define\s+GAM_REL_POS_MAX_DK\s+(\d+)", _HEADER).group(1))
# the widest joint_hidden the fused RNN-T loss runs, and the widest pred_hidden the prediction network trains at
RNNT_LOSS_MAX_JOINT_HIDDEN = int(re.search(r"#define\s+GAM_RNNT_LOSS_MAX_JOINT_HIDDEN\s+(\d+)", _HEADER).group(1))
PREDICT_BACKWARD_MAX_HIDDEN = int(re.search(r"#define\s+GAM_PREDICT_BACKWARD_MAX_HIDDEN\s+(\d+)", _HEADER).group(1))


def lib_path() -> Path:
    return Path(os.environ.get("GIGAAM_B200_LIB", _PKG / "libgigaam_b200.so"))


def load() -> C.CDLL:
    """Load (building first if needed) the shared library and declare the prototypes of the header."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not path.exists():
        from ._build import build_library
        path = build_library()
    lib = C.CDLL(str(path))
    for name, (restype, argtypes) in PROTOTYPES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    _LIB = lib
    return lib


class GamError(RuntimeError):
    pass


def check(lib: C.CDLL, handle, rc: int, what: str) -> None:
    if rc != 0:
        msg = lib.gam_last_error(handle)
        raise GamError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")
