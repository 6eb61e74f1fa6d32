"""ctypes binding of libgigaam_b200.so (include/gigaam_b200.h).  There is no CPU fallback: if the library is
missing it is built with nvcc, and if that is impossible the import of any compute class fails loudly."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path
from typing import Optional

_PKG = Path(__file__).resolve().parent
_LIB: Optional[C.CDLL] = None

c_f32p = C.c_void_p
c_vp = C.c_void_p


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

REL_POS_MAX_T = 768   # GAM_REL_POS_MAX_T in include/gigaam_b200.h: the default longest T' (GamConfig.max_encoded_frames = 0)


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


EXPORTS = ("gam_create", "gam_destroy", "gam_last_error", "gam_version", "gam_logmel_frames", "gam_encoded_frames",
           "gam_workspace_bytes", "gam_logmel", "gam_encode", "gam_ctc_greedy", "gam_rnnt_greedy", "gam_test_gemm",
           "gam_test_attention", "gam_launch_count", "gam_profile_begin", "gam_profile_end", "gam_profile_class_count",
           "gam_profile_class_name", "gam_logmel_workspace_bytes", "gam_logmel_tc", "gam_test_attention_relpos",
           "gam_decode_workspace_bytes", "gam_group_words", "gam_comm_unique_id", "gam_comm_init",
           "gam_comm_nccl_version", "gam_gather_hyps", "gam_test_attention_varlen", "gam_ctc_log_probs",
           "gam_rnnt_joint_workspace_bytes", "gam_rnnt_joint", "gam_rnnt_predict", "gam_test_gemm_conv",
           "gam_test_layernorm", "gam_test_ln_rope", "gam_test_ln_out_ln", "gam_test_unpack_rows", "gam_test_dwconv",
           "gam_test_pack_plan", "gam_test_subsample_conv1", "gam_test_mel_to_tmajor", "gam_emo_workspace_bytes",
           "gam_emo_head", "gam_test_frames_split", "gam_test_mel_log", "gam_test_rnnt_greedy",
           "gam_rnnt_predict_train", "gam_ctc_log_probs_backward_workspace_bytes", "gam_ctc_log_probs_backward",
           "gam_rnnt_joint_backward_workspace_bytes", "gam_rnnt_joint_backward", "gam_rnnt_predict_backward_workspace_bytes",
           "gam_rnnt_predict_backward", "gam_test_gemm_used_slots", "gam_decode_scored_workspace_bytes",
           "gam_ctc_greedy_scored", "gam_rnnt_greedy_scored", "gam_test_rnnt_greedy_scored", "gam_ctc_align_workspace_bytes",
           "gam_ctc_align", "gam_rnnt_align_scores_workspace_bytes", "gam_rnnt_align_scores", "gam_rnnt_align_workspace_bytes",
           "gam_rnnt_align", "gam_ctc_align_long_workspace_bytes", "gam_ctc_align_long", "gam_test_ctc_align_long",
           "gam_decode_state_bytes", "gam_decode_state_init", "gam_decode_resume_workspace_bytes", "gam_ctc_greedy_resume",
           "gam_rnnt_greedy_resume", "gam_ctc_spot", "gam_test_ctc_spot", "gam_ctc_bias_workspace_bytes", "gam_ctc_bias",
           "gam_ctc_align_long_gaps_workspace_bytes", "gam_ctc_align_long_gaps", "gam_test_ctc_align_long_gaps",
           "gam_ctc_spot_state_bytes", "gam_ctc_spot_state_init", "gam_ctc_spot_resume",
           "gam_ctc_align_long_skips_workspace_bytes", "gam_ctc_align_long_skips", "gam_test_ctc_align_long_skips",
           "gam_rnnt_loss_saved_bytes", "gam_rnnt_loss_workspace_bytes", "gam_rnnt_loss", "gam_rnnt_loss_backward_workspace_bytes",
           "gam_rnnt_loss_backward")


def lib_path() -> Path:
    return Path(os.environ.get("GIGAAM_B200_LIB", _PKG / "libgigaam_b200.so"))


def load() -> C.CDLL:
    """Load (building first if needed) the shared library and declare the prototypes."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not path.exists():
        from ._build import build_library
        path = build_library()
    lib = C.CDLL(str(path))
    H = C.c_void_p
    i32, i64 = C.c_int32, C.c_int64
    lib.gam_create.argtypes = [C.POINTER(GamConfig), C.POINTER(GamWeights), C.c_int, C.POINTER(H)]
    lib.gam_create.restype = C.c_int
    lib.gam_destroy.argtypes = [H]
    lib.gam_destroy.restype = None
    lib.gam_last_error.argtypes = [H]
    lib.gam_last_error.restype = C.c_char_p
    lib.gam_version.restype = C.c_int
    lib.gam_launch_count.argtypes = [H]
    lib.gam_launch_count.restype = i64
    lib.gam_logmel_frames.argtypes = [H, i64]
    lib.gam_logmel_frames.restype = i64
    lib.gam_encoded_frames.argtypes = [H, i64]
    lib.gam_encoded_frames.restype = i64
    lib.gam_workspace_bytes.argtypes = [H, i32, i64]
    lib.gam_workspace_bytes.restype = i64
    lib.gam_decode_workspace_bytes.argtypes = [H, i32, i32]
    lib.gam_decode_workspace_bytes.restype = i64
    lib.gam_decode_scored_workspace_bytes.argtypes = [H, i32, i32]
    lib.gam_decode_scored_workspace_bytes.restype = i64
    lib.gam_comm_unique_id.argtypes = [c_vp]
    lib.gam_comm_unique_id.restype = C.c_int
    lib.gam_comm_init.argtypes = [H, c_vp, i32, i32]
    lib.gam_comm_init.restype = C.c_int
    lib.gam_comm_nccl_version.restype = i32
    lib.gam_gather_hyps.argtypes = [H, c_vp, i64, c_vp, c_vp]
    lib.gam_gather_hyps.restype = C.c_int
    lib.gam_group_words.argtypes = [H, c_vp, c_vp, c_vp, i32, i32, c_vp, i32, i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    lib.gam_group_words.restype = C.c_int
    lib.gam_logmel.argtypes = [H, c_vp, i32, i64, c_vp, c_vp]
    lib.gam_logmel.restype = C.c_int
    lib.gam_encode.argtypes = [H, c_vp, c_vp, i32, i64, c_vp, i64, c_vp, c_vp, i32, c_vp]
    lib.gam_encode.restype = C.c_int
    for fn in (lib.gam_ctc_greedy, lib.gam_rnnt_greedy):
        fn.argtypes = [H, c_vp, c_vp, i32, i32, c_vp, i64, c_vp, c_vp, c_vp, i32, c_vp]
        fn.restype = C.c_int
    for fn in (lib.gam_ctc_greedy_scored, lib.gam_rnnt_greedy_scored):
        fn.argtypes = [H, c_vp, c_vp, i32, i32, c_vp, i64, c_vp, c_vp, c_vp, i32, c_vp, c_vp, c_vp, c_vp]
        fn.restype = C.c_int
    lib.gam_decode_state_bytes.argtypes = [H]
    lib.gam_decode_state_bytes.restype = i64
    lib.gam_decode_state_init.argtypes = [H, c_vp, i32, c_vp]
    lib.gam_decode_state_init.restype = C.c_int
    lib.gam_decode_resume_workspace_bytes.argtypes = [H, i32, i32]
    lib.gam_decode_resume_workspace_bytes.restype = i64
    for fn in (lib.gam_ctc_greedy_resume, lib.gam_rnnt_greedy_resume):
        fn.argtypes = [H, c_vp, i32, i32, c_vp, c_vp, c_vp, c_vp, c_vp, i64, c_vp, c_vp, c_vp, i32] + [c_vp] * 5 + [i64, c_vp]
        fn.restype = C.c_int
    lib.gam_ctc_log_probs.argtypes = [H, c_vp, i32, i32, c_vp, c_vp]
    lib.gam_ctc_log_probs.restype = C.c_int
    lib.gam_rnnt_joint_workspace_bytes.argtypes = [H, i32, i32, i32]
    lib.gam_rnnt_joint_workspace_bytes.restype = i64
    lib.gam_rnnt_joint.argtypes = [H, c_vp, c_vp, i32, i32, i32, c_vp, i64, c_vp, c_vp]
    lib.gam_rnnt_joint.restype = C.c_int
    lib.gam_rnnt_predict.argtypes = [H, c_vp, c_vp, c_vp, i32, i32, c_vp, c_vp, c_vp, c_vp]
    lib.gam_rnnt_predict.restype = C.c_int
    lib.gam_rnnt_predict_train.argtypes = [H, c_vp, c_vp, c_vp, i32, i32, c_vp, c_vp, c_vp, c_vp, c_vp]
    lib.gam_ctc_log_probs_backward_workspace_bytes.argtypes = [H, i32, i32]
    lib.gam_ctc_log_probs_backward.argtypes = [H, c_vp, i32, i32, c_vp, c_vp, c_vp, i64, c_vp, c_vp, c_vp, c_vp]
    lib.gam_rnnt_joint_backward_workspace_bytes.argtypes = [H, i32, i32, i32]
    lib.gam_rnnt_joint_backward.argtypes = [H, c_vp, c_vp, i32, i32, i32, c_vp, c_vp, c_vp, i64] + [c_vp] * 9
    lib.gam_rnnt_predict_backward_workspace_bytes.argtypes = [H, i32, i32]
    lib.gam_rnnt_predict_backward.argtypes = [H, c_vp, c_vp, c_vp, i32, i32] + [c_vp] * 8 + [c_vp, i64] + [c_vp] * 7
    for fn in (lib.gam_ctc_log_probs_backward_workspace_bytes, lib.gam_rnnt_joint_backward_workspace_bytes,
               lib.gam_rnnt_predict_backward_workspace_bytes):
        fn.restype = i64
    for fn in (lib.gam_rnnt_predict_train, lib.gam_ctc_log_probs_backward, lib.gam_rnnt_joint_backward, lib.gam_rnnt_predict_backward):
        fn.restype = C.c_int
    for fn in (lib.gam_ctc_align_workspace_bytes, lib.gam_rnnt_align_scores_workspace_bytes, lib.gam_rnnt_align_workspace_bytes,
               lib.gam_ctc_align_long_workspace_bytes, lib.gam_ctc_align_long_gaps_workspace_bytes,
               lib.gam_ctc_align_long_skips_workspace_bytes):
        fn.argtypes = [H, i32, i32, i32]
        fn.restype = i64
    lib.gam_ctc_align.argtypes = [H, c_vp, c_vp, c_vp, c_vp, i32, i32, i32, c_vp, i64] + [c_vp] * 6
    lib.gam_rnnt_align_scores.argtypes = [H, c_vp, c_vp, c_vp, i32, i32, i32, c_vp, i64, c_vp, c_vp, c_vp]
    lib.gam_rnnt_align.argtypes = [H, c_vp, c_vp, c_vp, c_vp, i32, i32, i32, c_vp, i64] + [c_vp] * 6
    lib.gam_ctc_align_long.argtypes = lib.gam_ctc_align.argtypes
    lib.gam_test_ctc_align_long.argtypes = [H, c_vp, c_vp, c_vp, c_vp, i32, i32, i32, c_vp, i64] + [c_vp] * 5 + [i32, c_vp, c_vp]
    lib.gam_ctc_align_long_gaps.argtypes = [H, c_vp, c_vp, c_vp, c_vp, c_vp, i32, i32, i32, C.c_float, c_vp, i64] + [c_vp] * 9
    lib.gam_test_ctc_align_long_gaps.argtypes = lib.gam_ctc_align_long_gaps.argtypes[:-1] + [i32, c_vp, c_vp]
    lib.gam_ctc_align_long_skips.argtypes = ([H, c_vp, c_vp, c_vp, c_vp, c_vp, i32, i32, i32, C.c_float, C.c_float, c_vp, i64]
                                             + [c_vp] * 11)
    lib.gam_test_ctc_align_long_skips.argtypes = lib.gam_ctc_align_long_skips.argtypes[:-1] + [i32, c_vp, c_vp]
    for fn in (lib.gam_ctc_align, lib.gam_rnnt_align_scores, lib.gam_rnnt_align, lib.gam_ctc_align_long, lib.gam_test_ctc_align_long,
               lib.gam_ctc_align_long_gaps, lib.gam_test_ctc_align_long_gaps, lib.gam_ctc_align_long_skips,
               lib.gam_test_ctc_align_long_skips):
        fn.restype = C.c_int
    for fn in (lib.gam_rnnt_loss_saved_bytes, lib.gam_rnnt_loss_workspace_bytes, lib.gam_rnnt_loss_backward_workspace_bytes):
        fn.argtypes = [H, i32, i32, i32]
        fn.restype = i64
    lib.gam_rnnt_loss.argtypes = [H] + [c_vp] * 5 + [i32, i32, i32, c_vp, i64, c_vp, c_vp, c_vp]
    lib.gam_rnnt_loss_backward.argtypes = [H] + [c_vp] * 5 + [i32, i32, i32, c_vp, c_vp, c_vp, i64] + [c_vp] * 9
    lib.gam_rnnt_loss.restype = lib.gam_rnnt_loss_backward.restype = C.c_int
    lib.gam_ctc_spot.argtypes = [H, c_vp, c_vp, i32, i32, c_vp, c_vp, i32, i32, C.c_float, i32] + [c_vp] * 5
    lib.gam_test_ctc_spot.argtypes = [H, c_vp, c_vp, i32, i32, c_vp, c_vp, i32, i32, C.c_float, i32] + [c_vp] * 4 + [i32, c_vp]
    lib.gam_ctc_spot_state_bytes.argtypes = [H, i32]
    lib.gam_ctc_spot_state_bytes.restype = i64
    lib.gam_ctc_spot_state_init.argtypes = [H, c_vp, i32, i32, i32, c_vp]
    lib.gam_ctc_spot_resume.argtypes = ([H, c_vp, i32, i32] + [c_vp] * 6 + [i32, i32, C.c_float, i32, c_vp, i64] + [c_vp] * 7
                                        + [c_vp])
    for fn in (lib.gam_ctc_spot, lib.gam_test_ctc_spot, lib.gam_ctc_spot_state_init, lib.gam_ctc_spot_resume):
        fn.restype = C.c_int
    lib.gam_ctc_bias_workspace_bytes.argtypes = [H, i32, i32, i32, i32]
    lib.gam_ctc_bias_workspace_bytes.restype = i64
    lib.gam_ctc_bias.argtypes = ([H, c_vp, c_vp, i32, i32, c_vp, c_vp, i32, i32] + [c_vp] * 4 + [i32, C.c_float, c_vp, i32] + [c_vp] * 3
                                 + [i32] + [c_vp] * 3 + [i64, c_vp, i64] + [c_vp] * 7)
    lib.gam_ctc_bias.restype = C.c_int
    lib.gam_emo_workspace_bytes.argtypes = [H, i32, i32]
    lib.gam_emo_workspace_bytes.restype = i64
    lib.gam_emo_head.argtypes = [H, c_vp, c_vp, i32, i32, c_vp, i64, c_vp, c_vp, c_vp, c_vp]
    lib.gam_emo_head.restype = C.c_int
    lib.gam_test_gemm.argtypes = [H, i32, c_vp, c_vp, i32, c_vp, c_vp, c_vp, c_vp, i32, i32, i32, i32, i32, C.c_float, i32, c_vp,
                                  c_vp]
    lib.gam_test_gemm_used_slots.argtypes = [H]
    lib.gam_test_gemm_used_slots.restype = C.c_int
    lib.gam_test_gemm_conv.argtypes = [H, i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, i32, i32, i32, i32, i32, i32, i32, i32, c_vp]
    lib.gam_test_layernorm.argtypes = [H, c_vp, c_vp, c_vp, c_vp, i32, c_vp, i32, c_vp]
    lib.gam_test_ln_rope.argtypes = [H, c_vp, c_vp, c_vp, c_vp, c_vp, i32, i32, c_vp, c_vp, i32, c_vp, c_vp, i32, i32, c_vp]
    lib.gam_test_ln_out_ln.argtypes = [H, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, i32, c_vp, i32, c_vp]
    lib.gam_test_unpack_rows.argtypes = [H, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, i32, i32, i32, i32, c_vp]
    lib.gam_test_dwconv.argtypes = [H, i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, i32, i32, i32, i32,
                                    c_vp]
    lib.gam_test_pack_plan.argtypes = [H, c_vp, i32, i32, i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    lib.gam_test_subsample_conv1.argtypes = [H, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, i32, i32, i64, i32, c_vp]
    lib.gam_test_mel_to_tmajor.argtypes = [H, c_vp, c_vp, c_vp, i32, i32, i64, c_vp]
    lib.gam_test_frames_split.argtypes = [H, c_vp, i32, i64, c_vp, c_vp, c_vp]
    lib.gam_test_mel_log.argtypes = [H, c_vp, c_vp, i32, i32, i32, c_vp, c_vp, c_vp, i32, c_vp, c_vp]
    lib.gam_test_rnnt_greedy.argtypes = [H, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, i32, i32, i32, i32, i32, c_vp, c_vp, c_vp,
                                         c_vp, c_vp]
    lib.gam_test_rnnt_greedy_scored.argtypes = [H, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, i32, i32, i32, i32, i32, c_vp, c_vp,
                                                c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    lib.gam_test_rnnt_greedy_scored.restype = C.c_int
    for fn in (lib.gam_test_gemm, lib.gam_test_gemm_conv, lib.gam_test_layernorm, lib.gam_test_ln_rope, lib.gam_test_ln_out_ln,
               lib.gam_test_unpack_rows, lib.gam_test_dwconv, lib.gam_test_pack_plan, lib.gam_test_subsample_conv1,
               lib.gam_test_mel_to_tmajor, lib.gam_test_frames_split, lib.gam_test_mel_log, lib.gam_test_rnnt_greedy):
        fn.restype = C.c_int
    lib.gam_test_attention.argtypes = [H, c_vp, c_vp, c_vp, i32, i32, c_vp]
    lib.gam_test_attention.restype = C.c_int
    lib.gam_test_attention_relpos.argtypes = [H, c_vp, c_vp, c_vp, c_vp, i32, i32, c_vp]
    lib.gam_test_attention_relpos.restype = C.c_int
    lib.gam_test_attention_varlen.argtypes = [H, c_vp, c_vp, c_vp, c_vp, c_vp, i32, i32, i32, c_vp]
    lib.gam_test_attention_varlen.restype = C.c_int
    lib.gam_logmel_workspace_bytes.argtypes = [H, i32, i64]
    lib.gam_logmel_workspace_bytes.restype = i64
    lib.gam_logmel_tc.argtypes = [H, c_vp, i32, i64, c_vp, c_vp, i64, c_vp]
    lib.gam_logmel_tc.restype = C.c_int
    lib.gam_profile_begin.argtypes = [H]
    lib.gam_profile_begin.restype = C.c_int
    lib.gam_profile_end.argtypes = [H, C.POINTER(C.c_double), C.POINTER(C.c_int64), i32]
    lib.gam_profile_end.restype = C.c_int
    lib.gam_profile_class_count.restype = C.c_int
    lib.gam_profile_class_name.argtypes = [i32]
    lib.gam_profile_class_name.restype = C.c_char_p
    _LIB = lib
    return lib


class GamError(RuntimeError):
    pass


def check(lib: C.CDLL, handle, rc: int, what: str) -> None:
    if rc != 0:
        msg = lib.gam_last_error(handle)
        raise GamError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")
