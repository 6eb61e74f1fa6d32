"""gigaam_b200 -- H100-native drop-in for the GigaAM inference hot path
(log-mel -> Conformer encoder -> CTC / RNN-T greedy decode) behind the reference's Python surface.

    import gigaam_b200 as gigaam
    model = gigaam.load_model("v2_ctc")            # same signature as gigaam.load_model (gigaam/__init__.py:110-116)
    model.transcribe("example.wav")                # -> TranscriptionResult
    gigaam.load_model("emo").get_probs("example.wav")  # -> {"angry": p, "sad": p, "neutral": p, "positive": p}
    enc, enc_len = model(wav, lengths)              # batched forward
    model.decoding.decode(model.head, enc, enc_len) # -> [(text, ids, frames)]
"""
from __future__ import annotations

import hashlib
import logging
import os
from typing import Dict, Optional, Union

import torch

from .engine import check_attention_heads, max_encoded_frames_config
from .model import GigaAM, GigaAMASR, GigaAMEmo, check_emo_head
from .preprocess import load_audio, read_audio
from .synthetic import synthetic_audio, synthetic_checkpoint
from .streaming import EmotionStreamServer, StreamServer
from .types import (Alignment, Detection, EmotionSpan, EmotionStreamUpdate, EmotionTimeline, LongformAlignment,
                    LongformTranscriptionResult, Segment, StreamResult, StreamUpdate, TranscriptionResult, Word)

__all__ = ["GigaAM", "GigaAMASR", "GigaAMEmo", "load_audio", "read_audio", "load_model", "synthetic_checkpoint", "synthetic_audio",
           "TranscriptionResult", "Word", "Segment", "LongformTranscriptionResult", "Alignment",
           "LongformAlignment", "Detection", "StreamServer", "StreamUpdate", "StreamResult", "EmotionSpan", "EmotionTimeline",
           "EmotionStreamServer", "EmotionStreamUpdate"]

_CACHE_DIR = os.path.expanduser("~/.cache/gigaam")
_MODEL_NAMES = ["emo", "v1_ctc", "v1_rnnt", "v1_ssl", "v2_ctc", "v2_rnnt", "v2_ssl", "v3_ctc", "v3_rnnt",
                "v3_e2e_ctc", "v3_e2e_rnnt", "v3_ssl"]
_SHORT_NAMES = ["ctc", "rnnt", "e2e_ctc", "e2e_rnnt", "ssl"]


def _normalize_device(device: Optional[Union[str, torch.device]]) -> torch.device:
    if device is None:
        return torch.device("cuda" if torch.cuda.is_available() else "cpu")
    return torch.device(device) if isinstance(device, str) else device


def _torch_load_ckpt(path: str) -> Dict:
    """Reference checkpoints pickle an omegaconf.DictConfig as their cfg; `ckpt.load_checkpoint` reads them with or
    without omegaconf installed."""
    from .ckpt import load_checkpoint
    return load_checkpoint(path)


def load_model(model_name: str, fp16_encoder: bool = True, use_flash: Optional[bool] = False,
               device: Optional[Union[str, torch.device]] = None, download_root: Optional[str] = None, *,
               checkpoint: Optional[Dict] = None, synthetic: Optional[bool] = None, seed: int = 0,
               max_encoded_frames: Optional[int] = None) -> Union[GigaAM, GigaAMASR, GigaAMEmo]:
    """Same positional signature and semantics as gigaam.load_model (gigaam/__init__.py:110-192).

    `use_flash` is accepted for compatibility: attention always runs on the project's tensor-core kernel.
    Keyword-only extensions (the boxes this runs on have no network): `checkpoint` = an in-memory
    `{"cfg", "state_dict"}`; `synthetic=True` (or env GIGAAM_B200_SYNTHETIC=1) builds the seeded synthetic
    checkpoint of that model shape when `<download_root>/<name>.ckpt` does not exist.

    `max_encoded_frames`: longest utterance the model encodes, in encoder frames of 40 ms (like the max shape of a
    TensorRT profile).  None keeps 768 frames (30.7 s); up to the encoder's `pos_emb_max_len` (5000 frames, up to
    3 199 999 samples at 16 kHz, for the shipped checkpoints) may be requested.  Longer input is refused with the limit in the
    message.  A v1 (rel_pos) model's projected position tables take 16 x (2 * max - 1) x 768 fp16 of device memory
    (38 MB at 768, 246 MB at 5000)."""
    device_obj = _normalize_device(device)
    pack_cache_base = None
    if download_root is None:
        download_root = _CACHE_DIR
    if checkpoint is None:
        local_path = os.path.expanduser(model_name)
        if os.path.isfile(local_path):  # fine-tuned Lightning checkpoint (gigaam/__init__.py:139-156)
            finetuned = _torch_load_ckpt(local_path)
            base = load_model(finetuned["hyper_parameters"]["model_name"], fp16_encoder, use_flash, device_obj,
                              download_root, synthetic=synthetic, seed=seed, max_encoded_frames=max_encoded_frames)
            sd = {k: v for k, v in finetuned["state_dict"].items() if k.startswith(("preprocessor.", "encoder.", "head."))}
            base.load_state_dict(sd)
            return base
        if model_name not in _SHORT_NAMES + _MODEL_NAMES:
            raise ValueError(f"Model '{model_name}' not found. Available model names: {_SHORT_NAMES + _MODEL_NAMES}")
        if model_name in _SHORT_NAMES:
            model_name = f"v3_{model_name}"
        path = os.path.join(download_root, model_name + ".ckpt")
        if os.path.isfile(path):
            checkpoint = _torch_load_ckpt(path)
            pack_cache_base = os.path.join(download_root, f"{model_name}.{hash_path(path)[:16]}")
            if model_name == "v1_rnnt" or "e2e" in model_name:
                checkpoint["cfg"]["decoding"]["model_path"] = os.path.join(download_root, model_name + "_tokenizer.model")
        else:
            if synthetic is None:
                synthetic = os.environ.get("GIGAAM_B200_SYNTHETIC", "0") == "1"
            if not synthetic:
                raise FileNotFoundError(
                    f"{path} not found and this build cannot download checkpoints (no network). Place the reference "
                    "checkpoint there, or pass synthetic=True for seeded random weights of the same shape.")
            checkpoint = synthetic_checkpoint(model_name, seed=seed)
    cfg = checkpoint["cfg"]
    if "emo" in model_name:
        check_emo_head(cfg, checkpoint["state_dict"])     # NotImplementedError before any device work
        model = GigaAMEmo(cfg)
    else:
        model = GigaAM(cfg) if "ssl" in model_name else GigaAMASR(cfg)
    max_encoded_frames_config(max_encoded_frames, model.encoder.cfg["pos_emb_max_len"])   # ValueError before any device work
    check_attention_heads(model.encoder.cfg)                                                 # likewise
    model.load_state_dict(checkpoint["state_dict"])
    model = model.eval()
    model.__dict__["_pack_cache_base"] = pack_cache_base    # packed-weight cache next to the checkpoint (model.py)
    model.__dict__["_max_encoded_frames"] = max_encoded_frames   # kept across the engine rebuilds of .to() / load_state_dict
    if device_obj.type == "cpu":
        logging.warning("gigaam_b200 has no CPU compute path; the model is constructed but forward() needs CUDA")
    if fp16_encoder and device_obj.type != "cpu":
        model.encoder = model.encoder.half()
    try:
        cfg["model_name"] = model_name
    except Exception:
        pass
    return model.to(device_obj)


def hash_path(ckpt_path: str) -> str:
    return hashlib.md5(open(ckpt_path, "rb").read()).hexdigest()
