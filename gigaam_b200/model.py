"""Model wrappers with the reference's surface (gigaam/model.py:16-140): GigaAM.forward / embed_audio /
prepare_wav, GigaAMASR.transcribe / _decode, GigaAMEmo.get_probs / forward_for_export (:262-293), `_device`, `_dtype`,
`cfg`, `preprocessor`, `encoder`, `head`, `decoding`, `id2name`.  Hydra `_target_` instantiation is replaced by a small
registry keyed on the same class names."""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
from torch import Tensor, nn

from . import _lib
from .decoder import CTCHead, Linear, RNNTHead
from .decoding import CTCGreedyDecoding, RNNTGreedyDecoding, _as_btd
from .encoder import ConformerEncoder
from .engine import Engine
from .preprocess import SAMPLE_RATE, FeatureExtractor, read_audio, resample_ratio, resampled_length
from .types import Alignment, Detection, EmotionTimeline, LongformAlignment, TranscriptionResult, Word

LONGFORM_THRESHOLD = 25 * SAMPLE_RATE
ALIGN_MAX_TOKENS = 4096   # kAlignMaxTokens of csrc/kernels.h
ALIGN_LONG_MAX_TOKENS = 65536   # kAlignLongMaxTokens of csrc/kernels.h
SPOT_MAX_TOKENS = 64   # kSpotMaxTokens of csrc/kernels.h
SPOT_FIRST_MAX_DET = 256   # spot(): detections kept per keyword by the first launch; a second one keeps them all
RESAMPLE_SPAN = 30 * SAMPLE_RATE   # outputs per row when a long recording is resampled in bounded spans
RESAMPLE_ROWS = 4                  # rows (spans) per gam_resample launch of those: 2 minutes of output

_REGISTRY = {
    "FeatureExtractor": FeatureExtractor, "ConformerEncoder": ConformerEncoder, "CTCHead": CTCHead,
    "RNNTHead": RNNTHead, "CTCGreedyDecoding": CTCGreedyDecoding, "RNNTGreedyDecoding": RNNTGreedyDecoding,
    "Linear": Linear,
}

EMO_MAX_CLASSES = 256   # kPoolMaxClasses of csrc/kernels.h: one class per thread of the softmax

_NO_POSTERIORS = ("{} needs a CTC head: an RNN-T model has no per-frame posteriors without its [T, U + 1] lattice, so there "
                  "is nothing to search; use a *_ctc model")


def _plain(obj):
    """OmegaConf-like containers -> plain dict / list."""
    if hasattr(obj, "items"):
        return {k: _plain(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)) or type(obj).__name__ == "ListConfig":
        return [_plain(v) for v in obj]
    return obj


def instantiate(section: Dict, default_cls: str):
    """Stand-in for hydra.utils.instantiate (gigaam/model.py:24-25,93-94): `_target_: gigaam.<mod>.<Class>`."""
    kw = dict(section)
    target = kw.pop("_target_", None)
    kw.pop("type", None)
    name = target.rsplit(".", 1)[-1] if target else default_cls
    if name not in _REGISTRY:
        raise ValueError(f"unknown component {target!r}")
    return _REGISTRY[name](**kw)


def normalize_cfg(cfg) -> Dict:
    """Bring a checkpoint cfg (Hydra-style, with `_target_`s) or a synthetic cfg to one plain-dict shape:
    sections `preprocessor`, `encoder`, optional `head` (with `type`) and `decoding`.  A cfg with `id2name` is an emo model
    (gigaam/model.py:270): its head's type is "emo"."""
    c = _plain(cfg)
    out = dict(c)
    head = c.get("head")
    if head is not None and "type" not in head:
        tgt = str(head.get("_target_", ""))
        head = dict(head)
        if "id2name" in c:
            head["type"] = "emo"
        else:
            head["type"] = "rnnt" if "RNNT" in tgt or "decoder" in head else "ctc"
        out["head"] = head
    return out


def check_emo_head(cfg, state_dict: Optional[Dict[str, Tensor]] = None) -> None:
    """Refuse an emo head this build cannot run, before any device work.  The supported head is a `_target_` whose last
    component is `Linear`, with in_features = d_model, a bias and out_features = len(id2name) in [1, 256] (the reference's
    checkpoint names a class outside `gigaam` that maps [B, 768] -> [B, C]).  Nothing else is approximated: the
    NotImplementedError names the target and the checkpoint's `head.*` keys, so that the head to add is known."""
    c = _plain(cfg)
    head, names = dict(c.get("head") or {}), list(c.get("id2name") or [])
    target = head.get("_target_")
    d_model = c["encoder"]["d_model"]
    keys = sorted(k for k in (state_dict or {}) if k.startswith("head."))
    why = None
    if target is None or str(target).rsplit(".", 1)[-1] != "Linear":
        why = "only a Linear head (torch.nn.Linear) is supported"
    elif head.get("in_features") != d_model:
        why = f"in_features {head.get('in_features')} != d_model {d_model}"
    elif not head.get("bias", True):
        why = "a Linear head without bias is not supported"
    elif head.get("out_features") != len(names):
        why = f"out_features {head.get('out_features')} != len(id2name) {len(names)}"
    elif not 1 <= len(names) <= EMO_MAX_CLASSES:
        why = f"{len(names)} classes outside [1, {EMO_MAX_CLASSES}]"
    if why is not None:
        raise NotImplementedError(f"emo head {target!r} is not supported: {why}"
                                  + (f" (checkpoint head keys: {keys})" if state_dict is not None else ""))


class GigaAM(nn.Module):
    """Giga Acoustic Model (self-supervised encoder) -- drop-in for gigaam.model.GigaAM."""

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        self._ncfg = normalize_cfg(cfg)
        self.preprocessor = instantiate(self._ncfg["preprocessor"], "FeatureExtractor")
        self.encoder = instantiate(self._ncfg["encoder"], "ConformerEncoder")
        self.preprocessor._bind(self)
        self.encoder._bind(self)
        self.__dict__["_engine_obj"] = None

    # ---- engine lifecycle: rebuilt lazily whenever parameters move / change dtype / get reloaded
    def _invalidate_engine(self) -> None:
        self.__dict__["_engine_obj"] = None

    def _get_engine(self) -> Engine:
        eng = self.__dict__.get("_engine_obj")
        if eng is None:
            dev = self._device
            if dev.type != "cuda":
                raise RuntimeError("gigaam_b200 has no CPU path: move the model to a CUDA (sm_90a, H100) device first")
            sd = {k: v for k, v in self.state_dict().items()}
            eng = Engine(self._engine_cfg(), sd, dev, pack_cache=self._pack_cache_path(),
                         max_encoded_frames=self.__dict__.get("_max_encoded_frames"))
            eng.head_signature = self._head_signature()
            self.__dict__["_engine_obj"] = eng
        elif eng.head_signature is not None:
            sig = self._head_signature()
            if sig != eng.head_signature:      # an optimizer step or copy_ changed a head weight: repack it in place
                eng.repack_head({f"head.{k}": v for k, v in self.head.state_dict().items()})
                eng.head_signature = sig
        return eng

    def _head_signature(self):
        """(storage, version counter) of every head parameter: changes with optimizer.step(), copy_() and friends."""
        head = self._modules.get("head")
        return None if head is None else tuple((p.data_ptr(), p._version) for p in head.parameters())

    def _check_frozen_encoder(self, *modules: nn.Module) -> None:
        if torch.is_grad_enabled() and any(p.requires_grad for m in modules for p in m.parameters()):
            raise NotImplementedError("the encoder is inference-only; freeze it (requires_grad_(False) on the encoder and "
                                      "preprocessor) and train the head on its output")

    def _pack_cache_path(self) -> Optional[str]:
        """On-disk cache of the packed weights, set by load_model for checkpoints read from a file: keyed by the
        checkpoint's md5 and the parameter dtype the engine was built from (fp16_encoder rounds before packing)."""
        base = self.__dict__.get("_pack_cache_base")
        return None if base is None else f"{base}.{str(self._dtype).split('.')[-1]}.b200pack"

    def _engine_cfg(self) -> Dict:
        c = self._ncfg
        pre = {k: v for k, v in c["preprocessor"].items() if k != "_target_"}
        enc = dict(self.encoder.cfg)
        out = dict(model_name=c.get("model_name", "custom"), preprocessor=pre, encoder=enc)
        if c.get("head") is not None:
            out["head"] = {k: v for k, v in c["head"].items() if k != "_target_"}
            out["decoding"] = {k: v for k, v in c.get("decoding", {}).items() if k != "_target_"}
        return out

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        res = super().load_state_dict(state_dict, strict=strict, assign=assign)
        # the weights may no longer be the checkpoint's: the next engine packs this state_dict instead of replaying the
        # checkpoint's pack cache (load_model sets the cache key again after loading the checkpoint itself)
        self.__dict__.pop("_pack_cache_base", None)
        self._invalidate_engine()
        return res

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        self._invalidate_engine()
        return out

    # ---- reference surface
    def forward(self, features: Tensor, feature_lengths: Tensor) -> Tuple[Tensor, Tensor]:
        """wav [B, N], lengths [B] -> (encoded [B, d_model, T'], encoded_len [B] int32)  (gigaam/model.py:27-37).  The
        encoder is inference-only: with grad enabled and an encoder or preprocessor parameter requiring grad this raises."""
        self._check_frozen_encoder(self.preprocessor, self.encoder)
        features, feature_lengths = self.preprocessor(features, feature_lengths)
        return self.encoder(features, feature_lengths)

    @property
    def _device(self) -> torch.device:
        return next(self.parameters()).device

    @property
    def _dtype(self) -> torch.dtype:
        return next(self.parameters()).dtype

    # ---- audio at any sample rate (INTEGRATION.md §7k)
    def _native(self, wav_file, sample_rate: int) -> Tuple[Tensor, int]:
        """(mono float32 waveform, its sample rate) of a path (`preprocess.read_audio`: the file's own rate) or of an
        in-memory waveform at `sample_rate`.  A rate gam_resample cannot take raises ValueError here, before any device work."""
        if isinstance(wav_file, str):
            wav, sr = read_audio(wav_file)
        else:
            wav, sr = torch.as_tensor(wav_file, dtype=torch.float32).reshape(-1), sample_rate
        if sr != SAMPLE_RATE:
            resample_ratio(sr)
        return wav, sr

    def _resample_host(self, wav: Tensor, sample_rate: int) -> Tensor:
        """A 1-D waveform at `sample_rate` -> its 16 kHz samples, a host float32 tensor.  The output is cut into spans of
        RESAMPLE_SPAN samples, RESAMPLE_ROWS of them per gam_resample launch (the span form: each row uploads only the input
        its outputs need), so device memory does not grow with the recording; every output is the one-shot call's."""
        eng = self._get_engine()
        _, o, n, w = eng.resample_plan(sample_rate)
        L, K = wav.numel(), 2 * w + o
        N = resampled_length(L, sample_rate)
        out = torch.empty(N, dtype=torch.float32)
        starts = list(range(0, N, RESAMPLE_SPAN))
        for g in range(0, len(starts), RESAMPLE_ROWS):
            spans = [(max(0, a // n * o - w), min(L, (min(a + RESAMPLE_SPAN, N) - 1) // n * o - w + K), a,
                      min(a + RESAMPLE_SPAN, N)) for a in starts[g:g + RESAMPLE_ROWS]]
            x = torch.zeros((len(spans), max(max(hi - lo for lo, hi, _, _ in spans), 1)), dtype=torch.float32)
            for r, (lo, hi, _, _) in enumerate(spans):
                x[r, :hi - lo] = wav[lo:hi]
            y = torch.empty((len(spans), RESAMPLE_SPAN), dtype=torch.float32, device=eng.device)
            y = eng.resample_spans(x.to(eng.device), torch.tensor(spans, dtype=torch.int64).t(), sample_rate, y).cpu()
            for r, (_, _, a, b) in enumerate(spans):
                out[a:b] = y[r, :b - a]
        return out

    def _resample_batch(self, wav: Tensor, lengths: Tensor, sample_rate: int) -> Tuple[Tensor, Tensor]:
        """A batch at `sample_rate` -> the 16 kHz batch (Engine.resample, rounded to the model's dtype as prepare_wav does) and
        its lengths; 16 kHz input is returned as it is.  A rate gam_resample cannot take raises ValueError before any device
        work."""
        if sample_rate == SAMPLE_RATE:
            return wav, lengths
        resample_ratio(sample_rate)
        y, y_len = self._get_engine().resample(wav, lengths, sample_rate)
        return y.to(self._dtype), y_len

    def prepare_wav(self, wav_file: Union[str, Tensor, np.ndarray], sample_rate: int = SAMPLE_RATE) -> Tuple[Tensor, Tensor]:
        """gigaam/model.py:47-55; additionally accepts an in-memory mono waveform (tensor / ndarray) at `sample_rate` Hz,
        resampled to 16 kHz on the GPU (a file is read at its own rate, `preprocess.read_audio`).  The 16 kHz samples are
        rounded to the model's dtype."""
        wav, sr = self._native(wav_file, sample_rate)
        if sr != SAMPLE_RATE:
            wav = self._get_engine().resample(wav[None], torch.tensor([wav.numel()]), sr)[0][0]
        wav = wav.to(self._device).to(self._dtype).unsqueeze(0)
        length = torch.full([1], wav.shape[-1], device=self._device)
        return wav, length

    def embed_audio(self, wav_file, sample_rate: int = SAMPLE_RATE) -> Tuple[Tensor, Tensor]:
        """gigaam/model.py:57-63; `sample_rate` as in `prepare_wav`."""
        wav, length = self.prepare_wav(wav_file, sample_rate)
        return self.forward(wav, length)

    # ---- the windowed entry points' recording intake
    @property
    def _max_frames(self) -> int:
        """The most encoder frames one window may have: the model's max_encoded_frames, else the position table's length."""
        return self.__dict__.get("_max_encoded_frames") or _lib.REL_POS_MAX_T

    def _encoded_length(self, n_samples: int) -> int:
        """Encoder frames of a recording of n_samples samples (the front end's and the subsampling's length rules), on the
        host."""
        mel = self.preprocessor.out_len(torch.tensor([int(n_samples)]))
        return int(self.encoder.pre_encode.calc_output_length(mel)[0])

    def _intake(self, wav_file, sample_rate: int, window: float, overlap: float, batch_size: int
                ) -> Tuple[Tensor, int, list, int]:
        """One recording for the windowed entry points -> (its 16 kHz samples in the model's dtype in pinned host memory,
        uploaded one batch of windows at a time; N samples; `longform.plan_windows`' windows over them; T encoder frames).
        The file is read or the waveform taken, the rate checked, the windows planned on the resampled length and batch_size
        checked before any device work: ValueError for each refusal.  Then the recording is resampled in bounded spans
        (`_resample_host`) and rounded to the model's dtype, as prepare_wav rounds it; it is pinned when the model is on a GPU."""
        from .longform import plan_windows
        wav, sr = self._native(wav_file, sample_rate)
        N = wav.numel() if sr == SAMPLE_RATE else resampled_length(wav.numel(), sr)
        windows, T = plan_windows(N, window, overlap, self._encoded_length, self._max_frames)
        if batch_size < 1:
            raise ValueError("batch_size must be >= 1")
        if sr != SAMPLE_RATE:
            wav = self._resample_host(wav, sr)
        host = wav.to(self._dtype)
        return (host.pin_memory() if self._device.type == "cuda" else host), N, windows, T   # a CPU model uploads nothing


class GigaAMASR(GigaAM):
    """Giga Acoustic Model for Speech Recognition -- drop-in for gigaam.model.GigaAMASR."""

    def __init__(self, cfg):
        super().__init__(cfg)
        head_cfg = self._ncfg["head"]
        dec_cfg = {k: v for k, v in self._ncfg["decoding"].items() if k != "type"}
        self._rnnt = head_cfg.get("type") == "rnnt"
        self.head = instantiate(head_cfg, "RNNTHead" if self._rnnt else "CTCHead")
        self.head._bind(self)
        self.decoding = instantiate(dec_cfg, "RNNTGreedyDecoding" if self._rnnt else "CTCGreedyDecoding")

    def _needs_head(self, rnnt: bool, message: str) -> None:
        """Raise NotImplementedError(message) unless the model has the head a call needs: RNN-T if `rnnt`, else CTC."""
        if self._rnnt != rnnt:
            raise NotImplementedError(message)

    def _decode(self, encoded: Tensor, encoded_len: Tensor, wav_lens: Tensor, word_timestamps: bool = False,
                confidence: bool = False) -> List[Tuple[str, Optional[List[Word]], Optional[float]]]:
        """gigaam/model.py:96-124; (text, words, confidence) per utterance (confidence None unless requested)."""
        out = self.decoding.decode_device(self.head, encoded, encoded_len, scores=confidence)
        return self._results(out, encoded_len, wav_lens, word_timestamps)

    def _results(self, out: Sequence[Optional[Tensor]], encoded_len: Tensor, wav_lens: Tensor, word_timestamps: bool,
                 rec: Optional[Sequence[Tensor]] = None) -> List[Tuple[str, Optional[List[Word]], Optional[float]]]:
        """Greedy or aligned tokens (ids, frames, counts[, token_logp[, path_logp, path_rows]]), on the device or already on the
        host, -> (text, words, confidence) per utterance.  Words are None unless `word_timestamps`; they are grouped on the
        device (csrc/words.cu) unless `rec` holds host copies of gam_group_words' records.  token_logp, when given, gives every
        word its confidence; path_logp / path_rows give the utterance's (None without them)."""
        from .timestamps_utils import compute_frame_shift, path_confidence, words_from_device
        tok = self.decoding.tokenizer

        def host(i: int) -> Optional[Tensor]:
            return out[i].cpu() if len(out) > i and out[i] is not None else None
        token_logp = host(3) if word_timestamps else None
        path_logp, path_rows = host(4), host(5)
        res = []
        if word_timestamps:
            if rec is None:
                rec = self._get_engine().group_words(out[0], out[1], out[2], self._word_flags())
            ws, we, wf, wn, nw = (t.cpu() for t in rec)
            enc_len, wav_len = encoded_len.cpu(), wav_lens.cpu()
        ids = out[0].cpu()
        for i, n in enumerate(out[2].cpu().tolist()):
            row = ids[i, :n].tolist()
            words = None
            if word_timestamps:
                k = int(nw[i])
                words = words_from_device(tok, row, ws[i, :k].tolist(), we[i, :k].tolist(), wf[i, :k].tolist(), wn[i, :k].tolist(),
                                          compute_frame_shift(int(wav_len[i]), int(enc_len[i])),
                                          None if token_logp is None else token_logp[i, :n].tolist())
            res.append((tok.decode(row), words, None if path_logp is None else path_confidence(path_logp[i], path_rows[i])))
        return res

    def _word_flags(self) -> Tensor:
        """Per-token flag table of the device word grouping (timestamps_utils.token_flag_table), built once."""
        flags = self.__dict__.get("_token_flags")
        if flags is None or flags.device != self._device:        # device-resident: the grouping runs inside CUDA graphs
            from .timestamps_utils import token_flag_table
            flags = token_flag_table(self.decoding.tokenizer).to(self._device)
            self.__dict__["_token_flags"] = flags
        return flags

    def forward_for_export(self, features: Tensor, feature_lengths: Tensor) -> Tuple[Tensor, Tensor]:
        """log-mel [B, F, M], lengths [B] -> (head(encoded), encoded_len) (gigaam/model.py:142-149): CTC log-probs
        [B, T', V+1].  An RNN-T head has no forward, so this raises for RNN-T models, as in the reference."""
        encoded, encoded_len = self.encoder(features, feature_lengths)
        return self.head(encoded), encoded_len

    @torch.inference_mode()
    def transcribe(self, wav_file, word_timestamps: bool = False, confidence: bool = False,
                   hotwords: Optional[Sequence[Union[str, Sequence[int]]]] = None, hotword_threshold: float = 0.5,
                   boost: Optional[Sequence[Union[str, Sequence[int]]]] = None, boost_weight: float = 1.0,
                   sample_rate: int = SAMPLE_RATE) -> TranscriptionResult:
        """gigaam/model.py:126-140.  `confidence=True` decodes with the scored kernels (the same text and words) and fills
        `confidence` of the result, and of every word when word timestamps are on (INTEGRATION.md, "Confidence").
        `hotwords` (CTC models only): names or terms that replace the greedy words they outscore by `hotword_threshold`
        (INTEGRATION.md §7h); None decodes exactly as without them.  `boost` (RNN-T models only): names or terms whose
        tokens get `boost_weight` nats added to their logits while the greedy decoder follows them (INTEGRATION.md §7j);
        scores stay the model's own.  None decodes exactly as without it.  `sample_rate`: the rate of in-memory audio, resampled
        to 16 kHz on the GPU before the 25 s check (INTEGRATION.md §7k); times stay seconds of the recording."""
        kw_ids = tables = None
        if hotwords is not None:              # boost is not looked at then
            kw_ids = self._hotword_ids(hotwords, hotword_threshold, "transcribe")
        elif boost is not None:
            tables = self._boost_tables(boost, boost_weight, "transcribe")
        wav, length = self.prepare_wav(wav_file, sample_rate)
        if length.item() > LONGFORM_THRESHOLD:
            raise ValueError("Too long wav file, use 'transcribe_longform' method.")
        encoded, encoded_len = self.forward(wav, length)
        if kw_ids is None and tables is None:
            text, words, conf = self._decode(encoded, encoded_len, length, word_timestamps, confidence)[0]
            return TranscriptionResult(text=text, words=words, confidence=conf)
        eng = self._get_engine()
        enc = _as_btd(encoded.to(dtype=torch.float32))
        if tables is not None:                # one boosted decoding call from a fresh record
            T = enc.shape[1]
            zero = torch.zeros(1, dtype=torch.int32, device=eng.device)
            out = eng.decode_buffers(1, eng.hyp_width(T), T, scores=confidence)
            eng.greedy_resume(enc, zero, encoded_len.to(device=eng.device, dtype=torch.int32), zero, eng.decode_state(1), out,
                              confidence, tuple(t.to(eng.device) for t in tables))
        else:                                 # greedy decoding, then the spotted hotwords spliced in
            g = self.decoding.decode_device(self.head, encoded, encoded_len, scores=confidence)
            lp = eng.ctc_log_probs(enc)
            ids, frames, counts, _, token_logp, path_logp = self._apply_hotwords(lp, encoded_len, kw_ids, hotword_threshold, *g[:5])
            del lp
            out = (ids, frames, counts, token_logp, path_logp, *g[5:])
        text, words, conf = self._results(out, encoded_len, length, word_timestamps)[0]
        return TranscriptionResult(text=text, words=words, confidence=conf)

    @torch.inference_mode()
    def transcribe_longform(self, wav_file, word_timestamps: bool = False, fr_batch_size: int = 16, fr_num_workers: int = 0,
                            segments: Optional[List[Tensor]] = None, boundaries: Optional[List[Tuple[float, float]]] = None,
                            confidence: bool = False, sample_rate: int = SAMPLE_RATE, **kwargs):
        """gigaam/model.py:195-259.  Segmentation is pluggable: pass `segments` / `boundaries` from any VAD (the
        reference's pyannote pipeline, gigaam/vad_utils.py, is third party and not vendored); without them the
        recording is cut at low-energy points (`longform.split_on_energy`, kwargs forwarded).  Segments are
        length-bucketed into batches of `fr_batch_size`; `fr_num_workers` is accepted for signature compatibility.
        `confidence=True` fills every segment's (and word's) `confidence`, scored inside the same device step.  `sample_rate`:
        the rate of an in-memory `wav_file`, resampled to 16 kHz first; `segments` are 16 kHz."""
        from .longform import split_on_energy, transcribe_segments
        if segments is None:
            wav, sr = self._native(wav_file, sample_rate)
            if sr != SAMPLE_RATE:
                wav = self._resample_host(wav, sr)
            segments, boundaries = split_on_energy(wav, SAMPLE_RATE, **kwargs)
        elif boundaries is None:
            raise ValueError("boundaries are required when segments are given")
        return transcribe_segments(self, segments, boundaries, word_timestamps, fr_batch_size, confidence)

    @torch.inference_mode()
    def align(self, wav_file, text: Union[str, Sequence[int]], word_timestamps: bool = True, sample_rate: int = SAMPLE_RATE
              ) -> Alignment:
        """Align a known transcript to one recording: `text` is a string (normalised and tokenised by
        `Tokenizer.encode`) or a sequence of token ids.  There is no 25 s limit: any length the loaded model encodes is
        accepted (INTEGRATION.md §7d).  `sample_rate` as in `prepare_wav`."""
        wav, length = self.prepare_wav(wav_file, sample_rate)
        return self.align_batch(wav, length, [text], word_timestamps)[0]

    @torch.inference_mode()
    def align_batch(self, wav: Tensor, lengths: Tensor, texts: Sequence[Union[str, Sequence[int]]],
                    word_timestamps: bool = True, sample_rate: int = SAMPLE_RATE) -> List[Alignment]:
        """Align texts[b] to wav[b, :lengths[b]] for every b (Viterbi words, forward log-likelihood, path confidence).
        Raises ValueError before any device work for an empty batch, len(texts) != B, more than 4096 tokens or an id outside
        [0, V) and for a `sample_rate` that cannot be resampled.  An utterance without an alignment (too few frames for its
        tokens) gets log_likelihood = -inf and no words.  `sample_rate`: the batch's rate, resampled to 16 kHz first."""
        from .decoding import align
        from .timestamps_utils import path_confidence
        B = self._batch_rows(wav, "align")
        if len(texts) != B:
            raise ValueError(f"align: {len(texts)} texts for a batch of {B} recordings")
        norm, ids = [], []
        for text in texts:
            name, row = self._text_ids(text, "align")
            if len(row) > ALIGN_MAX_TOKENS:
                raise ValueError(f"align: {len(row)} tokens exceed the limit of {ALIGN_MAX_TOKENS} per utterance")
            norm.append(name)
            ids.append(row)
        U = max(len(r) for r in ids)
        targets = torch.zeros((B, U), dtype=torch.int32)
        for b, row in enumerate(ids):
            targets[b, :len(row)] = torch.tensor(row, dtype=torch.int32)
        target_len = torch.tensor([len(r) for r in ids], dtype=torch.int32)
        wav, lengths = self._resample_batch(wav, lengths, sample_rate)
        encoded, encoded_len = self.forward(wav, lengths)
        dev = encoded.device
        targets_d, target_len_d = targets.to(dev), target_len.to(dev)
        frames, token_logp, viterbi_logp, log_likelihood, path_rows = align(self.head, encoded, encoded_len, targets_d, target_len_d)
        ll, vit = torch.stack([log_likelihood, viterbi_logp]).cpu().tolist()
        words: List[Optional[List[Word]]] = [None] * B
        if word_timestamps:
            words = [[] for _ in range(B)]
            if U > 0:
                found = self._results((targets_d, frames, target_len_d, token_logp), encoded_len, lengths, True)
                words = [w if math.isfinite(v) else [] for (_, w, _), v in zip(found, vit)]
        rows = path_rows.cpu().tolist()
        return [Alignment(text=norm[b], words=words[b], log_likelihood=ll[b], confidence=path_confidence(vit[b], rows[b]))
                for b in range(B)]

    def _text_ids(self, text: Union[str, Sequence[int]], what: str) -> Tuple[str, List[int]]:
        """(normalised text, token ids) of a string (`Tokenizer.encode`) or of a sequence of token ids, taken as it is:
        ValueError `what: token id ... outside [0, V)` for an id the vocabulary lacks."""
        tok = self.decoding.tokenizer
        if isinstance(text, str):
            row = tok.encode(text)
            return tok.normalize(text), row
        row = [int(i) for i in text]
        bad = [i for i in row if not 0 <= i < len(tok)]
        if bad:
            raise ValueError(f"{what}: token id {bad[0]} outside [0, {len(tok)})")
        return tok.decode(row), row

    def _refuse_edge_spaces(self, ids: List[List[int]], what: str, noun: str, why: str) -> None:
        """ValueError for a phrase whose first or last token is the space token; `why` tells what to pass instead."""
        tok = self.decoding.tokenizer
        for row in ids:
            if any(tok.id_to_str(row[i]) == " " for i in (0, -1)):
                raise ValueError(f"{what}: {noun} {tok.decode(row)!r} starts or ends with the space token; {why}")

    def _line_tokens(self, lines: Sequence[str]) -> Tuple[List[str], List[int], List[Tuple[int, int]]]:
        """Normalised lines, the token ids of the whole text and each line's token range [a, b).  Lines are joined so that
        no word spans two of them: a charwise vocabulary puts one space token between non-empty lines; SentencePiece
        lines start with U+2581, which opens a word by itself.  (A charwise vocabulary without a space token has no word
        boundaries at all: its lines are joined as they are.)"""
        tok = self.decoding.tokenizer
        space = tok.vocab.index(" ") if tok.charwise and " " in tok.vocab else None
        norm, ids, ranges = [], [], []
        for line in lines:
            if not isinstance(line, str):
                raise TypeError(f"align_longform: lines must be strings, got {type(line).__name__}")
            name, row = self._text_ids(line, "align_longform")
            norm.append(name)
            if row and ids and space is not None:
                ids.append(space)
            ranges.append((len(ids), len(ids) + len(row)))
            ids.extend(row)
        return norm, ids, ranges

    @torch.inference_mode()
    def align_longform(self, wav_file, text: Union[str, Sequence[str]], word_timestamps: bool = True, window: float = 30.0,
                       overlap: float = 4.0, batch_size: int = 16, *, gap_threshold: Optional[float] = None,
                       skip_threshold: Optional[float] = None, sample_rate: int = SAMPLE_RATE) -> LongformAlignment:
        """Align a known text, one string or a sequence of lines, to a recording of any length (INTEGRATION.md §7e).  The
        encoder runs over overlapping windows (`longform.plan_windows`), the windows' CTC log-probs are stitched into one
        sequence and gam_ctc_align_long aligns the whole text to it: up to 65 536 tokens, no frame limit.  Returns one
        Segment per line.  CTC models only: RNN-T raises NotImplementedError.  Raises ValueError before any device work for
        more than 65 536 tokens and for the window plan's refusals (longform.plan_windows).
        `gap_threshold` (theta in (0, 1], INTEGRATION.md §7e) lets audio between lines that the text lacks stay unaligned
        (gam_ctc_align_long_gaps): a frame at a line's edge is left unmatched where theta times the greedy decoder's
        probability beats blank, and the result's `unmatched` lists those stretches; ValueError for theta outside (0, 1] as
        float32, or NaN.
        `skip_threshold` (psi in (0, 1], the same checks) lets whole lines the recording lacks be skipped
        (gam_ctc_align_long_skips): skipping a line and the joining token before it costs psi per token, and the
        result's `skipped` lists the skipped lines.
        `sample_rate`: the rate of an in-memory `wav_file`, resampled to 16 kHz in bounded spans before the window plan."""
        from .longform import line_edges, line_segments, skipped_lines, stitch_ctc_log_probs, unmatched_intervals
        from .timestamps_utils import compute_frame_shift, gap_confidence, path_confidence, words_from_device
        self._needs_head(False, "align_longform needs a CTC head: RNN-T alignment walks a [T, U + 1] lattice, about 4.5e9 nodes "
                                "for an hour of speech, and banding it would no longer give the Viterbi path; use a *_ctc model, "
                                "or align() up to max_encoded_frames")

        def log_threshold(name, value):
            x = float(np.float32(value))
            if not 0.0 < x <= 1.0:              # NaN fails too
                raise ValueError(f"align_longform: {name} must be in (0, 1], got {value!r}")
            return float(np.float32(math.log(x)))   # spot's rounding of log theta
        log_theta = None if gap_threshold is None else log_threshold("gap_threshold", gap_threshold)
        log_psi = None if skip_threshold is None else log_threshold("skip_threshold", skip_threshold)
        lines = [text] if isinstance(text, str) else list(text)
        norm, ids, ranges = self._line_tokens(lines)
        if len(ids) > ALIGN_LONG_MAX_TOKENS:
            raise ValueError(f"align_longform: {len(ids)} tokens exceed the limit of {ALIGN_LONG_MAX_TOKENS}")
        host, N, windows, T = self._intake(wav_file, sample_rate, window, overlap, batch_size)
        lp = stitch_ctc_log_probs(self, host, windows, T, batch_size)
        eng = self._get_engine()
        U = len(ids)
        targets = torch.tensor([ids], dtype=torch.int32).reshape(1, U)
        targets_d = targets.to(eng.device)
        target_len_d = torch.tensor([U], dtype=torch.int32, device=eng.device)
        enc_len = torch.tensor([T], dtype=torch.int32, device=eng.device)
        skip_rows = skip_logp = None
        if log_theta is None and log_psi is None:
            frames, token_logp, viterbi_logp, log_likelihood, path_rows = eng.ctc_align_long(lp, enc_len, targets_d, target_len_d)
        else:
            edges = torch.tensor(line_edges(ranges, U), dtype=torch.uint8).reshape(1, U).to(eng.device)
            gaps = (edges, -math.inf if log_theta is None else log_theta)
            if log_psi is None:
                frames, token_logp, viterbi_logp, log_likelihood, path_rows, unmatched, u_rows, u_logp = eng.ctc_align_long(
                    lp, enc_len, targets_d, target_len_d, gaps=gaps)
            else:
                (frames, token_logp, viterbi_logp, log_likelihood, path_rows, unmatched, u_rows, u_logp, skip_rows,
                 skip_logp) = eng.ctc_align_long(lp, enc_len, targets_d, target_len_d, gaps=gaps, skips=log_psi)
        del lp
        vit, ll = float(viterbi_logp[0]), float(log_likelihood[0])
        shift = compute_frame_shift(N, T)
        fr, logp = frames[0].cpu().tolist(), token_logp[0].cpu().tolist()
        skipped = None
        if log_psi is not None:
            skipped = skipped_lines(ranges, fr) if math.isfinite(vit) else []
        words, word_first = None, None
        if word_timestamps:
            words, word_first = [], []
            kept = [i for i, f in enumerate(fr) if f >= 0] if skipped else None
            if U > 0 and math.isfinite(vit) and kept != []:     # a path that skips every line has no words
                if skipped:                                     # group the aligned tokens only
                    k_ids, k_logp = [ids[i] for i in kept], [logp[i] for i in kept]
                    k_idx = torch.tensor(kept, dtype=torch.int64, device=eng.device)
                    k_targets, k_frames = targets_d[:, k_idx].contiguous(), frames[:, k_idx].contiguous()
                    k_len = torch.tensor([len(kept)], dtype=torch.int32, device=eng.device)
                else:
                    k_ids, k_logp, k_targets, k_frames, k_len = ids, logp, targets_d, frames, target_len_d
                ws, we, wf, wn, k = (t[0].cpu().tolist() for t in eng.group_words(k_targets, k_frames, k_len, self._word_flags()))
                words = words_from_device(self.decoding.tokenizer, k_ids, ws[:k], we[:k], wf[:k], wn[:k], shift, k_logp)
                word_first = wf[:k] if kept is None else [kept[f] for f in wf[:k]]
        segs = line_segments(norm, ranges, fr, logp, shift, vit, words, word_first, skipped or ())
        if log_theta is None and log_psi is None:
            return LongformAlignment(segments=segs, log_likelihood=ll, confidence=path_confidence(vit, int(path_rows[0])))
        matched = int(path_rows[0]) - int(u_rows[0])
        conf = gap_confidence(vit, float(u_logp[0]), matched, 0.0 if skip_logp is None else float(skip_logp[0]))
        gaps_out = None if log_theta is None else unmatched_intervals(unmatched[0], shift)
        return LongformAlignment(segments=segs, log_likelihood=ll, confidence=conf, unmatched=gaps_out, skipped=skipped)

    @torch.inference_mode()
    def transcribe_windowed(self, wav_file, word_timestamps: bool = False, confidence: bool = False, window: float = 30.0,
                            overlap: float = 4.0, batch_size: int = 16, pause: float = 1.0, max_segment: float = 25.0,
                            hotwords: Optional[Sequence[Union[str, Sequence[int]]]] = None, hotword_threshold: float = 0.5,
                            boost: Optional[Sequence[Union[str, Sequence[int]]]] = None, boost_weight: float = 1.0,
                            sample_rate: int = SAMPLE_RATE):
        """Transcribe a recording of any length without a VAD (INTEGRATION.md §7f).  The encoder runs over overlapping
        windows (`longform.plan_windows`), and the greedy decoder runs over the windows' kept frames as ONE utterance: each
        window is decoded as soon as its batch is encoded, resuming the decoder state of the window before it
        (gam_*_greedy_resume), so no cut falls inside a word and device memory does not grow with the recording.  Segments
        are cut afterwards between words (`longform.segment_cuts`: at pauses of at least `pause` seconds, then inside
        segments longer than `max_segment` seconds).  Returns a LongformTranscriptionResult whose segments tile the
        recording.  Raises ValueError before any device work for the window plan's refusals, batch_size < 1, pause < 0 and
        max_segment <= 0.  `hotwords` as in `transcribe` (CTC models only): the windows' log-probs are also stitched into one
        [T, V+1] sequence from the same encoder pass, and the hotwords are applied to the whole recording before it is cut into
        segments.  `boost` and `boost_weight` as in `transcribe` (RNN-T models only): every window's decoding is boosted, the
        graph state carried across windows with the decoder's.  `sample_rate`: the rate of an in-memory `wav_file`, resampled to
        16 kHz in bounded spans into host memory before the window plan (INTEGRATION.md §7k)."""
        from .longform import check_segmenting, decode_windows, windowed_result
        kw_ids = None if hotwords is None else self._hotword_ids(hotwords, hotword_threshold, "transcribe_windowed")
        tables = None if boost is None else self._boost_tables(boost, boost_weight, "transcribe_windowed")
        check_segmenting(pause, max_segment)
        host, N, windows, T = self._intake(wav_file, sample_rate, window, overlap, batch_size)
        eng = self._get_engine()
        if tables is not None:
            out = decode_windows(self, host, windows, T, batch_size, confidence, boost=tuple(t.to(eng.device) for t in tables))
        elif kw_ids is None:
            out = decode_windows(self, host, windows, T, batch_size, confidence)
        else:
            lp = torch.empty((1, T, eng.num_classes), dtype=torch.float32, device=eng.device)
            out = decode_windows(self, host, windows, T, batch_size, confidence, log_probs=lp)
            enc_len = torch.tensor([T], dtype=torch.int32, device=eng.device)
            b_ids, b_frames, b_counts, _, b_logp, b_path = self._apply_hotwords(
                lp, enc_len, kw_ids, hotword_threshold, out.ids, out.frames, out.counts, out.token_logp, out.path_logp,
                out.frame_logp)
            del lp
            out = out._replace(ids=b_ids, frames=b_frames, counts=b_counts, token_logp=b_logp, path_logp=b_path)
        n = int(out.counts[0])
        return windowed_result(self, out.ids[0, :n].tolist(), out.frames[0, :n].tolist(),
                               out.token_logp[0, :n].tolist() if confidence else None,
                               out.frame_logp[0].cpu().numpy() if confidence else None,
                               out.frame_rows[0].cpu().numpy() if confidence else None, N, T, word_timestamps, pause, max_segment)

    def streaming(self, window: float = 8.0, overlap: float = 4.0, batch_size: int = 64, confidence: bool = False,
                  keywords: Optional[Sequence[Union[str, Sequence[int]]]] = None, threshold: float = 0.5,
                  boost: Optional[Sequence[Union[str, Sequence[int]]]] = None, boost_weight: float = 1.0,
                  sample_rate: int = SAMPLE_RATE, hotwords: Optional[Sequence[Union[str, Sequence[int]]]] = None,
                  hotword_threshold: float = 0.5):
        """A `streaming.StreamServer` for live audio (INTEGRATION.md §7i): open streams, push chunks, `step()` for captions
        and keyword alerts, `close()` for each stream's `transcribe_windowed` / `spot` result.  `boost` and `boost_weight` as
        in `transcribe` (RNN-T models only), for every stream of the server.  Raises before any device work: ValueError for
        the window plan's refusals, batch_size < 1, `spot`'s keyword and threshold checks and `boost`'s checks;
        NotImplementedError for keywords on an RNN-T model and for boost on a CTC model.  `sample_rate`: the rate of the pushed
        samples, resampled to 16 kHz as they arrive (INTEGRATION.md §7k); ValueError for a rate gam_resample cannot take.
        `hotwords` and `hotword_threshold` as in `transcribe` (CTC models only, checked the same way before any device work):
        captions commit text with the hotwords spliced in once no later detection can change it, and a closed stream equals
        `transcribe_windowed(..., hotwords=hotwords, hotword_threshold=hotword_threshold)`."""
        from .streaming import StreamServer
        tables = None if boost is None else self._boost_tables(boost, boost_weight, "streaming")
        return StreamServer(self, window, overlap, batch_size, confidence, keywords, threshold, boost=tables, sample_rate=sample_rate,
                            hotwords=hotwords, hotword_threshold=hotword_threshold)

    # ---- keyword spotting (INTEGRATION.md §7g)
    def _keyword_ids(self, keywords: Sequence[Union[str, Sequence[int]]], threshold: float) -> Tuple[List[str], List[List[int]]]:
        """Each keyword's text and token ids (`_phrase_ids`), then the threshold, checked before any device work: ValueError
        also for a threshold outside (0, 1] (in fp32)."""
        names, ids = self._phrase_ids(keywords, "spot", "keyword")
        if not 0.0 < float(np.float32(threshold)) <= 1.0:
            raise ValueError(f"spot: threshold={threshold} outside (0, 1]")
        return names, ids

    def _phrase_ids(self, phrases: Sequence[Union[str, Sequence[int]]], what: str, noun: str) -> Tuple[List[str], List[List[int]]]:
        """Each phrase's text and token ids, checked before any device work: a string is normalised and tokenised by
        `Tokenizer.encode` (as `align` does), a sequence of ids is taken as it is.  Raises ValueError for an empty list, a
        phrase without tokens, more than 64 tokens and an id outside [0, V); messages start with `what` and name the phrase
        a `noun`."""
        kws = [phrases] if isinstance(phrases, str) else list(phrases)
        if not kws:
            raise ValueError(f"{what}: no {noun}s")
        names, ids = [], []
        for kw in kws:
            name, row = self._text_ids(kw, what)
            if not row:
                raise ValueError(f"{what}: {noun} {kw!r} normalises to no tokens" if isinstance(kw, str)
                                 else f"{what}: a {noun} without tokens")
            if len(row) > SPOT_MAX_TOKENS:
                raise ValueError(f"{what}: {noun} {name!r} has {len(row)} tokens, more than {SPOT_MAX_TOKENS}")
            names.append(name)
            ids.append(row)
        return names, ids

    @staticmethod
    def _keyword_tensors(ids: List[List[int]], device) -> Tuple[Tensor, Tensor]:
        keywords = torch.zeros((len(ids), max(len(r) for r in ids)), dtype=torch.int32)
        for k, row in enumerate(ids):
            keywords[k, :len(row)] = torch.tensor(row, dtype=torch.int32)
        return keywords.to(device), torch.tensor([len(r) for r in ids], dtype=torch.int32, device=device)

    @staticmethod
    def _detections(names: List[str], ids: List[List[int]], dets: Sequence[Sequence[Tuple[int, int, float]]],
                    frame_shift: float) -> List[Detection]:
        """Each keyword's (start frame, end frame, score) detections in one recording -> its Detection records, sorted by
        start, then keyword."""
        out = [(s, k, Detection(keyword=name, keyword_index=k, start=s * frame_shift, end=e * frame_shift, score=sc,
                                confidence=math.exp(sc / len(ids[k]))))
               for k, name in enumerate(names) for s, e, sc in dets[k]]
        out.sort(key=lambda d: d[:2])
        return [d for _, _, d in out]

    @staticmethod
    def _stored(start: Tensor, end: Tensor, score: Tensor, count: Tensor) -> List[List[Tuple[int, int, float]]]:
        """Host copies of one recording's gam_ctc_spot outputs ([K, max_det], count [K]) -> each keyword's stored detections."""
        n = count.clamp(max=start.shape[1]).tolist()
        return [list(zip(start[k, :c].tolist(), end[k, :c].tolist(), score[k, :c].tolist())) for k, c in enumerate(n)]

    @torch.inference_mode()
    def spot_batch(self, wav: Tensor, lengths: Tensor, keywords: Sequence[Union[str, Sequence[int]]], threshold: float = 0.5,
                   max_det: int = 64, sample_rate: int = SAMPLE_RATE) -> List[List[Detection]]:
        """Spot every keyword in every recording wav[b, :lengths[b]] of a batch the model encodes in one pass (up to
        max_encoded_frames).  Returns one list per recording, sorted by start, then keyword index; at most `max_det`
        detections of each keyword are kept (the first ones in time).  Keywords are strings (normalised and tokenised as
        `align` does) or sequences of token ids, up to 64 tokens; `threshold` in (0, 1] is the lowest per-token likelihood
        ratio to greedy decoding that is reported (INTEGRATION.md §7g).  RNN-T models raise NotImplementedError; the keyword,
        threshold, batch and `sample_rate` checks raise ValueError, all before any device work.  `sample_rate`: the batch's rate,
        resampled to 16 kHz first."""
        from .decoding import spot
        from .timestamps_utils import compute_frame_shift
        self._needs_head(False, _NO_POSTERIORS.format("spot_batch"))
        names, ids = self._keyword_ids(keywords, threshold)
        if max_det < 1:
            raise ValueError(f"spot_batch: max_det={max_det} must be >= 1")
        B = self._batch_rows(wav, "spot_batch")
        wav, lengths = self._resample_batch(wav, lengths, sample_rate)
        encoded, encoded_len = self.forward(wav, lengths)
        kw, kw_len = self._keyword_tensors(ids, encoded.device)
        start, end, score, count = (t.cpu() for t in spot(self.head, encoded, encoded_len, kw, kw_len, threshold, max_det))
        enc_len, wav_len = encoded_len.cpu().tolist(), lengths.cpu().tolist()
        return [self._detections(names, ids, self._stored(start[b], end[b], score[b], count[b]),
                                 compute_frame_shift(int(wav_len[b]), int(enc_len[b])) if enc_len[b] > 0 else 0.0)
                for b in range(B)]

    @staticmethod
    def _batch_rows(wav: Tensor, what: str) -> int:
        """The rows of a [B, N] batch; ValueError for an empty batch (or one that is not 2-D)."""
        B = int(wav.shape[0]) if wav.dim() == 2 else 0
        if B == 0:
            raise ValueError(f"{what}: empty batch")
        return B

    @torch.inference_mode()
    def spot(self, wav_file, keywords: Sequence[Union[str, Sequence[int]]], threshold: float = 0.5, window: float = 30.0,
             overlap: float = 4.0, batch_size: int = 16, sample_rate: int = SAMPLE_RATE) -> List[Detection]:
        """Spot keywords in a recording of any length (INTEGRATION.md §7g): the CTC log-probs of the overlapping windows of
        `align_longform` are stitched into one sequence and gam_ctc_spot searches it for every keyword at once.  Returns
        every detection, sorted by start, then keyword index.  Keywords and threshold as in `spot_batch`.  CTC models only:
        RNN-T raises NotImplementedError.  Raises ValueError before any device work for the keyword and threshold checks,
        batch_size < 1 and the window plan's refusals (longform.plan_windows).  `sample_rate`: the rate of an in-memory
        `wav_file`, resampled to 16 kHz in bounded spans into host memory before the window plan."""
        from .longform import stitch_ctc_log_probs
        from .timestamps_utils import compute_frame_shift
        self._needs_head(False, _NO_POSTERIORS.format("spot"))
        names, ids = self._keyword_ids(keywords, threshold)
        host, N, windows, T = self._intake(wav_file, sample_rate, window, overlap, batch_size)
        lp = stitch_ctc_log_probs(self, host, windows, T, batch_size)
        eng = self._get_engine()
        kw, kw_len = self._keyword_tensors(ids, eng.device)
        enc_len = torch.tensor([T], dtype=torch.int32, device=eng.device)
        out = self._spot_all(lp, enc_len, kw, kw_len, ids, threshold)
        del lp
        return self._detections(names, ids, self._stored(*(t[0].cpu() for t in out)), compute_frame_shift(N, T))

    def _spot_all(self, lp: Tensor, enc_len: Tensor, kw: Tensor, kw_len: Tensor, ids: List[List[int]], threshold: float
                  ) -> Tuple[Tensor, ...]:
        """gam_ctc_spot over log-probs [B, T, V+1] keeping every detection: a first launch keeps up to SPOT_FIRST_MAX_DET per
        keyword, and one more with the largest count runs only when a count exceeds that."""
        eng = self._get_engine()
        # detections of one keyword do not overlap and span >= U frames each: T // U bounds the count
        max_det = max(1, min(lp.shape[1] // min(len(r) for r in ids), SPOT_FIRST_MAX_DET))
        out = eng.ctc_spot(lp, enc_len, kw, kw_len, threshold, max_det)
        most = int(out[3].max())
        if most > max_det:
            out = eng.ctc_spot(lp, enc_len, kw, kw_len, threshold, most)
        return out

    # ---- hotwords (INTEGRATION.md §7h)
    def _hotword_ids(self, hotwords: Sequence[Union[str, Sequence[int]]], threshold: float, what: str) -> List[List[int]]:
        """Token ids of the hotwords, checked before any device work: RNN-T models raise NotImplementedError, the keyword and
        threshold checks of `spot` raise ValueError, and so does a hotword that starts or ends with the space token (the
        splice keeps to word boundaries by itself)."""
        self._needs_head(False, _NO_POSTERIORS.format(what))
        _, ids = self._keyword_ids(hotwords, threshold)
        self._refuse_edge_spaces(ids, what, "hotword", "hotwords are spliced at word boundaries only, so pass the word without "
                                 "its spaces")
        return ids

    # ---- phrase boosting (INTEGRATION.md §7j)
    def _boost_tables(self, phrases: Sequence[Union[str, Sequence[int]]], weight: float, what: str) -> Tuple[Tensor, Tensor]:
        """The host tables of the boost graph of `phrases` (decoding.boost_graph), checked before any device work: CTC
        models raise NotImplementedError; `spot`'s phrase checks, a phrase that starts or ends with the space token, a weight
        that is not finite and > 0 and a graph of more than 65 536 states raise ValueError.  A charwise vocabulary anchors
        every phrase at a word start (its space token); SentencePiece pieces open their words themselves."""
        from .decoding import boost_graph
        self._needs_head(True, f"{what}: boost steers the RNN-T greedy decoder; for a CTC model use hotwords=, which splices "
                               "spotted phrases into the transcript")
        _, ids = self._phrase_ids(phrases, what, "phrase")
        self._refuse_edge_spaces(ids, what, "phrase", "a phrase is anchored at a word start by itself, so pass the words "
                                 "without edge spaces")
        tok = self.decoding.tokenizer
        anchor = tok.vocab.index(" ") if tok.charwise and " " in tok.vocab else None
        return boost_graph(ids, weight, anchor, len(tok) + 1, len(tok))

    def _apply_hotwords(self, lp: Tensor, enc_len: Tensor, ids: List[List[int]], threshold: float, g_ids: Tensor, g_frames: Tensor,
                        g_counts: Tensor, token_logp: Optional[Tensor] = None, path_logp: Optional[Tensor] = None,
                        frame_logp: Optional[Tensor] = None) -> Tuple[Tensor, ...]:
        """Spot the hotwords in lp [B, T, V+1] (every detection kept) and splice them into the greedy output (gam_ctc_bias):
        -> (ids, frames, counts, source, token_logp or None, path_logp or None); frame_logp is adjusted in place."""
        eng = self._get_engine()
        kw, kw_len = self._keyword_tensors(ids, eng.device)
        spotted = self._spot_all(lp, enc_len, kw, kw_len, ids, threshold)
        return eng.ctc_bias(lp, enc_len, kw, kw_len, spotted, threshold, self._word_flags(), g_ids, g_frames, g_counts, token_logp,
                            path_logp, frame_logp)

    @torch.inference_mode()
    def transcribe_batch(self, wav: Tensor, lengths: Tensor, sample_rate: int = SAMPLE_RATE) -> List[str]:
        """Batched entry (the path eval.py / transcribe_longform drive: model(wav, len) -> decoding.decode).  `sample_rate`:
        the batch's rate, resampled to 16 kHz first (ValueError, before any device work, for a rate that cannot be)."""
        wav, lengths = self._resample_batch(wav, lengths, sample_rate)
        encoded, encoded_len = self.forward(wav, lengths)
        return [t for t, _, _ in self.decoding.decode(self.head, encoded, encoded_len)]


class GigaAMEmo(GigaAM):
    """Giga Acoustic Model for Emotion Recognition -- drop-in for gigaam.model.GigaAMEmo (gigaam/model.py:262-293).

    Frames pooled for utterance b: n_b = encoded_len[b], except that a batch of ONE pools all T' frames (the rule of the
    encoder's packed rows, DESIGN §3.1).  `get_probs` is thus exactly the reference's (it pools every frame of its one
    utterance), and every utterance's probabilities are independent of the batch it is in.  The reference's
    `forward_for_export` averages over the padded T' instead; on ragged batches of more than one utterance its answer
    depends on the padding, and this build's padded frames are zeros, so that answer is not reproduced.  An utterance with
    n_b = 0 gives a NaN row (the mean of an empty set)."""

    def __init__(self, cfg):
        super().__init__(cfg)
        check_emo_head(cfg)
        self.head = instantiate(self._ncfg["head"], "Linear")
        self.head._bind(self)
        self.id2name = self._ncfg["id2name"]

    def _pooled_probs(self, encoded: Tensor, encoded_len: Optional[Tensor]) -> Tensor:
        _, _, probs = self._get_engine().emo_head(_as_btd(encoded), encoded_len)
        return probs

    @torch.inference_mode()
    def get_probs(self, wav_file, sample_rate: int = SAMPLE_RATE) -> Dict[str, float]:
        """gigaam/model.py:272-285: {class name: probability} of one recording (a path or an in-memory waveform at
        `sample_rate`, as in `prepare_wav`)."""
        wav, length = self.prepare_wav(wav_file, sample_rate)
        encoded, encoded_len = self.forward(wav, length)
        probs = self._pooled_probs(encoded, encoded_len)[0].tolist()
        return {self.id2name[i]: probs[i] for i in range(len(self.id2name))}

    def forward_for_export(self, features: Tensor, feature_lengths: Tensor) -> Tensor:
        """log-mel [B, F, M], lengths [B] -> probs [B, C] (gigaam/model.py:287-293), pooling each utterance over its own
        encoded_len frames (all T' for a batch of one; see the class docstring)."""
        encoded, encoded_len = self.encoder(features, feature_lengths)
        return self._pooled_probs(encoded, encoded_len)

    @torch.inference_mode()
    def emotion_timeline(self, wav_file, window: float = 30.0, overlap: float = 4.0, span: float = 4.0, hop: float = 1.0,
                         spans: Optional[Sequence[Tuple[float, float]]] = None, batch_size: int = 16,
                         sample_rate: int = SAMPLE_RATE) -> EmotionTimeline:
        """Emotions over a recording of any length (INTEGRATION.md, "Emotions over time").  The encoder runs over the
        overlapping windows of `transcribe_windowed` (`longform.plan_windows`), the head's logits of every kept frame are
        stitched into one [T, C] sequence (gam_emo_frame_logits), and every span's probabilities are the softmax of its mean
        frame logits (gam_emo_spans, one call).  Spans are `span` seconds long every `hop` seconds (`longform.emotion_spans`:
        one span [0, T) when the recording is shorter, a tail span that ends at T; gaps between spans when hop > span), or the
        caller's `spans` [(start, end), ...] in seconds, each boundary rounded to a 40 ms frame and clamped to the recording.
        Times use the recording's frame shift, as `transcribe_windowed` does.  Raises ValueError before any device work for a
        span or hop that is not a positive multiple of 0.04 s, caller spans that are NaN, negative or inverted, batch_size < 1,
        the window plan's refusals and a `sample_rate` that cannot be resampled."""
        from .longform import caller_span_frames, check_caller_spans, emotion_plan_frames, emotion_spans, stitch_emo_frame_logits
        span_f, hop_f = emotion_plan_frames(span, hop)
        caller = None if spans is None else check_caller_spans(spans)
        host, N, windows, T = self._intake(wav_file, sample_rate, window, overlap, batch_size)
        fl = stitch_emo_frame_logits(self, host, windows, T, batch_size)
        plan = emotion_spans(T, span_f, hop_f) if caller is None else caller_span_frames(caller, T)
        return self._timeline(fl, plan, N, T)

    def _timeline(self, frame_logits: Tensor, plan: Sequence[Tuple[int, int]], N: int, T: int) -> EmotionTimeline:
        """One gam_emo_spans call over the device frame logits [T, C] for the spans `plan` -> the EmotionTimeline."""
        from .longform import emotion_result
        from .timestamps_utils import compute_frame_shift
        eng = self._get_engine()
        se = torch.tensor(plan, dtype=torch.int32).reshape(-1, 2).t().contiguous().to(eng.device)
        _, probs = eng.emo_spans(frame_logits, se[0], se[1], logits=False)
        return emotion_result(self.id2name, plan, probs.cpu(), frame_logits.cpu(), compute_frame_shift(N, T))

    def streaming(self, window: float = 8.0, overlap: float = 4.0, span: float = 4.0, hop: float = 1.0, batch_size: int = 64,
                  sample_rate: int = SAMPLE_RATE):
        """A `streaming.EmotionStreamServer` for live audio (INTEGRATION.md, "Emotions over time"): open streams, push chunks,
        `step()` for the spans that became final, `close()` for each stream's `emotion_timeline` with the same window, overlap,
        span and hop, bit for bit.  Raises ValueError before any device work for the window plan's refusals, batch_size < 1,
        a span or hop that is not a positive multiple of 0.04 s and a `sample_rate` that cannot be resampled."""
        from .streaming import EmotionStreamServer
        return EmotionStreamServer(self, window, overlap, span, hop, batch_size, sample_rate)
