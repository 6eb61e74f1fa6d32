"""Long-form driver: the caller one step above the hot path (gigaam/model.py:195-259 `transcribe_longform`).

The reference cuts a recording into speech segments with a pyannote VAD pipeline (gigaam/vad_utils.py, third party,
needs a Hugging Face snapshot) and pushes them through `forward` + `_decode` in arrival order with a DataLoader.
Here the segmentation is pluggable -- any VAD can hand over `(segments, boundaries)`; without one a small
energy-based splitter keeps every piece under the 25 s limit of the encoder -- and the segments are *length-bucketed*
before batching, so a batch pads to its own longest member instead of the recording's longest segment (padding is
pure waste on this path: the kernels mask it but still stream it)."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch
from torch import Tensor

from .preprocess import SAMPLE_RATE
from .types import LongformTranscriptionResult, Segment, Word


def plan_batches(lengths: Sequence[int], batch_size: int) -> List[List[int]]:
    """Indices of the segments of every batch: longest first, neighbours in length share a batch."""
    if batch_size < 1:
        raise ValueError("batch_size must be >= 1")
    order = sorted(range(len(lengths)), key=lambda i: (-int(lengths[i]), i))
    return [order[i:i + batch_size] for i in range(0, len(order), batch_size)]


def padding_waste(lengths: Sequence[int], batches: List[List[int]]) -> float:
    """Fraction of padded samples over all batches (0 = none)."""
    total = sum(max(int(lengths[i]) for i in b) * len(b) for b in batches if b)
    real = sum(int(lengths[i]) for b in batches for i in b)
    return 0.0 if total == 0 else 1.0 - real / total


def split_on_energy(wav: Tensor, sample_rate: int = SAMPLE_RATE, max_duration: float = 22.0, min_duration: float = 15.0,
                    frame: float = 0.02) -> Tuple[List[Tensor], List[Tuple[float, float]]]:
    """Fallback segmentation when no VAD is plugged in: cut at the quietest 20 ms frame between `min_duration` and
    `max_duration` seconds after the previous cut.  Returns (segments, boundaries in seconds) like
    gigaam.vad_utils.segment_audio_file."""
    wav = wav.reshape(-1).float().cpu()
    n = wav.numel()
    hop = max(1, int(frame * sample_rate))
    lo, hi = int(min_duration * sample_rate), int(max_duration * sample_rate)
    segments: List[Tensor] = []
    bounds: List[Tuple[float, float]] = []
    start = 0
    while n - start > hi:
        window = wav[start + lo: start + hi]
        usable = window.numel() // hop * hop
        energy = window[:usable].reshape(-1, hop).pow(2).mean(dim=1)
        cut = start + lo + int(energy.argmin()) * hop + hop // 2
        segments.append(wav[start:cut])
        bounds.append((start / sample_rate, cut / sample_rate))
        start = cut
    if n - start > 0:
        segments.append(wav[start:])
        bounds.append((start / sample_rate, n / sample_rate))
    return segments, bounds


def transcribe_segments(model, segments: Sequence[Tensor], boundaries: Sequence[Tuple[float, float]], word_timestamps: bool = False,
                        batch_size: int = 16, confidence: bool = False) -> LongformTranscriptionResult:
    """Batched inference over pre-cut segments, results in the original order (gigaam/model.py:222-259).  The
    length-bucketed batches go through `pipeline.BatchPipeline`: the upload of batch i+1 and the read-back of batch i-1
    overlap the kernels of batch i, recurring shapes replay a CUDA graph, and word grouping stays on the device."""
    from .pipeline import BatchPipeline
    from .timestamps_utils import path_confidence
    if len(segments) != len(boundaries):
        raise ValueError("segments and boundaries differ in length")
    if not segments:
        return LongformTranscriptionResult(segments=[])
    lengths = [int(s.numel()) for s in segments]
    out: List[Optional[Segment]] = [None] * len(segments)
    dtype = model._dtype
    batches = plan_batches(lengths, batch_size)

    def host_batches():
        for batch in batches:
            longest = max(lengths[i] for i in batch)
            wav = torch.zeros((len(batch), longest), dtype=torch.float32)
            for row, i in enumerate(batch):
                # same fp16 rounding of the waveform as gigaam/model.py:239 (`.to(self._dtype)`)
                wav[row, : lengths[i]] = segments[i].reshape(-1).float().cpu().to(dtype).float()
            yield wav.pin_memory(), torch.tensor([lengths[i] for i in batch], dtype=torch.int64)

    # a graph per distinct (batch, padded length) only pays off when shapes recur; VAD segments rarely do
    shapes = [(len(b), max(lengths[i] for i in b)) for b in batches]
    pipe = BatchPipeline(model, use_graph=len(set(shapes)) < len(shapes), with_words=word_timestamps, with_scores=confidence)
    for batch, host in zip(batches, pipe.run_raw(host_batches())):
        ids, frames, counts, enc_len = host[:4]
        token_logp, path_logp, path_rows = host[-3:] if confidence else (None, None, None)
        if word_timestamps:
            wav_lens = torch.tensor([lengths[i] for i in batch])
            results = model._words_from_records(ids, counts, enc_len, wav_lens, list(host[4:9]), token_logp)
        else:
            results = [(t, None) for t, _, _ in model.decoding.to_hypotheses(ids, frames, counts)]
        for row, (text, words) in enumerate(results):
            i = batch[row]
            seg_start, seg_end = boundaries[i]
            shifted = None
            if word_timestamps:
                shifted = [Word(text=w.text, start=round(w.start + seg_start, 3), end=round(w.end + seg_start, 3),
                                confidence=w.confidence) for w in words or []]
            conf = path_confidence(path_logp[row], path_rows[row]) if confidence else None
            out[i] = Segment(text=text, start=seg_start, end=seg_end, words=shifted, confidence=conf)
    return LongformTranscriptionResult(segments=[s for s in out if s is not None])
