"""Long-form driver: the caller one step above the hot path (gigaam/model.py:195-259 `transcribe_longform`).

The reference cuts a recording into speech segments with a pyannote VAD pipeline (gigaam/vad_utils.py, third party,
needs a Hugging Face snapshot) and pushes them through `forward` + `_decode` in arrival order with a DataLoader.
Here the segmentation is pluggable -- any VAD can hand over `(segments, boundaries)`; without one a small
energy-based splitter keeps every piece under the 25 s limit of the encoder -- and the segments are *length-bucketed*
before batching, so a batch pads to its own longest member instead of the recording's longest segment (padding is
pure waste on this path: the kernels mask it but still stream it)."""
from __future__ import annotations

import bisect
import math
from typing import Callable, Iterator, List, NamedTuple, Optional, Sequence, Tuple

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
        decoded = list(host[:3]) + (list(host[-3:]) if confidence else [])
        results = model._results(decoded, host[3], torch.tensor([lengths[i] for i in batch]), word_timestamps,
                                 host[4:9] if word_timestamps else None)
        for row, (text, words, conf) in enumerate(results):
            i = batch[row]
            seg_start, seg_end = boundaries[i]
            shifted = None
            if word_timestamps:
                shifted = [Word(text=w.text, start=round(w.start + seg_start, 3), end=round(w.end + seg_start, 3),
                                confidence=w.confidence) for w in words or []]
            out[i] = Segment(text=text, start=seg_start, end=seg_end, words=shifted, confidence=conf)
    return LongformTranscriptionResult(segments=[s for s in out if s is not None])


# ------------------------------------------------------------------------------------------ long-form alignment windows
FRAME_SAMPLES = 640   # one encoder frame: hop 160 x subsampling 4, for both front ends


class Window(NamedTuple):
    """One encoder window of `plan_windows`: samples [start, end) of the recording; it supplies global frames
    [keep_start, keep_end), which are its local frames shifted by start / FRAME_SAMPLES."""
    start: int
    end: int
    keep_start: int
    keep_end: int


def _frame_multiple(seconds: float, what: str) -> int:
    """seconds -> samples, refusing a value that is not a whole number of 40 ms encoder frames."""
    frames = round(float(seconds) * SAMPLE_RATE / FRAME_SAMPLES)
    if not math.isclose(frames * FRAME_SAMPLES / SAMPLE_RATE, float(seconds), rel_tol=0.0, abs_tol=1e-9):
        raise ValueError(f"{what}={seconds} s is not a multiple of {FRAME_SAMPLES / SAMPLE_RATE} s (one encoder frame)")
    return frames * FRAME_SAMPLES


def plan_windows(n_samples: int, window_s: float, overlap_s: float, length_fn: Callable[[int], int],
                 max_frames: Optional[int] = None) -> Tuple[List[Window], int]:
    """Overlapping encoder windows over a recording of `n_samples` samples, and its encoder frame count T = length_fn(N).

    W = window samples, H = (window - overlap) samples, O = overlap frames.  n = 1 window if N <= W, else
    1 + ceil((N - W) / H); window w covers samples [w H, min(w H + W, N)) and keeps global frames [c_w, c_{w+1}) with
    c_0 = 0, c_w = w H / 640 + floor(O / 2) and c_n = T.  The encoders' length recursions are additive in whole frames
    (length_fn(N) = o / 640 + length_fn(N - o) for o a multiple of 640), so local frame j of window w is global frame
    w H / 640 + j, every frame is kept exactly once, and each window keeps frames at least O / 2 from its cut ends.  A window
    whose kept range is empty (the last one, with no overlap, when it is shorter than a frame) is still listed.
    Raises ValueError for an empty recording, one that encodes to no frame, a window or overlap that is not a multiple of
    40 ms, an overlap < 0 or >= the window, or a window of more than `max_frames` encoder frames."""
    n = int(n_samples)
    if n <= 0:
        raise ValueError("empty recording")
    W = _frame_multiple(window_s, "window")
    V = _frame_multiple(overlap_s, "overlap")
    if W <= 0:
        raise ValueError(f"window={window_s} s must be positive")
    if V < 0 or V >= W:
        raise ValueError(f"overlap={overlap_s} s must be >= 0 and shorter than the window ({window_s} s)")
    if max_frames is not None and length_fn(W) > max_frames:
        raise ValueError(f"window={window_s} s encodes to {length_fn(W)} frames, more than the model's max_encoded_frames "
                         f"{max_frames}")
    T = int(length_fn(n))
    if T <= 0:
        raise ValueError(f"{n} samples encode to no frame")
    H = W - V
    count = 1 if n <= W else 1 + -(-(n - W) // H)
    cuts = [0] + [w * H // FRAME_SAMPLES + V // FRAME_SAMPLES // 2 for w in range(1, count)] + [T]
    return [Window(w * H, min(w * H + W, n), cuts[w], cuts[w + 1]) for w in range(count)], T


def window_batches(model, wav: Tensor, windows: Sequence[Window], batch_size: int) -> Iterator[Tuple[List[Window], Tensor]]:
    """Encode the windows of `wav` ([N], already in the model's dtype, on the model's device or in pinned host memory) in
    window order through `model.forward` (the varlen path), in batches of up to `batch_size` windows of one length: no
    padding, so no row depends on its neighbours.  Windows that keep no frame are skipped.  A host waveform is uploaded one
    batch at a time.  Yields (the batch's windows, encoded [nb, d, T_w])."""
    for group in window_groups(windows, batch_size, lambda w: w):
        yield group, encode_rows(model, [wav[w.start:w.end] for w in group])


def window_groups(items: Sequence, batch_size: int, window_of: Callable[[object], Window]) -> List[List]:
    """`window_batches`' batches: consecutive items whose windows have one length, up to `batch_size` of them; items whose
    window keeps no frame are left out."""
    if batch_size < 1:
        raise ValueError("batch_size must be >= 1")
    groups: List[List] = []
    length = None
    for item in items:
        w = window_of(item)
        if w.keep_end <= w.keep_start:
            continue
        if groups and len(groups[-1]) < batch_size and length == w.end - w.start:
            groups[-1].append(item)
        else:
            groups.append([item])
            length = w.end - w.start
    return groups


def encode_rows(model, rows: Sequence[Tensor]) -> Tensor:
    """Encode equal-length waveforms (in the model's dtype, all on the model's device or all on the host) as one batch through
    `model.forward` (the varlen path) -> encoded [len(rows), d, T_w].  Host rows are staged in pinned memory and uploaded
    without blocking."""
    dev = model._device
    length = rows[0].numel()
    if rows[0].device == dev:
        batch = torch.stack(list(rows))
    else:
        staged = torch.empty((len(rows), length), dtype=rows[0].dtype, pin_memory=True)
        torch.stack(list(rows), out=staged)
        batch = staged.to(dev, non_blocking=True)
    lens = torch.full((len(rows),), length, dtype=torch.int64, device=dev)
    encoded, _ = model.forward(batch, lens)
    return encoded


def stitch_ctc_log_probs(model, wav: Tensor, windows: Sequence[Window], T: int, batch_size: int = 16) -> Tensor:
    """CTC log-probs [1, T, V+1] f32 of a whole recording (wav [N] on the model's device or in pinned host memory, already in
    the model's dtype):
    the windows are encoded by `window_batches`, `model.head` (gam_ctc_log_probs) gives each batch's log-probs, and each
    window's kept rows are copied into place.  Only one batch of window log-probs is alive at a time."""
    eng = model._get_engine()
    out = torch.empty((1, T, eng.num_classes), dtype=torch.float32, device=eng.device)
    for group, encoded in window_batches(model, wav, windows, batch_size):
        lp = model.head(encoded)
        for row, w in enumerate(group):
            first = w.start // FRAME_SAMPLES
            out[0, w.keep_start:w.keep_end] = lp[row, w.keep_start - first:w.keep_end - first]
        del lp, encoded
    return out


def stitch_emo_frame_logits(model, wav: Tensor, windows: Sequence[Window], T: int, batch_size: int = 16) -> Tensor:
    """Emotion frame logits [T, C] f32 on the device of a whole recording (wav as for `stitch_ctc_log_probs`): the windows are
    encoded by `window_batches`, and one gam_emo_frame_logits launch per batch writes each window's kept frames straight into
    place.  Only one batch of encoder output is alive at a time, and no [B, T_w, C] intermediate is built."""
    from .decoding import _as_btd
    eng = model._get_engine()
    out = torch.empty((T, eng.num_classes), dtype=torch.float32, device=eng.device)
    for group, encoded in window_batches(model, wav, windows, batch_size):
        rng = torch.tensor([[w.keep_start - w.start // FRAME_SAMPLES for w in group], [w.keep_end - w.start // FRAME_SAMPLES for w in group],
                            [w.keep_start for w in group]], dtype=torch.int32).to(eng.device)
        eng.emo_frame_logits(_as_btd(encoded), rng[0], rng[1], rng[2], out)
        del encoded
    return out


def emotion_spans(T: int, span: int, hop: int) -> List[Tuple[int, int]]:
    """The planned spans [a, b) of an emotion timeline over T frames, spans of `span` frames every `hop` frames: one span
    [0, T) when T <= span; else [k hop, k hop + span) for every k >= 0 with k hop + span <= T, and a tail span [T - span, T)
    when the last of those does not end at T.  With hop <= span the spans cover [0, T); with hop > span they leave gaps of
    hop - span frames between them (the tail span may still overlap the last one)."""
    if span < 1 or hop < 1:
        raise ValueError(f"span={span} and hop={hop} frames must be >= 1")
    if T <= span:
        return [(0, T)]
    out = [(k * hop, k * hop + span) for k in range((T - span) // hop + 1)]
    if out[-1][1] != T:
        out.append((T - span, T))
    return out


def emotion_plan_frames(span: float, hop: float) -> Tuple[int, int]:
    """(span, hop) seconds -> frames; ValueError for a value that is not a positive multiple of 40 ms."""
    out = []
    for name, value in (("span", span), ("hop", hop)):
        if not (isinstance(value, (int, float)) and math.isfinite(value)):
            raise ValueError(f"{name}={value!r} s must be a finite number of seconds")
        frames = _frame_multiple(value, name) // FRAME_SAMPLES
        if frames < 1:
            raise ValueError(f"{name}={value} s must be positive")
        out.append(frames)
    return out[0], out[1]


def check_caller_spans(spans: Sequence[Tuple[float, float]]) -> List[Tuple[float, float]]:
    """Caller spans (start, end) in seconds, checked: ValueError for no spans, a NaN or negative boundary, or end < start.
    end = start is an empty span, whose row is NaN."""
    out = [(float(a), float(b)) for a, b in spans]
    if not out:
        raise ValueError("spans: no spans")
    for a, b in out:
        if math.isnan(a) or math.isnan(b) or a < 0 or b < 0:
            raise ValueError(f"spans: ({a}, {b}) has a NaN or negative boundary")
        if b < a:
            raise ValueError(f"spans: ({a}, {b}) ends before it starts")
    return out


def caller_span_frames(spans: Sequence[Tuple[float, float]], T: int) -> List[Tuple[int, int]]:
    """Checked caller spans in seconds -> frames [round(start / 0.04), round(end / 0.04)), each clamped to [0, T]."""
    step = FRAME_SAMPLES / SAMPLE_RATE

    def frame(s: float) -> int:
        return T if s >= T * step else min(max(round(s / step), 0), T)
    return [(frame(a), frame(b)) for a, b in spans]


def emotion_result(names: Sequence[str], plan: Sequence[Tuple[int, int]], probs: Tensor, frame_logits: Tensor, frame_shift: float):
    """An EmotionTimeline from host tensors: spans [a, b) in frames, their probs [S, C] and the frame logits [T, C]; times are
    the frames times `frame_shift`."""
    from .types import EmotionSpan, EmotionTimeline
    rows = probs.tolist()
    spans = [EmotionSpan(start=a * frame_shift, end=b * frame_shift, probs=dict(zip(names, row))) for (a, b), row in zip(plan, rows)]
    return EmotionTimeline(names=list(names), spans=spans, probs=probs, frame_logits=frame_logits)


def decode_windows(model, wav: Tensor, windows: Sequence[Window], T: int, batch_size: int = 16, scores: bool = False,
                   log_probs: Optional[Tensor] = None, boost: Optional[Tuple[Tensor, Tensor]] = None):
    """Greedy-decode a whole recording of T encoder frames as one utterance: `window_batches` encodes the windows, and each
    window's kept frames are decoded in window order, resuming the previous window's decoder state on the device
    (Engine.greedy_resume).  Only one batch of encoder output is alive at a time.  Returns the Engine.DecodeBuffers of the
    one stream: ids / frames [1, max_out] (global frames), counts [1] and, with `scores`, token_logp, path_logp, path_rows and
    the per-frame frame_logp / frame_rows [1, T].  max_out = Engine.hyp_width(T), so the buffers never overflow.
    `log_probs` (CTC, f32 [1, T, V+1] on the device): also filled with the stitched log-probs of `stitch_ctc_log_probs`,
    from the same encoder pass.  `boost` (RNN-T, device tables of decoding.boost_graph) steers every window's decoding, the
    graph state carried in the decoder record."""
    from .decoding import _as_btd
    eng = model._get_engine()
    index = {w: i for i, w in enumerate(windows)}
    first = [w.start // FRAME_SAMPLES for w in windows]
    ranges = torch.tensor([[w.keep_start - f for w, f in zip(windows, first)], [w.keep_end - f for w, f in zip(windows, first)], first],
                          dtype=torch.int32).to(eng.device)
    state = eng.decode_state(1)
    out = eng.decode_buffers(1, eng.hyp_width(T), T, scores=scores)
    for group, encoded in window_batches(model, wav, windows, batch_size):
        enc = _as_btd(encoded)
        for row, w in enumerate(group):
            i = index[w]
            eng.greedy_resume(enc[row:row + 1], ranges[0, i:i + 1], ranges[1, i:i + 1], ranges[2, i:i + 1], state, out, scores, boost)
        if log_probs is not None:
            lp = model.head(encoded)
            for row, w in enumerate(group):
                log_probs[0, w.keep_start:w.keep_end] = lp[row, w.keep_start - first[index[w]]:w.keep_end - first[index[w]]]
            del lp
        del enc, encoded
    return out


def segment_cuts(word_spans: Sequence[Tuple[int, int]], T: int, frame_shift: float, pause: float, max_segment: float) -> List[int]:
    """Segment boundaries of a transcribed recording of T frames, from its words' frame spans [start, end) in order:
    [c_0 = 0, c_1, ..., c_n = T], segment k covering frames [c_k, c_{k+1}).  Cuts fall only between consecutive words whose
    spans do not overlap, at the gap's middle frame (end_prev + start_next) // 2: first at every gap of at least `pause`
    seconds, then, while a segment lasts more than `max_segment` seconds, at the middle of its longest inner gap (the first
    of equal ones), until it fits or has no such gap left."""
    starts = [s for s, _ in word_spans]
    gaps = [(e, s) for (_, e), (s, _) in zip(word_spans, word_spans[1:])]     # gap i: between word i and word i + 1
    cuts = [0] + [(e + s) // 2 for e, s in gaps if s >= e and (s - e) * frame_shift >= pause] + [T]
    out = [0]
    todo = list(zip(cuts, cuts[1:]))[::-1]
    while todo:
        a, b = todo.pop()
        if (b - a) * frame_shift > max_segment:
            i0, i1 = bisect.bisect_left(starts, a), bisect.bisect_left(starts, b)     # the words of [a, b)
            inner = [(gaps[i][1] - gaps[i][0], i) for i in range(i0, i1 - 1) if gaps[i][1] >= gaps[i][0]]
            if inner:
                e, s = gaps[max(inner, key=lambda g: g[0])[1]]    # max keeps the first of equal gaps
                mid = (e + s) // 2                               # a < e <= mid <= s < b
                todo.extend([(mid, b), (a, mid)])
                continue
        out.append(b)
    return out


def windowed_segments(tokenizer, ids: Sequence[int], frames: Sequence[int], cuts: Sequence[int], frame_shift: float, duration: float,
                      words: Optional[Sequence[Word]], word_starts: Sequence[int], frame_logp=None, frame_rows=None) -> List[Segment]:
    """One Segment per range [cuts[k], cuts[k+1]) of `segment_cuts`: the tokens whose frames fall inside it (text =
    tokenizer.decode of them), the words that start inside it (None when `words` is None), start / end = the cut frames
    times the frame shift (the last segment ends at `duration`) and, when frame_logp / frame_rows (per-frame sums of l and
    decision rows) are given, confidence = exp(sum of l over its frames / their rows), NaN without rows."""
    from .timestamps_utils import path_confidence
    out: List[Segment] = []
    n = len(cuts) - 1
    for k in range(n):
        a, b = cuts[k], cuts[k + 1]
        t0, t1 = bisect.bisect_left(frames, a), bisect.bisect_left(frames, b)
        w0, w1 = bisect.bisect_left(word_starts, a), bisect.bisect_left(word_starts, b)
        conf = None
        if frame_logp is not None:
            conf = path_confidence(float(frame_logp[a:b].sum()), int(frame_rows[a:b].sum()))
        out.append(Segment(text=tokenizer.decode(list(ids[t0:t1])), start=a * frame_shift, end=duration if k == n - 1 else b * frame_shift,
                           words=None if words is None else list(words[w0:w1]), confidence=conf))
    return out


def check_segmenting(pause: float, max_segment: float) -> None:
    """`segment_cuts`' settings: ValueError for pause < 0 and max_segment <= 0 (NaN fails both)."""
    if not pause >= 0:
        raise ValueError(f"pause={pause} s must be >= 0")
    if not max_segment > 0:
        raise ValueError(f"max_segment={max_segment} s must be positive")


def windowed_result(model, ids: List[int], frames: List[int], token_logp: Optional[List[float]], frame_logp, frame_rows, N: int,
                    T: int, word_timestamps: bool, pause: float, max_segment: float) -> LongformTranscriptionResult:
    """The result of a recording of N samples and T frames decoded as one utterance: its token ids and global frames, and
    with scores the tokens' log-probs and the per-frame sums of `decode_windows` (None without them).  Words are grouped
    on the device, segments cut by `segment_cuts` and built by `windowed_segments`.  `transcribe_windowed` and a closed
    stream both end here, so the same decoding gives them the same result."""
    from .timestamps_utils import compute_frame_shift, words_from_device
    eng, tok = model._get_engine(), model.decoding.tokenizer
    rows = torch.tensor([ids or [0], frames or [0]], dtype=torch.int32).pin_memory().to(eng.device, non_blocking=True)
    count = torch.full((1,), len(ids), dtype=torch.int32, device=eng.device)
    ws, we, wf, wn, k = (t[0].cpu().tolist() for t in eng.group_words(rows[:1], rows[1:], count, model._word_flags()))
    shift = compute_frame_shift(N, T)
    words = words_from_device(tok, ids, ws[:k], we[:k], wf[:k], wn[:k], shift, token_logp)
    cuts = segment_cuts(list(zip(ws[:k], we[:k])), T, shift, pause, max_segment)
    return LongformTranscriptionResult(segments=windowed_segments(tok, ids, frames, cuts, shift, N / SAMPLE_RATE,
                                                                   words if word_timestamps else None, ws[:k], frame_logp,
                                                                   frame_rows))


def line_segments(lines: Sequence[str], ranges: Sequence[Tuple[int, int]], frames: Sequence[int], token_logp: Sequence[float],
                  frame_shift: float, viterbi_logp: float, words: Optional[Sequence[Word]] = None,
                  word_first: Optional[Sequence[int]] = None, skipped: Sequence[int] = ()) -> List[Segment]:
    """One Segment per line of an aligned text.  ranges[i] = line i's token range [a, b) in the aligned sequence, frames /
    token_logp the alignment's per-token outputs, words (None: no word timestamps) the words of the whole sequence with
    word_first their first token.  A line spans the frames of its first and last token (its first word's start and its
    last word's end) and has confidence exp(mean token log-prob); a line without tokens, or one of the `skipped` lines,
    starts and ends where the line before it ended (0.0 first), has no words and confidence NaN.  Without a path (a
    Viterbi score that is not finite) every line has no words, NaN times and confidence 0.0."""
    if not math.isfinite(viterbi_logp):
        return [Segment(text=t, start=math.nan, end=math.nan, words=None if words is None else [], confidence=0.0) for t in lines]
    from .timestamps_utils import mean_logp_confidence
    starts = [a for a, _ in ranges]
    by_line: List[List[Word]] = [[] for _ in lines]
    for w, f in zip(words or [], word_first or []):
        by_line[bisect.bisect_right(starts, f) - 1].append(w)
    out: List[Segment] = []
    prev_end = 0.0
    skipped = set(skipped)
    for i, (text, (a, b)) in enumerate(zip(lines, ranges)):
        seg_words = None if words is None else by_line[i]
        if a == b or i in skipped:
            out.append(Segment(text=text, start=prev_end, end=prev_end, words=seg_words, confidence=math.nan))
            continue
        start, end = frames[a] * frame_shift, (frames[b - 1] + 1) * frame_shift
        out.append(Segment(text=text, start=start, end=end, words=seg_words, confidence=mean_logp_confidence(token_logp[a:b])))
        prev_end = end
    return out


def line_edges(ranges: Sequence[Tuple[int, int]], U: int) -> List[int]:
    """gam_ctc_align_long_gaps' line_edges of a text of U tokens whose lines have token ranges [a, b): bit 0 on the first
    token of every line, bit 1 on its last.  Empty lines have no tokens and set no bits."""
    edges = [0] * U
    for a, b in ranges:
        if b > a:
            edges[a] |= 1
            edges[b - 1] |= 2
    return edges


def unmatched_intervals(flags: Tensor, frame_shift: float) -> List[Tuple[float, float]]:
    """Maximal runs of unmatched frames (flags [T], nonzero = unmatched) -> (start, end) seconds, end exclusive."""
    f = torch.cat([torch.zeros(1, dtype=torch.int8), (flags.reshape(-1).cpu() != 0).to(torch.int8), torch.zeros(1, dtype=torch.int8)])
    d = torch.diff(f)
    starts = torch.nonzero(d == 1).reshape(-1).tolist()
    ends = torch.nonzero(d == -1).reshape(-1).tolist()
    return [(a * frame_shift, b * frame_shift) for a, b in zip(starts, ends)]


def skip_edges(edges: Sequence[int]) -> List[Tuple[int, int]]:
    """gam_ctc_align_long_skips' skip edges of a text with these line_edges, one per line end in order: (e_i, x_i), x_i the
    blank just after the i-th token with bit 1 set and e_i = x_{i-1} (0 for the first).  The edge jumps n_i = (x_i - e_i) / 2
    tokens: the line and any joining token before it."""
    out, e = [], 0
    for j, f in enumerate(edges):
        if f & 2:
            out.append((e, 2 * (j + 1)))
            e = 2 * (j + 1)
    return out


def skipped_lines(ranges: Sequence[Tuple[int, int]], frames: Sequence[int]) -> List[int]:
    """The lines a path with skips jumped, in ascending order: the lines with tokens whose last token has frame -1.  Only
    meaningful for an alignment that has a path."""
    return [i for i, (a, b) in enumerate(ranges) if b > a and frames[b - 1] < 0]
