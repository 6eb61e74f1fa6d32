"""Result records of the public API.  Field names, defaults, `str()` and the long-form helpers follow the reference's
result classes (gigaam/types.py:16-67) because callers and tests touch them (`result.words is None`, `str(result) == text`,
`for segment in result`); the implementation is a small slotted record base instead of dataclasses -- a long-form
transcript holds one `Word` per spoken word, and slotted objects are a third of the size."""
from __future__ import annotations

from typing import Any, Dict, Iterator, List, Optional, Tuple

import torch


class _Record:
    """Positional / keyword construction over `_fields`, value equality and a readable repr.  Fields in `_quiet` are
    left out of the repr while they hold their default (None), so records without them print as before."""
    __slots__ = ()
    _fields: Tuple[str, ...] = ()
    _defaults: Dict[str, Any] = {}
    _quiet: Tuple[str, ...] = ()

    def __init__(self, *args: Any, **kwargs: Any) -> None:
        if len(args) > len(self._fields):
            raise TypeError(f"{type(self).__name__} takes at most {len(self._fields)} positional arguments")
        given = dict(zip(self._fields, args))
        for key, value in kwargs.items():
            if key not in self._fields:
                raise TypeError(f"{type(self).__name__} has no field {key!r}")
            if key in given:
                raise TypeError(f"{type(self).__name__} got {key!r} twice")
            given[key] = value
        for name in self._fields:
            if name in given:
                setattr(self, name, given[name])
            elif name in self._defaults:
                setattr(self, name, self._defaults[name])
            else:
                raise TypeError(f"{type(self).__name__} missing required field {name!r}")

    def __eq__(self, other: object) -> bool:
        return type(other) is type(self) and all(getattr(self, n) == getattr(other, n) for n in self._fields)

    def __repr__(self) -> str:
        shown = (n for n in self._fields if n not in self._quiet or getattr(self, n) is not None)
        return f"{type(self).__name__}({', '.join(f'{n}={getattr(self, n)!r}' for n in shown)})"


class Word(_Record):
    """One word with its start / end time in seconds.  `confidence` (transcribe(..., confidence=True)) is
    exp(mean log-probability of the word's tokens)."""
    __slots__ = _fields = ("text", "start", "end", "confidence")
    _defaults = {"confidence": None}
    _quiet = ("confidence",)
    text: str
    start: float
    end: float
    confidence: Optional[float]


class TranscriptionResult(_Record):
    """`transcribe()` result: `words` stays None unless word timestamps were requested.  `confidence`
    (confidence=True) is exp(path log-probability / decision rows) of the greedy path, blank decisions included."""
    __slots__ = _fields = ("text", "words", "confidence")
    _defaults = {"words": None, "confidence": None}
    _quiet = ("confidence",)
    text: str
    words: Optional[List[Word]]
    confidence: Optional[float]

    def __str__(self) -> str:
        return self.text


class Segment(_Record):
    """One speech segment of a long recording (times in seconds from the start of the recording).  `confidence` as
    in TranscriptionResult, for the segment."""
    __slots__ = _fields = ("text", "start", "end", "words", "confidence")
    _defaults = {"words": None, "confidence": None}
    _quiet = ("confidence",)
    text: str
    start: float
    end: float
    words: Optional[List[Word]]
    confidence: Optional[float]


class Alignment(_Record):
    """`align()` result: `text` is the normalised text that was aligned (characters a charwise vocabulary lacks are gone),
    `words` its words with times and confidences from the Viterbi path (None without word timestamps), `log_likelihood`
    the forward score log p(text | audio) summed over all paths, and `confidence` = exp(Viterbi path score / path edges)."""
    __slots__ = _fields = ("text", "words", "log_likelihood", "confidence")
    _defaults = {"words": None}
    text: str
    words: Optional[List[Word]]
    log_likelihood: float
    confidence: float

    def __str__(self) -> str:
        return self.text


class Detection(_Record):
    """One keyword detection of `spot()` / `spot_batch()`: `keyword` (its normalised text, or the decoded ids) and its index in
    the list asked for, start / end in seconds (end exclusive: one frame after the first frame of the keyword's last token),
    `score` = log p(keyword path) - log p(greedy path) over the same frames (<= 0) and `confidence` = exp(score / tokens), the
    per-token likelihood ratio to the greedy decoder, 1.0 exactly where greedy decoding writes the keyword."""
    __slots__ = _fields = ("keyword", "keyword_index", "start", "end", "score", "confidence")
    keyword: str
    keyword_index: int
    start: float
    end: float
    score: float
    confidence: float


class LongformAlignment(_Record):
    """`align_longform()` result: one `Segment` per input line, in order (its normalised text, the start of its first token's
    frame and the end of its last, its words, and `confidence` = exp(mean log-probability of its tokens)), plus the
    whole recording's `log_likelihood` (forward score) and `confidence` = exp(Viterbi path score / frames), as in
    `Alignment`.  With `gap_threshold`, `unmatched` holds the (start, end) seconds of every maximal run of frames the text
    left unaligned, `log_likelihood` is the forward score of the graph with gaps and `confidence` = exp((Viterbi score -
    score of the unmatched frames) / matched frames) (NaN when no frame is matched); without it `unmatched` is None.
    With `skip_threshold`, `skipped` holds the ascending indices of the lines the alignment skipped (their segments have
    no time span and no words), `log_likelihood` is the forward score of the graph with skips and the skip edges' scores
    are also taken out of `confidence`; without it `skipped` is None."""
    __slots__ = _fields = ("segments", "log_likelihood", "confidence", "unmatched", "skipped")
    _defaults = {"unmatched": None, "skipped": None}
    _quiet = ("unmatched", "skipped")
    segments: List[Segment]
    log_likelihood: float
    confidence: float
    unmatched: Optional[List[Tuple[float, float]]]
    skipped: Optional[List[int]]

    @property
    def text(self) -> str:
        return " ".join(seg.text for seg in self.segments if seg.text)

    @property
    def words(self) -> List[Word]:
        return [word for seg in self.segments for word in (seg.words or [])]

    def __str__(self) -> str:
        return self.text

    def __len__(self) -> int:
        return len(self.segments)

    def __iter__(self) -> Iterator[Segment]:
        return iter(self.segments)


class LongformTranscriptionResult(_Record):
    """`transcribe_longform()` result: the segments in recording order."""
    __slots__ = _fields = ("segments",)
    segments: List[Segment]

    @property
    def text(self) -> str:
        return " ".join(seg.text for seg in self.segments)

    @property
    def words(self) -> List[Word]:
        return [word for seg in self.segments for word in (seg.words or [])]

    @property
    def has_word_timestamps(self) -> bool:
        return bool(self.segments) and self.segments[0].words is not None

    def __str__(self) -> str:
        return self.text

    def __len__(self) -> int:
        return len(self.segments)

    def __iter__(self) -> Iterator[Segment]:
        return iter(self.segments)


class StreamUpdate(_Record):
    """What one `StreamServer.step()` changed in a live stream.  `new_tokens` are the token ids committed by the step and
    `new_text` their text: concatenating a stream's `new_text` in order gives the tokenizer's decoding of every committed
    token.  `tentative_text` decodes the frames after the committed ones in the newest encoded window; it is replaced at the
    next step.  `committed_until` is the end of the committed frames in seconds at the nominal 0.04 s per frame.
    `detections` are the keyword detections made final by the step, `pending` the provisional ones (at most one per keyword),
    which a better overlapping candidate may still replace; their times use the nominal frame step too.
    With hotwords, `new_tokens` are the tokens released by the step, the hotwords already spliced in: every token at a frame
    before the release frame R, where no later detection can change the output.  `committed_until` is R, which never
    decreases and stops short of the decoded frames while a hotword path may still end there.  `tentative_text` decodes the
    held greedy tokens (frames from R on, no splices) followed by the newest window's tentative tokens."""
    __slots__ = _fields = ("stream", "new_tokens", "new_text", "tentative_text", "committed_until", "detections", "pending")
    stream: int
    new_tokens: List[int]
    new_text: str
    tentative_text: str
    committed_until: float
    detections: List[Detection]
    pending: List[Detection]


class StreamResult(_Record):
    """`StreamServer.close()` result: the stream's `transcript`, the `LongformTranscriptionResult` that `transcribe_windowed`
    gives for the same recording and settings, and its keyword `detections` as `spot` gives them (None without keywords)."""
    __slots__ = _fields = ("transcript", "detections")
    transcript: LongformTranscriptionResult
    detections: Optional[List[Detection]]

    def __str__(self) -> str:
        return str(self.transcript)


class EmotionSpan(_Record):
    """One span of an emotion timeline: `start` / `end` in seconds of the recording (end exclusive) and `probs`, {class name:
    probability} of the softmax of the span's mean frame logits, which is the head applied to the mean of its frames."""
    __slots__ = _fields = ("start", "end", "probs")
    start: float
    end: float
    probs: Dict[str, float]


class EmotionTimeline(_Record):
    """`GigaAMEmo.emotion_timeline()` result (INTEGRATION.md, "Emotions over time"): the class `names`, one `EmotionSpan` per
    span in order, `probs` (host f32 [S, C], the spans' probabilities in class order) and `frame_logits` (host f32 [T, C], the
    head's logits of every 40 ms encoder frame, W f_t + b).  The softmax of the mean of frame_logits over any range of frames
    is that range's emotion, so callers can pool spans of their own.  Two timelines are equal when their names and spans are,
    and their tensors have the same bits."""
    __slots__ = _fields = ("names", "spans", "probs", "frame_logits")
    names: List[str]
    spans: List[EmotionSpan]
    probs: torch.Tensor
    frame_logits: torch.Tensor

    def __eq__(self, other: object) -> bool:
        def bits(t: torch.Tensor) -> torch.Tensor:
            return t.contiguous().view(torch.int32)
        return (type(other) is type(self) and self.names == other.names and repr(self.spans) == repr(other.spans)
                and all(a.shape == b.shape and torch.equal(bits(a), bits(b))
                        for a, b in ((self.probs, other.probs), (self.frame_logits, other.frame_logits))))

    def __len__(self) -> int:
        return len(self.spans)

    def __iter__(self) -> Iterator[EmotionSpan]:
        return iter(self.spans)


class EmotionStreamUpdate(_Record):
    """What one `EmotionStreamServer.step()` added to a live stream: `new_spans`, the planned spans whose last frame became
    final in this step (times at the nominal 0.04 s per frame), and `final_until`, the end of the final frames in seconds.
    Concatenating a stream's `new_spans` gives its timeline's spans without the tail span, which only `close` adds."""
    __slots__ = _fields = ("stream", "new_spans", "final_until")
    stream: int
    new_spans: List[EmotionSpan]
    final_until: float
