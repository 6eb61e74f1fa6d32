"""Live streams (INTEGRATION.md §7i): many recordings that arrive a chunk at a time, transcribed and searched for keywords
while they are spoken.

Each stream is cut into `longform.plan_windows`' windows.  Window w of a stream is *ready* once the stream holds more than
w H + W samples (W the window, H = W - V the hop): it is then never the last window of the plan, whatever length the
stream reaches, so its samples and kept frames are final.  `StreamServer.step()` encodes every ready window of every
stream in batches of equal-length windows (`longform.window_groups` / `encode_rows`, no padding) and decodes each batch's
kept frames by rounds: one `Engine.greedy_resume` launch decodes the r-th window of every stream in the batch, with the
streams' decoder records gathered from a device pool and scattered back.  CTC log-probs of the same batch feed
`Engine.ctc_spot_resume` over the same frames.  `close()` encodes what is left, the last window included, and builds the
result with `transcribe_windowed`'s and `spot`'s code, so a closed stream gets their output bit for bit.

A server made with another `sample_rate` takes pushes at that rate.  Each step first resamples, in one `gam_resample`
launch for all streams (the span form, include/gigaam_b200.h), every 16 kHz output whose taps have all been pushed
(`resample_ready`), and appends it to the stream's 16 kHz samples; `close()` adds the tail with the end's zero padding.
Every 16 kHz sample is thus the one-shot resampler's, and the windows see the samples `transcribe_windowed(recording,
sample_rate=...)` sees.  The host keeps the raw samples that the outputs still pending can need.

With hotwords (CTC models), each decode round also spots the hotwords in a spot pool of their own and runs one
`Engine.ctc_bias_resume` launch over the round's streams: it releases the tokens whose hotword decisions are final (frames
before the release frame R) and the stream holds the rest for the next round: the log-prob rows [R, C) and the undecided
detections on the device, the greedy tokens and per-frame sums of that span on the host.  `close()` makes the last call with
finish, so a closed stream equals `transcribe_windowed(..., hotwords=...)`.

Device memory does not grow with a stream's duration: a stream owns one decoder record, one spot record per keyword and
per hotword, and with hotwords the held rows [R, C), bounded by the oldest live hotword path; every step's outputs are
step-local.  The host keeps each stream's unencoded samples, its token ids, frames, token
log-probs, per-frame sums and detections for `close`.  One caller drives a server; it is not thread-safe.

`EmotionStreamServer` (GigaAM-Emo) shares the windows, the sample buffers (`_Audio`) and the resampling stage
(`resample_streams`): each step writes the emotion head's logits of the ready windows' kept frames next to each stream's
held frames and scores the planned spans that became final; `close()` returns `emotion_timeline`'s result bit for bit."""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
from torch import Tensor

from .decoding import _as_btd
from .longform import (FRAME_SAMPLES, Window, _frame_multiple, check_segmenting, encode_rows, plan_windows, window_groups,
                       windowed_result)
from .preprocess import SAMPLE_RATE, resample_ratio, resampled_length
from .timestamps_utils import compute_frame_shift, token_flag_table
from .types import Detection, EmotionSpan, EmotionStreamUpdate, EmotionTimeline, StreamResult, StreamUpdate

FRAME_SECONDS = FRAME_SAMPLES / SAMPLE_RATE   # the nominal 40 ms frame step of updates


def ready_count(n_samples: int, W: int, V: int) -> int:
    """How many windows of a stream holding n_samples samples are ready: window w is once n_samples > w H + W, H = W - V.
    For N >= n_samples this is at most len(plan_windows(N)) - 1, so a ready window is never a plan's last one."""
    return 0 if n_samples <= W else (n_samples - W - 1) // (W - V) + 1


def resample_ready(n_raw: int, o: int, n: int, w: int) -> int:
    """How many 16 kHz outputs of a stream holding n_raw samples at the ratio o / n are final: output j n + p needs input
    samples up to j o + o + w - 1, so the outputs of every j < (n_raw - w) / o are.  They never exceed ceil(n N / o) for
    N >= n_raw, the length of any recording the stream can become."""
    return n * max(0, (n_raw - w) // o)


def ready_window(w: int, W: int, V: int) -> Window:
    """Window w of every plan in which it is not the last one (`longform.plan_windows`' rule): samples [w H, w H + W) and kept
    frames [c_w, c_{w+1}), c_0 = 0 and c_w = w H / 640 + floor(O / 2), O = V / 640."""
    H, half = W - V, V // FRAME_SAMPLES // 2
    return Window(w * H, w * H + W, 0 if w == 0 else w * H // FRAME_SAMPLES + half, (w + 1) * H // FRAME_SAMPLES + half)


class TextFeed:
    """A stream's committed text, a step at a time: `push(all_ids, n_new)` returns the text of the n_new ids just appended,
    so that the concatenated returns equal tokenizer.decode(all_ids).  Only the ids from the last word opener on (a token in
    `openers`: a space, or a SentencePiece piece starting with U+2581) are decoded again, which needs decoding to append
    text past a word opener (decode(ids + more) extends decode(ids) when ids starts with one)."""

    def __init__(self, tokenizer, openers):
        self.tokenizer = tokenizer
        self.openers = openers
        self.anchor = 0        # index of the last word opener (0 before the first)
        self.tail = ""         # decode(ids[anchor:]) as emitted

    def push(self, ids: Sequence[int], n_new: int) -> str:
        if n_new == 0:
            return ""
        text = self.tokenizer.decode(list(ids[self.anchor:]))
        new = text[len(self.tail):]
        self.tail = text
        for i in range(len(ids) - 1, max(self.anchor, len(ids) - n_new) - 1, -1):
            if ids[i] in self.openers:
                self.anchor = i
                self.tail = self.tokenizer.decode(list(ids[i:]))
                break
        return new


class _Audio:
    """The samples of one open stream: its 16 kHz samples that a window not yet encoded may need and, for a server at another
    rate, the raw samples that pending 16 kHz outputs can need."""

    def __init__(self, dtype: torch.dtype):
        self.n = 0                       # samples pushed
        self.chunks: List[Tensor] = []   # pushed since the last consolidation
        self.buf = torch.zeros(0, dtype=dtype)   # samples [buf_start, n) that a window not yet encoded may need
        self.buf_start = 0
        self.windows: List[Window] = []  # the windows handed to the encoder, in order
        # resampling streams: raw samples [raw_start, raw_n) that pending 16 kHz outputs can need, and the outputs made so far
        self.raw = torch.zeros(0, dtype=torch.float32)
        self.raw_chunks: List[Tensor] = []
        self.raw_start = self.raw_n = self.out_n = 0

    def append(self, chunk, resampling: bool, dtype: torch.dtype) -> None:
        """Append pushed samples: kept as float32 raw samples when `resampling`, else rounded to `dtype` as `prepare_wav` does."""
        x = torch.as_tensor(chunk, dtype=torch.float32).detach().reshape(-1).cpu()
        if resampling:
            if x.numel():
                self.raw_chunks.append(x)
                self.raw_n += x.numel()
            return
        x = x.to(dtype)
        if x.numel():
            self.chunks.append(x)
            self.n += x.numel()

    def samples(self, start: int, end: int) -> Tensor:
        if self.chunks:
            self.buf = torch.cat([self.buf] + self.chunks)
            self.chunks = []
        return self.buf[start - self.buf_start:end - self.buf_start]

    def trim(self, keep_from: int) -> None:
        """Drop the samples before `keep_from` (the next window's first sample)."""
        self.samples(keep_from, keep_from)
        cut = keep_from - self.buf_start
        if cut > 0:
            self.buf = self.buf[cut:].clone()
            self.buf_start = keep_from


def resample_streams(eng, sample_rate: int, ratio: Tuple[int, int, int], dtype: torch.dtype, streams: Sequence[_Audio],
                     final: bool) -> None:
    """Resample, in one launch, each stream's 16 kHz outputs that are final (all of them when `final`: the end of the
    recording is known), append them to its 16 kHz samples (rounded to `dtype`) and drop the raw samples no pending output
    needs.  `ratio` = (o, n, w) of preprocess.resample_ratio(sample_rate)."""
    o, n, w = ratio
    rows = []
    for s in streams:
        target = resampled_length(s.raw_n, sample_rate) if final else resample_ready(s.raw_n, o, n, w)
        if target > s.out_n:
            if s.raw_chunks:
                s.raw = torch.cat([s.raw] + s.raw_chunks)
                s.raw_chunks = []
            rows.append((s, target))
    if not rows:
        return
    x = torch.zeros((len(rows), max(1, max(s.raw.numel() for s, _ in rows))), dtype=torch.float32)
    for r, (s, _) in enumerate(rows):
        x[r, :s.raw.numel()] = s.raw
    spans = torch.tensor([[s.raw_start for s, _ in rows], [s.raw_n for s, _ in rows], [s.out_n for s, _ in rows],
                          [t for _, t in rows]], dtype=torch.int64)
    y = torch.empty((len(rows), max(t - s.out_n for s, t in rows)), dtype=torch.float32, device=eng.device)
    y = eng.resample_spans(x.to(eng.device), spans, sample_rate, y).cpu()
    for r, (s, target) in enumerate(rows):
        cnt = target - s.out_n
        s.chunks.append(y[r, :cnt].to(dtype))
        s.n += cnt
        s.out_n = target
        keep = min(max(s.raw_start, target // n * o - w), s.raw_n)   # the first tap of the next pending output
        s.raw = s.raw[keep - s.raw_start:].clone()
        s.raw_start = keep


class _Stream(_Audio):
    """Host side of one open stream."""

    def __init__(self, sid: int, slot: int, feed: TextFeed, K: int, dtype: torch.dtype):
        super().__init__(dtype)
        self.id, self.slot, self.feed = sid, slot, feed
        self.committed = 0               # frames decoded for good
        self.ids: List[int] = []
        self.frames: List[int] = []
        self.token_logp: List[float] = []
        self.frame_logp: List[np.ndarray] = []
        self.frame_rows: List[np.ndarray] = []
        self.dets: List[List[Tuple[int, int, float]]] = [[] for _ in range(K)]
        self.pending: List[Optional[Tuple[int, int, float]]] = [None] * K
        self.tentative: List[int] = []
        # hotwords: the span [hw_base, C) not yet released -- its rows and its undecided hotword detections on the device
        # (hw_det: start, end and score bits as i32 [D, 3, K], and the count per hotword [K]), its greedy tokens and
        # per-frame sums on the host; hw_left: the span starts on a word boundary
        self.hw_rows: Optional[Tensor] = None
        self.hw_det: Optional[Tuple[Tensor, Tensor]] = None
        self.hw_base = 0
        self.hw_left = True
        self.hw_ids = np.zeros(0, np.int32)
        self.hw_frames = np.zeros(0, np.int32)
        self.hw_logp = np.zeros(0, np.float32)
        self.hw_flp = np.zeros(0, np.float64)


class StreamServer:
    """Transcribe live audio streams, and spot keywords in them, with one encoder batch per step across all of them
    (INTEGRATION.md §7i).  Made by `GigaAMASR.streaming(...)`:

        srv = model.streaming(window=8.0, overlap=4.0, batch_size=64)
        a = srv.open()
        srv.push(a, chunk)              # host samples, any length
        for u in srv.step():            # a StreamUpdate for every stream that changed
            ...
        res = srv.close(a, word_timestamps=True)

    A closed stream's result is `transcribe_windowed(recording, word_timestamps, confidence, window, overlap, pause=pause,
    max_segment=max_segment)` (with the server's `boost` and `boost_weight`) and, with keywords, `spot(recording, keywords,
    threshold, window, overlap)`, bit for bit.  `boost`: the tables of a boost graph (GigaAMASR._boost_tables, moved to the
    device with the first stream) that steer every stream's decoding, committed and tentative.  `sample_rate`: the rate of the
    pushed samples; a closed stream's result is then `transcribe_windowed(recording, sample_rate=sample_rate, ...)`'s.
    `hotwords` / `hotword_threshold` (CTC models only): checked as `transcribe` checks them; a closed stream's result is then
    `transcribe_windowed(recording, hotwords=hotwords, hotword_threshold=hotword_threshold, ...)`'s, and updates commit text
    with the hotwords spliced in once no later detection can change it (INTEGRATION.md §7i)."""

    def __init__(self, model, window: float = 8.0, overlap: float = 4.0, batch_size: int = 64, confidence: bool = False,
                 keywords: Optional[Sequence[Union[str, Sequence[int]]]] = None, threshold: float = 0.5,
                 boost: Optional[Tuple[Tensor, Tensor]] = None, sample_rate: int = SAMPLE_RATE,
                 hotwords: Optional[Sequence[Union[str, Sequence[int]]]] = None, hotword_threshold: float = 0.5):
        self.sample_rate = sample_rate
        self._ratio = None if sample_rate == SAMPLE_RATE else resample_ratio(sample_rate)
        self.W = _frame_multiple(window, "window")
        self.V = _frame_multiple(overlap, "overlap")
        plan_windows(max(self.W, 1), window, overlap, model._encoded_length, model._max_frames)   # the window plan's refusals
        if batch_size < 1:
            raise ValueError("batch_size must be >= 1")
        self.names: List[str] = []
        self.kw_ids: List[List[int]] = []
        if keywords is not None:
            model._needs_head(False, "keywords in streams need a CTC head: an RNN-T model has no per-frame posteriors without "
                                     "its [T, U + 1] lattice; use a *_ctc model")
            self.names, self.kw_ids = model._keyword_ids(keywords, threshold)
        self.hw_ids: List[List[int]] = [] if hotwords is None else model._hotword_ids(hotwords, hotword_threshold, "streaming")
        self.hotword_threshold = hotword_threshold
        self.model, self.window, self.overlap = model, window, overlap
        self.batch_size, self.confidence, self.threshold = int(batch_size), bool(confidence), threshold
        self.boost = boost
        self._openers = set(torch.nonzero(token_flag_table(model.decoding.tokenizer) & 3).reshape(-1).tolist())
        self._streams: Dict[int, _Stream] = {}
        self._next_id = 0
        self._free: List[int] = []
        self._eng = None
        self._dec_pool: Optional[Tensor] = None    # uint8 [slots, decode record]
        self._spot_pool: Optional[Tensor] = None   # uint8 [slots, K, spot record]
        self._hw_pool: Optional[Tensor] = None     # uint8 [slots, hotwords, spot record]

    # ---- streams
    def open(self) -> int:
        """A new stream; returns its id."""
        if not self._free:
            self._grow()
        slot = self._free.pop()
        self._dec_pool[slot] = self._fresh_dec[0]
        if self.kw_ids:
            self._spot_pool[slot] = self._fresh_spot[0]
        if self.hw_ids:
            self._hw_pool[slot] = self._fresh_hw[0]
        sid = self._next_id
        self._next_id += 1
        self._streams[sid] = _Stream(sid, slot, TextFeed(self.model.decoding.tokenizer, self._openers), len(self.kw_ids),
                                     self.model._dtype)
        if self.hw_ids:
            K = len(self.hw_ids)
            self._streams[sid].hw_det = (torch.zeros((0, 3, K), dtype=torch.int32, device=self._eng.device),
                                         torch.zeros(K, dtype=torch.int32, device=self._eng.device))
        return sid

    def _grow(self) -> None:
        if self._eng is None:
            eng = self._eng = self.model._get_engine()
            self._fresh_dec = eng.decode_state(1)
            if self.boost is not None:
                self.boost = tuple(t.to(eng.device) for t in self.boost)
            if self.kw_ids:
                self._kw, self._kw_len = self.model._keyword_tensors(self.kw_ids, eng.device)
                self._fresh_spot = eng.spot_state(1, len(self.kw_ids), self._kw.shape[1])
                self._min_u = min(len(r) for r in self.kw_ids)
            if self.hw_ids:
                self._hw_kw, self._hw_kw_len = self.model._keyword_tensors(self.hw_ids, eng.device)
                self._fresh_hw = eng.spot_state(1, len(self.hw_ids), self._hw_kw.shape[1])
                self._hw_min_u = min(len(r) for r in self.hw_ids)
                self._flags = self.model._word_flags()
                self._flags_host = self._flags.cpu().tolist()
        old = 0 if self._dec_pool is None else self._dec_pool.shape[0]
        new = max(8, 2 * old)
        dec = self._fresh_dec.expand(new - old, -1)
        self._dec_pool = dec.clone() if self._dec_pool is None else torch.cat([self._dec_pool, dec])
        if self.kw_ids:
            spot = self._fresh_spot.expand(new - old, -1, -1)
            self._spot_pool = spot.clone() if self._spot_pool is None else torch.cat([self._spot_pool, spot])
        if self.hw_ids:
            hw = self._fresh_hw.expand(new - old, -1, -1)
            self._hw_pool = hw.clone() if self._hw_pool is None else torch.cat([self._hw_pool, hw])
        self._free.extend(range(new - 1, old - 1, -1))

    def _get(self, stream: int, what: str) -> _Stream:
        s = self._streams.get(stream)
        if s is None:
            raise ValueError(f"{what}: stream {stream!r} is not open")
        return s

    def push(self, stream: int, chunk) -> None:
        """Append mono samples at the server's sample rate (any length) to a stream.  16 kHz samples are rounded to the model's
        dtype as `prepare_wav` does; samples at another rate are kept as float32 and rounded once resampled.  Host only:
        nothing runs on the device until `step` or `close`."""
        self._get(stream, "push").append(chunk, self._ratio is not None, self.model._dtype)

    # ---- steps
    @torch.inference_mode()
    def step(self) -> List[StreamUpdate]:
        """Encode and decode every ready window of every open stream; returns a StreamUpdate for every stream that has new
        windows, in the order the streams were opened."""
        if self._ratio is not None:
            self._resample(list(self._streams.values()), final=False)
        news = {s: [ready_window(w, self.W, self.V) for w in range(len(s.windows), ready_count(s.n, self.W, self.V))]
                for s in self._streams.values()}
        jobs = [(s, ws[r]) for r in range(max((len(ws) for ws in news.values()), default=0)) for s, ws in news.items() if r < len(ws)]
        if not jobs:
            return []
        before = {s: (len(s.ids), [len(d) for d in s.dets]) for s in news if news[s]}
        self._run(jobs, tentative=True)
        out = []
        for s, (n0, d0) in before.items():
            s.trim(len(s.windows) * (self.W - self.V))
            new_ids = s.ids[n0:]
            dets = [self._detection(k, *d) for k in range(len(self.kw_ids)) for d in s.dets[k][d0[k]:]]
            pending = [self._detection(k, *p) for k, p in enumerate(s.pending) if p is not None]
            dets.sort(key=lambda d: (d.start, d.keyword_index))
            out.append(StreamUpdate(stream=s.id, new_tokens=new_ids, new_text=s.feed.push(s.ids, len(new_ids)),
                                    tentative_text=self.model.decoding.tokenizer.decode(s.hw_ids.tolist() + s.tentative),
                                    committed_until=s.committed * FRAME_SECONDS, detections=dets, pending=pending))
        return out

    def _resample(self, streams: List[_Stream], final: bool) -> None:
        """Resample, in one launch, each stream's 16 kHz outputs that are final (all of them when `final`: the end of the
        recording is known), append them to its 16 kHz samples and drop the raw samples no pending output needs."""
        resample_streams(self._eng, self.sample_rate, self._ratio, self.model._dtype, streams, final)

    def _detection(self, k: int, start: int, end: int, score: float) -> Detection:
        return Detection(keyword=self.names[k], keyword_index=k, start=start * FRAME_SECONDS, end=end * FRAME_SECONDS, score=score,
                         confidence=math.exp(score / len(self.kw_ids[k])))

    def _run(self, jobs: List[Tuple[_Stream, Window]], tentative: bool) -> None:
        """Encode, decode (and spot in) the jobs' windows, each stream's in order, then bring the results to the host."""
        last = {s: i for i, (s, _) in enumerate(jobs)}
        for s, w in jobs:
            s.windows.append(w)
        reads = []
        for group in window_groups(list(enumerate(jobs)), self.batch_size, lambda item: item[1][1]):
            encoded = encode_rows(self.model, [s.samples(w.start, w.end) for _, (s, w) in group])
            enc = _as_btd(encoded)
            lp = self.model.head(encoded) if self.kw_ids or self.hw_ids else None
            rounds: List[List[int]] = []
            seen: Dict[_Stream, int] = {}
            for row, (_, (s, _)) in enumerate(group):
                r = seen[s] = seen.get(s, -1) + 1
                if r == len(rounds):
                    rounds.append([])
                rounds[r].append(row)
            for rows in rounds:
                lp_rows = None if lp is None else self._rows(lp, rows)
                reads.append(self._decode_round([group[r][1] for r in rows], self._rows(enc, rows), lp_rows))
            if tentative:
                rows = [row for row, (i, (s, _)) in enumerate(group) if last[s] == i]
                if rows:   # a group may hold no stream's newest window
                    reads.append(self._tentative([group[r][1] for r in rows], self._rows(enc, rows)))
            del encoded, enc, lp
        for read in reads:           # one synchronisation per call, in job order
            read()

    def _rows(self, x: Tensor, rows: List[int]) -> Tensor:
        return x if rows == list(range(x.shape[0])) else x.index_select(0, torch.tensor(rows, device=x.device))

    def _decode_round(self, sel: List[Tuple[_Stream, Window]], enc: Tensor, lp: Optional[Tensor]):
        """One greedy_resume launch over the kept frames of one window of each stream in `sel` (and one spot launch); returns
        the host read-back."""
        eng, dev = self._eng, self._eng.device
        T_w = enc.shape[1]
        first = [w.start // FRAME_SAMPLES for _, w in sel]
        lo = [w.keep_start - f for (_, w), f in zip(sel, first)]
        hi = [w.keep_end - f for (_, w), f in zip(sel, first)]
        rng = torch.tensor([lo, hi, [0] * len(sel), first, [0] * len(sel)], dtype=torch.int32).to(dev)
        slots = torch.tensor([s.slot for s, _ in sel], device=dev)
        state = self._dec_pool.index_select(0, slots)
        out = eng.decode_buffers(len(sel), eng.hyp_width(T_w), T_w, scores=self.confidence)
        eng.greedy_resume(enc, rng[0], rng[1], rng[2], state, out, self.confidence, self.boost)
        self._dec_pool.index_copy_(0, slots, state)
        frames_max = max(h - l for l, h in zip(lo, hi))
        spot = None
        if self.kw_ids:
            spot = self._spot_round(slots, lp, rng[0], rng[1], rng[3], rng[4], frames_max)
        hot = None
        if self.hw_ids:
            hot = self._spot_round(slots, lp, rng[0], rng[1], rng[3], rng[4], frames_max, hotwords=True)
            for k, (s, _) in enumerate(sel):   # the round's rows join the held span
                rows = lp[k, lo[k]:hi[k]]
                s.hw_rows = rows.clone() if s.hw_rows is None else torch.cat([s.hw_rows, rows])

        def read():
            host = [None if t is None else t.cpu() for t in out]
            ids, frames, counts = host[:3]
            for k, ((s, w), f) in enumerate(zip(sel, first)):
                n = int(counts[k])
                if self.hw_ids:   # the round's greedy output joins the held span, released by _release below
                    s.hw_ids = np.concatenate([s.hw_ids, ids[k, :n].numpy()])
                    s.hw_frames = np.concatenate([s.hw_frames, (frames[k, :n] + f).numpy().astype(np.int32)])
                    if self.confidence:
                        s.hw_logp = np.concatenate([s.hw_logp, host[3][k, :n].numpy()])
                        s.hw_flp = np.concatenate([s.hw_flp, host[6][k, lo[k]:hi[k]].numpy()])
                else:
                    s.ids.extend(ids[k, :n].tolist())
                    s.frames.extend((frames[k, :n] + f).tolist())
                    if self.confidence:
                        s.token_logp.extend(host[3][k, :n].tolist())
                        s.frame_logp.append(host[6][k, lo[k]:hi[k]].numpy())
                if self.confidence:
                    s.frame_rows.append(host[7][k, lo[k]:hi[k]].numpy())
                s.committed = w.keep_end
            if spot is not None:
                self._read_spot([s for s, _ in sel], spot)
            if hot is not None:
                self._release([s for s, _ in sel], [w.keep_end for _, w in sel], hot, finish=False)
        return read

    def _spot_round(self, slots: Tensor, lp: Tensor, lo: Tensor, hi: Tensor, base: Tensor, finish: Tensor, frames: int,
                    hotwords: bool = False):
        """One ctc_spot_resume launch for the streams at `slots`, over the keywords (returns the device outputs) or the
        hotwords (returns the detections and the records after the launch)."""
        eng = self._eng
        kw_ids = self.hw_ids if hotwords else self.kw_ids
        n, K = slots.numel(), len(kw_ids)
        max_det = frames // min(len(r) for r in kw_ids) + 2   # a carried pending one, plus disjoint detections of >= U frames
        i32 = dict(dtype=torch.int32, device=eng.device)
        det = (torch.empty((n, K, max_det), **i32), torch.empty((n, K, max_det), **i32),
               torch.empty((n, K, max_det), dtype=torch.float32, device=eng.device), torch.zeros((n, K), **i32))
        if hotwords:
            state = self._hw_pool.index_select(0, slots)
            eng.ctc_spot_resume(lp, lo, hi, base, finish, self._hw_kw, self._hw_kw_len, self.hotword_threshold, state, det)
            self._hw_pool.index_copy_(0, slots, state)
            return det, state
        pend = (torch.empty((n, K), **i32), torch.empty((n, K), **i32), torch.empty((n, K), dtype=torch.float32, device=eng.device))
        state = self._spot_pool.index_select(0, slots)
        eng.ctc_spot_resume(lp, lo, hi, base, finish, self._kw, self._kw_len, self.threshold, state, det, pend)
        self._spot_pool.index_copy_(0, slots, state)
        return det + pend

    def _held_detections(self, streams: List[_Stream], new: Tuple[Tensor, ...]) -> Tuple[Tensor, ...]:
        """The undecided detections of `streams` (held on the device) followed by the round's new ones `new` = (start, end,
        score [n, K, md], count [n, K]), on the device: the bias-resume input (start, end, score [n, K, D], count [n, K])."""
        st, en, sc, cnt = new
        held = [s.hw_det for s in streams]
        Dc = max(p.shape[0] for p, _ in held)
        if Dc == 0:
            return new
        n, K, md = st.shape
        packed = torch.nn.utils.rnn.pad_sequence([p for p, _ in held], batch_first=True).permute(0, 2, 3, 1)   # [n, 3, K, Dc]
        cc = torch.stack([c for _, c in held])[..., None]
        j = torch.arange(Dc + md, device=st.device)[None, None, :]
        old = j < cc
        jc = j.clamp(max=Dc - 1).expand(n, K, -1)
        jn = (j - cc).clamp(0, md - 1)

        def merge(a, b):
            return torch.where(old, a.gather(2, jc), b.gather(2, jn))
        return (merge(packed[:, 0], st), merge(packed[:, 1], en),
                merge(packed[:, 2].view(torch.float32), sc), cc[..., 0] + cnt)

    def _release(self, streams: List[_Stream], ends: List[int], hot: Tuple[Tuple[Tensor, ...], Tensor], finish: bool) -> None:
        """One ctc_bias_resume launch over the held spans [hw_base, ends[b]) of `streams`, padded to the longest: the round's
        new hotword detections join the undecided ones on the device, the released tokens (and per-frame sums) are
        committed, and the span is trimmed to the release frame.  One read-back per call."""
        eng, dev = self._eng, self._eng.device
        det, state = hot
        det = self._held_detections(streams, det)
        n = len(streams)
        held = [e - s.hw_base for s, e in zip(streams, ends)]
        T = max(1, max(held))
        lp = torch.zeros((n, T, eng.num_classes), dtype=torch.float32, device=dev)
        for b, (s, h) in enumerate(zip(streams, held)):
            if h:
                lp[b, :h] = s.hw_rows[:h]
        max_out = max(T, max(s.hw_ids.size for s in streams))
        ids = np.zeros((n, max_out), np.int32)
        frames = np.zeros((n, max_out), np.int32)
        token_logp = np.zeros((n, max_out), np.float32) if self.confidence else None
        flp = np.zeros((n, T), np.float64) if self.confidence else None
        for b, s in enumerate(streams):
            m = s.hw_ids.size
            ids[b, :m], frames[b, :m] = s.hw_ids, s.hw_frames
            if self.confidence:
                token_logp[b, :m] = s.hw_logp
                flp[b, :s.hw_flp.size] = s.hw_flp
        rng = torch.tensor([held, [s.hw_base for s in streams], [int(finish)] * n, [int(s.hw_left) for s in streams],
                            [s.hw_ids.size for s in streams]], dtype=torch.int32).to(dev)
        flp_dev = None if flp is None else torch.from_numpy(flp).to(dev)
        out = eng.ctc_bias_resume(lp, rng[0], rng[1], rng[2], self._hw_kw, self._hw_kw_len, self.hotword_threshold, state, det,
                                  self._flags, torch.from_numpy(ids).to(dev), torch.from_numpy(frames).to(dev), rng[4], rng[3],
                                  None if token_logp is None else torch.from_numpy(token_logp).to(dev), flp_dev)
        o_ids, o_frames, o_counts, _, o_logp, until, c_st, c_en, c_sc, c_cnt = out
        carried = torch.stack([c_st, c_en, c_sc.view(torch.int32)], 1).permute(0, 3, 1, 2)   # [n, D, 3, K], stays on the device
        o_ids, o_frames, o_counts, until, c_width = (t.cpu().numpy() for t in (o_ids, o_frames, o_counts, until, c_cnt.amax(1)))
        o_logp = None if o_logp is None else o_logp.cpu().numpy()
        flp = None if flp_dev is None else flp_dev.cpu().numpy()
        for b, s in enumerate(streams):
            m, R = int(o_counts[b]), int(until[b])
            cut = R - s.hw_base
            s.ids.extend(o_ids[b, :m].tolist())
            s.frames.extend(o_frames[b, :m].tolist())
            if self.confidence:
                s.token_logp.extend(o_logp[b, :m].tolist())
                s.frame_logp.append(flp[b, :cut].copy())
                s.hw_flp = s.hw_flp[cut:]
            g = int(np.searchsorted(s.hw_frames, R))   # the held greedy tokens before R are released
            if g:
                s.hw_left = bool(self._flags_host[int(s.hw_ids[g - 1])] & 1)
            s.hw_ids, s.hw_frames, s.hw_logp = s.hw_ids[g:], s.hw_frames[g:], s.hw_logp[g:]
            s.hw_det = (carried[b, :int(c_width[b])], c_cnt[b])
            if s.hw_rows is not None:
                s.hw_rows = s.hw_rows[cut:]
            s.hw_base = R
            s.committed = R

    @staticmethod
    def _read_spot(streams: List[_Stream], spot: Tuple[Tensor, ...]) -> None:
        start, end, score, count, p_start, p_end, p_score = (t.cpu() for t in spot)
        counts, pending = count.tolist(), zip(p_start.tolist(), p_end.tolist(), p_score.tolist())
        for b, (s, (ps, pe, psc)) in enumerate(zip(streams, pending)):
            for k, c in enumerate(counts[b]):
                if c:
                    s.dets[k].extend(zip(start[b, k, :c].tolist(), end[b, k, :c].tolist(), score[b, k, :c].tolist()))
            s.pending = [None if a < 0 else (a, e, x) for a, e, x in zip(ps, pe, psc)]

    def _tentative(self, sel: List[Tuple[_Stream, Window]], enc: Tensor):
        """Decode the frames after the kept ones, [keep_end, T_w), of each stream's newest window from a copy of its committed
        decoder record; the output is only reported."""
        eng, dev = self._eng, self._eng.device
        T_w = enc.shape[1]
        lo = [w.keep_end - w.start // FRAME_SAMPLES for _, w in sel]
        rng = torch.tensor([lo, [T_w] * len(sel), [0] * len(sel)], dtype=torch.int32).to(dev)
        state = self._dec_pool.index_select(0, torch.tensor([s.slot for s, _ in sel], device=dev))
        out = eng.decode_buffers(len(sel), eng.hyp_width(T_w))
        eng.greedy_resume(enc, rng[0], rng[1], rng[2], state, out, boost=self.boost)

        def read():
            ids, counts = out.ids.cpu(), out.counts.cpu()
            for k, (s, _) in enumerate(sel):
                s.tentative = ids[k, :int(counts[k])].tolist()
        return read

    # ---- the end of a stream
    @torch.inference_mode()
    def close(self, stream: int, word_timestamps: bool = False, pause: float = 1.0, max_segment: float = 25.0) -> StreamResult:
        """End a stream: encode its remaining windows, the last one included, and return its StreamResult.  Raises ValueError
        for a stream that is not open, pause < 0, max_segment <= 0 and, after freeing the stream, for one whose samples
        encode to no frame (as `transcribe_windowed` does)."""
        s = self._get(stream, "close")
        check_segmenting(pause, max_segment)
        del self._streams[stream]
        self._free.append(s.slot)
        if self._ratio is not None:
            self._resample([s], final=True)
        windows, T = plan_windows(s.n, self.window, self.overlap, self.model._encoded_length, self.model._max_frames)
        N, done = s.n, len(s.windows)
        assert windows[:done] == s.windows, "a ready window differs from the plan of the whole stream"
        self._run([(s, w) for w in windows[done:]], tentative=False)
        detections = None
        if self.kw_ids:
            dev = self._eng.device
            one = torch.tensor([s.slot], device=dev)
            flags = torch.tensor([[0], [0], [0], [1]], dtype=torch.int32, device=dev)   # lo = hi = 0, finish
            lp = torch.zeros((1, 1, self._eng.num_classes), dtype=torch.float32, device=dev)
            self._read_spot([s], self._spot_round(one, lp, flags[0], flags[1], flags[2], flags[3], 0))
            detections = self.model._detections(self.names, self.kw_ids, s.dets, compute_frame_shift(N, T))
        if self.hw_ids:   # the last hotword call: the pending detections are emitted and everything held is released
            dev = self._eng.device
            one = torch.tensor([s.slot], device=dev)
            flags = torch.tensor([[0], [0], [0], [1]], dtype=torch.int32, device=dev)
            lp = torch.zeros((1, 1, self._eng.num_classes), dtype=torch.float32, device=dev)
            self._release([s], [T], self._spot_round(one, lp, flags[0], flags[1], flags[2], flags[3], 0, hotwords=True), finish=True)
        transcript = windowed_result(self.model, s.ids, s.frames, s.token_logp if self.confidence else None,
                                     np.concatenate(s.frame_logp) if self.confidence else None,
                                     np.concatenate(s.frame_rows) if self.confidence else None, N, T, word_timestamps, pause,
                                     max_segment)
        return StreamResult(transcript=transcript, detections=detections)

    @property
    def streams(self) -> List[int]:
        """The ids of the open streams."""
        return list(self._streams)


class _EmoStream(_Audio):
    """Host side of one open emotion stream."""

    def __init__(self, sid: int, dtype: torch.dtype):
        super().__init__(dtype)
        self.id = sid
        self.final = 0                   # frames whose logits are final
        self.k = 0                       # the next planned span [k hop, k hop + span) to emit
        self.dev_from = 0                # first frame a future span can read: the device holds frames [dev_from, final)
        self.dev: Optional[Tensor] = None
        self.logits: List[Tensor] = []   # host frame logits of frames [0, final), in pieces
        self.spans: List[Tuple[int, int]] = []   # the spans emitted, in frames
        self.probs: List[Tensor] = []    # their probabilities, in pieces


class EmotionStreamServer:
    """Emotions of live audio streams, with one encoder batch per step across all of them (INTEGRATION.md, "Emotions over
    time").  Made by `GigaAMEmo.streaming(...)`:

        srv = model.streaming(window=8.0, overlap=4.0, span=4.0, hop=1.0)
        a = srv.open()
        srv.push(a, chunk)              # host samples, any length
        for u in srv.step():            # an EmotionStreamUpdate for every stream that got final frames
            ...
        timeline = srv.close(a)

    Windows are `StreamServer`'s: window w is encoded once it is ready (`ready_count`, `ready_window`), and one
    gam_emo_frame_logits launch per batch writes the kept frames' logits into each stream's frames.  A planned span
    [k hop, k hop + span) is emitted once its last frame is final, by one gam_emo_spans call per step over every stream's new
    spans; the tail span of `longform.emotion_spans` comes only at `close`, which returns `emotion_timeline(recording, window,
    overlap, span, hop)` bit for bit.  The device holds, per stream, only the frames a future span can still read (from the
    next planned span's start, or span frames before the final frames for a tail span), so device memory does not grow with a
    stream's duration.  The host keeps each stream's frame logits (4 C bytes per 40 ms, returned by `close`) and the spans
    already emitted.  One caller drives a server; it is not thread-safe."""

    def __init__(self, model, window: float = 8.0, overlap: float = 4.0, span: float = 4.0, hop: float = 1.0, batch_size: int = 64,
                 sample_rate: int = SAMPLE_RATE):
        from .longform import emotion_plan_frames
        self.sample_rate = sample_rate
        self._ratio = None if sample_rate == SAMPLE_RATE else resample_ratio(sample_rate)
        self.W = _frame_multiple(window, "window")
        self.V = _frame_multiple(overlap, "overlap")
        plan_windows(max(self.W, 1), window, overlap, model._encoded_length, model._max_frames)   # the window plan's refusals
        if batch_size < 1:
            raise ValueError("batch_size must be >= 1")
        self.span, self.hop = emotion_plan_frames(span, hop)
        self.model, self.window, self.overlap, self.batch_size = model, window, overlap, int(batch_size)
        self.names: List[str] = list(model.id2name)
        self._streams: Dict[int, _EmoStream] = {}
        self._next_id = 0
        self._eng = None

    def open(self) -> int:
        """A new stream; returns its id."""
        sid = self._next_id
        self._next_id += 1
        self._streams[sid] = _EmoStream(sid, self.model._dtype)
        return sid

    def _get(self, stream: int, what: str) -> _EmoStream:
        s = self._streams.get(stream)
        if s is None:
            raise ValueError(f"{what}: stream {stream!r} is not open")
        return s

    def push(self, stream: int, chunk) -> None:
        """Append mono samples at the server's sample rate (any length) to a stream, as `StreamServer.push` does.  Host only."""
        self._get(stream, "push").append(chunk, self._ratio is not None, self.model._dtype)

    def _engine(self):
        if self._eng is None:
            self._eng = self.model._get_engine()
        return self._eng

    @torch.inference_mode()
    def step(self) -> List[EmotionStreamUpdate]:
        """Encode every ready window of every open stream and emit the planned spans that became final; returns an
        EmotionStreamUpdate for every stream that has new windows, in the order the streams were opened."""
        streams = list(self._streams.values())
        if self._ratio is not None and streams:
            resample_streams(self._engine(), self.sample_rate, self._ratio, self.model._dtype, streams, final=False)
        news = {s: [ready_window(w, self.W, self.V) for w in range(len(s.windows), ready_count(s.n, self.W, self.V))] for s in streams}
        news = {s: ws for s, ws in news.items() if ws}
        if not news:
            return []
        jobs = [(s, ws[r]) for r in range(max(len(ws) for ws in news.values())) for s, ws in news.items() if r < len(ws)]
        ends = {s: ws[-1].keep_end for s, ws in news.items()}
        spans = {}
        for s, end in ends.items():
            last = (end - self.span) // self.hop if end >= self.span else -1    # the last k whose span ends by `end`
            spans[s] = [(k * self.hop, k * self.hop + self.span) for k in range(s.k, last + 1)]
            s.k = max(s.k, last + 1)
        probs = self._run(jobs, ends, spans)
        out = []
        for s in news:
            s.trim(len(s.windows) * (self.W - self.V))
            new = [EmotionSpan(start=a * FRAME_SECONDS, end=b * FRAME_SECONDS, probs=dict(zip(self.names, row)))
                   for (a, b), row in zip(spans[s], probs[s].tolist())]
            out.append(EmotionStreamUpdate(stream=s.id, new_spans=new, final_until=s.final * FRAME_SECONDS))
        return out

    def _run(self, jobs: List[Tuple[_EmoStream, Window]], ends: Dict[_EmoStream, int],
             spans: Dict[_EmoStream, List[Tuple[int, int]]]) -> Dict[_EmoStream, Tensor]:
        """Encode the jobs' windows and write their kept frames' logits next to each stream's held frames in one step buffer
        (one gam_emo_frame_logits launch per batch), score every stream's `spans` in one gam_emo_spans call, bring the new
        frame logits and the probabilities to the host and keep on the device only the frames a future span can read.
        `ends[s]` is stream s's final frame count after the jobs.  Returns each stream's probs [len(spans[s]), C] (host)."""
        eng = self._engine()
        base, total = {}, 0
        for s, end in ends.items():
            base[s] = total
            total += end - s.dev_from
        buf = torch.empty((max(total, 1), eng.num_classes), dtype=torch.float32, device=eng.device)
        for s in ends:
            if s.dev is not None and s.dev.shape[0]:
                buf[base[s]:base[s] + s.dev.shape[0]] = s.dev
        for s, w in jobs:
            s.windows.append(w)
        for group in window_groups(jobs, self.batch_size, lambda job: job[1]):
            encoded = encode_rows(self.model, [s.samples(w.start, w.end) for s, w in group])
            first = [w.start // FRAME_SAMPLES for _, w in group]
            rng = torch.tensor([[w.keep_start - f for (_, w), f in zip(group, first)], [w.keep_end - f for (_, w), f in zip(group, first)],
                                [base[s] + w.keep_start - s.dev_from for s, w in group]], dtype=torch.int32).to(eng.device)
            eng.emo_frame_logits(_as_btd(encoded), rng[0], rng[1], rng[2], buf)
            del encoded
        plan = [(base[s] + a - s.dev_from, base[s] + b - s.dev_from) for s in ends for a, b in spans[s]]
        assert all(a >= s.dev_from for s in ends for a, _ in spans[s]), "a span reads a frame the device no longer holds"
        probs = torch.zeros((0, eng.num_classes), dtype=torch.float32)
        if plan:
            se = torch.tensor(plan, dtype=torch.int32).t().contiguous().to(eng.device)
            probs = eng.emo_spans(buf, se[0], se[1], logits=False)[1].cpu()
        host = buf.cpu()
        out, row = {}, 0
        for s, end in ends.items():
            out[s] = probs[row:row + len(spans[s])]
            row += len(spans[s])
            s.probs.append(out[s])
            s.spans.extend(spans[s])
            s.logits.append(host[base[s] + s.final - s.dev_from:base[s] + end - s.dev_from].clone())
            # a future span starts at the next planned span or, as the tail span, at or after end - span
            keep = min(max(s.dev_from, min(s.k * self.hop, end - self.span)), end)
            s.dev = buf[base[s] + keep - s.dev_from:base[s] + end - s.dev_from].clone()
            s.dev_from, s.final = keep, end
        return out

    @torch.inference_mode()
    def close(self, stream: int) -> EmotionTimeline:
        """End a stream: encode its remaining windows, the last one included, and return its EmotionTimeline, which is
        `emotion_timeline(recording, window, overlap, span, hop)`'s bit for bit.  Raises ValueError for a stream that is not
        open and, after freeing the stream, for one whose samples encode to no frame."""
        from .longform import emotion_result, emotion_spans
        s = self._get(stream, "close")
        del self._streams[stream]
        if self._ratio is not None:
            resample_streams(self._engine(), self.sample_rate, self._ratio, self.model._dtype, [s], final=True)
        windows, T = plan_windows(s.n, self.window, self.overlap, self.model._encoded_length, self.model._max_frames)
        N, done = s.n, len(s.windows)
        assert windows[:done] == s.windows, "a ready window differs from the plan of the whole stream"
        plan = emotion_spans(T, self.span, self.hop)
        assert plan[:len(s.spans)] == s.spans, "an emitted span differs from the plan of the whole stream"
        self._run([(s, w) for w in windows[done:]], {s: T}, {s: plan[len(s.spans):]})
        return emotion_result(self.names, s.spans, torch.cat(s.probs), torch.cat(s.logits), compute_frame_shift(N, T))

    @property
    def streams(self) -> List[int]:
        """The ids of the open streams."""
        return list(self._streams)
