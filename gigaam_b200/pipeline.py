"""Host-side batch pipeline around the reference surface (`model(wav, len)` + `model.decoding.decode`):
the H2D copy of batch i+1 (copy stream, pinned source) and the D2H copy + detokenisation of batch i-1 overlap the
device work of batch i, and the ~270 kernel launches of a batch are replayed as ONE CUDA graph per input shape
(captured from the very same `model(...)` / `decode_device(...)` calls), so the GPU waits neither for PCIe nor for
the host's launch loop.  Nothing here changes what is computed; it is the serving loop a caller such as the
reference's `transcribe_longform` / `train_utils/eval.py` would drive."""
from __future__ import annotations

from typing import Dict, Iterable, Iterator, List, Tuple

import torch

Tensor = torch.Tensor


class _ShapeGraph:
    """The whole device step for one (B, N) input shape, captured once: static inputs -> static outputs."""

    def __init__(self, model, B: int, N: int, dev: torch.device, with_words: bool = False, gather=None, with_scores: bool = False):
        self.with_words = with_words
        self.with_scores = with_scores
        self.gather = gather
        self.wav = torch.zeros((B, N), dtype=torch.float32, device=dev)
        self.len = torch.full((B,), N, dtype=torch.int64, device=dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(2):                      # eager warm-up: plans, workspaces, tensor maps
                self._step(model)
        side.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph, stream=side):
            self.out = self._step(model)
        torch.cuda.current_stream(dev).wait_stream(side)
        # the graph baked the pointers of the engine's scratch buffers for this shape: own them, so the engine's
        # per-kind LRU may forget the shape without freeing memory this graph still writes
        self._held = model._get_engine().held_workspaces(B, N)

    def _step(self, model):
        return device_step(model, self.wav, self.len, self.with_words, self.gather, self.with_scores)


def device_step(model, wav: Tensor, lengths: Tensor, with_words: bool = False, gather=None, with_scores: bool = False):
    """wav -> device-resident hypotheses (ids, frames, counts, encoded_len[, word records][, token_logp, path_logp,
    path_rows]): the kernels of one batch.  With `gather` (dist.HypothesisGather; every rank runs the same number of
    equally shaped steps) the shard's packed hypotheses are all-gathered inside the step and ids / frames / counts are
    those of the GLOBAL batch; scores are not part of that layout.  `with_scores` decodes with the scored kernels."""
    if gather is not None and with_scores:
        raise ValueError("scores are not gathered across ranks")
    enc, enc_len = model(wav, lengths)
    if gather is not None:
        from .dist import unpack_gathered
        eng = model._get_engine()
        B, T = enc.shape[0], enc.shape[2]
        packed = eng.packed_hypotheses(B, T)
        model.decoding.decode_device(model.head, enc, enc_len, packed)
        ids, frames, counts = unpack_gathered(gather.all_gather(packed), B * gather.world, gather.world, B, eng.hyp_width(T))
        return ids, frames, counts, enc_len
    out = model.decoding.decode_device(model.head, enc, enc_len, scores=with_scores)
    ids, frames, counts = out[:3]
    words = tuple(model._get_engine().group_words(ids, frames, counts, model._word_flags())) if with_words else ()
    return (ids, frames, counts, enc_len) + words + tuple(out[3:])


class BatchPipeline:
    """`run(host_batches)` yields the hypotheses of every batch.  `with_words=True` also groups tokens into words on the
    device (csrc/words.cu) and `run_raw` then yields the host copies of the raw records for word timestamps.
    `with_scores=True` decodes with the scored kernels inside the same step (and graph): `run_raw` appends token_logp,
    path_logp and path_rows."""

    def __init__(self, model, use_graph: bool = True, max_graphs: int = 4, with_words: bool = False, gather=None,
                 with_scores: bool = False):
        self.model = model
        self.with_words = with_words
        self.with_scores = with_scores
        self.gather = gather          # dist.HypothesisGather: results are then those of all ranks' batches
        self.dev = model._device
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self.use_graph = use_graph
        self.max_graphs = max_graphs
        self._graphs: Dict[Tuple[int, int], _ShapeGraph] = {}

    def _upload(self, batch):
        wav, lengths = batch
        with torch.cuda.stream(self.copy_stream):
            wav_d = wav.to(self.dev, non_blocking=True)
            len_d = lengths.to(self.dev, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        return wav_d, len_d, ev

    def _graph_for(self, B: int, N: int) -> _ShapeGraph:
        g = self._graphs.get((B, N))
        if g is None:
            if len(self._graphs) >= self.max_graphs:
                self._graphs.pop(next(iter(self._graphs)))
            g = _ShapeGraph(self.model, B, N, self.dev, self.with_words, self.gather, self.with_scores)
            self._graphs[(B, N)] = g
        return g

    @torch.inference_mode()
    def run(self, host_batches: Iterable[Tuple[Tensor, Tensor]]) -> Iterator[List[Tuple[str, List[int], List[int]]]]:
        """host_batches: iterable of (wav [B, N] float32 pinned host tensor, lengths [B] int64) -> hypotheses per batch."""
        for host in self.run_raw(host_batches):
            yield self.model.decoding.to_hypotheses(*host[:3])

    @torch.inference_mode()
    def run_raw(self, host_batches: Iterable[Tuple[Tensor, Tensor]]) -> Iterator[List[Tensor]]:
        """Like `run`, but yields the pinned host copies of the device step's outputs: ids, frames, counts, encoded_len
        (+ word_start, word_end, word_first, word_ntok, n_words with `with_words`; + token_logp, path_logp, path_rows with
        `with_scores`)."""
        model = self.model
        compute = torch.cuda.current_stream(self.dev)
        it = iter(host_batches)
        try:
            nxt = self._upload(next(it))
        except StopIteration:
            return
        prev = None
        while nxt is not None:
            wav_d, len_d, ev = nxt
            try:
                nxt = self._upload(next(it))          # next batch's PCIe transfer runs under this batch's kernels
            except StopIteration:
                nxt = None
            compute.wait_event(ev)
            wav_d.record_stream(compute)
            len_d.record_stream(compute)
            if self.use_graph:
                g = self._graph_for(wav_d.shape[0], wav_d.shape[1])
                g.wav.copy_(wav_d, non_blocking=True)   # device-to-device refill of the graph's static input
                g.len.copy_(len_d, non_blocking=True)
                g.graph.replay()
                outs = g.out
            else:
                outs = device_step(model, wav_d, len_d, self.with_words, self.gather, self.with_scores)
            host = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in outs]
            for h, t in zip(host, outs):
                h.copy_(t, non_blocking=True)           # stream-ordered before the next replay overwrites the outputs
            done = torch.cuda.Event()
            done.record(compute)
            if prev is not None:
                prev[1].synchronize()
                yield prev[0]
            prev = (host, done)
        if prev is not None:
            prev[1].synchronize()
            yield prev[0]
