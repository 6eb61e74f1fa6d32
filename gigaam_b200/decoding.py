"""Greedy decoders with the reference's interface (gigaam/decoding.py).  `decode(head, encoded, lengths)`
returns the same `List[(text, token_ids, token_frames)]`; head projection, argmax, CTC collapse and the whole
RNN-T prediction/joint loop run on the device, then one D2H copy brings ids / frames / counts back for the
host-side detokenisation (which the reference also does on the host, decoding.py:93-96,207)."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib


class Tokenizer:
    """gigaam/decoding.py:10-44 -- charwise vocabulary or a SentencePiece model."""

    def __init__(self, vocab: List[str], model_path: Optional[str] = None):
        self.charwise = model_path is None
        if self.charwise:
            self.vocab = vocab
        else:
            from sentencepiece import SentencePieceProcessor
            self.model = SentencePieceProcessor()
            self.model.load(model_path)

    def normalize(self, text: str) -> str:
        """The text `encode` tokenises (the reference fine-tuner's rule, gigaam/utils.py:228-239): ё -> е, whitespace runs
        collapsed to one space and trimmed, lower case; a charwise vocabulary also drops every character it lacks."""
        text = " ".join(text.replace("ё", "е").replace("Ё", "Е").split()).lower()
        if self.charwise:
            vocab = set(self.vocab)
            text = "".join(c for c in text if c in vocab)
        return text

    def encode(self, text: str) -> List[int]:
        """Token ids of `normalize(text)`: one id per character for a charwise vocabulary, SentencePiece's `encode` otherwise
        (gigaam/utils.py:218-226)."""
        text = self.normalize(text)
        if self.charwise:
            c2i = {c: i for i, c in enumerate(self.vocab)}
            return [c2i[c] for c in text]
        return list(self.model.encode(text))

    def decode(self, tokens: List[int]) -> str:
        if self.charwise:
            return "".join(self.vocab[tok] for tok in tokens)
        return self.model.decode(tokens)

    def __len__(self):
        return len(self.vocab) if self.charwise else len(self.model)

    def id_to_str(self, token_id: int) -> str:
        if self.charwise:
            return self.vocab[token_id]
        return self.model.IdToPiece(token_id)


def _as_btd(encoded: Tensor) -> Tensor:
    """[B, d, T] (the encoder's transposed view) -> contiguous [B, T, d] without a copy when possible."""
    x = encoded.transpose(1, 2)
    return x if x.is_contiguous() else x.contiguous()


class _GreedyBase:
    def __init__(self, vocabulary: List[str], model_path: Optional[str] = None):
        self.tokenizer = Tokenizer(vocabulary, model_path)
        self.blank_id = len(self.tokenizer)

    def decode_device(self, head, encoded: Tensor, lengths: Tensor, packed: Optional[Tensor] = None, scores: bool = False
                      ) -> Tuple[Tensor, ...]:
        """Device-resident result: ids [B, max_out] i32, frames [B, max_out] i32, counts [B] i32 (views of `packed`, an
        `Engine.packed_hypotheses` buffer, when one is given: the layout the multi-GPU gather ships).  `scores=True`
        appends token_logp [B, max_out] f32, path_logp [B] f32 and path_rows [B] i32 (`Engine.greedy`)."""
        eng = head._engine()
        assert eng.num_classes == len(self.tokenizer) + 1, \
            f"Num classes {eng.num_classes} != len(vocab)+1 {len(self.tokenizer) + 1}"
        enc = _as_btd(encoded.to(device=eng.device, dtype=torch.float32))
        return eng.greedy(enc, lengths, packed, scores=scores)

    @torch.inference_mode()
    def decode(self, head, encoded: Tensor, lengths: Tensor, return_scores: bool = False) -> List[Tuple]:
        """[(text, token_ids, token_frames)] per utterance; with `return_scores`, (text, token_ids, token_frames,
        token_logprobs, path_logprob, path_rows): the log-probability of every emitted token, the sum over every decision
        row of the greedy path and the number of those rows (include/gigaam_b200.h, gam_ctc_greedy_scored)."""
        if not return_scores:
            ids, frames, counts = self.decode_device(head, encoded, lengths)
            return self.to_hypotheses(ids.cpu(), frames.cpu(), counts.cpu())
        out = [t.cpu() for t in self.decode_device(head, encoded, lengths, scores=True)]
        return self.to_scored_hypotheses(*out)

    def to_hypotheses(self, ids: Tensor, frames: Tensor, counts: Tensor) -> List[Tuple[str, List[int], List[int]]]:
        out = []
        for b, n in enumerate(counts.tolist()):
            tok = ids[b, :n].tolist()
            out.append((self.tokenizer.decode(tok), tok, frames[b, :n].tolist()))
        return out

    def to_scored_hypotheses(self, ids: Tensor, frames: Tensor, counts: Tensor, token_logp: Tensor, path_logp: Tensor,
                             path_rows: Tensor) -> List[Tuple[str, List[int], List[int], List[float], float, int]]:
        return [hyp + (token_logp[b, :len(hyp[1])].tolist(), float(path_logp[b]), int(path_rows[b]))
                for b, hyp in enumerate(self.to_hypotheses(ids, frames, counts))]


class CTCGreedyDecoding(_GreedyBase):
    """gigaam/decoding.py:47-96"""


class RNNTGreedyDecoding(_GreedyBase):
    """gigaam/decoding.py:99-207"""

    def __init__(self, vocabulary: List[str], model_path: Optional[str] = None, max_symbols_per_step: int = 10):
        super().__init__(vocabulary, model_path)
        self.max_symbols = max_symbols_per_step


def align(head, encoded: Tensor, encoded_len: Tensor, targets: Tensor, target_lengths: Tensor) -> Tuple[Tensor, ...]:
    """Viterbi and forward alignment of known transcripts (include/gigaam_b200.h, gam_ctc_align / gam_rnnt_align).
    encoded [B, d, T] (the encoder's output), encoded_len [B], targets [B, U] token ids in [0, V) (entries at or past
    target_lengths[b] are ignored), target_lengths [B] -> device tensors (frames [B, U] i32, token_logp [B, U] f32,
    viterbi_logp [B] f32, log_likelihood [B] f32, path_rows [B] i32).  CTC: gam_ctc_log_probs, then gam_ctc_align.  RNN-T:
    the prediction network over cat[blank, y] (one launch per step), the gathered joint scores, then gam_rnnt_align.  No host
    synchronisation: the call can be captured in a CUDA graph."""
    eng = head._engine()
    enc = _as_btd(encoded.to(device=eng.device, dtype=torch.float32))
    targets = targets.to(device=eng.device)
    target_lengths = target_lengths.to(device=eng.device)
    if eng.head_type == 1:
        return eng.ctc_align(eng.ctc_log_probs(enc), encoded_len, targets, target_lengths)
    y, x = _rnnt_inputs(eng, targets, target_lengths)
    dec, _, _ = eng.rnnt_predict(x, None, None)
    blank_lp, label_lp = eng.rnnt_align_scores(enc, dec, y)
    return eng.rnnt_align(blank_lp, label_lp, encoded_len, target_lengths)


def _rnnt_inputs(eng, targets: Tensor, target_lengths: Tensor) -> Tuple[Tensor, Tensor]:
    """The RNN-T prologue of align and rnnt_loss: device targets [B, U] -> (y [B, U] i64 with every entry at or past
    target_lengths[b] replaced by blank, x = cat[blank, y] [B, U+1], the prediction network's input)."""
    B, U = targets.shape
    blank = eng.num_classes - 1
    # the prediction network reads every step of its input: padding becomes blank so that it cannot poison the utterance
    used = torch.arange(U, device=eng.device)[None, :] < target_lengths.to(torch.int64)[:, None]
    y = torch.where(used, targets.to(torch.int64), torch.full_like(targets, blank, dtype=torch.int64))
    x = torch.cat([torch.full((B, 1), blank, dtype=torch.int64, device=eng.device), y], 1).contiguous()
    return y, x


_REDUCTIONS = ("none", "mean", "sum")


def rnnt_loss(head, encoded: Tensor, encoded_len: Tensor, targets: Tensor, target_lengths: Tensor, reduction: str = "mean"
              ) -> Tensor:
    """The RNN-T loss -log p(y | x), summed over all alignments, without the [B, T, U+1, V+1] lattice (include/gigaam_b200.h,
    gam_rnnt_loss).  encoded [B, d, T] (the encoder's output), encoded_len [B], targets [B, U] token ids in [0, V) (entries at or
    past target_lengths[b] are ignored), target_lengths [B] -> loss [B] for reduction="none", else its batch mean or sum: the
    values of torchaudio.functional.rnnt_loss(..., blank=V, reduction=...) on the lattice of head.joint.joint.  Differentiable:
    the prediction network runs through head.decoder.predict and the joint through the fused loss, so gradients reach
    decoder.embed / decoder.lstm, joint.enc / joint.pred / joint.joint_net.1 and `encoded` when it requires grad.  An
    utterance with encoded_len 0 has loss +inf and no gradient.  No host synchronisation: the call can be captured in a CUDA
    graph.  CTC heads raise NotImplementedError (use F.ctc_loss on model.head(encoded)); another reduction, a joint_hidden or
    pred_hidden the fused loss does not run, and a gradient through a prediction network wider than the predict backward
    runs raise ValueError before any device work."""
    if reduction not in _REDUCTIONS:
        raise ValueError(f"rnnt_loss: reduction must be one of {_REDUCTIONS}, got {reduction!r}")
    if getattr(head, "decoder", None) is None or getattr(head, "joint", None) is None:
        raise NotImplementedError("rnnt_loss needs an RNN-T head; for a CTC model use torch.nn.functional.ctc_loss on the "
                                  "log-probs of model.head(encoded), transposed to [T, B, V+1]")
    J = head.joint_cfg["joint_hidden"]
    if J % 4 != 0 or J > _lib.RNNT_LOSS_MAX_JOINT_HIDDEN:
        raise ValueError(f"rnnt_loss: joint_hidden {J} is not supported: the fused loss runs joint_hidden <= "
                         f"{_lib.RNNT_LOSS_MAX_JOINT_HIDDEN}, a multiple of 4")
    H = head.decoder.pred_hidden
    if H % 16 != 0:   # the projection GEMM's k-step (gam_api.cu, proj_shapes_ok)
        raise ValueError(f"rnnt_loss: pred_hidden {H} is not supported: the fused loss projects pred_hidden in steps of 16, "
                         f"so it must be a multiple of 16")
    head.decoder._check_trainable()
    eng = head._engine()
    enc = _as_btd(encoded.to(device=eng.device, dtype=torch.float32))
    targets = targets.to(device=eng.device)
    target_lengths = target_lengths.to(device=eng.device)
    y, x = _rnnt_inputs(eng, targets, target_lengths)
    dec, _ = head.decoder.predict(x, None)
    loss = head.joint._loss(enc, dec, y, encoded_len.to(device=eng.device), target_lengths)
    if reduction == "mean":
        return loss.mean()
    return loss.sum() if reduction == "sum" else loss


BOOST_MAX_STATES = 65536   # kBoostMaxStates of csrc/kernels.h


def boost_graph(phrases: Sequence[Sequence[int]], weight: float, anchor: Optional[int], V1: int, blank: int
                ) -> Tuple[Tensor, Tensor]:
    """The boost graph of `phrases` (token-id sequences) for gam_rnnt_greedy_boost: (next int32 [S, V1], bonus float32 [S, V1])
    on the host, state 0 initial (include/gigaam_b200.h and INTEGRATION.md §7j have the definition).

    Each phrase is a pattern; with `anchor` (the space token of a charwise vocabulary, else None) it is prefixed by the
    anchor, so that a match can only start at a word start.  The states are all prefixes of all patterns, the empty one
    included; state 0 is the anchor's (the start of a transcript is a word start), or the empty prefix without an anchor.
    next(s, v) is the longest suffix of s.v that is a state (Aho-Corasick), and bonus(s, v) = fp32(weight) when next(s, v)
    ends in a phrase token (it is neither empty nor the bare anchor), else 0.  Blank gets no bonus and does not move the
    state.  Duplicate phrases are merged.

    There is deliberately no penalty for abandoning a partial match, as some beam-search boosters take back the bonus of a
    failed match: greedy decisions never compare accumulated totals, so such a penalty would only make the decoder hold on to
    a wrong partial match, and that costs deletions.

    Raises ValueError for a weight that is not finite and > 0 in fp32, and for a graph of more than 65 536 states."""
    with np.errstate(over="ignore"):
        w = np.float32(weight)
    if not (np.isfinite(w) and w > 0):
        raise ValueError(f"boost: weight={weight} must be finite and > 0 (in fp32)")
    pats = {tuple(([] if anchor is None else [int(anchor)]) + [int(t) for t in p]) for p in phrases}
    prefixes = {p[:k] for p in pats for k in range(len(p) + 1)}
    if len(prefixes) > BOOST_MAX_STATES:
        raise ValueError(f"boost: the phrases make a graph of {len(prefixes)} states, more than {BOOST_MAX_STATES}")
    start = () if anchor is None else (int(anchor),)
    # states by length (the initial one first): a state's suffix link is shorter, so its row is complete when it is copied
    order = sorted(prefixes - {start}, key=lambda t: (len(t), t))
    order.insert(0, start)
    idx = {t: i for i, t in enumerate(order)}
    children: dict = {}
    for t in order:
        if t:
            children.setdefault(t[:-1], []).append(t)
    S = len(order)
    nxt = np.zeros((S, V1), dtype=np.int32)
    link = {}
    root = idx[()]
    for t in sorted(order, key=len):        # Aho-Corasick: the row of t is its suffix link's row, with t's children over it
        i = idx[t]
        if len(t) == 0:
            nxt[i] = i
        else:
            link[t] = root if len(t) == 1 else int(nxt[link[t[:-1]], t[-1]])
            nxt[i] = nxt[link[t]]
        for c in children.get(t, ()):
            nxt[i, c[-1]] = idx[c]
    # a bonus where the next state ends in a phrase token: neither the empty prefix nor the bare anchor
    ends_in_phrase = np.array([len(t) > len(start) or (anchor is None and len(t) > 0) for t in order], dtype=bool)
    bonus = np.where(ends_in_phrase[nxt], w, np.float32(0)).astype(np.float32)
    bonus[:, blank] = 0
    nxt[:, blank] = np.arange(S, dtype=np.int32)
    return torch.from_numpy(nxt), torch.from_numpy(bonus)


def spot(head, encoded: Tensor, encoded_len: Tensor, keywords: Tensor, keyword_len: Tensor, threshold: float, max_det: int
         ) -> Tuple[Tensor, ...]:
    """CTC keyword spotting (include/gigaam_b200.h, gam_ctc_spot).  encoded [B, d, T] (the encoder's output), encoded_len [B],
    keywords [K, Umax] token ids in [0, V) (entries at or past keyword_len[k] are ignored), keyword_len [K] in [1, 64],
    threshold in (0, 1] -> device tensors (start [B, K, max_det] i32, end [B, K, max_det] i32, score [B, K, max_det] f32,
    count [B, K] i32): gam_ctc_log_probs, then gam_ctc_spot.  No host synchronisation: the call can be captured in a CUDA
    graph.  RNN-T heads raise NotImplementedError: they have no frame posteriors without a lattice."""
    eng = head._engine()
    if eng.head_type != 1:
        raise NotImplementedError("keyword spotting needs a CTC head: an RNN-T model has no per-frame posteriors without its "
                                  "[T, U + 1] lattice; use a *_ctc model")
    enc = _as_btd(encoded.to(device=eng.device, dtype=torch.float32))
    return eng.ctc_spot(eng.ctc_log_probs(enc), encoded_len, keywords, keyword_len, threshold, max_det)
