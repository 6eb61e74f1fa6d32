"""Word timestamps from the (token id, frame) pairs the greedy kernels emit, with the reference's semantics
(gigaam/timestamps_utils.py:8-53): a word starts at its first token's frame and ends one frame after its last token;
words split on a space token or a SentencePiece piece starting with U+2581.

The grouping itself runs on the device (csrc/words.cu through `gam_group_words`, driven by a per-token flag table built
once from the tokenizer): `words_from_device` only multiplies frames by the frame shift and joins the pieces of each
word's token range.  `frames_to_words` is the reference's host function with the same signature, kept as public surface
and as the checker of the device path in the tests."""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import torch

from .preprocess import SAMPLE_RATE
from .types import Word

_SP_SPACE = "▁"


def compute_frame_shift(audio_length_samples: int, seq_len: int) -> float:
    return audio_length_samples / SAMPLE_RATE / seq_len


def frames_to_words(tokenizer, token_ids: List[int], token_frames: List[int], frame_shift: float) -> List[Word]:
    words: List[Word] = []
    pieces: List[str] = []
    frames: List[int] = []

    def flush() -> None:
        text = "".join(pieces).strip()
        if text:
            words.append(Word(text=text, start=frames[0] * frame_shift, end=(frames[-1] + 1) * frame_shift))
        pieces.clear()
        frames.clear()

    for tok, fr in zip(token_ids, token_frames):
        piece = tokenizer.id_to_str(tok)
        if piece == " ":
            flush()
            continue
        if piece.startswith(_SP_SPACE):
            flush()
            piece = piece[1:]
        pieces.append(piece)
        frames.append(fr)
    flush()
    return words


def token_flag_table(tokenizer) -> torch.Tensor:
    """uint8 [V] flags of include/gigaam_b200.h:gam_group_words -- 1: the piece is " "; 2: it starts with U+2581;
    4: nothing visible is left of it after removing that prefix and strip()."""
    flags = torch.zeros(len(tokenizer), dtype=torch.uint8)
    for tok in range(len(tokenizer)):
        piece = tokenizer.id_to_str(tok)
        if piece.startswith(_SP_SPACE):
            flags[tok] = 2 | (4 if piece[1:].strip() == "" else 0)
        elif piece == " ":
            flags[tok] = 1
        elif piece.strip() == "":
            flags[tok] = 4
    return flags


def mean_logp_confidence(logps: Sequence[float]) -> float:
    """exp(mean of the log-probabilities), summed in order in float64; NaN for an empty sequence or a NaN member."""
    return math.exp(sum(float(x) for x in logps) / len(logps)) if len(logps) else math.nan


def path_confidence(path_logp: float, path_rows: int) -> float:
    """exp(path_logp / path_rows): the per-decision likelihood of a greedy path, blank decisions included; NaN when the
    path has no decision rows."""
    return math.exp(float(path_logp) / int(path_rows)) if int(path_rows) > 0 else math.nan


def gap_confidence(viterbi_logp: float, unmatched_logp: float, matched_rows: int, skip_logp: float = 0.0) -> float:
    """exp((viterbi_logp - unmatched_logp - skip_logp) / matched_rows): an alignment with gaps' Viterbi score per matched
    frame, the unmatched frames' scores and the skip edges' penalties taken out; NaN when no frame is matched."""
    if int(matched_rows) <= 0:
        return math.nan
    return math.exp((float(viterbi_logp) - float(unmatched_logp) - float(skip_logp)) / int(matched_rows))


def words_from_device(tokenizer, ids: Sequence[int], word_start: Sequence[int], word_end: Sequence[int],
                      word_first: Sequence[int], word_ntok: Sequence[int], frame_shift: float,
                      token_logp: Optional[Sequence[float]] = None) -> List[Word]:
    """Word records of one utterance (host copies of gam_group_words' outputs) -> List[Word].  With `token_logp` (the
    scored decoder's per-token log-probabilities) every word gets confidence = exp(mean over its tokens)."""
    out: List[Word] = []
    for s, e, f, n in zip(word_start, word_end, word_first, word_ntok):
        pieces = [tokenizer.id_to_str(t) for t in ids[f:f + n]]
        if pieces and pieces[0].startswith(_SP_SPACE):
            pieces[0] = pieces[0][1:]
        conf = None if token_logp is None else mean_logp_confidence(token_logp[f:f + n])
        out.append(Word(text="".join(pieces).strip(), start=s * frame_shift, end=e * frame_shift, confidence=conf))
    return out
