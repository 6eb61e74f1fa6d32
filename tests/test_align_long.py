"""Alignment of long recordings: `longform.plan_windows`, the stitched CTC log-probs, gam_ctc_align_long (one cluster of up
to 16 CTAs per utterance, include/gigaam_b200.h) and `GigaAMASR.align_longform` (INTEGRATION.md §7e).

gam_ctc_align_long computes every state of every frame with the operations of gam_ctc_align, so on inputs both accept its
five outputs must be the same bits, whatever the cluster size; beyond gam_ctc_align's limits it is checked against the
float32 replay of tests/test_align.py (frames, token log-probs and path scores bit for bit, the forward score within the
derived bound).

CPU: the window plan for both front ends, a random-scheduler model of the per-frame cluster protocol (with negative
controls), line / token bookkeeping, the record and the refusals.  GPU: bit identity with gam_ctc_align at forced cluster
sizes, CTA boundaries placed on the edges that cross them, sizes past the old limits, one hour at the token limit, the
stitching, and the public call end to end (single window == align, multi-line segments, determinism, a CUDA-graph replay).
"""
import math
import random
import time

import numpy as np
import pytest
import torch

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, longform, synthetic
from gigaam_b200.longform import FRAME_SAMPLES, line_segments, plan_windows
from gigaam_b200.timestamps_utils import token_flag_table
from gigaam_b200.types import LongformAlignment, Segment, Word

from test_align import F32, INF, NAN, _log_probs, ctc_forward64, ctc_forward_bound, ctc_replay
from test_attention_protocol_model import ProtocolError, _schedule

_CPU_MODELS = {}


def _cpu_model(name):
    if name not in _CPU_MODELS:
        _CPU_MODELS[name] = gigaam.load_model(name, device="cpu", checkpoint=synthetic.synthetic_checkpoint(name, n_layers=1))
    return _CPU_MODELS[name]


# ------------------------------------------------------------------------------------------ CPU: the window plan
@pytest.mark.parametrize("name", ["v2_ctc", "v3_e2e_ctc"])
def test_plan_windows_keep_every_frame_once_inside_its_window(name):
    length = _cpu_model(name)._encoded_length
    rng = random.Random(0)
    sizes = [1, 319, 320, 639, 640, 641, 16000, 479999, 480000, 480001, 480640, 896000, 16000 * 600 + 17]
    sizes += [rng.randrange(1, 3_000_000) for _ in range(60)]
    plans = [(30.0, 4.0), (30.0, 0.0), (10.0, 2.0), (20.0, 19.96), (5.0, 0.04), (0.08, 0.04)]
    for n in sizes:
        for window, overlap in plans:
            if length(n) <= 0:
                with pytest.raises(ValueError, match="no frame"):
                    plan_windows(n, window, overlap, length)
                continue
            wins, T = plan_windows(n, window, overlap, length)
            W = round(window * 25) * FRAME_SAMPLES
            assert T == length(n)
            assert (len(wins) == 1) == (n <= W)
            if n <= W:
                assert wins == [longform.Window(0, n, 0, T)]
            kept = []
            for w in wins:
                assert 0 <= w.start < w.end <= n and w.start % FRAME_SAMPLES == 0 and w.end - w.start <= W
                first, out = w.start // FRAME_SAMPLES, length(w.end - w.start)
                # the additive length rule the plan rests on
                assert length(n) == first + length(n - w.start) or w.end < n
                if w.keep_end > w.keep_start:
                    assert first <= w.keep_start and w.keep_end <= first + out, (n, window, overlap, w)
                kept.extend(range(w.keep_start, w.keep_end))
            assert kept == list(range(T)), (n, window, overlap)
            assert wins[-1].end == n


def test_plan_windows_refusals():
    length = _cpu_model("v2_ctc")._encoded_length
    with pytest.raises(ValueError, match="empty"):
        plan_windows(0, 30.0, 4.0, length)
    with pytest.raises(ValueError, match="multiple"):
        plan_windows(16000, 30.01, 4.0, length)
    with pytest.raises(ValueError, match="multiple"):
        plan_windows(16000, 30.0, 0.5, length)
    with pytest.raises(ValueError, match="overlap"):
        plan_windows(16000, 30.0, -0.04, length)
    with pytest.raises(ValueError, match="overlap"):
        plan_windows(16000, 30.0, 30.0, length)
    with pytest.raises(ValueError, match="max_encoded_frames"):
        plan_windows(16000, 31.0, 4.0, length, 768)         # 776 frames
    assert plan_windows(16000, 30.0, 4.0, length, 768)[1] == length(16000)    # 751 frames fit


# ------------------------------------------------------------------------------------------ CPU: the cluster protocol
class ClusterBarrier:
    """barrier.cluster: one arrival per CTA per phase; a wait for phase j passes once j + 1 phases have completed."""

    def __init__(self, n):
        self.n, self.arrived, self.completions = n, set(), 0

    def arrive(self, who, phase):
        if who in self.arrived or phase != self.completions:
            raise ProtocolError(f"CTA {who} arrives for phase {phase} during phase {self.completions}")
        self.arrived.add(who)
        if len(self.arrived) == self.n:
            self.arrived, self.completions = set(), self.completions + 1


def _cluster_sweep(C, frames, rng, buffers=2, skip_barrier_at=None):
    """ctc_align_long_kernel's per-frame protocol: CTA k reads frame t - 1 from its own buffer and from CTA k - 1's, then
    writes frame t into buffer t % buffers, then arrives on the cluster barrier and waits for it.  Buffer contents are tagged
    with the frame they hold; every read must see frame t - 1.  The steps are split so that the random scheduler can put
    any other CTA's step between them."""
    buf = [[0] * buffers for _ in range(C)]     # frame 0 written by every CTA before the first barrier
    bar = ClusterBarrier(C)

    def cta(k):
        phase = 0
        bar.arrive(k, phase)                    # the barrier that opens frame 1
        yield lambda p=phase: bar.completions > p
        phase += 1
        for t in range(1, frames):
            if buf[k][(t - 1) % buffers] != t - 1:
                raise ProtocolError(f"CTA {k} frame {t}: own buffer holds frame {buf[k][(t - 1) % buffers]}")
            yield lambda: True
            if k > 0 and buf[k - 1][(t - 1) % buffers] != t - 1:
                raise ProtocolError(f"CTA {k} frame {t}: CTA {k - 1}'s buffer holds frame {buf[k - 1][(t - 1) % buffers]}")
            yield lambda: True
            buf[k][t % buffers] = t
            yield lambda: True
            if t == skip_barrier_at:
                continue
            bar.arrive(k, phase)
            yield lambda p=phase: bar.completions > p
            phase += 1
    roles = {f"cta{k}": cta(k) for k in range(C)}
    _schedule(rng, roles, {})


def test_cluster_protocol_model_double_buffer_one_barrier_per_frame():
    for seed in range(200):
        rng = random.Random(seed)
        _cluster_sweep(rng.choice([2, 3, 5, 16]), rng.randrange(2, 24), rng)


@pytest.mark.parametrize("kind", ["one buffer", "missing barrier"])
def test_cluster_protocol_model_negative_controls(kind):
    caught = 0
    for seed in range(200):
        rng = random.Random(seed)
        try:
            if kind == "one buffer":
                _cluster_sweep(4, 12, rng, buffers=1)
            else:
                _cluster_sweep(4, 12, rng, skip_barrier_at=5)
        except ProtocolError:
            caught += 1
    assert caught > 0, kind


# ------------------------------------------------------------------------------------------ CPU: lines, tokens, records
def _word_token_ranges(tok, ids):
    """Token ranges of the words gam_group_words forms (its flag rules, on the host)."""
    flags = token_flag_table(tok).tolist()
    words, cur, visible = [], None, False
    for i, t in enumerate(ids):
        f = flags[t]
        if f & 1 or f & 2:
            if cur is not None and visible:
                words.append(cur)
            cur, visible = None, False
            if f & 1:
                continue
        if cur is None:
            cur = [i, i + 1]
        cur[1] = i + 1
        visible = visible or not f & 4
    if cur is not None and visible:
        words.append(cur)
    return words


def _check_lines(model, lines):
    norm, ids, ranges = model._line_tokens(lines)
    tok = model.decoding.tokenizer
    assert norm == [tok.normalize(x) for x in lines]
    for (a, b), text in zip(ranges, lines):
        assert ids[a:b] == tok.encode(text)
    assert all(r[0] <= s[0] for r, s in zip(ranges, ranges[1:]))
    for a, b in _word_token_ranges(tok, ids):
        inside = [i for i, (lo, hi) in enumerate(ranges) if lo <= a and b <= hi]
        assert len(inside) == 1, (a, b, ranges)
    return norm, ids, ranges


def test_line_tokens_charwise_keep_words_inside_lines():
    model = _cpu_model("v2_ctc")
    tok = model.decoding.tokenizer
    norm, ids, ranges = _check_lines(model, ["Привет мир", "", "  как   дела  ", "x", "Ёлка"])
    assert ranges[1][0] == ranges[1][1] and ranges[3][0] == ranges[3][1]          # empty after normalisation
    assert ids.count(tok.vocab.index(" ")) == 1 + 1 + 1 + 1                       # one in line 0, one in line 2, two between lines
    assert norm[4] == "елка"


def test_line_tokens_sentencepiece_keep_words_inside_lines(tmp_path):
    spm = pytest.importorskip("sentencepiece")
    corpus = tmp_path / "corpus.txt"
    lines = ["привет как дела", "все хорошо спасибо", "ежик в тумане", "где мой телефон", "сегодня хорошая погода"] * 40
    corpus.write_text("\n".join(lines), encoding="utf-8")
    spm.SentencePieceTrainer.train(input=str(corpus), model_prefix=str(tmp_path / "m"), vocab_size=32, model_type="unigram",
                                   character_coverage=1.0, minloglevel=2)
    model = _cpu_model("v2_ctc")
    saved = model.decoding.tokenizer
    try:
        model.decoding.tokenizer = gigaam.decoding.Tokenizer([], str(tmp_path / "m.model"))
        _, ids, ranges = _check_lines(model, ["Привет как дела", "", "ежик в тумане", "где мой"])
        assert sum(b - a for a, b in ranges) == len(ids)                          # no separator tokens
    finally:
        model.decoding.tokenizer = saved


def test_line_segments_rules():
    lines = ["аб", "", "вг де", ""]
    ranges = [(0, 2), (3, 3), (3, 8), (8, 8)]
    frames = [1, 2, -1, 10, 11, 13, 14, 20]
    logp = [-0.5, -0.25, 0.0, -1.0, -1.0, -1.0, -1.0, -1.0]
    words = [Word("аб", 0.04, 0.12, 0.5), Word("вг", 0.4, 0.48, 0.4), Word("де", 0.56, 0.84, 0.3)]
    segs = line_segments(lines, ranges, frames, logp, 0.04, -3.0, words, [0, 3, 6])
    assert [s.words for s in segs] == [words[:1], [], words[1:], []]
    assert (segs[0].start, segs[0].end) == (1 * 0.04, 3 * 0.04)
    assert (segs[1].start, segs[1].end) == (segs[0].end, segs[0].end) and math.isnan(segs[1].confidence)
    assert (segs[2].start, segs[2].end) == (10 * 0.04, 21 * 0.04)
    assert segs[2].confidence == math.exp(-1.0) and segs[0].confidence == math.exp(-0.375)
    assert segs[3].start == segs[3].end == segs[2].end
    first_empty = line_segments(["", "а"], [(0, 0), (0, 1)], [4], [-1.0], 0.04, -1.0)
    assert first_empty[0].start == first_empty[0].end == 0.0 and first_empty[0].words is None
    for vit in (-INF, NAN):
        none = line_segments(lines, ranges, frames, logp, 0.04, vit, words, [0, 3, 6])
        assert all(s.words == [] and math.isnan(s.start) and math.isnan(s.end) and s.confidence == 0.0 for s in none)
    assert all(s.words is None for s in line_segments(lines, ranges, frames, logp, 0.04, -INF))


def test_longform_alignment_record():
    seg = Segment("аб", 0.0, 0.08, [Word("аб", 0.0, 0.08, 0.5)], 0.5)
    empty = Segment("", 0.08, 0.08, [], math.nan)
    a = LongformAlignment([seg, empty, Segment("в", 0.1, 0.2, [Word("в", 0.1, 0.2, 0.9)], 0.9)], -3.5, 0.7)
    assert a.text == "аб в" and str(a) == "аб в" and len(a) == 3 and list(a)[0] is seg
    assert [w.text for w in a.words] == ["аб", "в"]
    assert a == LongformAlignment(segments=list(a.segments), log_likelihood=-3.5, confidence=0.7)
    assert a != LongformAlignment(list(a.segments), -3.5, 0.75)
    assert repr(a).startswith("LongformAlignment(segments=[Segment(text='аб'")
    assert gigaam.LongformAlignment is LongformAlignment


def test_align_longform_refuses_before_device_work():
    model = _cpu_model("v2_ctc")
    wav = np.zeros(16000, np.float32)
    with pytest.raises(ValueError, match="exceed"):
        model.align_longform(wav, "а" * 65537)
    with pytest.raises(ValueError, match="exceed"):
        model.align_longform(wav, ["а" * 40000, "б" * 25536])                   # 65 536 letters + one separator
    with pytest.raises(ValueError, match="empty"):
        model.align_longform(np.zeros(0, np.float32), "а")
    with pytest.raises(ValueError, match="max_encoded_frames"):
        model.align_longform(wav, "а", window=31.0)
    with pytest.raises(ValueError, match="multiple"):
        model.align_longform(wav, "а", overlap=1.01)
    with pytest.raises(ValueError, match="overlap"):
        model.align_longform(wav, "а", overlap=-1.0)
    with pytest.raises(ValueError, match="overlap"):
        model.align_longform(wav, "а", window=10.0, overlap=10.0)
    with pytest.raises(ValueError, match="batch_size"):
        model.align_longform(wav, "а", batch_size=0)
    rnnt = _cpu_model("v2_rnnt")
    with pytest.raises(NotImplementedError, match="CTC"):
        rnnt.align_longform(wav, "а")


# ------------------------------------------------------------------------------------------ GPU helpers
def _dev():
    return torch.device("cuda", 0)


_MODELS = {}


def _model(name, max_frames=None):
    key = (name, max_frames)
    if key not in _MODELS:
        ck = synthetic.synthetic_checkpoint(name, seed=0, n_layers=1)
        _MODELS[key] = gigaam.load_model(name, fp16_encoder=False, device=_dev(), checkpoint=ck, max_encoded_frames=max_frames)
    return _MODELS[key]


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _same(a, b):
    return all(torch.equal(_bits(x), _bits(y)) for x, y in zip(a, b))


def _sizes_allowed(eng, U):
    """Forced cluster sizes gam_test_ctc_align_long accepts at U tokens (it refuses one that leaves a CTA without states)."""
    out = []
    lp = torch.zeros(1, 1, eng.num_classes, device=_dev())
    for c in range(1, 17):
        try:
            eng.ctc_align_long(lp, torch.tensor([1]), torch.zeros(1, U, dtype=torch.int32), torch.tensor([0]), cluster_ctas=c)
            out.append(c)
        except _lib.GamError as e:
            assert "without states" in str(e) or "holds" in str(e), str(e)
    return out


def _ragged_batch(rng, V1, ties):
    """The batch of test_align.py::test_ctc_stage2_ragged_batch_against_replay: ragged lengths, ties, -inf, NaN in used
    and unused entries, bad ids."""
    B, T, U = 12, 300, 100
    lp = _log_probs(rng, (B, T, V1), ties=ties)
    targets = rng.integers(0, V1 - 1, (B, U)).astype(np.int32)
    targets[1, 10:20] = targets[1, 10]
    enc_len = [300, 250, 200, 120, 300, 40, 0, 300, 300, 300, 150, 301]
    target_len = [100, 60, 80, 100, 0, 50, 10, 30, 30, 30, 40, 20]
    lp[2, 5, :] = -INF
    lp[3, :, targets[3, 0]] = -INF
    lp[7, 40, targets[7, 3]] = NAN
    lp[8, 250, :] = NAN
    enc_len[8] = 250
    unused = sorted(set(range(V1 - 1)) - set(targets[9, :30].tolist()))[0]
    lp[9, :, unused] = NAN
    targets[10, 5] = V1 - 1
    targets[11, 3] = -4
    return lp, enc_len, targets, target_len


def _run_both(eng, lp, enc_len, targets, target_len, sizes):
    args = (torch.from_numpy(lp).to(_dev()), torch.tensor(enc_len), torch.from_numpy(targets), torch.tensor(target_len))
    want = eng.ctc_align(*args)
    for c in sizes:
        got = eng.ctc_align_long(*args, cluster_ctas=c)
        assert eng.last_align_long_plan[0] == c
        assert _same(got, want), c
    assert _same(eng.ctc_align_long(*args), want)
    return want


# ------------------------------------------------------------------------------------------ GPU: kernel
@pytest.mark.gpu
@pytest.mark.parametrize("V1", [34, 257])
def test_bit_identical_to_ctc_align_on_the_ragged_batch(V1):
    eng = _model("v2_ctc" if V1 == 34 else "v3_e2e_ctc")._get_engine()
    rng = np.random.default_rng(V1)
    sizes = _sizes_allowed(eng, 100)
    assert sizes[:3] == [1, 2, 3] and sizes[-1] == 13              # S = 201: 13 CTAs of 16 states; 14 to 16 leave one empty
    for ties in (False, True):
        _run_both(eng, *_ragged_batch(rng, V1, ties), [1, 2, 3, sizes[-1]])
    with pytest.raises(_lib.GamError, match="without states"):
        eng.ctc_align_long(torch.zeros(1, 4, V1, device=_dev()), torch.tensor([4]), torch.zeros(1, 100, dtype=torch.int32),
                           torch.tensor([3]), cluster_ctas=16)


@pytest.mark.gpu
def test_bit_identical_to_ctc_align_at_its_token_limit():
    eng = _model("v3_e2e_ctc", 5000)._get_engine()
    rng = np.random.default_rng(7)
    T, U, V1 = 5000, 4096, 257
    lp = _log_probs(rng, (2, T, V1))
    targets = rng.integers(0, V1 - 1, (2, U)).astype(np.int32)
    assert _sizes_allowed(eng, U)[-1] == 16
    _run_both(eng, lp, [T, 4500], targets, [U, 2000], [1, 2, 3, 16])
    assert eng.last_align_long_plan == (16, 528)


def _check_replay(out, lp, enc_len, targets, target_len):
    fr, tok, vit, ll, rows = (t.cpu().numpy() for t in out)
    for b in range(lp.shape[0]):
        Tb, Ub = enc_len[b], target_len[b]
        y = targets[b, :Ub].tolist()
        r_fr, r_tok, r_vit, r_rows = ctc_replay(lp[b], Tb, y, targets.shape[1])
        assert np.array_equal(fr[b], r_fr), b
        assert np.array_equal(tok[b].view(np.uint32), r_tok.view(np.uint32)), b
        assert F32(vit[b]).view(np.uint32) == F32(r_vit).view(np.uint32), b
        assert rows[b] == r_rows
        want, mags = ctc_forward64(lp[b], Tb, y)
        assert abs(ll[b] - want) <= ctc_forward_bound(mags, want), (b, ll[b], want)


@pytest.mark.gpu
def test_cta_boundaries_on_the_edges_that_cross_them():
    """P = 48 (C = 2) and P = 32 (C = 3) states per CTA at U = 40.  Utterance 0 repeats the labels on both sides of each
    boundary (no skip edge crosses), utterance 1 has only distinct neighbours (the skip edge s - 2 of the second state of a
    CTA crosses), and utterances 2 / 3 end with S - 1 on a boundary (S - 2 | S - 1 in different CTAs for C = 2 / 3)."""
    eng = _model("v2_ctc")._get_engine()
    V1, T, U = 34, 160, 40
    rng = np.random.default_rng(11)
    targets = np.zeros((4, U), np.int32)
    targets[1] = np.arange(U) % (V1 - 1)
    targets[0] = targets[1]
    for s in (48, 32, 64):                          # label states s + 1 repeat their left neighbour
        targets[0, s // 2] = targets[0, s // 2 - 1]
    targets[2], targets[3] = targets[1], targets[1]
    target_len = [U, U, 24, 16]
    enc_len = [T, T, T, T - 30]
    for c, p in ((2, 48), (3, 32)):
        for ties in (False, True):
            lp = _log_probs(rng, (4, T, V1), ties=ties)
            out = eng.ctc_align_long(torch.from_numpy(lp).to(_dev()), torch.tensor(enc_len), torch.from_numpy(targets),
                                     torch.tensor(target_len), cluster_ctas=c)
            assert eng.last_align_long_plan == (c, p)
            _check_replay(out, lp, enc_len, targets, target_len)


@pytest.mark.gpu
def test_beyond_the_old_limits_against_the_replay():
    eng = _model("v2_ctc")._get_engine()
    rng = np.random.default_rng(5)
    V1 = 34
    T, U = 20000, 8000
    lp = _log_probs(rng, (1, T, V1))
    targets = rng.integers(0, V1 - 1, (1, U)).astype(np.int32)
    out = eng.ctc_align_long(torch.from_numpy(lp).to(_dev()), torch.tensor([T]), torch.from_numpy(targets), torch.tensor([U]))
    assert eng.lib.gam_ctc_align_workspace_bytes(eng.handle, 1, T, U) == -1          # past gam_ctc_align's limits
    _check_replay(out, lp, [T], targets, [U])
    # ragged B = 3 around the CTA boundaries of C = 3 at U = 3000 (P = 2016 states)
    T, U = 7000, 3000
    lp = _log_probs(rng, (3, T, V1))
    targets = rng.integers(0, V1 - 1, (3, U)).astype(np.int32)
    enc_len, target_len = [7000, 6000, 5000], [3000, 1008, 1007]      # S - 1 = 2016 = the first boundary, and S - 1 = 2014
    out = eng.ctc_align_long(torch.from_numpy(lp).to(_dev()), torch.tensor(enc_len), torch.from_numpy(targets),
                             torch.tensor(target_len), cluster_ctas=3)
    assert eng.last_align_long_plan == (3, 2016)
    _check_replay(out, lp, enc_len, targets, target_len)


@pytest.mark.gpu
@pytest.mark.parametrize("V1", [34, 257])
def test_one_hour_at_the_token_limit(V1):
    """T = 90 000 frames (one hour), U = 65 536 tokens on planted log-probs: token i is peaked at frame f_i (log-prob 0
    there, -30 elsewhere), blank peaked on every other frame.  The best path is the planted one; its score is the fp32 sum
    of its entries in t order."""
    eng = _model("v2_ctc" if V1 == 34 else "v3_e2e_ctc")._get_engine()
    T, U = 90000, 65536
    g = torch.Generator().manual_seed(V1)
    steps = torch.randint(1, V1 - 1, (U,), generator=g)                      # no label repeats its neighbour
    y = (torch.cumsum(steps, 0) % (V1 - 1)).to(torch.int32)
    gaps = torch.full((U,), 1, dtype=torch.int64)
    gaps[torch.randperm(U, generator=g)[:T - U - 2000]] += 1
    f = torch.cumsum(gaps, 0) - 1 + 1000
    assert int(f[-1]) < T
    lp = torch.full((1, T, V1), -30.0, device=_dev())
    lp[0, :, V1 - 1] = 0.0
    lp[0, f.to(_dev()), y.long().to(_dev())] = 0.0
    lp[0, f.to(_dev()), V1 - 1] = -30.0
    lp[0, f[::7].to(_dev()), y[::7].long().to(_dev())] = -0.25            # a few non-zero terms make the sum's order matter
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = eng.ctc_align_long(lp, torch.tensor([T]), y[None], torch.tensor([U]))
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    print(f"\none hour, V+1 = {V1}: {wall * 1e3:.0f} ms wall, peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
    frames, _, vit, ll, rows = (t.cpu() for t in out)
    assert torch.equal(frames[0].long(), f)
    path = np.zeros(T, F32)
    path[f.numpy()] = np.where(np.arange(U) % 7 == 0, F32(-0.25), F32(0.0))
    s = F32(0.0)
    for x in path:
        s = F32(s + x)
    assert F32(vit[0]) == s and int(rows[0]) == T and math.isfinite(float(ll[0]))
    with pytest.raises(ValueError):
        eng.ctc_align_long(lp[:, :10], torch.tensor([10]), torch.zeros(1, U + 1, dtype=torch.int32), torch.tensor([1]))


# ------------------------------------------------------------------------------------------ GPU: stitching, end to end
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v3_e2e_ctc"])
def test_stitched_rows_equal_each_window_alone(name):
    model = _model(name)
    wav, _ = synthetic.synthetic_audio(1, 600.0, seed=3)
    wav = wav[0].to(_dev())
    n = wav.numel() - 12345
    wav = wav[:n]
    windows, T = plan_windows(n, 30.0, 4.0, model._encoded_length, 768)
    assert len(windows) > 20 and T == model._get_engine().encoded_frames(model._get_engine().logmel_frames(n))
    lp = longform.stitch_ctc_log_probs(model, wav, windows, T, batch_size=8)
    for w in windows:
        with torch.inference_mode():
            enc, enc_len = model(wav[None, w.start:w.end], torch.tensor([w.end - w.start], device=_dev()))
            alone = model.head(enc)[0]
        first = w.start // FRAME_SAMPLES
        assert int(enc_len[0]) == alone.shape[0] >= w.keep_end - first
        assert torch.equal(_bits(lp[0, w.keep_start:w.keep_end]), _bits(alone[w.keep_start - first:w.keep_end - first])), w


def _greedy_text(model, wav):
    return model.transcribe(wav.cpu()).text


@pytest.mark.gpu
def test_single_window_equals_align():
    model = _model("v2_ctc")
    wav, _ = synthetic.synthetic_audio(1, 20.0, seed=5)
    wav = wav[0]
    text = _greedy_text(model, wav) or "а"
    for t in (text, text[: len(text) // 2], ""):
        a = model.align(wav, t)
        lf = model.align_longform(wav, t)
        assert len(lf.segments) == 1 and lf.segments[0].text == a.text
        assert lf.log_likelihood == a.log_likelihood and lf.confidence == a.confidence
        assert lf.segments[0].words == a.words, t


@pytest.mark.gpu
def test_multi_line_text_over_five_minutes():
    model = _model("v2_ctc")
    wav, _ = synthetic.synthetic_audio(1, 300.0, seed=9)
    wav = wav[0]
    lines = []
    for k in range(0, wav.numel(), 20 * 16000):
        t = _greedy_text(model, wav[k:k + 20 * 16000])
        lines.append(t[: len(t) // 2])             # half of each piece's greedy text: the whole text stays feasible
    lines.insert(3, "")
    res = model.align_longform(wav, lines)
    assert len(res.segments) == len(lines)
    assert math.isfinite(res.log_likelihood) and 0.0 < res.confidence <= 1.0
    starts = [s.start for s in res.segments]
    assert starts == sorted(starts)
    for seg in res.segments:
        assert seg.start <= seg.end
        for w in seg.words:
            assert seg.start <= w.start <= w.end <= seg.end
        if not seg.text:
            assert seg.words == [] and math.isnan(seg.confidence)
    assert res.segments[-1].end <= wav.numel() / 16000 + 1e-9
    again = model.align_longform(wav, lines)
    assert repr(again) == repr(res)
    plain = model.align_longform(wav, lines, word_timestamps=False)
    assert all(s.words is None for s in plain.segments)
    assert [(s.start, s.end) for s in plain.segments] == [(s.start, s.end) for s in res.segments]


@pytest.mark.gpu
def test_graph_capture_of_ctc_align_long():
    eng = _model("v2_ctc")._get_engine()
    rng = np.random.default_rng(2)
    lp = torch.from_numpy(_log_probs(rng, (2, 3000, 34))).to(_dev())
    targets = torch.from_numpy(rng.integers(0, 33, (2, 1200)).astype(np.int32)).to(_dev())
    enc_len = torch.tensor([3000, 2500], dtype=torch.int32, device=_dev())
    tlen = torch.tensor([1200, 700], dtype=torch.int32, device=_dev())
    want = [t.clone() for t in eng.ctc_align_long(lp, enc_len, targets, tlen)]
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        eng.ctc_align_long(lp, enc_len, targets, tlen)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            captured = eng.ctc_align_long(lp, enc_len, targets, tlen)
    torch.cuda.current_stream().wait_stream(stream)
    for t in captured:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert _same(captured, want)
