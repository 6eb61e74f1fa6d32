"""Transcription of recordings of any length without a VAD: resumable greedy decoding (gam_ctc_greedy_resume /
gam_rnnt_greedy_resume, include/gigaam_b200.h), `longform.decode_windows`, the segmentation rules and
`GigaAMASR.transcribe_windowed` (INTEGRATION.md §7f).

The point of the resumable decoders is one invariant: an utterance decoded in consecutive ranges of frames, with the state
carried on the device, gives one gam_*_greedy(_scored) call's ids, frames, counts, token log-probs and path scores bit for
bit.  CPU: the segmentation rules, the refusals and the exported symbols.  GPU: the invariant for both heads (with chunk edges
on pending RNN-T steps and on CTC repeats, and for 32 RNN-T streams decoded in groups of 8), truncation, the stitched encoder output, one window == transcribe, and flat
device memory.
"""
import ctypes
import math
import random

import numpy as np
import pytest
import torch

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, longform, synthetic
from gigaam_b200.longform import FRAME_SAMPLES, plan_windows, segment_cuts, windowed_segments
from gigaam_b200.types import LongformTranscriptionResult, Word

_CPU_MODELS = {}


def _cpu_model(name):
    if name not in _CPU_MODELS:
        _CPU_MODELS[name] = gigaam.load_model(name, device="cpu", checkpoint=synthetic.synthetic_checkpoint(name, n_layers=1))
    return _CPU_MODELS[name]


# ------------------------------------------------------------------------------------------ CPU: segmentation
def test_cuts_at_pauses_fall_at_gap_middles():
    spans = [(2, 5), (6, 9), (40, 44), (45, 50), (80, 81)]
    # gaps of 1, 31, 1 and 30 frames; 0.04 s per frame, pause 1.0 s = 25 frames
    assert segment_cuts(spans, 100, 0.04, 1.0, 1e9) == [0, (9 + 40) // 2, (50 + 80) // 2, 100]
    assert segment_cuts(spans, 100, 0.04, 1.22, 1e9) == [0, (9 + 40) // 2, 100]                   # 30 frames = 1.2 s
    assert segment_cuts(spans, 100, 0.04, 0.0, 1e9) == [0, 5, 24, 44, 65, 100]                     # every gap, even of 1 frame
    assert segment_cuts([], 100, 0.04, 0.0, 1.0) == [0, 100]
    assert segment_cuts([(3, 9)], 100, 0.04, 0.0, 1.0) == [0, 100]                                 # no inner gap left
    # overlapping spans (RNN-T tokens of one frame) are never cut
    assert segment_cuts([(0, 5), (4, 9), (9, 12)], 20, 0.04, 0.0, 1e9) == [0, 9, 20]


def test_max_segment_splits_at_the_longest_inner_gap():
    spans = [(0, 10), (12, 20), (30, 40), (41, 50), (55, 60), (61, 99)]     # inner gaps 2, 10, 1, 5, 1
    cuts = segment_cuts(spans, 100, 0.04, 100.0, 2.0)                        # 2.0 s = 50 frames
    assert cuts[0] == 0 and cuts[-1] == 100
    assert (20 + 30) // 2 in cuts                                            # the 10-frame gap first
    assert (50 + 55) // 2 in cuts                                            # then the 5-frame gap of [25, 100)
    for a, b in zip(cuts, cuts[1:]):
        inner = [(e, s) for (_, e), (s, _) in zip(spans, spans[1:]) if a < e and s < b]
        assert (b - a) * 0.04 <= 2.0 or not inner, (a, b)
    # equal gaps: the first one
    assert segment_cuts([(0, 10), (14, 20), (24, 30)], 30, 1.0, 100.0, 20.0) == [0, 12, 30]


class _Tok:
    vocab = ["а", "б", " "]

    def decode(self, ids):
        return "".join(self.vocab[i] for i in ids)


def test_segments_tile_the_recording_and_rows_add_up():
    rng = np.random.default_rng(0)
    T, shift = 500, 0.04
    frames = sorted(rng.choice(np.arange(3, T - 3), 60, replace=False).tolist())
    ids = rng.integers(0, 2, 60).tolist()
    ids[::6] = [2] * len(ids[::6])
    word_spans = [(f, f + 1) for f in frames[::6]]
    cuts = segment_cuts(word_spans, T, shift, 0.2, 3.0)
    words = [Word(str(i), s * shift, e * shift, None) for i, (s, e) in enumerate(word_spans)]
    frame_logp = rng.normal(-0.5, 0.2, T)
    frame_rows = rng.integers(0, 3, T).astype(np.int32)
    duration = T * shift + 0.013
    segs = windowed_segments(_Tok(), ids, frames, cuts, shift, duration, words, [s for s, _ in word_spans], frame_logp, frame_rows)
    assert segs[0].start == 0.0 and segs[-1].end == duration
    assert all(a.end == b.start for a, b in zip(segs, segs[1:]))
    assert "".join(s.text for s in segs) == _Tok().decode(ids)
    assert sum(len(s.words) for s in segs) == len(words)
    total = 0
    for k, s in enumerate(segs):
        a, b = cuts[k], cuts[k + 1]
        rows = int(frame_rows[a:b].sum())
        total += rows
        want = math.exp(float(frame_logp[a:b].sum()) / rows) if rows else math.nan
        assert s.confidence == want or (math.isnan(want) and math.isnan(s.confidence))
        for w in s.words:
            assert s.start <= w.start < s.end
    assert total == int(frame_rows.sum())
    plain = windowed_segments(_Tok(), ids, frames, cuts, shift, duration, None, [s for s, _ in word_spans])
    assert all(s.words is None and s.confidence is None for s in plain)


def test_no_token_recording_gives_one_empty_segment():
    cuts = segment_cuts([], 80, 0.04, 1.0, 25.0)
    segs = windowed_segments(_Tok(), [], [], cuts, 0.04, 3.21, [], [], np.full(80, -0.1), np.ones(80, np.int32))
    assert len(segs) == 1 and segs[0].text == "" and segs[0].words == []
    assert (segs[0].start, segs[0].end) == (0.0, 3.21)
    assert segs[0].confidence == pytest.approx(math.exp(-0.1))
    assert math.isnan(windowed_segments(_Tok(), [], [], cuts, 0.04, 3.21, None, [], np.zeros(80), np.zeros(80, np.int32))[0].confidence)


def test_transcribe_windowed_refuses_before_device_work():
    model = _cpu_model("v2_ctc")
    wav = np.zeros(16000, np.float32)
    with pytest.raises(ValueError, match="empty"):
        model.transcribe_windowed(np.zeros(0, np.float32))
    with pytest.raises(ValueError, match="multiple"):
        model.transcribe_windowed(wav, window=30.01)
    with pytest.raises(ValueError, match="multiple"):
        model.transcribe_windowed(wav, overlap=0.5)
    with pytest.raises(ValueError, match="overlap"):
        model.transcribe_windowed(wav, overlap=-0.04)
    with pytest.raises(ValueError, match="overlap"):
        model.transcribe_windowed(wav, window=10.0, overlap=10.0)
    with pytest.raises(ValueError, match="max_encoded_frames"):
        model.transcribe_windowed(wav, window=31.0)
    with pytest.raises(ValueError, match="batch_size"):
        model.transcribe_windowed(wav, batch_size=0)
    with pytest.raises(ValueError, match="pause"):
        model.transcribe_windowed(wav, pause=-0.5)
    with pytest.raises(ValueError, match="max_segment"):
        model.transcribe_windowed(wav, max_segment=0.0)
    with pytest.raises(ValueError, match="max_segment"):
        _cpu_model("v2_rnnt").transcribe_windowed(wav, max_segment=-1.0)
    assert not hasattr(gigaam.GigaAM, "transcribe_windowed")


def test_resume_symbols_are_exported():
    lib = _lib.load()
    for name in ("gam_decode_state_bytes", "gam_decode_state_init", "gam_decode_resume_workspace_bytes", "gam_ctc_greedy_resume",
                 "gam_rnnt_greedy_resume"):
        assert name in _lib.EXPORTS and hasattr(lib, name)


# ------------------------------------------------------------------------------------------ GPU helpers
def _dev():
    return torch.device("cuda", 0)


_MODELS = {}


def _model(name, blank_shift=0.0):
    key = (name, blank_shift)
    if key not in _MODELS:
        ck = synthetic.synthetic_checkpoint(name, seed=0, n_layers=1)
        if blank_shift:
            ck["state_dict"]["head.joint.joint_net.1.bias"][-1] += blank_shift
        _MODELS[key] = gigaam.load_model(name, fp16_encoder=False, device=_dev(), checkpoint=ck)
    return _MODELS[key]


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _splits(rng, L, how):
    """Consecutive ranges [b_i, b_{i+1}) covering [0, L): one, two, seven or a random number of chunks, some empty."""
    if how == 1:
        return [0, L]
    if how in (2, 7):
        return [0] + sorted(rng.randint(0, L) for _ in range(how - 1)) + [L]
    cuts = sorted(rng.randint(0, L) for _ in range(rng.randint(1, 12)))
    return [0] + cuts + [cuts[-1]] + [L]                           # a repeated cut: an empty chunk


def _resume_all(eng, enc, lens, bounds, max_out, scores, frame_base=None):
    """Decode every row of enc in its chunks; returns the buffers and whether a chunk edge fell on a pending step."""
    B, T, _ = enc.shape
    state = eng.decode_state(B)
    out = eng.decode_buffers(B, max_out, T + 5, scores=scores)
    fb = torch.zeros(B, dtype=torch.int32, device=_dev()) if frame_base is None else frame_base
    pending = False
    for c in range(max(len(b) for b in bounds) - 1):
        lo = [b[c] if c + 1 < len(b) else lens[i] for i, b in enumerate(bounds)]
        hi = [b[c + 1] if c + 1 < len(b) else lens[i] for i, b in enumerate(bounds)]
        eng.greedy_resume(enc, torch.tensor(lo, dtype=torch.int32, device=_dev()), torch.tensor(hi, dtype=torch.int32, device=_dev()),
                          fb, state, out, scores)
        if eng.head_type == 2:
            pend = state.view(torch.int32)[:, 1].cpu()
            pending |= any(int(pend[i]) == 1 and lo[i] < hi[i] < lens[i] for i in range(B))
    return out, state, pending


def _check_same(out, want, scores):
    n = want[2].cpu()
    assert torch.equal(out.counts.cpu(), n)
    for b in range(len(n)):
        k = int(n[b])
        assert torch.equal(out.ids[b, :k].cpu(), want[0][b, :k].cpu()), b
        assert torch.equal(out.frames[b, :k].cpu(), want[1][b, :k].cpu()), b
        if scores:
            assert torch.equal(_bits(out.token_logp[b, :k]).cpu(), _bits(want[3][b, :k]).cpu()), b
    if scores:
        assert torch.equal(_bits(out.path_logp).cpu(), _bits(want[4]).cpu())
        assert torch.equal(out.path_rows.cpu(), want[5].cpu())
        assert torch.equal(out.frame_rows.sum(1).cpu(), want[5].cpu())


# ------------------------------------------------------------------------------------------ GPU: the invariant
@pytest.mark.gpu
@pytest.mark.parametrize("name,blank_shift", [("v2_rnnt", 0.0), ("v2_rnnt", -1000.0), ("v3_e2e_rnnt", -1000.0), ("v3_e2e_rnnt", -4.0)])
def test_rnnt_resume_is_bit_identical(name, blank_shift):
    eng = _model(name, blank_shift)._get_engine()
    g = torch.Generator().manual_seed(len(name) + int(blank_shift))
    B, T = 4, 700
    enc = (torch.randn(B, T, eng.d_model, generator=g) * 0.5).to(_dev())
    lens = [700, 613, 1, 257]
    lens_d = torch.tensor(lens, dtype=torch.int32)
    max_out = eng.hyp_width(T)
    rng = random.Random(7)
    saw_pending = False
    for scores in (False, True):
        want = eng.greedy(enc, lens_d, scores=scores)
        for how in (1, 2, 7, "random", "random"):
            bounds = [_splits(rng, L, how if b % 2 == 0 else rng.choice([1, 2, 7, "random"])) for b, L in enumerate(lens)]
            out, state, pending = _resume_all(eng, enc, lens, bounds, max_out, scores)
            saw_pending |= pending
            _check_same(out, want, scores)
            assert torch.equal(state.view(torch.int32)[:, 2].cpu(), want[2].cpu())          # the true count
    if blank_shift < -100:
        assert saw_pending, "no chunk edge fell on a pending LSTM step"


@pytest.mark.gpu
def test_rnnt_resume_of_many_streams_is_bit_identical():
    """32 streams decode in groups of 8 (NH = 2), the width a one-shot call of that batch takes too; the folds do not depend
    on the group width, so resuming them in random chunks still gives the one-shot bits."""
    eng = _model("v3_e2e_rnnt", -4.0)._get_engine()
    B, T, H, V1 = 32, 120, 320, eng.num_classes
    # the launch plan of this batch, read with all lengths 0: NH (plan[0]) = 2
    f32 = [torch.zeros(shape, device=_dev()) for shape in ((B, 1, H), (V1, 4 * H), (H, 4 * H), (H, H), (H,), (V1, H), (V1,))]
    i32 = [torch.zeros(shape, dtype=torch.int32, device=_dev()) for shape in ((B,), (B, 1), (B, 1), (B,))]
    plan = (ctypes.c_int32 * 7)()
    rc = eng.lib.gam_test_rnnt_greedy(eng.handle, f32[0].data_ptr(), i32[0].data_ptr(), *[t.data_ptr() for t in f32[1:]], B, 1, V1, 1, 1,
                                      *[t.data_ptr() for t in i32[1:]], ctypes.cast(plan, ctypes.c_void_p), eng._stream())
    _lib.check(eng.lib, eng.handle, rc, "gam_test_rnnt_greedy")
    assert plan[0] == 2, list(plan)
    g = torch.Generator().manual_seed(32)
    enc = (torch.randn(B, T, eng.d_model, generator=g) * 0.5).to(_dev())
    rng = random.Random(32)
    lens = [rng.randint(1, T) for _ in range(B)]
    lens_d = torch.tensor(lens, dtype=torch.int32)
    for scores in (False, True):
        want = eng.greedy(enc, lens_d, scores=scores)
        bounds = [_splits(rng, L, rng.choice([1, 2, 7, "random"])) for L in lens]
        out, state, _ = _resume_all(eng, enc, lens, bounds, eng.hyp_width(T), scores)
        _check_same(out, want, scores)
        assert torch.equal(state.view(torch.int32)[:, 2].cpu(), want[2].cpu())


@pytest.mark.gpu
def test_rnnt_resume_truncates_as_the_one_shot_kernel():
    model = _model("v2_rnnt", -1000.0)
    eng = model._get_engine()
    g = torch.Generator().manual_seed(3)
    B, T, max_out = 2, 300, 777                        # every frame emits max_symbols tokens: 3000 > 777
    enc = (torch.randn(B, T, eng.d_model, generator=g) * 0.5).to(_dev())
    lens = torch.tensor([300, 250], dtype=torch.int32, device=_dev())
    ids = torch.full((B, max_out), -1, dtype=torch.int32, device=_dev())
    frames, counts = torch.full_like(ids, -1), torch.zeros(B, dtype=torch.int32, device=_dev())
    tok, path, rows = torch.zeros(B, max_out, device=_dev()), torch.zeros(B, device=_dev()), torch.zeros(B, dtype=torch.int32, device=_dev())
    ws = torch.empty(int(eng.lib.gam_decode_scored_workspace_bytes(eng.handle, B, T)), dtype=torch.uint8, device=_dev())
    rc = eng.lib.gam_rnnt_greedy_scored(eng.handle, enc.data_ptr(), lens.data_ptr(), B, T, ws.data_ptr(), ws.numel(), ids.data_ptr(),
                                        frames.data_ptr(), counts.data_ptr(), max_out, tok.data_ptr(), path.data_ptr(), rows.data_ptr(),
                                        eng._stream())
    _lib.check(eng.lib, eng.handle, rc, "gam_rnnt_greedy_scored")
    assert int(counts.min()) == max_out
    bounds = [[0, 37, 120, 121, 300], [0, 250]]
    out, state, _ = _resume_all(eng, enc, [300, 250], bounds, max_out, True)
    _check_same(out, (ids, frames, counts, tok, path, rows), True)
    assert state.view(torch.int32)[:, 2].tolist() == [3000, 2500]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v3_e2e_ctc"])
def test_ctc_resume_is_bit_identical(name):
    eng = _model(name)._get_engine()
    g = torch.Generator().manual_seed(11)
    B, T = 4, 700
    enc = (torch.randn(B, T, eng.d_model, generator=g) * 0.5).to(_dev())
    lens = [700, 613, 1, 333]
    lens_d = torch.tensor(lens, dtype=torch.int32)
    # planted: frames 99 and 100 of row 0 get the row of an emitted frame, so one label runs across the edge at 100
    ids0, frames0, counts0 = eng.greedy(enc, lens_d)
    f = int(frames0[0, int(counts0[0]) // 2])
    enc[0, 99] = enc[0, f]
    enc[0, 100] = enc[0, f]
    rng = random.Random(5)
    for scores in (False, True):
        want = eng.greedy(enc, lens_d, scores=scores)
        n0 = int(want[2][0])
        at = [int(x) for x in want[1][0, :n0].cpu()]
        assert 100 not in at                                         # the run through frame 100 collapsed to one token
        for how in (1, 2, 7, "random", "random"):
            bounds = [_splits(rng, L, how if b % 2 == 0 else rng.choice([1, 2, 7, "random"])) for b, L in enumerate(lens)]
            bounds[0] = sorted(set(bounds[0]) | {100})
            out, _, _ = _resume_all(eng, enc, lens, bounds, T, scores)
            _check_same(out, want, scores)


# ------------------------------------------------------------------------------------------ GPU: the public path
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v2_rnnt"])
def test_windowed_decode_equals_the_stitched_encoder_output(name):
    model = _model(name)
    eng = model._get_engine()
    wav, _ = synthetic.synthetic_audio(1, 300.0, seed=4)
    wav = wav[0][: 300 * 16000 - 4321]
    windows, T = plan_windows(wav.numel(), 30.0, 4.0, model._encoded_length, 768)
    rows = []
    with torch.inference_mode():
        for w in windows:
            enc, _ = model(wav[None, w.start:w.end].to(_dev()), torch.tensor([w.end - w.start], device=_dev()))
            first = w.start // FRAME_SAMPLES
            rows.append(enc.transpose(1, 2)[0, w.keep_start - first:w.keep_end - first])
        stitched = torch.cat(rows)[None].contiguous()
        assert stitched.shape[1] == T
        want = eng.greedy(stitched, torch.tensor([T]), scores=True)
        out = longform.decode_windows(model, wav.pin_memory(), windows, T, batch_size=4, scores=True)
    _check_same(out, want, True)
    assert int(out.counts[0]) > 10


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v2_rnnt"])
def test_one_window_equals_transcribe(name):
    model = _model(name)
    wav, _ = synthetic.synthetic_audio(1, 20.0, seed=6)
    wav = wav[0]
    ref = model.transcribe(wav, word_timestamps=True, confidence=True)
    res = model.transcribe_windowed(wav, word_timestamps=True, confidence=True, pause=1e9)
    assert isinstance(res, LongformTranscriptionResult) and len(res.segments) == 1
    seg = res.segments[0]
    assert seg.text == ref.text and seg.words == ref.words
    assert (seg.start, seg.end) == (0.0, wav.numel() / 16000)
    assert seg.confidence == pytest.approx(ref.confidence, rel=1e-6)
    plain = model.transcribe_windowed(wav, pause=1e9)
    assert plain.segments[0].text == ref.text and plain.segments[0].words is None and plain.segments[0].confidence is None


@pytest.mark.gpu
def test_segments_tile_a_long_recording():
    model = _model("v2_rnnt")
    wav, _ = synthetic.synthetic_audio(1, 150.0, seed=8)
    wav = wav[0]
    res = model.transcribe_windowed(wav, word_timestamps=True, confidence=True, pause=0.2, max_segment=10.0)
    segs = res.segments
    assert segs[0].start == 0.0 and segs[-1].end == wav.numel() / 16000
    assert all(a.end == b.start for a, b in zip(segs, segs[1:]))
    for s in segs:
        assert all(s.start <= w.start and w.end <= s.end + 1e-9 for w in s.words)
    again = model.transcribe_windowed(wav, word_timestamps=True, confidence=True, pause=0.2, max_segment=10.0)
    assert repr(again) == repr(res)


@pytest.mark.gpu
def test_device_memory_stays_flat():
    model = _model("v2_ctc")
    peaks = {}
    for minutes in (2, 20, 2, 20):
        wav, _ = synthetic.synthetic_audio(1, 60.0 * minutes, seed=minutes)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        model.transcribe_windowed(wav[0], batch_size=4, confidence=True, word_timestamps=True)
        torch.cuda.synchronize()
        peaks[minutes] = torch.cuda.max_memory_allocated() - base
    print(f"\npeak above baseline: 2 min {peaks[2] / 2**20:.1f} MiB, 20 min {peaks[20] / 2**20:.1f} MiB")
    assert peaks[20] - peaks[2] < 64 * 2**20
