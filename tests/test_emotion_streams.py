"""Emotions of live streams (INTEGRATION.md, "Emotions over time"): `GigaAMEmo.streaming` and `EmotionStreamServer`.

A closed stream equals `emotion_timeline` over the same samples, window, overlap, span and hop, bit for bit; the spans a
stream emits while it runs are the timeline's spans without the tail span, with the same probabilities; device memory does
not grow with a stream's duration.  All on the GPU (the refusals are in tests/test_emotion_timeline.py)."""
import random

import pytest
import torch

import gigaam_b200 as gigaam
from gigaam_b200 import synthetic
from gigaam_b200.longform import emotion_spans

FRAME = 0.04
_MODEL = {}


def _model():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (there is no CPU fallback to test instead)"
    if "emo" not in _MODEL:
        _MODEL["emo"] = gigaam.load_model("emo", device=torch.device("cuda", 0), synthetic=True)
    return _MODEL["emo"]


def _frames(span):
    return round(span.start / FRAME), round(span.end / FRAME)


def _check_stream(model, wav, updates, closed, rate, span, hop, window=8.0, overlap=4.0):
    want = model.emotion_timeline(wav, window=window, overlap=overlap, span=span, hop=hop, sample_rate=rate)
    assert closed == want, "a closed stream differs from emotion_timeline"
    T = want.frame_logits.shape[0]
    plan = emotion_spans(T, round(span / FRAME), round(hop / FRAME))
    emitted = [s for u in updates for s in u.new_spans]
    regular = plan if T <= round(span / FRAME) else [p for p in plan if (p[0] % round(hop / FRAME)) == 0 and p[1] <= T]
    assert len(emitted) <= len(regular)
    assert [_frames(s) for s in emitted] == regular[:len(emitted)]
    for i, s in enumerate(emitted):
        assert list(s.probs) == want.names
        assert torch.equal(torch.tensor(list(s.probs.values()), dtype=torch.float32), want.probs[i])
    # every regular span whose frames were final before the close was emitted by a step
    final = max((round(u.final_until / FRAME) for u in updates), default=0)
    assert len(emitted) == sum(1 for a, b in regular if b <= final and not (T <= round(span / FRAME) and b < round(span / FRAME)))
    return len(emitted)


@pytest.mark.gpu
def test_streams_equal_the_timeline_bit_for_bit():
    """Five streams of different lengths pushed in random chunks (one-sample pushes included), opened and closed at different
    steps, with a hop shorter than the span; and a server at 8 kHz with a hop longer than the span."""
    model = _model()
    rng = random.Random(5)
    for rate, span, hop, secs in ((16000, 4.0, 1.0, [31.3, 12.0, 47.9, 8.0, 3.1]), (8000, 2.0, 3.0, [26.7, 40.1])):
        srv = model.streaming(window=8.0, overlap=4.0, span=span, hop=hop, batch_size=3, sample_rate=rate)
        wavs = [synthetic.synthetic_audio(1, s, seed=70 + i)[0][0] for i, s in enumerate(secs)]
        if rate != 16000:
            wavs = [w[::2].contiguous() for w in wavs]
        pos = [0] * len(wavs)
        ids = {}
        updates = {i: [] for i in range(len(wavs))}
        emitted = 0
        opened = 0
        steps = 0
        while ids or opened < len(wavs):
            if opened < len(wavs) and (steps % 3 == 0 or not ids):
                ids[opened] = srv.open()
                opened += 1
            for i, sid in list(ids.items()):
                n = rng.choice([1, 1, 17, 640, 3000, 8000, 24000, 40000])
                srv.push(sid, wavs[i][pos[i]:pos[i] + n].numpy())
                pos[i] += n
            by_stream = {u.stream: u for u in srv.step()}
            for i, sid in ids.items():
                if sid in by_stream:
                    u = by_stream[sid]
                    assert u.final_until >= (updates[i][-1].final_until if updates[i] else 0)
                    updates[i].append(u)
            for i, sid in list(ids.items()):
                if pos[i] >= wavs[i].numel():
                    closed = srv.close(sid)
                    del ids[i]
                    emitted += _check_stream(model, wavs[i], updates[i], closed, rate, span, hop)
                    with pytest.raises(ValueError, match="not open"):
                        srv.push(sid, [0.0])
            steps += 1
        assert srv.streams == []
        assert emitted >= 10


@pytest.mark.gpu
def test_stream_that_never_reaches_a_window_or_a_span():
    model = _model()
    srv = model.streaming(window=8.0, overlap=4.0, span=6.0, hop=1.0)
    wav = synthetic.synthetic_audio(1, 5.0, seed=3)[0][0]
    a = srv.open()
    srv.push(a, wav.numpy())
    assert srv.step() == []
    closed = srv.close(a)
    assert closed == model.emotion_timeline(wav, window=8.0, overlap=4.0, span=6.0, hop=1.0)
    # the timeline's times use the recording's frame shift, N / 16000 / T: the one span ends at the recording's end
    assert len(closed.spans) == 1 and (closed.spans[0].start, closed.spans[0].end) == (0.0, 5.0)


@pytest.mark.gpu
def test_stream_device_memory_stays_flat():
    """A 20-minute stream's peak above the baseline stays within the margin `StreamServer`'s test allows over a 2-minute one,
    and the frames held on the device stay bounded by the span plus a window."""
    model = _model()
    model._get_engine()
    peaks, held = {}, {}
    for minutes in (2, 20):
        wav, _ = synthetic.synthetic_audio(1, 60.0 * minutes, seed=minutes)
        wav = wav[0]
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        most = 0
        with torch.inference_mode():
            srv = model.streaming(window=8.0, overlap=4.0, span=4.0, hop=1.0)
            a = srv.open()
            for pos in range(0, wav.numel(), 48000):
                srv.push(a, wav[pos:pos + 48000].numpy())
                srv.step()
                s = srv._streams[a]
                most = max(most, 0 if s.dev is None else s.dev.shape[0])
            tl = srv.close(a)
            del srv
        torch.cuda.synchronize()
        peaks[minutes] = torch.cuda.max_memory_allocated() - base
        held[minutes] = most
        assert abs(tl.frame_logits.shape[0] - 60 * minutes / FRAME) <= 2
    print(f"\npeak above baseline: 2 min {peaks[2] / 2**20:.1f} MiB, 20 min {peaks[20] / 2**20:.1f} MiB; held frames {held}")
    assert peaks[20] - peaks[2] < 64 * 2**20
    assert held[20] <= 100 + 8.0 / FRAME and held[20] == held[2]
