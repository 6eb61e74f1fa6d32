"""Emotions over time (INTEGRATION.md, "Emotions over time"): gam_emo_frame_logits, gam_emo_spans and
`GigaAMEmo.emotion_timeline`.

The head is Linear(768, C) on the mean of the encoder frames, so softmax(W mean_t f_t + b) = softmax(mean_t l_t) with the
per-frame logits l_t = W f_t + b.  CPU: the span plan, the refusals (before any device work), the exports.  GPU: both kernels
element by element against float64 with bounds derived from their fp32 arithmetic, containment of their reads and writes,
stitching bit for bit, one window against get_probs, and graph replay."""
import math
import random

import pytest
import torch

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, synthetic
from gigaam_b200.longform import (FRAME_SAMPLES, caller_span_frames, emotion_spans, encode_rows, plan_windows,
                                  stitch_emo_frame_logits)
from gigaam_b200.decoding import _as_btd

D = 768
U = 2.0 ** -24        # unit roundoff of fp32
CHUNK = 32            # kPoolChunk of csrc/kernels.h


def gamma(k):
    """gamma_k = k u / (1 - k u): relative bound of k consecutive fp32 roundings (Higham, Accuracy and Stability, §3.1)."""
    return k * U / (1 - k * U)


# ------------------------------------------------------------------------------------------ CPU: the span plan
@pytest.mark.parametrize("T,span,hop", [(1, 100, 25), (99, 100, 25), (100, 100, 25), (101, 100, 25), (125, 100, 25),
                                        (126, 100, 25), (1000, 100, 100), (1003, 100, 7), (5000, 1, 1), (37, 5, 5)])
def test_span_plan_covers_the_recording_when_hop_fits_the_span(T, span, hop):
    plan = emotion_spans(T, span, hop)
    if T <= span:
        assert plan == [(0, T)]
        return
    regular = [(k * hop, k * hop + span) for k in range((T - span) // hop + 1)]
    assert plan[:len(regular)] == regular and all(b <= T for _, b in regular)
    tail = plan[len(regular):]
    # the tail span is the only span that ends at T off the hop grid, and it exists exactly when no regular span ends at T
    assert tail == ([] if regular[-1][1] == T else [(T - span, T)])
    assert all(b - a == span for a, b in plan)
    covered = torch.zeros(T, dtype=torch.bool)
    for a, b in plan:
        covered[a:b] = True
    assert bool(covered.all())
    assert plan[-1][1] == T


def test_span_plan_with_hop_longer_than_the_span_leaves_gaps():
    plan = emotion_spans(100, 10, 25)
    assert plan == [(0, 10), (25, 35), (50, 60), (75, 85), (90, 100)]
    assert emotion_spans(85, 10, 25) == [(0, 10), (25, 35), (50, 60), (75, 85)]
    with pytest.raises(ValueError):
        emotion_spans(10, 0, 1)


def test_caller_spans_round_to_frames_and_clamp():
    assert caller_span_frames([(0.0, 0.04), (0.019, 0.021), (1.0, 1e9), (0.5, math.inf), (3.0, 3.0)], 50) == \
        [(0, 1), (0, 1), (25, 50), (12, 50), (50, 50)]


# ------------------------------------------------------------------------------------------ CPU: refusals, exports
def _no_device_work(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("device work before the arguments were checked")
    monkeypatch.setattr(gigaam.model.Engine, "__init__", refuse)
    monkeypatch.setattr(gigaam.GigaAM, "_resample_host", refuse)


@pytest.fixture(scope="module")
def cpu_emo():
    return gigaam.load_model("emo", device="cpu", synthetic=True)


@pytest.mark.parametrize("kw,needle", [
    (dict(span=0.05), "span=0.05"), (dict(span=0.0), "span=0.0"), (dict(span=-0.04), "span=-0.04"), (dict(hop=0.0), "hop=0.0"),
    (dict(hop=0.01), "hop=0.01"), (dict(span=math.nan), "span=nan"), (dict(hop=math.inf), "hop=inf"),
    (dict(spans=[(1.0, 0.5)]), "ends before"), (dict(spans=[(math.nan, 1.0)]), "NaN"), (dict(spans=[(0.0, math.nan)]), "NaN"),
    (dict(spans=[(-0.04, 1.0)]), "negative"), (dict(spans=[]), "no spans"),
    (dict(batch_size=0), "batch_size"), (dict(window=0.05), "window=0.05"), (dict(overlap=30.0), "overlap"),
    (dict(window=40.0), "max_encoded_frames"), (dict(sample_rate=12345), "sample_rate"), (dict(sample_rate=0), "sample_rate"),
])
def test_timeline_refusals_come_before_any_device_work(monkeypatch, cpu_emo, kw, needle):
    _no_device_work(monkeypatch)
    with pytest.raises(ValueError, match=None) as e:
        cpu_emo.emotion_timeline(torch.zeros(16000 * 3), **kw)
    assert needle in str(e.value), str(e.value)


def test_empty_recording_is_refused(monkeypatch, cpu_emo):
    _no_device_work(monkeypatch)
    with pytest.raises(ValueError, match="empty"):
        cpu_emo.emotion_timeline(torch.zeros(0))


@pytest.mark.parametrize("kw", [dict(span=0.05), dict(hop=0.0), dict(batch_size=0), dict(window=0.05), dict(overlap=8.0),
                                dict(sample_rate=12345)])
def test_stream_server_refusals_come_before_any_device_work(monkeypatch, cpu_emo, kw):
    _no_device_work(monkeypatch)
    with pytest.raises(ValueError):
        cpu_emo.streaming(**kw)


def test_exports_and_public_types():
    lib = _lib.load()
    for name in ("gam_emo_frame_logits", "gam_emo_spans"):
        assert name in _lib.EXPORTS and hasattr(lib, name)
    assert len(_lib.PROTOTYPES["gam_emo_frame_logits"][1]) == 10 and len(_lib.PROTOTYPES["gam_emo_spans"][1]) == 9
    names = [lib.gam_profile_class_name(i).decode() for i in range(lib.gam_profile_class_count())]
    assert "emo_frame_logits" in names and "emo_spans" in names
    for name in ("EmotionSpan", "EmotionTimeline", "EmotionStreamServer", "EmotionStreamUpdate"):
        assert name in gigaam.__all__ and hasattr(gigaam, name)
    assert hasattr(gigaam.GigaAMEmo, "emotion_timeline") and not hasattr(gigaam.GigaAMASR, "emotion_timeline")
    assert not hasattr(gigaam.GigaAM, "emotion_timeline") and not hasattr(gigaam.GigaAM, "streaming")


def test_timeline_equality_is_bitwise():
    names = ["a", "b"]
    p = torch.tensor([[0.25, float("nan")]])
    t = gigaam.EmotionTimeline(names=names, spans=[gigaam.EmotionSpan(0.0, 1.0, {"a": 0.25, "b": float("nan")})], probs=p,
                               frame_logits=torch.zeros(3, 2))
    same = gigaam.EmotionTimeline(names=names, spans=[gigaam.EmotionSpan(0.0, 1.0, {"a": 0.25, "b": float("nan")})],
                                  probs=p.clone(), frame_logits=torch.zeros(3, 2))
    assert t == same
    assert t != gigaam.EmotionTimeline(names=names, spans=same.spans, probs=p, frame_logits=-torch.zeros(3, 2))


# ------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (there is no CPU fallback to test instead)"
    return torch.device("cuda", 0)


_MODELS = {}


def _head_model(C, dev):
    """A 1-layer emo model with C classes: only its head is used by the kernel tests."""
    if C not in _MODELS:
        cfg = synthetic.emo_cfg(1, None if C == 4 else C)
        ck = {"cfg": cfg, "state_dict": synthetic.synthetic_state_dict(cfg, C)}
        _MODELS[C] = (gigaam.load_model("emo", device=dev, checkpoint=ck), ck["state_dict"])
    return _MODELS[C]


def _full_model(dev):
    if "full" not in _MODELS:
        _MODELS["full"] = gigaam.load_model("emo", device=dev, synthetic=True)
    return _MODELS["full"]


SENTINEL = -12345.5


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 4, 5, 256])
def test_frame_logits_against_float64(dev, C):
    model, sd = _head_model(C, dev)
    eng = model._get_engine()
    g = torch.Generator().manual_seed(C)
    B, T, n_frames = 9, 300, 1200
    # (lo, hi, dst): ragged, empty (lo == hi, lo > hi), clamped (lo < 0, hi > T), and rows that fall off either end
    ranges = [(0, 300, 500), (5, 6, 300), (17, 17, 301), (40, 10, 302), (-30, 64, 303), (250, 400, 400), (100, 200, -50),
              (0, 300, 1100), (31, 98, 800)]
    x = torch.randn(B, T, D, generator=g) * (torch.rand(B, 1, 1, generator=g) * 4 + 0.1) + torch.randn(B, 1, 1, generator=g) * 5
    for b, (lo, hi, _) in enumerate(ranges):
        mask = torch.ones(T, dtype=torch.bool)
        mask[max(lo, 0):min(max(hi, 0), T)] = False
        x[b, mask] = float("nan")                      # rows outside [lo, hi) are never read
    lo, hi, dst = (torch.tensor(c, dtype=torch.int32, device=dev) for c in zip(*ranges))
    out = torch.full((n_frames, C), SENTINEL, device=dev)
    with torch.inference_mode():
        eng.emo_frame_logits(x.to(dev), lo, hi, dst, out)
        torch.cuda.synchronize()
    out = out.cpu()
    W, bias = sd["head.weight"].double(), sd["head.bias"].double()
    written = torch.zeros(n_frames, dtype=torch.bool)
    for b, (l, h, d) in enumerate(ranges):
        l = min(max(l, 0), T)                          # the first kept frame lands on row dst
        for t in range(l, min(max(h, 0), T)):
            row = d + t - l
            if not 0 <= row < n_frames:
                continue
            assert not written[row]
            written[row] = True
            f = x[b, t].double()
            want = W @ f + bias
            # per lane 24 fmaf, 5 xor-tree adds, + bias: at most 30 roundings per term
            tol = gamma(30) * (W.abs() @ f.abs() + bias.abs())
            assert bool(((out[row].double() - want).abs() <= tol).all()), (b, t)
    assert int(written.sum()) > 500
    assert bool((out[~written] == SENTINEL).all()), "a row outside every [lo, hi) was written"


@pytest.mark.gpu
@pytest.mark.parametrize("C", [4, 33])
def test_frame_logits_have_the_bits_of_the_pooled_head_on_one_frame(dev, C):
    """A mean over one frame is the frame itself, so gam_emo_head's logits of a one-frame utterance are that frame's logits
    in the same summation order, bit for bit."""
    model, _ = _head_model(C, dev)
    eng = model._get_engine()
    x = torch.randn(1, 40, D, generator=torch.Generator().manual_seed(2)).to(dev) * 3
    out = torch.empty((40, C), device=dev)
    zero = torch.zeros(1, dtype=torch.int32, device=dev)
    with torch.inference_mode():
        eng.emo_frame_logits(x, zero, zero + 40, zero, out)
        alone = torch.stack([eng.emo_head(x[:, t:t + 1].contiguous(), None)[1][0] for t in range(40)])
    assert torch.equal(out, alone)


def _softmax_tol(v, C):
    """The softmax bound of gam_emo_head (tests/test_emotion.py) for the kernel's own logits v (float64)."""
    d = v - v.max()
    want = torch.softmax(v, 0)
    r = (1 + 4 * U) * torch.exp(U * d.abs()) - 1
    rho = (C * U / math.e + 4 * U) * (1 + gamma(12)) + gamma(12)
    return want, want * ((1 + r) * (1 + U) / (1 - rho) - 1) + 2.0 ** -126


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 4, 5, 256])
def test_spans_against_float64(dev, C):
    model, _ = _head_model(C, dev)
    eng = model._get_engine()
    g = torch.Generator().manual_seed(10 + C)
    n = 6000
    fl = torch.randn(n, C, generator=g) * (torch.rand(1, C, generator=g) * 6) + torch.randn(1, C, generator=g) * 3
    spans = [(100, 100), (200, 150), (7, 8), (0, 31), (40, 72), (64, 97), (0, 5000), (999, 5999), (5, 37), (40, 72), (-20, 12),
             (5990, 7000), (3000, 3033), (2000, 2031), (0, n)]
    spans += [tuple(sorted(torch.randint(0, n + 1, (2,), generator=g).tolist())) for _ in range(40)]
    st = torch.tensor([a for a, _ in spans], dtype=torch.int32, device=dev)
    en = torch.tensor([b for _, b in spans], dtype=torch.int32, device=dev)
    with torch.inference_mode():
        logits, probs = eng.emo_spans(fl.to(dev), st, en)
        torch.cuda.synchronize()
    logits, probs = logits.cpu(), probs.cpu()
    for i, (a, b) in enumerate(spans):
        a, b = min(max(a, 0), n), min(max(b, 0), n)
        m = max(b - a, 0)
        if m == 0:
            assert bool(logits[i].isnan().all() and probs[i].isnan().all()), i
            continue
        xs = fl[a:b].double()
        want = xs.mean(0)
        # 32-frame runs summed from their first frame (<= 31 roundings), the run sums from 0 (ceil(m / 32) roundings), then
        # one division: |mean_hat - mean| <= gamma_k (1 + u) mean|x| + u |mean|, k = 31 + ceil(m / 32)
        k = 31 + math.ceil(m / CHUNK)
        tol = gamma(k) * (1 + U) * xs.abs().mean(0) + U * want.abs()
        assert bool(((logits[i].double() - want).abs() <= tol).all()), (i, m)
        want_p, tol_p = _softmax_tol(logits[i].double(), C)
        assert bool(((probs[i].double() - want_p).abs() <= tol_p).all()), (i, m)
    # each span's bits do not depend on its position or its neighbours
    perm = list(range(len(spans)))
    random.Random(C).shuffle(perm)
    with torch.inference_mode():
        l2, p2 = eng.emo_spans(fl.to(dev), st[perm].contiguous(), en[perm].contiguous())
        l1, p1 = eng.emo_spans(fl.to(dev), st[:1].contiguous(), en[:1].contiguous())
    for j, i in enumerate(perm):
        assert torch.equal(l2[j].cpu().view(torch.int32), logits[i].view(torch.int32))
        assert torch.equal(p2[j].cpu().view(torch.int32), probs[i].view(torch.int32))
    assert torch.equal(p1[0].cpu().view(torch.int32), probs[0].view(torch.int32))


@pytest.mark.gpu
def test_a_nan_frame_makes_every_span_containing_it_nan(dev):
    model, _ = _head_model(4, dev)
    eng = model._get_engine()
    fl = torch.randn(200, 4)
    fl[77] = float("nan")
    spans = [(0, 77), (0, 78), (77, 78), (78, 200), (60, 100)]
    st = torch.tensor([a for a, _ in spans], dtype=torch.int32, device=dev)
    en = torch.tensor([b for _, b in spans], dtype=torch.int32, device=dev)
    with torch.inference_mode():
        _, probs = eng.emo_spans(fl.to(dev), st, en)
    probs = probs.cpu()
    assert [bool(probs[i].isnan().all()) for i in range(len(spans))] == [False, True, True, False, True]
    assert bool(probs[[0, 3]].isfinite().all())


@pytest.mark.gpu
def test_refusals_of_the_c_abi(dev):
    model, _ = _head_model(4, dev)
    eng = model._get_engine()
    x = torch.zeros(2, 10, D, device=dev)
    i32 = torch.zeros(2, dtype=torch.int32, device=dev)
    out = torch.zeros(10, 4, device=dev)
    for args, needle in (((x, 0, 10, i32, i32, i32, out, 10), "B=0"), ((x, 65536, 10, i32, i32, i32, out, 10), "65535"),
                         ((x, 2, 0, i32, i32, i32, out, 10), "T=0"), ((x, 2, 10, i32, i32, i32, out, 0), "n_frames=0"),
                         ((x, 2, 10, None, i32, i32, out, 10), "NULL"), ((x, 2, 10, i32, i32, i32, None, 10), "NULL")):
        with pytest.raises(_lib.GamError, match=needle):
            eng._call("gam_emo_frame_logits", *args)
    for args, needle in (((out, 10, i32, i32, 0, None, out), "S=0"), ((out, 0, i32, i32, 2, None, out), "n_frames=0"),
                         ((out, 10, None, i32, 2, None, out), "NULL"), ((None, 10, i32, i32, 2, None, out), "NULL")):
        with pytest.raises(_lib.GamError, match=needle):
            eng._call("gam_emo_spans", *args)
    asr = gigaam.load_model("v2_ctc", device=dev, checkpoint=synthetic.synthetic_checkpoint("v2_ctc", n_layers=1))
    with pytest.raises(_lib.GamError, match="no emo head"):
        asr._get_engine()._call("gam_emo_spans", out, 10, i32, i32, 2, None, out)


@pytest.mark.gpu
def test_stitched_frames_equal_each_window_encoded_alone_and_timelines_ignore_the_batch(dev):
    model = _full_model(dev)
    eng = model._get_engine()
    wav = synthetic.synthetic_audio(1, 75.3, seed=31)[0][0]
    host = wav.to(model._dtype).pin_memory()
    windows, T = plan_windows(wav.numel(), 10.0, 2.0, model._encoded_length, model._max_frames)
    assert len(windows) >= 8
    with torch.inference_mode():
        stitched = stitch_emo_frame_logits(model, host, windows, T, 3)
        for w in windows:
            if w.keep_end <= w.keep_start:
                continue
            enc = _as_btd(encode_rows(model, [host[w.start:w.end]]))
            first = w.start // FRAME_SAMPLES
            one = torch.full((enc.shape[1], eng.num_classes), SENTINEL, device=dev)
            rng = torch.tensor([[w.keep_start - first], [w.keep_end - first], [0]], dtype=torch.int32, device=dev)
            eng.emo_frame_logits(enc, rng[0], rng[1], rng[2], one)
            assert torch.equal(one[:w.keep_end - w.keep_start], stitched[w.keep_start:w.keep_end]), w
    timelines = [model.emotion_timeline(wav, window=10.0, overlap=2.0, batch_size=bs) for bs in (1, 3, 16)]
    assert torch.equal(timelines[0].frame_logits, stitched.cpu())
    assert timelines[0] == timelines[1] == timelines[2]
    tl = timelines[0]
    assert tl.names == synthetic.EMO_CLASSES and tl.probs.shape == (len(tl.spans), 4) and tl.frame_logits.shape == (T, 4)
    assert [(round(s.start / (wav.numel() / 16000 / T)), round(s.end / (wav.numel() / 16000 / T))) for s in tl] == emotion_spans(T, 100, 25)
    assert all(abs(sum(s.probs.values()) - 1) < 1e-5 for s in tl)
    # caller spans, the same frame logits: a span equals the plan's span with the same frames, bit for bit
    mine = model.emotion_timeline(wav, window=10.0, overlap=2.0, spans=[(1.0, 5.0), (0.0, 1e6), (3.0, 3.0)])
    assert torch.equal(mine.frame_logits, tl.frame_logits)
    assert torch.equal(mine.probs[0], tl.probs[1]) and bool(mine.probs[2].isnan().all())


@pytest.mark.gpu
def test_one_window_agrees_with_get_probs(dev):
    """A recording shorter than the window, one span [0, T): get_probs pools the frames then applies the head; the timeline
    applies the head to each frame then pools the logits.  Both start from the same encoder output, so they agree within the
    sum of their float64 bounds."""
    model = _full_model(dev)
    eng = model._get_engine()
    wav = synthetic.synthetic_audio(1, 12.7, seed=8)[0][0]
    tl = model.emotion_timeline(wav, span=40.0)
    got = model.get_probs(wav)
    with torch.inference_mode():
        w, length = model.prepare_wav(wav)
        enc = _as_btd(model.forward(w, length)[0])
        T = enc.shape[1]
        again = torch.empty((T, 4), device=dev)
        zero = torch.zeros(1, dtype=torch.int32, device=dev)
        eng.emo_frame_logits(enc, zero, zero + T, zero, again)
    assert len(tl.spans) == 1 and tl.frame_logits.shape[0] == T
    assert torch.equal(again.cpu(), tl.frame_logits), "the timeline's window encode differs from get_probs' encode"
    f = enc[0].cpu().double()
    sd = model.state_dict()
    W, bias = sd["head.weight"].cpu().double(), sd["head.bias"].cpu().double()
    want = W @ f.mean(0) + bias
    k = 31 + math.ceil(T / CHUNK)
    # get_probs: pooled within gamma_k (1 + u) mean|f| + u |mean|, then logits within gamma_30 of |W| |p| + |b|
    p_tol = gamma(k) * (1 + U) * f.abs().mean(0) + U * f.mean(0).abs()
    eps_a = W.abs() @ p_tol + gamma(30) * (W.abs() @ (f.mean(0).abs() + p_tol) + bias.abs())
    # timeline: each frame's logits within gamma_30 (|W||f_t| + |b|), then their mean within the chunked-sum bound
    fl = (W @ f.t()).t() + bias
    l_tol = gamma(30) * ((W.abs() @ f.abs().t()).t() + bias.abs())
    eps_b = l_tol.mean(0) + gamma(k) * (1 + U) * (fl.abs() + l_tol).mean(0) + U * (fl.mean(0).abs() + l_tol.mean(0))
    p_star = torch.softmax(want, 0)
    rho = (4 * U / math.e + 4 * U) * (1 + gamma(12)) + gamma(12)
    tol = 0
    for eps in (eps_a, eps_b):
        e = float(eps.max())
        r = (1 + 4 * U) * math.exp(U * float((want - want.min()).abs().max() + 2 * e)) - 1
        tol = tol + p_star * ((1 + r) * (1 + U) / (1 - rho) * math.exp(2 * e) - 1) + 2.0 ** -126
    a = torch.tensor([got[n] for n in tl.names], dtype=torch.float64)
    b = tl.probs[0].double()
    assert bool(((a - b).abs() <= tol).all()), ((a - b).abs(), tol)


@pytest.mark.gpu
def test_graph_replay_of_frame_logits_then_spans(dev):
    model, _ = _head_model(5, dev)
    eng = model._get_engine()
    g = torch.Generator().manual_seed(4)
    x = torch.randn(3, 200, D, generator=g).to(dev)
    rng = torch.tensor([[0, 10, 50], [200, 150, 51], [0, 200, 340]], dtype=torch.int32, device=dev)
    spans = torch.tensor([[0, 30, 0, 100], [341, 64, 0, 341]], dtype=torch.int32, device=dev)
    fl = torch.empty((341, 5), device=dev)

    def run():
        eng.emo_frame_logits(x, rng[0], rng[1], rng[2], fl)
        return eng.emo_spans(fl, spans[0], spans[1])

    with torch.inference_mode():
        eager = [t.clone() for t in run()]
        eager_fl = fl.clone()
        fl.fill_(float("nan"))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            run()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = run()
        fl.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(fl, eager_fl)
    for a, b in zip(out, eager):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
