"""Audio at any sample rate (include/gigaam_b200.h, gam_resample; INTEGRATION.md §7k).

CPU: `preprocess.resample_table` and the output-length rule against torchaudio, the WAV reader at every bit depth and channel
count (a 16-bit, 16 kHz file reads as it always did), the refusals, `sample_rate=16000` making exactly the calls it made
before, and the stream readiness rule against a brute-force restatement.

GPU: the kernel against torchaudio's float64 resample with a per-element bound derived from the arithmetic, NaN containment
in a ragged batch, bit-identity of batches, output spans and streams with one call, closed resampling streams against
`transcribe_windowed` / `spot`, the public calls end to end and against the oracle, CUDA-graph replay and flat device memory."""
import ctypes as C
import io
import math
import random
import wave

import numpy as np
import pytest
import torch
import torchaudio.functional as AF
from torchaudio.functional.functional import _get_sinc_resample_kernel

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, preprocess, synthetic
from gigaam_b200.preprocess import read_audio, resample_ratio, resample_table, resampled_length
from gigaam_b200.streaming import resample_ready

RATES = [8000, 11025, 12000, 22050, 24000, 32000, 44100, 48000, 96000, 37800]   # 37800: o = 189 > n = 80

_CPU_MODELS = {}


def _cpu_model(name):
    if name not in _CPU_MODELS:
        _CPU_MODELS[name] = gigaam.load_model(name, device="cpu", checkpoint=synthetic.synthetic_checkpoint(name, n_layers=1))
    return _CPU_MODELS[name]


def _ta_kernel(sr):
    g = math.gcd(sr, 16000)
    k, w = _get_sinc_resample_kernel(sr, 16000, g, dtype=torch.float64)
    return k.reshape(k.shape[0], -1), w


# ------------------------------------------------------------------------------------------ CPU: the definition
@pytest.mark.parametrize("sr", RATES)
def test_table_is_torchaudios_float64_kernel_rounded_once(sr):
    h64, w = _ta_kernel(sr)
    o, n, w_ours = resample_ratio(sr)
    assert w_ours == w and h64.shape == (n, 2 * w + o)
    assert torch.equal(resample_table(sr), h64.float())


@pytest.mark.parametrize("sr", [8000, 44100, 48000, 37800, 11025])
def test_output_length_is_torchaudios(sr):
    assert resampled_length(0, sr) == 0          # torchaudio cannot take an empty signal
    for L in list(range(1, 40)) + [441, 1000, 4409, 16001]:
        want = AF.resample(torch.zeros(1, L, dtype=torch.float64), sr, 16000).shape[-1]
        assert resampled_length(L, sr) == want, (sr, L)


def test_the_issue_rates_fit_and_12345_does_not():
    sizes = {sr: resample_table(sr).numel() for sr in RATES[:-1]}
    assert min(sizes.values()) == 28 and max(sizes.values()) == 291200 and sizes[11025] == 291200
    with pytest.raises(ValueError, match="2469:3200"):
        resample_ratio(12345)


@pytest.mark.parametrize("bad", [0, -8000, 8000.5, 8000.0, True, "8000", None])
def test_rate_refusals(bad):
    with pytest.raises(ValueError, match="positive integer"):
        resample_ratio(bad)


def test_public_calls_refuse_a_bad_rate_before_device_work():
    model = _cpu_model("v2_ctc")     # a CPU model has no engine: any device work would raise RuntimeError instead
    wav = np.zeros(8000, np.float32)
    calls = [lambda: model.transcribe(wav, sample_rate=12345), lambda: model.transcribe_windowed(wav, sample_rate=0),
             lambda: model.transcribe_longform(wav, sample_rate=-1), lambda: model.align(wav, "да", sample_rate=12345),
             lambda: model.align_longform(wav, "да", sample_rate=7.5), lambda: model.spot(wav, ["да"], sample_rate=12345),
             lambda: model.embed_audio(wav, sample_rate=True), lambda: model.streaming(sample_rate=12345),
             lambda: model.transcribe(wav, hotwords=["да"], sample_rate=0),
             lambda: model.transcribe_batch(torch.zeros(1, 100), torch.tensor([100]), sample_rate=12345),
             lambda: model.align_batch(torch.zeros(1, 100), torch.tensor([100]), ["да"], sample_rate=12345),
             lambda: model.spot_batch(torch.zeros(1, 100), torch.tensor([100]), ["да"], sample_rate=12345)]
    for call in calls:
        with pytest.raises(ValueError, match="sample_rate"):
            call()
    with pytest.raises(ValueError, match="sample_rate"):
        _cpu_model("v2_rnnt").transcribe(wav, boost=["да"], sample_rate=12345)


def test_engine_refuses_inverted_spans(monkeypatch):
    from gigaam_b200.engine import Engine

    calls = []

    class Stub:
        device = torch.device("cpu")

        def resample_plan(self, sr):
            return torch.zeros(15, 2), 1, 2, 7

        def _call(self, *a):
            calls.append(a[0])
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    x, out = torch.zeros(2, 10), torch.zeros(2, 10)
    Engine.resample_spans(Stub(), x, torch.tensor([[0, 0], [5, 10], [0, 2], [3, 12]]), 8000, out)
    assert calls == ["gam_resample"]
    # in_end < in_begin, out_end < out_begin, out_begin < 0, more samples or outputs than a row holds
    for bad in ([[6, 0], [5, 5]], [[0, 0], [5, 5]], [[0, 0], [11, 5]]):
        for outs in ([[0, 0], [3, 3]],) if bad != [[0, 0], [5, 5]] else ([[4, 0], [3, 3]], [[-1, 0], [3, 3]], [[0, 0], [11, 3]]):
            with pytest.raises(ValueError):
                Engine.resample_spans(Stub(), x, torch.tensor(bad + outs), 8000, out)
    assert calls == ["gam_resample"]


def test_exported():
    assert "gam_resample" in _lib.EXPORTS
    restype, args = _lib.PROTOTYPES["gam_resample"]
    assert restype == C.c_int32 and len(args) == 13 and args[2] == C.c_int64 and args[3] == C.c_int32


# ------------------------------------------------------------------------------------------ CPU: the WAV reader
def _wav_bytes(frames: np.ndarray, width: int, rate: int) -> bytes:
    buf = io.BytesIO()
    with wave.open(buf, "wb") as wf:
        wf.setnchannels(frames.shape[1])
        wf.setsampwidth(width)
        wf.setframerate(rate)
        if width == 1:
            raw = (frames + 128).astype(np.uint8).tobytes()
        elif width == 3:
            v = frames.astype(np.int32).reshape(-1)
            raw = np.stack([v & 255, (v >> 8) & 255, (v >> 16) & 255], 1).astype(np.uint8).tobytes()
        else:
            raw = frames.astype({2: np.int16, 4: np.int32}[width]).tobytes()
        wf.writeframes(raw)
    return buf.getvalue()


@pytest.mark.parametrize("width", [1, 2, 3, 4])
@pytest.mark.parametrize("channels", [1, 2, 3])
def test_wav_reader(tmp_path, monkeypatch, width, channels):
    monkeypatch.setattr(preprocess, "run", lambda *a, **k: (_ for _ in ()).throw(FileNotFoundError()))   # no ffmpeg
    bits = 8 * width
    rng = np.random.default_rng(width * 10 + channels)
    top = 2 ** (bits - 1)
    frames = rng.integers(-top, top, size=(1001, channels), dtype=np.int64)
    frames[:2] = [[-top] * channels, [top - 1] * channels]
    path = tmp_path / "a.wav"
    path.write_bytes(_wav_bytes(frames, width, 44100))
    wav, rate = read_audio(str(path))
    assert rate == 44100 and wav.dtype == torch.float32 and wav.shape == (1001,)
    mono = np.trunc(frames.mean(axis=1)) if channels > 1 else frames[:, 0]
    assert np.array_equal(wav.numpy(), (mono / top).astype(np.float32))
    with pytest.raises(RuntimeError, match="44100 Hz"):
        preprocess.load_audio(str(path))


@pytest.mark.parametrize("channels", [1, 2])
def test_16_bit_16_khz_reads_as_before(tmp_path, monkeypatch, channels):
    monkeypatch.setattr(preprocess, "run", lambda *a, **k: (_ for _ in ()).throw(FileNotFoundError()))
    frames = np.random.default_rng(3).integers(-32768, 32768, size=(4000, channels))
    path = tmp_path / "b.wav"
    path.write_bytes(_wav_bytes(frames, 2, 16000))
    pcm = frames.astype(np.int16).reshape(-1)            # the reader this project had before
    if channels > 1:
        pcm = pcm.reshape(-1, channels).astype(np.float32).mean(axis=1).astype(np.int16)
    want = torch.frombuffer(bytearray(pcm.tobytes()), dtype=torch.int16).float() / 32768.0
    wav, rate = read_audio(str(path))
    assert rate == 16000 and torch.equal(wav, want) and torch.equal(preprocess.load_audio(str(path)), want)


# ------------------------------------------------------------------------------------------ CPU: 16 kHz is untouched
def test_16_khz_makes_the_calls_it_made_before(monkeypatch):
    import gigaam_b200.longform as longform
    from gigaam_b200.engine import DecodeBuffers, Engine
    model = _cpu_model("v2_ctc")
    log = []
    enc = torch.zeros((1, 768, 25))
    monkeypatch.setattr(Engine, "resample", lambda *a: pytest.fail("resampled"))
    monkeypatch.setattr(Engine, "resample_spans", lambda *a: pytest.fail("resampled"))
    monkeypatch.setattr(model, "_resample_host", lambda *a: pytest.fail("resampled"))
    monkeypatch.setattr(model, "forward", lambda wav, length: (log.append(("forward", wav.dtype, tuple(wav.shape),
                                                                           length.tolist())), (enc, torch.tensor([25])))[1])
    monkeypatch.setattr(model, "_decode", lambda *a: (log.append(("decode",) + tuple(a[3:])), [("txt", None, None)])[1])
    monkeypatch.setattr(model.decoding, "decode", lambda head, e, l: (log.append("decode_batch"), [("txt", None, None)])[1])
    wav = np.zeros(16000, np.float32)
    runs = []
    for kwargs in ({}, {"sample_rate": 16000}):
        log.clear()
        assert model.transcribe(wav, word_timestamps=True, **kwargs).text == "txt"
        model.transcribe_batch(torch.zeros(2, 300), torch.tensor([300, 200]), **kwargs)
        model.embed_audio(wav, **kwargs)
        runs.append(list(log))
    assert runs[0] == runs[1] and len(runs[0]) == 5

    class Recorder:
        device = torch.device("cpu")
        num_classes = 35

        def group_words(self, ids, frames, counts, flags):
            B, m = ids.shape
            return [torch.zeros((B, m), dtype=torch.int32) for _ in range(4)] + [torch.zeros(B, dtype=torch.int32)]
    monkeypatch.setattr(model, "_get_engine", lambda: Recorder())
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)

    def fake_decode(m, host, windows, T, batch_size, scores, *extra, **kw):
        log.append(("decode_windows", host.dtype, host.numel(), tuple(windows), T))
        i32 = dict(dtype=torch.int32)
        return DecodeBuffers(torch.zeros((1, T), **i32), torch.zeros((1, T), **i32), torch.zeros(1, **i32))
    monkeypatch.setattr(longform, "decode_windows", fake_decode)
    runs = []
    for kwargs in ({}, {"sample_rate": 16000}):
        log.clear()
        model.transcribe_windowed(wav, **kwargs)
        runs.append(list(log))
    assert runs[0] == runs[1] and len(runs[0]) == 1
    srv = model.streaming(sample_rate=16000)
    assert srv.sample_rate == 16000 and srv._ratio is None


# ------------------------------------------------------------------------------------------ CPU: stream readiness
@pytest.mark.parametrize("sr", [8000, 44100, 48000, 37800, 22050])
def test_stream_readiness_against_brute_force(sr):
    o, n, w = resample_ratio(sr)
    K = 2 * w + o
    for n_raw in list(range(0, 3 * K + 3 * o)) + [5000, 5001]:
        # output m = j n + p is final when every tap's sample j o + k - w (k < K) that lies in the signal has been pushed
        ready = [m for m in range(n * (n_raw + K) // o + 2 * n) if (m // n) * o + K - 1 - w < n_raw]
        assert ready == list(range(len(ready)))
        assert resample_ready(n_raw, o, n, w) == len(ready), (sr, n_raw)
        for N in (n_raw, n_raw + 1, n_raw + o + 7):
            assert len(ready) <= resampled_length(N, sr)


# ------------------------------------------------------------------------------------------ GPU
def _dev():
    return torch.device("cuda", 0)


_MODELS = {}


def _model(name, n_layers=1):
    if (name, n_layers) not in _MODELS:
        ck = synthetic.synthetic_checkpoint(name, seed=0, n_layers=n_layers)
        _MODELS[name, n_layers] = (gigaam.load_model(name, fp16_encoder=False, device=_dev(), checkpoint=ck), ck)
    return _MODELS[name, n_layers][0]


def _signals(sr, long):
    rng = np.random.default_rng(sr)
    t = np.arange(3000) / sr
    sq = np.where(np.sin(2 * np.pi * 0.013 * sr * t) >= 0, 1.0, -1.0)
    ext = np.where(np.arange(3000) % 2 == 0, -1.0, 32767 / 32768)
    imp = np.zeros(2000)
    imp[0] = imp[-1] = 1.0
    sigs = [rng.standard_normal(3000) * 0.3, np.sin(2 * np.pi * 0.45 * sr * t), sq, ext, imp, np.zeros(2500), np.zeros(0),
            rng.standard_normal(1), rng.standard_normal(7)]
    o, n, w = resample_ratio(sr)
    sigs.append(rng.uniform(-1, 1, 2 * w + o - 1))
    if long:
        sigs.append(rng.uniform(-1, 1, (1 << 20) + 37))
    return [torch.tensor(s, dtype=torch.float32) for s in sigs]


def _bound(x, sr):
    """Per-element bound on |ours - torchaudio float64|: sum |h64 - h32||x| + gamma_K sum |h32 x| (+ the float64 side's)."""
    h64, w = _ta_kernel(sr)
    o, n, _ = resample_ratio(sr)
    K = h64.shape[1]
    h32 = h64.float().double()
    xp = torch.nn.functional.pad(x.double().abs()[None, None], (w, w + o))
    conv = lambda h: torch.nn.functional.conv1d(xp, h[:, None, :], stride=o).transpose(1, 2).reshape(-1)
    u = 2.0 ** -24
    gamma = K * u / (1 - K * u)
    L = resampled_length(x.numel(), sr)
    return (conv((h64 - h32).abs()) + gamma * conv(h32.abs()) + 2 * K * 2.0 ** -53 * conv(h64.abs()))[:L]


@pytest.mark.gpu
@pytest.mark.parametrize("sr", RATES)
def test_kernel_against_torchaudio_float64(sr):
    eng = _model("v2_ctc")._get_engine()
    sigs = _signals(sr, long=sr in (8000, 44100, 48000))
    L = max(s.numel() for s in sigs)
    x = torch.full((len(sigs), L), float("nan"))
    for b, s in enumerate(sigs):
        x[b, :s.numel()] = s
    lens = torch.tensor([s.numel() for s in sigs])
    y, y_len = eng.resample(x.to(_dev()), lens, sr)
    y = y.cpu()
    worst = 0.0
    for b, s in enumerate(sigs):
        want = AF.resample(s.double()[None], sr, 16000)[0] if s.numel() else torch.zeros(0, dtype=torch.float64)
        assert int(y_len[b]) == want.numel() == resampled_length(s.numel(), sr)
        got = y[b, :want.numel()].double()
        err, bound = (got - want).abs(), _bound(s, sr)
        assert (err <= bound).all(), (sr, b, float((err - bound).max()))
        nz = bound > 0
        if nz.any():
            worst = max(worst, float((err[nz] / bound[nz]).max()))
        assert (y[b, want.numel():] == 0).all()
    print(f"\n{sr} Hz: worst error / bound {worst:.3f}")


@pytest.mark.gpu
def test_nan_reaches_exactly_the_outputs_whose_span_holds_it():
    eng = _model("v2_ctc")._get_engine()
    for sr in (8000, 44100, 48000):
        o, n, w = resample_ratio(sr)
        K = 2 * w + o
        lens = [1000, 0, 37, 1500]
        x = torch.full((4, 1600), float("nan"))
        for b, L in enumerate(lens):
            x[b, :L] = torch.rand(L) - 0.5
        q = 500
        x[3, q] = float("nan")
        out_len = [resampled_length(L, sr) for L in lens]
        spans = torch.tensor([[0] * 4, lens, [0] * 4, out_len])
        y = torch.full((4, max(out_len) + 50), float("nan"), device=_dev())
        y = eng.resample_spans(x.to(_dev()), spans, sr, y).cpu()
        for b, L in enumerate(lens):
            assert torch.isnan(y[b, out_len[b]:]).all()              # unused output space is not written
            m = torch.arange(out_len[b])
            first = (m // n) * o - w
            hit = (first <= q) & (q < first + K) if b == 3 else torch.zeros_like(m, dtype=torch.bool)
            assert torch.equal(torch.isnan(y[b, :out_len[b]]), hit), (sr, b)
            assert hit.any() == (b == 3)


def _spans_call(eng, sig, sr, cuts):
    """Resample `sig` output span by output span, each row uploading only the samples its outputs need."""
    o, n, w = resample_ratio(sr)
    K, L = 2 * w + o, sig.numel()
    rows = []
    for a, b in zip(cuts, cuts[1:]):
        lo = max(0, a // n * o - w) if b > a else 0
        hi = min(L, (b - 1) // n * o - w + K) if b > a else 0
        rows.append((max(0, min(lo, hi)), max(0, hi), a, b))
    P = max(1, max(hi - lo for lo, hi, _, _ in rows))
    x = torch.full((len(rows), P), float("nan"))
    for r, (lo, hi, _, _) in enumerate(rows):
        x[r, :hi - lo] = sig[lo:hi]
    y = torch.full((len(rows), max(1, max(b - a for _, _, a, b in rows))), float("nan"), device=_dev())
    y = eng.resample_spans(x.to(_dev()), torch.tensor(rows).t(), sr, y).cpu()
    return torch.cat([y[r, :b - a] for r, (_, _, a, b) in enumerate(rows)])


@pytest.mark.gpu
@pytest.mark.parametrize("sr", [8000, 11025, 44100, 48000])
def test_batches_and_output_spans_are_bit_identical(sr):
    eng = _model("v2_ctc")._get_engine()
    rng = random.Random(sr)
    sig = torch.rand(20011) * 2 - 1
    one, one_len = eng.resample(sig[None].to(_dev()), torch.tensor([sig.numel()]), sr)
    one = one[0].cpu()
    N = int(one_len[0])
    others = [torch.rand(rng.randint(0, 30000)) for _ in range(5)]
    x = torch.zeros(7, 30000)
    lens = [o.numel() for o in others[:3]] + [sig.numel()] + [o.numel() for o in others[3:]] + [0]
    for b, s in enumerate(others[:3] + [sig] + others[3:] + [torch.zeros(0)]):
        x[b, :s.numel()] = s
    batch, _ = eng.resample(x.to(_dev()), torch.tensor(lens), sr)
    assert torch.equal(batch[3, :N].cpu().view(torch.int32), one.view(torch.int32))
    for step in (1, 7, 101, "random"):
        if step == "random":
            cuts = sorted({0, N} | {rng.randint(0, N) for _ in range(40)})
            cuts.insert(3, cuts[2])                                  # an empty span
        else:
            cuts = list(range(0, N, step if step > 1 else 37)) + [N]
            if step == 1:
                cuts = sorted(set(cuts) | {a + 1 for a in cuts[:-1]})   # spans of one output among others
        got = _spans_call(eng, sig, sr, cuts)
        assert torch.equal(got.view(torch.int32), one.view(torch.int32)), (sr, step)


def _chunks(rng, L, how):
    sizes, i = [], 0
    while i < L:
        k = {"one": 1, "prime": rng.choice([2, 3, 5, 7, 11, 13, 331, 1009])}.get(how) or rng.choice([0, 0, 1, 17, 400, 3001])
        sizes.append(min(k, L - i))
        i += sizes[-1]
    return sizes


@pytest.mark.gpu
@pytest.mark.parametrize("sr", [8000, 44100])
def test_stream_resampling_equals_one_call(sr):
    model = _model("v2_ctc")
    eng = model._get_engine()
    rng = random.Random(sr)
    sig = torch.rand(6007 if sr == 8000 else 30011) * 2 - 1
    want, _ = eng.resample(sig[None].to(_dev()), torch.tensor([sig.numel()]), sr)
    want = want[0].cpu()
    with torch.inference_mode():
        srv = model.streaming(sample_rate=sr)
        for how in ("one", "prime", "random"):
            s = srv._streams[srv.open()]
            i = 0
            for k, size in enumerate(_chunks(rng, sig.numel() if how != "one" else min(sig.numel(), 3000), how)):
                srv.push(s.id, sig[i:i + size].numpy())
                i += size
                if k % (97 if how == "one" else 3) == 0:
                    srv._resample([s], final=False)
                    assert s.raw_start <= max(0, s.out_n // resample_ratio(sr)[1] * resample_ratio(sr)[0])
            srv._resample([s], final=True)
            ref = want if i == sig.numel() else eng.resample(sig[None, :i].to(_dev()), torch.tensor([i]), sr)[0][0].cpu()
            assert s.n == ref.numel()
            assert torch.equal(s.samples(0, s.n).view(torch.int32), ref.view(torch.int32)), how


def _recordings(seed, sr, n=3):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        sec = float(rng.uniform(3.0, 27.0))
        wav, _ = synthetic.synthetic_audio(1, sec * sr / 16000, seed=seed * 10 + i)
        out.append(wav[0].clone())
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("sr", [8000, 44100])
@pytest.mark.parametrize("name", ["v2_ctc", "v2_rnnt"])
def test_closed_streams_equal_transcribe_windowed(name, sr):
    model = _model(name)
    wavs = _recordings(len(name) + sr % 7, sr)
    rng = random.Random(sr)
    ctc = name.endswith("ctc")
    keywords = ["да", [3], [5]] if ctc else None
    with torch.inference_mode():
        srv = model.streaming(window=8.0, overlap=4.0, batch_size=4, confidence=True, keywords=keywords, threshold=0.2,
                              sample_rate=sr)
        ids = [srv.open() for _ in wavs]
        pos = [0] * len(wavs)
        while any(p < w.numel() for p, w in zip(pos, wavs)):
            for i, w in enumerate(wavs):
                k = rng.choice([0, 1, 160, 799, 4001, 12345])
                srv.push(ids[i], w[pos[i]:pos[i] + k].numpy())
                pos[i] += k
            srv.step()
        results = [srv.close(i, word_timestamps=True, pause=0.3, max_segment=6.0) for i in ids]
    n_tok = 0
    for w, res in zip(wavs, results):
        want = model.transcribe_windowed(w, word_timestamps=True, confidence=True, window=8.0, overlap=4.0, pause=0.3,
                                         max_segment=6.0, sample_rate=sr)
        assert repr(res.transcript) == repr(want)
        n_tok += sum(len(s.words) for s in want.segments)
        if ctc:
            assert repr(res.detections) == repr(model.spot(w, keywords, threshold=0.2, window=8.0, overlap=4.0, sample_rate=sr))
    assert n_tok > 0


@pytest.mark.gpu
@pytest.mark.parametrize("sr", [8000, 44100])
def test_transcribe_at_a_rate_equals_transcribe_of_the_resampled_wave(sr):
    for name in ("v2_ctc", "v2_rnnt"):
        model = _model(name)
        wav = _recordings(3, sr, n=1)[0][:int(20 * sr)]
        y, _ = model._get_engine().resample(wav[None].to(_dev()), torch.tensor([wav.numel()]), sr)
        a = model.transcribe(wav, word_timestamps=True, confidence=True, sample_rate=sr)
        b = model.transcribe(y[0], word_timestamps=True, confidence=True)
        assert repr(a) == repr(b)
        assert model.transcribe_batch(wav[None], torch.tensor([wav.numel()]), sample_rate=sr) == [b.text]
        assert torch.equal(model.prepare_wav(wav, sample_rate=sr)[0], y.to(model._dtype))
        assert torch.equal(torch.from_numpy(np.asarray(model._resample_host(wav, sr))), y[0].cpu())


@pytest.mark.gpu
def test_encoder_on_the_resampled_wave_against_the_oracle():
    from oracle import gigaam_oracle as orc
    from test_gpu_parity import ENC_REL_TOL
    model = _model("v2_ctc", n_layers=2)
    ck = _MODELS["v2_ctc", 2][1]
    for sr in (8000, 44100):
        wav = _recordings(5, sr, n=1)[0][:int(8 * sr)]
        ours, ours_len = model.prepare_wav(wav, sample_rate=sr)
        ta = AF.resample(wav.double()[None], sr, 16000).float()
        assert ta.shape == ours.shape
        with torch.inference_mode():
            enc, enc_len = model(ours, ours_len)
            enc_o, len_o = orc.model_forward(ta, torch.tensor([ta.shape[1]]), ck["state_dict"], ck["cfg"])
        assert torch.equal(enc_len.cpu(), len_o)
        rel = float((enc.cpu() - enc_o).norm() / enc_o.norm())
        print(f"\n{sr} Hz: encoder rel {rel:.3e}")
        assert rel < ENC_REL_TOL


@pytest.mark.gpu
def test_refusals_of_the_entry_point():
    eng = _model("v2_ctc")._get_engine()
    table, o, n, w = eng.resample_plan(44100)
    x = torch.zeros(1, 10, device=_dev())
    spans = torch.tensor([[0], [10], [0], [4]], device=_dev())
    y = torch.zeros(1, 4, device=_dev())
    ok = (x, 10, 1, spans, table, table.shape[0], table.shape[1], o, n, y, 4)
    eng._call("gam_resample", *ok)
    for i, bad, msg in [(0, None, "NULL"), (3, None, "NULL"), (4, None, "NULL"), (9, None, "NULL"), (2, 0, "B=0"),
                        (1, -1, "pitch"), (10, -1, "pitch"), (5, table.shape[0] - 1, "does not match"),
                        (6, n + 1, "does not match"), (7, o + 1, "does not match"), (8, n + 1, "does not match"),
                        (7, 0, "does not match")]:
        args = list(ok)
        args[i] = bad
        with pytest.raises(_lib.GamError, match=msg):
            eng._call("gam_resample", *args)
    with pytest.raises(ValueError, match="16 kHz"):
        eng.resample_plan(16000)


@pytest.mark.gpu
def test_cuda_graph_replay_is_bit_exact():
    eng = _model("v2_ctc")._get_engine()
    sr = 44100
    table, o, n, w = eng.resample_plan(sr)
    lens = [30000, 12345, 0]
    x = torch.zeros(3, 30000, device=_dev())
    spans = torch.tensor([[0] * 3, lens, [0] * 3, [resampled_length(L, sr) for L in lens]], device=_dev())
    y = torch.zeros(3, max(resampled_length(L, sr) for L in lens), device=_dev())
    s = torch.cuda.Stream(_dev())
    with torch.cuda.stream(s):
        eng.resample_spans(x, spans, sr, y)          # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        eng.resample_spans(x, spans, sr, y)
    for seed in (1, 2):
        torch.manual_seed(seed)
        x.copy_(torch.rand(3, 30000, device=_dev()) - 0.5)
        y.zero_()
        g.replay()
        torch.cuda.synchronize()
        want = eng.resample(x, torch.tensor(lens), sr)[0]
        assert torch.equal(y.view(torch.int32), want.view(torch.int32))


@pytest.mark.gpu
def test_device_memory_stays_flat_at_48_khz():
    model = _model("v2_ctc")
    peaks = {}
    for minutes in (2, 20, 2, 20):
        wav, _ = synthetic.synthetic_audio(1, 180.0 * minutes, seed=minutes)     # 3 x 16000 samples a second: 48 kHz
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        model.transcribe_windowed(wav[0], batch_size=4, sample_rate=48000)
        torch.cuda.synchronize()
        peaks[minutes] = torch.cuda.max_memory_allocated() - base
    print(f"\npeak above baseline at 48 kHz: 2 min {peaks[2] / 2**20:.1f} MiB, 20 min {peaks[20] / 2**20:.1f} MiB")
    assert peaks[20] - peaks[2] < 64 * 2**20
