"""Live streams: resumable keyword spotting (gam_ctc_spot_resume, include/gigaam_b200.h), the window schedule of
`streaming.StreamServer` and the server itself (INTEGRATION.md §7i).

CPU: the windows a stream encodes before and at `close` are exactly `plan_windows(N)` for any chunking, the refusals, the
`new_text` concatenation invariant and the exported symbols.  GPU: a window's encoder output (and CTC log-probs) do not
depend on its batch, closed streams equal `transcribe_windowed` and `spot` bit for bit, resumed spotting equals the one-shot
kernel, tentative text equals a replay from the committed state, and device memory stays flat.
"""
import random

import numpy as np
import pytest
import torch

import gigaam_b200 as gigaam
from gigaam_b200 import _lib, synthetic
from gigaam_b200.longform import FRAME_SAMPLES, plan_windows
from gigaam_b200.streaming import StreamServer, TextFeed, ready_count, ready_window

_CPU_MODELS = {}


def _cpu_model(name):
    if name not in _CPU_MODELS:
        _CPU_MODELS[name] = gigaam.load_model(name, device="cpu", checkpoint=synthetic.synthetic_checkpoint(name, n_layers=1))
    return _CPU_MODELS[name]


def _length_fn(n):
    """The encoders' length rule: frames of n samples (both front ends: hop 160, subsampling 4)."""
    return _cpu_model("v2_ctc")._encoded_length(n)


# ------------------------------------------------------------------------------------------ CPU: the window schedule
def _chunkings(rng, N, W, H):
    """Chunk sizes covering N samples: 1-sample chunks, chunks that end exactly at w H + W, and random ones."""
    yield [1] * N if N <= 3 * 640 else [1] * 700 + [N - 700]
    edges = sorted({min(w * H + W, N) for w in range(N // H + 2)} | {N})
    yield [b - a for a, b in zip([0] + edges, edges) if b > a]
    sizes, left = [], N
    while left:
        sizes.append(min(left, rng.choice([1, 17, 640, 5000, rng.randint(1, 3 * W)])))
        left -= sizes[-1]
    yield sizes


@pytest.mark.parametrize("window,overlap", [(8.0, 4.0), (30.0, 4.0), (2.0, 0.0), (1.2, 0.88)])
def test_ready_windows_are_the_plan_of_the_whole_stream(window, overlap):
    W, V = round(window * 16000), round(overlap * 16000)
    H = W - V
    rng = random.Random(int(window * 100 + overlap))
    lengths = [1, 639, 640, W - 1, W, W + 1, W + H, 3 * H + W, 3 * H + W + 1, 5 * H + W - 1] + [rng.randint(1, 12 * W) for _ in range(8)]
    for N in lengths:
        if _length_fn(N) <= 0:
            continue
        plan, _ = plan_windows(N, window, overlap, _length_fn)
        for sizes in _chunkings(rng, N, W, H):
            handed, n = [], 0
            for c in sizes:
                n += c
                if rng.random() < 0.5:       # steps at random moments between pushes
                    handed += [ready_window(w, W, V) for w in range(len(handed), ready_count(n, W, V))]
            handed += [ready_window(w, W, V) for w in range(len(handed), ready_count(n, W, V))]
            assert len(handed) == len(plan) - 1 or (N <= W and not handed)
            handed += plan[len(handed):]     # close: the ready ones not yet encoded (none here), then the last one
            assert handed == plan, (N, sizes[:5])


def test_a_ready_window_is_never_the_last():
    W, V = 8 * 16000, 4 * 16000
    for n in range(W - 3, W + 5 * (W - V) + 3, 997):
        r = ready_count(n, W, V)
        plan, _ = plan_windows(n, 8.0, 4.0, _length_fn)
        assert r == len(plan) - 1 if n > W else r == 0
        if r:
            assert ready_window(r - 1, W, V).end < n          # more than w H + W samples are held


# ------------------------------------------------------------------------------------------ CPU: text and refusals
class _OpenerTok:
    """A SentencePiece-like tokenizer: pieces joined, U+2581 read as a space, the first piece's leading one dropped."""
    pieces = ["▁a", "b", "▁c", "d", "ee", "▁", "▁fgh", "i"]

    def decode(self, ids):
        text = "".join(self.pieces[i] for i in ids).replace("▁", " ")
        return text[1:] if text.startswith(" ") else text


def test_new_text_concatenates_to_the_decoded_stream():
    rng = random.Random(3)
    tok = _OpenerTok()
    openers = {i for i, p in enumerate(tok.pieces) if p.startswith("▁")}
    for _ in range(200):
        feed, ids, text = TextFeed(tok, openers), [], ""
        for _ in range(rng.randint(1, 12)):
            new = [rng.randrange(len(tok.pieces)) for _ in range(rng.choice([0, 1, 2, 5]))]
            ids += new
            text += feed.push(ids, len(new))
            assert text == tok.decode(ids)
            assert feed.anchor == max([0] + [i for i, t in enumerate(ids) if t in openers])
    # charwise: the space token opens words
    m = _cpu_model("v2_ctc")
    tk = m.decoding.tokenizer
    feed, ids, text = TextFeed(tk, {tk.vocab.index(" ")}), [], ""
    for chunk in (tk.encode("при"), tk.encode("вет как"), [], [tk.vocab.index(" ")] + tk.encode("дела")):
        ids += chunk
        text += feed.push(ids, len(chunk))
    assert text == tk.decode(ids) == "привет как дела"


def test_streaming_refuses_before_device_work():
    model = _cpu_model("v2_ctc")
    with pytest.raises(ValueError, match="multiple"):
        model.streaming(window=8.01)
    with pytest.raises(ValueError, match="multiple"):
        model.streaming(overlap=0.5)
    with pytest.raises(ValueError, match="overlap"):
        model.streaming(overlap=-0.04)
    with pytest.raises(ValueError, match="overlap"):
        model.streaming(window=4.0, overlap=4.0)
    with pytest.raises(ValueError, match="max_encoded_frames"):
        model.streaming(window=31.0)
    with pytest.raises(ValueError, match="positive"):
        model.streaming(window=0.0)
    with pytest.raises(ValueError, match="batch_size"):
        model.streaming(batch_size=0)
    with pytest.raises(ValueError, match="no keywords"):
        model.streaming(keywords=[])
    with pytest.raises(ValueError, match="threshold"):
        model.streaming(keywords=["да"], threshold=1.5)
    with pytest.raises(ValueError, match="outside"):
        model.streaming(keywords=[[999]])
    with pytest.raises(ValueError, match="more than 64"):
        model.streaming(keywords=[[1] * 65])
    with pytest.raises(NotImplementedError, match="CTC head"):
        _cpu_model("v2_rnnt").streaming(keywords=["да"])
    srv = model.streaming()
    with pytest.raises(ValueError, match="not open"):
        srv.push(0, np.zeros(10, np.float32))
    with pytest.raises(ValueError, match="not open"):
        srv.close(7)
    assert srv.streams == [] and srv.step() == []
    assert srv._eng is None                                                 # nothing reached the device


def test_stream_symbols_are_exported():
    lib = _lib.load()
    for name in ("gam_ctc_spot_state_bytes", "gam_ctc_spot_state_init", "gam_ctc_spot_resume"):
        assert name in _lib.EXPORTS and hasattr(lib, name)
    for name in ("StreamServer", "StreamUpdate", "StreamResult"):
        assert name in gigaam.__all__ and hasattr(gigaam, name)
    assert gigaam.StreamServer is StreamServer and hasattr(gigaam.GigaAMASR, "streaming")


# ------------------------------------------------------------------------------------------ GPU helpers
def _dev():
    return torch.device("cuda", 0)


_MODELS = {}


def _model(name):
    if name not in _MODELS:
        ck = synthetic.synthetic_checkpoint(name, seed=0, n_layers=1)
        _MODELS[name] = gigaam.load_model(name, fp16_encoder=False, device=_dev(), checkpoint=ck)
    return _MODELS[name]


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


# ------------------------------------------------------------------------------------------ GPU: the prerequisite
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v3_e2e_ctc", "v2_rnnt"])
def test_window_encoding_does_not_depend_on_its_batch(name):
    """A window's encoder output (and CTC log-probs) are the same bits alone and at any row of a batch of 2-64 equal-length
    windows: what lets a stream server batch windows of unrelated streams."""
    from gigaam_b200.longform import encode_rows
    model = _model(name)
    wav, _ = synthetic.synthetic_audio(1, 140.0, seed=21)
    W = 8 * 16000
    rows = [wav[0, i * 16000: i * 16000 + W].to(model._dtype) for i in range(64)]
    with torch.inference_mode():
        alone = [encode_rows(model, [r]) for r in rows]
        ctc = model._ncfg["head"]["type"] == "ctc"
        alone_lp = [model.head(e) for e in alone] if ctc else None
        rng = random.Random(5)
        for size in (2, 3, 5, 16, 17, 64):
            pick = rng.sample(range(64), size)
            enc = encode_rows(model, [rows[i] for i in pick])
            lp = model.head(enc) if ctc else None
            for j, i in enumerate(pick):
                assert torch.equal(_bits(enc[j]), _bits(alone[i][0])), (size, j)
                if ctc:
                    assert torch.equal(_bits(lp[j]), _bits(alone_lp[i][0])), (size, j)


# ------------------------------------------------------------------------------------------ GPU: transcripts
def _drive(srv, wavs, rng, on_update=None):
    """Push every recording in random chunks, interleaved, stepping at random moments and closing each stream once all of
    it is pushed.  Returns {index: StreamResult} and the updates per index."""
    ids = [srv.open() for _ in wavs]
    pos = [0] * len(wavs)
    styles = [rng.choice(["tiny", "big", "edges", "random"]) for _ in wavs]
    results, updates = {}, {i: [] for i in range(len(wavs))}
    W, H = srv.W, srv.W - srv.V
    while len(results) < len(wavs):
        for i, w in enumerate(wavs):
            if i in results or rng.random() < 0.3:
                continue
            N = w.numel()
            if pos[i] < N:
                if styles[i] == "tiny":
                    c = rng.choice([1, 3, 160])
                elif styles[i] == "big":
                    c = rng.randint(16000, 200000)
                elif styles[i] == "edges":        # end exactly at the next w H + W
                    c = max(1, ((pos[i] - W) // H + 1) * H + W - pos[i]) if pos[i] >= W else W - pos[i]
                else:
                    c = rng.randint(1, 80000)
                c = min(c, N - pos[i])
                srv.push(ids[i], w[pos[i]:pos[i] + c].numpy())
                pos[i] += c
            elif rng.random() < 0.5:
                results[i] = srv.close(ids[i], word_timestamps=True, pause=0.3, max_segment=6.0)
        if rng.random() < 0.4:
            for u in srv.step():
                i = ids.index(u.stream)
                updates[i].append(u)
                if on_update:
                    on_update(i, u)
    return results, updates


def _recordings(seed, n=12):
    rng = random.Random(seed)
    W, H = 8 * 16000, 4 * 16000
    lengths = [W - 1000, W, 2 * H + W, H + W + 1, 640 * 3 + 5] + [rng.randint(W, 70 * 16000) for _ in range(n - 5)]
    wav, _ = synthetic.synthetic_audio(1, 72.0, seed=seed)
    out = []
    for k, N in enumerate(lengths):
        start = rng.randint(0, wav.shape[1] - N)
        out.append(wav[0, start:start + N].clone())
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("confidence", [False, True])
@pytest.mark.parametrize("name", ["v2_ctc", "v2_rnnt", "v3_e2e_rnnt"])
def test_closed_streams_equal_transcribe_windowed(name, confidence):
    model = _model(name)
    wavs = _recordings(len(name) + confidence)
    rng = random.Random(17 + confidence)
    with torch.inference_mode():
        srv = model.streaming(window=8.0, overlap=4.0, batch_size=5, confidence=confidence)
        results, updates = _drive(srv, wavs, rng)
        assert srv.streams == []
        with pytest.raises(ValueError, match="not open"):
            srv.push(0, np.zeros(5, np.float32))
        with pytest.raises(ValueError, match="not open"):
            srv.close(3)
        b = srv.open()
        with pytest.raises(ValueError, match="empty"):
            srv.close(b)
        assert srv.streams == [] and len(srv._free) == srv._dec_pool.shape[0]      # every slot is free again
        tok = model.decoding.tokenizer
        for i, w in enumerate(wavs):
            want = model.transcribe_windowed(w, word_timestamps=True, confidence=confidence, window=8.0, overlap=4.0, pause=0.3,
                                              max_segment=6.0)
            got = results[i].transcript
            assert repr(got) == repr(want), i
            assert results[i].detections is None
            committed = [t for u in updates[i] for t in u.new_tokens]
            assert "".join(u.new_text for u in updates[i]) == tok.decode(committed)
            times = [u.committed_until for u in updates[i]]
            assert times == sorted(times)
    assert sum(len(u) for u in updates.values()) > 12


# ------------------------------------------------------------------------------------------ GPU: resumable spotting
def _planted_log_probs(g, B, T, V1, keywords, nan_rows):
    """Random log-probs with the keywords planted a few times each (one frame or more per token, a blank between tokens
    now and then), near misses and NaN rows."""
    logits = torch.randn(B, T, V1, generator=g) * 1.5
    blank = V1 - 1
    rng = random.Random(int(torch.randint(0, 1 << 30, (1,), generator=g)))
    for b in range(B):
        for _ in range(T // 40):
            kw = rng.choice(keywords)
            t = rng.randrange(T)
            for j, tok in enumerate(kw):
                for _ in range(rng.choice([1, 1, 2, 3])):
                    if t >= T:
                        break
                    logits[b, t, tok] += rng.choice([6.0, 6.0, 2.0])
                    t += 1
                if j + 1 < len(kw) and (kw[j + 1] == tok or rng.random() < 0.3) and t < T:
                    logits[b, t, blank] += 6.0
                    t += 1
        for t in nan_rows:
            logits[b, t, rng.randrange(V1)] = float("nan")
    return logits.log_softmax(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v3_e2e_ctc"])
def test_resumed_spotting_equals_the_one_shot_kernel(name):
    eng = _model(name)._get_engine()
    V1 = eng.num_classes
    g = torch.Generator().manual_seed(V1)
    rng = random.Random(V1)
    keywords = [[5], [3, 3], [1, 2, 1, 2], [7, 8, 9], [4, 4, 4, 6], [rng.randrange(V1 - 1) for _ in range(64)],
                [rng.randrange(V1 - 1) for _ in range(12)], [2]]
    K, Umax = len(keywords), 64
    kw = torch.zeros(K, Umax, dtype=torch.int32)
    for k, r in enumerate(keywords):
        kw[k, :len(r)] = torch.tensor(r)
    kw_len = torch.tensor([len(r) for r in keywords], dtype=torch.int32)
    kw_d, kw_len_d = kw.to(_dev()), kw_len.to(_dev())
    B, T = 3, 1500
    nan_rows = [200, 201, 777]
    lp = _planted_log_probs(g, B, T, V1, keywords, nan_rows).to(_dev()).contiguous()
    lens = [1500, 1311, 640]
    thr = 0.4
    start, end, score, count = (t.cpu() for t in eng.ctc_spot(lp, torch.tensor(lens), kw_d, kw_len_d, thr, 512))
    assert int(count.min()) >= 0 and int(count.sum()) > 3 * K
    saw_pending_edge = False
    for trial in range(6):
        bounds = []
        for b in range(B):
            L = lens[b]
            dets = [(int(start[b, k, i]), int(end[b, k, i])) for k in range(K) for i in range(int(count[b, k]))]
            edges = {rng.randrange(L + 1) for _ in range(rng.randint(1, 15))}
            for s, e in rng.sample(dets, min(6, len(dets))):
                edges |= {s + 1, e - 1, e}                          # inside a detection, at its last frame, just after it
            edges |= {t for t in (200, 201, 202, 777, 778) if rng.random() < 0.5}
            if trial == 0:
                edges = set(range(0, L + 1, 1 if b == 2 else 97))    # one frame per call on one row
            bounds.append(sorted({0, L} | {min(x, L) for x in edges}))
        state = eng.spot_state(B, K, Umax)
        got = [[[] for _ in range(K)] for _ in range(B)]
        calls = max(len(x) for x in bounds) - 1
        for c in range(calls):
            lo = [x[c] if c + 1 < len(x) else lens[b] for b, x in enumerate(bounds)]
            hi = [x[c + 1] if c + 1 < len(x) else lens[b] for b, x in enumerate(bounds)]
            fin = [int(c == calls - 1)] * B
            rngs = torch.tensor([lo, hi, [0] * B, fin], dtype=torch.int32).to(_dev())
            max_det = max(h - l for l, h in zip(lo, hi)) + 2     # a carried detection plus disjoint ones of >= 1 frame
            i32 = dict(dtype=torch.int32, device=_dev())
            det = (torch.full((B, K, max_det), -7, **i32), torch.full((B, K, max_det), -7, **i32),
                   torch.full((B, K, max_det), 7.0, device=_dev()), torch.zeros((B, K), **i32))
            pend = (torch.empty((B, K), **i32), torch.empty((B, K), **i32), torch.empty((B, K), device=_dev()))
            eng.ctc_spot_resume(lp, rngs[0], rngs[1], rngs[2], rngs[3], kw_d, kw_len_d, thr, state, det, pend)
            d = [t.cpu() for t in det + pend]
            for b in range(B):
                for k in range(K):
                    n = int(d[3][b, k])
                    assert (d[0][b, k, n:] == -7).all()              # nothing past the appended detections is written
                    for i in range(n):
                        got[b][k].append((int(d[0][b, k, i]), int(d[1][b, k, i]), int(_bits(d[2][b, k, i]))))
                        j = len(got[b][k]) - 1                       # final: the one-shot kernel's j-th detection, for good
                        assert got[b][k][j] == (int(start[b, k, j]), int(end[b, k, j]), int(_bits(score[b, k, j]))), (b, k, j)
                    if int(d[4][b, k]) >= 0:
                        saw_pending_edge |= hi[b] < lens[b]
                        assert int(d[5][b, k]) <= hi[b] and float(d[6][b, k]) <= 0.0
                    else:
                        assert int(d[5][b, k]) == -1 and float(d[6][b, k]) == float("-inf")
        for b in range(B):
            for k in range(K):
                assert len(got[b][k]) == int(count[b, k]), (trial, b, k)
        tot = state.view(torch.int32)[:, :, 3].cpu()                 # the record's true count
        assert torch.equal(tot, count), trial
    assert saw_pending_edge


@pytest.mark.gpu
def test_spot_resume_refusals():
    eng = _model("v2_ctc")._get_engine()
    lib, h = eng.lib, eng.handle
    assert lib.gam_ctc_spot_state_bytes(h, 0) == -1 and lib.gam_ctc_spot_state_bytes(h, 65) == -1
    assert lib.gam_ctc_spot_state_bytes(h, 1) == 64 and lib.gam_ctc_spot_state_bytes(h, 64) == 32 + 32 * 32
    assert _model("v2_rnnt")._get_engine().lib.gam_ctc_spot_state_bytes(_model("v2_rnnt")._get_engine().handle, 4) == -1
    V1 = eng.num_classes
    lp = torch.zeros(1, 4, V1, device=_dev())
    z = torch.zeros(4, dtype=torch.int32, device=_dev())
    kw = torch.ones(1, 2, dtype=torch.int32, device=_dev())
    klen = torch.full((1,), 2, dtype=torch.int32, device=_dev())
    st = eng.spot_state(1, 1, 2)
    out = [torch.zeros(8, dtype=torch.int32, device=_dev()) for _ in range(7)]
    args = lambda rec=st.shape[2], state=st.data_ptr(), lo=z.data_ptr(): (  # noqa: E731
        h, lp.data_ptr(), 1, 4, lo, z.data_ptr(), z.data_ptr(), z.data_ptr(), kw.data_ptr(), klen.data_ptr(), 1, 2, 0.5, 4, state, rec,
        *[t.data_ptr() for t in out], eng._stream())
    assert lib.gam_ctc_spot_resume(*args()) == 0
    assert lib.gam_ctc_spot_resume(*args(rec=st.shape[2] + 32)) != 0
    assert b"record_bytes" in lib.gam_last_error(h)
    assert lib.gam_ctc_spot_resume(*args(state=None)) != 0
    assert lib.gam_ctc_spot_resume(*args(lo=None)) != 0
    assert b"required" in lib.gam_last_error(h)
    with pytest.raises(_lib.GamError, match="threshold"):
        eng.ctc_spot_resume(lp, z[:1], z[:1], z[:1], z[:1], kw, klen, 1.5, st, tuple(t.view(1, 1, 8) for t in out[:3]) + (out[3][:1].view(1, 1),))


@pytest.mark.gpu
def test_stream_keywords_equal_spot():
    model = _model("v2_ctc")
    wavs = _recordings(5, n=7)
    tok = model.decoding.tokenizer
    words = {w for x in wavs for w in model.transcribe_windowed(x, window=8.0, overlap=4.0).text.split() if len(w) >= 2}
    keywords = sorted(words)[:6] + ["да", [1, 1], [tok.vocab.index(" "), 2], [3], [5]]
    with torch.inference_mode():
        srv = model.streaming(window=8.0, overlap=4.0, batch_size=3, keywords=keywords, threshold=0.2)
        seen = {}

        def check(i, u):
            seen.setdefault(i, []).extend(u.detections)

        results, updates = _drive(srv, wavs, random.Random(9), check)
        n_det = 0
        for i, w in enumerate(wavs):
            want = model.spot(w, keywords, threshold=0.2, window=8.0, overlap=4.0)
            assert repr(results[i].detections) == repr(want), i
            n_det += len(want)
            # the final detections of the updates are the closed stream's, at nominal 40 ms frames
            ups = seen.get(i, [])
            assert len(ups) <= len(want)
            shift = w.numel() / 16000 / model._encoded_length(w.numel())
            keyed = {(k, round(s)) for k, s in ((d.keyword_index, d.start / shift) for d in want)}
            assert all((d.keyword_index, round(d.start / 0.04)) in keyed for d in ups), i
    assert n_det > 0


# ------------------------------------------------------------------------------------------ GPU: tentative text
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v2_ctc", "v2_rnnt"])
def test_tentative_text_is_a_replay_from_the_committed_state(name):
    from gigaam_b200.decoding import _as_btd
    from gigaam_b200.longform import encode_rows
    model = _model(name)
    eng = model._get_engine()
    tok = model.decoding.tokenizer
    wav, _ = synthetic.synthetic_audio(1, 40.0, seed=33)
    wav = wav[0].to(model._dtype)
    rng = random.Random(2)
    with torch.inference_mode():
        srv = model.streaming(window=8.0, overlap=4.0, batch_size=2)
        a = srv.open()
        pos, checked = 0, 0
        while pos < wav.numel():
            c = min(rng.randint(8000, 150000), wav.numel() - pos)
            srv.push(a, wav[pos:pos + c].numpy())
            pos += c
            for u in srv.step():
                windows = [ready_window(w, srv.W, srv.V) for w in range(ready_count(pos, srv.W, srv.V))]
                state = eng.decode_state(1)
                out = eng.decode_buffers(1, eng.hyp_width(200))
                for w in windows:
                    enc = _as_btd(encode_rows(model, [wav[w.start:w.end]]))
                    f = w.start // FRAME_SAMPLES
                    r = torch.tensor([[w.keep_start - f], [w.keep_end - f], [0]], dtype=torch.int32).to(_dev())
                    out = out._replace(counts=torch.zeros(1, dtype=torch.int32, device=_dev()))
                    eng.greedy_resume(enc, r[0], r[1], r[2], state, out)
                copy = state.clone()
                T_w = enc.shape[1]
                tail = eng.decode_buffers(1, eng.hyp_width(T_w))
                r = torch.tensor([[windows[-1].keep_end - windows[-1].start // FRAME_SAMPLES], [T_w], [0]], dtype=torch.int32).to(_dev())
                eng.greedy_resume(enc, r[0], r[1], r[2], copy, tail)
                n = int(tail.counts[0])
                assert u.tentative_text == tok.decode(tail.ids[0, :n].tolist())
                assert u.committed_until == windows[-1].keep_end * 0.04
                checked += 1
        srv.close(a)
    assert checked >= 3


# ------------------------------------------------------------------------------------------ GPU: memory
@pytest.mark.gpu
def test_stream_device_memory_stays_flat():
    """A 20-minute stream's peak above the baseline stays within the margin transcribe_windowed's test allows over a
    2-minute one, measured the same way."""
    model = _model("v2_ctc")
    peaks = {}
    for minutes in (2, 20, 2, 20):
        wav, _ = synthetic.synthetic_audio(1, 60.0 * minutes, seed=minutes)
        wav = wav[0]
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        with torch.inference_mode():
            srv = model.streaming(window=8.0, overlap=4.0, confidence=True, keywords=["да", "нет"])
            a = srv.open()
            for pos in range(0, wav.numel(), 48000):
                srv.push(a, wav[pos:pos + 48000].numpy())
                srv.step()
            srv.close(a, word_timestamps=True)
            del srv
        torch.cuda.synchronize()
        peaks[minutes] = torch.cuda.max_memory_allocated() - base
    print(f"\npeak above baseline: 2 min {peaks[2] / 2**20:.1f} MiB, 20 min {peaks[20] / 2**20:.1f} MiB")
    assert peaks[20] - peaks[2] < 64 * 2**20
