"""Timing of the emotion head (CUDA events, L2 flushed before every timed launch / step).

    python tools/emo_probe.py [OUT.json]     # prints a table and one JSON line (also written to OUT.json)

  * gam_emo_head alone (both kernels: chunk sums, then mean + Linear + softmax) at B x T' = 64 x 251, 32 x 1251 and
    1 x 5000, with the bandwidth achieved on the bytes it reads (the encoder output once, the chunk sums once, W per
    utterance);
  * get_probs of the full 16-layer synthetic emo model against model(wav, len) of v1_ssl (the same encoder, no head) at
    10 s and 60 s, both loaded with max_encoded_frames=5000, with the emo_head class's share of the profiled kernel time.
The GPU name, power limit and SM clock are read by the same process, before the timings.
"""
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402

dev = torch.device("cuda", 0)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(dev)


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def head_alone(eng, B, T, reps=20):
    d, C = eng.d_model, eng.num_classes
    enc = torch.randn(B, T, d, device=dev)
    enc_len = torch.full((B,), T, dtype=torch.int32, device=dev)
    nbytes = int(eng.lib.gam_emo_workspace_bytes(eng.handle, B, T))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    pooled = torch.empty(B, d, device=dev)
    logits, probs = torch.empty(B, C, device=dev), torch.empty(B, C, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def launch():
        rc = eng.lib.gam_emo_head(eng.handle, enc.data_ptr(), enc_len.data_ptr(), B, T, ws.data_ptr(), nbytes, pooled.data_ptr(),
                                  logits.data_ptr(), probs.data_ptr(), stream)
        assert rc == 0, eng.lib.gam_last_error(eng.handle)
    launch()
    ms = timed(launch, reps)
    read = enc.numel() * 4 + nbytes + B * C * (d + 1) * 4     # encoder output, chunk sums, W and b per utterance
    return ms, read


def step_ms(fn, reps=5):
    with torch.inference_mode():
        fn()
        return timed(fn, reps)


def main():
    info = gpu_info()
    print(f"# {info}", flush=True)
    res = {"gpu": info, "emo_head": [], "step": []}
    emo = gigaam.load_model("emo", device=dev, synthetic=True, max_encoded_frames=5000)
    ssl = gigaam.load_model("v1_ssl", device=dev, synthetic=True, max_encoded_frames=5000)
    eng = emo._get_engine()
    for B, T in ((64, 251), (32, 1251), (1, 5000)):
        ms, read = head_alone(eng, B, T)
        row = dict(B=B, T=T, us=round(ms * 1e3, 2), bytes_read=read, gb_s=round(read / ms / 1e6, 1))
        res["emo_head"].append(row)
        print(f"gam_emo_head B={B:3d} T'={T:5d}: {ms * 1e3:8.2f} us, {read / 1e6:7.1f} MB read, {row['gb_s']:7.1f} GB/s", flush=True)
    for secs in (10.0, 60.0):
        wav = gigaam.synthetic_audio(1, secs, seed=1)[0]
        wav_d, wav_len = wav.to(dev), torch.tensor([wav.shape[1]], device=dev)
        t_emo = step_ms(lambda: emo.get_probs(wav_d[0]))
        t_ssl = step_ms(lambda: ssl(wav_d, wav_len))
        e = emo._get_engine()
        with torch.inference_mode():
            flush.zero_()
            torch.cuda.synchronize()
            e.profile_begin()
            emo.get_probs(wav_d[0])
            prof = e.profile_end()
        total = sum(v[0] for v in prof.values())
        head = prof.get("emo_head", (0.0, 0))[0]
        row = dict(audio=f"{secs:.0f} s", get_probs_ms=round(t_emo, 3), ssl_step_ms=round(t_ssl, 3), emo_head_ms=round(head, 4),
                   emo_head_share=round(head / total, 5) if total else None)
        res["step"].append(row)
        print(f"{secs:4.0f} s: get_probs {t_emo:7.3f} ms, v1_ssl model(wav, len) {t_ssl:7.3f} ms, emo_head {head * 1e3:6.1f} us "
              f"({100 * row['emo_head_share']:.3f} % of the profiled kernel time)", flush=True)
    print(json.dumps(res))
    if len(sys.argv) > 1:
        Path(sys.argv[1]).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
