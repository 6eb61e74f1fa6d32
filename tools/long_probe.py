"""Timing of long utterances (CUDA events, L2 flushed before every timed launch / step), on models loaded with
max_encoded_frames=5000.

    python tools/long_probe.py [OUT.json]     # prints a table and one JSON line (also written to OUT.json)

  * the rotary and rel_pos attention kernels alone (packed rows, the path gam_encode takes) at T' = 768, 1536, 3072 and
    5000, for one utterance and for a ragged packed batch;
  * model(wav, len) of the full 16-layer v2_ctc and v1_ctc at 30, 60 and 120 s and at T' = 5000 for one utterance, with
    the attention class's share from the library's per-launch profile (gam_profile_*).
The GPU name, power limit and SM clock are read by the same process, before the timings.
"""
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402
from gigaam_b200.engine import Engine  # noqa: E402

dev = torch.device("cuda", 0)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
MAX_T = 5000


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


def attention_ms(eng, relpos, lens, reps=10):
    d = 768
    parts = 4 if relpos else 3
    rows, T = sum(lens), max(lens)
    g = torch.Generator().manual_seed(rows + relpos)
    qkv = torch.randn(rows, parts * d, generator=g).half().to(dev)
    pos = torch.randn(2 * MAX_T - 1, d, generator=g).half().to(dev)
    out = torch.zeros(rows, d, dtype=torch.float16, device=dev)
    klen = torch.tensor(lens, dtype=torch.int32, device=dev)
    cu = torch.tensor([0] + [sum(lens[: i + 1]) for i in range(len(lens))], dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream().cuda_stream

    def launch():
        rc = eng.lib.gam_test_attention_varlen(eng.handle, qkv.data_ptr(), pos.data_ptr() if relpos else None, klen.data_ptr(),
                                               cu.data_ptr(), out.data_ptr(), len(lens), T, rows, stream)
        assert rc == 0, eng.lib.gam_last_error(eng.handle)
    launch()
    return timed(launch, reps)


def attention_flop(lens):
    # S = QK^T and P.V, 16 heads of 48: 4 * n^2 * 768 per utterance (rel_pos adds its position product on top)
    return sum(4.0 * n * n * 768 for n in lens)


def step(model, n_samples, reps=5):
    wav, wav_len = gigaam.synthetic_audio(1, n_samples / 16000.0, seed=1)
    wav = wav[:, :n_samples].contiguous().to(dev)
    wav_len = torch.tensor([n_samples], device=dev)
    with torch.inference_mode():
        enc, _ = model(wav, wav_len)
        ms = timed(lambda: model(wav, wav_len), reps)
        eng = model._get_engine()
        flush.zero_()
        torch.cuda.synchronize()
        eng.profile_begin()
        model(wav, wav_len)
        prof = eng.profile_end()
    total = sum(v[0] for v in prof.values())
    return enc.shape[2], ms, prof.get("attention", (0.0, 0))[0], total


def main():
    info = gpu_info()
    print(f"# {info}", flush=True)
    res = {"gpu": info, "attention": [], "step": []}
    engines = {}
    for which, relpos in (("v2_ctc", False), ("v1_ctc", True)):
        ck = gigaam.synthetic_checkpoint(which, n_layers=1)
        engines[relpos] = Engine(ck["cfg"], ck["state_dict"], dev, max_encoded_frames=MAX_T)
    g = torch.Generator().manual_seed(0)
    for T in (768, 1536, 3072, 5000):
        ragged = [T] + [int(x) for x in torch.randint(T // 8, T + 1, (7,), generator=g)]
        for lens, label in (([T], "B=1"), (ragged, "ragged B=8")):
            for relpos in (False, True):
                ms = attention_ms(engines[relpos], relpos, lens)
                tf = attention_flop(lens) / ms / 1e9
                row = dict(kernel="rel_pos" if relpos else "rotary", T=T, batch=label, rows=sum(lens), ms=round(ms, 4),
                           tflops_qk_pv=round(tf, 1))
                res["attention"].append(row)
                print(f"attention {row['kernel']:7s} T'={T:5d} {label:10s} rows={sum(lens):6d}: {ms:8.3f} ms  "
                      f"({tf:5.1f} TFLOP/s on S and P.V)", flush=True)
    del engines
    for which in ("v2_ctc", "v1_ctc"):
        ck = gigaam.synthetic_checkpoint(which, seed=0)
        model = gigaam.load_model(which, device=dev, checkpoint=ck, max_encoded_frames=MAX_T)
        for label, n in (("30 s", 480_000), ("60 s", 960_000), ("120 s", 1_920_000), ("T'=5000", 3_199_519)):
            T, ms, att, prof_total = step(model, n)
            row = dict(model=which, audio=label, T=T, step_ms=round(ms, 2), attention_ms=round(att, 2),
                       attention_share=round(att / prof_total, 3) if prof_total else None)
            res["step"].append(row)
            print(f"model(wav, len) {which} {label:8s} T'={T:5d}: {ms:8.2f} ms, attention {att:7.2f} ms "
                  f"({100 * row['attention_share']:.1f} % of the profiled kernel time)", flush=True)
        del model
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if len(sys.argv) > 1:
        Path(sys.argv[1]).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
