"""Time and peak memory of the RNN-T loss, forward + backward, by two routes.

    python tools/rnnt_loss_probe.py [--out DIR]

fused:   decoding.rnnt_loss (csrc/rnnt_loss.cu: three floats per lattice node, the joint recomputed tile by tile).
lattice: RNNTDecoder.predict + RNNTJoint.joint's [B, T', U+1, V+1] log-probs + torchaudio's rnnt_loss, with the joint
         backward of csrc/head_grads.cu; run only below 2^31 lattice elements, which torchaudio's CUDA loss requires.
Synthetic 2-layer models with every head parameter trainable; encoder outputs and targets are random, U_b = U for every
utterance.  Each time is the median of the repetitions (CUDA events around forward + backward, after a warm-up); the peak
is torch.cuda.max_memory_allocated above what was allocated before the call.  The card name, power limit and SM clock are
read in the same run.  The last line is one JSON record of everything printed.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402
from gigaam_b200 import decoding  # noqa: E402

dev = torch.device("cuda", 0)
CONFIGS = [("v3_e2e_rnnt", 32, 250, 60), ("v2_rnnt", 32, 376, 60), ("v3_e2e_rnnt", 8, 750, 150), ("v3_e2e_rnnt", 32, 750, 150),
           ("v3_e2e_rnnt", 1, 5000, 1000)]
# torchaudio's CUDA rnnt_loss indexes the lattice with 32-bit ints (the reference fine-tuner halves its sub-batch until
# B T (U+1) V < 2^31 for this reason), so the lattice route runs only below that many elements
LATTICE_MAX_ELEMENTS = 2 ** 31 - 1


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(dev)


def lattice_loss(model, enc, enc_len, y, tlen):
    import torchaudio.functional as ta
    V1 = model._get_engine().num_classes
    _, x = decoding._rnnt_inputs(model._get_engine(), y, tlen)
    dec, _ = model.head.decoder.predict(x, None)
    lp = model.head.joint.joint(enc.transpose(1, 2), dec)
    return ta.rnnt_loss(lp, y.int(), enc_len.int(), tlen.int(), blank=V1 - 1, reduction="mean", fused_log_softmax=False)


def measure(fn, reps):
    times = []
    for i in range(reps + 1):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn().backward()
        b.record()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        if i > 0:
            times.append(a.elapsed_time(b))
    return sorted(times)[len(times) // 2], peak


def probe(name, B, T, U, reps):
    ck = gigaam.synthetic_checkpoint(name, seed=0, n_layers=2)
    model = gigaam.load_model(name, device=dev, checkpoint=ck, max_encoded_frames=max(T, 768))
    model.head.requires_grad_(True)
    V1 = model._get_engine().num_classes
    g = torch.Generator(device=dev).manual_seed(0)
    enc = torch.randn(B, 768, T, generator=g, device=dev)
    enc_len = torch.full((B,), T, dtype=torch.int32, device=dev)
    y = torch.randint(0, V1 - 1, (B, U), generator=g, device=dev)
    tlen = torch.full((B,), U, dtype=torch.int32, device=dev)
    nodes = B * T * (U + 1)
    rec = dict(model=name, B=B, T=T, U=U, V1=V1, nodes=nodes, lattice_gb=round(nodes * V1 * 4 / 1e9, 2))
    ms, peak = measure(lambda: decoding.rnnt_loss(model.head, enc, enc_len, y, tlen), reps)
    rec.update(fused_ms=round(ms, 2), fused_peak_gb=round(peak / 1e9, 3), fused_bytes_per_node=round(peak / nodes, 1))
    if nodes * V1 <= LATTICE_MAX_ELEMENTS:
        ms, peak = measure(lambda: lattice_loss(model, enc, enc_len, y, tlen), reps)
        rec.update(lattice_ms=round(ms, 2), lattice_peak_gb=round(peak / 1e9, 3))
        model.head.zero_grad(set_to_none=True)
        torch.cuda.empty_cache()
    else:
        rec.update(lattice_ms="not run: lattice above 2^31 elements")
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON record to DIR/rnnt_loss_probe.json")
    args = ap.parse_args()
    info = dict(card=card())
    print(info, flush=True)
    info["rows"] = [probe(*c, reps=args.reps) for c in CONFIGS]
    line = json.dumps(info)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "rnnt_loss_probe.json").write_text(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
