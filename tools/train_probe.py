"""Timing of one frozen-encoder training step per head type, with CUDA events.

    python tools/train_probe.py

For a 2-layer synthetic v2_ctc and v2_rnnt model, B = 16 utterances of 10 s and 20-token targets, one step is timed in five
phases: the encoder forward (no grad), the head forward (CTCHead.forward, or RNNTDecoder.predict + RNNTJoint.joint), the
loss (torch's ctc_loss, or torchaudio's rnnt_loss on log-probs), the backward (the head kernels of csrc/head_grads.cu),
and AdamW.  Each phase is the median of the repetitions.  The card name and power limit are read in the same run.  The
last line is one JSON record of everything printed.
"""
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402

dev = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(dev)


def probe(name, B=16, seconds=10.0, n_tok=20, reps=10):
    ck = gigaam.synthetic_checkpoint(name, seed=0, n_layers=2)
    model = gigaam.load_model(name, device=dev, checkpoint=ck)
    model.head.requires_grad_(True)
    V1 = model._get_engine().num_classes
    wav, wav_len = gigaam.synthetic_audio(B, seconds, seed=1)
    wav, wav_len = wav.to(dev), wav_len.to(dev)
    tgt = torch.randint(0, V1 - 1, (B, n_tok), device=dev)
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4, weight_decay=1e-3)
    if "rnnt" in name:
        import torchaudio.functional as ta
    phases = {k: [] for k in ("encoder", "head", "loss", "backward", "optimizer")}
    for i in range(reps + 2):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
        opt.zero_grad(set_to_none=True)
        ev[0].record()
        with torch.no_grad():
            enc, enc_len = model(wav, wav_len)
        ev[1].record()
        if "rnnt" in name:
            blank = torch.full((B, 1), V1 - 1, dtype=torch.long, device=dev)
            dec, _ = model.head.decoder.predict(torch.cat([blank, tgt], 1), None)
            lp = model.head.joint.joint(enc.transpose(1, 2), dec)
            ev[2].record()
            loss = ta.rnnt_loss(lp, tgt.int(), enc_len.int(), torch.full((B,), n_tok, dtype=torch.int32, device=dev),
                                blank=V1 - 1, reduction="mean", fused_log_softmax=False)
        else:
            lp = model.head(enc)
            ev[2].record()
            loss = F.ctc_loss(lp.transpose(0, 1), tgt, enc_len.long(), torch.full((B,), n_tok, dtype=torch.long, device=dev),
                              blank=V1 - 1, reduction="none", zero_infinity=True).mean()
        ev[3].record()
        loss.backward()
        ev[4].record()
        opt.step()
        ev[5].record()
        torch.cuda.synchronize()
        if i >= 2:
            for k, (a, b) in zip(phases, zip(ev[:-1], ev[1:])):
                phases[k].append(a.elapsed_time(b))
    med = {k: sorted(v)[len(v) // 2] for k, v in phases.items()}
    med["step"] = sum(med.values())
    print(f"{name}: B={B} x {seconds:.0f} s, {n_tok} tokens: " + ", ".join(f"{k} {v:.2f} ms" for k, v in med.items()))
    return med


if __name__ == "__main__":
    rec = {"card": card(), "v2_ctc": probe("v2_ctc"), "v2_rnnt": probe("v2_rnnt")}
    print(f"card: {rec['card']}")
    print(json.dumps(rec))
