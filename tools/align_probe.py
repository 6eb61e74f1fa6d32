"""Cost of aligning known transcripts (decoding.align: gam_ctc_align, gam_rnnt_align_scores, gam_rnnt_align), stage by stage,
with CUDA events.

    python tools/align_probe.py

Each shape aligns random target ids of length U to random encoder output [B, T', d] (alignment cost does not depend on the
values) with one-layer synthetic heads, after a warm-up; each figure is the median of the repetitions.  Stages: CTC,
log-probs (gam_ctc_log_probs) and the DP (gam_ctc_align); RNN-T, the prediction network (U + 1 LSTM launches), the gathered
joint scores (stage 1) and the DP (stage 2).  Stage 1's FLOP/s counts the projections and the V + 1 logits of every node and
is set against the H100 SXM data-sheet FP32 rate of 67 TFLOP/s (not a measured peak).  Peak memory is
torch.cuda.max_memory_allocated over one whole align call (weights, inputs, workspaces and
outputs included), set beside the fp32 lattice gam_rnnt_joint would need.  The card
name, power limit and SM clock are read in the same run; the last line is one JSON record of everything printed."""
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402
from gigaam_b200 import decoding  # noqa: E402

dev = torch.device("cuda", 0)
SHAPES = [("v2_ctc", 64, 251, 150), ("v3_e2e_rnnt", 32, 250, 60), ("v2_rnnt", 1, 5000, 3000), ("v3_e2e_rnnt", 1, 5000, 1000)]
FP32_DATASHEET = 67e12


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(dev)


def median_ms(fn, warmup=3, reps=20):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def probe(name, B, T, U):
    ck = gigaam.synthetic_checkpoint(name, seed=0, n_layers=1)
    model = gigaam.load_model(name, fp16_encoder=False, device=dev, checkpoint=ck, max_encoded_frames=max(T, 768))
    eng = model._get_engine()
    V1 = eng.num_classes
    g = torch.Generator().manual_seed(0)
    enc = torch.randn(B, T, eng.d_model, generator=g).to(dev)
    enc_len = torch.full((B,), T, dtype=torch.int32, device=dev)
    targets = torch.randint(0, V1 - 1, (B, U), generator=g, dtype=torch.int32).to(dev)
    tlen = torch.full((B,), U, dtype=torch.int32, device=dev)
    encoded = enc.transpose(1, 2)
    rec = dict(shape=f"{name} {B}x{T}", U=U, classes=V1)
    with torch.inference_mode():
        if eng.head_type == 1:
            lp = eng.ctc_log_probs(enc)
            rec["log_probs_ms"] = median_ms(lambda: eng.ctc_log_probs(enc))
            rec["dp_ms"] = median_ms(lambda: eng.ctc_align(lp, enc_len, targets, tlen))
        else:
            x = torch.cat([torch.full((B, 1), V1 - 1, dtype=torch.int64, device=dev), targets.long()], 1).contiguous()
            dec, _, _ = eng.rnnt_predict(x, None, None)
            blank, label = eng.rnnt_align_scores(enc, dec, targets)
            rec["predict_ms"] = median_ms(lambda: eng.rnnt_predict(x, None, None))
            rec["scores_ms"] = median_ms(lambda: eng.rnnt_align_scores(enc, dec, targets))
            rec["dp_ms"] = median_ms(lambda: eng.rnnt_align(blank, label, enc_len, tlen))
            J, H, d = eng.gam_config.joint_hidden, eng.pred_hidden, eng.d_model
            flops = 2.0 * B * T * (U + 1) * J * V1 + 2.0 * B * T * d * J + 2.0 * B * (U + 1) * H * J
            rec["scores_tflops"] = round(flops / (rec["scores_ms"] * 1e-3) / 1e12, 2)
            rec["scores_share_of_fp32_datasheet"] = round(flops / (rec["scores_ms"] * 1e-3) / FP32_DATASHEET, 3)
            rec["lattice_gb_not_built"] = round(B * T * (U + 1) * V1 * 4 / 1e9, 2)
        rec["align_call_ms"] = median_ms(lambda: decoding.align(model.head, encoded, enc_len, targets, tlen))
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        decoding.align(model.head, encoded, enc_len, targets, tlen)
        torch.cuda.synchronize()
        # everything live during the call: weights, inputs, cached workspaces, intermediates and outputs
        rec["align_peak_device_mb"] = round(torch.cuda.max_memory_allocated(dev) / 1e6, 1)
        rec["align_workspaces_mb"] = round(sum(t.numel() for c in (eng._ws_align, eng._ws_joint) for t in c.tensors()) / 1e6, 1)
    for k, v in rec.items():
        if isinstance(v, float):
            rec[k] = round(v, 4)
    print(rec)
    del model, eng
    torch.cuda.empty_cache()
    return rec


def main():
    gpu = card()
    print("card (name, power limit, SM clock, max SM clock):", gpu)
    recs = [probe(*s) for s in SHAPES]
    print(json.dumps(dict(card=gpu, shapes=recs)))


if __name__ == "__main__":
    main()
