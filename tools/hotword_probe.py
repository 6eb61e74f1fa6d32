"""Cost of CTC hotwords (gam_ctc_bias), alone and after gam_ctc_spot, with CUDA events.

    python tools/hotword_probe.py [--quick]

Random log_softmax rows [1, T, V+1] stand in for stitched long-form log-probs: 10 and 60 minutes of audio (T = 15 000 and
90 000 frames of 40 ms) at V + 1 = 34 (v2_ctc, charwise) and 257 (v3_e2e_ctc, SentencePiece), with 10, 100 and 1000 random
hotwords of 3 to 12 tokens, threshold 0.5.  The greedy input is the argmax collapse of the rows and the flag table is the
model's.  Spot runs as `transcribe` runs it (GigaAMASR._spot_all: max_det = min(T / shortest, 256), and one more launch with
the largest count when a count exceeds that), so every detection is a candidate.  "bias" times gam_ctc_bias alone on those
outputs; "spot + bias" times both.  Each figure is the median of 5 timed calls after 2 warm-up calls.  The card's name, power
limit and SM clocks are read in the same run, before and after.  The last line is one JSON record of everything printed."""
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402

dev = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(dev)


def median_ms(fn, warmup=2, reps=5):
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


def greedy(lp):
    """CTC greedy of lp [1, T, V+1] on the device: ids / frames [1, T] i32, counts [1] i32."""
    T, blank = lp.shape[1], lp.shape[2] - 1
    lab = lp[0].argmax(-1)
    prev = torch.cat([torch.full((1,), blank, device=dev, dtype=lab.dtype), lab[:-1]])
    frames = torch.nonzero((lab != blank) & (lab != prev)).flatten()
    ids = torch.zeros((1, T), dtype=torch.int32, device=dev)
    fr = torch.zeros((1, T), dtype=torch.int32, device=dev)
    ids[0, :frames.numel()] = lab[frames].int()
    fr[0, :frames.numel()] = frames.int()
    return ids, fr, torch.tensor([frames.numel()], dtype=torch.int32, device=dev)


def main(quick):
    rec = {"card_before": card(), "rows": []}
    print(f"card: {rec['card_before']}")
    g = torch.Generator().manual_seed(0)
    for name in ("v2_ctc", "v3_e2e_ctc"):
        ck = gigaam.synthetic_checkpoint(name, seed=0, n_layers=1)
        model = gigaam.load_model(name, fp16_encoder=False, device=dev, checkpoint=ck)
        eng = model._get_engine()
        flags = model._word_flags()
        V1 = eng.num_classes
        ok = (flags[:V1 - 1] & 1) == 0                                   # hotwords neither start nor end with a space
        letters = torch.nonzero(ok.cpu()).flatten()
        for minutes in ((10,) if quick else (10, 60)):
            T = minutes * 60 * 25
            lp = torch.randn(1, T, V1, generator=g).mul_(2.0).log_softmax(-1).to(dev)
            enc_len = torch.tensor([T], dtype=torch.int32, device=dev)
            ids, frames, counts = greedy(lp)
            for K in ((10, 100) if quick else (10, 100, 1000)):
                lens = torch.randint(3, 13, (K,), generator=g, dtype=torch.int32)
                kw = letters[torch.randint(0, letters.numel(), (K, 12), generator=g)].int()
                kw_d, lens_d = kw.to(dev), lens.to(dev)
                rows = [kw[k, :int(lens[k])].tolist() for k in range(K)]
                spotted = model._spot_all(lp, enc_len, kw_d, lens_d, rows, 0.5)

                def bias():
                    return eng.ctc_bias(lp, enc_len, kw_d, lens_d, spotted, 0.5, flags, ids, frames, counts)

                def both():
                    s = model._spot_all(lp, enc_len, kw_d, lens_d, rows, 0.5)
                    return eng.ctc_bias(lp, enc_len, kw_d, lens_d, s, 0.5, flags, ids, frames, counts)
                ms_bias, ms_both = median_ms(bias), median_ms(both)
                out = bias()
                dets = int(spotted[3].sum())
                changed = int((out[3][0, :int(out[2][0])] >= 0).sum())
                row = dict(V1=V1, minutes=minutes, frames=T, keywords=K, max_det=int(spotted[0].shape[2]), detections=dets,
                           tokens_from_hotwords=changed,
                           bias_ms=round(ms_bias, 3), spot_bias_ms=round(ms_both, 3))
                rec["rows"].append(row)
                print(f"V+1 = {V1:4d}, {minutes:2d} min ({T} frames), K = {K:4d}, {dets:6d} detections, {changed:5d} tokens "
                      f"from hotwords: bias {ms_bias:8.3f} ms, spot + bias {ms_both:8.3f} ms")
            del lp
    rec["card_after"] = card()
    print(f"card after: {rec['card_after']}")
    print(json.dumps(rec))


if __name__ == "__main__":
    main("--quick" in sys.argv)
