"""Cost of long-form alignment (GigaAMASR.align_longform: window encoding, CTC log-probs, stitching, gam_ctc_align_long and
word grouping), with CUDA events.

    python tools/align_long_probe.py [--quick] [--gaps] [--skips]

Part 1, the kernel: gam_ctc_align_long on random log-probs [1, 2000, 34] for U = 1k ... 64k tokens at forced cluster sizes
C = 1, 4 and 16 (where the states fit), as time per frame.  The backtrack's share is the difference to the same call with one
target class at -inf on every frame: that sweep does the same work, but there is no path to walk back.
Part 2, the whole call on synthetic 16-layer models (fp16 encoder) over 10 and 60 minutes of synthetic audio, at V + 1 = 34
(v2_ctc) and 257 (v3_e2e_ctc), with random targets of U = min(T / 2, 65 536) tokens: each stage timed on its own, and the
peak device memory (torch.cuda.max_memory_allocated) of one whole pass.
Part 3, alignment with gaps: gam_ctc_align_long_gaps (its row-max pre-pass and sweep) against gam_ctc_align_long on the same
random log-probs at V + 1 = 34 and 257, for T = 2000 frames at U = 1k ... 64k tokens in lines of 500 tokens, and for an hour
(T = 90 000, U = 65 536), at the library's cluster size; medians of 7 (3 for the hour), the two calls alternating.  --gaps runs
part 3 alone.
Part 4, alignment with skipped lines: gam_ctc_align_long_skips against gam_ctc_align_long_gaps at part 3's shapes and theta,
psi = 0.5, with lines of 500 tokens and of 12 tokens (short lines: many skip edges, an exit blank in most warps), the two
calls alternating as in part 3.  A skip source is read from another CTA only when its line crosses a CTA boundary, so at
most C - 1 lines per recording do (none at U <= 4 096, where the library's plan is C = 1).  --skips runs part 4 alone.
The card's name, power limit and SM clocks are read in the same run; the last line is one JSON record of everything printed."""
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402
from gigaam_b200 import _lib, longform  # noqa: E402

dev = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(dev)


def median_ms(fn, warmup=2, reps=7):
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


def kernel_part(quick):
    ck = gigaam.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1)
    eng = gigaam.load_model("v2_ctc", fp16_encoder=False, device=dev, checkpoint=ck)._get_engine()
    T, V1 = 2000, eng.num_classes
    g = torch.Generator().manual_seed(0)
    lp = torch.randn(1, T, V1, generator=g).log_softmax(-1).to(dev)
    dead = lp.clone()
    dead[..., 0] = -float("inf")
    rows = []
    for U in ([1024, 65536] if quick else [1024, 4096, 16384, 32768, 65536]):
        y = (torch.randint(0, V1 - 2, (1, U), generator=g) + 1).to(torch.int32)
        y[0, 0] = 0
        args = (torch.tensor([T]), y.to(dev), torch.tensor([U]))
        for C in (1, 4, 16):
            try:
                ms = median_ms(lambda: eng.ctc_align_long(lp, *args, cluster_ctas=C))
            except _lib.GamError:           # this C leaves a CTA without states, or its share does not fit
                continue
            plan = eng.last_align_long_plan
            no_bt = median_ms(lambda: eng.ctc_align_long(dead, *args, cluster_ctas=C))
            rows.append(dict(U=U, S=2 * U + 1, C=C, P=plan[1], ms=round(ms, 3), us_per_frame=round(ms * 1e3 / T, 3),
                             backtrack_ms=round(ms - no_bt, 3), backtrack_share=round((ms - no_bt) / ms, 3)))
            print(f"U={U:6d} S={2 * U + 1:6d} C={C:2d} P={plan[1]:5d}: {ms:8.3f} ms = {ms * 1e3 / T:7.3f} us/frame, "
                  f"backtrack {ms - no_bt:6.3f} ms ({(ms - no_bt) / ms:.1%})", flush=True)
    return rows


def timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return out, a.elapsed_time(b)


def call_part(name, minutes, batch_size=16):
    model = gigaam.load_model(name, device=dev, checkpoint=gigaam.synthetic_checkpoint(name, seed=0))
    eng = model._get_engine()
    wav, _ = gigaam.synthetic_audio(1, 60.0 * minutes, seed=1)
    wav, _ = model.prepare_wav(wav[0])
    wav = wav[0]
    windows, T = longform.plan_windows(wav.numel(), 30.0, 4.0, model._encoded_length, 768)
    U = min(T // 2, 65536)
    g = torch.Generator().manual_seed(1)
    y = torch.randint(0, eng.num_classes - 1, (1, U), generator=g, dtype=torch.int32).to(dev)
    groups = []
    for w in windows:
        if groups and len(groups[-1]) < batch_size and groups[-1][0].end - groups[-1][0].start == w.end - w.start:
            groups[-1].append(w)
        else:
            groups.append([w])

    def encode(head):
        with torch.inference_mode():
            for group in groups:
                n = group[0].end - group[0].start
                enc, _ = model.forward(torch.stack([wav[w.start:w.end] for w in group]), torch.full((len(group),), n, device=dev))
                if head:
                    model.head(enc)

    def stitch():
        with torch.inference_mode():
            return longform.stitch_ctc_log_probs(model, wav, windows, T, batch_size)

    encode(True)                                  # warm-up: every window shape
    torch.cuda.reset_peak_memory_stats()
    _, enc_ms = timed(lambda: encode(False))
    _, enc_head_ms = timed(lambda: encode(True))
    lp, stitch_ms = timed(stitch)
    args = (torch.tensor([T]), y, torch.tensor([U]))
    eng.ctc_align_long(lp, *args)
    out, dp_ms = timed(lambda: eng.ctc_align_long(lp, *args))
    frames = out[0]
    flags = model._word_flags()
    tl = torch.tensor([U], dtype=torch.int32, device=dev)
    _, words_ms = timed(lambda: [t.cpu() for t in eng.group_words(y, frames, tl, flags)])
    peak = torch.cuda.max_memory_allocated() / 2**30
    row = dict(model=name, minutes=minutes, V1=eng.num_classes, windows=len(windows), T=T, U=U, encode_ms=round(enc_ms, 1),
               log_probs_ms=round(enc_head_ms - enc_ms, 1), stitch_copy_ms=round(stitch_ms - enc_head_ms, 1), dp_ms=round(dp_ms, 1),
               words_ms=round(words_ms, 1), peak_gib=round(peak, 2), viterbi_finite=bool(torch.isfinite(out[2]).all()))
    print(row, flush=True)
    del lp, out, model, eng
    torch.cuda.empty_cache()
    return row


def gaps_part(quick):
    rows = []
    for name in ("v2_ctc", "v3_e2e_ctc"):
        ck = gigaam.synthetic_checkpoint(name, seed=0, n_layers=1)
        eng = gigaam.load_model(name, fp16_encoder=False, device=dev, checkpoint=ck)._get_engine()
        V1 = eng.num_classes
        g = torch.Generator().manual_seed(V1)
        sizes = [(2000, 1024), (2000, 65536)] if quick else [(2000, u) for u in (1024, 4096, 16384, 32768, 65536)]
        for T, U in sizes + [(90000, 65536)]:
            lp = torch.randn(1, T, V1, generator=g).log_softmax(-1).to(dev)
            y = torch.randint(0, V1 - 1, (1, U), generator=g, dtype=torch.int32).to(dev)
            edges = torch.tensor(longform.line_edges([(a, min(a + 500, U)) for a in range(0, U, 500)], U), dtype=torch.uint8)
            args = (torch.tensor([T]), y, torch.tensor([U]))
            gaps = (edges[None].to(dev), -0.6931472)
            reps, warm = (3, 1) if T > 2000 else (7, 2)
            plain_ms, gap_ms = [], []
            for _ in range(warm):
                eng.ctc_align_long(lp, *args)
                eng.ctc_align_long(lp, *args, gaps=gaps)
            for _ in range(reps):                 # alternating, so that drift of the clocks hits both
                plain_ms.append(median_ms(lambda: eng.ctc_align_long(lp, *args), warmup=0, reps=1))
                gap_ms.append(median_ms(lambda: eng.ctc_align_long(lp, *args, gaps=gaps), warmup=0, reps=1))
            a, b = statistics.median(plain_ms), statistics.median(gap_ms)
            rows.append(dict(V1=V1, T=T, U=U, plain_ms=round(a, 3), gaps_ms=round(b, 3), ratio=round(b / a, 3)))
            print(f"V+1={V1:4d} T={T:6d} U={U:6d}: gam_ctc_align_long {a:9.3f} ms, gaps {b:9.3f} ms ({b / a:.3f}x)", flush=True)
            del lp
        del eng
        torch.cuda.empty_cache()
    return rows


def skips_part(quick):
    rows = []
    for name in ("v2_ctc", "v3_e2e_ctc"):
        ck = gigaam.synthetic_checkpoint(name, seed=0, n_layers=1)
        eng = gigaam.load_model(name, fp16_encoder=False, device=dev, checkpoint=ck)._get_engine()
        V1 = eng.num_classes
        g = torch.Generator().manual_seed(V1)
        sizes = [(2000, 1024), (2000, 65536)] if quick else [(2000, u) for u in (1024, 4096, 16384, 32768, 65536)]
        for T, U in sizes + [(90000, 65536)]:
            lp = torch.randn(1, T, V1, generator=g).log_softmax(-1).to(dev)
            y = torch.randint(0, V1 - 1, (1, U), generator=g, dtype=torch.int32).to(dev)
            args = (torch.tensor([T]), y, torch.tensor([U]))
            for line in (500, 12):
                edges = torch.tensor(longform.line_edges([(a, min(a + line, U)) for a in range(0, U, line)], U), dtype=torch.uint8)
                gaps = (edges[None].to(dev), -0.6931472)
                reps, warm = (3, 1) if T > 2000 else (7, 2)
                gap_ms, skip_ms = [], []
                for _ in range(warm):
                    eng.ctc_align_long(lp, *args, gaps=gaps)
                    out = eng.ctc_align_long(lp, *args, gaps=gaps, skips=-0.6931472)
                for _ in range(reps):             # alternating, so that drift of the clocks hits both
                    gap_ms.append(median_ms(lambda: eng.ctc_align_long(lp, *args, gaps=gaps), warmup=0, reps=1))
                    skip_ms.append(median_ms(lambda: eng.ctc_align_long(lp, *args, gaps=gaps, skips=-0.6931472), warmup=0, reps=1))
                a, b = statistics.median(gap_ms), statistics.median(skip_ms)
                rows.append(dict(V1=V1, T=T, U=U, line=line, gaps_ms=round(a, 3), skips_ms=round(b, 3), ratio=round(b / a, 3),
                                 skipped=int(out[8][0])))
                print(f"V+1={V1:4d} T={T:6d} U={U:6d} lines of {line:3d}: gaps {a:9.3f} ms, skips {b:9.3f} ms ({b / a:.3f}x), "
                      f"{int(out[8][0])} lines skipped", flush=True)
            del lp
        del eng
        torch.cuda.empty_cache()
    return rows


def main():
    quick = "--quick" in sys.argv
    info = card()
    print(info, flush=True)
    if "--skips" in sys.argv:
        rec = dict(card=info, skips=skips_part(quick))
    elif "--gaps" in sys.argv:
        rec = dict(card=info, gaps=gaps_part(quick))
    else:
        rec = dict(card=info, kernel=kernel_part(quick), calls=[], gaps=gaps_part(quick))
        for name in ("v2_ctc", "v3_e2e_ctc"):
            for minutes in ((10,) if quick else (10, 60)):
                rec["calls"].append(call_part(name, minutes))
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
