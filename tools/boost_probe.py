"""Cost of phrase boosting in the RNN-T greedy decoder (gam_rnnt_greedy_boost against gam_rnnt_greedy_resume), with CUDA
events around each call.

    python tools/boost_probe.py [--reps N]

Synthetic v2_rnnt (V1 = 34, charwise: phrases anchored at the space token) and v3_e2e_rnnt (V1 = 1025) heads, at the
per-GPU decoding shapes of BASELINE configs 3 (32 utterances x 15 s) and 4 (256 x 10 s over 8 GPUs: 32 x 10 s per GPU),
scores off.  The encoder output is the (1-layer synthetic) encoder's on seeded synthetic audio.  Graphs: every bonus 0 (one state), 100 and 1 000 random
phrases of 2-8 tokens at weight 1.0.  The unboosted and boosted calls alternate, so both see the same clocks; reported:
milliseconds per call (median), the boosted / unboosted ratio, the graph's states and its table memory (S x V1 x 8 bytes),
and how many tokens the boosted decode emitted next to the unboosted one.  The card's name and power limit are read in the
same run; the last line is one JSON record of everything printed."""
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import gigaam_b200 as gigaam  # noqa: E402
from gigaam_b200.decoding import _as_btd, boost_graph  # noqa: E402

dev = torch.device("cuda", 0)
SHAPES = (("config 3: 32 x 15 s", 32, 15.0), ("config 4 per GPU: 32 x 10 s", 32, 10.0))


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(dev)


def main():
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 30
    print(card(), flush=True)
    rows = []
    for name in ("v2_rnnt", "v3_e2e_rnnt"):
        model = gigaam.load_model(name, fp16_encoder=True, device=dev, checkpoint=gigaam.synthetic_checkpoint(name, seed=0, n_layers=1))
        eng = model._get_engine()
        tok = model.decoding.tokenizer
        V1 = eng.num_classes
        anchor = tok.vocab.index(" ") if tok.charwise and " " in tok.vocab else None
        words = [i for i in range(V1 - 1) if i != anchor]
        rng = np.random.default_rng(0)
        graphs = {"zero bonuses": (torch.zeros((1, V1), dtype=torch.int32), torch.zeros((1, V1)))}
        for n in (100, 1000):
            ph = [rng.choice(words, size=rng.integers(2, 9)).tolist() for _ in range(n)]
            graphs[f"{n} phrases"] = boost_graph(ph, 1.0, anchor, V1, V1 - 1)
        for shape, B, seconds in SHAPES:
            wav, lengths = gigaam.synthetic_audio(B, seconds, seed=1)
            with torch.inference_mode():
                encoded, _ = model.forward(wav.to(dev).to(model._dtype), lengths.to(dev))
            enc = _as_btd(encoded.float()).clone()
            T = enc.shape[1]
            i32 = dict(dtype=torch.int32, device=dev)
            lo, hi, fb = torch.zeros(B, **i32), torch.full((B,), T, **i32), torch.zeros(B, **i32)
            fresh = eng.decode_state(B)
            for gname, (nxt, bonus) in graphs.items():
                tables = (nxt.to(dev), bonus.to(dev))
                times = {False: [], True: []}
                emitted = {}
                for r in range(reps + 3):
                    for boosted in (False, True):
                        state = fresh.clone()
                        out = eng.decode_buffers(B, eng.hyp_width(T))
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record()
                        eng.greedy_resume(enc, lo, hi, fb, state, out, False, tables if boosted else None)
                        b.record()
                        torch.cuda.synchronize()
                        if r >= 3:                 # the first rounds warm modules, launch attributes and workspaces
                            times[boosted].append(a.elapsed_time(b))
                        emitted[boosted] = int(out.counts.sum())
                base, boost = statistics.median(times[False]), statistics.median(times[True])
                row = dict(model=name, V1=V1, shape=shape, graph=gname, states=int(nxt.shape[0]),
                           table_MiB=round(nxt.shape[0] * V1 * 8 / 2**20, 3), unboosted_ms=round(base, 3),
                           boosted_ms=round(boost, 3), ratio=round(boost / base, 3), tokens_unboosted=emitted[False],
                           tokens_boosted=emitted[True])
                print(row, flush=True)
                rows.append(row)
    print(json.dumps(dict(card=card(), reps=reps, rows=rows)))


if __name__ == "__main__":
    main()
