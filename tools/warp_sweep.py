"""Throughput of the production (warp-per-shard) kernel on one GPU over the BASELINE shapes and its knobs (CUDA events,
inputs resident; not the bench):
    python tools/warp_sweep.py [--out gpurun_out/warp_sweep.md] [--shapes c2,c3,c4,d200,d100] [--configs ...]"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import word2bits_b200 as w2b
from tools.quick_perf import synth

SHAPES = {  # name: (D, negative, bitlevel, window)
    "c2": (800, 24, 1, 10), "c3": (400, 12, 2, 10), "c4": (400, 24, 0, 10), "d200": (200, 24, 1, 8), "d100": (100, 5, 1, 5),
}


def peak():
    import json
    try:
        return float(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 3350.0  # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/warp_sweep.md")
    ap.add_argument("--shapes", default="c2,c3,c4,d200,d100")
    ap.add_argument("--configs", default="0:0:0:1,0:1:0:1,0:0:3:1,0:0:0:2,1:0:0:1",
                    help="kernel:prefetch:slots:shard-multiple (kernel 0 = warp kernel, 1 = register kernel; slots 0 = planner)")
    ap.add_argument("--vocab", type=int, default=400000)
    ap.add_argument("--tokens", type=int, default=40_000_000)
    ap.add_argument("--words", type=int, default=2_000_000, help="words per step over all shards")
    ap.add_argument("--steps", type=int, default=3)
    a = ap.parse_args()
    ids, cn = synth(a.vocab, a.tokens)
    pk = peak()
    rows = ["| shape | kernel | prefetch | slots | shards | words/shard/step | positions/s | algorithmic GB/s | of %.0f GB/s | loss/position |" % pk,
            "|---|---|---|---|---|---|---|---|---|---|"]
    for name in a.shapes.split(","):
        D, neg, b, W = SHAPES[name]
        for cfg in a.configs.split(","):
            kernel, prefetch, slots, mult = [int(x) for x in cfg.split(":")]
            t = w2b.Trainer(None, vocab_size=a.vocab + 1, size=D, window=W, negative=neg, bitlevel=b, iter=1,
                            threads=None, kernel=kernel, prefetch=prefetch, slots=slots, init=False)
            S = t.threads * mult
            t.close()
            t = w2b.Trainer(None, vocab_size=a.vocab + 1, size=D, window=W, negative=neg, bitlevel=b, iter=1,
                            threads=S, kernel=kernel, prefetch=prefetch, slots=slots)
            t.set_vocab_counts(cn, int(a.tokens))
            t.set_corpus(ids, np.arange(S, dtype=np.int64) * (a.tokens // S), np.full(S, -1, np.int32), True)
            wps = max(1500, a.words // S)
            t.train_step(wps // 4)
            pos = rows_ = 0
            ms = loss = 0.0
            for _ in range(a.steps):
                st = t.train_step(wps)
                pos += st["positions"]; rows_ += st["context_rows"] + st["target_rows"]; ms += st["kernel_ms"]; loss += st["loss"]
            t.close()
            gbs = rows_ * D * 4 * 2 / 1e9 / (ms / 1e3)
            line = "| %s D=%d neg=%d b=%d | %d | %d | %s | %d | %d | %.2f M | %.0f | %.3f | %.4f |" % (
                name, D, neg, b, kernel, prefetch, slots or "plan", S, wps, pos / ms / 1e3, gbs, gbs / pk, loss / max(pos, 1))
            print(line, flush=True)
            rows.append(line)
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        f.write("# production (warp-per-shard) kernel, tools/warp_sweep.py (CUDA events; %d steps)\n\n" % a.steps)
        f.write("\n".join(rows) + "\n")


if __name__ == "__main__":
    main()
