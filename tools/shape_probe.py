"""Throughput of the production kernel at arbitrary row widths / bit levels / -reg (not the bench):
    python tools/shape_probe.py 150:1:0 1200:2:0 800:1:0.001      # D:bitlevel:reg ...
Prints positions/s and algorithmic GB/s against the HBM peak (MEASURED_PEAKS.json, else the H100 data sheet)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import word2bits_b200 as w2b
from tools.quick_perf import synth
from tools.warp_sweep import peak

specs = sys.argv[1:] or ["150:1:0", "250:1:0", "300:1:0", "1200:1:0", "1536:0:0", "2048:1:0", "800:1:0.001", "200:1:0.001"]
N = 20_000_000
ids, cn = synth(400000, N)
for spec in specs:
    D, b, reg = spec.split(":")
    D, b, reg = int(D), int(b), float(reg)
    t = w2b.Trainer(None, vocab_size=400001, size=D, window=10 if D >= 400 else 8, negative=24, bitlevel=b, iter=1,
                    threads=None, reg=reg)
    S = t.threads
    t.set_vocab_counts(cn, N)
    t.set_corpus(ids, np.arange(S, dtype=np.int64) * (N // S), np.full(S, -1, np.int32), True)
    t.train_step(500)
    st = t.train_step(2000)
    gbs = (st["context_rows"] + st["target_rows"]) * D * 8 / 1e9 / (st["kernel_ms"] / 1e3)
    print("D=%d b=%d reg=%g shards=%d: %.1f M positions/s, %.0f GB/s algorithmic (%.2f of %.0f)" % (
        D, b, reg, S, st["positions"] / st["kernel_ms"] / 1e3, gbs, gbs / peak(), peak()), flush=True)
    t.close()
