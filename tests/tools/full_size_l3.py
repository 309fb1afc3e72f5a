"""Epoch losses at the benchmarked shape (V ~ 300k-word Zipf vocabulary, D=800, window 10, negative 24, bitlevel 1) as a
function of the shard count, GPU vs the unmodified reference with as many pthreads (test infrastructure; the numbers
behind the bars of tests/test_gpu_parity.py::test_full_size_shape_loss_tracks_the_reference):
    python tests/tools/full_size_l3.py [tokens] [shard counts ...]"""
import os, sys, tempfile, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import bench
import word2bits_b200 as w2b
from oracle import pyoracle as po

tokens = int(sys.argv[1]) if len(sys.argv) > 1 else 3_000_000
shards = [int(x) for x in sys.argv[2:]] or [16, 132, 1584]
cdf, _ = bench.zipf_cdf(400000)
ids = bench.synth_ids(tokens, 99, cdf)
path = bench._write_text(ids, os.path.join(tempfile.gettempdir(), "l3_"))
D, W, neg, b, iters = 800, 10, 24, 1, 2
print("host cores:", len(os.sched_getaffinity(0)))
try:
    c = w2b.Corpus(path, 1)
    for S in shards:
        ref = po.Ref("o3")
        ref.configure(path, D, W, neg, b, threads=S, iters=iters, min_count=1)
        ref.learn_vocab(); ref.init_net(); ref.init_unigram()
        t0 = time.time()
        lr = [ref.train_epoch() for _ in range(iters)]
        tr = time.time() - t0
        for prefetch in (0, 1):
            t = w2b.Trainer(c, size=D, window=W, negative=neg, bitlevel=b, threads=S, iter=iters, prefetch=prefetch)
            lg = [t.train_epoch()[0] for _ in range(iters)]
            t.close()
            print("S=%5d prefetch=%d: GPU %s  reference(%d threads, %.0fs) %s  rel gap %s" % (
                S, prefetch, ["%.0f" % x for x in lg], S, tr, ["%.0f" % x for x in lr],
                ["%.4f" % (abs(a - r) / abs(r)) for a, r in zip(lg, lr)]), flush=True)
finally:
    os.unlink(path)
