"""Nearest-neighbour queries for the top-k tests (tests/test_oracle_topk.py, tests/test_gpu_topk.py), over the vector
files tests/analogy_cases.py and tests/packed_cases.py build, plus one 40 000-word fp32 file whose 3000 queries
cross several vocabulary chunks.  build(name, directory) -> (vectors file the GPU reads (packed or not), unpacked
file, words file, words, bitlevel, threshold)."""
import os

import numpy as np

from tests import analogy_cases as ac
from tests import packed_cases as pc

# name: (source, source case, how many words to query (None: every word of the file), seed)
CASES = {
    "V4_b1": ("analogy", "V4_b1", None, 0),
    "V5_b1": ("analogy", "V5_b1", None, 1),
    "V255_b1": ("analogy", "V255_b1", None, 2),
    "edges_b0": ("analogy", "edges_b0", None, 3),          # zero rows, duplicate names
    "edges_b1": ("analogy", "edges_b1", None, 4),
    "V2000_threshold700_b1": ("analogy", "V2000_threshold700_b1", 900, 5),  # words beyond the threshold
    "all_equal": ("analogy", "all_equal", 300, 6),
    "small_positive": ("analogy", "small_positive", None, 7),
    "D800_b0": ("analogy", "D800_b0", 300, 8),
    "packed_ties_D8_b1": ("packed", "ties_D8_b1", None, 9),
    "packed_edges_b2": ("packed", "edges_b2", None, 10),
    "packed_D130_b1": ("packed", "D130_b1", 300, 11),
    "packed_all_equal_b1": ("packed", "all_equal_b1", 300, 12),
    "packed_V40000_chunks_b1": ("packed", "V40000_chunks_b1", 3000, 13),
    "V40000_chunks_b0": ("big", None, 3000, 14),
}


def build(name, d):
    src, case, n, seed = CASES[name]
    os.makedirs(d, exist_ok=True)
    if src == "analogy":
        vf, _, b, th = ac.build(case, d)
        gf = vf
    elif src == "packed":
        gf, vf, _, b, th = pc.build(case, d)
    else:
        vf, _, b, th = ac.planted(d, D=48, V=40000, nq=1, seed=seed)
        gf = vf
    names, _ = pc.read_vectors(vf)
    rng = np.random.default_rng(seed)
    words = list(names) if n is None else [names[i] for i in rng.integers(0, len(names), n)]
    # a word not in the vocabulary, repeated query words, another case
    words += ["missingword", words[0], words[-1].lower(), words[0].upper()]
    wf = os.path.join(d, "words.txt")
    with open(wf, "w") as f:
        f.write("\n".join(words) + "\n")
    return gf, vf, wf, words, b, th
