"""Inputs of the analogy-evaluator tests (tests/test_oracle_analogy.py, tests/test_gpu_evaluator.py) and of
tests/golden/make_reference_outputs.py, which stores what src/compute-accuracy.c answers on each of them.
Every case is generated from a seed: build(name, directory) -> (vectors file, questions file, bitlevel, threshold)."""
import os

import numpy as np

from oracle import pyoracle as po


def write_vectors(path, names, vec):
    with open(path, "wb") as f:
        f.write(b"%d %d\n" % (len(names), vec.shape[1]))
        for w, row in zip(names, vec):
            f.write(w.encode() + b" " + np.ascontiguousarray(row, np.float32).tobytes() + b"\n")


def write_questions(path, questions, per_section=120):
    """questions: list of 4-word lists; a new section every per_section questions."""
    with open(path, "w") as f:
        for i, q in enumerate(questions):
            if i % per_section == 0:
                f.write(": section-%d\n" % (i // per_section))
            f.write(" ".join(q) + "\n")


def read_questions(path):
    """The question lines of a file written by write_questions, in file order."""
    return [l.split() for l in open(path) if l.strip() and not l.startswith(":")]


def planted(d, D, V, nq, bits=0, quantized_input=False, threshold=0, seed=0, zero_rows=0, dup_names=0,
            oddities=False):
    """Planted a:b offsets (like questions-words.txt on trained vectors) plus noise words.  A fifth of the
    questions take four random vocabulary words (so query words repeat and the fourth word can be a query word),
    3 % have an out-of-vocabulary word; case is mixed.  quantized_input: the file already holds the levels of
    `bits` (what `word2bits -bitlevel b` writes)."""
    rng = np.random.default_rng(seed)
    pairs = max(1, min(300, (V - 1) // 3))
    off = rng.normal(size=D).astype(np.float32) * 1.5
    a = rng.normal(size=(pairs, D)).astype(np.float32)
    b = a + off + 1.1 * rng.normal(size=(pairs, D)).astype(np.float32)
    noise = rng.normal(size=(max(0, V - 1 - 2 * pairs), D)).astype(np.float32)
    vec = np.concatenate([np.zeros((1, D), np.float32) + 0.01, a, b, noise])[:V]
    names = (["</s>"] + ["Alpha%d" % i for i in range(pairs)] + ["beta%d" % i for i in range(pairs)] +
             ["noise%d" % i for i in range(len(noise))])[:V]
    if quantized_input:
        vec = po.quantize(vec * 0.3, bits)
    for r in rng.choice(np.arange(1, V), size=min(zero_rows, V - 1), replace=False):
        vec[r] = 0.0  # normalises to NaN: never an answer, and a question that uses it has none
    for r in rng.choice(np.arange(1 + 2 * pairs, V), size=min(dup_names, max(0, V - 1 - 2 * pairs)), replace=False):
        names[r] = names[rng.integers(1, r)]  # the first row of a name is the one questions refer to
    vocab_q = min(V, threshold) if threshold else V
    qs = []
    for _ in range(nq):
        if rng.random() < 0.8 and 2 * pairs + 1 <= vocab_q:
            i, j = rng.integers(0, pairs, 2)
            q = ["alpha%d" % i, "BETA%d" % i, "Alpha%d" % j, "beta%d" % j]
        else:
            q = [names[k] for k in rng.integers(0, vocab_q, 4)]
        if rng.random() < 0.03:
            q[rng.integers(0, 4)] = "missingword"
        qs.append(q)
    if oddities:  # a zero row as query word, all-repeated query words, fourth word = third word
        z = [k for k in range(V) if not np.any(vec[k])]
        if z:
            qs.append([names[1], names[2], names[z[0]], names[3]])
        qs += [[names[1]] * 4, [names[1], names[1], names[2], names[2]], [names[2], names[1], names[3], names[3]]]
    vf, qf = os.path.join(d, "vec.bin"), os.path.join(d, "questions.txt")
    write_vectors(vf, names, vec)
    write_questions(qf, qs)
    return vf, qf, bits, threshold


def all_equal(d, D=32, V=1500, nq=200, seed=3):
    """Every vector equal: every score ties, so the tensor-core filter's candidate list overflows (more than 1024
    per question) and the evaluator scores everything on the SIMT cores; the first non-query index wins."""
    rng = np.random.default_rng(seed)
    vec = np.tile(rng.normal(size=(1, D)).astype(np.float32), (V, 1))
    names = ["w%d" % i for i in range(V)]
    qs = [[names[k] for k in rng.integers(0, 8, 4)] for _ in range(nq)]
    vf, qf = os.path.join(d, "vec.bin"), os.path.join(d, "questions.txt")
    write_vectors(vf, names, vec)
    write_questions(qf, qs)
    return vf, qf, 0, 0


def tf32(x):
    """What a TF32 tensor-core operand keeps of float32 x: the low 13 mantissa bits dropped."""
    return (np.ascontiguousarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def small_positive_rows(D=32, seed=11, tries=200000):
    """(C, W) raw rows such that, after the reference's normalisation, the score of W against C is positive but
    below 2^-9 |C| (the tensor-core filter's error bound) while the TF32 score is negative."""
    rng = np.random.default_rng(seed)
    c = rng.normal(size=D).astype(np.float32)
    cn = po.analogy_normalize(c[None], 0)[0]
    cn64, ct = cn.astype(np.float64), tf32(cn).astype(np.float64)
    for _ in range(tries // 1000):
        r = rng.normal(size=(1000, D))
        r -= np.outer(r @ cn64, cn64)                     # orthogonal to C ...
        r += np.outer(rng.uniform(0, 2e-3, 1000), cn64)   # ... plus a little of C
        w = po.analogy_normalize(r.astype(np.float32), 0)
        exact = np.zeros(len(w), np.float32)
        for k in range(D):                                # the reference's unfused order
            exact = exact + cn[k] * w[:, k]
        approx = tf32(w).astype(np.float64) @ ct
        ok = np.nonzero((exact > 0) & (exact < 2.0 ** -9) & (approx < 0))[0]
        if len(ok):
            return c, r[ok[0]].astype(np.float32)
    raise AssertionError("no row found")


def small_positive(d, D=32, V=300, seed=11):
    """Question `a a c ?` (so vec = c) whose only positively scoring word w has an exact score in (0, eps) and a
    negative TF32 score: the reference answers w, a filter that keeps only TF32 scores > 0 answers nothing."""
    rng = np.random.default_rng(seed)
    c, w = small_positive_rows(D, seed)
    neg = -(c[None] * rng.uniform(0.5, 2.0, (V - 3, 1))).astype(np.float32) + 0.05 * rng.normal(size=(V - 3, D)).astype(np.float32)
    vec = np.concatenate([rng.normal(size=(1, D)).astype(np.float32), c[None], w[None], neg])
    names = ["a", "c", "w"] + ["n%d" % i for i in range(V - 3)]
    vf, qf = os.path.join(d, "vec.bin"), os.path.join(d, "questions.txt")
    write_vectors(vf, names, vec)
    write_questions(qf, [["a", "a", "c", "w"], ["A", "a", "C", "n0"]])
    return vf, qf, 0, 0


CASES = {}
for _D in (1, 3, 7, 8, 12, 31, 32, 33, 72, 130, 200, 800, 1200, 2000):
    for _b in (0, 1):
        CASES["D%d_b%d" % (_D, _b)] = (planted, dict(D=_D, V=1001, nq=300, bits=_b, seed=_D))
for _V in (4, 5, 255, 256, 257, 5000):
    CASES["V%d_b1" % _V] = (planted, dict(D=48, V=_V, nq=200, bits=1, seed=_V))
CASES["V2000_threshold700_b1"] = (planted, dict(D=48, V=2000, nq=400, bits=1, threshold=700, seed=7))
for _n in (1, 63, 64, 65, 127, 128, 129, 3000):
    CASES["nq%d_b1" % _n] = (planted, dict(D=48, V=1001, nq=_n, bits=1, seed=100 + _n + (_n == 1)))
for _b in (0, 1, 2, 3, 4, 8):
    CASES["bits%d_fp32" % _b] = (planted, dict(D=48, V=1001, nq=300, bits=_b, seed=200 + _b))
    CASES["bits%d_quantized" % _b] = (planted, dict(D=48, V=1001, nq=300, bits=_b, quantized_input=True,
                                                   seed=300 + _b))
for _b in (0, 1):
    CASES["edges_b%d" % _b] = (planted, dict(D=40, V=600, nq=300, bits=_b, zero_rows=20, dup_names=30,
                                             oddities=True, seed=400 + _b))
CASES["all_equal"] = (all_equal, {})
CASES["small_positive"] = (small_positive, {})


def build(name, d):
    fn, kw = CASES[name]
    os.makedirs(d, exist_ok=True)
    return fn(d, **kw)


def per_question_file(qf, answers, names, path):
    """Each question of qf scored on its own: one section per question the reference sees, its fourth word
    replaced by the chosen word's name (kept when there is no answer).  Returns {section: expected count}."""
    want, known = {}, set(names)
    with open(path, "w") as f:
        for k, (q, c) in enumerate(zip(read_questions(qf), answers)):
            if c < 0 and not all(w.upper() in known for w in q):
                continue  # skipped by the reference: no section
            f.write(": q%d\n%s %s %s %s\n" % (k, q[0], q[1], q[2], names[c] if c >= 0 else q[3]))
            want["q%d" % k] = 1 if c >= 0 else 0
    return want


def per_question_counts(report):
    """{section: correct count} from a report of per_question_file."""
    got, sec = {}, None
    for line in report.splitlines():
        if line.endswith(":") and not line.startswith("ACCURACY"):
            sec = line[:-1]
        elif line.startswith("ACCURACY TOP1:") and sec is not None:
            got[sec] = int(line.split("(")[1].split("/")[0])
    return got


def vocab_names(vf, threshold=0):
    """Upper-cased names of the vector file (what the reference compares questions with), file order."""
    with open(vf, "rb") as f:
        V, D = (int(x) for x in f.readline().split())
        if threshold and V > threshold:
            V = threshold
        names = []
        for _ in range(V):
            w = b""
            while True:
                ch = f.read(1)
                if ch in (b"", b" "):
                    break
                if ch != b"\n":
                    w += ch
            names.append(w.decode("latin1").upper())
            f.read(4 * D)
    return names
