"""Inputs of the packed-evaluator tests (tests/test_oracle_packed.py, tests/test_gpu_evaluator_packed.py) and of
tests/golden/make_reference_packed.py.  A case is one of tests/analogy_cases.py's generators run on 1-bit or 2-bit
levels; its vectors are then written twice, as the word2vec-binary file the reference reads and as the packed file
(the format of w2b_write_packed) the bit-domain evaluator reads.
build(name, directory) -> (packed file, unpacked file, questions file, bitlevel, threshold)."""
import json
import os

import numpy as np

from oracle import pyoracle as po
from tests import analogy_cases as ac


def reference_answers():
    """{case: report and digest of the answers} of the reference compute_accuracy on the unpacked files
    (tests/golden/make_reference_packed.py)."""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_packed.json")) as f:
        return json.load(f)


def level_codes(vec, bits):
    """Per value the packed code: bit 0 = negative, bit 1 (2-bit files) = the larger magnitude."""
    vec = np.asarray(vec, np.float32)
    return (vec < 0).astype(np.uint8) | ((np.abs(vec) > 0.5).astype(np.uint8) << 1 if bits == 2 else 0)


def pack_rows(vec, bits):
    """Levels (V x D float32) -> V x ceil(D*bits/8) uint8: value j in bits [j*bits, (j+1)*bits) of its row."""
    code = level_codes(vec, bits)
    planes = [(code >> k) & 1 for k in range(bits)]
    return np.packbits(np.stack(planes, axis=2).reshape(len(code), -1), axis=1, bitorder="little")


def unpack_rows(rows, D, bits):
    """The float32 levels w2b_read_packed restores."""
    b = np.unpackbits(rows, axis=1, bitorder="little")[:, : D * bits].reshape(len(rows), D, bits)
    mag = np.float32(1.0) / np.float32(3.0) if bits == 1 else np.where(b[:, :, 1] == 1, np.float32(0.75), np.float32(0.25))
    return np.where(b[:, :, 0] == 1, -mag, mag).astype(np.float32)


def write_packed(path, names, rows, D, bits):
    with open(path, "wb") as f:
        f.write(b"%d %d %d\n" % (len(names), D, bits))
        for w, r in zip(names, rows):
            f.write(w.encode() + b" " + r.tobytes() + b"\n")


def read_vectors(vf):
    """(names as written, V x D float32) of a word2vec-binary file written by analogy_cases.write_vectors."""
    with open(vf, "rb") as f:
        V, D = (int(x) for x in f.readline().split())
        names, vec = [], np.empty((V, D), np.float32)
        for k in range(V):
            w = b""
            while (ch := f.read(1)) not in (b"", b" "):
                w += ch
            names.append(w.decode())
            vec[k] = np.frombuffer(f.read(4 * D), np.float32)
            f.read(1)
    return names, vec


def planted(d, bits, **kw):
    return ac.planted(d, bits=bits, quantized_input=True, **kw)


def all_equal(d, bits, D=32, V=1500, nq=200, seed=3):
    """Every row equal: every score ties, the candidate list overflows and the fp32 SIMT scorer takes over."""
    vf, qf, _, th = ac.all_equal(d, D=D, V=V, nq=nq, seed=seed)
    names, vec = read_vectors(vf)
    ac.write_vectors(vf, names, po.quantize(vec, bits))
    return vf, qf, bits, th


CASES = {}
for _D in (1, 3, 7, 8, 31, 32, 33, 63, 64, 65, 127, 128, 130, 200, 800, 1200, 2000):
    for _b in (1, 2):
        CASES["D%d_b%d" % (_D, _b)] = (planted, dict(D=_D, V=1001, nq=300, bits=_b, seed=_D))
for _V in (4, 5, 255, 256, 257, 5000):
    for _b in (1, 2):
        CASES["V%d_b%d" % (_V, _b)] = (planted, dict(D=200, V=_V, nq=200, bits=_b, seed=_V))
CASES["V40000_chunks_b2"] = (planted, dict(D=64, V=40000, nq=300, bits=2, seed=9))  # several chunks of the Gram matrix
CASES["V40000_chunks_b1"] = (planted, dict(D=96, V=40000, nq=300, bits=1, seed=10))
CASES["V2000_threshold700_b2"] = (planted, dict(D=100, V=2000, nq=400, bits=2, threshold=700, seed=7))
for _n in (1, 63, 64, 65, 3000):
    CASES["nq%d_b2" % _n] = (planted, dict(D=72, V=1001, nq=_n, bits=2, seed=100 + _n + (_n == 1)))
for _b in (1, 2):  # duplicate names, out-of-vocabulary words, all-repeated query words
    CASES["edges_b%d" % _b] = (planted, dict(D=40, V=600, nq=300, bits=_b, dup_names=30, oddities=True, seed=400 + _b))
CASES["all_equal_b1"] = (all_equal, dict(bits=1))
CASES["ties_D8_b1"] = (planted, dict(D=8, V=1001, nq=300, bits=1, seed=8))


def build(name, d):
    fn, kw = CASES[name]
    os.makedirs(d, exist_ok=True)
    vf, qf, bits, th = fn(d, **kw)
    names, vec = read_vectors(vf)
    pf = os.path.join(d, "vec.packed")
    rows = pack_rows(vec, bits)
    assert np.array_equal(unpack_rows(rows, vec.shape[1], bits).view(np.uint32), vec.view(np.uint32)), "not on the levels"
    write_packed(pf, names, rows, vec.shape[1], bits)
    return pf, vf, qf, bits, th


# ---- the Gram kernel's formulas, restated on numpy bit planes (uint32 words, padding bits 0)
def planes(vec, bits):
    """(sign plane, magnitude plane) of levels vec: V x ceil(D/32) uint32 each, value j in bit j % 32 of word j // 32."""
    def plane(bit):
        p = np.packbits(bit.astype(np.uint8), axis=1, bitorder="little")
        p = np.pad(p, ((0, 0), (0, -p.shape[1] % 4)))
        return p.view(np.uint32)
    code = level_codes(vec, bits)
    return plane(code & 1), plane(code >> 1)


def popc(x):
    return np.unpackbits(np.ascontiguousarray(x).view(np.uint8), axis=-1).reshape(*x.shape[:-1], -1).sum(-1).astype(np.int64)


def gram_from_planes(nw, hw, nc, hc, D, bits):
    """Integer dot products of rows w against rows c from their planes, in level units."""
    x = nw[:, None, :] ^ nc[None, :, :]
    if bits == 1:
        return D - 2 * popc(x)
    a, b = hw[:, None, :], hc[None, :, :]
    A = D + 2 * popc(a) + 2 * popc(b) + 4 * popc(a & b)
    B = popc(x) + 2 * popc(x & a) + 2 * popc(x & b) + 4 * popc(x & a & b)
    return A - 2 * B


def integer_levels(vec, bits):
    """Levels in units of the smallest: +-1 (1 bit), +-1 / +-3 (2 bits)."""
    return np.rint(np.asarray(vec, np.float64) * (3 if bits == 1 else 4)).astype(np.int64)
