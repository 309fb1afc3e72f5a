"""Text vector files (-binary 0) for the text-reader tests (tests/test_text_vectors.py, tests/test_gpu_text_vectors.py):
tokens in the "%lf" rendering and exact decimal expansions of float midpoints, glibc strtof as the reference value of
a token, and the text twin of a word2vec-binary file."""
import ctypes as C
import os

import numpy as np

_libc = C.CDLL("libc.so.6")
_libc.strtof.restype = C.c_float
_libc.strtof.argtypes = [C.c_char_p, C.c_void_p]


def strtof_bits(tokens):
    """uint32 bits of glibc strtof of every token (str or bytes)."""
    return np.array([np.float32(_libc.strtof(t if isinstance(t, bytes) else t.encode(), None)).view(np.uint32)
                     for t in tokens], np.uint32)


def strtof_fast(tokens):
    """strtof_bits for many tokens: numpy's correctly rounded decimal-to-double conversion, then to float32.  Rounding
    twice gives strtof's float unless the double lands exactly on a midpoint between two floats (every binary32
    midpoint is a double, and rounding is monotone); those tokens, and NaNs, go to strtof itself."""
    a = np.asarray(tokens, dtype="S")
    d = np.char.lower(a)
    nan = np.char.find(d, b"nan") >= 0
    x = np.where(nan, b"0", a).astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        f = x.astype(np.float32)
        g = np.nextafter(f, np.where(x > f, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
        mid = (f.astype(np.float64) + g.astype(np.float64)) * 0.5
    out = f.view(np.uint32).copy()
    slow = np.nonzero(nan | ((x != f) & (x == mid)))[0]
    out[slow] = strtof_bits([bytes(a[i]) for i in slow])
    return out


def lf(x):
    """C's "%lf" of float32 x (the reference's fprintf(fo, "%lf ", ...)): Python's %f rounds the same way; a NaN
    keeps its sign as glibc prints it."""
    x = float(x)
    if x != x:
        return "-nan" if np.signbit(x) else "nan"
    return "%f" % x


def midpoint(b):
    """(digits, e): the midpoint between the floats with bits b and b + 1 is int(digits) x 10^e exactly."""
    be, frac = b >> 23, b & 0x7FFFFF
    m, k = (frac | 0x800000, be - 150) if be else (frac, -149)
    M, K = 2 * m + 1, k - 1
    return (str(M << K), 0) if K >= 0 else (str(M * 5 ** (-K)), K)


def plain(digits, e):
    """int(digits) x 10^e written without an exponent."""
    if e >= 0:
        return digits + "0" * e
    digits = digits.rjust(1 - e, "0")
    return digits[:e] + "." + digits[e:]


def midpoint_tokens(bits_list):
    """Per midpoint: its exact expansion, the same +-1 in the last digit, and truncated to 17, 19, 20 and 40
    significant digits."""
    out = []
    for b in bits_list:
        d, e = midpoint(int(b))
        out += [plain(d, e), plain(str(int(d) + 1), e), plain(str(int(d) - 1), e)]
        for n in (17, 19, 20, 40):
            if len(d) > n:
                out.append("%se%d" % (d[:n], e + len(d) - n))
    return out


def write_text(path, names, vec):
    """The reference's -binary 0 file: "V D\\n", then per word "<word> " + "%lf " per value + "\\n"."""
    with open(path, "w", encoding="latin1") as f:
        f.write("%d %d\n" % vec.shape)
        fmt = "%f " * vec.shape[1]
        for w, row in zip(names, vec):
            vals = fmt % tuple(row.tolist()) if np.isfinite(row).all() else "".join(lf(x) + " " for x in row)
            f.write(w + " " + vals + "\n")


def read_tokens(path):
    """(names, rows of tokens) of a text vector file, split on the host."""
    with open(path, "rb") as f:
        f.readline()
        names, rows = [], []
        for line in f:
            name, _, rest = line.partition(b" ")
            names.append(name.decode("latin1"))
            rows.append(rest.split())
    return names, rows


def strtof_table(path):
    """(names, V x D float32): strtof of every token of a text vector file."""
    names, rows = read_tokens(path)
    flat = strtof_fast([t for r in rows for t in r])
    return names, flat.view(np.float32).reshape(len(rows), -1)


def twin(vf, d):
    """The text twin of word2vec-binary file vf: (text file, binary file holding the strtof values of its tokens)."""
    from tests import packed_cases as pc
    from tests import analogy_cases as ac
    names, vec = pc.read_vectors(vf)
    tf = os.path.join(d, "vec.txt")
    write_text(tf, names, vec)
    _, val = strtof_table(tf)
    bf = os.path.join(d, "vec_strtof.bin")
    ac.write_vectors(bf, names, val)
    return tf, bf
