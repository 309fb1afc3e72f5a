"""Float64 rounding-error bounds and the kernels' scalar functions, shared by the per-position test
(test_gpu_position_f64.py) and the per-step trajectory test (test_trajectory_f64.py).

With u = 2^-24 and gamma_n = n*u / (1 - n*u), a float32 sum of n terms in any order is off by at most gamma_n times
the sum of the terms' absolute values; a term that passes through at most h roundings (a summation tree of depth h)
is off by gamma_h."""
import numpy as np

from oracle import pyoracle as po
from tests.util import bits

U = 2.0 ** -24
TINY = 2.0 ** -126  # atomic and bulk-reduce adds flush denormal inputs and results (DESIGN §2, deviation 3)
SUB = 2.0 ** -149   # absolute rounding error of an operation whose result is denormal


def gamma(n):
    n = np.asarray(n, np.float64)
    return n * U / (1 - n * U)


def grad_scalar(f, label, alpha, exptab, slot_shift=0):
    """g (:473-475) as the kernels compute it in float32 from the f they used; slot_shift reads a neighbouring slot."""
    f, alpha = np.float32(f), np.float32(alpha)
    if f > 6:
        return np.float32(np.float32(label - 1) * alpha)
    if f < -6:
        return np.float32(np.float32(label) * alpha)
    idx = int(np.float32(np.float32(f + np.float32(6)) * np.float32(83)))  # int() truncates toward zero
    return np.float32(np.float32(np.float32(label) - exptab[idx + slot_shift]) * alpha)


def quantizer(b, minus_zero_takes_sign):
    """The kernel's quantize: the oracle's, except that -0.0 takes the negative level where the kernel copies the
    sign bit (the warp kernel's compile-time bit levels 1 and 2, DESIGN §1 a1)."""
    def q(x):
        out = po.quantize(x, b)
        if minus_zero_takes_sign:
            nz = bits(x) == 0x80000000
            out[nz] = -out[nz]
        return out
    return q


def special_values(b):
    """|x| = 0.5 and its neighbours, -0.0, denormals, the smallest normal, and quantization thresholds of bit level b."""
    half = np.float32(0.5)
    vals = [half, np.nextafter(half, np.float32(0)), np.nextafter(half, np.float32(1)), np.float32(0.0),
            np.float32(1e-40), np.float32(2.0 ** -126), np.float32(2.0 ** -127), np.float32(0.25), np.float32(0.75)]
    if b >= 4:
        seg = 2 ** (b - 1)
        for k in (0, 1, seg // 2 - 1, seg - 1):
            t = np.float32((k + 0.5) / seg)
            vals += [t, np.nextafter(t, np.float32(0)), np.nextafter(t, np.float32(1))]
    vals = np.array(vals, np.float32)
    return np.concatenate([vals, -vals])  # -0.0 among them
