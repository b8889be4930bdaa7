"""The arithmetic identity behind the DFMA descent of the exact sampler
(csrc/tree_dev.cuh, spec_round<R>): for finite x and finite left >= 0,

    fma(-1.0, left, x) == x - left      (one rounding, like __dsub_rn)
    fma(-0.0, left, x) == x             (bit for bit, including signed zeros)

IEEE-754 guarantees it; this checks it on the host FPU (gcc + libm's fma, which
is correctly rounded like the GPU's DFMA) over random and edge-case operands."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

SRC = r"""
#include <math.h>
#include <stdint.h>
#include <string.h>
static uint64_t bits(double v) { uint64_t b; memcpy(&b, &v, 8); return b; }
long check(const double *x, const double *left, long n) {
    long bad = 0;
    for (long i = 0; i < n; i++) {
        volatile double a = x[i], b = left[i];
        double sub = a - b;
        if (bits(fma(-1.0, b, a)) != bits(sub)) bad++;
        if (bits(fma(-0.0, b, a)) != bits(a)) bad++;
    }
    return bad;
}
"""


def test_fma_forms_are_bit_identical_to_subtract_and_identity():
    with tempfile.TemporaryDirectory() as d:
        c, so = os.path.join(d, "f.c"), os.path.join(d, "f.so")
        open(c, "w").write(SRC)
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", c, "-o", so,
                               "-lm"])
        lib = ctypes.CDLL(so)
        lib.check.restype = ctypes.c_long
        lib.check.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_long]
        rng = np.random.RandomState(0)
        n = 400000
        # priorities-like magnitudes, plus wide exponent ranges, denormals and zeros
        x = np.concatenate([rng.rand(n) * 1e3, np.ldexp(rng.rand(n), rng.randint(-1070, 1000, n)),
                            [0.0, -0.0, 5e-324, 1.7976931348623157e308, 1.0, 1.0]])
        left = np.concatenate([rng.rand(n) * 1e3, np.ldexp(rng.rand(n), rng.randint(-1070, 1000, n)),
                               [0.0, 0.0, 5e-324, 1.0, 1.0 - 2 ** -53, 1e-300]])
        x = np.ascontiguousarray(x, dtype=np.float64)
        left = np.ascontiguousarray(np.abs(left), dtype=np.float64)
        assert lib.check(x.ctypes.data, left.ctypes.data, len(x)) == 0
