"""float_ru (csrc/pwpp_math.cuh), compiled for the CPU, against the double compare it replaces in the fit kernels.

The seed, margin and inner-seed tests of the fit kernels compare a float z with a per-round double threshold t. They
evaluate z < float_ru(t) instead of (double) z < t. This checks, on thresholds at and next to float boundaries (subnormal,
zero, huge, infinite, NaN) and on every float next to them, that the two compares agree and that float_ru(t) is the
smallest float >= t."""
import ctypes as C
import os
import subprocess

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM = r"""
#include "pwpp_math.cuh"
extern "C" void float_ru_n(const double* t, long long n, float* out) { for (long long i = 0; i < n; ++i) out[i] = pwpp::float_ru(t[i]); }
"""


def _float_ru_lib(tmp_path):
    src = tmp_path / "float_ru.cpp"
    src.write_text(SHIM)
    so = tmp_path / "libfloat_ru.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared",
                           "-I" + os.path.join(REPO, "patchwork-plusplus_b200", "csrc"), str(src), "-o", str(so)])
    lib = C.CDLL(str(so))
    lib.float_ru_n.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p]
    return lib


def _thresholds():
    f = np.array([0.0, -0.0, 1.0, -1.0, 1.5, -1.7, 0.3, -0.3, 1.6 * 0.02, 80.0, -2.5e-3, 1e-40, -1e-40, 1e-45, -1e-45,
                  np.finfo(np.float32).tiny, np.finfo(np.float32).max, -np.finfo(np.float32).max], np.float32)
    rng = np.random.default_rng(7)
    f = np.concatenate([f, rng.normal(scale=3.0, size=2000).astype(np.float32)])
    up = np.nextafter(f, np.float32(np.inf)).astype(np.float64)
    dn = np.nextafter(f, np.float32(-np.inf)).astype(np.float64)
    fd = f.astype(np.float64)
    t = [fd, (fd + up) / 2, (fd + dn) / 2, fd + (up - fd) * 1e-6, fd - (fd - dn) * 1e-6, np.nextafter(fd, np.inf), np.nextafter(fd, -np.inf)]
    special = np.array([np.inf, -np.inf, np.nan, 1e300, -1e300, 5e-324, -5e-324, 3.5e38, -3.5e38,
                        float(np.finfo(np.float32).max) * (1 + 2.0 ** -25), -float(np.finfo(np.float32).max) * (1 + 2.0 ** -25)])
    return np.concatenate(t + [special])


def test_float_ru_is_exact_replacement_of_the_double_compare(tmp_path):
    lib = _float_ru_lib(tmp_path)
    t = np.ascontiguousarray(_thresholds())
    tf = np.empty(len(t), np.float32)
    lib.float_ru_n(t.ctypes.data, len(t), tf.ctypes.data)
    with np.errstate(invalid="ignore", over="ignore"):
        ok = ~np.isnan(t)
        assert np.isnan(tf[~ok]).all()
        # smallest float >= t
        assert (tf[ok].astype(np.float64) >= t[ok]).all()
        below = np.nextafter(tf[ok], np.float32(-np.inf)).astype(np.float64)
        assert ((below < t[ok]) | (tf[ok] == -np.inf)).all()
        # every float around the threshold, plus the specials, decides the same way in both compares
        zs = [tf, np.nextafter(tf, np.float32(np.inf)), np.nextafter(tf, np.float32(-np.inf)), t.astype(np.float32)]
        zs += [np.full(len(t), v, np.float32) for v in (np.inf, -np.inf, np.nan, 0.0, -0.0)]
        for z in zs:
            assert np.array_equal(z.astype(np.float64) < t, z < tf)
