"""PWPP_ORDER_REFERENCE_EXACT on the SIMT twin (the kernels themselves, run on the CPU; tests/simt/simt_order_exact.cpp: the twin's
launch sequence with the fix-up behind k_order when the option order is 2): the index LISTS equal those of the unmodified
reference build (oracle/_ref/libpwref.so, std::sort as built by libstdc++) element for element, ties in z included. A frame whose
label SETS differ from the reference's (an fp32-vs-double flip, DESIGN.md section 3) cannot have equal lists and is skipped; all
but two frames of every group must be compared. The same on the GPU: tests/test_gpu_order_exact.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_py as O
from helpers import CheckedReference, SimtTwin
from param_sets import PARAM_SETS
from pwpp_ctypes import PwppParams, default_params

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_order_exact.so")


def build_lib():
    """tests/simt/simt_order_exact.cpp with the twin's compile line (tests/conftest.py: build_simt)."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_order_exact.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_order_exact.cpp")])
    return LIB


class ExactTwin(SimtTwin):
    """helpers.SimtTwin on libpwpp_simt_order_exact.so, estimating through simt_estimate_exact_multi."""

    def __init__(self, params=None, num_streams=1, **options):
        lib = C.CDLL(build_lib())
        self._bind(lib, "simt_")
        lib.simt_create.argtypes = [C.POINTER(PwppParams), C.c_int]; lib.simt_create.restype = C.c_void_p
        lib.simt_select.argtypes = [C.c_void_p, C.c_int]
        lib.simt_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        lib.simt_estimate_exact_multi.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
        lib.simt_order_exact_counts.argtypes = [C.c_void_p]
        self._lib = lib
        self.params = params if params is not None else default_params()
        self._h = lib.simt_create(C.byref(self.params), num_streams)
        self._ns = [0] * num_streams
        for k, v in options.items():
            assert lib.simt_set_option(self._h, k.encode(), int(v)) == 0, k

    def estimate(self, pts):
        self.estimate_multi([pts])

    def estimate_multi(self, frames):
        frames = [np.ascontiguousarray(a, dtype=np.float32) for a in frames]
        ptrs = (C.c_void_p * len(frames))(*[a.ctypes.data for a in frames])
        ns = (C.c_int64 * len(frames))(*[a.shape[0] for a in frames])
        self._lib.simt_estimate_exact_multi(self._h, len(frames), ptrs, ns, frames[0].shape[1])
        self._ns[:len(frames)] = [a.shape[0] for a in frames]
        self.select(0)

    def counts(self):
        """The fix-up's counters of the process: patches simulated, heap fall-backs, NaN bins."""
        out = np.zeros(3, np.uint64)
        self._lib.simt_order_exact_counts(out.ctypes.data)
        return out


pytestmark = pytest.mark.skipif(not O.have_reference_build(), reason="needs the reference build (oracle/_ref/libpwref.so)")


def wall_frame():
    """A wall inside a zone-0 bin: R-VPF removes points in several iterations (the case of test_gpu_reference.py)."""
    rng = np.random.default_rng(11)
    return np.r_[np.c_[4 + rng.random(6000) * 0.05, rng.random(6000) * 0.6, -1.7 + rng.random(6000) * 2.0, rng.random(6000)],
                 np.c_[3 + rng.random(6000) * 4, rng.random(6000) * 0.6, -1.7 + rng.normal(0, 0.02, 6000), rng.random(6000)]].astype(np.float32)


def compare(ref, tw, what):
    """1 when the lists were compared (and are equal), 0 when the label sets differ."""
    g_r, n_r = ref.getGroundIndices(), ref.getNongroundIndices()
    g_t, n_t = tw.getGroundIndices(), tw.getNongroundIndices()
    if not (np.array_equal(np.sort(g_r), np.sort(g_t)) and np.array_equal(np.sort(n_r), np.sort(n_t))):
        return 0
    for name, a, b in (("ground", g_r, g_t), ("non-ground", n_r, n_t)):
        assert np.array_equal(a, b), f"{what}: {name} list differs (first at {np.nonzero(a != b)[0][:3]})"
    return 1


@pytest.mark.parametrize("patch", [0, 1])
def test_fixtures_fresh_and_as_one_sequence(kitti, patch):
    compared = 0
    for f, a in enumerate(kitti):
        ref, tw = CheckedReference(stable_sort=False), ExactTwin(order=2, patch=patch)
        ref.estimate(a); tw.estimate(a)
        compared += compare(ref, tw, f"fixture {f} fresh")
    assert compared >= len(kitti) - 2
    ref, tw, compared = CheckedReference(stable_sort=False), ExactTwin(order=2, patch=patch), 0
    for f, a in enumerate(kitti):
        ref.estimate(a); tw.estimate(a)
        compared += compare(ref, tw, f"fixture {f} in sequence")
    assert compared >= len(kitti) - 2


def test_ties_differ_from_the_stable_order(kitti):
    """The fixtures hold ties inside one part: the exact lists are not the stable-sort lists (what PWPP_ORDER_REFERENCE gives)."""
    tw_exact, tw_stable = ExactTwin(order=2), SimtTwin(order=1)
    tw_exact.estimate(kitti[0]); tw_stable.estimate(kitti[0])
    assert not np.array_equal(tw_exact.getGroundIndices(), tw_stable.getGroundIndices())
    assert np.array_equal(np.sort(tw_exact.getGroundIndices()), np.sort(tw_stable.getGroundIndices()))


def test_second_parameter_set_synthetic_and_wall():
    import conftest
    import synth
    mk, cols = PARAM_SETS["no_rvpf_tgr"]
    frames = [(mk(), np.ascontiguousarray(conftest.load_kitti(f)[:, :cols])) for f in (1, 4)]
    for s in range(3):
        b = synth.make_frame(20260922, s).numpy()
        if s == 2:
            b[:, 2] = np.round(b[:, 2] / 0.01) * 0.01   # centimetre-quantised z: thousands of exact ties per bin
        frames.append((None, b))
    frames.append((None, wall_frame()))
    compared = 0
    for k, (prm, a) in enumerate(frames):
        for patch in (0, 1):
            ref, tw = CheckedReference(prm, stable_sort=False), ExactTwin(prm, order=2, patch=patch)
            ref.estimate(a); tw.estimate(a)
            compared += compare(ref, tw, f"frame {k} patch={patch}")
    assert compared >= 2 * len(frames) - 2


def test_sort_kernels_at_their_size_limits():
    """One flat patch per frame at the limits of the sort and fix-up kernels (the sizes of test_order.py), all frames in one call."""
    rng = np.random.default_rng(5)
    sizes = [10, 15, 16, 17, 31, 33, 63, 64, 65, 127, 129, 255, 256, 257, 511, 512, 513, 1023, 1025, 2047, 2048, 2049, 4095, 4096, 4097, 8191, 8192]
    frames = [np.c_[5 + rng.random(n) * 0.5, rng.random(n) * 0.5, -1.7 + np.round(rng.normal(0, 0.03, n), 3), rng.random(n)].astype(np.float32)
              for n in sizes]
    tw = ExactTwin(num_streams=len(frames), order=2)
    before = tw.counts()
    tw.estimate_multi(frames)
    compared = 0
    for f, (n, a) in enumerate(zip(sizes, frames)):
        ref = CheckedReference(stable_sort=False)
        ref.estimate(a)
        tw.select(f)
        compared += compare(ref, tw, f"size {n}")
    assert compared >= len(frames) - 2
    assert tw.counts()[0] > before[0]   # millimetre-rounded z: ties, so the simulation ran
