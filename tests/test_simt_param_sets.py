"""Several parameter sets in one launch sequence, executed on the CPU by the SIMT stand-in (tests/simt/simt_param_sets.cpp, the twin
of tests/simt/simt_twin.cpp with the set tables of pwpp_create_sets): every kernel reads the record of its frame's set. Each
stream is compared with its own CANON64 oracle built with its set and fed the same frames in the same order, through both
front-end variants and with a stream table that names streams of every set in mixed order."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_py as O
from helpers import SimtTwin, assert_bins_close, assert_sets_equal, assert_state_close
from param_sets import PARAM_SETS
from pwpp_ctypes import PwppBinResult, PwppParams

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_param_sets.so")


@pytest.fixture(scope="module", autouse=True)
def _build_sets_twin():
    """Same compile line as the twin (tests/conftest.py: build_simt)."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_param_sets.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_param_sets.cpp")])


def narrow_rings():
    """The default set with rings narrower than 1.5 m in zone 0: build_geometry sends it to the exact binning kernel."""
    p = PARAM_SETS["default"][0]()
    p.num_rings_each_zone[:] = [8, 4, 4, 4]   # zone 0: 1.2 m rings
    p.sensor_height = 1.9
    return p


class SetsTwin(SimtTwin):
    """helpers.SimtTwin on libpwpp_simt_param_sets.so."""

    def __init__(self, sets, stream_set, **options):
        lib = C.CDLL(LIB)
        self._bind(lib, "simt_")
        lib.simt_create_sets.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]; lib.simt_create_sets.restype = C.c_void_p
        lib.simt_bin_ids.argtypes = [C.c_void_p, C.c_void_p]
        lib.simt_bin_results.argtypes = [C.c_void_p, C.c_void_p]
        lib.simt_select.argtypes = [C.c_void_p, C.c_int]
        lib.simt_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        lib.simt_estimate_sets.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        lib.simt_estimate_sets.restype = C.c_int
        self._lib = lib
        self._sets = (PwppParams * len(sets))(*sets)
        ids = (C.c_int * len(stream_set))(*stream_set)
        self._h = lib.simt_create_sets(self._sets, len(sets), ids, len(stream_set))
        assert self._h
        self.nbins = 0
        self._ns = [0] * len(stream_set)
        for k, v in options.items():
            assert lib.simt_set_option(self._h, k.encode(), int(v)) == 0, k

    def estimate_sets(self, streams, frames):
        frames = [np.ascontiguousarray(a, dtype=np.float32) for a in frames]
        ids = (C.c_int * len(frames))(*streams)
        ptrs = (C.c_void_p * len(frames))(*[a.ctypes.data for a in frames])
        ns = (C.c_int64 * len(frames))(*[a.shape[0] for a in frames])
        fast = C.c_int(-1)
        rc = self._lib.simt_estimate_sets(self._h, len(frames), ids, ptrs, ns, frames[0].shape[1], C.byref(fast))
        assert rc == 0
        self._ns[:len(frames)] = [a.shape[0] for a in frames]
        return fast.value

    def frame_bins(self, nbins):
        arr = (PwppBinResult * nbins)()
        self._lib.simt_bin_results(self._h, C.byref(arr))
        return arr


def _same(one, tw, f, s, nbins, what):
    """Bit for bit what the unchanged one-set twin computes for the stream: bins, index lists, patch records, state."""
    tw.select(f)
    assert np.array_equal(one.bin_ids(), tw.bin_ids()), f"{what}: bin ids differ from the one-set twin"
    assert np.array_equal(one.getGroundIndices(), tw.getGroundIndices()), f"{what}: ground list differs from the one-set twin"
    assert np.array_equal(one.getNongroundIndices(), tw.getNongroundIndices()), f"{what}: non-ground list differs from the one-set twin"
    assert bytes(one.bin_results()) == bytes(tw.frame_bins(nbins)), f"{what}: patch records differ from the one-set twin"
    tw.select(s)
    assert bytes(one.state()) == bytes(tw.state()), f"{what}: state differs from the one-set twin"
    for r in range(4):
        for w in (0, 1):
            assert one.history(r, w).tobytes() == tw.history(r, w).tobytes(), f"{what}: history ring {r} kind {w}"


def _check(orc, tw, f, s, a, what):
    """Frame f of the call (stream s) against its oracle. Returns False when the frame has a fitted patch of fewer than 5 points (the
    `ros` set fits patches down to one point, num_min_pts = 0): such planes are ill-conditioned, the frame is compared outside
    those patches only, as in tests/test_simt_kernels.py, and later frames of the stream no longer follow the oracle's state."""
    tw.select(f)
    ids = orc.bin_ids()
    assert np.array_equal(ids, tw.bin_ids()), f"{what}: bin ids differ"
    g_o, ng_o, g_t, ng_t = orc.getGroundIndices(), orc.getNongroundIndices(), tw.getGroundIndices(), tw.getNongroundIndices()
    degenerate = (orc.bin_min_fit_n() < 3) | np.array([r.fitted and r.n < 5 for r in orc.bin_results()])
    if degenerate.any():
        keep = ~np.r_[degenerate, np.zeros(3, bool)][ids]
        mo = np.zeros(len(a), bool); mo[g_o] = True
        mt = np.zeros(len(a), bool); mt[g_t] = True
        assert np.array_equal(mo[keep], mt[keep]), f"{what}: labels differ outside degenerate patches"
        return False
    assert_sets_equal(g_o, ng_o, g_t, ng_t, len(a), what)
    assert_bins_close(orc.bin_results(), tw.frame_bins(orc.nbins), orc.nbins, what)
    assert np.abs(orc.getCenters().astype(np.float64) - tw.getCenters()).max(initial=0) <= 1e-6, what
    tw.select(s)
    assert_state_close(orc.state(), tw.state(), f"{what} state")
    for r in range(4):
        for w in (0, 1):
            assert np.allclose(tw.history(r, w), orc.history(r, w), rtol=1e-6, atol=1e-9), f"{what}: history ring {r} kind {w}"
    return True


def _run(tw, sets, stream_set, schedule, expect_fast, opts, kitti):
    """Every frame: bit for bit the one-set twin of its stream's set, and the oracle while the stream's frames are well-posed."""
    orcs, ones, clean = {}, {}, {}
    for c, (streams, scans) in enumerate(schedule):
        assert tw.estimate_sets(streams, [kitti[k] for k in scans]) == expect_fast[c]
        for f, (s, k) in enumerate(zip(streams, scans)):
            p = sets[stream_set[s]]
            orc = orcs.setdefault(s, O.Oracle(params=p, arith=O.ARITH_CANON64))
            one = ones.setdefault(s, SimtTwin(p, **opts))
            orc.estimate(kitti[k]); one.estimate(kitti[k])
            what = f"{opts} call {c} frame {f} (stream {s}, set {stream_set[s]})"
            _same(one, tw, f, s, orc.nbins, what)
            if clean.get(s, True):
                clean[s] = _check(orc, tw, f, s, kitti[k], what)
    return clean


@pytest.mark.parametrize("opts", [dict(), dict(front=0, patch=1)], ids=["cluster_front", "three_kernel_front"])
def test_mixed_sets_in_one_launch_sequence(kitti, opts):
    """Three sets of tests/param_sets.py, six streams interleaved over them; three calls with mixed, permuted stream tables.
    Every frame runs with its own set's geometry (bin ids), thresholds (index lists, patch records) and state (histories)."""
    sets = [PARAM_SETS[n][0]() for n in ("default", "ros", "no_rvpf_tgr")]
    stream_set = [0, 1, 2, 0, 1, 2]
    schedule = [([0, 1, 2, 3, 4, 5], [0, 1, 2, 3, 4, 5]), ([5, 2, 4, 0], [1, 3, 0, 2]), ([1, 3, 2], [4, 5, 1])]
    clean = _run(SetsTwin(sets, stream_set, **opts), sets, stream_set, schedule, [1, 1, 1], opts, kitti)
    assert clean[0] and clean[3], f"the default-set streams left the full oracle comparison: {clean}"


def test_a_set_without_the_fp32_filter_sends_the_call_to_the_exact_kernel(kitti):
    """A call that names a set whose geometry the fp32 filter does not cover bins every frame with the exact kernel; a call
    that names only covered sets takes the filter. Both are exact, so each frame matches its own oracle either way."""
    sets = [PARAM_SETS["default"][0](), narrow_rings()]
    schedule = [([0, 1, 2], [0, 1, 2]), ([2, 0], [3, 4])]
    clean = _run(SetsTwin(sets, [0, 1, 0]), sets, [0, 1, 0], schedule, [0, 1], dict(), kitti)
    assert all(clean.values())
