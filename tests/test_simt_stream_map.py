"""The kernels with a non-identity stream table, executed on the CPU by the SIMT stand-in (tests/simt/simt_streams.cpp, the
twin of tests/simt/simt_twin.cpp with a stream-table entry point): frame f of a call advances stream streams[f] of a larger
state array. Every stream is compared with its own CANON64 oracle fed the same frames in the same order, and the streams a
call does not name keep their state and histories."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_py as O
from helpers import SimtTwin, assert_bins_close, assert_sets_equal, assert_state_close
from pwpp_ctypes import PwppParams, default_params

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_streams.so")


@pytest.fixture(scope="module", autouse=True)
def _build_stream_twin():
    """Same compile line as the twin (tests/conftest.py: build_simt)."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_streams.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_streams.cpp")])


class StreamTwin(SimtTwin):
    """helpers.SimtTwin on libpwpp_simt_streams.so."""

    def __init__(self, num_streams, **options):
        lib = C.CDLL(LIB)
        self._bind(lib, "simt_")
        lib.simt_create.argtypes = [C.POINTER(PwppParams), C.c_int]; lib.simt_create.restype = C.c_void_p
        lib.simt_bin_ids.argtypes = [C.c_void_p, C.c_void_p]
        lib.simt_bin_results.argtypes = [C.c_void_p, C.c_void_p]
        lib.simt_num_bins.argtypes = [C.c_void_p]
        lib.simt_select.argtypes = [C.c_void_p, C.c_int]
        lib.simt_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        lib.simt_estimate_streams.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        lib.simt_estimate_streams.restype = C.c_int
        self._lib = lib
        self.params = default_params()
        self._h = lib.simt_create(C.byref(self.params), num_streams)
        self.nbins = lib.simt_num_bins(self._h)
        self._ns = [0] * num_streams
        for k, v in options.items():
            assert lib.simt_set_option(self._h, k.encode(), int(v)) == 0, k

    def estimate_streams(self, streams, frames):
        frames = [np.ascontiguousarray(a, dtype=np.float32) for a in frames]
        ids = (C.c_int * len(frames))(*streams)
        ptrs = (C.c_void_p * len(frames))(*[a.ctypes.data for a in frames])
        ns = (C.c_int64 * len(frames))(*[a.shape[0] for a in frames])
        rc = self._lib.simt_estimate_streams(self._h, len(frames), ids, ptrs, ns, frames[0].shape[1])
        if rc == 0:
            self._ns = [a.shape[0] for a in frames] + self._ns[len(frames):]
        return rc

    def snapshot(self, s):
        """State and histories of stream s, as bytes."""
        self.select(s)
        return bytes(self.state()) + b"".join(self.history(r, w).tobytes() for r in range(4) for w in (0, 1))


def _check_frame(orc, tw, a, what):
    assert np.array_equal(orc.bin_ids(), tw.bin_ids()), f"{what}: bin ids differ"
    assert (orc.bin_min_fit_n() >= 3).all(), f"{what}: the frame has a degenerate patch (choose another input)"
    assert_sets_equal(orc.getGroundIndices(), orc.getNongroundIndices(), tw.getGroundIndices(), tw.getNongroundIndices(), len(a), what)
    assert_bins_close(orc.bin_results(), tw.bin_results(), orc.nbins, what)


def _check_stream(orc, tw, s, what):
    tw.select(s)
    assert_state_close(orc.state(), tw.state(), what)
    for r in range(4):
        for w in (0, 1):
            assert np.allclose(tw.history(r, w), orc.history(r, w), rtol=1e-6, atol=1e-9), f"{what}: history ring {r} kind {w}"


def test_permuted_subset_of_the_streams(kitti):
    """Seven streams, three calls naming a permuted subset each: the kernels read and write the state of the named stream
    (front end, every fit class's zone-0 margin, k_gle's state and history rows), with both front-end variants."""
    schedule = [([5, 2, 0], [0, 1, 2]), ([2, 6, 5], [3, 4, 5]), ([0, 5], [1, 3])]
    for opts in (dict(), dict(front=0, patch=1)):
        tw = StreamTwin(7, **opts)
        orcs = {}
        fresh = tw.snapshot(4)
        for c, (streams, scans) in enumerate(schedule):
            untouched = {s: tw.snapshot(s) for s in range(7) if s not in streams}
            assert tw.estimate_streams(streams, [kitti[k] for k in scans]) == 0
            for f, (s, k) in enumerate(zip(streams, scans)):
                orc = orcs.setdefault(s, O.Oracle(arith=O.ARITH_CANON64))
                orc.estimate(kitti[k])
                tw.select(f)
                _check_frame(orc, tw, kitti[k], f"{opts} call {c} frame {f} (stream {s})")
                _check_stream(orc, tw, s, f"{opts} call {c} stream {s}")
            for s, snap in untouched.items():
                assert tw.snapshot(s) == snap, f"{opts} call {c}: stream {s} was not named but changed"
        assert tw.snapshot(4) == fresh   # never named


def test_a_repeated_or_unknown_stream_is_refused():
    """The twin runs one launch sequence: a table with a repeated id, or an id outside the state array, is refused."""
    tw = StreamTwin(3)
    a = np.array([[5, 0, -1.7, 0.5]], np.float32)
    assert tw.estimate_streams([1, 1], [a, a]) == -1
    assert tw.estimate_streams([3], [a]) == -1
    assert tw.estimate_streams([-1], [a]) == -1
