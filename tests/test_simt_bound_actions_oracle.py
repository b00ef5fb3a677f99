"""Why a bound call skips a frame by redirecting it instead of running it with a count of 0, checked on the CPU: one run of a bound
call with actions, executed by the SIMT stand-in (tests/simt/simt_bound_actions_twin.cpp) as the library launches it: the action
table kernel (k_bound_table_actions) writes the run's stream table and sizes, then the launch sequence runs with them. Against
the CANON64 oracle, with max_elevation_storage = max_flatness_storage = 20, so a stream's histories are full after a few KITTI
frames. Then:
  - PWPP_FRAME_SKIP of a stream the run names: the table kernel points the frame at its scratch slot, the stream's state and
    history rows stay bit for bit, the scratch slot stays at its constructor state, and the other frame of the run matches its
    own oracle;
  - PWPP_FRAME_RUN with a count of 0 on the same full stream moves its state, exactly as the oracle's empty frame does;
  - PWPP_FRAME_RESET with a count of 0 ("reset only") and then frames: the stream equals a fresh oracle fed the same frames."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_py as O
from pwpp_ctypes import PwppParams, default_params
from test_simt_stream_map import StreamTwin, _check_frame, _check_stream

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_bound_actions_twin.so")
REAL = 2      # the twin's streams: 0 and 1 real, 2 and 3 the scratch slots of a run's frames 0 and 1
RUN, SKIP, RESET = 0, 1, 2
SKIPPED = 2


def storage20():
    p = default_params()
    p.max_elevation_storage = p.max_flatness_storage = 20
    return p


@pytest.fixture(scope="module")
def twin_lib():
    """Same compile line as the twin (tests/conftest.py: build_simt)."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_bound_actions_twin.cpp", "simt_streams.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(REPO, "include", "pwpp.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_bound_actions_twin.cpp")])
    return LIB


class ActionTwin(StreamTwin):
    """StreamTwin on the harness that runs a bound call's run with actions, created with parameters p."""

    def __init__(self, lib_path, num_streams, p):
        lib = C.CDLL(lib_path)
        self._bind(lib, "simt_")
        lib.simt_create.argtypes = [C.POINTER(PwppParams), C.c_int]; lib.simt_create.restype = C.c_void_p
        lib.simt_bin_ids.argtypes = [C.c_void_p, C.c_void_p]
        lib.simt_bin_results.argtypes = [C.c_void_p, C.c_void_p]
        lib.simt_num_bins.argtypes = [C.c_void_p]
        lib.simt_select.argtypes = [C.c_void_p, C.c_int]
        lib.simt_estimate_streams.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        lib.simt_estimate_streams.restype = C.c_int
        lib.simt_bound_actions_run.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
        lib.simt_bound_actions_run.restype = C.c_int
        self._lib = lib
        self.params = p
        self._h = lib.simt_create(C.byref(self.params), num_streams)
        self.nbins = lib.simt_num_bins(self._h)
        self._ns = [0] * num_streams

    def bound_run(self, streams, actions, frames):
        """One run of a bound call: frame f of stream streams[f] with actions[f] and frames[f] as its records (count = capacity);
        returns the status the table kernel wrote. Results by position as after estimate_streams."""
        nf = len(frames)
        frames = [np.ascontiguousarray(a, dtype=np.float32) for a in frames]
        ids = (C.c_int * nf)(*streams)
        acts = (C.c_int * nf)(*actions)
        scratch = (C.c_int * nf)(*[REAL + f for f in range(nf)])
        ptrs = (C.c_void_p * nf)(*[a.ctypes.data for a in frames])
        ns = (C.c_int64 * nf)(*[a.shape[0] for a in frames])
        status = (C.c_int * nf)()
        assert self._lib.simt_bound_actions_run(self._h, nf, ids, acts, scratch, ptrs, ns, 4, status) == 0
        self._ns = [a.shape[0] if actions[f] in (RUN, RESET) else 0 for f, a in enumerate(frames)] + self._ns[nf:]
        return list(status)


def scan(kitti, k):
    """Scan k of the six KITTI fixtures, cycled."""
    return np.ascontiguousarray(kitti[k % 6], dtype=np.float32)


EMPTY = np.zeros((0, 4), np.float32)


def test_skip_redirect_zero_count_and_reset_against_the_oracle(kitti, twin_lib):
    p = storage20()
    tw = ActionTwin(twin_lib, REAL + 2, p)
    orcs = [O.Oracle(params=p, arith=O.ARITH_CANON64) for _ in range(REAL)]
    fresh_scratch = [tw.snapshot(REAL + f) for f in range(2)]
    for k in range(4):   # both streams to full histories, one run of two frames each time
        a, b = scan(kitti, k), scan(kitti, k + 1)
        assert tw.bound_run([0, 1], [RUN, RUN], [a, b]) == [0, 0]
        for f, (s, x) in enumerate(((0, a), (1, b))):
            orcs[s].estimate(x)
            tw.select(f)
            _check_frame(orcs[s], tw, x, f"warm-up {k} frame {f}")
            _check_stream(orcs[s], tw, s, f"warm-up {k} stream {s}")
    tw.select(0)
    assert all(tw.state().n_elevation[r] == 20 for r in range(4)), "the histories are not full yet"

    # SKIP of stream 0 in a run that names it (frame 1), beside a frame of stream 1: its frame carries records, which must not
    # be read; the table kernel redirects it to scratch slot REAL + 1
    before = tw.snapshot(0)
    b = scan(kitti, 9)
    assert tw.bound_run([1, 0], [RUN, SKIP], [b, scan(kitti, 2)]) == [0, SKIPPED]
    assert tw.snapshot(0) == before, "a skipped frame changed its stream"
    assert [tw.snapshot(REAL + f) for f in range(2)] == fresh_scratch, "a scratch slot left its constructor state"
    orcs[1].estimate(b)
    tw.select(0)
    _check_frame(orcs[1], tw, b, "the run's other frame")
    _check_stream(orcs[1], tw, 1, "the run's other stream")

    # RUN with a count of 0 on the same full stream: the threshold update runs on the trimmed histories and moves the state, as
    # in the oracle
    assert tw.bound_run([0], [RUN], [EMPTY]) == [0]
    orcs[0].estimate(EMPTY)
    assert tw.snapshot(0) != before, "an empty frame on a full stream should move its state"
    _check_stream(orcs[0], tw, 0, "count 0")

    # RESET with a count of 0, then frames: a fresh oracle fed the same (empty, then KITTI) frames
    assert tw.bound_run([0], [RESET], [EMPTY]) == [0]
    fresh = O.Oracle(params=p, arith=O.ARITH_CANON64)
    fresh.estimate(EMPTY)
    _check_stream(fresh, tw, 0, "reset only")
    for k in range(4, 7):
        a = scan(kitti, k)
        assert tw.bound_run([0], [RUN], [a]) == [0]
        fresh.estimate(a)
        tw.select(0)
        _check_frame(fresh, tw, a, f"frame {k} after the reset")
        _check_stream(fresh, tw, 0, f"frame {k} after the reset")
