"""The width selector of bound calls with a width ladder (csrc/pwpp_ladder.cuh, k_ladder_select), executed on the CPU by the SIMT
stand-in (tests/simt/simt_bound_ladder.cpp) and compared with a numpy statement of include/pwpp.h's width rule.

A position runs when the table kernel left it status 0, PWPP_COUNT_OUT_OF_RANGE, PWPP_SLOT_OUT_OF_RANGE or
PWPP_OFFSETS_OUT_OF_RANGE, and is rejected for PWPP_FRAME_SKIPPED, PWPP_ACTION_INVALID, PWPP_STREAM_OUT_OF_RANGE or
PWPP_STREAM_DUPLICATE. With L = 1 + the last position that runs (0 when none does), the run launches the smallest ladder width
w >= max(L, 1). The kernel writes w to d_width and the index of w in the ladder to the graph's SWITCH node
(cudaGraphSetConditional, recorded by the stand-in)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_bound_ladder.so")
RUNS = (0, 1, 4, 5)        # 0, PWPP_COUNT_OUT_OF_RANGE, PWPP_SLOT_OUT_OF_RANGE, PWPP_OFFSETS_OUT_OF_RANGE
REJECTED = (2, 3, 6, 7)    # PWPP_FRAME_SKIPPED, PWPP_ACTION_INVALID, PWPP_STREAM_OUT_OF_RANGE, PWPP_STREAM_DUPLICATE
LS_THREADS = 256           # the selector's CTA
MAX_WIDTHS = 8             # PWPP_MAX_LADDER_WIDTHS, nframes included


def declare(L, name):
    fn = getattr(L, name)
    fn.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    fn.restype = C.c_int

    def select(status, widths):
        """(width written to d_width, index given to cudaGraphSetConditional) for one launch."""
        st = np.ascontiguousarray(status, dtype=np.int32)
        w = np.ascontiguousarray(widths, dtype=np.int32)
        width, index = np.full(1, -7, np.int32), np.full(1, -7, np.int32)
        assert fn(len(st), st.ctypes.data, w.ctypes.data, len(w), width.ctypes.data, index.ctypes.data) == 0, f"{name}: CUDA error"
        return int(width[0]), int(index[0])
    return select


def build_lib():
    """Same compile line as test_simt_bound_streams.py's library."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_bound_ladder.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_bound_ladder.cpp")])
    return declare(C.CDLL(LIB), "simt_ladder_select")


@pytest.fixture(scope="module")
def select():
    return build_lib()


def expected(status, widths):
    """The width rule: (w, its index in the ladder)."""
    runs = np.flatnonzero(~np.isin(np.asarray(status), REJECTED))
    need = max(int(runs[-1]) + 1 if len(runs) else 0, 1)
    i = next(k for k, w in enumerate(widths) if w >= need)
    return widths[i], i


def ladder(rng, nf, n):
    """A random strictly increasing ladder of n widths ending with nf."""
    inner = sorted(rng.choice(np.arange(1, nf), n - 1, replace=False).tolist()) if n > 1 else []
    return inner + [nf]


def rejected(rng, nf):
    return rng.choice(REJECTED, nf)


def every_code_at_every_position():
    """Every status code at every position of a 20-position call whose other positions are rejected, on ladder {1, 4, 16}."""
    rng = np.random.default_rng(1)
    for code in RUNS + REJECTED:
        for p in range(20):
            st = rejected(rng, 20)
            st[p] = code
            yield f"code{code}-pos{p}", st, [1, 4, 16, 20]


def nothing_and_everything():
    rng = np.random.default_rng(2)
    for nf in (2, 5, 64, 300):
        w = [1, 4, 16, nf] if nf > 16 else [1, nf]
        yield f"none-nf{nf}", rejected(rng, nf), w
        yield f"all-nf{nf}", rng.choice(RUNS, nf), w
        yield f"zeros-nf{nf}", np.zeros(nf, np.int32), w


def ladders_of_every_length():
    """Ladders of one (nframes alone) to PWPP_MAX_LADDER_WIDTHS widths, the last running position swept over the call."""
    rng = np.random.default_rng(3)
    nf = 64
    for n in range(1, MAX_WIDTHS + 1):
        w = ladder(rng, nf, n)
        for last in [-1, 0] + sorted(set(w[:-1]) | {x - 1 for x in w[:-1]} | {x + 1 for x in w[:-1] if x + 1 < nf}) + [nf - 1]:
            st = rejected(rng, nf)
            if last >= 0:
                st[last] = rng.choice(RUNS)
                st[:last] = np.where(rng.random(last) < 0.5, rng.choice(RUNS, last), st[:last])
            yield f"n{n}-last{last}", st, w


def wide_calls():
    """nframes above the CTA's thread count, so that every thread scans several positions and the last running one can sit in
    any thread's slice and any warp."""
    rng = np.random.default_rng(4)
    for nf in (LS_THREADS + 1, 2 * LS_THREADS + 3, 1000, 4097):
        w = sorted({1, 4, 16, LS_THREADS, nf - 1, nf})
        for last in sorted({-1, 0, 3, 31, 32, LS_THREADS - 1, LS_THREADS, LS_THREADS + 1, nf - 2, nf - 1} - {nf}):
            st = rejected(rng, nf)
            if last >= 0:
                st[last] = rng.choice(RUNS)
                st[:last] = np.where(rng.random(last) < 0.3, rng.choice(RUNS, last), st[:last])
            yield f"nf{nf}-last{last}", st, w


GROUPS = {"every_code": every_code_at_every_position, "nothing_everything": nothing_and_everything,
          "ladder_lengths": ladders_of_every_length, "wide": wide_calls}


def run_group(select, group):
    n = 0
    for name, st, w in GROUPS[group]():
        assert select(st, w) == expected(st, w), f"{name}: status {np.asarray(st).tolist()[:64]} widths {w}"
        n += 1
    assert n > 0


@pytest.mark.parametrize("group", list(GROUPS))
def test_width_rule(select, group):
    run_group(select, group)


def test_model_examples():
    """The numpy statement itself on hand-made cases."""
    assert expected([2, 2, 2], [1, 3]) == (1, 0)             # nothing runs: the narrowest width
    assert expected([0, 2, 2], [1, 3]) == (1, 0)
    assert expected([2, 1, 2], [1, 3]) == (3, 1)
    assert expected([7, 6, 5, 3], [1, 2, 4]) == (4, 2)       # OFFSETS_OUT_OF_RANGE runs
    assert expected([4, 6, 3, 7], [1, 2, 4]) == (1, 0)       # SLOT_OUT_OF_RANGE runs; the rest is rejected
