"""The frame-table kernel of bound calls (csrc/pwpp_records.cuh, k_bound_table), executed on the CPU by the SIMT stand-in
(tests/simt/simt_bound_table.cpp) and compared word for word with numpy.

From the device counts of a bound call the kernel accepts every count in [0, max_n[f]] (any other makes an empty frame and
sets status[f] = PWPP_COUNT_OUT_OF_RANGE), writes the int64 exclusive scan of the accepted counts, the scan of their
ceil(n / 4096) chunks, and copies the bound call's stream and set tables. Every output array is filled with a sentinel first;
the words after its nframes (+ 1) entries must keep it."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_bound_table.so")
CHUNK_PTS = 4096
OUT_OF_RANGE = 1        # PWPP_COUNT_OUT_OF_RANGE
SENT64, SENT32 = -0x5A5A5A5A5A5A5A5B, -0x5A5A5A5B
PAD = 16                # sentinel words after every output array


@pytest.fixture(scope="module")
def lib():
    """Same compile line as test_simt_records.py's library."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_bound_table.cpp", "simt_records.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_bound_table.cpp")])
    L = C.CDLL(LIB)
    L.simt_bound_table.argtypes = [C.c_int] + [C.c_void_p] * 9
    L.simt_bound_table.restype = None
    return L


def expected(counts, max_n, streams, sets):
    ok = (counts >= 0) & (counts <= max_n)
    n = np.where(ok, counts, 0)
    pt_off = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    chunk_off = np.concatenate([[0], np.cumsum((n + CHUNK_PTS - 1) // CHUNK_PTS)]).astype(np.int32)
    return pt_off, chunk_off, streams.astype(np.int32), sets.astype(np.int32), np.where(ok, 0, OUT_OF_RANGE).astype(np.int32)


def run(lib, counts, max_n, streams, sets):
    nf = len(counts)
    counts, max_n = np.ascontiguousarray(counts, np.int64), np.ascontiguousarray(max_n, np.int64)
    streams, sets = np.ascontiguousarray(streams, np.int32), np.ascontiguousarray(sets, np.int32)
    out = [np.full(nf + 1 + PAD, SENT64, np.int64), np.full(nf + 1 + PAD, SENT32, np.int32)] + [np.full(nf + PAD, SENT32, np.int32) for _ in range(3)]
    lib.simt_bound_table(nf, counts.ctypes.data, max_n.ctypes.data, streams.ctypes.data, sets.ctypes.data, *[o.ctypes.data for o in out])
    want = expected(counts, max_n, streams, sets)
    names = ("pt_off", "chunk_off", "stream", "pset", "status")
    for name, o, w in zip(names, out, want):
        assert np.array_equal(o[:len(w)], w), f"{name}: first mismatch at {np.flatnonzero(o[:len(w)] != w)[:5]}"
        assert np.all(o[len(w):] == (SENT64 if o.dtype == np.int64 else SENT32)), f"{name}: a word after the table changed"
    return want


# the counts every frame count is tried with, relative to a capacity cap
def count_menu(cap):
    return [0, 1, 4095, 4096, 4097, cap, cap + 1, -1]


@pytest.mark.parametrize("nf", [1, 2, 4, 5, 1000, 65535])
def test_counts_at_every_boundary(lib, nf):
    """Every count of the menu cycles through the frames (so each slice of the CTA sees several of them), with capacities of
    4097 points and more, and the stream and set tables hold distinct values per frame."""
    rng = np.random.default_rng(nf)
    max_n = rng.integers(4097, 20000, nf)
    kinds = np.arange(nf) % 8 if nf > 8 else rng.integers(0, 8, nf)
    counts = np.array([count_menu(int(c))[k] for c, k in zip(max_n, kinds)], np.int64)
    streams = rng.integers(0, 65535, nf)
    sets = rng.integers(0, 8, nf)
    pt_off, _, _, _, status = run(lib, counts, max_n, streams, sets)
    assert status.sum() == np.count_nonzero((counts < 0) | (counts > max_n))


@pytest.mark.parametrize("nf", [1, 2, 4, 5, 1000, 65535])
def test_every_count_of_one_kind(lib, nf):
    """All frames on one count of the menu at a time: all empty, all full, all out of range."""
    max_n = np.full(nf, 4097, np.int64)
    for c in count_menu(4097):
        run(lib, np.full(nf, c, np.int64), max_n, np.arange(nf) % 7, np.arange(nf) % 3)


@pytest.mark.parametrize("nf", [1, 5, 1000, 65535])
def test_zero_capacity(lib, nf):
    """max_n = 0: a count of 0 is accepted, 1 and -1 are out of range; mixed with frames of capacity."""
    rng = np.random.default_rng(7)
    max_n = np.where(np.arange(nf) % 2, 0, 5000).astype(np.int64)
    counts = rng.choice([-1, 0, 1, 5000], nf).astype(np.int64)
    run(lib, counts, max_n, np.zeros(nf), np.zeros(nf))
    run(lib, np.zeros(nf, np.int64), np.zeros(nf, np.int64), np.zeros(nf), np.zeros(nf))


def test_large_totals_scan_in_64_bits(lib):
    """65535 frames of up to 2^31 - 4097 points: the point scan passes 2^32, and the chunk scan stays below 2^31."""
    nf = 65535
    max_n = np.full(nf, 2 ** 31 - 4097, np.int64)
    # every 32nd frame full (2048 x 524288 chunks): the chunk total stays an int, as the bind requires of the capacities
    counts = np.where(np.arange(nf) % 32 == 0, max_n, np.arange(nf) * 100).astype(np.int64)
    pt_off = run(lib, counts, max_n, np.arange(nf), np.arange(nf) % 8)[0]
    assert pt_off[-1] > 2 ** 32
