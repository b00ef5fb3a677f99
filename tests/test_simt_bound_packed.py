"""The frame-table kernels of packed bound calls (csrc/pwpp_records.cuh, k_bound_table_packed and k_bound_table_packed_actions),
executed on the CPU by the SIMT stand-in (tests/simt/simt_bound_packed.cpp) and compared word for word with a numpy model of the
rule; then the record unpack of the run, which reads the run's record table the table kernel wrote, over a packed buffer placed
flush against guard pages.

A frame that runs reads lo = offsets[f] and hi = offsets[f + 1]: offsets outside 0 <= lo <= hi <= capacity give
PWPP_OFFSETS_OUT_OF_RANGE and an empty frame, a count hi - lo above max_n[f] PWPP_COUNT_OUT_OF_RANGE, and an accepted frame's run
record table entry points at base + lo * step. Every other frame keeps src = base with n = 0; a skipped frame reads no offset.
Every output array is filled with a sentinel first and the words after its table must keep it."""
import ctypes as C
import mmap
import os
import subprocess

import numpy as np
import pytest

from test_simt_bound_actions import ACTION_MENU, INVALID, OUT_OF_RANGE, PAD, RESET, RUN, SENT32, SENT64, SKIP, SKIPPED, bind_tables, check_states
from test_simt_bound_rings import layout, make_records

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_bound_packed.so")
CHUNK_PTS = 4096
OFFSETS_OUT_OF_RANGE = 5   # PWPP_OFFSETS_OUT_OF_RANGE
I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1


def build_lib():
    """Same compile line as test_simt_bound_rings.py's library."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_bound_packed.cpp", "simt_records.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_bound_packed.cpp")])
    return C.CDLL(LIB)


@pytest.fixture(scope="module")
def lib():
    L = build_lib()
    L.simt_stream_state_bytes.restype = C.c_int
    L.simt_record_frame_bytes.restype = C.c_int
    L.simt_bound_table_packed.argtypes = [C.c_int] + [C.c_void_p] * 16 + [C.c_int64, C.c_void_p, C.c_void_p]
    L.simt_bound_table_packed.restype = None
    L.simt_unpack_run.argtypes = [C.c_int] + [C.c_void_p] * 4
    L.simt_unpack_run.restype = None
    assert L.simt_record_frame_bytes() == 48
    return L


def run_table(lib, base, step, capacity, offsets, max_n, streams, sets, actions, num_streams):
    """One packed table launch; checks every output word against the numpy model and returns (pt_off, status, the run's record
    table as nframes rows of 48 bytes)."""
    nf = len(max_n)
    max_n = np.ascontiguousarray(max_n, np.int64)
    offsets = np.ascontiguousarray(offsets, np.int64)
    assert len(offsets) == nf + 1
    streams, sets = np.ascontiguousarray(streams, np.int32), np.ascontiguousarray(sets, np.int32)
    lay = layout(step)
    runs, scratch, dep = bind_tables(streams.tolist(), num_streams)
    sb = lib.simt_stream_state_bytes()
    nslots = num_streams + (max(np.diff(runs)) if nf else 0)
    init = np.ascontiguousarray(((np.arange(nslots)[:, None] * 7 + np.arange(sb)[None, :]) % 251 + 1).astype(np.uint8))
    states = np.full((nslots + PAD, sb), 0x5A, np.uint8)
    out = [np.full(nf + 1 + PAD, SENT64, np.int64), np.full(nf + 1 + PAD, SENT32, np.int32)] + [np.full(nf + PAD, SENT32, np.int32) for _ in range(4)]
    brun = np.full((nf + PAD) * 48, 0x5A, np.uint8)
    acts = None if actions is None else np.ascontiguousarray(actions, np.int32)
    lib.simt_bound_table_packed(nf, max_n.ctypes.data, streams.ctypes.data, sets.ctypes.data, *[o.ctypes.data for o in out[:5]],
                                None if acts is None else acts.ctypes.data, out[5].ctypes.data, scratch.ctypes.data, dep.ctypes.data,
                                init.ctypes.data, states.ctypes.data, C.c_void_p(base), C.byref(lay), capacity, offsets.ctypes.data,
                                brun.ctypes.data)
    # the model: each frame judged by its own two entries
    runs_ = np.ones(nf, bool) if acts is None else (acts == RUN) | (acts == RESET)
    lo, hi = offsets[:-1], offsets[1:]
    off_ok = runs_ & (lo >= 0) & (hi >= lo) & (hi <= capacity)
    c = np.where(off_ok, hi - np.where(off_ok, lo, 0), -1)
    ok = off_ok & (c <= max_n)
    n = np.where(ok, c, 0)
    pt_off = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    chunk_off = np.concatenate([[0], np.cumsum((n + CHUNK_PTS - 1) // CHUNK_PTS)]).astype(np.int32)
    skip_st = np.zeros(nf, np.int32) if acts is None else np.where(acts == SKIP, SKIPPED, INVALID)
    status = np.where(runs_, np.where(ok, 0, np.where(off_ok, OUT_OF_RANGE, OFFSETS_OUT_OF_RANGE)), skip_st).astype(np.int32)
    stream = np.where(runs_, streams, scratch).astype(np.int32)
    want = [pt_off, chunk_off, stream, sets, status]
    names = ["pt_off", "chunk_off", "stream", "pset", "status"]
    if acts is not None:
        want.append(acts)
        names.append("act")
    for name, o, w in zip(names, out, want):
        assert np.array_equal(o[:len(w)], w), f"{name}: first mismatch at {np.flatnonzero(o[:len(w)] != w)[:5]}"
        assert np.all(o[len(w):] == (SENT64 if o.dtype == np.int64 else SENT32)), f"{name}: a word after the table changed"
    if acts is None:
        assert np.all(out[5] == SENT32), "act was written without actions"
    rec = brun.reshape(-1, 48)
    src = rec[:nf, :8].copy().view(np.uint64).reshape(-1)
    want_src = np.where(ok, np.uint64(base) + (np.where(ok, lo, 0) * step).astype(np.uint64), np.uint64(base))
    assert np.array_equal(src, want_src), f"brun src: first mismatch at {np.flatnonzero(src != want_src)[:5]}"
    assert np.all(rec[:nf, 8:12].copy().view(np.int32) == step), "brun step"
    assert np.all(rec[nf:] == 0x5A), "a record after the table changed"
    reset = np.zeros(nslots + PAD, bool)
    if acts is not None:
        reset[np.unique(streams[(acts == RESET) & (dep == 0)])] = True
    check_states(states, init, reset, "packed table")
    return pt_off, status, rec[:nf].copy()


def random_offsets(rng, nf, capacity):
    """Monotone offsets of a packed batch over [0, capacity], then every invalid kind at random frames: a negative entry, a
    decreasing pair, an entry past capacity, a frame longer than its max_n; max_n just above, at or below each count."""
    cuts = np.sort(rng.integers(0, capacity + 1, nf + 1))
    cuts[0] = rng.integers(0, 3)
    counts = np.diff(cuts)
    max_n = counts + rng.integers(0, 50, nf)
    exact = rng.random(nf) < 0.2
    max_n[exact] = counts[exact]   # a frame at exactly max_n
    off = cuts.astype(np.int64)
    for k in rng.integers(0, nf + 1, max(1, nf // 20)):
        off[k] = rng.choice([-1, I64_MIN, capacity + 1, I64_MAX, max(int(off[k]) - 7, I64_MIN)])
    long_ = rng.integers(0, nf, max(1, nf // 20))
    max_n[long_] = [max(min(int(off[k + 1]) - int(off[k]) - 1, capacity), 0) for k in long_]
    return off, np.maximum(max_n, 0)


@pytest.mark.parametrize("nf", [1, 1023, 1024, 1025, 4097])
@pytest.mark.parametrize("with_actions", [False, True], ids=["packed", "packed_actions"])
def test_offsets_counts_and_actions(lib, nf, with_actions):
    """Valid, negative, decreasing, past-capacity and longer-than-max_n frames over 1 to 4097 frames, so that threads own slices of
    several frames; with actions every action of the menu, a skipped frame's offsets being garbage."""
    rng = np.random.default_rng(nf + 11 * with_actions)
    capacity = 40 * nf + 5
    off, max_n = random_offsets(rng, nf, capacity)
    actions = None
    if with_actions:
        actions = np.array(ACTION_MENU * (nf // len(ACTION_MENU) + 1))[:nf] if nf > 7 else rng.choice(ACTION_MENU, nf)
    num_streams = max(8, nf // 4) if nf > 5 else 3
    streams = rng.integers(0, num_streams, nf) if with_actions else rng.permutation(max(nf, 1))[:nf]
    run_table(lib, 0x7f0000001003, 22, capacity, off, max_n, streams, rng.integers(0, 8, nf), actions, num_streams if with_actions else max(nf, 1))


def test_each_invalid_kind(lib):
    """One frame of each kind between valid ones: negative lo, decreasing pair, hi past capacity, count above max_n, the empty
    frame at capacity, and a frame of exactly max_n. A decreasing pair lets the valid frames around the invalid one overlap."""
    cap = 100
    off = [0, 10, -3, 20, 15, 30, 101, 100, 100, 100]
    max_n = [10, 50, 50, 50, 10, 50, 50, 70, 0]
    _, status, _ = run_table(lib, 0x10000, 16, cap, off, max_n, np.arange(9), np.zeros(9), None, 9)
    bad = OFFSETS_OUT_OF_RANGE
    assert status.tolist() == [0, bad, bad, bad, OUT_OF_RANGE, bad, bad, 0, 0]
    _, status, _ = run_table(lib, 0x10000, 16, cap, [0, 10, 5, 15], [10, 10, 9], np.arange(3), np.zeros(3), None, 3)
    assert status.tolist() == [0, OFFSETS_OUT_OF_RANGE, OUT_OF_RANGE]
    pt_off, status, _ = run_table(lib, 0x10000, 16, 15, [0, 10, 5, 15], [10, 10, 10], np.arange(3), np.zeros(3), None, 3)
    assert status.tolist() == [0, OFFSETS_OUT_OF_RANGE, 0] and pt_off[-1] == 20   # more accepted records than capacity


def test_reset_on_invalid_offsets_and_skips_read_nothing(lib):
    """RESET with invalid offsets still resets (dep 0 here: in the table kernel); skipped frames with garbage offsets around
    them; a stream repeated in a later run (dep 1) is not reset by the table kernel."""
    cap = 1000
    off = [0, 100, -5, 300, I64_MAX, 500, 600, 700]
    streams = [0, 1, 2, 3, 0, 4, 1]
    for acts in ([RESET, RESET, RESET, SKIP, RESET, 9, RESET], [SKIP, SKIP, SKIP, SKIP, SKIP, SKIP, SKIP], [RUN, RESET, SKIP, RUN, RESET, RUN, RESET]):
        _, status, _ = run_table(lib, 0x20000, 13, cap, off, [1000] * 7, streams, np.arange(7) % 3, np.array(acts), 5)
        for f, a in enumerate(acts):
            if a in (RUN, RESET):
                lo, hi = off[f], off[f + 1]
                assert status[f] == (0 if 0 <= lo <= hi <= cap else OFFSETS_OUT_OF_RANGE)


@pytest.mark.parametrize("action", ACTION_MENU)
def test_one_action_everywhere(lib, action):
    """All frames on one action over offsets that are all garbage for the skipped ones."""
    rng = np.random.default_rng(5)
    nf = 300
    off = rng.choice([0, 1, -1, I64_MAX, I64_MIN, 50], nf + 1).astype(np.int64)
    _, status, _ = run_table(lib, 0x30000, 16, 60, off, np.full(nf, 60), rng.permutation(nf), np.arange(nf) % 4,
                             np.full(nf, action, np.int32), nf)
    if action not in (RUN, RESET):
        assert np.all(status == (SKIPPED if action == SKIP else INVALID))


@pytest.mark.parametrize("step", [13, 16, 22])
def test_unpack_through_the_run_table_reads_only_the_buffer(lib, step):
    """A packed buffer placed with its extent [base, base + capacity * step) flush against a PROT_NONE page after it, then right
    after one before it; frames at both ends of the buffer at full length, an empty frame at capacity, and frames whose offsets
    point past either end. The unpack through the run's table must give each frame its records: any read outside faults."""
    rng = np.random.default_rng(step)
    page = mmap.PAGESIZE
    libc = C.CDLL(None, use_errno=True)
    libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    capacity = 700
    raw, pts = make_records(rng, capacity, step)
    extent = capacity * step
    data_pages = (extent + page - 1) // page + 1
    m = mmap.mmap(-1, (data_pages + 2) * page)
    base0 = C.addressof(C.c_char.from_buffer(m))
    assert libc.mprotect(base0, page, 0) == 0 and libc.mprotect(base0 + (data_pages + 1) * page, page, 0) == 0
    off = np.array([0, 300, 300, 450, capacity, capacity, capacity + 1, -1, 200, 450, capacity], np.int64)
    max_n = np.array([300, 0, 150, 250, 0, 5, 5, 700, 250, 250], np.int64)
    try:
        for start in (base0 + (data_pages + 1) * page - extent, base0 + page):   # flush against the guard after / before
            C.memmove(start, raw.ctypes.data, extent)
            pt_off, status, brun = run_table(lib, start, step, capacity, off, max_n, np.arange(10), np.zeros(10), None, 10)
            assert status.tolist() == [0, 0, 0, 0, 0, OFFSETS_OUT_OF_RANGE, OFFSETS_OUT_OF_RANGE, OFFSETS_OUT_OF_RANGE, 0, 0]
            brun = np.ascontiguousarray(brun)
            dst = np.full((int(pt_off[-1]) + 1, 4), np.nan, np.float32)
            lib.simt_unpack_run(10, brun.ctypes.data, max_n.ctypes.data, pt_off.ctypes.data, dst.ctypes.data)
            for f in range(10):
                got = dst[pt_off[f]:pt_off[f + 1]]
                want = pts[off[f]:off[f + 1]] if status[f] == 0 else np.zeros((0, 4), np.float32)
                assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"frame {f}: unpacked points"
    finally:
        libc.mprotect(base0, (data_pages + 2) * page, mmap.PROT_READ | mmap.PROT_WRITE)
