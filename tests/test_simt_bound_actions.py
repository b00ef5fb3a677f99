"""The frame-table kernel of bound calls with per-frame actions (csrc/pwpp_records.cuh, k_bound_table_actions) and the reset
kernel launched before a dependent run (k_bound_reset), executed on the CPU by the SIMT stand-in
(tests/simt/simt_bound_actions.cpp) and compared word for word with numpy.

The table kernel copies every action, skips every frame whose action is neither PWPP_FRAME_RUN nor PWPP_FRAME_RESET (its count
is not read: n = 0, status PWPP_FRAME_SKIPPED or PWPP_ACTION_INVALID, stream table entry = its scratch slot), accepts the other
frames' counts as k_bound_table does, and restores the constructor state of the stream of every RESET frame whose stream has no
frame in an earlier run. k_bound_reset restores those of the remaining RESET frames of one run. Every output array is filled
with a sentinel first and the words after its table must keep it; the state array is sentinel-filled and the init array
patterned, so a state that changed shows which kernel wrote it."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_bound_actions.so")
CHUNK_PTS = 4096
RUN, SKIP, RESET = 0, 1, 2                       # PWPP_FRAME_*
OUT_OF_RANGE, SKIPPED, INVALID = 1, 2, 3         # PWPP_COUNT_OUT_OF_RANGE, PWPP_FRAME_SKIPPED, PWPP_ACTION_INVALID
I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1
ACTION_MENU = [RUN, SKIP, RESET, -1, 3, I32_MIN, I32_MAX]
SENT64, SENT32 = -0x5A5A5A5A5A5A5A5B, -0x5A5A5A5B
PAD = 16                # sentinel words (and state rows) after every output array


@pytest.fixture(scope="module")
def lib():
    """Same compile line as test_simt_bound_table.py's library."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_bound_actions.cpp", "simt_records.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_bound_actions.cpp")])
    L = C.CDLL(LIB)
    L.simt_stream_state_bytes.restype = C.c_int
    L.simt_bound_table_actions.argtypes = [C.c_int] + [C.c_void_p] * 15
    L.simt_bound_table_actions.restype = None
    L.simt_bound_reset.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 5
    L.simt_bound_reset.restype = None
    return L


def bind_tables(streams, num_streams):
    """What pwpp_bind_call_actions derives from the stream table: the runs (maximal spans of pairwise distinct streams), the
    scratch slot of every frame (num_streams + its place in its run) and whether its stream has a frame in an earlier run."""
    nf = len(streams)
    runs, last = [0], {}
    for f, s in enumerate(streams):
        if s in last and last[s] >= runs[-1]:
            runs.append(f)
        last[s] = f
    runs.append(nf)
    scratch, dep = np.zeros(nf, np.int32), np.zeros(nf, np.int32)
    first_run = {}
    for r in range(len(runs) - 1):
        for f in range(runs[r], runs[r + 1]):
            first_run.setdefault(streams[f], r)
            scratch[f] = num_streams + f - runs[r]
            dep[f] = first_run[streams[f]] < r
    return runs, scratch, dep


def expected(counts, max_n, streams, sets, actions, scratch):
    runs_ = (actions == RUN) | (actions == RESET)
    ok = (counts >= 0) & (counts <= max_n)
    n = np.where(runs_ & ok, counts, 0)
    pt_off = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    chunk_off = np.concatenate([[0], np.cumsum((n + CHUNK_PTS - 1) // CHUNK_PTS)]).astype(np.int32)
    status = np.where(runs_, np.where(ok, 0, OUT_OF_RANGE), np.where(actions == SKIP, SKIPPED, INVALID)).astype(np.int32)
    stream = np.where(runs_, streams, scratch).astype(np.int32)
    return pt_off, chunk_off, stream, sets.astype(np.int32), status, actions.astype(np.int32)


def run(lib, counts, max_n, streams, sets, actions, num_streams):
    """One table launch, then one reset launch per run that holds a dependent frame, as pwpp_run_bound_call issues them; every
    output word and every state row is checked after each launch."""
    nf = len(counts)
    counts, max_n = np.ascontiguousarray(counts, np.int64), np.ascontiguousarray(max_n, np.int64)
    streams, sets = np.ascontiguousarray(streams, np.int32), np.ascontiguousarray(sets, np.int32)
    actions = np.ascontiguousarray(actions, np.int32)
    runs, scratch, dep = bind_tables(streams.tolist(), num_streams)
    sb = lib.simt_stream_state_bytes()
    nslots = num_streams + (max(np.diff(runs)) if nf else 0)
    init = ((np.arange(nslots)[:, None] * 7 + np.arange(sb)[None, :]) % 251 + 1).astype(np.uint8)   # never the sentinel byte
    init = np.ascontiguousarray(init)
    states = np.full((nslots + PAD, sb), 0x5A, np.uint8)
    out = [np.full(nf + 1 + PAD, SENT64, np.int64), np.full(nf + 1 + PAD, SENT32, np.int32)] + [np.full(nf + PAD, SENT32, np.int32) for _ in range(4)]
    lib.simt_bound_table_actions(nf, counts.ctypes.data, max_n.ctypes.data, streams.ctypes.data, sets.ctypes.data, *[o.ctypes.data for o in out[:5]],
                                 actions.ctypes.data, out[5].ctypes.data, scratch.ctypes.data, dep.ctypes.data, init.ctypes.data, states.ctypes.data)
    want = expected(counts, max_n, streams, sets, actions, scratch)
    names = ("pt_off", "chunk_off", "stream", "pset", "status", "act")
    for name, o, w in zip(names, out, want):
        assert np.array_equal(o[:len(w)], w), f"{name}: first mismatch at {np.flatnonzero(o[:len(w)] != w)[:5]}"
        assert np.all(o[len(w):] == (SENT64 if o.dtype == np.int64 else SENT32)), f"{name}: a word after the table changed"
    reset = np.zeros(nslots + PAD, bool)
    reset[np.unique(streams[(actions == RESET) & (dep == 0)])] = True
    check_states(states, init, reset, "k_bound_table_actions")
    for r in range(len(runs) - 1):
        f0, f1 = runs[r], runs[r + 1]
        if not dep[f0:f1].any():
            continue
        lib.simt_bound_reset(f0, f1, out[5].ctypes.data, dep.ctypes.data, streams.ctypes.data, init.ctypes.data, states.ctypes.data)
        sel = (actions[f0:f1] == RESET) & (dep[f0:f1] == 1)
        reset[streams[f0:f1][sel]] = True
        check_states(states, init, reset, f"k_bound_reset of run {r}")
    return want


def check_states(states, init, reset, who):
    rows = len(init)
    got_init = np.all(states[:rows] == init, axis=1)
    got_sent = np.all(states == 0x5A, axis=1)
    assert np.array_equal(got_init, reset[:rows]), f"{who}: streams reset {np.flatnonzero(got_init)[:8]}, want {np.flatnonzero(reset[:rows])[:8]}"
    assert np.all(got_sent[:rows] | got_init), f"{who}: a state row was partly written"
    assert np.all(got_sent[rows:]), f"{who}: a row after the state array changed"


def stream_table(rng, nf, num_streams, repeats):
    """nf stream ids below num_streams; with repeats some streams come back within a few frames (dependent runs)."""
    if not repeats:
        return rng.permutation(num_streams)[:nf]
    return rng.integers(0, num_streams, nf)


@pytest.mark.parametrize("nf", [1, 2, 4, 5, 1000, 65535])
def test_every_action_with_garbage_counts(lib, nf):
    """Every action of the menu (the three PWPP_FRAME_* values and the invalid -1, 3, INT32_MIN, INT32_MAX) cycles through the
    frames; a skipped frame's count is garbage (out of range either way, or the int64 extremes), a running frame's count sits
    at a boundary of its capacity."""
    rng = np.random.default_rng(nf)
    max_n = rng.integers(4097, 20000, nf)
    actions = np.array(ACTION_MENU * (nf // len(ACTION_MENU) + 1))[:nf] if nf > 7 else rng.choice(ACTION_MENU, nf)
    menu = lambda c: [0, 1, 4095, 4096, 4097, c, c + 1, -1]   # noqa: E731
    counts = np.array([menu(int(c))[k % 8] for k, c in enumerate(max_n)], np.int64)
    runs_ = (actions == RUN) | (actions == RESET)
    garbage = rng.choice([-1, -2 ** 63, 2 ** 63 - 1, 10 ** 12, 5], nf)
    counts = np.where(runs_, counts, garbage)
    num_streams = max(8, nf // 4) if nf > 5 else 3
    streams = stream_table(rng, nf, num_streams, True)
    run(lib, counts, max_n, streams, rng.integers(0, 8, nf), actions, num_streams)


@pytest.mark.parametrize("nf", [1, 5, 1000, 65535])
@pytest.mark.parametrize("action", ACTION_MENU)
def test_one_action_everywhere(lib, nf, action):
    """All frames on one action, distinct streams: all running, all skipped, all reset by the table kernel, all invalid."""
    rng = np.random.default_rng(3)
    max_n = np.full(nf, 5000, np.int64)
    counts = rng.choice([0, 1, 5000, 5001, -1], nf).astype(np.int64)
    streams = rng.permutation(nf)
    _, _, stream, _, status, _ = run(lib, counts, max_n, streams, np.arange(nf) % 4, np.full(nf, action, np.int32), nf)
    if action in (SKIP, -1, 3, I32_MIN, I32_MAX):
        assert np.all(stream >= nf)


def test_repeat_table(lib):
    """The stream table [2, 0, 2, 1, 3, 0, 1]: runs [0, 2), [2, 6), [6, 7). RESET of a stream's first frame is the table kernel's,
    RESET of a later frame (frames 2, 5, 6) the reset kernel's before its run; SKIP of stream 2's first frame with RUN of its
    second; scratch slots restart at every run."""
    streams = np.array([2, 0, 2, 1, 3, 0, 1])
    runs, scratch, dep = bind_tables(streams.tolist(), 4)
    assert runs == [0, 2, 6, 7]
    assert scratch.tolist() == [4, 5, 4, 5, 6, 7, 4]
    assert dep.tolist() == [0, 0, 1, 0, 0, 1, 1]
    max_n = np.full(7, 100, np.int64)
    for actions in ([SKIP, RUN, RESET, RESET, RUN, RESET, RESET], [RESET] * 7, [RUN, SKIP, RUN, SKIP, RESET, RUN, RESET],
                    [SKIP] * 7, [3, RESET, -1, RUN, RESET, I32_MAX, RESET]):
        run(lib, np.array([5, 0, 100, 101, -1, 7, 0]), max_n, streams, np.zeros(7), np.array(actions), 4)


def test_large_totals_scan_in_64_bits(lib):
    """65535 frames of up to 2^31 - 4097 points with every fourth frame skipped: the point scan passes 2^32 past skipped frames."""
    nf = 65535
    max_n = np.full(nf, 2 ** 31 - 4097, np.int64)
    counts = np.where(np.arange(nf) % 32 == 0, max_n, np.arange(nf) * 100).astype(np.int64)
    actions = np.where(np.arange(nf) % 4 == 3, SKIP, RUN)
    pt_off = run(lib, counts, max_n, np.arange(nf), np.arange(nf) % 8, actions, nf)[0]
    assert pt_off[-1] > 2 ** 32
