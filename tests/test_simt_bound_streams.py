"""The frame-table kernels of bound calls with a stream table (csrc/pwpp_records.cuh, k_bound_table_streams,
k_bound_table_rings_streams, k_bound_table_packed_streams), the reset kernel before every later run (k_bound_reset over the
run's copy of the streams) and the state rows (k_bound_states_streams), executed on the CPU by the SIMT stand-in
(tests/simt/simt_bound_streams.cpp) and compared word for word with a numpy statement of the rules.

Every frame reads its stream once into the ctx's copy. The action is judged first (SKIP or an invalid action), then the stream:
s < 0 is a hole (PWPP_FRAME_SKIPPED), s >= num_streams is PWPP_STREAM_OUT_OF_RANGE, and a second frame of one run that would run
on the same stream is PWPP_STREAM_DUPLICATE (the lowest position wins; frames skipped by their action claim nothing). Then the
ring slot or packed offsets, then the count. A rejected frame runs on its scratch slot as an empty frame; its set is its stream's,
or its bound stream's for an invalid id. RESET frames of run 0 are reset by the table kernel, those of later runs by
k_bound_reset; no rejected frame resets anything. The claim table must be all -1 again after the kernel."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_simt_bound_actions import ACTION_MENU, I32_MAX, I32_MIN, INVALID, OUT_OF_RANGE, PAD, RESET, RUN, SENT32, SENT64, SKIP, SKIPPED, bind_tables

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_bound_streams.so")
CHUNK_PTS = 4096
SLOT_OOR, OFFSETS_OOR, STREAM_OOR, DUPLICATE = 4, 5, 6, 7
STREAM_GARBAGE = [I32_MIN, -1, I32_MAX]   # with num_streams and num_streams + 1, added per case
KINDS = {"plain": 0, "rings": 1, "packed": 2}
BASE = 0x7f0000001000


class Backend:
    """The three entry points of a kernel library (prefix simt_ or probe_) called with numpy arrays. The SIMT stand-in takes the
    host arrays as they are; the device probe takes device copies (to_device / back), every array copied back after each call."""

    def __init__(self, L, prefix, to_device=None, back=None):
        self.L, self.prefix, self.to_device, self.back = L, prefix, to_device, back
        self.sb = getattr(L, prefix + "stream_state_bytes")()
        self.rowb = getattr(L, prefix + "pwpp_state_bytes")()

    def __call__(self, name, *args):
        if self.to_device is None:
            conv = [a.ctypes.data if isinstance(a, np.ndarray) else a for a in args]
            getattr(self.L, self.prefix + name)(*conv)
            return
        dev = [self.to_device(a) if isinstance(a, np.ndarray) else None for a in args]
        conv = [d.data_ptr() if d is not None else a for a, d in zip(args, dev)]
        assert getattr(self.L, self.prefix + name)(*conv) == 0, f"{self.prefix}{name}: CUDA error"
        for a, d in zip(args, dev):
            if d is not None:
                self.back(a, d)


def declare(L, prefix):
    """The argument types of the entry points, the same for both libraries."""
    g = lambda n: getattr(L, prefix + n)   # noqa: E731
    g("stream_state_bytes").restype = C.c_int
    g("pwpp_state_bytes").restype = C.c_int
    g("bound_table_streams").argtypes = ([C.c_int, C.c_int] + [C.c_void_p] * 19 + [C.c_int, C.c_int] + [C.c_void_p] * 2 + [C.c_int] +
                                         [C.c_void_p] * 2 + [C.c_int64] + [C.c_void_p] * 2)
    g("bound_reset").argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 5
    g("bound_states_streams").argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    for n in ("bound_table_streams", "bound_reset", "bound_states_streams"):
        g(n).restype = C.c_int if prefix == "probe_" else None
    return L


def build_lib():
    """Same compile line as test_simt_bound_packed.py's library."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_bound_streams.cpp", "simt_records.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_bound_streams.cpp")])
    return declare(C.CDLL(LIB), "simt_")


@pytest.fixture(scope="module")
def lib():
    return Backend(build_lib(), "simt_")


def model(kind, counts, max_n, b_pset, actions, read, runs, num_streams, set_of, scratch, slots, ring_counts, offsets, capacity):
    """The rules of include/pwpp.h's stream-table block, frame by frame."""
    nf = len(read)
    acts = np.full(nf, RUN, np.int64) if actions is None else actions.astype(np.int64)
    runs_ = (acts == RUN) | (acts == RESET)
    v = np.where(runs_, 0, np.where(acts == SKIP, SKIPPED, INVALID))
    v = np.where(runs_ & (read < 0), SKIPPED, v)
    v = np.where(runs_ & (read >= num_streams), STREAM_OOR, v)
    for r in range(len(runs) - 1):
        seen = set()
        for f in range(runs[r], runs[r + 1]):
            if v[f] == 0:
                if read[f] in seen:
                    v[f] = DUPLICATE
                seen.add(int(read[f]))
    n = np.zeros(nf, np.int64)
    status = v.copy()
    slot_copy = np.full(nf, -1, np.int64)
    src = np.full(nf, BASE, np.int64)
    stride = 16 * max(1, int(max_n.max()) if nf else 1)
    for f in range(nf):
        if v[f]:
            continue
        bad = OUT_OF_RANGE
        if kind == 1:
            slot_copy[f] = s = int(slots[f])
            if 0 <= s < len(ring_counts):
                c = int(ring_counts[s])
                src[f] = BASE + s * stride
            else:
                c, bad = -1, SLOT_OOR
        elif kind == 2:
            lo, hi = int(offsets[f]), int(offsets[f + 1])
            c = hi - lo if 0 <= lo <= hi <= capacity else -1
            bad = OUT_OF_RANGE if c >= 0 else OFFSETS_OOR
            if 0 <= c <= max_n[f]:
                src[f] = BASE + lo * 16
        else:
            c = int(counts[f])
        ok = 0 <= c <= max_n[f]
        n[f] = c if ok else 0
        status[f] = 0 if ok else bad
    pt_off = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    chunk_off = np.concatenate([[0], np.cumsum((n + CHUNK_PTS - 1) // CHUNK_PTS)]).astype(np.int32)
    valid = (read >= 0) & (read < num_streams)
    sets = np.where(valid, set_of[np.where(valid, read, 0)], b_pset)
    stream = np.where(v == 0, read, scratch)
    act = np.where(runs_ & (v != 0), SKIP, acts)
    return dict(pt_off=pt_off, chunk_off=chunk_off, stream=stream.astype(np.int32), pset=sets.astype(np.int32), status=status.astype(np.int32),
                act=act.astype(np.int32), slot=slot_copy.astype(np.int32), src=src, accepted=v == 0, acts=acts)


def run(lib, kind, bound, read, actions=None, counts=None, max_n=None, set_of=None, slots=None, ring_counts=None, offsets=None, capacity=0):
    """One table launch, the reset launches of runs 1.. (with actions) and the state rows of every run, as pwpp_run_bound_call
    issues them with a stream table; every output word, the claim table and every state row are checked."""
    bound = np.asarray(bound, np.int64)
    nf = len(bound)
    num_streams = int(bound.max()) + 1 if set_of is None else len(set_of)
    set_of = np.ascontiguousarray(np.arange(num_streams) % 3 if set_of is None else set_of, np.int32)
    read_in = np.ascontiguousarray(read, np.int32)
    rng = np.random.default_rng(nf)
    max_n = np.ascontiguousarray(rng.integers(1, 9000, nf) if max_n is None else max_n, np.int64)
    counts = np.ascontiguousarray(rng.integers(-2, 9100, nf) if counts is None else counts, np.int64)
    runs, scratch, _ = bind_tables(bound.tolist(), num_streams)
    dep = np.ascontiguousarray(np.concatenate([np.full(runs[r + 1] - runs[r], int(r > 0)) for r in range(len(runs) - 1)]), np.int32)
    b_pset = np.ascontiguousarray(set_of[bound], np.int32)
    acts = None if actions is None else np.ascontiguousarray(actions, np.int32)
    slots = np.ascontiguousarray(np.zeros(nf) if slots is None else slots, np.int32)
    ring_counts = np.ascontiguousarray([0] if ring_counts is None else ring_counts, np.int64)
    offsets = np.ascontiguousarray(np.zeros(nf + 1) if offsets is None else offsets, np.int64)
    runs_arr = np.ascontiguousarray(runs, np.int32)
    sb = lib.sb
    nslots = num_streams + max(np.diff(runs))
    init = np.ascontiguousarray(((np.arange(nslots)[:, None] * 7 + np.arange(sb)[None, :]) % 251 + 1).astype(np.uint8))
    states = np.full((nslots + PAD, sb), 0x5A, np.uint8)
    out = [np.full(nf + 1 + PAD, SENT64, np.int64), np.full(nf + 1 + PAD, SENT32, np.int32)] + [np.full(nf + PAD, SENT32, np.int32) for _ in range(3)]
    act, read_copy, slot = (np.full(nf + PAD, SENT32, np.int32) for _ in range(3))
    claim = np.full(num_streams + PAD, -1, np.int32)
    claim[num_streams:] = SENT32
    brun = np.full((nf + PAD) * 48, 0x5A, np.uint8)
    lib("bound_table_streams", KINDS[kind], nf, counts, max_n, b_pset, *out, acts, act if acts is not None else None, scratch,
        dep if acts is not None else None, init, states, read_in, read_copy, claim, set_of, runs_arr, len(runs) - 1, num_streams, slots, slot,
        len(ring_counts), ring_counts, C.c_void_p(BASE), capacity, offsets, brun)
    w = model(KINDS[kind], counts, max_n, b_pset, acts, read_in.astype(np.int64), runs, num_streams, set_of, scratch, slots, ring_counts, offsets,
              capacity)
    for name, o in zip(("pt_off", "chunk_off", "stream", "pset", "status"), out):
        want = w[name]
        assert np.array_equal(o[:len(want)], want), f"{name}: first mismatch at {np.flatnonzero(o[:len(want)] != want)[:5]}"
        assert np.all(o[len(want):] == (SENT64 if o.dtype == np.int64 else SENT32)), f"{name}: a word after the table changed"
    assert np.array_equal(read_copy[:nf], read_in) and np.all(read_copy[nf:] == SENT32), "the read copy"
    assert np.all(claim[:num_streams] == -1) and np.all(claim[num_streams:] == SENT32), "the claim table is not all -1 after the kernel"
    if acts is not None:
        assert np.array_equal(act[:nf], w["act"]) and np.all(act[nf:] == SENT32), "the action copy"
    else:
        assert np.all(act == SENT32), "act was written without actions"
    if kind == "rings":
        assert np.array_equal(slot[:nf], w["slot"]) and np.all(slot[nf:] == SENT32), "the slot copy"
    if kind != "plain":
        rec = brun.reshape(-1, 48)
        got = rec[:nf, :8].copy().view(np.int64).reshape(-1)
        assert np.array_equal(got, w["src"]), f"brun src: first mismatch at {np.flatnonzero(got != w['src'])[:5]}"
        assert np.all(rec[nf:] == 0x5A), "a record after the table changed"
    # resets: run 0's by the table kernel, the later runs' by k_bound_reset from the read copy
    reset = np.zeros(nslots + PAD, bool)
    acc, a = w["accepted"], w["acts"]
    if acts is not None:
        r0 = acc[:runs[1]] & (a[:runs[1]] == RESET)
        reset[read_in[:runs[1]][r0]] = True
    check_states(states, init, reset, "table kernel")
    rows = np.full((nf + PAD, lib.rowb), 0x5A, np.uint8)
    valid = (read_in >= 0) & (read_in < num_streams)
    for r in range(len(runs) - 1):
        f0, f1 = runs[r], runs[r + 1]
        if acts is not None and r > 0:
            lib("bound_reset", f0, f1, act, dep, read_copy, init, states)
            sel = acc[f0:f1] & (a[f0:f1] == RESET)
            reset[read_in[f0:f1][sel]] = True
            check_states(states, init, reset, f"k_bound_reset of run {r}")
        lib("bound_states_streams", f0, f1, read_copy, num_streams, states, rows)
        v = valid[f0:f1]   # a row is its stream's state after the run (only the resets write states here)
        assert np.array_equal(rows[f0:f1][v, :8], states[read_in[f0:f1][v], :8]), f"state rows of run {r}"
    assert np.all(rows[:nf][~valid] == 0x5A), "a state row of a hole or an out-of-range id was written"
    assert np.all(rows[nf:] == 0x5A), "a state row after the table changed"
    return w


def check_states(states, init, reset, who):
    rows = len(init)
    got_init = np.all(states[:rows] == init, axis=1)
    assert np.array_equal(got_init, reset[:rows]), f"{who}: streams reset {np.flatnonzero(got_init)[:8]}, want {np.flatnonzero(reset[:rows])[:8]}"
    assert np.all(np.all(states[:rows] == 0x5A, axis=1) | got_init), f"{who}: a state row was partly written"
    assert np.all(states[rows:] == 0x5A), f"{who}: a row after the state array changed"


def garbage(ns):
    return STREAM_GARBAGE + [ns, ns + 1]


def schedule(rng, bound, ns, p_bad=0.15, p_dup=0.15):
    """A scheduler's pick over the bound shape: distinct streams from ns, with holes, out-of-range ids and duplicates mixed in."""
    nf = len(bound)
    read = rng.permutation(ns)[:nf] if nf <= ns else rng.integers(0, ns, nf)
    u = rng.random(nf)
    read = np.where(u < p_bad, rng.choice(garbage(ns), nf), read)
    dup = (u >= p_bad) & (u < p_bad + p_dup) & (np.arange(nf) > 0)
    read[dup] = read[np.maximum(np.flatnonzero(dup) - rng.integers(1, 4, dup.sum()), 0)]
    return read


SHAPES = {"one_run": np.arange(64), "backlog": np.concatenate([np.arange(64), np.arange(32)]), "repeat": np.zeros(9, np.int64),
          "wide_odd_runs": np.concatenate([np.arange(601), np.arange(600), np.arange(302)]),   # 2 frames per thread, runs at 601, 1201
          "runs_of_7": np.arange(2100) % 7}                                                      # 3 frames per thread, runs of 7
SHAPE_STREAMS = {"one_run": 256, "backlog": 256, "repeat": 5, "wide_odd_runs": 1000, "runs_of_7": 9}


def slices_crossing_runs(bound):
    """How many threads of the one-CTA table kernel own a slice of frames that spans a run boundary."""
    nf = len(bound)
    runs, _, _ = bind_tables(list(bound), int(max(bound)) + 1)
    per = (nf + 1023) // 1024
    return sum(1 for t in range(1024) for b in runs[1:-1] if t * per < b < min(t * per + per, nf))


def test_wide_shapes_cross_run_boundaries_inside_slices():
    """The wide shapes do what they are there for: some thread's slice holds the end of one run and the start of the next."""
    assert slices_crossing_runs(SHAPES["wide_odd_runs"]) == 2
    assert slices_crossing_runs(SHAPES["runs_of_7"]) > 100


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("with_actions", [False, True], ids=["no_actions", "actions"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_schedules(lib, kind, with_actions, shape):
    """Seeded schedules over five shapes: one run of 64; a 64 + 32 backlog (two runs); a repeat table (runs of length 1); 1503
    frames in three runs starting at odd positions and 2100 frames in runs of 7, so that thread slices (2 and 3 frames) span run
    boundaries. Every action of the menu with every stream case; behind an invalid stream, invalid slots or offsets."""
    schedules(lib, kind, with_actions, shape)


def schedules(lib, kind, with_actions, shape):
    rng = np.random.default_rng(sum(map(ord, kind + shape)) + with_actions)
    bound = SHAPES[shape]
    nf = len(bound)
    ns = SHAPE_STREAMS[shape]
    set_of = rng.integers(0, 4, ns)
    for tick in range(3):
        read = schedule(rng, bound, ns)
        actions = rng.choice(ACTION_MENU, nf, p=[0.5, 0.15, 0.2, 0.05, 0.04, 0.03, 0.03]) if with_actions else None
        kw = {}
        if kind == "rings":
            kw = dict(slots=rng.choice([0, 1, 2, 3, -1, 4, I32_MAX], nf), ring_counts=rng.integers(-1, 9000, 4))
        elif kind == "packed":
            cap = 20 * nf
            cuts = np.sort(rng.integers(0, cap + 1, nf + 1))
            cuts[rng.integers(0, nf + 1, max(1, nf // 10))] = rng.choice([-1, cap + 1, 2 ** 62], max(1, nf // 10))
            kw = dict(offsets=cuts, capacity=cap, max_n=np.full(nf, 60))
        run(lib, kind, bound, read, actions, set_of=set_of, **kw)


def test_duplicates_first_occurrence_skipped_by_action(lib):
    """Stream 3 named by frames 0, 1 and 2 of one run: frame 0 skipped by its action, so frame 1 wins and frame 2 is the duplicate;
    across runs the same stream is not a duplicate."""
    bound = [0, 1, 2, 3, 0, 1]
    w = run(lib, "plain", bound, [3, 3, 3, 1, 3, 3], actions=[SKIP, RESET, RUN, RUN, RESET, RUN], counts=[5, 6, 7, 8, 9, 10],
            max_n=[100] * 6, set_of=np.arange(4))
    assert w["status"].tolist() == [SKIPPED, 0, DUPLICATE, 0, 0, DUPLICATE]
    w = run(lib, "plain", bound, [3, 3, 3, 1, 3, 3], actions=None, counts=[5, 6, 7, 8, 9, 10], max_n=[100] * 6, set_of=np.arange(4))
    assert w["status"].tolist() == [0, DUPLICATE, DUPLICATE, 0, 0, DUPLICATE]


@pytest.mark.parametrize("kind", list(KINDS))
def test_every_action_with_every_stream_case(lib, kind):
    """The product of the action menu and the stream cases (valid, hole, each garbage id, duplicate), one pair per frame."""
    ns = 50
    cases = ["valid", "dup"] + garbage(ns)
    pairs = [(a, c) for a in ACTION_MENU for c in cases]
    nf = len(pairs)
    bound = np.arange(nf) % ns   # runs of 50
    read, actions = [], []
    for f, (a, c) in enumerate(pairs):
        actions.append(a)
        read.append(f % ns if c == "valid" else (read[-1] if c == "dup" and f % ns else 7) if c == "dup" else c)
    kw = {}
    if kind == "rings":
        kw = dict(slots=np.arange(nf) % 3 - 1, ring_counts=[10, 20])
    elif kind == "packed":
        kw = dict(offsets=np.arange(nf + 1) * 3 - 2, capacity=3 * nf, max_n=np.full(nf, 5))
    run(lib, kind, bound, read, actions, set_of=np.arange(ns) % 4, **kw)


def test_identity_matches_bound_streams(lib):
    """d_streams equal to the bound streams: every frame accepted on its bound stream and set, nothing flagged."""
    bound = np.concatenate([np.arange(40), np.arange(10)])
    w = run(lib, "plain", bound, bound, actions=None, set_of=np.arange(40) % 3)
    assert not np.isin(w["status"], [SKIPPED, STREAM_OOR, DUPLICATE]).any()
    assert np.array_equal(w["stream"], bound) and np.array_equal(w["pset"], (np.arange(40) % 3)[bound])


def test_all_holes(lib):
    """Every frame a hole: every frame skipped to its scratch slot, no state touched, no row written."""
    nf = 1100
    run(lib, "plain", np.arange(nf), np.full(nf, -1), actions=np.full(nf, RESET, np.int32), set_of=np.arange(nf) % 2)
