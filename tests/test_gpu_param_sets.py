"""Several parameter sets in one context (pwpp_create_sets) on the GPU.

Every stream of a multi-set context must compute, bit for bit, what a one-set context built from its own set computes on the
same frames with the same call shape, and every frame must match the CANON64 oracle run with its stream's set. The sets are the
three of tests/param_sets.py plus a geometry the fp32 binning filter does not cover (1.2 m rings in zone 0), assigned to eight
streams interleaved. The comparison context for set k is a one-set context of eight streams all on set k, given the very same
calls: the frame count, frame sizes and stream table of a call are what select its kernels (tests/test_gpu_edges.py), so both
contexts run the same kernels on every frame of set k. Call shapes: a batch call (cluster front end), one-frame calls made twice
each (the second replays the small-call graph), a stream-table call with repeated streams, and a batch above 400k points per
frame (dense cluster kernel); each asserts the launch rules that select its kernels."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_py as O
from param_sets import PARAM_SETS
from test_gpu_parity import compare_frame

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
NAMES = ["default", "ros", "no_rvpf_tgr", "narrow_rings"]
STREAM_SET = [0, 1, 2, 3, 0, 1, 2, 3]


def _tuning(name):
    for line in open(os.path.join(REPO, "patchwork-plusplus_b200", "csrc", "pwpp_tuning.h")):
        if line.startswith(f"#define {name} "):
            return int(line.split()[2])
    raise KeyError(name)


SMALL_CALL = _tuning("PWPP_SMALL_CALL_DEFAULT")
DENSE_MEAN = 400000     # mean frame size of a launch range above which the dense cluster kernel runs (pwpp_capi.cu)


def narrow_rings():
    p = PARAM_SETS["default"][0]()
    p.num_rings_each_zone[:] = [8, 4, 4, 4]   # zone 0: 1.2 m rings
    p.sensor_height = 1.9
    return p


def make_set(name):
    return narrow_rings() if name == "narrow_rings" else PARAM_SETS[name][0]()


def fp32_filter_ok(p):
    """build_geometry (csrc/pwpp_host.hpp): the fp32 binning filter covers the set's geometry."""
    lo, hi = p.min_range, p.max_range
    z = [lo, (7 * lo + hi) / 8, (3 * lo + hi) / 4, (lo + hi) / 2, hi]
    return hi <= 250 and all((z[k + 1] - z[k]) / p.num_rings_each_zone[k] >= 1.5 and p.num_sectors_each_zone[k] <= 128 for k in range(4))


def launch_ranges(streams, sizes):
    """The launch ranges of one pwpp_estimate_host call of one pipeline chunk: maximal runs of frames with distinct streams.
    Per range: (frames, small-call kernels, dense cluster kernel, fp32 binning filter)."""
    out, run = [], []
    for f, s in enumerate(streams):
        if s in [streams[g] for g in run]:
            out.append(run); run = []
        run.append(f)
    out.append(run)
    sets = [make_set(n) for n in NAMES]
    return [(len(r), len(r) <= SMALL_CALL, np.mean([sizes[f] for f in r]) > DENSE_MEAN, all(fp32_filter_ok(sets[STREAM_SET[streams[f]]]) for f in r))
            for r in out]


def engines(order):
    import pwpp_b200
    multi = pwpp_b200.Engine([make_set(n) for n in NAMES], device=0, num_streams=8, stream_set=STREAM_SET)
    ones = [pwpp_b200.Engine(make_set(n), device=0, num_streams=8) for n in NAMES]
    for e in [multi] + ones:
        e.set_output_order(order)
    return multi, ones


def snapshot(eng, s):
    return bytes(eng.state(s)) + b"".join(eng.history(s, r, w).tobytes() for r in range(4) for w in (0, 1))


def assert_same(multi, one, f, s, what):
    """Frame f (stream s) of the last call: the multi-set context against the one-set context of the stream's set."""
    nb = multi.stream_num_bins(s)
    assert nb == one.nbins, what
    assert np.array_equal(multi.bin_ids(f), one.bin_ids(f)), f"{what}: bin ids"
    assert np.array_equal(multi.ground_indices(f), one.ground_indices(f)), f"{what}: ground list"
    assert np.array_equal(multi.nonground_indices(f), one.nonground_indices(f)), f"{what}: non-ground list"
    assert bytes(multi.bin_results(f)) == bytes(one.bin_results(f)), f"{what}: patch records"
    assert multi.num_patches(f) == one.num_patches(f), f"{what}: patch count"
    assert multi.centers(f).tobytes() == one.centers(f).tobytes(), f"{what}: centers"
    assert multi.normals(f).tobytes() == one.normals(f).tobytes(), f"{what}: normals"
    assert snapshot(multi, s) == snapshot(one, s), f"{what}: state / histories"


class Oracles:
    """The CANON64 oracle of every stream, with its set, fed the stream's frames in order. A stream stops being compared in full
    after a frame with degenerate patches (the `ros` set fits patches of one point: ill-conditioned planes, after which the
    states may legitimately part), as in tests/test_gpu_parity.py."""

    def __init__(self):
        self.orc = {s: O.Oracle(make_set(NAMES[STREAM_SET[s]]), O.ARITH_CANON64) for s in range(8)}
        self.clean = {s: True for s in range(8)}
        self.compared = 0

    def check(self, eng, f, s, a, what):
        self.orc[s].estimate(a)
        if self.clean[s]:
            nd = compare_frame(eng, f, self.orc[s], a, what, min_pts_floor=5 if NAMES[STREAM_SET[s]] == "ros" else 0)
            self.clean[s] = nd == 0
            self.compared += 1


def run_call(multi, ones, streams, frames, orcs, what):
    multi.estimate_host(frames, streams=streams)
    for one in ones:
        one.estimate_host(frames, streams=streams)
    for f, s in enumerate(streams):
        k = STREAM_SET[s]
        assert_same(multi, ones[k], f, s, f"{what} frame {f} (stream {s}, set {NAMES[k]})")
        if orcs is not None:
            orcs.check(multi, f, s, frames[f], f"{what} frame {f} (stream {s}, set {NAMES[k]}) vs oracle")


@pytest.fixture(scope="module")
def dense(kitti):
    return [np.concatenate([kitti[(i + j) % 6] for j in range(4)]) for i in range(4)]


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
def test_every_stream_equals_its_one_set_context_and_the_oracle(kitti, dense, order):
    multi, ones = engines(order)
    orcs = Oracles() if order == 0 else None
    sizes = lambda fr: [len(a) for a in fr]   # noqa: E731
    # 1. batch call, every stream once: one range of 8 frames on the cluster front end, exact binning (the narrow set is in it)
    streams, frames = list(range(8)), [kitti[s % 6] for s in range(8)]
    assert launch_ranges(streams, sizes(frames)) == [(8, False, False, False)]
    run_call(multi, ones, streams, frames, orcs, "batch")
    # 2. one-frame calls, each twice (the second replays the small-call graph); the graph key follows the binning kernel
    for rep in range(2):
        for s in range(8):
            fr = [kitti[(s + 1 + rep) % 6]]
            assert launch_ranges([s], sizes(fr)) == [(1, True, False, NAMES[STREAM_SET[s]] != "narrow_rings")]
            run_call(multi, ones, [s], fr, orcs, f"one-frame rep {rep} stream {s}")
    # 3. stream table with repeated streams: a run of two frames (small call, fp32 filter) and a mixed run of six that falls
    #    back to the exact front end
    streams = [0, 5, 0, 3, 5, 2, 7, 1]
    frames = [kitti[(3 + f) % 6] for f in range(8)]
    assert launch_ranges(streams, sizes(frames)) == [(2, True, False, True), (6, False, False, False)]
    run_call(multi, ones, streams, frames, orcs, "stream table")
    # 4. frames above 400k points: the dense cluster kernel, fp32 filter (no narrow-ring stream named)
    streams = [0, 1, 2, 4, 5]
    frames = [dense[f % 4] for f in range(5)]
    assert launch_ranges(streams, sizes(frames)) == [(5, False, True, True)]
    run_call(multi, ones, streams, frames, orcs, "dense")
    if orcs is not None:
        # the default-set stream that starts on a recorded scan has no degenerate patch in any call: compared in full throughout
        assert orcs.clean[0], orcs.clean
        assert orcs.compared >= 20, orcs.compared


def test_one_set_equals_pwpp_create(kitti):
    """pwpp_create_sets with one set is pwpp_create, bit for bit."""
    import pwpp_b200
    p = make_set("default")
    a = pwpp_b200.Engine([p], device=0, num_streams=3, stream_set=[0, 0, 0])
    b = pwpp_b200.Engine(p, device=0, num_streams=3)
    assert a.nbins == b.nbins == a.stream_num_bins(2)
    for call in ([0, 1, 2], [2], [1, 1, 0]):
        frames = [kitti[(s + len(call)) % 6] for s in call]
        a.estimate_host(frames, streams=call)
        b.estimate_host(frames, streams=call)
        for f, s in enumerate(call):
            assert_same(a, b, f, s, f"call {call} frame {f}")
            assert len(a.export_state(s)) == len(b.export_state(s))


def test_reset_storage_bound_and_state_blobs(kitti):
    """Reset restores each stream's own set; each set keeps its own storage bound; blobs move between multi- and one-set contexts
    of the same parameters, and are refused by a stream whose history capacity differs."""
    import pwpp_b200
    multi, ones = engines(0)
    fresh = {s: snapshot(multi, s) for s in range(8)}
    for s in range(8):
        st, p = multi.state(s), make_set(NAMES[STREAM_SET[s]])
        assert st.sensor_height == p.sensor_height and list(st.elevation_thr) == list(p.elevation_thr), s
        assert multi.stream_set[s] == STREAM_SET[s] == int(multi.lib.pwpp_stream_set(multi._h, s))
    # ten batch calls: the no_rvpf_tgr streams (max_*_storage 40 / 50) trim their histories, the default ones (1000) do not
    for t in range(10):
        frames = [kitti[(s + t) % 6] for s in range(8)]
        run_call(multi, ones, list(range(8)), frames, None, f"tick {t}")
    small = [s for s in range(8) if NAMES[STREAM_SET[s]] == "no_rvpf_tgr"]
    big = [s for s in range(8) if NAMES[STREAM_SET[s]] == "default"]
    for s in small:
        st = multi.state(s)
        assert max(st.n_elevation) == 50 and max(st.n_flatness) <= 40, (s, list(st.n_elevation), list(st.n_flatness))
    for s in big:
        assert max(multi.state(s).n_elevation) > 50, s
    # blob of a multi-set stream -> one-set context with the same parameters: the continuation is bit-identical
    s = small[0]
    blob = multi.export_state(s)
    solo = pwpp_b200.Engine(make_set("no_rvpf_tgr"), device=0, num_streams=1)
    assert len(blob) == multi.lib.pwpp_stream_state_blob_size(multi._h, s) == solo.lib.pwpp_state_blob_size(solo._h)
    assert multi.lib.pwpp_state_blob_size(multi._h) > len(blob)   # the largest set's blob
    solo.import_state(0, blob)
    twin = pwpp_b200.Engine(make_set("no_rvpf_tgr"), device=0, num_streams=1)
    twin.import_state(0, ones[2].export_state(s))
    a = kitti[5]
    multi.estimate_host([a], streams=[s]); solo.estimate_host([a]); twin.estimate_host([a])
    assert np.array_equal(multi.ground_indices(0), solo.ground_indices(0))
    assert bytes(multi.bin_results(0)) == bytes(solo.bin_results(0)) == bytes(twin.bin_results(0))
    assert multi.export_state(s) == solo.export_state(0)
    # and back: a one-set blob into the multi-set stream
    multi.import_state(small[1], solo.export_state(0))
    assert snapshot(multi, small[1]) == snapshot(solo, 0)
    # a stream whose set has another history capacity refuses it
    with pytest.raises(pwpp_b200.PwppError):
        multi.import_state(big[0], blob)
    # reset: every stream back to its own set's constructor state
    multi.reset(small[0])
    assert snapshot(multi, small[0]) == fresh[small[0]]
    multi.reset()
    assert all(snapshot(multi, s) == fresh[s] for s in range(8))


def test_invalid_arguments_fail_before_allocation():
    """num_sets outside [1, 8], a NULL or out-of-range stream_set, or an invalid set: an error naming the problem, no context."""
    import pwpp_b200
    from pwpp_ctypes import PwppParams
    lib = pwpp_b200.load_library()
    sets = (PwppParams * 9)(*[make_set("default") for _ in range(9)])
    ok = (C.c_int32 * 4)(0, 1, 2, 0)

    def create(n, table, k=4):
        h = C.c_void_p(123)
        rc = lib.pwpp_create_sets(sets, n, table, 0, k, 0, C.byref(h))
        assert h.value is None, "no context on failure"
        return rc, lib.pwpp_last_error().decode()

    for n in (0, 9, -1):
        rc, msg = create(n, ok)
        assert rc == -1 and "num_sets" in msg, (n, msg)
    rc, msg = create(3, None)
    assert rc == -1 and "stream_set" in msg, msg
    rc, msg = create(3, (C.c_int32 * 4)(0, 1, 3, 0))
    assert rc == -1 and "stream 2" in msg and "set 3" in msg, msg
    rc, msg = create(3, (C.c_int32 * 4)(0, -1, 0, 0))
    assert rc == -1 and "stream 1" in msg, msg
    sets[2].num_zones = 3
    rc, msg = create(3, ok)
    assert rc == -4 and "parameter set 2" in msg, msg
    sets[2].num_zones = 4
    sets[1].min_range = 90.0
    rc, msg = create(3, ok)
    assert rc == -1 and "parameter set 1" in msg, msg
