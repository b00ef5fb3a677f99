"""Bound calls (pwpp_bind_call / pwpp_run_bound_call): frame sizes read on the GPU, no host synchronisation, capturable into the
caller's CUDA graph.

Every result is compared bit for bit with a twin context created identically and driven by pwpp_estimate_device_records with
the same frames and the counts as host sizes (0 for an out-of-range count): bin ids, index lists, centers, normals, xyz,
patch records, state and histories, in both output orders (each bound separately). Frames live in device buffers of their
capacity, 1..15 bytes past an allocation's base; counts in an int64 CUDA tensor that is rewritten in place between runs."""
import ctypes as C

import numpy as np
import pytest

from param_sets import _default, _no_rvpf_tgr, _ros
from test_gpu_records import LAYOUTS, outputs, records, stream

pytestmark = pytest.mark.gpu

NAMES = ["xyzi16", "velodyne22", "pcl_xyzi32", "f64_xyz"]   # float4-16, a 22-byte record, PCL's 32 bytes, FLOAT64 x/y/z
ERR_INVALID_ARG, ERR_CAPACITY = -1, -5


def engine(num_streams, order, sets=None):
    import pwpp_b200
    if sets is None:
        e = pwpp_b200.Engine(device=0, num_streams=num_streams)
    else:
        e = pwpp_b200.Engine(sets, device=0, num_streams=num_streams, stream_set=list(range(num_streams)))
    e.set_output_order(order)
    return e


class Pair:
    """A bound context and its twin. Frame f is a device buffer of max_n[f] records of layout names[f]."""

    def __init__(self, streams, names, max_n, order=0, num_streams=None, sets=None):
        import torch
        import pwpp_b200
        ns = num_streams or (max(streams) + 1)
        self.streams, self.names, self.max_n = list(streams), list(names), [int(k) for k in max_n]
        self.eng, self.twin = engine(ns, order, sets), engine(ns, order, sets)
        self.lays = [pwpp_b200.layout_from_dtype(LAYOUTS[nm]) for nm in names]
        self.bufs, self.ptrs = [], []
        for f, (nm, m) in enumerate(zip(names, self.max_n)):
            mis = 1 + (5 * f) % 15
            t = torch.empty(mis + m * LAYOUTS[nm].itemsize, dtype=torch.uint8, device="cuda")
            self.bufs.append((t, mis))
            self.ptrs.append(t.data_ptr() + mis)
        self.counts = torch.zeros(len(streams), dtype=torch.int64, device="cuda")
        self.eng.bind_call(self.ptrs, self.max_n, self.lays, self.counts, streams=self.streams)

    def load(self, scans, seed, counts=None):
        """Writes frame f = a record array of scans[(f + seed) % len] (cut to its capacity) and the counts (default: the records
        written); returns the sizes the twin runs with."""
        import torch
        self.data = []
        for f, nm in enumerate(self.names):
            a = scans[(f + seed) % len(scans)][: self.max_n[f]]
            r, _ = records(a, LAYOUTS[nm], seed=seed * 100 + f)
            t, mis = self.bufs[f]
            if len(r):
                t[mis: mis + r.nbytes] = torch.from_numpy(r.view(np.uint8).copy()).cuda()
            self.data.append(r)
        c = np.array([len(r) for r in self.data] if counts is None else counts, np.int64)
        self.counts.copy_(torch.from_numpy(c))
        torch.cuda.synchronize()
        return [int(k) if 0 <= k <= m else 0 for k, m in zip(c, self.max_n)]

    def run_twin(self, sizes):
        self.twin.estimate_device_records(self.ptrs, sizes, self.lays, streams=self.streams)
        self.twin.synchronize()

    def check(self, sizes, what):
        """The bound call's results (after bound_call_results) against the twin's last call, and every stream's state."""
        idx, off, ng, st = self.eng.bound_call_results()
        self.eng.synchronize()
        assert np.array_equal(off.cpu().numpy(), np.concatenate([[0], np.cumsum(sizes)])), f"{what}: offsets"
        want_st = [0 if 0 <= k <= m else 1 for k, m in zip(self.counts.cpu().numpy(), self.max_n)]
        assert st.cpu().numpy().tolist() == want_st, f"{what}: status"
        nf = len(self.streams)
        assert np.array_equal(ng.cpu().numpy(), [self.twin.num_ground(f) for f in range(nf)]), f"{what}: num_ground"
        for f in range(nf):
            assert outputs(self.eng, f) == outputs(self.twin, f), f"{what}: frame {f}"
        for s in sorted(set(self.streams)):
            assert stream(self.eng, s) == stream(self.twin, s), f"{what}: stream {s}"

    def step(self, scans, seed, what, counts=None):
        """One eager run on the ctx's stream, the twin's call, and the comparison."""
        sizes = self.load(scans, seed, counts)
        self.eng.run_bound_call()
        self.run_twin(sizes)
        self.check(sizes, what)
        return sizes


@pytest.fixture(scope="module")
def scans(kitti):
    return list(kitti)


def big(scans, k, n):
    """A dense frame of n points: KITTI scans stacked (shifted apart in x so they do not overlap exactly)."""
    parts, i = [], 0
    while sum(len(p) for p in parts) < n:
        a = scans[(k + i) % len(scans)].copy()
        a[:, 0] += 0.37 * i
        parts.append(a)
        i += 1
    return np.ascontiguousarray(np.concatenate(parts)[:n])


CASES = {
    # name: (streams, capacities as a function of the scan sizes, repeat count)
    "one_frame": ([0], lambda sz: [sz + 1000]),
    "four_frames": ([0, 1, 2, 3], lambda sz: [sz + 7 * k for k in range(4)]),
    "five_frames": ([4, 0, 3, 1, 2], lambda sz: [sz] * 5),
    "stream_table_with_repeats": ([2, 0, 2, 1, 3, 0, 1], lambda sz: [sz + 4096] * 7),
    "sixty_four_frames": (list(range(64)), lambda sz: [sz + 13 * k for k in range(64)]),
    "dense_capacities_small_counts": (list(range(8)), lambda sz: [600000] * 8),
}


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
@pytest.mark.parametrize("case", list(CASES))
def test_direct_runs_equal_the_twin(scans, case, order):
    """Three runs with state carried; layouts mixed within the call. The dense-capacities case runs the dense cluster front end
    on frames of KITTI size, whose twin call takes the regular one."""
    streams, caps = CASES[case]
    sz = max(len(a) for a in scans)
    names = [NAMES[f % len(NAMES)] for f in range(len(streams))]
    p = Pair(streams, names, caps(sz), order)
    for run in range(3):
        p.step(scans, run, f"{case} run {run}")


def test_dense_counts_and_capacities(scans):
    """Frames of 450 000 to 500 000 points: bound call and twin both on the dense front end."""
    dense = [big(scans, k, 450000 + 25000 * k) for k in range(3)]
    p = Pair(list(range(3)), NAMES[:3], [500000] * 3)
    for run in range(2):
        p.step(dense, run, f"run {run}")


def test_four_parameter_sets(scans):
    sets = [_default(), _ros(), _no_rvpf_tgr(), _default()]
    sets[3].sensor_height = 1.6
    sz = max(len(a) for a in scans)
    p = Pair([3, 1, 0, 2, 1], ["xyzi16", "velodyne22", "pcl_xyzi32", "f64_xyz", "xyzi16"], [sz] * 5, num_streams=4, sets=sets)
    for run in range(2):
        p.step(scans, run, f"run {run}")


def test_out_of_range_counts_run_as_empty_frames(scans):
    """Counts of -1 and max_n + 1 in frames 1 and 3: those frames equal the twin's n = 0 frames, their streams advance as after
    an empty call, status flags exactly them, and every other frame is unchanged."""
    sz = max(len(a) for a in scans)
    p = Pair([0, 1, 2, 3, 4], NAMES + ["xyzi16"], [sz] * 5)
    for run in range(2):
        counts = [len(scans[(f + run) % 6]) for f in range(5)]
        counts[1], counts[3] = -1, sz + 1
        sizes = p.step(scans, run, f"run {run}", counts=counts)
        assert sizes[1] == sizes[3] == 0
        assert p.eng.bound_call_results()[3].cpu().numpy().tolist() == [0, 1, 0, 1, 0]


def test_graph_capture_and_replays(scans):
    """run_bound_call captured once by torch.cuda.graph (global capture mode), replayed 8 times with new frames and counts
    written into the same tensors; state carries across replays and matches the twin after each. A direct call that fits the
    frozen buffers between two replays runs as usual, and the replays after it stay right."""
    import torch
    sz = max(len(a) for a in scans)
    p = Pair([0, 1, 2, 3, 0], NAMES + ["velodyne22"], [sz + 100] * 5, order=1)
    p.step(scans, 0, "eager run before the capture")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        p.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    for rep in range(8):
        counts = None if rep != 5 else [len(scans[(f + rep + 1) % 6]) // 2 for f in range(5)]
        sizes = p.load(scans, rep + 1, counts)
        g.replay()
        torch.cuda.synchronize()
        p.run_twin(sizes)
        p.check(sizes, f"replay {rep}")
        if rep == 3:   # a direct call of two frames that fits the buffers, on both contexts
            data = [records(scans[k], LAYOUTS["xyzi16"], seed=k)[0] for k in (4, 5)]
            bufs = [torch.from_numpy(r.view(np.uint8).copy()).cuda() for r in data]
            torch.cuda.synchronize()
            for e in (p.eng, p.twin):
                e.estimate_device_records([b.data_ptr() for b in bufs], [len(r) for r in data], p.lays[:1] * 2, streams=[1, 3])
                e.synchronize()
            for f in range(2):
                assert outputs(p.eng, f) == outputs(p.twin, f), f"direct call frame {f}"
            torch.cuda.synchronize()


def test_no_host_synchronisation(scans):
    """With a long sleep kernel ahead on the stream, run_bound_call and a graph replay return while the stream is still busy."""
    import torch
    sz = max(len(a) for a in scans)
    p = Pair([0, 1], ["xyzi16", "velodyne22"], [sz] * 2)
    p.step(scans, 0, "eager run")   # every kernel loaded before the timing-sensitive part
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda._sleep(2_000_000_000)
        p.eng.run_bound_call(st.cuda_stream)
        assert not st.query(), "run_bound_call waited for the stream"
    st.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        p.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    with torch.cuda.stream(st):
        torch.cuda._sleep(2_000_000_000)
        g.replay()
        assert not st.query(), "the replay waited"
    st.synchronize()
    torch.cuda.synchronize()


def test_freeze_and_validation(scans):
    import torch
    import pwpp_b200
    sz = max(len(a) for a in scans)
    p = Pair([0, 1], ["xyzi16", "pcl_xyzi32"], [sz, sz])
    p.step(scans, 0, "first run")

    # launch count: one table launch, one unpack, the twin's sequence without its unpack
    p.load(scans, 1)
    l0 = p.eng.launch_count()
    p.eng.run_bound_call()
    m0 = p.twin.launch_count()
    p.run_twin([len(r) for r in p.data])
    assert p.eng.launch_count() - l0 == 1 + 1 + (p.twin.launch_count() - m0 - 1)
    p.check([len(r) for r in p.data], "second run")

    # the record results refuse a bound call, with a message
    with pytest.raises(pwpp_b200.PwppError, match="bound call"):
        p.eng.device_record_lists()
    with pytest.raises(pwpp_b200.PwppError, match="bound call"):
        p.eng.ground_records(0)

    # a direct call larger than the frozen buffers: PWPP_ERR_CAPACITY, no state change; after unbinding it runs
    big_frames = [big(scans, k, 3 * sz) for k in range(2)]
    data = [records(a, LAYOUTS["xyzi16"], seed=k)[0] for k, a in enumerate(big_frames)]
    bufs = [torch.from_numpy(r.view(np.uint8).copy()).cuda() for r in data]
    torch.cuda.synchronize()
    before = [stream(p.eng, s) for s in range(2)]
    l0 = p.eng.launch_count()
    args = ([b.data_ptr() for b in bufs], [len(r) for r in data], [p.lays[0]] * 2)
    with pytest.raises(pwpp_b200.PwppError, match=f"error {ERR_CAPACITY}"):
        p.eng.estimate_device_records(*args, streams=[0, 1])
    assert p.eng.launch_count() == l0 and [stream(p.eng, s) for s in range(2)] == before
    with pytest.raises(pwpp_b200.PwppError, match=f"error {ERR_CAPACITY}"):
        p.eng.estimate_host([big_frames[0]])
    assert [stream(p.eng, s) for s in range(2)] == before

    # the output order is frozen too
    with pytest.raises(pwpp_b200.PwppError, match=f"error {ERR_INVALID_ARG}"):
        p.eng.set_output_order(1)

    # binding twice is refused; after unbinding, the large call runs and equals the twin's
    with pytest.raises(pwpp_b200.PwppError, match="already bound"):
        p.eng.bind_call(p.ptrs, p.max_n, p.lays, p.counts, streams=p.streams)
    p.eng.unbind_call()
    with pytest.raises(pwpp_b200.PwppError, match="no call is bound"):
        p.eng.run_bound_call()
    for e in (p.eng, p.twin):
        e.estimate_device_records(*args, streams=[0, 1])
        e.synchronize()
    for f in range(2):
        assert outputs(p.eng, f) == outputs(p.twin, f)
    for s in range(2):
        assert stream(p.eng, s) == stream(p.twin, s)
    p.eng.set_output_order(1)


def test_bind_errors_name_the_frame(scans):
    import torch
    import pwpp_b200
    e = engine(4, 0)
    lay = pwpp_b200.layout_from_dtype(LAYOUTS["xyzi16"])
    buf = torch.zeros(16 * 1000, dtype=torch.uint8, device="cuda")
    counts = torch.zeros(4, dtype=torch.int64, device="cuda")
    ptrs, max_n, lays = [buf.data_ptr()] * 4, [1000] * 4, [lay] * 4

    def bind(streams=(0, 1, 2, 3), ptrs=ptrs, max_n=max_n, lays=lays, counts_ptr=None):
        nf = len(streams)
        ids = np.ascontiguousarray(streams, np.int32)
        p = (C.c_void_p * nf)(*ptrs)
        n = (C.c_int64 * nf)(*max_n)
        ly = (pwpp_b200.PwppPointLayout * nf)(*lays)
        rc = e.lib.pwpp_bind_call(e._h, nf, ids.ctypes.data, p, n, ly, C.c_void_p(counts.data_ptr() if counts_ptr is None else counts_ptr))
        return rc, e.lib.pwpp_last_error().decode()

    rc, msg = bind(streams=(0, 1, 7, 2))
    assert rc == ERR_INVALID_ARG and "frame 2" in msg
    bad = pwpp_b200.PwppPointLayout()
    C.memmove(C.byref(bad), C.byref(lay), C.sizeof(lay))
    bad.offset[2] = 14
    rc, msg = bind(lays=[lay, lay, lay, bad])
    assert rc == ERR_INVALID_ARG and "frame 3" in msg and "field z" in msg
    rc, msg = bind(ptrs=[ptrs[0], None, ptrs[0], ptrs[0]])
    assert rc == ERR_INVALID_ARG and "frame 1" in msg
    rc, msg = bind(max_n=[1000, 1000, -1, 1000])
    assert rc == ERR_INVALID_ARG and "frame 2" in msg
    rc, msg = bind(max_n=[1000, 2 ** 31, 1000, 1000])
    assert rc == ERR_INVALID_ARG and "frame 1" in msg
    rc, msg = bind(counts_ptr=0)
    assert rc == ERR_INVALID_ARG and "d_counts" in msg
    nf = 4
    for which in range(4):   # NULL streams / frames / max_n / layouts
        args = [np.zeros(4, np.int32).ctypes.data, (C.c_void_p * nf)(*ptrs), (C.c_int64 * nf)(*max_n), (pwpp_b200.PwppPointLayout * nf)(*lays)]
        args[which] = None
        assert e.lib.pwpp_bind_call(e._h, nf, *args, C.c_void_p(counts.data_ptr())) == ERR_INVALID_ARG
    # nothing is bound after the failures: a valid bind succeeds, with a max_n = 0 frame that may have a NULL pointer
    rc, msg = bind(ptrs=[ptrs[0], 0, ptrs[0], ptrs[0]], max_n=[1000, 0, 1000, 1000])
    assert rc == 0, msg
