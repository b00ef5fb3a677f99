"""Width ladders of bound calls (pwpp_bind_width_ladder): at every run or replay the GPU picks how many positions the call
launches, and nothing it returns changes.

Every case binds the same input tensors into two contexts with the same parameter sets, streams and history, created with the
default PWPP_SMALL_CALL (so a 4-wide launch of a longer run must keep that run's batch kernels): `eng` with the ladder
{1, 4, 16}, `twin` the same call without one. After every run or replay both are compared bit for bit: the indices, offsets,
num_ground, status and read copies; the record, getter (xyz and state rows), packed-xyz and packed-record buffers in full (every buffer starts filled with the
same sentinel, so bytes past the counts must stay unwritten on both sides); the patch rows; every host getter of every position;
and every stream's export blob. The width the ladder launched is checked against the width rule of include/pwpp.h."""
import ctypes as C

import numpy as np
import pytest

from param_sets import _default, _ros
from test_gpu_bound_streams import SETS, Fleet, blobs, runs_of, tick_schedule
from test_gpu_records import LAYOUTS, outputs

pytestmark = pytest.mark.gpu

RUN, SKIP, RESET = 0, 1, 2
REJECTED = (2, 3, 6, 7)   # PWPP_FRAME_SKIPPED, PWPP_ACTION_INVALID, PWPP_STREAM_OUT_OF_RANGE, PWPP_STREAM_DUPLICATE
ERR_INVALID_ARG = -1
LADDER = [1, 4, 16]
SENTINEL = 0xA5


class Pair(Fleet):
    """Fleet's inputs (plain, rings or packed, actions and a stream table optional) bound into two contexts: `eng` with `ladder`,
    `twin` without. Every result kind is enabled on both."""

    def __init__(self, scans, shape, ns, kind="plain", table=True, with_actions=True, sets=None, ladder=LADDER, order=None):
        import torch
        import pwpp_b200
        self.scans, self.kind = scans, kind
        self.shape, self.ns, self.nf = list(shape), ns, len(shape)
        self.stream_set = [s % 4 for s in range(ns)]
        self.eng, self.twin = [pwpp_b200.Engine(sets or SETS, device=0, num_streams=ns, stream_set=self.stream_set) for _ in range(2)]
        if order is not None:
            for e in (self.eng, self.twin):
                e.set_output_order(order)
        self.max_n = max(len(a) for a in scans) + 7
        self.stride = self.max_n * 16
        self.dscans = [torch.as_tensor(a, device="cuda") for a in scans]
        self.lay = pwpp_b200.layout_from_dtype(LAYOUTS["xyzi16"])
        self.actions = torch.zeros(self.nf, dtype=torch.int32, device="cuda") if with_actions else None
        self.streams = torch.tensor(self.shape, dtype=torch.int32, device="cuda")
        nf, caps, lays = self.nf, [self.max_n] * self.nf, [self.lay] * self.nf
        if kind == "rings":
            self.bufs = [torch.zeros((2, self.stride), dtype=torch.uint8, device="cuda") for _ in range(nf)]
            self.ring_counts = [torch.zeros(2, dtype=torch.int64, device="cuda") for _ in range(nf)]
            self.slots = torch.zeros(nf, dtype=torch.int32, device="cuda")
        elif kind == "packed":
            self.points = torch.zeros((nf * self.max_n, 4), dtype=torch.float32, device="cuda")
            self.offsets = torch.zeros(nf + 1, dtype=torch.int64, device="cuda")
        else:
            self.bufs = [torch.zeros((self.max_n, 4), dtype=torch.float32, device="cuda") for _ in range(nf)]
            self.counts = torch.zeros(nf, dtype=torch.int64, device="cuda")
        for e in (self.eng, self.twin):
            if kind == "rings":
                e.bind_call_rings(list(zip(self.bufs, self.ring_counts)), caps, lays, self.slots, streams=self.shape, actions=self.actions)
            elif kind == "packed":
                e.bind_call_packed(self.points, self.offsets, caps, layout=self.lay, streams=self.shape, actions=self.actions)
            else:
                e.bind_call(self.bufs, caps, lays, self.counts, streams=self.shape, actions=self.actions)
            e.bind_record_results()
            e.bind_getter_results()
            e.bind_packed_xyz()
            e.bind_packed_records()
            if table:
                e.bind_stream_table(self.streams)
        self.table = table
        self.runs = runs_of(self.shape)
        self.widths = list(ladder) + [nf]
        self.eng.bind_width_ladder(ladder)
        for e in (self.eng, self.twin):
            for t in self.full_buffers(e).values():
                if t.is_contiguous() and t.numel():
                    t.view(torch.uint8).fill_(SENTINEL)
        torch.cuda.synchronize()

    def full_buffers(self, e):
        """Every device result buffer of the bound call, whole: bytes past the counts included."""
        idx, off, ng, st = e.bound_call_results()
        out = {"idx": idx, "off": off, "ng": ng}
        g, n, _, cnt = e.bound_record_results()
        out.update(rec_g=g, rec_n=n)
        d = e.bound_getter_results()
        out.update(ground_xyz=d["ground_xyz"], nonground_xyz=d["nonground_xyz"])
        px = e.bound_packed_xyz()
        out.update(px_g=px["ground"], px_n=px["nonground"])
        pr = e.bound_packed_records()
        out.update(pr_g=pr["ground"], pr_n=pr["nonground"])
        return out

    def results(self, e):
        """Everything of the last run that the contract covers, as host bytes."""
        import torch
        out = {k: v.cpu().numpy().tobytes() for k, v in self.full_buffers(e).items()}
        _, _, _, st = e.bound_call_results()
        out["status"] = st.cpu().numpy().tobytes()
        if self.table:
            out["streams_read"] = e.bound_call_streams().cpu().numpy().tobytes()
        if self.kind == "rings":
            out["slots_read"] = e.bound_call_slots().cpu().numpy().tobytes()
        out["rec_counts"] = e.bound_record_results()[3].cpu().numpy().tobytes()
        d = e.bound_getter_results()
        npat = d["num_patches"].cpu().numpy()
        out["num_patches"] = npat.tobytes()
        out["xyz_counts"] = d["xyz_counts"].cpu().numpy().tobytes()
        for k in ("height", "elevation_thr", "flatness_thr", "n_elevation", "n_flatness"):
            out[k] = d[k].cpu().numpy().tobytes()
        for f in range(self.nf):
            out[f"centers{f}"] = d["centers"][f, :npat[f]].cpu().numpy().tobytes()
            out[f"normals{f}"] = d["normals"][f, :npat[f]].cpu().numpy().tobytes()
        for k in ("ground_offsets", "nonground_offsets"):
            out["px_" + k] = e.bound_packed_xyz()[k].cpu().numpy().tobytes()
            out["pr_" + k] = e.bound_packed_records()[k].cpu().numpy().tobytes()
        torch.cuda.synchronize()
        for f in range(self.nf):
            out[f"host{f}"] = outputs(e, f)
        out["blobs"] = blobs(e, self.ns).cpu().numpy().tobytes()
        return out

    def compare(self, what):
        import torch
        torch.cuda.synchronize()
        a, b = self.results(self.eng), self.results(self.twin)
        assert a.keys() == b.keys()
        bad = [k for k in a if a[k] != b[k]]
        assert not bad, f"{what}: the ladder changed {bad[:8]}"
        st = np.frombuffer(a["status"], np.int32)
        want = expected_width(st, self.widths)
        assert int(self.eng.bound_call_width().item()) == want, f"{what}: width"
        assert int(self.twin.bound_call_width().item()) == self.nf, f"{what}: the twin's width"
        return want

    def run(self, graphs=None):
        """One run of both calls: eager, or a replay of their captured graphs."""
        if graphs:
            for g in graphs:
                g.replay()
        else:
            self.eng.run_bound_call()
            self.twin.run_bound_call()

    def capture(self):
        import torch
        gs = []
        for e in (self.eng, self.twin):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                e.run_bound_call(torch.cuda.current_stream().cuda_stream)
            gs.append(g)
        return gs


def expected_width(status, widths):
    """include/pwpp.h's width rule."""
    runs = np.flatnonzero(~np.isin(status, REJECTED))
    need = max(int(runs[-1]) + 1 if len(runs) else 0, 1)
    return next(w for w in widths if w >= need)


def present(rng, nf, ns, k, compact):
    """A scheduler's pick of k present sensors out of ns on nf positions: compacted to the front, or scattered, holes elsewhere;
    RESET and SKIP actions on a few of them."""
    read = np.full(nf, -1, np.int64)
    pos = np.arange(k) if compact else np.sort(rng.choice(nf, k, replace=False))
    read[pos] = rng.choice(ns, k, replace=False)
    acts = np.where(rng.random(nf) < 0.1, RESET, RUN)
    acts[pos[rng.random(k) < 0.08]] = SKIP
    return read, acts


@pytest.mark.parametrize("mode", ["graph", "eager"])
def test_fleet_of_256_streams(kitti, mode):
    """A 64-position call with a stream table and actions over 256 streams on four parameter sets (the ROS set, num_min_pts = 0,
    among them): k present sensors for k in {0, 1, 2, 4, 5, 16, 17, 63, 64}, compacted to the front and scattered, replayed from
    torch.cuda.graph or run eagerly. Every width of the ladder is launched."""
    p = Pair(list(kitti), list(range(64)), 256)
    rng = np.random.default_rng(64)
    assert int(p.eng.bound_call_width().item()) == 0, "the width before the ladder's first run"
    graphs = p.capture() if mode == "graph" else None
    seen = set()
    for t, (k, compact) in enumerate((k, c) for k in (0, 1, 2, 4, 5, 16, 17, 63, 64) for c in (True, False)):
        read, acts = present(rng, 64, 256, k, compact)
        p.load(t, read, acts)
        p.run(graphs)
        seen.add(p.compare(f"k={k} {'compacted' if compact else 'scattered'}"))
    assert seen == {1, 4, 16, 64}


@pytest.mark.parametrize("kind,table", [("plain", False), ("rings", False), ("rings", True), ("packed", False), ("packed", True)],
                         ids=["actions", "rings", "rings_table", "packed", "packed_table"])
def test_binds(kitti, kind, table):
    """Plain frames with actions, scan rings and packed batches, with and without a stream table: absent sensors skipped by
    their action or left out of the table, replayed from one captured graph."""
    nf, ns = 24, 32
    p = Pair(list(kitti), list(range(nf)), ns, kind=kind, table=table)
    graphs = p.capture()
    rng = np.random.default_rng(24)
    for t, k in enumerate((0, 1, 3, 4, 5, 12, 16, 17, 24, 2)):
        pos = np.arange(k) if t % 2 == 0 else np.sort(rng.choice(nf, k, replace=False))
        acts = np.full(nf, SKIP)
        acts[pos] = np.where(rng.random(k) < 0.15, RESET, RUN)
        if t == 9:
            acts[5] = 9   # an invalid action is rejected
        read = np.arange(nf) if not table else np.where(acts == SKIP, -1, rng.permutation(ns)[:nf])
        if table:
            acts = np.where(acts == SKIP, RUN, acts)   # the table leaves them out
        p.load(t, read, acts)
        p.run(graphs)
        p.compare(f"tick {t}, k={k}")


def test_backlog_shape(kitti):
    """The shape [0..63, 0..31] (two runs): widths 1, 4 and 16 cut run 0, and run 1 lies wholly past them."""
    shape = list(range(64)) + list(range(32))
    p = Pair(list(kitti), shape, 256)
    graphs = p.capture()
    rng = np.random.default_rng(96)
    for t in range(8):
        if t % 2:
            read, acts = tick_schedule(rng, shape, 256, p.runs)
        else:
            read, acts = present(rng, 96, 256, [1, 3, 12, 40][t // 2], True)
        p.load(t, read, acts)
        p.run(graphs)
        p.compare(f"tick {t}")


def test_reference_exact_order(kitti):
    """PWPP_ORDER_REFERENCE_EXACT: the libstdc++ order of equal z and its fix-up kernels in every width's body."""
    p = Pair(list(kitti), list(range(16)), 32, order=2, ladder=[1, 4])
    graphs = p.capture()
    rng = np.random.default_rng(16)
    for t, k in enumerate((1, 3, 4, 9, 16)):
        read, acts = present(rng, 16, 32, k, t % 2 == 0)
        p.load(t, read, acts)
        p.run(graphs if t % 2 else None)
        p.compare(f"tick {t}")


def test_launch_count_rule(kitti):
    """A laddered run launches one more kernel than the same call without a ladder (the selector), whatever width runs."""
    p = Pair(list(kitti), list(range(64)), 256)
    rng = np.random.default_rng(1)
    for t, k in enumerate((0, 1, 5, 64)):
        read, acts = present(rng, 64, 256, k, True)
        p.load(t, read, acts)
        a, b = p.eng.launch_count(), p.twin.launch_count()
        p.run()
        assert p.eng.launch_count() - a == p.twin.launch_count() - b + 1, f"k={k}"
        p.compare(f"k={k}")


def test_enable_errors(kitti):
    """Every refused enable returns PWPP_ERR_INVALID_ARG and leaves the call as it was."""
    import torch
    import pwpp_b200
    e = pwpp_b200.Engine(device=0, num_streams=4)
    w = np.array([1, 2], np.int32)
    assert e.lib.pwpp_bind_width_ladder(e._h, 1, w.ctypes.data) == ERR_INVALID_ARG   # no call bound
    # neither actions nor a stream table
    bufs = [torch.zeros((100, 4), dtype=torch.float32, device="cuda") for _ in range(4)]
    counts = torch.zeros(4, dtype=torch.int64, device="cuda")
    lay = pwpp_b200.layout_from_dtype(LAYOUTS["xyzi16"])
    e.bind_call(bufs, [100] * 4, [lay] * 4, counts, streams=[0, 1, 2, 3])
    assert e.lib.pwpp_bind_width_ladder(e._h, 1, w.ctypes.data) == ERR_INVALID_ARG
    p = Pair(list(kitti), list(range(8)), 16, ladder=[2])
    lib, h = p.eng.lib, p.eng._h
    bad = [(None, 1), ([], 0), ([1, 2, 3, 4, 5, 6, 7, 8], 8), ([2, 2], 2), ([3, 2], 2), ([0], 1), ([8], 1), ([-1], 1)]
    for ws, n in bad:   # on the twin, which has no ladder yet
        arr = None if ws is None else np.array(ws + [0], np.int32)
        assert p.twin.lib.pwpp_bind_width_ladder(p.twin._h, n, None if arr is None else arr.ctypes.data) == ERR_INVALID_ARG, (ws, n)
    assert lib.pwpp_bind_width_ladder(h, 1, w.ctypes.data) == ERR_INVALID_ARG   # a second enable
    for fn in ("pwpp_bind_record_results", "pwpp_bind_getter_results", "pwpp_bind_packed_xyz", "pwpp_bind_packed_records"):
        assert getattr(lib, fn)(h, 1) == ERR_INVALID_ARG, fn
    assert lib.pwpp_bind_stream_table(h, C.c_void_p(p.streams.data_ptr())) == ERR_INVALID_ARG
    assert "before the width ladder" in lib.pwpp_last_error().decode()
    rng = np.random.default_rng(8)
    for t, k in enumerate((2, 8)):
        read, acts = present(rng, 8, 16, k, True)
        p.load(t, read, acts)
        p.run()
        p.compare(f"after the refused enables, k={k}")


def test_unbind_leaves_other_graphs_valid(kitti):
    """Call 1 of the laddered context gets a ladder and a captured graph, then is unbound: call 0's graph keeps replaying, bit
    for bit the twin's."""
    import torch
    p = Pair(list(kitti), list(range(16)), 64, sets=[_default(), _ros(), _default(), _ros()], ladder=[1, 4, 8])
    g0 = p.capture()
    e = p.eng
    e.select_bound_call(1)
    bufs = [torch.zeros((p.max_n, 4), dtype=torch.float32, device="cuda") for _ in range(8)]
    counts = torch.zeros(8, dtype=torch.int64, device="cuda")
    acts = torch.zeros(8, dtype=torch.int32, device="cuda")
    e.bind_call(bufs, [p.max_n] * 8, [p.lay] * 8, counts, streams=list(range(8)), actions=acts)
    e.bind_width_ladder([2])
    g1 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g1):
        e.run_bound_call(torch.cuda.current_stream().cuda_stream)
    e.unbind_call()
    e.select_bound_call(0)
    del g1
    rng = np.random.default_rng(3)
    for t, k in enumerate((1, 6, 16)):
        read, acts_ = present(rng, 16, 64, k, True)
        p.load(t, read, acts_)
        p.run(g0)
        p.compare(f"after the unbind, k={k}")
