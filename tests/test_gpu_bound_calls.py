"""Several bound calls per context (pwpp_select_bound_call): one captured graph per batch shape over the same sensor streams.

One context with four parameter sets holds bound calls of different kinds and widths, each captured into its own graph and
replayed in a seeded random order. After every replay the call is compared with a twin context driven by direct
pwpp_estimate_device_records calls of the accepted frames, run by run (test_gpu_bound_streams.Fleet.check): index lists, offsets,
status, every stream's export blob. The call's own result buffers must also survive the replays of the other calls untouched.
Contexts are created with PWPP_SMALL_CALL=0 so that calls of any size take the batch kernels on both sides."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_bound_actions import batch_kernels
from test_gpu_bound_streams import RUN, SKIP, RESET, SETS, Fleet, runs_of, tick_schedule
from test_gpu_records import LAYOUTS, outputs

pytestmark = pytest.mark.gpu

NS = 96   # streams of the context: more than the widest call has positions
ERR_INVALID_ARG, ERR_CAPACITY = -1, -5


def contexts(order=None):
    import pwpp_b200
    with batch_kernels():
        eng, twin = [pwpp_b200.Engine(SETS, device=0, num_streams=NS, stream_set=[s % 4 for s in range(NS)]) for _ in range(2)]
    if order is not None:
        eng.set_output_order(order)
        twin.set_output_order(order)
    return eng, twin


class Call(Fleet):
    """Bound call k of the shared context `eng` (twin `twin`): Fleet's bind, load and check, on the selected call. `results`
    names the call's own result buffers: "records" (pwpp_bind_record_results), "getters" (pwpp_bind_getter_results, xyz and
    state) and "packed" (pwpp_bind_packed_xyz and pwpp_bind_packed_records)."""

    def __init__(self, eng, twin, k, scans, shape, kind, table, with_actions, results=()):
        import torch
        import pwpp_b200
        self.eng, self.twin, self.k = eng, twin, k
        self.scans, self.kind, self.results = scans, kind, results
        self.shape, self.ns, self.nf = list(shape), NS, len(shape)
        self.max_n = max(len(a) for a in scans) + 7
        self.stride = self.max_n * 16
        self.dscans = [torch.as_tensor(a, device="cuda") for a in scans]
        self.lay = pwpp_b200.layout_from_dtype(LAYOUTS["xyzi16"])
        self.actions = torch.zeros(self.nf, dtype=torch.int32, device="cuda") if with_actions else None
        self.streams = torch.tensor(self.shape, dtype=torch.int32, device="cuda")
        nf, caps, lays = self.nf, [self.max_n] * self.nf, [self.lay] * self.nf
        self.select()
        if kind == "rings":
            self.bufs = [torch.zeros((2, self.stride), dtype=torch.uint8, device="cuda") for _ in range(nf)]
            self.ring_counts = [torch.zeros(2, dtype=torch.int64, device="cuda") for _ in range(nf)]
            self.slots = torch.zeros(nf, dtype=torch.int32, device="cuda")
            eng.bind_call_rings(list(zip(self.bufs, self.ring_counts)), caps, lays, self.slots, streams=self.shape, actions=self.actions)
        elif kind == "packed":
            self.points = torch.zeros((nf * self.max_n, 4), dtype=torch.float32, device="cuda")
            self.offsets = torch.zeros(nf + 1, dtype=torch.int64, device="cuda")
            eng.bind_call_packed(self.points, self.offsets, caps, layout=self.lay, streams=self.shape, actions=self.actions)
        else:
            self.bufs = [torch.zeros((self.max_n, 4), dtype=torch.float32, device="cuda") for _ in range(nf)]
            self.counts = torch.zeros(nf, dtype=torch.int64, device="cuda")
            eng.bind_call(self.bufs, caps, lays, self.counts, streams=self.shape, actions=self.actions)
        if "records" in results:
            eng.bind_record_results()
        if "getters" in results:
            eng.bind_getter_results()
        if "packed" in results:
            eng.bind_packed_xyz()
            eng.bind_packed_records()
        self.table = table
        if table:
            eng.bind_stream_table(self.streams)
        self.runs = runs_of(self.shape)

    def select(self):
        self.eng.select_bound_call(self.k)

    def tick(self, rng, t):
        """Loads tick t: with a table a scheduler's pick of streams (holes, duplicates, out-of-range ids), without one the bound
        streams; with actions seeded SKIP and RESET."""
        if self.table:
            read, acts = tick_schedule(rng, self.shape, NS, self.runs)
        else:
            read, acts = self.shape, rng.choice([RUN, SKIP, RESET], self.nf, p=[0.8, 0.12, 0.08])
        self.load(t, read, acts if self.actions is not None else [RUN] * self.nf)

    def check(self, what):
        self.select()
        super().check(what)

    def capture(self):
        import torch
        self.select()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
        return g

    def own(self):
        """Copies of every buffer the call owns: status, the read copies of its streams and slots, and its enabled results."""
        import torch
        self.select()
        e = self.eng
        out = {"status": e.bound_call_results()[3]}
        if self.table:
            out["read"] = e.bound_call_streams()
        if self.kind == "rings":
            out["slots"] = e.bound_call_slots()
        if "records" in self.results:
            g, n, _, cnt = e.bound_record_results()
            out.update(rec_g=g, rec_n=n, rec_counts=cnt)
        if "getters" in self.results:
            d = e.bound_getter_results()
            out.update({k: d[k] for k in ("ground_xyz", "nonground_xyz", "xyz_counts", "height", "elevation_thr", "flatness_thr",
                                          "n_elevation", "n_flatness")})
        if "packed" in self.results:
            px, pr = e.bound_packed_xyz(), e.bound_packed_records()
            out.update(px_g=px["ground"], px_n=px["nonground"], px_go=px["ground_offsets"], px_no=px["nonground_offsets"],
                       pr_g=pr["ground"], pr_n=pr["nonground"])
        torch.cuda.synchronize()
        return {k: v.clone() for k, v in out.items()}


def ladder(scans, order=None):
    """A context holding three bound calls of different kinds and widths, and its twin."""
    eng, twin = contexts(order)
    return [Call(eng, twin, 0, scans, [0], "plain", table=True, with_actions=False, results=("getters",)),
            Call(eng, twin, 1, scans, list(range(8)), "rings", table=False, with_actions=True, results=("records",)),
            Call(eng, twin, 2, scans, list(range(64)), "packed", table=True, with_actions=False, results=("packed",))]


def first_runs(calls):
    """One eager run of every call (each over its bound streams), checked, then one graph per call."""
    for c in calls:
        c.load(0, c.shape, [RUN] * c.nf)
        c.select()
        c.eng.run_bound_call()
        c.check(f"call {c.k}: eager run")
    return [c.capture() for c in calls]


def assert_same(a, b, what):
    """Bit for bit: rows past a count were never written and may hold any pattern, NaN included."""
    import torch
    bits = {2: torch.int16, 4: torch.int32, 8: torch.int64}
    assert a.keys() == b.keys(), what
    for k in a:
        x, y = a[k], b[k]
        if x.is_floating_point():
            x, y = x.view(bits[x.element_size()]), y.view(bits[y.element_size()])
        assert torch.equal(x, y), f"{what}: {k}"


def replay(calls, graphs, rng, ticks, t0, what, snaps=None):
    """`ticks` replays in a seeded random order, each call's inputs rewritten before its replay and checked after it; with
    `snaps` also every other call's own buffers against their snapshot after that call's last run."""
    import torch
    for t in range(ticks):
        k = int(rng.integers(len(calls)))
        c = calls[k]
        if c is None:
            continue
        c.tick(rng, t0 + t)
        graphs[k].replay()
        torch.cuda.synchronize()
        c.check(f"{what}: tick {t}, call {k}")
        if snaps is not None:
            snaps[k] = c.own()
            for j, s in snaps.items():
                if j != k and calls[j] is not None:
                    assert_same(calls[j].own(), s, f"{what}: tick {t}, call {j}'s own buffers after a replay of call {k}")


def test_interleaved_replays_equal_the_twin_and_leave_the_other_calls_alone(kitti):
    """A 1-frame plain call with a stream table and getter results, an 8-frame call over 2-slot rings with actions and record
    results, and a 64-position packed call with a stream table and packed results: 36 replays in a seeded order."""
    calls = ladder(list(kitti))
    graphs = first_runs(calls)
    replay(calls, graphs, np.random.default_rng(7), 36, 1, "ladder", snaps={})


def test_unbind_keeps_the_other_graphs(kitti):
    """Unbinding the middle call leaves the other two graphs valid; a rebind of a shape that fits captures and replays."""
    calls = ladder(list(kitti))
    graphs = first_runs(calls)
    rng = np.random.default_rng(11)
    replay(calls, graphs, rng, 6, 1, "before the unbind")
    calls[1].select()
    calls[1].eng.unbind_call()
    replay([calls[0], None, calls[2]], graphs, rng, 8, 10, "after the unbind")
    calls[1] = Call(calls[0].eng, calls[0].twin, 1, list(kitti), [5, 6, 7, 8], "rings", table=False, with_actions=True, results=("records",))
    graphs[1] = calls[1].capture()
    replay(calls, graphs, rng, 12, 20, "after the rebind")


def test_growth_after_a_capture_is_refused(kitti):
    """After the captures, a bind that needs more points, a bind with actions whose run needs more scratch slots and a
    stream-table enable that does: PWPP_ERR_CAPACITY, and the replays that follow still equal the twin."""
    import torch
    import pwpp_b200
    calls = ladder(list(kitti))
    graphs = first_runs(calls)
    eng = calls[0].eng
    lay = pwpp_b200.layout_from_dtype(LAYOUTS["xyzi16"])
    eng.select_bound_call(3)
    big = 2 * 64 * calls[2].max_n   # twice the points the widest call reserved
    buf = torch.zeros((big, 4), dtype=torch.float32, device="cuda")
    cnt = torch.zeros(65, dtype=torch.int64, device="cuda")
    act = torch.zeros(65, dtype=torch.int32, device="cuda")
    with pytest.raises(pwpp_b200.PwppError, match=r"points \(the sum of max_n\) needs larger work buffers"):
        eng.bind_call([buf], [big], [lay], cnt[:1])
    small = [buf[1000 * f:1000 * (f + 1)] for f in range(65)]   # 65 frames of 1000 points fit the work buffers
    with pytest.raises(pwpp_b200.PwppError, match="needs 65 scratch state slots"):
        eng.bind_call(small, [1000] * 65, [lay] * 65, cnt, actions=act)
    eng.bind_call(small, [1000] * 65, [lay] * 65, cnt)   # no actions: no scratch slots, and the work buffers fit
    table = torch.arange(65, dtype=torch.int32, device="cuda")
    assert eng.lib.pwpp_bind_stream_table(eng._h, C.c_void_p(table.data_ptr())) == ERR_CAPACITY
    assert "needs 65 scratch state slots" in eng.lib.pwpp_last_error().decode()
    eng.unbind_call()
    replay(calls, graphs, np.random.default_rng(5), 12, 1, "after the refused binds")


def test_fresh_context_grows_small_then_large(kitti):
    """Binding a 1-frame call, then a 16-position packed call with a stream table and actions, before any run grows the work
    buffers and the scratch slots; both then capture and replay equal to the twin."""
    eng, twin = contexts()
    calls = [Call(eng, twin, 0, list(kitti), [0], "plain", table=False, with_actions=False),
             Call(eng, twin, 1, list(kitti), list(range(16)), "packed", table=True, with_actions=True)]
    graphs = first_runs(calls)
    replay(calls, graphs, np.random.default_rng(3), 10, 1, "small then large")


def test_host_getters_follow_the_call_that_ran_last(kitti):
    """The host getters and the Engine's serve the call whose run came last, not the selected one, also after its unbind."""
    import torch
    calls = ladder(list(kitti))
    eng = calls[0].eng
    rng = np.random.default_rng(13)
    for c in calls:
        c.tick(rng, 1)
    calls[0].select()
    eng.run_bound_call()
    calls[2].select()
    eng.run_bound_call()
    torch.cuda.synchronize()
    want = [outputs(eng, f) for f in range(64)]
    calls[0].select()   # selecting is not running
    assert [outputs(eng, f) for f in range(64)] == want
    assert eng.selected_bound_call == 0 and eng.lib.pwpp_selected_bound_call(eng._h) == 0
    calls[2].select()
    eng.unbind_call()
    assert [outputs(eng, f) for f in range(64)] == want, "after the unbind of the last call"


def test_selection_and_per_call_errors(kitti):
    """select outside [0, 32) is refused and keeps the selection; "already bound" is per call; with only call 5 bound,
    set_output_order, clone and a direct call that would grow a work buffer are refused, and allowed after its unbind."""
    import pwpp_b200
    eng, twin = contexts()
    for k in (-1, pwpp_b200.MAX_BOUND_CALLS):
        with pytest.raises(pwpp_b200.PwppError, match="outside"):
            eng.select_bound_call(k)
        assert eng.selected_bound_call == 0 and eng.lib.pwpp_selected_bound_call(eng._h) == 0
    assert eng.lib.pwpp_select_bound_call(eng._h, pwpp_b200.MAX_BOUND_CALLS) == ERR_INVALID_ARG
    assert eng.lib.pwpp_selected_bound_call(eng._h) == 0
    c = Call(eng, twin, 5, [a[:20000] for a in kitti], [0, 1], "plain", table=False, with_actions=False)
    with pytest.raises(pwpp_b200.PwppError, match="already bound"):
        Call(eng, twin, 5, [a[:20000] for a in kitti], [2], "plain", table=False, with_actions=False)
    Call(eng, twin, 6, [a[:20000] for a in kitti], [2], "plain", table=False, with_actions=False)
    eng.select_bound_call(6)
    eng.unbind_call()
    eng.select_bound_call(0)
    with pytest.raises(pwpp_b200.PwppError, match="output order"):
        eng.set_output_order(eng.ORDER_BIN)
    with pytest.raises(pwpp_b200.PwppError, match="bound call"):
        eng.clone()
    with pytest.raises(pwpp_b200.PwppError, match="does not fit the work buffers"):
        eng.estimate_host([np.ascontiguousarray(kitti[0])] * 3)
    c.load(0, c.shape, [RUN, RUN])
    c.select()
    eng.run_bound_call()
    c.check("call 5 after the refused calls")
    eng.unbind_call()
    eng.set_output_order(eng.ORDER_REFERENCE)
    eng.clone().close()
    eng.estimate_host([np.ascontiguousarray(kitti[0])] * 3)


def test_launch_counts_equal_single_call_contexts(kitti):
    """Every call of the ladder adds per run exactly what the same bind adds alone in a fresh context."""
    calls = ladder(list(kitti))
    rng = np.random.default_rng(17)
    for c in calls:
        eng, twin = contexts()
        alone = Call(eng, twin, 0, list(kitti), c.shape, c.kind, c.table, c.actions is not None, c.results)
        deltas = []
        for x in (c, alone):
            x.tick(rng, 1)
            x.select()
            x.eng.run_bound_call()
            n0 = x.eng.launch_count()
            x.eng.run_bound_call()
            deltas.append(x.eng.launch_count() - n0)
            x.eng.synchronize()
        assert deltas[0] == deltas[1], f"call {c.k}"
        eng.close()
        twin.close()


def test_exact_order_with_two_widths(kitti):
    """PWPP_ORDER_REFERENCE_EXACT: a 1-frame call and an 8-frame ring call, bound narrow first (the exact-order scratch grows at
    the second bind), replayed interleaved."""
    import pwpp_b200
    eng, twin = contexts(pwpp_b200.Engine.ORDER_REFERENCE_EXACT)
    calls = [Call(eng, twin, 0, list(kitti), [0], "plain", table=True, with_actions=False),
             Call(eng, twin, 1, list(kitti), list(range(8)), "rings", table=False, with_actions=True)]
    graphs = first_runs(calls)
    replay(calls, graphs, np.random.default_rng(19), 8, 1, "exact order")
