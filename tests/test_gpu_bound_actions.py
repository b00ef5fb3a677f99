"""Per-frame actions of bound calls (pwpp_bind_call_actions): a frame is run, skipped (its stream keeps its state bit for bit) or
its stream is reset first, decided on the GPU at every run or replay.

Every run is compared bit for bit with a twin context driven by pwpp_estimate_device_records calls that name only the present
frames, with pwpp_reset_stream between call segments where a RESET falls: every present frame's results at its position in the
bound call, the empty results of skipped frames (those of a one-frame call with no points), d_status, and every stream's state,
histories and export blob, in both output orders.

Most contexts here are created with PWPP_SMALL_CALL=0, so a call of any size takes the batch kernels: a twin call that names only
the present frames of a run may hold four frames or fewer where the bound call's run holds more, and the latency kernels of
such small calls are a different kernel variant (their patch records are not compared with the batch kernels' here). The
default-mode cases keep every run of the bound call at four frames or fewer and split the twin's calls at the runs as well, so
both sides take the latency kernels of small calls and every output is compared there too."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

from param_sets import _default, _no_rvpf_tgr, _ros
from test_gpu_bound_call import NAMES, Pair, engine
from test_gpu_records import LAYOUTS, outputs, records, stream

pytestmark = pytest.mark.gpu

RUN, SKIP, RESET = 0, 1, 2
OUT_OF_RANGE, SKIPPED, INVALID = 1, 2, 3
ERR_INVALID_ARG = -1
SENTINEL = 0x5A


@pytest.fixture(scope="module")
def scans(kitti):
    return list(kitti)


@contextlib.contextmanager
def batch_kernels():
    """Contexts created inside take the batch kernels for calls of every size."""
    old = os.environ.get("PWPP_SMALL_CALL")
    os.environ["PWPP_SMALL_CALL"] = "0"
    try:
        yield
    finally:
        if old is None:
            del os.environ["PWPP_SMALL_CALL"]
        else:
            os.environ["PWPP_SMALL_CALL"] = old


def storage20():
    p = _default()
    p.max_elevation_storage = p.max_flatness_storage = 20
    return p


class ActionPair(Pair):
    """Pair's bound context rebound with an actions tensor; the twin runs only the present frames."""

    def __init__(self, streams, names, max_n, order=0, num_streams=None, sets=None, single=None, batch=True):
        import torch
        self._sets, self._single = sets, single
        self.kernels = batch_kernels if batch else contextlib.nullcontext
        self.run_starts = set(runs_of(streams)) if not batch else set()
        with self.kernels():
            super().__init__(streams, names, max_n, order, num_streams, sets)
        if single is not None:   # one parameter set other than the default on every stream: both contexts re-created with it
            import pwpp_b200
            ns = num_streams or (max(streams) + 1)
            self.eng.unbind_call()
            with self.kernels():
                self.eng, self.twin = [pwpp_b200.Engine(single, device=0, num_streams=ns) for _ in range(2)]
            for e in (self.eng, self.twin):
                e.set_output_order(order)
        else:
            self.eng.unbind_call()
        self.order = order
        self.ns = num_streams or (max(streams) + 1)
        self.actions = torch.zeros(len(streams), dtype=torch.int32, device="cuda")
        self.eng.bind_call(self.ptrs, self.max_n, self.lays, self.counts, streams=self.streams, actions=self.actions)
        self._empty = {}

    def set_actions(self, acts):
        import torch
        self.actions.copy_(torch.tensor(list(acts), dtype=torch.int32))
        torch.cuda.synchronize()
        self.acts = [int(a) for a in acts]

    def empty(self, f):
        """Outputs of an empty frame of frame f's stream set and layout: a one-frame call with no points on a fresh context."""
        s = self.streams[f]
        key = self.eng.stream_set[s]
        if key not in self._empty:
            import pwpp_b200
            with self.kernels():
                if self._single is not None:
                    e = pwpp_b200.Engine(self._single, device=0, num_streams=self.ns)
                    e.set_output_order(self.order)
                else:
                    e = engine(self.ns, self.order, self._sets)
            e.estimate_device_records([self.ptrs[f]], [0], [self.lays[f]], streams=[s])
            e.synchronize()
            self._empty[key] = outputs(e, 0)
            e.close()
        return self._empty[key]

    def check_actions(self, sizes, what, records_check=False):
        """The bound call's last run against the twin driven segment by segment; sizes as Pair.load returns them."""
        idx, off, ng, st = self.eng.bound_call_results()
        self.eng.synchronize()
        nf = len(self.streams)
        acts = self.acts
        present = [a in (RUN, RESET) for a in acts]
        eff = [k if p else 0 for k, p in zip(sizes, present)]
        assert np.array_equal(off.cpu().numpy(), np.concatenate([[0], np.cumsum(eff)])), f"{what}: offsets"
        counts = self.counts.cpu().numpy()
        want_st = [(0 if 0 <= c <= m else OUT_OF_RANGE) if p else (SKIPPED if a == SKIP else INVALID)
                   for c, m, p, a in zip(counts, self.max_n, present, acts)]
        assert st.cpu().numpy().tolist() == want_st, f"{what}: status"
        ngs = ng.cpu().numpy()
        got = [outputs(self.eng, f) for f in range(nf)]
        if records_check:
            import torch
            torch.cuda.synchronize()
            gb, nb, roff, rcnt = self.eng.bound_record_results()
            bufs = [gb.cpu().numpy(), nb.cpu().numpy()]
            rcnt = rcnt.cpu().numpy()
        for f in range(nf):
            if not present[f]:
                assert got[f] == self.empty(f), f"{what}: skipped frame {f}"
                assert ngs[f] == 0
                if records_check:
                    assert rcnt[f].tolist() == [0, 0]
                    for b in bufs:
                        assert (b[roff[f]: roff[f + 1]] == SENTINEL).all(), f"{what}: skipped frame {f}: its region was written"
        seg = []

        def flush():
            if not seg:
                return
            self.twin.estimate_device_records([self.ptrs[f] for f in seg], [sizes[f] for f in seg], [self.lays[f] for f in seg],
                                              streams=[self.streams[f] for f in seg])
            self.twin.synchronize()
            for k, f in enumerate(seg):
                assert got[f] == outputs(self.twin, k), f"{what}: frame {f}"
                assert ngs[f] == self.twin.num_ground(k), f"{what}: frame {f} num_ground"
                if records_check:
                    step = LAYOUTS[self.names[f]].itemsize
                    want = [self.twin.num_ground(k), self.twin.num_nonground(k)]
                    assert rcnt[f].tolist() == want, f"{what}: frame {f} record counts"
                    for z, tw in enumerate((self.twin.ground_records(k), self.twin.nonground_records(k))):
                        region = bufs[z][roff[f]: roff[f + 1]]
                        n = want[z] * step
                        assert np.array_equal(region[:n], np.ascontiguousarray(tw).view(np.uint8).reshape(-1)), f"{what}: frame {f} part {z}"
                        assert (region[n:] == SENTINEL).all()
            seg.clear()

        for f in range(nf):
            if f in self.run_starts:   # default mode: the twin's calls no larger than the bound call's runs
                flush()
            if acts[f] == RESET:
                flush()
                self.twin.reset(self.streams[f])
            if present[f]:
                seg.append(f)
        flush()
        for s in sorted(set(self.streams)):
            assert stream(self.eng, s) == stream(self.twin, s), f"{what}: stream {s}"

    def step(self, scans, seed, acts, what, counts=None, records_check=False):
        sizes = self.load(scans, seed, counts)
        self.set_actions(acts)
        if records_check:
            fill(self)
        self.eng.run_bound_call()
        self.check_actions(sizes, what, records_check)
        return sizes


def runs_of(streams):
    """First frame of every run of a stream table (maximal spans of pairwise distinct streams), as the bind splits it."""
    starts, last = [0], {}
    for f, s in enumerate(streams):
        if s in last and last[s] >= starts[-1]:
            starts.append(f)
        last[s] = f
    return starts


def fill(p):
    import torch
    g, ng, _, _ = p.eng.bound_record_results()
    for b in (g, ng):
        if b is not None:
            b.fill_(SENTINEL)
    torch.cuda.synchronize()


def ragged(rng, nf, p_skip, p_reset):
    u = rng.random(nf)
    return np.where(u < p_skip, SKIP, np.where(u < p_skip + p_reset, RESET, RUN)).tolist()


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
def test_ragged_64_sensors_in_a_captured_graph(scans, order):
    """64 sensors in one captured graph, 20 replays with 10-50 % of the frames skipped and occasional resets; actions and counts
    rewritten in place before every replay, the twin naming only the present frames."""
    import torch
    sz = max(len(a) for a in scans)
    nf = 64
    p = ActionPair(list(range(nf)), [NAMES[f % 4] for f in range(nf)], [sz + 13 * k for k in range(nf)], order, sets=None,
                   single=storage20())
    rng = np.random.default_rng(64 + order)
    p.step(scans, 0, [RUN] * nf, "eager run before the capture")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        p.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    for rep in range(20):
        acts = ragged(rng, nf, 0.1 + 0.4 * rep / 19, 0.05)
        sizes = p.load(scans, rep + 1)
        p.set_actions(acts)
        g.replay()
        torch.cuda.synchronize()
        p.check_actions(sizes, f"replay {rep}")


REPEAT = [2, 0, 2, 1, 3, 0, 1]
REPEAT_ACTIONS = [
    [SKIP, RUN, RUN, RUN, RUN, RUN, RUN],            # SKIP of stream 2's first frame, RUN of its second
    [RUN, RUN, RESET, RUN, RUN, RUN, RUN],           # RESET of a second frame: a dependent run
    [RESET, RESET, RESET, RESET, RESET, RESET, RESET],
    [RUN, SKIP, RESET, SKIP, RUN, RESET, RESET],
    [SKIP] * 7,
    [RESET, RUN, SKIP, RUN, SKIP, SKIP, RESET],
]


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
def test_repeat_table(scans, order):
    sz = max(len(a) for a in scans)
    p = ActionPair(REPEAT, [NAMES[f % 4] for f in range(7)], [sz + 4096] * 7, order, single=storage20())
    for k, acts in enumerate(REPEAT_ACTIONS * 2):
        p.step(scans, k, acts, f"run {k}: {acts}")


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
def test_small_runs_in_default_mode(scans, order):
    """Default kernel selection: the bound call's runs of four frames or fewer take the latency kernels of small calls (the three
    stand-alone front-end kernels, the CTA-per-patch fits), which read the redirected stream table too; so do the twin's calls,
    split at the same runs. Four sensors, then the repeat table with dependent resets."""
    sz = max(len(a) for a in scans)
    p = ActionPair([0, 1, 2, 3], NAMES, [sz] * 4, order, single=storage20(), batch=False)
    rng = np.random.default_rng(11 + order)
    for k in range(6):
        p.step(scans, k, [RUN] * 4 if k < 2 else ragged(rng, 4, 0.35, 0.15), f"four sensors run {k}")
    q = ActionPair(REPEAT, [NAMES[f % 4] for f in range(7)], [sz] * 7, order, single=storage20(), batch=False)
    for k, acts in enumerate(REPEAT_ACTIONS):
        q.step(scans, k, acts, f"repeat table run {k}: {acts}")


def test_four_parameter_sets(scans):
    """Scratch slots under sets of different history capacities."""
    sets = [_default(), _ros(), _no_rvpf_tgr(), storage20()]
    sets[0].sensor_height = 1.6
    sz = max(len(a) for a in scans)
    p = ActionPair([3, 1, 0, 2, 1, 3], ["xyzi16", "velodyne22", "pcl_xyzi32", "f64_xyz", "xyzi16", "velodyne22"], [sz] * 6, num_streams=4,
                   sets=sets)
    rng = np.random.default_rng(4)
    for k in range(6):
        p.step(scans, k, [RUN] * 6 if k == 0 else ragged(rng, 6, 0.3, 0.15), f"run {k}")


def test_skip_keeps_a_full_stream_and_a_zero_count_does_not(scans):
    """Storage 20: after a few frames every history is full. SKIP leaves the export blob bit for bit; RUN with count 0 moves it
    (the threshold update runs on the trimmed histories), which is why a skip is not a count of 0."""
    sz = max(len(a) for a in scans)
    p = ActionPair([0], ["xyzi16"], [sz], single=storage20())
    for k in range(6):
        p.step(scans, k, [RUN], f"warm-up {k}")
    assert all(p.eng.state(0).n_elevation[r] == 20 for r in range(4))
    before = p.eng.export_state(0)
    p.step(scans, 6, [SKIP], "skip")
    assert p.eng.export_state(0) == before
    p.step(scans, 7, [RUN], "count 0", counts=[0])
    assert p.eng.export_state(0) != before


def test_reset_with_zero_and_out_of_range_counts(scans):
    """RESET with count 0 is "reset only": the state equals a fresh context's, bit for bit. With an out-of-range count the reset
    is applied too, and the frame runs as an empty frame with PWPP_COUNT_OUT_OF_RANGE."""
    import pwpp_b200
    sz = max(len(a) for a in scans)
    p = ActionPair([0, 1, 0], ["xyzi16", "velodyne22", "pcl_xyzi32"], [sz] * 3, single=storage20())
    fresh = pwpp_b200.Engine(storage20(), device=0, num_streams=2)
    for k in range(3):
        p.step(scans, k, [RUN] * 3, f"warm-up {k}")
    p.step(scans, 3, [RESET, RESET, RUN], "reset only", counts=[0, 0, 5])
    assert bytes(p.eng.state(1)) == bytes(fresh.state(1))
    p.step(scans, 4, [RUN, RUN, RESET], "reset of a second frame only", counts=[100, 100, 0])
    assert bytes(p.eng.state(0)) == bytes(fresh.state(0))
    p.step(scans, 5, [RESET, RESET, RESET], "out of range", counts=[-1, sz + 1, 2 ** 40])
    assert p.eng.bound_call_results()[3].cpu().numpy().tolist() == [OUT_OF_RANGE] * 3


def test_invalid_actions_skip_the_frame(scans):
    sz = max(len(a) for a in scans)
    p = ActionPair([0, 1, 2, 3, 4], NAMES + ["xyzi16"], [sz] * 5, single=storage20())
    p.step(scans, 0, [RUN] * 5, "warm-up", )
    for k, acts in enumerate([[-1, 3, RUN, -2 ** 31, 2 ** 31 - 1], [3, RUN, SKIP, RESET, 7]]):
        p.step(scans, k + 1, acts, f"invalid {acts}", counts=[-5, 10 ** 9, 100, -1, 2 ** 62])


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
def test_all_run_equals_bind_call(scans, order):
    """All-RUN actions give exactly pwpp_bind_call's results, state and launch count (no repeated streams: no reset launch)."""
    sz = max(len(a) for a in scans)
    streams = [4, 0, 3, 1, 2]
    p = ActionPair(streams, NAMES + ["velodyne22"], [sz] * 5, order)
    with batch_kernels():
        plain = engine(5, order)
    plain.bind_call(p.ptrs, p.max_n, p.lays, p.counts, streams=streams)
    for k in range(3):
        p.load(scans, k)
        p.set_actions([RUN] * 5)
        l0, m0 = p.eng.launch_count(), plain.launch_count()
        p.eng.run_bound_call()
        plain.run_bound_call()
        assert p.eng.launch_count() - l0 == plain.launch_count() - m0
        r1, r2 = p.eng.bound_call_results(), plain.bound_call_results()
        p.eng.synchronize()
        plain.synchronize()
        for a, b in zip(r1, r2):
            assert np.array_equal(a.cpu().numpy(), b.cpu().numpy())
        for f in range(5):
            assert outputs(p.eng, f) == outputs(plain, f)
        for s in range(5):
            assert stream(p.eng, s) == stream(plain, s)


def test_record_results_of_skipped_frames(scans):
    """Record results with sentinel-filled part buffers: skipped frames count 0 and their regions keep the sentinel."""
    sz = max(len(a) for a in scans)
    p = ActionPair(REPEAT, [NAMES[f % 4] for f in range(7)], [sz] * 7, 1, single=storage20())
    p.eng.bind_record_results()
    for k, acts in enumerate(REPEAT_ACTIONS):
        p.step(scans, k, acts, f"run {k}", records_check=True)


def test_graph_replays_rewrite_actions_in_place(scans):
    """Eight replays of one captured graph; actions and counts rewritten in place before each, a direct call between two of them,
    and a replay behind a long sleep kernel returns at once (no host synchronisation)."""
    import torch
    sz = max(len(a) for a in scans)
    p = ActionPair([0, 1, 2, 3, 0], NAMES + ["velodyne22"], [sz + 100] * 5, 1, single=storage20())
    p.step(scans, 0, [RUN] * 5, "eager run")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        p.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    schedule = [[SKIP, RUN, RUN, RUN, RESET], [RUN, SKIP, SKIP, RUN, RUN], [RESET, RUN, 9, RUN, SKIP], [RUN] * 5,
                [SKIP] * 5, [RUN, RESET, RUN, SKIP, RESET], [RESET] * 5, [RUN, RUN, RUN, RUN, SKIP]]
    for rep, acts in enumerate(schedule):
        counts = None if rep != 5 else [len(scans[(f + rep + 1) % 6]) // 2 for f in range(5)]
        sizes = p.load(scans, rep + 1, counts)
        p.set_actions(acts)
        if rep == 2:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                torch.cuda._sleep(2_000_000_000)
                g.replay()
                assert not st.query(), "the replay waited"
            st.synchronize()
        else:
            g.replay()
        torch.cuda.synchronize()
        p.check_actions(sizes, f"replay {rep}")
        if rep == 3:   # a direct call that fits the frozen buffers, on both contexts
            data = [records(scans[k], LAYOUTS["xyzi16"], seed=k)[0] for k in (4, 5)]
            bufs = [torch.from_numpy(r.view(np.uint8).copy()).cuda() for r in data]
            torch.cuda.synchronize()
            for e in (p.eng, p.twin):
                e.estimate_device_records([b.data_ptr() for b in bufs], [len(r) for r in data], p.lays[:1] * 2, streams=[1, 3])
                e.synchronize()
            for f in range(2):
                assert outputs(p.eng, f) == outputs(p.twin, f), f"direct call frame {f}"
            torch.cuda.synchronize()


def test_one_frame_host_calls_around_the_bind(scans):
    """A one-frame host call (the small-call graph) before the bind and after bind + unbind: the state buffers moved for the
    scratch slots, so the graph is captured again, and the results still equal a context that never bound."""
    import pwpp_b200
    sz = max(len(a) for a in scans)
    a, b = [pwpp_b200.Engine(device=0, num_streams=2) for _ in range(2)]
    import torch
    counts, actions = torch.zeros(2, dtype=torch.int64, device="cuda"), torch.zeros(2, dtype=torch.int32, device="cuda")
    buf = torch.zeros(sz * 16, dtype=torch.uint8, device="cuda")
    lay = pwpp_b200.layout_from_dtype(LAYOUTS["xyzi16"])
    for k in range(2):
        for e in (a, b):
            e.estimate_host([scans[k]], streams=[1])
        assert outputs(a, 0) == outputs(b, 0) and stream(a, 1) == stream(b, 1)
    a.bind_call([buf.data_ptr()] * 2, [sz] * 2, [lay] * 2, counts, actions=actions)
    a.unbind_call()
    for k in range(2, 5):
        for e in (a, b):
            e.estimate_host([scans[k]], streams=[1])
        assert outputs(a, 0) == outputs(b, 0) and stream(a, 1) == stream(b, 1)


def test_launch_count_rule(scans):
    """Compared with the same call bound without actions: one reset launch per run that holds a frame whose stream ran in an
    earlier run ([2, 0 | 2, 1, 3, 0 | 1]: runs 1 and 2), whatever the actions are."""
    sz = max(len(a) for a in scans)
    p = ActionPair(REPEAT, [NAMES[f % 4] for f in range(7)], [sz] * 7)
    with batch_kernels():
        plain = engine(4, 0)
    plain.bind_call(p.ptrs, p.max_n, p.lays, p.counts, streams=REPEAT)
    for acts in ([RUN] * 7, [SKIP] * 7, [RESET] * 7):
        p.load(scans, 0)
        p.set_actions(acts)
        l0, m0 = p.eng.launch_count(), plain.launch_count()
        p.eng.run_bound_call()
        plain.run_bound_call()
        assert p.eng.launch_count() - l0 == plain.launch_count() - m0 + 2


def test_bind_errors(scans):
    import torch
    import pwpp_b200
    e = engine(4, 0)
    lay = pwpp_b200.layout_from_dtype(LAYOUTS["xyzi16"])
    buf = torch.zeros(16 * 1000, dtype=torch.uint8, device="cuda")
    counts = torch.zeros(4, dtype=torch.int64, device="cuda")
    actions = torch.zeros(4, dtype=torch.int32, device="cuda")
    nf = 4
    args = [np.arange(4, dtype=np.int32).ctypes.data, (C.c_void_p * nf)(*[buf.data_ptr()] * 4), (C.c_int64 * nf)(*[1000] * 4),
            (pwpp_b200.PwppPointLayout * nf)(*[lay] * 4)]
    rc = e.lib.pwpp_bind_call_actions(e._h, nf, *args, None, C.c_void_p(actions.data_ptr()))
    assert rc == ERR_INVALID_ARG and "d_counts" in e.lib.pwpp_last_error().decode()
    ids = np.array([0, 1, 9, 2], np.int32)
    rc = e.lib.pwpp_bind_call_actions(e._h, nf, ids.ctypes.data, *args[1:], C.c_void_p(counts.data_ptr()), C.c_void_p(actions.data_ptr()))
    assert rc == ERR_INVALID_ARG and "frame 2" in e.lib.pwpp_last_error().decode()
    for bad in (actions.to(torch.int64), actions[:3], actions.cpu(), torch.zeros(8, dtype=torch.int32, device="cuda")[::2]):
        with pytest.raises(pwpp_b200.PwppError, match="actions"):
            e.bind_call([buf.data_ptr()] * 4, [1000] * 4, [lay] * 4, counts, actions=bad)
    e.bind_call([buf.data_ptr()] * 4, [1000] * 4, [lay] * 4, counts, actions=actions)
    with pytest.raises(pwpp_b200.PwppError, match="already bound"):
        e.bind_call([buf.data_ptr()] * 4, [1000] * 4, [lay] * 4, counts, actions=actions)
    e.unbind_call()
