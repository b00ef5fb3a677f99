"""Getter results of bound calls (pwpp_bind_getter_results / pwpp_bound_getter_results): ground and non-ground xyz, patch centers
and normals, and every frame's state, at fixed device addresses inside the caller's graph.

Every run is checked first as test_gpu_bound_rings.py checks it (index lists, record parts and stream states against a twin
context), then against a second twin that makes one direct call per present frame on the frame the run read (a reset first for
a RESET frame): every xyz row against pwpp_copy_*_xyz bit for bit, centers, normals and patch counts against pwpp_copy_centers /
pwpp_copy_normals / pwpp_num_patches, and each state row against pwpp_get_state of the frame's stream right after that frame (for
a skipped frame: the stream as its earlier frames left it)."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_bound_actions import INVALID, RESET, RUN, SKIP, ragged
from test_gpu_bound_rings import I32_MAX, RingPair
from test_gpu_records import LAYOUTS

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG = -1
SENTINEL = -7.25e33
STATE_FIELDS = ("height", "elevation_thr", "flatness_thr", "n_elevation", "n_flatness")


def _host(G):
    import torch
    return {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in G.items()}


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else (np.uint64 if a.dtype == np.float64 else a.dtype))


class GetterPair(RingPair):
    """A ring-bound context with getter results and its twins: RingPair's, and `tw`, which runs one present frame per call."""

    def __init__(self, *a, what=(True, True, True), **k):
        super().__init__(*a, **k)
        import pwpp_b200
        with self.kernels():
            self.tw = pwpp_b200.Engine(self._single, device=0, num_streams=self.ns)
        self.tw.set_output_order(self.order)
        self.what = what
        if any(what):
            self.eng.bind_getter_results(*what)

    def frame_read(self, f):
        """(pointer, size) of the records frame f of the last run segmented (size 0 for an invalid slot or count)."""
        r, s = self.ring_of[f], self.slot_list[f]
        if not 0 <= s < self.S:
            return self.slot_ptr(f, 0), 0
        c = int(self.rings[r][1][s].item())
        return (self.slot_ptr(f, s), c) if 0 <= c <= self.max_n[f] else (self.slot_ptr(f, 0), 0)

    def check(self, what):
        super().check(what)
        self.check_getters(what)

    def check_getters(self, what):
        import torch
        torch.cuda.synchronize()
        G = _host(self.eng.bound_getter_results())
        ro = G["row_off"]
        assert ro.tolist() == np.cumsum([0] + self.max_n).tolist()
        assert (G["ground_xyz"] is None) == (not self.what[0]) and (G["nonground_xyz"] is None) == (not self.what[1])
        assert (G["xyz_counts"] is None) == (not (self.what[0] or self.what[1])) and (G["height"] is None) == (not self.what[2])
        for f, s in enumerate(self.streams):
            empty = np.zeros((0, 3), np.float32)
            want = {"g": empty, "n": empty, "c": empty, "nm": empty}
            if self.acts[f] in (RUN, RESET):
                if self.acts[f] == RESET:
                    self.tw.reset(s)
                ptr, n = self.frame_read(f)
                self.tw.estimate_device_records([ptr], [n], [self.lays[f]], streams=[s])
                self.tw.synchronize()
                want = {"g": self.tw.ground_xyz(0), "n": self.tw.nonground_xyz(0), "c": self.tw.centers(0), "nm": self.tw.normals(0)}
            ng, nn, npch = len(want["g"]), len(want["n"]), len(want["c"])
            if G["xyz_counts"] is not None:
                assert G["xyz_counts"][f].tolist() == [ng, nn], f"{what}: frame {f} xyz counts"
            for key, part in (("ground_xyz", "g"), ("nonground_xyz", "n")):
                if G[key] is not None:
                    rows = G[key][ro[f]: ro[f] + len(want[part])]
                    assert np.array_equal(_bits(rows), _bits(want[part])), f"{what}: frame {f} {key}"
            assert int(G["num_patches"][f]) == npch, f"{what}: frame {f} num_patches"
            assert np.array_equal(_bits(G["centers"][f, :npch]), _bits(want["c"])), f"{what}: frame {f} centers"
            assert np.array_equal(_bits(G["normals"][f, :npch]), _bits(want["nm"])), f"{what}: frame {f} normals"
            if G["height"] is not None:
                st = self.tw.state(s)
                want_st = (np.float64(st.sensor_height), np.array(st.elevation_thr[:]), np.array(st.flatness_thr[:]),
                           np.array(st.n_elevation[:], np.int32), np.array(st.n_flatness[:], np.int32))
                for k, w in zip(STATE_FIELDS, want_st):
                    assert np.array_equal(_bits(np.atleast_1d(G[k][f])), _bits(np.atleast_1d(w))), f"{what}: frame {f} state {k}"


@pytest.fixture(scope="module")
def scans(kitti):
    return list(kitti)


def test_one_frame_kitti_graph_with_changing_counts(scans):
    """One KITTI frame captured in a CUDA graph and replayed with changing counts (0, 1, a part of the scan, the whole scan, an
    out-of-range count): before each replay both xyz buffers are filled with a sentinel, and no row past a count may change."""
    import torch
    sz = max(len(a) for a in scans)
    p = GetterPair([0], ["xyzi16"], [sz], num_slots=1, actions=False)
    G = p.eng.bound_getter_results()
    p.write(0, 0, scans[0], seed=0)
    p.set_slots([0])
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        p.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    for t, count in enumerate([None, 0, 1, 20000, None, sz + 1, None]):
        p.write(0, 0, scans[t % 6], seed=t, count=count)
        for key in ("ground_xyz", "nonground_xyz"):
            G[key].fill_(SENTINEL)
        torch.cuda.synchronize()
        g.replay()
        p.check(f"replay {t}, count {count}")
        c = G["xyz_counts"].cpu().numpy()
        for z, key in enumerate(("ground_xyz", "nonground_xyz")):
            assert (G[key][int(c[0, z]):].cpu().numpy() == np.float32(SENTINEL)).all(), f"replay {t}: {key} written past its count"


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
def test_sixteen_sensors_on_rings_with_actions(scans, order):
    """16 sensors of three layouts (16-byte, velodyne22, FLOAT64 xyz) on 3-slot rings, record results on beside the getters,
    captured once and replayed with a seeded schedule of SKIP, RESET, invalid actions, invalid slots and out-of-range counts
    (RESET with count 0 included)."""
    import torch
    nf = 16
    names = [["xyzi16", "velodyne22", "f64_xyz"][f % 3] for f in range(nf)]
    sz = max(len(a) for a in scans)
    p = GetterPair(list(range(nf)), names, [sz + 11 * f for f in range(nf)], num_slots=3, order=order, record_results=True)
    rng = np.random.default_rng(16 + order)
    cur = [0] * nf
    for f in range(nf):
        p.write(f, 0, scans[f % 6], seed=f)
    p.set_slots(cur, [RUN] * nf)
    p.eng.run_bound_call()
    p.check("eager run")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        p.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    for t in range(10):
        acts = ragged(rng, nf, 0.15, 0.1)
        acts[t % nf] = INVALID + 40
        slots = list(cur)
        for f in range(nf):
            if acts[f] == SKIP:
                continue
            nxt = (cur[f] + 1) % 3
            count = None
            if f == (3 * t + 1) % nf:
                count = sz + 999   # out of range
            elif f == (5 * t + 2) % nf:
                count, acts[f] = 0, RESET   # reset only
            p.write(f, nxt, scans[(f + t + 1) % 6], seed=1000 * t + f, count=count)
            cur[f] = slots[f] = nxt
        slots[(7 * t + 3) % nf] = [-1, 3, I32_MAX][t % 3]   # an invalid slot
        p.set_slots(slots, acts)
        g.replay()
        p.check(f"replay {t}")


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
def test_backlog_stream_bound_twice(scans, order):
    """One sensor's backlog: stream 0 bound twice on one ring (the second entry reads the next slot, or is skipped). Its two state
    rows are the twin's state after each of its two direct calls: the state launch runs after each of the call's two runs."""
    sz = max(len(a) for a in scans)
    p = GetterPair([0, 1, 0], ["velodyne22", "xyzi16", "velodyne22"], [sz] * 3, num_slots=4, ring_of=[0, 1, 0], order=order)
    t = 0
    for k in range(6):
        backlog = k % 3 != 1
        s0 = t % 4
        p.write(0, s0, scans[t % 6], seed=t)
        if backlog:
            p.write(0, (t + 1) % 4, scans[(t + 1) % 6], seed=t + 1)
        p.write(1, k % 4, scans[(k + 2) % 6], seed=50 + k)
        p.set_slots([s0, k % 4, (t + 1) % 4 if backlog else I32_MAX], [RUN if k != 3 else RESET, RUN, RUN if backlog else SKIP])
        p.eng.run_bound_call()
        p.check(f"run {k}")
        t += 2 if backlog else 1


@pytest.mark.parametrize("what", [(True, False, False), (False, True, False), (False, False, True), (True, True, False)],
                         ids=["ground", "nonground", "state", "xyz"])
def test_single_parts(scans, what):
    """Each part alone (and both xyz parts without the state): the other pointers are NULL, the enabled ones as with all parts."""
    sz = max(len(a) for a in scans)
    p = GetterPair([0, 1, 2], ["xyzi16", "velodyne22", "f64_xyz"], [sz] * 3, num_slots=2, what=what)
    for k in range(3):
        for r in range(3):
            p.write(r, k % 2, scans[(r + k) % 6], seed=10 * k + r)
        p.set_slots([k % 2] * 3, [RUN, SKIP if k == 1 else RUN, RESET if k == 2 else RUN])
        p.eng.run_bound_call()
        p.check(f"run {k}")


def test_graph_captured_before_the_enable_does_not_write(scans):
    """A graph captured before bind_getter_results replays without the getter launches: the buffers keep what they held."""
    import torch
    sz = max(len(a) for a in scans)
    p = GetterPair([0, 1], ["xyzi16", "velodyne22"], [sz] * 2, num_slots=1, actions=False, what=(False, False, False))
    for r in range(2):
        p.write(r, 0, scans[r], seed=r)
    p.set_slots([0, 0])
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        p.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    p.eng.bind_getter_results()
    p.what = (True, True, True)
    G = p.eng.bound_getter_results()
    for key in ("ground_xyz", "nonground_xyz"):
        G[key].fill_(SENTINEL)
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    for key in ("ground_xyz", "nonground_xyz"):
        assert (G[key].cpu().numpy() == np.float32(SENTINEL)).all(), key
    assert (G["xyz_counts"].cpu().numpy() == 0).all() and (G["height"].cpu().numpy() == 0).all()
    RingPair.check(p, "replay of the graph captured before the enable")   # the replay itself ran as usual
    for f, s in enumerate(p.streams):   # the getters' twin follows the streams
        ptr, n = p.frame_read(f)
        p.tw.estimate_device_records([ptr], [n], [p.lays[f]], streams=[s])
    p.eng.run_bound_call()   # a run after the enable writes them
    p.check("run after the enable")


def test_direct_call_between_replays_leaves_xyz_and_state(scans):
    """A direct call between two runs never writes the xyz or state buffers (it does overwrite the patch rows)."""
    import torch
    sz = max(len(a) for a in scans)
    p = GetterPair([0, 1], ["xyzi16", "velodyne22"], [sz] * 2, num_slots=1, actions=False)
    for r in range(2):
        p.write(r, 0, scans[r + 2], seed=r)
    p.set_slots([0, 0])
    p.eng.run_bound_call()
    p.check("first run")
    before = {k: v.clone() for k, v in p.eng.bound_getter_results().items() if isinstance(v, torch.Tensor) and k not in ("centers", "normals", "num_patches")}
    p.eng.estimate_host([scans[5]], streams=[1])
    p.eng.synchronize()
    after = p.eng.bound_getter_results()
    for k, v in before.items():
        assert torch.equal(_bits_t(v), _bits_t(after[k])), k
    p.tw.estimate_host([scans[5]], streams=[1])   # the twin follows the stream
    p.twin.estimate_host([scans[5]], streams=[1])
    p.eng.run_bound_call()
    p.check("run after the direct call")


def _bits_t(t):
    import torch
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int64)


def test_launch_count_errors_and_unbind(scans):
    """One xyz launch per run with either xyz part, one state launch per run of the call, nothing for the patches; the enable's
    errors; unbind releases the buffers and a later bind starts with the results off."""
    import torch
    import pwpp_b200
    sz = max(len(a) for a in scans)
    streams = [2, 0, 2, 1, 0]   # runs [0, 2), [2, 5): two runs

    def launches(what):
        p = GetterPair(streams, ["xyzi16"] * 5, [sz] * 5, num_slots=1, ring_of=[0, 1, 2, 3, 4], what=what)
        for r in range(5):
            p.write(r, 0, scans[r], seed=r)
        p.set_slots([0] * 5, [RUN] * 5)
        l0 = p.eng.launch_count()
        p.eng.run_bound_call()
        torch.cuda.synchronize()
        return p.eng.launch_count() - l0, p
    base, p = launches((False, False, False))
    assert launches((True, False, False))[0] == base + 1
    assert launches((True, True, False))[0] == base + 1
    assert launches((False, False, True))[0] == base + 2
    assert launches((True, True, True))[0] == base + 3
    e = p.eng
    for what in (0, 8, -1):
        assert e.lib.pwpp_bind_getter_results(e._h, what) == ERR_INVALID_ARG
        assert "what must be" in e.lib.pwpp_last_error().decode()
    e.bind_getter_results(state=False)
    with pytest.raises(pwpp_b200.PwppError, match="already enabled"):
        e.bind_getter_results()
    assert e.lib.pwpp_bound_getter_results(e._h, None) == ERR_INVALID_ARG
    e.unbind_call()
    with pytest.raises(pwpp_b200.PwppError, match="no call is bound"):
        e.bind_getter_results()
    with pytest.raises(pwpp_b200.PwppError, match="no call is bound"):
        e.bound_getter_results()
    g = pwpp_b200.PwppBoundGetters()
    assert e.lib.pwpp_bound_getter_results(e._h, C.byref(g)) == ERR_INVALID_ARG
    e.bind_call([p.slot_ptr(0, 0)], [sz], [p.lays[0]], torch.zeros(1, dtype=torch.int64, device="cuda"), streams=[0])
    G = e.bound_getter_results()
    assert G["ground_xyz"] is None and G["nonground_xyz"] is None and G["xyz_counts"] is None and G["height"] is None
    assert G["centers"] is not None and G["num_patches"].shape == (1,)
    e.unbind_call()


def test_fixture_scans_against_the_oracle(kitti):
    """The six fixture scans in one bound call of default parameters: every frame's ground xyz rows are the oracle's ground
    points and its non-ground rows the oracle's non-ground points."""
    import torch
    import oracle_py as O
    import pwpp_b200
    eng = pwpp_b200.Engine(device=0, num_streams=6)
    lay = pwpp_b200.layout_from_dtype(LAYOUTS["xyzi16"])
    bufs = [torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in kitti]
    counts = torch.tensor([len(a) for a in kitti], dtype=torch.int64, device="cuda")
    eng.bind_call(bufs, [len(a) for a in kitti], [lay] * 6, counts)
    eng.bind_getter_results()
    eng.run_bound_call()
    torch.cuda.synchronize()
    G = _host(eng.bound_getter_results())

    def rows(a):
        a = np.ascontiguousarray(a, np.float32)
        return np.sort(a.view(np.uint32).view([("x", "<u4"), ("y", "<u4"), ("z", "<u4")]).reshape(-1))
    for f, a in enumerate(kitti):
        orc = O.Oracle(arith=O.ARITH_CANON64)
        orc.estimate(np.ascontiguousarray(a, np.float32))
        ng, nn = G["xyz_counts"][f]
        o = G["row_off"][f]
        assert np.array_equal(rows(G["ground_xyz"][o:o + ng]), rows(orc.getGround())), f"scan {f}: ground"
        assert np.array_equal(rows(G["nonground_xyz"][o:o + nn]), rows(orc.getNonground())), f"scan {f}: non-ground"
    eng.unbind_call()
