"""Bound calls over scan rings (pwpp_bind_call_rings): the slot of every frame is read on the GPU at every run or replay, and the
scan is segmented where it was written.

Every run is compared bit for bit with a twin context driven by pwpp_estimate_device_records on the records of the slots read,
naming only the present frames (as test_gpu_bound_actions.py does): every present frame's results at its position in the bound
call, the empty results of skipped frames, d_status, the offsets, num_ground, both record parts and every stream's state,
histories and export blob. The identity case compares a ring-bound context with one bound by pwpp_bind_call_actions instead."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_bound_actions import INVALID, OUT_OF_RANGE, RESET, RUN, SKIP, SKIPPED, ActionPair, batch_kernels, ragged, storage20
from test_gpu_bound_call import NAMES, engine
from test_gpu_records import LAYOUTS, _dt, outputs, records, stream

pytestmark = pytest.mark.gpu

SLOT_OUT_OF_RANGE = 4
ERR_INVALID_ARG = -1
I32_MAX = 2 ** 31 - 1
LAYOUTS = dict(LAYOUTS, f64_rec48=_dt(["x", "y", "z", "intensity", "t"], ["<f8", "<f8", "<f8", "<f4", "<f8"], [0, 8, 16, 24, 32], 48))


@pytest.fixture(scope="module")
def scans(kitti):
    return list(kitti)


class RingPair(ActionPair):
    """A ring-bound context and its twin. Ring r has num_slots slots of names of its first frame; frame f reads ring ring_of[f].
    Rings are bound alternately as (uint8 (num_slots, stride) buffer, counts) and as (misaligned flat buffer, counts, stride)."""

    def __init__(self, streams, names, max_n, num_slots=3, ring_of=None, order=0, single=None, actions=True, record_results=False):
        import torch
        import pwpp_b200
        nf = len(streams)
        self.streams, self.names, self.max_n = list(streams), list(names), [int(k) for k in max_n]
        self.ring_of = list(range(nf)) if ring_of is None else list(ring_of)
        self.ns = max(streams) + 1
        self.order, self._single, self._sets = order, single or storage20(), None
        self.kernels, self.run_starts = batch_kernels, set()
        with self.kernels():
            self.eng, self.twin = [pwpp_b200.Engine(self._single, device=0, num_streams=self.ns) for _ in range(2)]
        for e in (self.eng, self.twin):
            e.set_output_order(order)
        self.lays = [pwpp_b200.layout_from_dtype(LAYOUTS[nm]) for nm in names]
        self.S = num_slots
        self.rings, self.ring_desc = {}, []
        for r in sorted(set(self.ring_of)):
            fr = [f for f in range(nf) if self.ring_of[f] == r]
            step = LAYOUTS[names[fr[0]]].itemsize
            stride = max(self.max_n[f] for f in fr) * step + 3 * r
            counts = torch.zeros(num_slots, dtype=torch.int64, device="cuda")
            if r % 2 == 0:
                buf = torch.zeros(num_slots, stride, dtype=torch.uint8, device="cuda")
                self.rings[r] = (buf, counts, buf.data_ptr(), stride)
                self.ring_desc.append((buf, counts))
            else:
                mis = 1 + (5 * r) % 15
                flat = torch.zeros(mis + num_slots * stride, dtype=torch.uint8, device="cuda")
                self.rings[r] = (flat[mis:], counts, flat.data_ptr() + mis, stride)
                self.ring_desc.append((flat[mis:], counts, stride))
        descs = {r: d for r, d in zip(sorted(self.rings), self.ring_desc)}
        self.slots = torch.zeros(nf, dtype=torch.int32, device="cuda")
        self.actions = torch.zeros(nf, dtype=torch.int32, device="cuda") if actions else None
        self.eng.bind_call_rings([descs[r] for r in self.ring_of], self.max_n, self.lays, self.slots, streams=self.streams, actions=self.actions)
        if record_results:
            self.eng.bind_record_results()
        self.records = record_results
        self._empty = {}
        self.acts = [RUN] * nf

    def slot_ptr(self, f, s):
        _, _, base, stride = self.rings[self.ring_of[f]]
        return base + s * stride

    def write(self, r, s, scan, seed, count=None):
        """Writes the records of scan into slot s of ring r and its count (default: the records written)."""
        import torch
        buf, counts, base, stride = self.rings[r]
        f = self.ring_of.index(r)
        a = scan[: self.max_n[f]]
        rec, _ = records(a, LAYOUTS[self.names[f]], seed=seed)
        flat = buf.view(-1)
        if len(rec):
            flat[s * stride: s * stride + rec.nbytes].copy_(torch.from_numpy(rec.view(np.uint8).copy()).cuda(non_blocking=False))
        counts[s] = len(rec) if count is None else count

    def set_slots(self, slots, acts=None):
        import torch
        self.slots.copy_(torch.tensor(list(slots), dtype=torch.int32))
        if acts is not None:
            self.actions.copy_(torch.tensor(list(acts), dtype=torch.int32))
            self.acts = [int(a) for a in acts]
        torch.cuda.synchronize()
        self.slot_list = [int(s) for s in slots]

    def check(self, what):
        """The last run against the twin, which runs the present frames at the slots they read."""
        import torch
        torch.cuda.synchronize()
        nf = len(self.streams)
        idx, off, ng, st = self.eng.bound_call_results()
        self.eng.synchronize()
        present = [a in (RUN, RESET) for a in self.acts]
        sizes, ptrs, want_st = [], [], []
        for f in range(nf):
            r, s = self.ring_of[f], self.slot_list[f]
            _, counts, _, _ = self.rings[r]
            if not present[f]:
                sizes.append(0); ptrs.append(self.slot_ptr(f, 0)); want_st.append(SKIPPED if self.acts[f] == SKIP else INVALID)
            elif not 0 <= s < self.S:
                sizes.append(0); ptrs.append(self.slot_ptr(f, 0)); want_st.append(SLOT_OUT_OF_RANGE)
            else:
                c = int(counts[s].item())
                ok = 0 <= c <= self.max_n[f]
                sizes.append(c if ok else 0); ptrs.append(self.slot_ptr(f, s)); want_st.append(0 if ok else OUT_OF_RANGE)
        assert st.cpu().numpy().tolist() == want_st, f"{what}: status"
        assert np.array_equal(off.cpu().numpy(), np.concatenate([[0], np.cumsum(sizes)])), f"{what}: offsets"
        want_slots = [s if p else -1 for s, p in zip(self.slot_list, present)]
        assert self.eng.bound_call_slots().cpu().numpy().tolist() == want_slots, f"{what}: slots read"
        ngs = ng.cpu().numpy()
        got = [outputs(self.eng, f) for f in range(nf)]
        if self.records:
            gb, nb, roff, rcnt = self.eng.bound_record_results()
            bufs, rcnt = [gb.cpu().numpy(), nb.cpu().numpy()], rcnt.cpu().numpy()
        seg = []

        def flush():
            if not seg:
                return
            self.twin.estimate_device_records([ptrs[f] for f in seg], [sizes[f] for f in seg], [self.lays[f] for f in seg],
                                              streams=[self.streams[f] for f in seg])
            self.twin.synchronize()
            for k, f in enumerate(seg):
                assert got[f] == outputs(self.twin, k), f"{what}: frame {f}"
                assert ngs[f] == self.twin.num_ground(k), f"{what}: frame {f} num_ground"
                if self.records:
                    step = LAYOUTS[self.names[f]].itemsize
                    want = [self.twin.num_ground(k), self.twin.num_nonground(k)]
                    assert rcnt[f].tolist() == want, f"{what}: frame {f} record counts"
                    for z, tw in enumerate((self.twin.ground_records(k), self.twin.nonground_records(k))):
                        region = bufs[z][roff[f]: roff[f + 1]]
                        assert np.array_equal(region[:want[z] * step], np.ascontiguousarray(tw).view(np.uint8).reshape(-1)), f"{what}: frame {f} part {z}"
            seg.clear()

        for f in range(nf):
            if not present[f]:
                self.ptrs = ptrs
                assert got[f] == self.empty(f), f"{what}: skipped frame {f}"
                assert ngs[f] == 0
                if self.records:
                    assert rcnt[f].tolist() == [0, 0]
                continue
            if self.acts[f] == RESET:
                flush()
                self.twin.reset(self.streams[f])
            seg.append(f)
        flush()
        for s in sorted(set(self.streams)):
            assert stream(self.eng, s) == stream(self.twin, s), f"{what}: stream {s}"


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
def test_one_slot_rings_equal_bind_call_actions(scans, order):
    """pwpp_bind_call_actions(frames, max_n, layouts, d_counts, d_actions) is the ring call with one-slot rings
    {frames[f], max_n[f] * point_step, d_counts + f, 1} and slots all zero: results, record parts, state and launch counts
    bit for bit over several runs with ragged actions."""
    import torch
    import pwpp_b200
    sz = max(len(a) for a in scans)
    streams = [4, 0, 3, 1, 2, 0]
    p = ActionPair(streams, NAMES + ["velodyne22", "xyzi16"], [sz + 7 * k for k in range(6)], order, single=storage20())
    with batch_kernels():
        q = pwpp_b200.Engine(storage20(), device=0, num_streams=5)
    q.set_output_order(order)
    rings = [(p.bufs[f][0][p.bufs[f][1]:], p.counts[f:f + 1], p.max_n[f] * LAYOUTS[p.names[f]].itemsize) for f in range(6)]
    slots = torch.zeros(6, dtype=torch.int32, device="cuda")
    q.bind_call_rings(rings, p.max_n, p.lays, slots, streams=streams, actions=p.actions)
    assert [r[0].data_ptr() for r in rings] == p.ptrs
    for e in (p.eng, q):
        e.bind_record_results()
    rng = np.random.default_rng(order)
    for k in range(4):
        p.load(scans, k, None if k != 2 else [5, -1, sz + 1, 0, 100, 2 ** 40])
        p.set_actions([RUN] * 6 if k == 0 else ragged(rng, 6, 0.3, 0.2))
        l0, m0 = p.eng.launch_count(), q.launch_count()
        p.eng.run_bound_call()
        q.run_bound_call()
        assert p.eng.launch_count() - l0 == q.launch_count() - m0
        r1, r2 = p.eng.bound_call_results(), q.bound_call_results()
        p.eng.synchronize()
        q.synchronize()
        for a, b in zip(r1, r2):
            assert np.array_equal(a.cpu().numpy(), b.cpu().numpy()), f"run {k}: device results"
        g1, n1, o1, c1 = p.eng.bound_record_results()
        g2, n2, o2, c2 = q.bound_record_results()
        assert np.array_equal(o1, o2) and torch.equal(c1, c2), f"run {k}: record counts"
        for f in range(6):
            o, m = int(o1[f]), int(c1[f, 0])
            st = LAYOUTS[p.names[f]].itemsize
            assert torch.equal(g1[o:o + m * st], g2[o:o + m * st]) and torch.equal(n1[o:o + int(c1[f, 1]) * st], n2[o:o + int(c1[f, 1]) * st])
            assert outputs(p.eng, f) == outputs(q, f), f"run {k}: frame {f}"
        for s in range(5):
            assert stream(p.eng, s) == stream(q, s), f"run {k}: stream {s}"
        want = [0 if a in (RUN, RESET) else -1 for a in p.acts]
        assert q.bound_call_slots().cpu().numpy().tolist() == want


def test_sixteen_sensors_in_a_captured_graph(scans):
    """16 sensors on 3-slot rings of three layouts, captured once in a torch CUDA graph and replayed 24 times with a seeded slot
    and action schedule. Between replays a copy kernel on the same stream writes the next scan into the slot no run is reading
    ((t + 1) % 3) and the producer publishes it; record results on."""
    import torch
    nf = 16
    names = [["pcl_xyzi32", "velodyne22", "f64_rec48"][f % 3] for f in range(nf)]
    sz = max(len(a) for a in scans)
    p = RingPair(list(range(nf)), names, [sz + 11 * f for f in range(nf)], num_slots=3, record_results=True)
    rng = np.random.default_rng(16)
    cur = [0] * nf
    for f in range(nf):
        p.write(f, 0, scans[f % 6], seed=f)
    p.set_slots(cur, [RUN] * nf)
    p.eng.run_bound_call()
    p.check("eager run")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        p.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    for t in range(24):
        acts = ragged(rng, nf, 0.1, 0.05)
        for f in range(nf):   # the producer: a new scan for most sensors, written into the slot after the current one
            if acts[f] == SKIP:
                continue
            nxt = (cur[f] + 1) % 3
            p.write(f, nxt, scans[(f + t + 1) % 6], seed=1000 * t + f, count=None if rng.random() > 0.05 else sz + 999)
            cur[f] = nxt
        p.set_slots(cur, acts)
        g.replay()
        p.check(f"replay {t}")


def test_invalid_slots_skip_with_garbage_and_reset(scans):
    """Invalid slots (-1, num_slots, INT_MAX) give status 4 and the twin's empty-frame state, the other frames unaffected; SKIP
    with a garbage slot and count; RESET with an invalid slot resets the stream and runs it empty."""
    sz = max(len(a) for a in scans)
    p = RingPair([0, 1, 2, 3], ["xyzi16", "velodyne22", "pcl_xyzi32", "f64_xyz"], [sz] * 4, num_slots=2)
    for r in range(4):
        for s in range(2):
            p.write(r, s, scans[(r + s) % 6], seed=10 * r + s)
    for k, (slots, acts) in enumerate([([0, 1, 0, 1], [RUN] * 4), ([-1, 2, I32_MAX, 0], [RUN] * 4), ([1, 0, 1, 0], [RUN] * 4),
                                       ([I32_MAX, 0, -7, 1], [SKIP, RUN, 9, RUN]), ([5, 1, 0, -1], [RESET, RUN, RUN, RESET]),
                                       ([0, 1, 0, 1], [RUN, RESET, SKIP, RUN])]):
        if k == 3:   # garbage counts in the slots the skipped frames would name
            p.rings[0][1].fill_(-5)
            p.rings[2][1].fill_(2 ** 62)
        if k == 4:
            for r in (0, 2):
                for s in range(2):
                    p.write(r, s, scans[(r + s + 3) % 6], seed=100 + 10 * r + s)
        p.set_slots(slots, acts)
        p.eng.run_bound_call()
        p.check(f"run {k}: slots {slots} actions {acts}")


def test_backlog_one_ring_two_entries(scans):
    """One sensor's backlog: its ring bound to two entries of stream 0 (the second reads the next slot, or is skipped when there
    is no backlog), beside a sensor of its own."""
    sz = max(len(a) for a in scans)
    p = RingPair([0, 1, 0], ["velodyne22", "xyzi16", "velodyne22"], [sz] * 3, num_slots=4, ring_of=[0, 1, 0])
    t = 0
    for k in range(8):
        backlog = k % 3 == 1
        s0 = t % 4
        p.write(0, s0, scans[t % 6], seed=t)
        if backlog:
            p.write(0, (t + 1) % 4, scans[(t + 1) % 6], seed=t + 1)
        p.write(1, k % 4, scans[(k + 2) % 6], seed=50 + k)
        p.set_slots([s0, k % 4, (t + 1) % 4 if backlog else I32_MAX], [RUN, RUN, RUN if backlog else SKIP])
        p.eng.run_bound_call()
        p.check(f"run {k}")
        t += 2 if backlog else 1


def test_slots_rewritten_after_the_run(scans):
    """d_slots rewritten after a replay without a host synchronisation: bound_call_slots keeps what the run used."""
    import torch
    sz = max(len(a) for a in scans)
    p = RingPair([0, 1], ["xyzi16", "pcl_xyzi32"], [sz] * 2, num_slots=3, actions=False)
    assert p.eng.bound_call_slots().cpu().numpy().tolist() == [-1, -1]
    for r in range(2):
        for s in range(3):
            p.write(r, s, scans[(r + s) % 6], seed=r * 3 + s)
    p.set_slots([2, 1])
    p.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    p.slots.copy_(torch.tensor([0, 5], dtype=torch.int32, device="cuda"))   # (stream-ordered after the run, no host synchronisation)
    torch.cuda.synchronize()
    assert p.eng.bound_call_slots().cpu().numpy().tolist() == [2, 1]
    p.check("slots rewritten after the run")


def test_launch_count_rule(scans):
    """A ring-bound call launches exactly what the same call bound with pwpp_bind_call_actions launches, with and without
    actions, repeated streams included."""
    import torch
    sz = max(len(a) for a in scans)
    streams = [2, 0, 2, 1, 3, 0, 1]
    for actions in (False, True):
        p = RingPair(streams, [NAMES[f % 4] for f in range(7)], [sz] * 7, num_slots=2, actions=actions)
        with batch_kernels():
            plain = engine(4, 0)
        bufs = [torch.zeros(sz * 48, dtype=torch.uint8, device="cuda") for _ in range(7)]
        counts = torch.zeros(7, dtype=torch.int64, device="cuda")
        plain.bind_call([b.data_ptr() for b in bufs], [sz] * 7, p.lays, counts, streams=streams,
                        actions=torch.zeros(7, dtype=torch.int32, device="cuda") if actions else None)
        p.set_slots([0] * 7, [RESET] * 7 if actions else None)
        l0, m0 = p.eng.launch_count(), plain.launch_count()
        p.eng.run_bound_call()
        plain.run_bound_call()
        assert p.eng.launch_count() - l0 == plain.launch_count() - m0
        torch.cuda.synchronize()


def test_bind_errors(scans):
    import torch
    import pwpp_b200
    e = engine(4, 0)
    lay = pwpp_b200.layout_from_dtype(LAYOUTS["xyzi16"])
    buf = torch.zeros(16 * 1000 * 3, dtype=torch.uint8, device="cuda")
    counts = torch.zeros(3, dtype=torch.int64, device="cuda")
    slots = torch.zeros(4, dtype=torch.int32, device="cuda")
    nf = 4

    def call(descs, d_slots=slots.data_ptr(), max_n=1000, ids=(0, 1, 2, 3)):
        arr = (pwpp_b200.PwppScanRing * nf)()
        for f, (base, stride, cnt, ns) in enumerate(descs):
            arr[f].base, arr[f].slot_stride, arr[f].d_counts, arr[f].num_slots = base, stride, cnt, ns
        rc = e.lib.pwpp_bind_call_rings(e._h, nf, np.array(ids, np.int32).ctypes.data, arr, (C.c_int64 * nf)(*[max_n] * nf),
                                        (pwpp_b200.PwppPointLayout * nf)(*[lay] * nf), C.c_void_p(d_slots), None)
        return rc, e.lib.pwpp_last_error().decode()

    good = (buf.data_ptr(), 16000, counts.data_ptr(), 3)
    for bad, msg in (((0, 16000, counts.data_ptr(), 3), "NULL"), ((buf.data_ptr(), 16000, 0, 3), "d_counts"), ((buf.data_ptr(), 16000, counts.data_ptr(), 0), "num_slots"),
                     ((buf.data_ptr(), 15999, counts.data_ptr(), 3), "slot_stride"), ((buf.data_ptr(), 2 ** 62, counts.data_ptr(), 3), "overflows"),
                     ((buf.data_ptr(), -1, counts.data_ptr(), 3), "slot_stride")):
        rc, err = call([good, good, bad, good])
        assert rc == ERR_INVALID_ARG and "frame 2" in err and msg in err, err
    rc, err = call([good] * 4, d_slots=0)
    assert rc == ERR_INVALID_ARG and "d_slots" in err
    rc, err = call([good, good, good, good], ids=(0, 1, 9, 2))
    assert rc == ERR_INVALID_ARG and "frame 2" in err
    rc = e.lib.pwpp_bind_call_rings(e._h, nf, np.arange(4, dtype=np.int32).ctypes.data, None, (C.c_int64 * nf)(*[1000] * nf),
                                    (pwpp_b200.PwppPointLayout * nf)(*[lay] * nf), C.c_void_p(slots.data_ptr()), None)
    assert rc == ERR_INVALID_ARG and "rings" in e.lib.pwpp_last_error().decode()
    rc, err = call([(0, 0, counts.data_ptr(), 1)] * 4, max_n=0)   # NULL base is fine when max_n is 0
    assert rc == 0, err
    with pytest.raises(pwpp_b200.PwppError, match="already bound"):
        e.bind_call([buf.data_ptr()] * 4, [1000] * 4, [lay] * 4, torch.zeros(4, dtype=torch.int64, device="cuda"))
    e.unbind_call()
    with pytest.raises(pwpp_b200.PwppError, match="no call is bound"):
        e.bound_call_slots()
    e.bind_call([buf.data_ptr()] * 4, [1000] * 4, [lay] * 4, torch.zeros(4, dtype=torch.int64, device="cuda"))
    with pytest.raises(pwpp_b200.PwppError, match="no rings"):
        e.bound_call_slots()
    e.unbind_call()
    ring = (buf.view(3, 16000), counts)
    for bad, msg in (((buf, counts), "first dimension"), ((buf.view(3, 16000), counts.int()), "counts"), ((buf[1:], counts, 16000), "past the buffer")):
        with pytest.raises(pwpp_b200.PwppError, match=msg):
            e.bind_call_rings([ring, ring, bad, ring], [1000] * 4, [lay] * 4, slots)
    for bad in (slots.to(torch.int64), slots[:3], slots.cpu()):
        with pytest.raises(pwpp_b200.PwppError, match="slots"):
            e.bind_call_rings([ring] * 4, [1000] * 4, [lay] * 4, bad)
    e.bind_call_rings([ring] * 4, [1000] * 4, [lay] * 4, slots)
    e.unbind_call()
