"""Packed records of bound calls (pwpp_bind_packed_records) on the GPU, through the C-ABI and the Engine.

After every run the packed parts are compared byte for byte with two independent references: the capacity-layout record
results of the same run (pwpp_bind_record_results, enabled on the same call) compacted in numpy by their count pairs, and
records[idx] taken from the frame's source bytes with the bound call's own index lists. The offsets must equal numpy's
exclusive scan of the count pairs, and no byte past the total may change. Every bind kind (plain, actions, rings, packed) with
velodyne22, pcl_xyzi32 and float32 (N, 4) records; CUDA graph replays with changing counts, slots and offsets, with every kind
of action and invalid entry, in both output orders; packed xyz beside packed records; one part only; an enable after a capture;
a direct call between runs; the launch-count rule; the errors and unbind."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_bound_actions import INVALID, OUT_OF_RANGE, RESET, RUN, SKIP
from test_gpu_records import LAYOUTS, records

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_UNSUPPORTED = -1, -4
SENTINEL = 0xA5
BIND_KINDS = ["plain", "actions", "rings", "packed"]
RECORD_KINDS = ["velodyne22", "pcl_xyzi32", "f32x4"]


@pytest.fixture(scope="module")
def scans(kitti):
    import synth
    return [kitti[0], kitti[1][:40000], synth.make_frame(1, 3).numpy()[:30000], kitti[3][:20000], synth.make_frame(1, 4).numpy()[:5000],
            kitti[5][:60000]]


def layout_of(kind):
    import pwpp_b200
    if kind == "f32x4":
        dt = np.dtype({"names": ["x", "y", "z", "intensity"], "formats": ["<f4"] * 4, "offsets": [0, 4, 8, 12], "itemsize": 16})
    else:
        dt = LAYOUTS[kind]
    return dt, pwpp_b200.layout_from_dtype(dt)


class Rig:
    """A bound call over `scans` as records of `kind`, bound as `bind`, with record results and packed records enabled.
    host[f] holds every byte frame f may read (uint8, rows of step); set() chooses what the next run reads, want() says which
    rows of host[f] each frame reads under the bind's rules."""

    SLACK = 50

    def __init__(self, scans, kind, bind, order=0, parts=3, record_results=True):
        import torch
        import pwpp_b200
        self.kind, self.bind, self.nf = kind, bind, len(scans)
        dt, self.lay = layout_of(kind)
        self.step = dt.itemsize
        rng = np.random.default_rng(11)
        self.max_n = [len(a) + self.SLACK for a in scans]
        self.rows = [len(a) for a in scans]

        def recs(a, k):
            if kind == "f32x4":
                return np.ascontiguousarray(a[:, :4]).astype(np.float32).view(np.uint8).reshape(len(a), 16)
            return np.ascontiguousarray(records(a, dt, seed=k)[0]).view(np.uint8).reshape(len(a), self.step)

        def junk(n):
            if kind == "f32x4":
                return rng.uniform(-30, 30, (n, 4)).astype(np.float32).view(np.uint8).reshape(n, 16)
            return rng.integers(0, 256, (n, self.step), dtype=np.uint8)
        self.eng = pwpp_b200.Engine(device=0, num_streams=self.nf)
        self.eng.set_output_order(order)
        self.actions = torch.zeros(self.nf, dtype=torch.int32, device="cuda") if bind != "plain" else None
        self.acts = [RUN] * self.nf
        if bind in ("plain", "actions"):
            self.host = [np.concatenate([recs(a, k), junk(self.SLACK)]) for k, a in enumerate(scans)]
            self.bufs = [torch.from_numpy(h.reshape(-1).copy()).cuda() for h in self.host]
            self.counts = torch.tensor(self.rows, dtype=torch.int64, device="cuda")
            self.cfg = list(self.rows)
            self.eng.bind_call(self.bufs, self.max_n, [self.lay] * self.nf, self.counts, actions=self.actions)
        elif bind == "rings":
            # two slots per ring: the scan, then the scan's rows in reverse (other records, same sizes)
            self.host = []
            self.ring_bufs, self.ring_counts = [], []
            for k, a in enumerate(scans):
                r = recs(a, k)
                slots = np.stack([np.concatenate([r, junk(self.SLACK)]), np.concatenate([r[::-1], junk(self.SLACK)])])
                self.host.append(slots)
                self.ring_bufs.append(torch.from_numpy(slots.reshape(2, -1).copy()).cuda())
                self.ring_counts.append(torch.tensor([len(a), len(a) - 7], dtype=torch.int64, device="cuda"))
            self.slots = torch.zeros(self.nf, dtype=torch.int32, device="cuda")
            self.cfg = ([0] * self.nf, [[len(a), len(a) - 7] for a in scans])
            self.eng.bind_call_rings(list(zip(self.ring_bufs, self.ring_counts)), self.max_n, [self.lay] * self.nf, self.slots,
                                     actions=self.actions)
        else:
            flat = np.concatenate([recs(a, k) for k, a in enumerate(scans)] + [junk(100)])
            self.host = flat
            self.capacity = len(flat)
            if kind == "f32x4":
                self.points = torch.from_numpy(flat.view(np.float32).reshape(-1, 4).copy()).cuda()
            else:
                self.points = torch.from_numpy(flat.reshape(-1).copy()).cuda()
            self.base_entries = np.concatenate([[0], np.cumsum(self.rows)]).tolist()
            self.offsets = torch.tensor(self.base_entries, dtype=torch.int64, device="cuda")
            self.cfg = list(self.base_entries)
            self.eng.bind_call_packed(self.points, self.offsets, self.max_n, layout=None if kind == "f32x4" else self.lay, actions=self.actions)
        if record_results:
            self.eng.bind_record_results()
        if parts:
            self.eng.bind_packed_records(ground=bool(parts & 1), nonground=bool(parts & 2))

    def set(self, cfg, acts=None):
        """The next run's counts (plain / actions), (slots, ring counts) (rings) or offsets entries (packed), and actions."""
        import torch
        self.cfg = cfg
        if self.bind in ("plain", "actions"):
            self.counts.copy_(torch.tensor(cfg, dtype=torch.int64))
        elif self.bind == "rings":
            self.slots.copy_(torch.tensor(cfg[0], dtype=torch.int32))
            for c, t in zip(cfg[1], self.ring_counts):
                t.copy_(torch.tensor(c, dtype=torch.int64))
        else:
            self.offsets.copy_(torch.tensor(cfg, dtype=torch.int64))
        if acts is not None:
            self.actions.copy_(torch.tensor(acts, dtype=torch.int32))
            self.acts = list(acts)
        torch.cuda.synchronize()

    def want(self):
        """For every frame, the rows it reads under the rules (an empty array for a skipped or invalid frame)."""
        out = []
        for f in range(self.nf):
            empty = np.empty((0, self.step), np.uint8)
            if self.acts[f] not in (RUN, RESET):
                out.append(empty)
            elif self.bind in ("plain", "actions"):
                c = self.cfg[f]
                out.append(self.host[f][:c] if 0 <= c <= self.max_n[f] else empty)
            elif self.bind == "rings":
                s = self.cfg[0][f]
                c = self.cfg[1][f][s] if 0 <= s < 2 else -1
                out.append(self.host[f][s][:c] if 0 <= c <= self.max_n[f] else empty)
            else:
                lo, hi = self.cfg[f], self.cfg[f + 1]
                ok = 0 <= lo <= hi <= self.capacity and hi - lo <= self.max_n[f]
                out.append(self.host[lo:hi] if ok else empty)
        return out

    def fill(self):
        """Sentinel in both packed parts before a run."""
        import torch
        P = self.eng.bound_packed_records()
        for key in ("ground", "nonground"):
            if P[key] is not None:
                P[key].fill_(SENTINEL)
        torch.cuda.synchronize()

    def random_cfg(self, rng, invalid=True):
        """A run's configuration: sizes anywhere up to max_n, some frames emptied; with `invalid`, out-of-range counts, slots
        and offsets; and actions with SKIP, RESET and invalid values when the bind has actions."""
        nf = self.nf
        acts = None
        if self.actions is not None:
            acts = [int(rng.choice([RUN, RUN, RUN, SKIP, RESET, 7 if invalid else RUN])) for _ in range(nf)]
        if self.bind in ("plain", "actions"):
            cfg = [int(rng.integers(0, self.max_n[f] + 1)) if rng.random() > 0.15 else 0 for f in range(nf)]
            if invalid:
                cfg[int(rng.integers(nf))] = -3
                cfg[int(rng.integers(nf))] = self.max_n[0] + 10 ** 6
        elif self.bind == "rings":
            slots = [int(rng.integers(0, 2)) for _ in range(nf)]
            counts = [[int(rng.integers(0, self.max_n[f] + 1)), int(rng.integers(0, self.max_n[f] + 1))] for f in range(nf)]
            if invalid:
                slots[int(rng.integers(nf))] = 5
                f = int(rng.integers(nf))
                counts[f][slots[f] if 0 <= slots[f] < 2 else 0] = self.max_n[f] + 1
            cfg = (slots, counts)
        else:
            sizes = [int(rng.integers(0, self.max_n[f] + 1)) if rng.random() > 0.15 else 0 for f in range(nf)]
            start = int(rng.integers(0, 40))
            cfg = [start] + [start + int(x) for x in np.cumsum(sizes)]
            cfg[-1] = min(cfg[-1], self.capacity)
            cfg = [min(x, cfg[-1]) for x in cfg]
            if invalid:
                k = int(rng.integers(1, nf))
                cfg[k] = cfg[k - 1] - 1 if cfg[k - 1] > 0 else -1   # a decreasing entry
        return cfg, acts

    def check(self, what, sentinel=True):
        """The last run's packed records against the compacted capacity-layout results and records[idx]; the offsets against
        the exclusive scan of the count pairs; nothing written past the total."""
        import torch
        torch.cuda.synchronize()
        idx, off, ng, st = (t.cpu().numpy() for t in self.eng.bound_call_results())
        self.eng.synchronize()
        P = self.eng.bound_packed_records()
        assert P["point_step"] == self.step
        w = self.want()
        assert np.array_equal(np.diff(off), [len(x) for x in w]), f"{what}: frame sizes"
        R = self.eng.bound_record_results()
        cnt = R[3].cpu().numpy().astype(np.int64)
        assert np.array_equal(cnt[:, 0], ng), f"{what}: ground counts"
        for z, key in enumerate(("ground", "nonground")):
            want_off = np.concatenate([[0], np.cumsum(cnt[:, z])])
            got_off = P[key + "_offsets"]
            if P[key] is None:
                assert got_off is None
                continue
            assert got_off.cpu().numpy().tolist() == want_off.tolist(), f"{what}: {key} offsets"
            total = int(want_off[-1]) * self.step
            buf = P[key].cpu().numpy().reshape(-1)
            # the capacity-layout results of the same run, compacted by their counts
            cap = R[z].cpu().numpy()
            compact = np.concatenate([cap[R[2][f]:R[2][f] + cnt[f, z] * self.step] for f in range(self.nf)])
            assert np.array_equal(buf[:total], compact), f"{what}: packed {key} differs from the record results"
            # records[idx] from the frame's own source rows and lists
            lists = [idx[off[f]:off[f] + ng[f]] if z == 0 else idx[off[f] + ng[f]:off[f] + ng[f] + cnt[f, 1]] for f in range(self.nf)]
            direct = np.concatenate([w[f][lists[f]].reshape(-1) for f in range(self.nf)] + [np.empty(0, np.uint8)])
            assert np.array_equal(buf[:total], direct), f"{what}: packed {key} differs from records[idx]"
            if sentinel:
                assert (buf[total:] == SENTINEL).all(), f"{what}: {key}: a byte past the total was written"
        return st


@pytest.mark.parametrize("kind", RECORD_KINDS)
@pytest.mark.parametrize("bind", BIND_KINDS)
def test_every_bind_kind(scans, bind, kind):
    """Two runs as bound (the stream state carries), then a run with changed sizes, slots or offsets and actions."""
    rig = Rig(scans, kind, bind)
    rng = np.random.default_rng(sum(map(ord, bind + kind)))
    for k in range(2):
        rig.fill()
        rig.eng.run_bound_call()
        rig.check(f"run {k}")
    cfg, acts = rig.random_cfg(rng)
    rig.set(cfg, acts)
    rig.fill()
    rig.eng.run_bound_call()
    rig.check("changed")


@pytest.mark.parametrize("order", [0, 1], ids=["order_bin", "order_reference"])
@pytest.mark.parametrize("bind", ["plain", "actions", "rings", "packed"])
def test_graph_replays(scans, bind, order):
    """One CUDA graph replayed 24 times with changing counts, slots and offsets, SKIP, RESET and invalid actions and
    out-of-range entries; each replay checked."""
    import torch
    kind = {"plain": "velodyne22", "actions": "f32x4", "rings": "pcl_xyzi32", "packed": "velodyne22"}[bind]
    rig = Rig(scans, kind, bind, order=order)
    rng = np.random.default_rng(100 + order + 7 * BIND_KINDS.index(bind))
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            rig.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    seen = set()
    for k in range(24):
        cfg, acts = rig.random_cfg(rng, invalid=k % 3 != 0)
        rig.set(cfg, acts)
        rig.fill()
        g.replay()
        torch.cuda.synchronize()
        seen |= set(rig.check(f"replay {k}").tolist())
    assert 0 in seen and len(seen) > 1, seen


def test_packed_xyz_beside_packed_records(scans):
    """Both enabled: the same two offsets arrays; for the float32 (N, 4) layout the first 12 bytes of every packed record are
    the packed xyz row, bit for bit."""
    import torch
    for bind in ("packed", "rings"):
        rig = Rig(scans, "f32x4", bind)
        rig.eng.bind_packed_xyz()
        rng = np.random.default_rng(5)
        for k in range(3):
            if k:
                rig.set(*rig.random_cfg(rng))
            rig.fill()
            rig.eng.run_bound_call()
            rig.check(f"{bind} run {k}")
            P, X = rig.eng.bound_packed_records(), rig.eng.bound_packed_xyz()
            for key in ("ground", "nonground"):
                assert P[key + "_offsets"].data_ptr() == X[key + "_offsets"].data_ptr(), key
                t = int(P[key + "_offsets"][-1])
                rec = P[key][:t].view(torch.float32)
                assert rec.shape == (t, 4)
                assert torch.equal(rec[:, :3].contiguous().view(torch.int32), X[key][:t].contiguous().view(torch.int32)), f"{bind} {key}"
        p = rig.eng.bound_packed_records()
        got = C.c_void_p(), C.c_void_p()
        assert rig.eng.lib.pwpp_bound_packed_xyz(rig.eng._h, None, None, C.byref(got[0]), C.byref(got[1])) == 0
        assert got[0].value == p["ground_offsets"].data_ptr() and got[1].value == p["nonground_offsets"].data_ptr()


@pytest.mark.parametrize("parts", [1, 2])
def test_one_part_only(scans, parts):
    """Only one part enabled: that part and its offsets are returned, the other is None; the scan still writes both arrays."""
    rig = Rig(scans, "velodyne22", "actions", parts=parts)
    P = rig.eng.bound_packed_records()
    on, off = ("ground", "nonground") if parts == 1 else ("nonground", "ground")
    assert P[on] is not None and P[on + "_offsets"] is not None and P[off] is None and P[off + "_offsets"] is None
    rng = np.random.default_rng(parts)
    for k in range(3):
        if k:
            rig.set(*rig.random_cfg(rng))
        rig.fill()
        rig.eng.run_bound_call()
        rig.check(f"run {k}")


def test_enable_after_a_capture(scans):
    """A graph captured before the enable leaves the packed buffers as they were; one captured after writes them."""
    import torch
    rig = Rig(scans, "pcl_xyzi32", "packed", parts=0)
    s = torch.cuda.Stream()
    g0 = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g0, stream=s):
            rig.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    rig.eng.bind_packed_records()
    rig.fill()
    g0.replay()
    torch.cuda.synchronize()
    P = rig.eng.bound_packed_records()
    for key in ("ground", "nonground"):
        assert (P[key].cpu().numpy() == SENTINEL).all(), f"{key}: a graph captured before the enable wrote it"
    g1 = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g1, stream=s):
            rig.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    rig.fill()
    g1.replay()
    torch.cuda.synchronize()
    rig.check("graph captured after the enable")


def test_direct_call_between_runs(scans):
    """Direct calls between runs leave the packed records and their offsets untouched."""
    import torch
    rig = Rig(scans, "velodyne22", "plain")
    rig.fill()
    rig.eng.run_bound_call()
    rig.check("run")
    P = rig.eng.bound_packed_records()
    before = {k: P[k].clone() for k in ("ground", "nonground", "ground_offsets", "nonground_offsets")}
    rig.eng.estimate_host([scans[4]])
    dt, lay = layout_of("velodyne22")
    r = torch.from_numpy(np.ascontiguousarray(records(scans[4], dt)[0]).view(np.uint8).reshape(-1).copy()).cuda()
    rig.eng.estimate_device_records([r.data_ptr()], [len(scans[4])], [lay])
    rig.eng.synchronize()
    torch.cuda.synchronize()
    for k, v in before.items():
        assert torch.equal(P[k], v), f"{k} changed under a direct call"


def test_launch_count_rule(scans):
    """Per run: packed records alone or packed xyz alone add two launches (one scan and one gather); both add three (one scan)."""
    for first in ("records", "xyz"):
        rig = Rig(scans[:3], "velodyne22", "actions", parts=0, record_results=False)
        e = rig.eng

        def per_run():
            n0 = e.launch_count()
            e.run_bound_call()
            return e.launch_count() - n0
        e.run_bound_call()
        base = per_run()
        (e.bind_packed_records if first == "records" else e.bind_packed_xyz)()
        assert per_run() == base + 2, first
        (e.bind_packed_xyz if first == "records" else e.bind_packed_records)()
        assert per_run() == base + 3, first
        e.synchronize()


def test_errors_and_unbind(scans):
    """No bound call, bad parts, already enabled, mixed point steps (naming the frame); after unbind the getter errs."""
    import torch
    import pwpp_b200
    e = pwpp_b200.Engine(device=0, num_streams=3)
    lib, h = e.lib, e._h
    outs = [C.c_void_p() for _ in range(4)]
    step = C.c_int32()

    def bound():
        return lib.pwpp_bound_packed_records(h, *[C.byref(o) for o in outs], C.byref(step))
    assert lib.pwpp_bind_packed_records(h, 3) == ERR_INVALID_ARG and "no call is bound" in lib.pwpp_last_error().decode()
    assert bound() == ERR_INVALID_ARG
    # mixed steps: frames 0 and 1 velodyne22, frame 2 pcl_xyzi32
    lays = [layout_of(k)[1] for k in ("velodyne22", "velodyne22", "pcl_xyzi32")]
    bufs = [torch.zeros(1000 * 32, dtype=torch.uint8, device="cuda") for _ in range(3)]
    counts = torch.tensor([1000, 1000, 1000], dtype=torch.int64, device="cuda")
    e.bind_call(bufs, [1000] * 3, lays, counts)
    assert lib.pwpp_bind_packed_records(h, 3) == ERR_UNSUPPORTED
    msg = lib.pwpp_last_error().decode()
    assert "frame 2" in msg and "point_step" in msg, msg
    assert bound() == ERR_INVALID_ARG
    e.bind_record_results()   # mixed steps keep the capacity layout
    e.unbind_call()
    # one step, different field layouts: accepted
    dt = LAYOUTS["velodyne22"]
    other = pwpp_b200.layout_from_dtype(np.dtype({"names": ["x", "y", "z", "intensity"], "formats": ["<f4"] * 4, "offsets": [6, 10, 14, 0],
                                                  "itemsize": dt.itemsize}))
    e.bind_call(bufs, [1000] * 3, [layout_of("velodyne22")[1], other, layout_of("velodyne22")[1]], counts)
    for bad in (0, 4, -1):
        assert lib.pwpp_bind_packed_records(h, bad) == ERR_INVALID_ARG
    assert bound() == ERR_INVALID_ARG and "not enabled" in lib.pwpp_last_error().decode()
    assert lib.pwpp_bind_packed_records(h, 2) == 0
    assert lib.pwpp_bind_packed_records(h, 2) == ERR_INVALID_ARG and "already" in lib.pwpp_last_error().decode()
    assert bound() == 0
    assert outs[0].value is None and outs[1].value and outs[2].value is None and outs[3].value and step.value == 22
    e.run_bound_call()
    e.synchronize()
    e.unbind_call()
    assert bound() == ERR_INVALID_ARG and "no call is bound" in lib.pwpp_last_error().decode()
