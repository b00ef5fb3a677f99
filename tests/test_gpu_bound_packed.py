"""Bound calls over packed batches (pwpp_bind_call_packed) and packed xyz results (pwpp_bind_packed_xyz) on the GPU.

Every run is compared bit for bit with a twin context driven by one pwpp_estimate_device_records call on the slices the offsets
name (an invalid frame as an empty frame): index lists, device offsets, num_ground, status, centers, normals, xyz getters, bin
results and every stream's state, histories and export blob. The identity case compares a packed bind with a
pwpp_bind_call_actions bind of the same slices, record and getter results included. Packed xyz is compared with the
concatenation of the host xyz getters over the frames, for a plain, an actions, a rings and a packed bind. Data: the six KITTI
fixtures and synthetic frames, as 16-, 22- and 32-byte records and as float32 N x 4 and N x 3 tensors."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_bound_actions import INVALID, OUT_OF_RANGE, RESET, RUN, SKIP, SKIPPED
from test_gpu_records import LAYOUTS, outputs, records, stream

pytestmark = pytest.mark.gpu

OFFSETS_OUT_OF_RANGE = 5
ERR_INVALID_ARG = -1


@pytest.fixture(scope="module")
def scans(kitti):
    import synth
    return list(kitti) + [synth.make_frame(1, 3).numpy(), synth.make_frame(1, 4).numpy()[:5000]]


def _engine(ns):
    import pwpp_b200
    return pwpp_b200.Engine(device=0, num_streams=ns)


class Packed:
    """A packed batch of scans in one CUDA buffer (`kind`: a LAYOUTS name, or "f32x4" / "f32x3" for a float32 tensor), frames
    back to back and 100 junk records after them; a context bound over it and a twin."""

    def __init__(self, scans, kind, slack=64, actions=False, streams=None):
        import torch
        import pwpp_b200
        self.kind, self.scans = kind, scans
        nf = len(scans)
        self.streams = list(range(nf)) if streams is None else list(streams)
        ns = max(self.streams) + 1
        self.max_n = [len(a) + slack for a in scans]
        if kind.startswith("f32x"):
            cols = int(kind[-1])
            recs = [np.ascontiguousarray(a[:, :cols]) for a in scans]
            self.step = 4 * cols
            self.lay = pwpp_b200.layout_from_dtype(np.dtype({"names": ["x", "y", "z", "intensity"][:cols], "formats": ["<f4"] * cols,
                                                             "offsets": [0, 4, 8, 12][:cols], "itemsize": 4 * cols}))
        else:
            dt = LAYOUTS[kind]
            recs = [records(a, dt, seed=k)[0] for k, a in enumerate(scans)]
            self.step = dt.itemsize
            self.lay = pwpp_b200.layout_from_dtype(dt)
        raw = [np.ascontiguousarray(r).view(np.uint8).reshape(-1) for r in recs]
        junk = np.random.default_rng(7).integers(0, 256, 100 * self.step, dtype=np.uint8)
        if kind.startswith("f32x"):
            junk = np.random.default_rng(7).uniform(-30, 30, 100 * cols).astype(np.float32).view(np.uint8)
        self.base_entries = np.concatenate([[0], np.cumsum([len(a) for a in scans])]).tolist()
        flat = np.concatenate(raw + [junk])
        self.capacity = len(flat) // self.step
        if kind.startswith("f32x"):
            self.points = torch.from_numpy(flat.view(np.float32).reshape(-1, cols).copy()).cuda()
        else:
            self.points = torch.from_numpy(flat.copy()).cuda()
        self.base = self.points.data_ptr()
        self.offsets = torch.zeros(nf + 1, dtype=torch.int64, device="cuda")
        self.actions = torch.zeros(nf, dtype=torch.int32, device="cuda") if actions else None
        self.eng, self.twin = _engine(ns), _engine(ns)
        self.eng.bind_call_packed(self.points, self.offsets, self.max_n, layout=None if kind.startswith("f32x") else self.lay,
                                  streams=self.streams, actions=self.actions)
        self.acts = [RUN] * nf
        self.set_offsets(self.base_entries)

    def set_offsets(self, entries, acts=None):
        """The nframes + 1 offsets entries (and the actions) of the next run."""
        import torch
        ent = [int(x) for x in entries]
        self.entries = ent
        self.offsets.copy_(torch.tensor(ent, dtype=torch.int64))
        if acts is not None:
            self.actions.copy_(torch.tensor(acts, dtype=torch.int32))
            self.acts = list(acts)
        torch.cuda.synchronize()

    def want(self):
        """(pointer, size, status) of every frame under the rule."""
        out = []
        for f, a in enumerate(self.acts):
            lo, hi = self.entries[f], self.entries[f + 1]
            if a not in (RUN, RESET):
                out.append((self.base, 0, SKIPPED if a == SKIP else INVALID))
            elif not 0 <= lo <= hi <= self.capacity:
                out.append((self.base, 0, OFFSETS_OUT_OF_RANGE))
            elif hi - lo > self.max_n[f]:
                out.append((self.base, 0, OUT_OF_RANGE))
            else:
                out.append((self.base + lo * self.step, hi - lo, 0))
        return out

    def check(self, what):
        """The last run against the twin's one call over the same slices (all frames RUN or invalid: no skips here)."""
        import torch
        torch.cuda.synchronize()
        idx, off, ng, st = self.eng.bound_call_results()
        self.eng.synchronize()
        w = self.want()
        assert st.cpu().numpy().tolist() == [s for _, _, s in w], f"{what}: status"
        assert np.array_equal(off.cpu().numpy(), np.concatenate([[0], np.cumsum([n for _, n, _ in w])])), f"{what}: offsets"
        for f, a in enumerate(self.acts):
            if a == RESET:
                self.twin.reset(self.streams[f])
        self.twin.estimate_device_records([p for p, _, _ in w], [n for _, n, _ in w], [self.lay] * len(w), streams=self.streams)
        self.twin.synchronize()
        ngs = ng.cpu().numpy()
        for f in range(len(w)):
            assert outputs(self.eng, f) == outputs(self.twin, f), f"{what}: frame {f}"
            assert ngs[f] == self.twin.num_ground(f), f"{what}: frame {f} num_ground"
        for s in set(self.streams):
            assert stream(self.eng, s) == stream(self.twin, s), f"{what}: stream {s}"


KINDS = ["xyzi16", "velodyne22", "pcl_xyzi32", "f32x4", "f32x3"]


@pytest.mark.parametrize("kind", KINDS)
def test_runs_equal_direct_calls_on_the_slices(scans, kind):
    """Eight frames packed with gaps; two runs (the stream state carries), then shifted slices and an emptied frame."""
    p = Packed(scans, kind)
    p.eng.run_bound_call()
    p.check("first run")
    p.eng.run_bound_call()
    p.check("second run")
    e = list(p.base_entries)
    e[2] += 50   # frame 1 grows by 50 records (within max_n), frame 2 starts 50 later
    e[4] = e[3]  # frame 3 is emptied, frame 4 takes its records (then it is longer than max_n)
    e[-1] += 20  # the last frame reaches into the records after the batch
    p.set_offsets(e)
    p.eng.run_bound_call()
    p.check("shifted and emptied")


def test_graph_replays_with_changing_offsets(scans):
    """One captured graph replayed with different offsets between replays: frames shifted, emptied, one at exactly max_n, and
    invalid entries (negative, decreasing, past capacity, longer than max_n); with packed xyz on, and the launch count of a run."""
    import torch
    p = Packed(scans[:6], "velodyne22", slack=8)
    p.eng.bind_packed_xyz()
    before = p.eng.launch_count()
    p.eng.run_bound_call()
    per_run = p.eng.launch_count() - before
    p.check("first run")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            p.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    b = p.base_entries
    steps = [
        ("as written", b),
        ("shifted", [b[0]] + [x + 3 for x in b[1:]]),
        ("emptied", b[:2] + [b[1]] + b[3:]),
        ("exactly max_n", [b[0], b[0] + p.max_n[0]] + b[2:]),
        ("invalid", [-4, b[1], 3, b[3], b[4], b[5], p.capacity + 1]),
        ("frames overlap", [b[0], b[2], b[1] + 5, b[3], b[4], b[5], b[6]]),
    ]
    for what, ent in steps:
        p.set_offsets(ent)
        g.replay()
        torch.cuda.synchronize()
        p.check(f"replay {what}")
        check_packed_xyz(p.eng, [p.twin], what)
    assert p.eng.launch_count() - before == 2 * per_run, "a replay is not an enqueue"


def check_packed_xyz(eng, twins, what, present=None):
    """Packed xyz of the bound call against the host xyz getters of its twin's frames (frame f of twins[0], or per-frame twins)."""
    import torch
    torch.cuda.synchronize()
    P = eng.bound_packed_xyz()
    tw = twins[0]
    nf = len(P["nonground_offsets"] if P["ground_offsets"] is None else P["ground_offsets"]) - 1
    for key, okey, get in (("ground", "ground_offsets", tw.ground_xyz), ("nonground", "nonground_offsets", tw.nonground_xyz)):
        if P[key] is None:
            continue
        rows = [get(f) for f in range(nf)]
        want_off = np.concatenate([[0], np.cumsum([len(r) for r in rows])])
        got_off = P[okey].cpu().numpy()
        assert got_off.tolist() == want_off.tolist(), f"{what}: {okey}"
        want = np.concatenate(rows).astype(np.float32)
        got = P[key].cpu().numpy()[:want_off[-1]]
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{what}: packed {key}"


def test_identity_with_bind_call_actions(scans):
    """The packed bind and a pwpp_bind_call_actions bind of the same slices give the same results bit for bit over runs with
    skips, resets and invalid offsets: index lists, offsets, num_ground, status, record results, getter results, packed xyz."""
    import torch
    import pwpp_b200
    sc = scans[:6]
    p = Packed(sc, "pcl_xyzi32", actions=True)
    q = _engine(len(sc))
    counts = torch.zeros(len(sc), dtype=torch.int64, device="cuda")
    acts_q = torch.zeros(len(sc), dtype=torch.int32, device="cuda")
    for e in (p.eng,):
        e.bind_record_results()
        e.bind_getter_results()
        e.bind_packed_xyz()

    b = p.base_entries
    plans = [([RUN] * 6, b), ([RUN, SKIP, RESET, 9, RUN, RESET], [b[0], b[1], -7, b[3], b[4] + 2, b[5], b[6]]),
             ([RUN, RUN, RUN, RUN, RESET, RUN], b[:3] + [b[2] - 9] + b[4:])]
    bound_q = None
    for k, (acts, ent) in enumerate(plans):
        p.set_offsets(ent, acts)
        w = p.want()
        if bound_q is not None:
            q.unbind_call()
        # the identity: frames[f] = base + lo * step, counts[f] = hi - lo (a frame with invalid offsets: an out-of-range count
        # gives the same empty frame, but its own status, so the statuses are compared apart)
        ptrs = [p.base + max(p.entries[f], 0) * p.step if 0 <= p.entries[f] <= p.capacity else p.base for f in range(6)]
        cnt = [p.entries[f + 1] - p.entries[f] if st != OFFSETS_OUT_OF_RANGE else -1 for f, (_, _, st) in enumerate(w)]
        counts.copy_(torch.tensor(cnt, dtype=torch.int64))
        acts_q.copy_(torch.tensor(acts, dtype=torch.int32))
        q.bind_call(ptrs, p.max_n, [p.lay] * 6, counts, actions=acts_q)
        q.bind_record_results()
        q.bind_getter_results()
        q.bind_packed_xyz()
        bound_q = True
        p.eng.run_bound_call()
        q.run_bound_call()
        torch.cuda.synchronize()
        a, b = p.eng.bound_call_results(), q.bound_call_results()
        for name, x, y in zip(("indices", "offsets", "num_ground"), a[:3], b[:3]):
            assert torch.equal(x, y), f"plan {k}: {name}"
        sa, sb = a[3].cpu().numpy(), b[3].cpu().numpy()
        assert sa.tolist() == [st for _, _, st in w]
        assert [int(y) if x != OFFSETS_OUT_OF_RANGE else OFFSETS_OUT_OF_RANGE for x, y in zip(sa, sb)] == sa.tolist()
        for f in range(6):
            assert outputs(p.eng, f) == outputs(q, f), f"plan {k}: frame {f}"
        ra, rb = p.eng.bound_record_results(), q.bound_record_results()
        assert torch.equal(ra[3], rb[3]) and np.array_equal(ra[2], rb[2]), f"plan {k}: record counts"
        for z in range(2):
            for f in range(6):
                m = int(ra[3][f, z]) * p.step
                assert torch.equal(ra[z][ra[2][f]:ra[2][f] + m], rb[z][rb[2][f]:rb[2][f] + m]), f"plan {k}: records {z} frame {f}"
        ga, gb = p.eng.bound_getter_results(), q.bound_getter_results()
        for key in ("xyz_counts", "num_patches", "height", "elevation_thr", "flatness_thr", "n_elevation", "n_flatness"):
            assert torch.equal(ga[key], gb[key]), f"plan {k}: getter {key}"
        pa, pb = p.eng.bound_packed_xyz(), q.bound_packed_xyz()
        for key in ("ground_offsets", "nonground_offsets"):
            assert torch.equal(pa[key], pb[key]), f"plan {k}: {key}"
        for key, okey in (("ground", "ground_offsets"), ("nonground", "nonground_offsets")):
            t = int(pa[okey][-1])
            assert torch.equal(pa[key][:t].view(torch.int32), pb[key][:t].view(torch.int32)), f"plan {k}: packed {key}"
        check_packed_xyz(p.eng, [p.eng], f"plan {k}")


def test_invalid_offsets_advance_the_stream_as_an_empty_call(scans):
    """Each invalid kind on one frame of a four-frame batch: that frame's status, an empty frame whose stream advances as after
    an empty direct call; the other frames are unaffected (the twin runs them as usual)."""
    p = Packed(scans[:4], "xyzi16")
    b = p.base_entries
    for what, ent in (("negative", [b[0], b[1], -1, b[3], b[4]]),
                      ("decreasing", [b[0], b[1], b[1] - 1, b[3], b[4]]),
                      ("past capacity", b[:4] + [p.capacity + 1]),
                      ("longer than max_n", [b[0], b[0] + p.max_n[0] + 1] + b[2:])):
        p.set_offsets(ent)
        p.eng.run_bound_call()
        p.check(what)


def test_packed_xyz_of_every_bind_kind(scans):
    """Packed xyz equals the concatenation of the host xyz getters over the frames for a plain, an actions, a rings and a packed
    bind; its offsets equal the scan of the host counts; enabling it adds two launches per run and none without it."""
    import torch
    import pwpp_b200
    sc = scans[:4]
    dt = LAYOUTS["xyzi16"]
    lay = pwpp_b200.layout_from_dtype(dt)
    bufs = [torch.from_numpy(np.ascontiguousarray(records(a, dt, seed=k)[0]).view(np.uint8).reshape(-1).copy()).cuda() for k, a in enumerate(sc)]
    max_n = [len(a) + 10 for a in sc]
    counts = torch.tensor([len(a) for a in sc], dtype=torch.int64, device="cuda")
    for kind in ("plain", "actions", "rings", "packed"):
        e = _engine(4)
        if kind in ("plain", "actions"):
            acts = torch.tensor([RUN, SKIP, RESET, RUN], dtype=torch.int32, device="cuda") if kind == "actions" else None
            e.bind_call(bufs, max_n, [lay] * 4, counts, actions=acts)
        elif kind == "rings":
            slots = torch.zeros(4, dtype=torch.int32, device="cuda")
            e.bind_call_rings([(b.view(1, -1), counts[k:k + 1]) for k, b in enumerate(bufs)], [len(a) for a in sc], [lay] * 4, slots)
        else:
            pts = torch.cat(bufs)
            off = torch.tensor(np.concatenate([[0], np.cumsum([len(a) for a in sc])]), dtype=torch.int64, device="cuda")
            e.bind_call_packed(pts, off, max_n, layout=lay)
        e.run_bound_call()
        n0 = e.launch_count()
        e.run_bound_call()
        plain = e.launch_count() - n0
        e.bind_packed_xyz(ground=kind != "rings", nonground=True)
        n0 = e.launch_count()
        e.run_bound_call()
        assert e.launch_count() - n0 == plain + 2, kind
        e.bound_call_results()
        e.synchronize()
        P = e.bound_packed_xyz()
        assert (P["ground"] is None) == (kind == "rings") and (P["ground_offsets"] is None) == (kind == "rings")
        check_packed_xyz(e, [e], kind)
        go = P["nonground_offsets"].cpu().numpy()
        assert go.tolist() == np.concatenate([[0], np.cumsum([e.num_nonground(f) for f in range(4)])]).tolist()
        e.unbind_call()


def test_bind_errors_unbind_and_freeze(scans):
    """Bind errors name the field and change no state; packed xyz errors; unbind releases the buffers; the freeze holds."""
    import torch
    import pwpp_b200
    e = _engine(2)
    lib, h = e.lib, e._h
    lay = pwpp_b200.layout_from_dtype(LAYOUTS["xyzi16"])
    pts = torch.zeros(1000, 4, dtype=torch.float32, device="cuda")
    off = torch.tensor([0, 500, 1000], dtype=torch.int64, device="cuda")
    ids = np.arange(2, dtype=np.int32)
    mx = (C.c_int64 * 2)(600, 600)
    P, O = C.c_void_p(pts.data_ptr()), C.c_void_p(off.data_ptr())

    def bind(base=P, layout=C.byref(lay), cap=1000, offs=O, max_n=mx):
        return lib.pwpp_bind_call_packed(h, 2, ids.ctypes.data, base, layout, cap, max_n, offs, None)
    for args, word in ((dict(layout=None), "layout"), (dict(offs=None), "d_offsets"), (dict(base=None), "base"), (dict(cap=-1), "capacity"),
                       (dict(cap=2 ** 62), "overflows"), (dict(max_n=(C.c_int64 * 2)(600, -1)), "frame 1")):
        assert bind(**args) == ERR_INVALID_ARG, word
        assert word in lib.pwpp_last_error().decode(), (word, lib.pwpp_last_error())
    assert lib.pwpp_bind_packed_xyz(h, 3) == ERR_INVALID_ARG and "no call is bound" in lib.pwpp_last_error().decode()
    e.estimate_host([scans[0]])   # no state changed: a direct call still runs
    assert bind() == 0
    for bad in (0, 4, -1):
        assert lib.pwpp_bind_packed_xyz(h, bad) == ERR_INVALID_ARG
    outs = [C.c_void_p() for _ in range(4)]
    assert lib.pwpp_bound_packed_xyz(h, *[C.byref(o) for o in outs]) == ERR_INVALID_ARG
    assert lib.pwpp_bind_packed_xyz(h, 2) == 0
    assert lib.pwpp_bind_packed_xyz(h, 2) == ERR_INVALID_ARG and "already" in lib.pwpp_last_error().decode()
    assert lib.pwpp_bound_packed_xyz(h, *[C.byref(o) for o in outs]) == 0
    assert outs[0].value is None and outs[1].value and outs[2].value is None and outs[3].value
    big = [np.tile(scans[0], (8, 1))]
    with pytest.raises(pwpp_b200.PwppError):   # frozen: a call that would grow a work buffer
        e.estimate_host(big)
    e.unbind_call()
    assert lib.pwpp_bound_packed_xyz(h, *[C.byref(o) for o in outs]) == ERR_INVALID_ARG
    e.estimate_host(big)   # the freeze is lifted
