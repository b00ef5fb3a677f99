"""Stream tables of bound calls (pwpp_bind_stream_table): every frame's sensor stream read on the GPU at every run or replay, so
one bound call serves more streams than it has frames.

Every tick is compared with a twin context of the same parameter sets and num_streams, driven by direct
pwpp_estimate_device_records calls that name, run by run, only the frames the bound call accepted (with pwpp_reset_stream for the
accepted RESET frames before their run): every accepted position's outputs (bin ids, both index lists, patches, xyz, bin
records), offsets, status, and every stream's export blob. Contexts are created with PWPP_SMALL_CALL=0 so that calls of any size
take the batch kernels on both sides."""
import numpy as np
import pytest

from param_sets import _default, _no_rvpf_tgr, _ros
from test_gpu_bound_actions import batch_kernels
from test_gpu_records import LAYOUTS, outputs

pytestmark = pytest.mark.gpu

RUN, SKIP, RESET = 0, 1, 2
OUT_OF_RANGE, SKIPPED, INVALID, STREAM_OOR, DUPLICATE = 1, 2, 3, 6, 7
ERR_INVALID_ARG = -1


def fine129():
    p = _default()
    p.num_sectors_each_zone[0] = 129   # a geometry the fp32 binning filter does not cover: the exact binning path
    return p


SETS = [_default(), _ros(), _no_rvpf_tgr(), fine129()]


class Fleet:
    """A bound call over `shape` positions on a ctx of `ns` streams over four parameter sets (`sets`), and its twin. kind "plain":
    a device buffer of max_n 16-byte records per position; "rings": a ring of two slots per position, each tick written into
    the slot (tick + f) % 2; "packed": one buffer with the frames back to back and device offsets. With `results` the bound
    call also gathers record, getter (xyz and state), packed xyz and packed record results."""

    def __init__(self, scans, shape, ns, table=True, with_actions=True, kind="plain", results=False, sets=None):
        import torch
        import pwpp_b200
        self.scans, self.kind = scans, kind
        self.shape, self.ns, self.nf = list(shape), ns, len(shape)
        self.stream_set = [s % 4 for s in range(ns)]
        with batch_kernels():
            self.eng, self.twin = [pwpp_b200.Engine(sets or SETS, device=0, num_streams=ns, stream_set=self.stream_set) for _ in range(2)]
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
            self.eng.bind_call_rings(list(zip(self.bufs, self.ring_counts)), caps, lays, self.slots, streams=self.shape, actions=self.actions)
        elif kind == "packed":
            self.points = torch.zeros((nf * self.max_n, 4), dtype=torch.float32, device="cuda")
            self.offsets = torch.zeros(nf + 1, dtype=torch.int64, device="cuda")
            self.eng.bind_call_packed(self.points, self.offsets, caps, layout=self.lay, streams=self.shape, actions=self.actions)
        else:
            self.bufs = [torch.zeros((self.max_n, 4), dtype=torch.float32, device="cuda") for _ in range(nf)]
            self.counts = torch.zeros(nf, dtype=torch.int64, device="cuda")
            self.eng.bind_call(self.bufs, caps, lays, self.counts, streams=self.shape, actions=self.actions)
        if results:
            self.eng.bind_record_results()
            self.eng.bind_getter_results()
            self.eng.bind_packed_xyz()
            self.eng.bind_packed_records()
        self.table = table
        if table:
            self.eng.bind_stream_table(self.streams)
        self.runs = runs_of(self.shape)

    def load(self, tick, read, acts):
        import torch
        sizes, self.ptrs, off = [], [], 0
        for f in range(self.nf):
            a = self.dscans[(tick + f) % len(self.dscans)]
            n = len(a) - (f % 5) * 11
            if self.kind == "rings":
                slot = (tick + f) % 2
                self.bufs[f][slot, :16 * n].copy_(a[:n].view(torch.uint8).reshape(-1))
                self.ring_counts[f][slot] = n
                self.slots[f] = slot
                self.ptrs.append(self.bufs[f].data_ptr() + slot * self.stride)
            elif self.kind == "packed":
                self.points[off:off + n].copy_(a[:n])
                self.ptrs.append(self.points.data_ptr() + 16 * off)
                off += n
            else:
                self.bufs[f][:n].copy_(a[:n])
                self.ptrs.append(self.bufs[f].data_ptr())
            sizes.append(n)
        if self.kind == "packed":
            self.offsets.copy_(torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64))
        elif self.kind == "plain":
            self.counts.copy_(torch.tensor(sizes, dtype=torch.int64))
        self.streams.copy_(torch.tensor(list(read), dtype=torch.int32))
        if self.actions is not None:
            self.actions.copy_(torch.tensor(list(acts), dtype=torch.int32))
        torch.cuda.synchronize()
        self.read, self.acts, self.sizes = [int(s) for s in read], [int(a) for a in acts], sizes

    def expected_status(self):
        st = []
        for r in range(len(self.runs) - 1):
            seen = set()
            for f in range(self.runs[r], self.runs[r + 1]):
                a, s = self.acts[f], self.read[f]
                if a not in (RUN, RESET):
                    st.append(SKIPPED if a == SKIP else INVALID)
                elif s < 0:
                    st.append(SKIPPED)
                elif s >= self.ns:
                    st.append(STREAM_OOR)
                elif s in seen:
                    st.append(DUPLICATE)
                else:
                    seen.add(s)
                    st.append(0)
        return st

    def check(self, what):
        """The bound call's last run against the twin, run by run over the accepted frames."""
        import torch
        idx, off, ng, st = self.eng.bound_call_results()
        torch.cuda.synchronize()
        want_st = self.expected_status()
        assert st.cpu().numpy().tolist() == want_st, f"{what}: status"
        if self.table:
            assert self.eng.bound_call_streams().cpu().numpy().tolist() == self.read, f"{what}: the read copy"
        acc = [s == 0 for s in want_st]
        eff = [n if a else 0 for n, a in zip(self.sizes, acc)]
        assert np.array_equal(off.cpu().numpy(), np.concatenate([[0], np.cumsum(eff)])), f"{what}: offsets"
        mine = {f: outputs(self.eng, f) for f in range(self.nf) if acc[f]}
        for r in range(len(self.runs) - 1):
            fr = [f for f in range(self.runs[r], self.runs[r + 1]) if acc[f]]
            for f in fr:
                if self.acts[f] == RESET:
                    self.twin.reset(self.read[f])
            if not fr:
                continue
            self.twin.estimate_device_records([self.ptrs[f] for f in fr], [self.sizes[f] for f in fr], [self.lay] * len(fr),
                                              streams=[self.read[f] for f in fr])
            self.twin.synchronize()
            for k, f in enumerate(fr):
                assert mine[f] == outputs(self.twin, k), f"{what}: frame {f} (stream {self.read[f]}) outputs"
        a, b = blobs(self.eng, self.ns), blobs(self.twin, self.ns)
        assert torch.equal(a, b), f"{what}: stream states differ at {torch.nonzero((a != b).any(1)).flatten()[:8].tolist()}"


def blobs(eng, ns):
    """Every stream's export blob, one zero-filled row each (a set with a smaller history capacity leaves its row's tail as it
    was)."""
    import torch
    rows = torch.zeros((ns, (eng.state_blob_size() + 15) // 16 * 16), dtype=torch.uint8, device="cuda")
    eng.export_states(list(range(ns)), out=rows)
    torch.cuda.synchronize()
    return rows


def runs_of(shape):
    runs, last = [0], {}
    for f, s in enumerate(shape):
        if s in last and last[s] >= runs[-1]:
            runs.append(f)
        last[s] = f
    runs.append(len(shape))
    return runs


def tick_schedule(rng, shape, ns, runs):
    """A scheduler's pick: distinct streams per run, a backlog stream in both runs, holes, duplicates inside a run, out-of-range
    ids, and SKIP / RESET actions."""
    nf = len(shape)
    picked = rng.permutation(ns)
    read = np.empty(nf, np.int64)
    read[:runs[1]] = picked[:runs[1]]
    if len(runs) > 2:
        read[runs[1]:] = np.concatenate([picked[:3], picked[runs[1]:runs[1] + nf - runs[1] - 3]])   # a backlog in both runs
    u = rng.random(nf)
    read[u < 0.06] = -1
    read[(u >= 0.06) & (u < 0.1)] = rng.choice([ns, ns + 5, 2 ** 31 - 1], int(((u >= 0.06) & (u < 0.1)).sum()))
    dup = np.flatnonzero((u >= 0.1) & (u < 0.15))
    for f in dup:
        r = max(k for k in range(len(runs) - 1) if runs[k] <= f)
        if f > runs[r]:
            read[f] = read[rng.integers(runs[r], f)]
    acts = rng.choice([RUN, SKIP, RESET], nf, p=[0.8, 0.12, 0.08])
    return read, acts


@pytest.mark.parametrize("kind", ["plain", "rings", "packed"])
def test_fleet_schedule_in_one_captured_graph(kitti, kind):
    """256 streams on four sets, a 64 + 32 bind (two runs), 24 seeded ticks replayed from one captured graph; plain frames, scan
    rings and a packed batch."""
    import torch
    shape = list(range(64)) + list(range(32))
    fl = Fleet(list(kitti), shape, 256, kind=kind)
    rng = np.random.default_rng(256)
    fl.load(0, shape, [RUN] * fl.nf)
    fl.eng.run_bound_call()
    fl.check("eager run before the capture")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fl.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    for t in range(24):
        read, acts = tick_schedule(rng, shape, 256, fl.runs)
        fl.load(t + 1, read, acts)
        g.replay()
        torch.cuda.synchronize()
        fl.check(f"tick {t}")


def bound_results(eng, nf):
    """Every result of the bound call's last run, as host arrays: indices, offsets, counts, status, and the valid part of every
    record, getter (xyz, patches, state rows), packed xyz and packed record result."""
    import torch
    idx, off, ng, st = eng.bound_call_results()
    torch.cuda.synchronize()
    h = lambda t: t.cpu().numpy()   # noqa: E731
    off_h = h(off)
    out = {"idx": h(idx[:int(off_h[-1])]), "off": off_h, "ng": h(ng), "status": h(st)}
    g, n, roff, cnt = eng.bound_record_results()
    cnt = h(cnt)
    for f in range(nf):
        out[f"rec_g{f}"] = h(g[roff[f]:roff[f] + 16 * cnt[f, 0]])
        out[f"rec_n{f}"] = h(n[roff[f]:roff[f] + 16 * cnt[f, 1]])
    d = eng.bound_getter_results()
    xc, npat = h(d["xyz_counts"]), h(d["num_patches"])
    out["xyz_counts"], out["num_patches"] = xc, npat
    for f in range(nf):
        r = int(d["row_off"][f])
        out[f"gx{f}"] = h(d["ground_xyz"][r:r + xc[f, 0]])
        out[f"nx{f}"] = h(d["nonground_xyz"][r:r + xc[f, 1]])
        out[f"c{f}"] = h(d["centers"][f, :npat[f]])
        out[f"nm{f}"] = h(d["normals"][f, :npat[f]])
    for k in ("height", "elevation_thr", "flatness_thr", "n_elevation", "n_flatness"):
        out[k] = h(d[k])
    px = eng.bound_packed_xyz()
    go, no = h(px["ground_offsets"]), h(px["nonground_offsets"])
    out.update(px_go=go, px_no=no, px_g=h(px["ground"][:go[-1]]), px_n=h(px["nonground"][:no[-1]]))
    pr = eng.bound_packed_records()
    go, no = h(pr["ground_offsets"]), h(pr["nonground_offsets"])
    out.update(pr_go=go, pr_no=no, pr_g=h(pr["ground"][:go[-1]]), pr_n=h(pr["nonground"][:no[-1]]))
    return out


@pytest.mark.parametrize("kind,with_actions", [("plain", False), ("plain", True), ("rings", True), ("packed", True)],
                         ids=["plain", "actions", "rings", "packed"])
def test_identity_equals_the_bind_without_a_table(kitti, kind, with_actions):
    """d_streams equal to the bound streams: bit for bit the results of the same bind without a table, with record, getter
    (xyz and state), packed xyz and packed record results enabled, and the same stream states, for all four bind kinds."""
    shape = [3, 1, 4, 0, 5, 9, 2, 6, 3, 5]
    a = Fleet(list(kitti), shape, 12, table=True, with_actions=with_actions, kind=kind, results=True)
    b = Fleet(list(kitti), shape, 12, table=False, with_actions=with_actions, kind=kind, results=True)
    for t in range(3):
        acts = [RUN, RESET, SKIP, RUN, RUN, RESET, RUN, SKIP, RESET, RUN] if t and with_actions else [RUN] * 10
        for x in (a, b):
            x.load(t, shape, acts)
            x.eng.run_bound_call()
        ra, rb = bound_results(a.eng, 10), bound_results(b.eng, 10)
        assert ra.keys() == rb.keys()
        for k in ra:
            assert ra[k].shape == rb[k].shape and ra[k].tobytes() == rb[k].tobytes(), f"tick {t}: {k}"
        for f in range(10):
            assert outputs(a.eng, f) == outputs(b.eng, f), f"tick {t} frame {f}"
        assert np.array_equal(blobs(a.eng, 12).cpu().numpy(), blobs(b.eng, 12).cpu().numpy()), f"tick {t}: stream states"


def storage20():
    """The four sets with 20-sample histories, so that a few frames fill them."""
    sets = [_default(), _ros(), _no_rvpf_tgr(), fine129()]
    for p in sets:
        p.max_elevation_storage = p.max_flatness_storage = 20
    return sets


def test_stream_named_only_by_rejected_frames_keeps_its_state(kitti):
    """Stream 5 runs until its histories are full, then is named only by rejected frames (an action SKIP, an invalid action,
    next to holes, out-of-range ids and RESETs of other streams): its export blob stays bit for bit. (A duplicate always leaves
    its stream to the frame that won it, which runs it.)"""
    shape = list(range(4))
    fl = Fleet(list(kitti), shape, 8, sets=storage20())
    for t in range(25):
        fl.load(t, [5, 1, 2, 3], [RUN] * 4)
        fl.eng.run_bound_call()
    fl.eng.synchronize()
    st = fl.eng.state(5)
    assert max(st.n_elevation) == 20 and max(st.n_flatness) == 20, "stream 5's histories are not full"
    blob = fl.eng.export_state(5)
    for t, (read, acts) in enumerate([([5, 1, 2, 3], [SKIP, RUN, RUN, RUN]), ([1, 5, 2, 3], [RUN, 7, RUN, RESET]),
                                      ([-1, 9, 5, 2], [RUN, RUN, SKIP, RESET])]):
        fl.load(t, read, acts)
        fl.eng.run_bound_call()
        fl.eng.synchronize()
        assert fl.eng.export_state(5) == blob, f"case {t}"


def test_bin_records_after_unbinding_a_table_call(kitti):
    """The host getters of the last call keep serving it after pwpp_unbind_call, with each frame's set the stream it read."""
    fl = Fleet(list(kitti), [0, 1], 8, with_actions=False)
    fl.load(0, [3, -1], [RUN, RUN])
    fl.eng.run_bound_call()
    fl.eng.bound_call_results()
    fl.eng.unbind_call()
    assert len(fl.eng.bin_results(0)) == fl.eng.stream_num_bins(3)
    assert len(fl.eng.bin_results(1)) == fl.eng.stream_num_bins(1)   # a hole: its bound stream's set


def test_bin_records_follow_the_set_of_the_stream_read(kitti):
    """A position whose stream (and so set) changed since the previous replay returns its new set's number of bin records."""
    fl = Fleet(list(kitti), [0, 1], 8, with_actions=False)
    for t, read in enumerate([[0, 1], [3, 2], [-1, 6]]):
        fl.load(t, read, [RUN, RUN])
        fl.eng.run_bound_call()
        fl.eng.bound_call_results()
        for f in range(2):
            s = read[f] if 0 <= read[f] < 8 else [0, 1][f]
            assert len(fl.eng.bin_results(f)) == fl.eng.stream_num_bins(s), f"tick {t} frame {f}"


def test_launch_count_rule(kitti):
    """With actions a bound call has one reset launch before every run after the first, with or without a stream table; a
    stream table adds no launch."""
    shape = list(range(6)) + list(range(3)) + [0]
    counts = {}
    for table in (False, True):
        for with_actions in (False, True):
            fl = Fleet(list(kitti), shape, 8, table=table, with_actions=with_actions)
            fl.load(0, shape, [RUN] * len(shape))
            fl.eng.run_bound_call()
            c0 = fl.eng.launch_count()
            fl.eng.run_bound_call()
            counts[table, with_actions] = fl.eng.launch_count() - c0
            fl.eng.synchronize()
    runs = len(runs_of(shape)) - 1
    assert counts[True, False] == counts[False, False]
    assert counts[True, True] == counts[False, True] == counts[False, False] + runs - 1


def test_bind_errors_leave_the_bound_call_unchanged(kitti):
    """Enable without a bound call, with NULL, twice, after a run and after a capture: PWPP_ERR_INVALID_ARG each time."""
    import torch
    import ctypes as C
    import pwpp_b200
    with batch_kernels():
        e = pwpp_b200.Engine(device=0, num_streams=4)
    t = torch.zeros(2, dtype=torch.int32, device="cuda")
    assert e.lib.pwpp_bind_stream_table(e._h, C.c_void_p(t.data_ptr())) == ERR_INVALID_ARG
    fl = Fleet(list(kitti), [0, 1], 4, table=False)
    lib, h = fl.eng.lib, fl.eng._h
    assert lib.pwpp_bind_stream_table(h, None) == ERR_INVALID_ARG
    fl.eng.bind_stream_table(fl.streams)
    fl.table = True
    assert lib.pwpp_bind_stream_table(h, C.c_void_p(fl.streams.data_ptr())) == ERR_INVALID_ARG
    fl.load(0, [2, 3], [RUN, RUN])
    fl.eng.run_bound_call()
    fl.check("after the refused enables")
    ran = Fleet(list(kitti), [0, 1], 4, table=False)
    ran.load(0, [0, 1], [RUN, RUN])
    ran.eng.run_bound_call()
    ran.check("the first run")
    assert ran.eng.lib.pwpp_bind_stream_table(ran.eng._h, C.c_void_p(ran.streams.data_ptr())) == ERR_INVALID_ARG
    ran.load(1, [0, 1], [RUN, RUN])
    ran.eng.run_bound_call()
    ran.check("after a refused enable past a run")
    cap = Fleet(list(kitti), [0, 1], 4, table=False)
    cap.load(0, [0, 1], [RUN, RUN])
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    assert cap.eng.lib.pwpp_bind_stream_table(cap.eng._h, C.c_void_p(cap.streams.data_ptr())) == ERR_INVALID_ARG
    g.replay()
    torch.cuda.synchronize()
    cap.check("after a refused enable past a capture")
