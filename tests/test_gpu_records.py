"""Sensor records of any PointCloud2 layout on the GPU (pwpp_estimate_host_records / pwpp_estimate_device_records).

Every case compares the records path with the existing path given the equivalent array: the fields numpy converts to float32,
N x 4, or N x 3 when the layout has no intensity. Bin ids, index lists (both output orders), patch records, centers, normals,
xyz getters, state and histories must be bit-identical. Layouts: xyz12, xyzi16, PCL xyzi32, a 22-byte record, a 48-byte record
with FLOAT32 intensity at 16, UINT8 and UINT16 intensity, FLOAT64 x/y/z and FLOAT64 intensity. Data: the six KITTI fixtures
and a scan with reflected-noise (RNR) hits added."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


def _dt(names, formats, offsets, itemsize):
    return np.dtype({"names": names, "formats": formats, "offsets": offsets, "itemsize": itemsize})


XYZI = ["x", "y", "z", "intensity"]
LAYOUTS = {
    "xyz12": _dt(XYZI[:3], ["<f4"] * 3, [0, 4, 8], 12),
    "xyzi16": _dt(XYZI, ["<f4"] * 4, [0, 4, 8, 12], 16),
    "pcl_xyzi32": _dt(XYZI, ["<f4"] * 4, [0, 4, 8, 16], 32),
    "velodyne22": _dt(XYZI + ["ring", "time"], ["<f4"] * 4 + ["<u2", "<f4"], [0, 4, 8, 12, 16, 18], 22),
    "rec48": _dt(XYZI + ["t"], ["<f4"] * 4 + ["<f8"], [0, 4, 8, 16, 24], 48),
    "u8_intensity": _dt(XYZI, ["<f4"] * 3 + ["u1"], [0, 4, 8, 12], 13),
    "u16_intensity": _dt(XYZI, ["<f4"] * 3 + ["<u2"], [0, 4, 8, 12], 14),
    "f64_xyz": _dt(["intensity", "x", "y", "z"], ["<f4", "<f8", "<f8", "<f8"], [0, 4, 12, 20], 28),
    "f64_intensity": _dt(XYZI, ["<f4"] * 3 + ["<f8"], [0, 4, 8, 12], 20),
}
WITH_I = [k for k in LAYOUTS if "intensity" in LAYOUTS[k].names]


def records(a, dt, seed=0):
    """Records of layout dt holding scan a (N x 4 float32; FLOAT64 fields get an offset that rounds, integer intensity is the
    scaled value), and the equivalent float32 array numpy makes of them."""
    rng = np.random.default_rng(seed)
    r = np.frombuffer(rng.integers(0, 256, len(a) * dt.itemsize, dtype=np.uint8).tobytes(), dtype=dt).copy()
    for c, name in enumerate("xyz"):
        ft = dt.fields[name][0]
        r[name] = a[:, c].astype(ft) + (rng.uniform(-1e-7, 1e-7, len(a)) if ft == np.float64 else 0)
    cols = ["x", "y", "z"]
    if "intensity" in dt.names:
        ft = dt.fields["intensity"][0]
        if ft.kind == "u":
            top = np.iinfo(ft).max
            r["intensity"] = np.clip(np.floor(a[:, 3] * np.float32(top)), 0, top).astype(ft)
        else:
            r["intensity"] = a[:, 3].astype(ft) + (rng.uniform(-1e-9, 1e-9, len(a)) if ft == np.float64 else 0)
        cols.append("intensity")
    with np.errstate(over="ignore"):
        eq = np.stack([r[c].astype(np.float32) for c in cols], axis=1)
    return r, np.ascontiguousarray(eq)


def padded(eq, nan_w=False):
    """N x 4 float32 of an equivalent array (an N x 3 one gets w = 0, or NaN: the intensity of a frame without the field)."""
    if eq.shape[1] == 4:
        return eq
    w = np.full((len(eq), 1), np.nan if nan_w else 0.0, np.float32)
    return np.ascontiguousarray(np.concatenate([eq, w], axis=1))


@pytest.fixture(scope="module")
def scans(kitti):
    """The six fixtures plus one with reflected-noise hits: low, steep, dark points below the sensor."""
    rng = np.random.default_rng(5)
    m = 400
    hits = np.stack([rng.uniform(3, 8, m), rng.uniform(-3, 3, m), rng.uniform(-6, -4, m), np.where(np.arange(m) % 2, 0.0, 0.1)], axis=1)
    return list(kitti) + [np.ascontiguousarray(np.concatenate([kitti[0], hits.astype(np.float32)]))]


def engine(num_streams=1, order=0, **kw):
    import pwpp_b200
    e = pwpp_b200.Engine(device=0, num_streams=num_streams, **kw)
    e.set_output_order(order)
    return e


def outputs(eng, f):
    parts = [eng.bin_ids(f), eng.ground_indices(f), eng.nonground_indices(f), eng.centers(f), eng.normals(f), eng.ground_xyz(f),
             eng.nonground_xyz(f)]
    return b"|".join(np.ascontiguousarray(p).tobytes() for p in parts) + bytes(eng.bin_results(f))


def stream(eng, s):
    return bytes(eng.state(s)) + b"".join(eng.history(s, r, w).tobytes() for r in range(4) for w in (0, 1)) + eng.export_state(s)


def assert_same(rec, ref, f, g, s, what):
    assert outputs(rec, f) == outputs(ref, g), what
    assert stream(rec, s) == stream(ref, s), f"{what}: state"


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "page_locked"])
@pytest.mark.parametrize("name", list(LAYOUTS))
def test_host_one_frame_calls(scans, name, pinned, order):
    """One stream, one frame per call through all seven scans (state carried), twice over: the second pass's calls replay the
    small-call graph the first captured. Each records call launches the existing call's kernels plus one unpack."""
    import pwpp_b200
    rec, ref = engine(order=order), engine(order=order)
    lay = pwpp_b200.layout_from_dtype(LAYOUTS[name])
    for rep in range(2):
        for k, a in enumerate(scans):
            r, eq = records(a, LAYOUTS[name], seed=k)
            l0, m0 = rec.launch_count(), ref.launch_count()
            if pinned:
                ptr = rec.lib.pwpp_host_alloc(r.nbytes)
                buf = np.ctypeslib.as_array((C.c_uint8 * r.nbytes).from_address(ptr))
                buf[:] = r.view(np.uint8)
                rec.estimate_host_records([(buf, lay)])
                rec.lib.pwpp_host_free(ptr)
            else:
                rec.estimate_host_records([r])
            ref.estimate_host([eq])
            assert rec.launch_count() - l0 == ref.launch_count() - m0 + 1, f"{name} scan {k}: launches"
            assert set(rec.call_times_us()) == {"h2d", "kernels", "d2h", "device_total"}
            assert_same(rec, ref, 0, 0, 0, f"{name} pass {rep} scan {k}")


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
def test_host_batch_over_several_pipeline_chunks(scans, order):
    """80 frames of mixed layouts (all with intensity) in one call: the pipeline splits it into chunks of ~4M points, each with
    its own unpack, and the frames run on the cluster front end. Two calls, the second carrying the first's state."""
    nf = 80
    rec, ref = engine(nf, order), engine(nf, order)
    for call in range(2):
        data = [records(scans[(f + call) % 7], LAYOUTS[WITH_I[f % len(WITH_I)]], seed=f) for f in range(nf)]
        l0, m0 = rec.launch_count(), ref.launch_count()
        rec.estimate_host_records([r for r, _ in data])
        ref.estimate_host([eq for _, eq in data])
        total = sum(len(eq) for _, eq in data)
        per_chunk = min(nf, max(1, (4 << 20) // max(1, total // nf)))
        nchunks = -(-nf // per_chunk)
        assert nchunks >= 2 and nf // nchunks > 4   # several chunks, each above the small-call limit
        assert rec.launch_count() - l0 == ref.launch_count() - m0 + nchunks
        for f in range(nf):
            assert_same(rec, ref, f, f, f, f"call {call} frame {f}")


@pytest.mark.parametrize("name", list(LAYOUTS))
def test_device_records_misaligned_separate_allocations(scans, name):
    """Seven frames on the device, each its own allocation that ends at its last record, starting 1..15 bytes past the
    allocation's base. The caller's buffers are overwritten after the call: the xyz getters still read the unpacked points."""
    import torch
    import pwpp_b200
    lay = pwpp_b200.layout_from_dtype(LAYOUTS[name])
    has_i = "intensity" in LAYOUTS[name].names
    rec, ref = engine(7), engine(7)
    for call in range(2):
        data = [records(scans[(f + 3 * call) % 7], LAYOUTS[name], seed=f + 10 * call) for f in range(7)]
        bufs, ptrs = [], []
        for f, (r, _) in enumerate(data):
            mis = 1 + (4 * f + call) % 15
            t = torch.empty(mis + r.nbytes, dtype=torch.uint8, device="cuda")
            t[mis:] = torch.from_numpy(r.view(np.uint8)).cuda()
            bufs.append(t)
            ptrs.append(t.data_ptr() + mis)
        pts = torch.from_numpy(np.concatenate([padded(eq) for _, eq in data])).cuda()
        offs = np.cumsum([0] + [len(eq) for _, eq in data]).astype(np.int64)
        torch.cuda.synchronize()
        l0, m0 = rec.launch_count(), ref.launch_count()
        rec.estimate_device_records(ptrs, [len(r) for r, _ in data], [lay] * 7)
        ref.estimate_device(pts.data_ptr(), offs, has_intensity=has_i)
        rec.synchronize(); ref.synchronize()
        assert rec.launch_count() - l0 == ref.launch_count() - m0 + 1
        for t in bufs:
            t.fill_(0x7F)
        torch.cuda.synchronize()
        for f in range(7):
            assert_same(rec, ref, f, f, f, f"{name} call {call} frame {f}")


@pytest.mark.parametrize("path", ["host", "device"])
def test_stream_table_with_repeats_and_mixed_layouts(scans, path):
    """Stream tables naming streams several times, every frame with its own layout, frames without intensity among frames with
    it. The reference context gets the same stream table with the equivalent float4 points (NaN intensity for the frames
    without the field)."""
    import torch
    import pwpp_b200
    calls = [([2, 0, 2, 1, 3, 0, 1], ["xyz12", "pcl_xyzi32", "velodyne22", "xyz12", "u16_intensity", "f64_xyz", "rec48"]),
             ([3, 3, 1], ["u8_intensity", "xyz12", "f64_intensity"]),
             ([0, 1, 2, 3, 0], ["xyzi16", "xyz12", "velodyne22", "pcl_xyzi32", "f64_xyz"])]
    rec, ref = engine(4), engine(4)
    for c, (streams, names) in enumerate(calls):
        data = [records(scans[(3 * c + f) % 7], LAYOUTS[names[f]], seed=f) for f in range(len(streams))]
        lays = [pwpp_b200.layout_from_dtype(r.dtype) for r, _ in data]
        if path == "host":
            rec.estimate_host_records([r for r, _ in data], streams=streams)
        else:
            bufs = [torch.from_numpy(r.view(np.uint8).copy()).cuda() for r, _ in data]
            torch.cuda.synchronize()
            rec.estimate_device_records([b.data_ptr() for b in bufs], [len(r) for r, _ in data], lays, streams=streams)
            rec.synchronize()
        pts = torch.from_numpy(np.concatenate([padded(eq, nan_w=True) for _, eq in data])).cuda()
        offs = np.cumsum([0] + [len(eq) for _, eq in data]).astype(np.int64)
        torch.cuda.synchronize()
        ref.estimate_device(pts.data_ptr(), offs, has_intensity=True, streams=streams)
        ref.synchronize()
        assert any(eq.shape[1] == 3 for _, eq in data) and any(eq.shape[1] == 4 for _, eq in data)
        for f, s in enumerate(streams):
            assert outputs(rec, f) == outputs(ref, f), f"call {c} position {f} stream {s}"
        for s in range(4):
            assert stream(rec, s) == stream(ref, s), f"call {c} stream {s}"


def test_frame_without_intensity_equals_its_n_by_3_call(scans):
    """A frame without an intensity field between two frames with one is segmented exactly as a separate N x 3 call of it."""
    for k in (0, 6):
        rec, ref = engine(3, 1), engine(3, 1)
        data = [records(scans[1], LAYOUTS["pcl_xyzi32"]), records(scans[k], LAYOUTS["xyz12"]), records(scans[2], LAYOUTS["u8_intensity"])]
        rec.estimate_host_records([r for r, _ in data], streams=[0, 1, 2])
        ref.estimate_host([data[1][1]], streams=[1])
        assert data[1][1].shape[1] == 3
        assert outputs(rec, 1) == outputs(ref, 0), f"scan {k}"
        assert stream(rec, 1) == stream(ref, 1)


def test_parameter_sets_each_stream_its_own_layout(scans):
    """A three-set context; each stream has its own set and its own record layout."""
    import torch
    import pwpp_b200
    from param_sets import PARAM_SETS
    sets = [PARAM_SETS[n][0]() for n in ("default", "ros", "no_rvpf_tgr")]
    lay_of = ["pcl_xyzi32", "xyz12", "u16_intensity"]
    rec = engine(3, 0, params=sets, stream_set=[0, 1, 2])
    ref = engine(3, 0, params=[PARAM_SETS[n][0]() for n in ("default", "ros", "no_rvpf_tgr")], stream_set=[0, 1, 2])
    for c, streams in enumerate(([0, 1, 2], [2, 0, 1], [1, 2, 1, 0])):
        data = [records(scans[(c + f) % 7], LAYOUTS[lay_of[s]], seed=f) for f, s in enumerate(streams)]
        rec.estimate_host_records([r for r, _ in data], streams=streams)
        pts = torch.from_numpy(np.concatenate([padded(eq, nan_w=True) for _, eq in data])).cuda()
        offs = np.cumsum([0] + [len(eq) for _, eq in data]).astype(np.int64)
        torch.cuda.synchronize()
        ref.estimate_device(pts.data_ptr(), offs, has_intensity=True, streams=streams)
        ref.synchronize()
        for f, s in enumerate(streams):
            assert outputs(rec, f) == outputs(ref, f), f"call {c} position {f} stream {s}"
        for s in range(3):
            assert stream(rec, s) == stream(ref, s), f"call {c} stream {s}"


def test_invalid_arguments_launch_nothing_and_change_no_state(scans):
    import torch
    import pwpp_b200
    eng = engine(3)
    r, _ = records(scans[1], LAYOUTS["pcl_xyzi32"])
    eng.estimate_host_records([r, r, r])
    blobs = [eng.export_state(s) for s in range(3)]
    launches = eng.launch_count()
    lib = eng.lib
    good = pwpp_b200.layout_from_dtype(r.dtype)

    def lay(step=32, off=(0, 4, 8, 16), types=(7, 7, 7, 7)):
        L = pwpp_b200.PwppPointLayout()
        L.point_step, L.offset[:], L.datatype[:] = step, list(off), list(types)
        return L

    d = torch.from_numpy(r.view(np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    INVALID, UNSUPPORTED = -1, -4
    cases = [  # (streams, ptr, n, layout, status, message part)
        (None, 1, len(r), good, INVALID, "streams is NULL"),
        ([5], 1, len(r), good, INVALID, "stream id 5"),
        ([0], 1, -1, good, INVALID, "frame 0: n < 0"),
        ([0], 0, len(r), good, INVALID, "frame 0: frame pointer is NULL"),
        ([0], 1, len(r), lay(types=(7, 7, 7, 11)), INVALID, "field intensity: unknown datatype 11"),
        ([0], 1, len(r), lay(off=(0, 4, 8, 30)), INVALID, "field intensity: bytes [30, 34)"),
        ([0], 1, len(r), lay(types=(7, 5, 7, 7)), UNSUPPORTED, "field y: x, y and z must be FLOAT32 or FLOAT64"),
        ([0], 1, len(r), lay(step=1025), UNSUPPORTED, "PWPP_MAX_POINT_STEP"),
        ([0], 1, len(r), lay(step=0), INVALID, "point_step 0"),
    ]
    for device in (False, True):
        for streams, p, n, L, status, text in cases:
            ids = (C.c_int32 * 1)(*streams) if streams is not None else None
            ptr = (C.c_void_p * 1)((d.data_ptr() if device else r.ctypes.data) if p else None)
            ns = (C.c_int64 * 1)(n)
            lays = (pwpp_b200.PwppPointLayout * 1)(L)
            if device:
                rc = lib.pwpp_estimate_device_records(eng._h, 1, ids, ptr, ns, lays, None)
            else:
                rc = lib.pwpp_estimate_host_records(eng._h, 1, ids, ptr, ns, lays)
            assert rc == status and text.encode() in lib.pwpp_last_error(), (device, text, rc, lib.pwpp_last_error())
        ids = (C.c_int32 * 1)(0)
        ptr = (C.c_void_p * 1)(r.ctypes.data)
        ns = (C.c_int64 * 1)(len(r))
        lays = (pwpp_b200.PwppPointLayout * 1)(good)
        fn = (lambda *a: lib.pwpp_estimate_device_records(*a, None)) if device else lib.pwpp_estimate_host_records
        assert fn(eng._h, 1, ids, None, ns, lays) == INVALID
        assert fn(eng._h, 1, ids, ptr, None, lays) == INVALID
        assert fn(eng._h, 1, ids, ptr, ns, None) == INVALID
        assert fn(eng._h, 0, ids, ptr, ns, lays) == INVALID
    assert eng.launch_count() == launches
    for s in range(3):
        assert eng.export_state(s) == blobs[s], f"stream {s} changed after a refused call"
    with pytest.raises(pwpp_b200.PwppError, match="native byte order"):
        pwpp_b200.layout_from_dtype(np.dtype([("x", ">f4"), ("y", ">f4"), ("z", ">f4")]))
    with pytest.raises(pwpp_b200.PwppError, match="no field 'z'"):
        pwpp_b200.layout_from_dtype(np.dtype([("x", "<f4"), ("y", "<f4")]))


def test_pointcloud2_message_of_any_layout_drives_the_real_engine(scans, tmp_path):
    """tests/pc2_records_driver.cpp: patchwork::estimateGround(pw, PointCloud2Message) for the five layouts of pc2_driver.cpp plus
    UINT8 intensity, default parameters. With intensity (any datatype) RNR runs: the result equals the engine's N x 4 call, and
    the scan's reflected-noise points make it differ from the N x 3 call. Without intensity it equals the N x 3 call."""
    import pwpp_b200
    exe = os.path.join(os.path.dirname(pwpp_b200.LIB_PATH), "pc2_records_driver")
    assert os.path.exists(exe), "lib/pc2_records_driver was not built (patchwork-plusplus_b200/build.py)"
    a = np.ascontiguousarray(np.concatenate([scans[2][:60000], scans[6][-400:]]))
    a.tofile(tmp_path / "scan.bin")
    out = subprocess.run([exe, str(tmp_path / "scan.bin")], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.splitlines()
    assert {"bigendian refused", "count2 refused", "noz refused"} <= set(lines)
    names = {"xyz12", "xyzi16", "pcl_xyzi32", "velodyne22", "ouster48_noint", "xyzi13_u8"}
    rows = {t[0]: [int(x) for x in t[1:]] for t in (l.split() for l in lines) if t and t[0] in names}
    assert set(rows) == names

    def expect(arr):
        eng = engine(1, 1)
        eng.estimate_host([np.ascontiguousarray(arr)])
        g, ng = eng.ground_indices(0).astype(np.int64), eng.nonground_indices(0)
        cn = 0
        for v in ng.tolist():
            cn = (cn * 1000003 + v) % 1000000007
        return [len(g), len(ng), int((g * (g % 97 + 1)).sum()), cn]

    u8 = a.copy()
    u8[:, 3] = np.clip(np.floor(a[:, 3] * np.float32(255)), 0, 255)
    n4, n3, nu8 = expect(a), expect(a[:, :3]), expect(u8)
    assert n4[3] != n3[3]   # RNR changed the non-ground list
    for name, row in rows.items():
        want = n3 if name in ("xyz12", "ouster48_noint") else (nu8 if name == "xyzi13_u8" else n4)
        assert row == want, name
