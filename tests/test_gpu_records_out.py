"""Ground and non-ground clouds in the sensor's own record layout (pwpp_device_record_results, pwpp_host_record_results,
pwpp_copy_ground_records, pwpp_copy_nonground_records; Engine.ground_records / nonground_records / device_record_lists).

Every list's records must equal input_records[that list's indices] byte for byte: the layouts of tests/test_gpu_records.py
(their non-coordinate bytes are random, so padding and unused fields are checked too), the six KITTI fixtures and the scan
with reflected-noise hits. Paths: host records from pageable and page-locked memory, device records 1..15 bytes past an
allocation's base, repeated one-frame calls (the small-call graph replays), a call of several pipeline chunks, stream tables
with repeats, a three-set context, both output orders."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import test_gpu_records as R

pytestmark = pytest.mark.gpu

scans = R.scans   # the six fixtures plus the RNR-hit scan


def check_frame(eng, f, r, what):
    """Frame f's record results against its input records r (a structured array or (n, step) uint8 rows)."""
    rows = r.view(np.uint8).reshape(len(r), -1)
    g, ng = eng.ground_indices(f), eng.nonground_indices(f)
    gr, nr = eng.ground_records(f), eng.nonground_records(f)
    assert gr.dtype == r.dtype and nr.dtype == r.dtype, what
    assert gr.tobytes() == rows[g].tobytes(), f"{what}: ground records"
    assert nr.tobytes() == rows[ng].tobytes(), f"{what}: non-ground records"


def check_views(eng, data, what):
    """Host view, device view and h_offsets: frame f's region at offsets[f] (16-byte aligned, room for its n records), ground
    records then non-ground records; the two views agree on every listed byte."""
    import torch
    d_rec, d_off = eng.device_record_lists()
    eng.synchronize()
    h_rec, h_off = eng.host_record_lists()
    assert (d_off == h_off).all() and h_off[0] == 0 and (h_off % 16 == 0).all(), what
    d_host = d_rec.cpu().numpy() if d_rec.numel() else np.empty(0, np.uint8)
    assert d_rec.dtype == torch.uint8 and len(d_host) == h_off[-1] == len(h_rec)
    for f, r in enumerate(data):
        step = r.dtype.itemsize
        assert h_off[f + 1] - h_off[f] == (len(r) * step + 15) // 16 * 16, f"{what}: region of frame {f}"
        m = (eng.num_ground(f) + eng.num_nonground(f)) * step
        lists = np.concatenate([eng.ground_indices(f), eng.nonground_indices(f)])
        want = r.view(np.uint8).reshape(len(r), step)[lists].ravel()
        assert np.array_equal(h_rec[h_off[f]:h_off[f] + m], want), f"{what}: host view of frame {f}"
        assert np.array_equal(d_host[h_off[f]:h_off[f] + m], want), f"{what}: device view of frame {f}"


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "page_locked"])
@pytest.mark.parametrize("name", list(R.LAYOUTS))
def test_host_one_frame_calls(scans, name, pinned, order):
    """One stream, one frame per call through all seven scans, twice over (the second pass replays the small-call graph). The
    first request of a call gathers once (one launch); later requests and the per-frame getters launch nothing more."""
    import pwpp_b200
    eng = R.engine(order=order)
    lay = pwpp_b200.layout_from_dtype(R.LAYOUTS[name])
    for rep in range(2):
        for k, a in enumerate(scans):
            r, _ = R.records(a, R.LAYOUTS[name], seed=k + 7 * rep)
            if pinned:
                ptr = eng.lib.pwpp_host_alloc(r.nbytes)
                buf = np.ctypeslib.as_array((C.c_uint8 * r.nbytes).from_address(ptr))
                buf[:] = r.view(np.uint8)
                eng.estimate_host_records([(buf, lay)])
                rows = buf.reshape(len(r), -1).copy()
                eng.lib.pwpp_host_free(ptr)   # (the host path keeps its own copy of the records)
            else:
                eng.estimate_host_records([r])
                rows = r
            l0 = eng.launch_count()
            check_frame(eng, 0, rows, f"{name} pass {rep} scan {k}")
            assert eng.launch_count() == l0 + 1
            if pinned:
                assert eng.ground_records(0).shape == (eng.num_ground(0), r.dtype.itemsize)
            check_views(eng, [r], f"{name} pass {rep} scan {k}")
            assert eng.launch_count() == l0 + 1


@pytest.mark.parametrize("name", list(R.LAYOUTS))
def test_device_records_misaligned(scans, name):
    """Seven frames on the device, each its own allocation starting 1..15 bytes past its base; both views and the getters."""
    import torch
    import pwpp_b200
    lay = pwpp_b200.layout_from_dtype(R.LAYOUTS[name])
    eng = R.engine(7)
    for call in range(2):
        data = [R.records(scans[(f + 3 * call) % 7], R.LAYOUTS[name], seed=f + 10 * call)[0] for f in range(7)]
        bufs, ptrs = [], []
        for f, r in enumerate(data):
            mis = 1 + (4 * f + call) % 15
            t = torch.empty(mis + r.nbytes, dtype=torch.uint8, device="cuda")
            t[mis:] = torch.from_numpy(r.view(np.uint8)).cuda()
            bufs.append(t)
            ptrs.append(t.data_ptr() + mis)
        torch.cuda.synchronize()
        eng.estimate_device_records(ptrs, [len(r) for r in data], [lay] * 7, dtypes=[r.dtype for r in data])
        check_views(eng, data, f"{name} call {call}")
        for f, r in enumerate(data):
            check_frame(eng, f, r, f"{name} call {call} frame {f}")


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
def test_host_batch_over_several_pipeline_chunks(scans, order):
    """80 frames of mixed layouts in one call (several pipeline chunks): one gather covers every frame."""
    nf = 80
    eng = R.engine(nf, order)
    data = [R.records(scans[f % 7], R.LAYOUTS[R.WITH_I[f % len(R.WITH_I)]], seed=f)[0] for f in range(nf)]
    eng.estimate_host_records(data)
    total = sum(len(r) for r in data)
    assert -(-nf // min(nf, max(1, (4 << 20) // max(1, total // nf)))) >= 2
    l0 = eng.launch_count()
    check_views(eng, data, "batch")
    for f, r in enumerate(data):
        check_frame(eng, f, r, f"frame {f}")
    assert eng.launch_count() == l0 + 1


@pytest.mark.parametrize("path", ["host", "device"])
def test_stream_table_with_repeats_and_mixed_layouts(scans, path):
    """Stream tables naming streams several times, every frame with its own layout, frames without intensity among frames with it."""
    import torch
    import pwpp_b200
    calls = [([2, 0, 2, 1, 3, 0, 1], ["xyz12", "pcl_xyzi32", "velodyne22", "xyz12", "u16_intensity", "f64_xyz", "rec48"]),
             ([3, 3, 1], ["u8_intensity", "xyz12", "f64_intensity"])]
    eng = R.engine(4, 1)
    for c, (streams, names) in enumerate(calls):
        data = [R.records(scans[(3 * c + f) % 7], R.LAYOUTS[names[f]], seed=f)[0] for f in range(len(streams))]
        if path == "host":
            eng.estimate_host_records(data, streams=streams)
        else:
            bufs = [torch.from_numpy(r.view(np.uint8).copy()).cuda() for r in data]
            torch.cuda.synchronize()
            eng.estimate_device_records([b.data_ptr() for b in bufs], [len(r) for r in data], [pwpp_b200.layout_from_dtype(r.dtype) for r in data],
                                        streams=streams, dtypes=[r.dtype for r in data])
        for f, r in enumerate(data):
            check_frame(eng, f, r, f"call {c} position {f}")
        check_views(eng, data, f"call {c}")


def test_parameter_sets_each_stream_its_own_layout(scans):
    from param_sets import PARAM_SETS
    sets = [PARAM_SETS[n][0]() for n in ("default", "ros", "no_rvpf_tgr")]
    lay_of = ["pcl_xyzi32", "xyz12", "u16_intensity"]
    eng = R.engine(3, 0, params=sets, stream_set=[0, 1, 2])
    for c, streams in enumerate(([0, 1, 2], [2, 0, 1], [1, 2, 1, 0])):
        data = [R.records(scans[(c + f) % 7], R.LAYOUTS[lay_of[s]], seed=f)[0] for f, s in enumerate(streams)]
        eng.estimate_host_records(data, streams=streams)
        for f, r in enumerate(data):
            check_frame(eng, f, r, f"call {c} position {f}")
        check_views(eng, data, f"call {c}")


def test_getters_refuse_calls_without_records(scans, kitti):
    """Before any call and after a float call every record getter fails with a message (and returns no stale records); a
    frame outside the call fails; the next records call makes them work again."""
    import pwpp_b200
    eng = R.engine(2)
    lib, h = eng.lib, eng._h
    out = np.zeros(1 << 20, np.uint8)
    a, b = C.c_void_p(), C.c_void_p()

    def all_fail(text):
        assert lib.pwpp_copy_ground_records(h, 0, out.ctypes.data) == -1 and text in lib.pwpp_last_error()
        assert lib.pwpp_copy_nonground_records(h, 0, out.ctypes.data) == -1
        assert lib.pwpp_host_record_results(h, C.byref(a), C.byref(b)) == -1
        assert lib.pwpp_device_record_results(h, C.byref(a), C.byref(b)) == -1
    all_fail(b"")
    r, _ = R.records(scans[1], R.LAYOUTS["velodyne22"])
    eng.estimate_host_records([r, r])
    check_frame(eng, 1, r, "first records call")
    assert lib.pwpp_copy_ground_records(h, 2, out.ctypes.data) == -1 and b"frame index" in lib.pwpp_last_error()
    assert lib.pwpp_copy_nonground_records(h, -1, out.ctypes.data) == -1
    l0 = eng.launch_count()
    eng.estimate_host([kitti[0]])
    all_fail(b"did not take records")
    with pytest.raises(pwpp_b200.PwppError, match="did not take records"):
        eng.ground_records(0)
    with pytest.raises(pwpp_b200.PwppError, match="did not take records"):
        eng.device_record_lists()
    import torch
    pts = torch.from_numpy(R.padded(kitti[2])).cuda()
    torch.cuda.synchronize()
    eng.estimate_device(pts.data_ptr(), [0, len(kitti[2])])
    all_fail(b"did not take records")
    assert eng.launch_count() > l0
    r2, _ = R.records(scans[4], R.LAYOUTS["rec48"], seed=3)
    eng.estimate_host_records([r2])
    check_frame(eng, 0, r2, "records call after float calls")
    assert lib.pwpp_copy_ground_records(h, 1, out.ctypes.data) == -1   # the call had one frame


@pytest.mark.parametrize("path", ["host", "device"])
def test_fetching_leaves_results_and_state_untouched(scans, path):
    """Two contexts get the same calls; one fetches the record results (both views) after every call, between frames of the
    same streams. Results and state stay bit-identical to the context that never asks, and a call that does not ask
    launches exactly the kernels of one that never asked."""
    import torch
    import pwpp_b200
    seq = [([0, 1], ["velodyne22", "pcl_xyzi32"]), ([1, 0, 1], ["pcl_xyzi32", "velodyne22", "pcl_xyzi32"]), ([0], ["velodyne22"]),
           ([0], ["velodyne22"]), ([1, 0], ["pcl_xyzi32", "velodyne22"])]
    ask, quiet = R.engine(2, 1), R.engine(2, 1)
    for c, (streams, names) in enumerate(seq):
        data = [R.records(scans[(2 * c + f) % 7], R.LAYOUTS[names[f]], seed=c + f)[0] for f in range(len(streams))]
        deltas, keep = [], []   # (each context's device buffers stay alive until its results are fetched)
        for eng in (ask, quiet):
            l0 = eng.launch_count()
            if path == "host":
                eng.estimate_host_records(data, streams=streams)
            else:
                bufs = [torch.from_numpy(r.view(np.uint8).copy()).cuda() for r in data]
                keep.append(bufs)
                torch.cuda.synchronize()
                eng.estimate_device_records([b.data_ptr() for b in bufs], [len(r) for r in data],
                                            [pwpp_b200.layout_from_dtype(r.dtype) for r in data], streams=streams, dtypes=[r.dtype for r in data])
                eng.synchronize()
            deltas.append(eng.launch_count() - l0)
        assert deltas[0] == deltas[1], f"call {c}: launches {deltas}"
        l1 = ask.launch_count()
        check_views(ask, data, f"call {c}")
        for f, r in enumerate(data):
            check_frame(ask, f, r, f"call {c} position {f}")
        assert ask.launch_count() == l1 + 1
        for f in range(len(streams)):
            assert R.outputs(ask, f) == R.outputs(quiet, f), f"call {c} position {f}"
        for s in range(2):
            assert R.stream(ask, s) == R.stream(quiet, s), f"call {c} stream {s}"


def test_records_payload_drives_the_real_engine(scans, tmp_path):
    """tests/pc2_records_out_driver.cpp: estimateGround(pw, message) then makeRecordsPayload for ground and non-ground, for
    velodyne22, pcl_xyzi32 and xyz12 messages with random filler bytes: the payload carries the input's point_step and fields,
    height 1, width = count, row_step, and records[indices] byte for byte; the getters throw after a float call."""
    import pwpp_b200
    exe = os.path.join(os.path.dirname(pwpp_b200.LIB_PATH), "pc2_records_out_driver")
    assert os.path.exists(exe), "lib/pc2_records_out_driver was not built (patchwork-plusplus_b200/build.py)"
    np.ascontiguousarray(scans[6]).tofile(tmp_path / "scan.bin")
    out = subprocess.run([exe, str(tmp_path / "scan.bin")], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    for name in ("velodyne22", "pcl_xyzi32", "xyz12"):
        row = [l.split() for l in lines if l.startswith(name + " ")]
        assert row and row[0][1] == "ok", (name, lines)
        assert int(row[0][2]) > 0 and int(row[0][3]) > 0
    assert "float call refused" in lines
