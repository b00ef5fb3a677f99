"""Stream state on the GPU through the C-ABI and the Engine: pwpp_export_states_device / pwpp_import_states_device (snapshot,
rollback, fork and migration of streams inside the caller's stream order, capturable) and pwpp_clone (a copy of a whole ctx).

The contexts hold three parameter sets with small history storage (the histories fill up and are trimmed within a few scans;
one set's history capacity is odd). Every comparison is bit for bit: device rows against pwpp_export_state's blobs, and the
frames after an import or a clone against the source stream continuing (index lists, bin ids, centers, normals, xyz, patch
records, pwpp_get_state, histories and the exported blob)."""
import os
import subprocess

import numpy as np
import pytest

from param_sets import _default, _no_rvpf_tgr, _ros
from test_gpu_bound_call import NAMES, Pair
from test_gpu_records import outputs, stream

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
OK, SKIPPED, OUT_OF_RANGE, BLOB_MISMATCH, DUPLICATE = 0, 1, 2, 3, 4
ERR_INVALID_ARG = -1
SENT = 0xA5


def sets3():
    a, b, c = _default(), _ros(), _no_rvpf_tgr()
    a.max_elevation_storage = a.max_flatness_storage = 20
    b.max_elevation_storage, b.max_flatness_storage = 7, 5     # history capacity 7 + 4 * 54 + 64 = 287: odd
    return [a, b, c]


def engine3(ns=6, order=1):
    import pwpp_b200
    e = pwpp_b200.Engine(sets3(), device=0, num_streams=ns, stream_set=[s % 3 for s in range(ns)])
    e.set_output_order(order)
    return e


def no_plane_scan(a):
    """Scan a with the first bin of zone 0 (ring 0, sector 0) emptied and refilled with 40 points at z = 1e30: their mean is the
    low-point representative, and 1e30 + th_seeds rounds to 1e30 in double, so no point passes a seed test. The patch has no
    plane of its own, and as the first patch of the frame it takes the plane the stream carried
    from its previous frame (StreamState's stale plane, part of the blob)."""
    r = np.hypot(a[:, 0], a[:, 1])
    th = np.degrees(np.arctan2(a[:, 1], a[:, 0]))
    keep = ~((r > 2.5) & (r < 7.8) & (th > -2) & (th < 24))
    rng = np.random.default_rng(9)
    extra = np.stack([4.0 + rng.uniform(0, 0.2, 40), 0.3 + rng.uniform(0, 0.2, 40), np.full(40, 1e30), np.ones(40)], 1)
    return np.ascontiguousarray(np.concatenate([a[keep], extra.astype(np.float32)]))


def drive(eng, scans, streams, rounds, seed=0):
    """rounds calls over `streams`, frame f of call r = scans[(r + f + seed) % 6]."""
    for r in range(rounds):
        eng.estimate_host([scans[(r + f + seed) % len(scans)] for f in range(len(streams))], streams=list(streams))
    eng.synchronize()


def host_rows(eng, rows, streams):
    return [bytes(rows[i, :len(eng.export_state(s))].cpu().numpy().tobytes()) for i, s in enumerate(streams)]


@pytest.fixture(scope="module")
def scans(kitti):
    return list(kitti)


def test_device_export_is_export_state_for_every_stream(scans):
    import torch
    e = engine3()
    drive(e, scans, range(6), 8)
    stride = (e.state_blob_size() + 15) // 16 * 16 + 32
    rows = torch.full((6, stride), SENT, dtype=torch.uint8, device="cuda")
    perm = [4, 0, 5, 2, 1, 3]
    _, st = e.export_states(perm, out=rows)
    torch.cuda.synchronize()
    assert st.cpu().tolist() == [OK] * 6
    r = rows.cpu().numpy()
    for i, s in enumerate(perm):
        blob = e.export_state(s)
        assert r[i, :len(blob)].tobytes() == blob, f"row {i} (stream {s})"
        assert (r[i, len(blob):] == SENT).all(), f"row {i}: bytes past the stream's blob were written"
        st_ = e.state(s)
        assert max(st_.n_elevation) > 0 and max(st_.n_flatness) > 0


def test_import_continues_bit_for_bit(scans):
    """Streams 0..2 run k scans, a no-plane patch among them; their device rows go into streams 3..5 of the same ctx (one per
    set) and into streams 0..2 of another ctx. Then all three copies of every stream run the same frames."""
    import torch
    src, dst = engine3(), engine3()
    special = no_plane_scan(scans[1])
    drive(src, scans, range(3), 5)
    src.estimate_host([special, scans[2], scans[3]], streams=[0, 1, 2])
    src.synchronize()
    np_bins = [b for b in src.bin_results(0) if b.n == 40 and b.fitted and b.n_ground == 0 and np.all(np.isfinite(b.mean))]
    assert np_bins, "the no-plane patch did not occur"
    drive(dst, scans, range(3), 2, seed=3)     # the target streams hold other state before the import
    rows, st = src.export_states([0, 1, 2])
    assert src.import_states(rows, [3, 4, 5]).cpu().tolist() == [OK] * 3
    assert dst.import_states(rows, torch.tensor([0, 1, 2], dtype=torch.int32, device="cuda")).cpu().tolist() == [OK] * 3
    torch.cuda.synchronize()
    for s in range(3):
        assert stream(src, s) == stream(src, s + 3) == stream(dst, s), f"stream {s} after the import"
    for r in range(4):
        frames = [special if r == 1 else scans[(r + f) % 6] for f in range(3)]
        src.estimate_host(frames + frames, streams=[0, 1, 2, 3, 4, 5])
        dst.estimate_host(frames + frames, streams=[0, 1, 2, 3, 4, 5])   # the same call size: the same kernel variants
        for f in range(3):
            assert outputs(src, f) == outputs(src, f + 3) == outputs(dst, f), f"round {r} frame {f}"
            assert stream(src, f) == stream(src, f + 3) == stream(dst, f), f"round {r} stream {f}"


def test_host_and_device_blobs_interoperate(scans):
    import torch
    src, a, b = engine3(), engine3(), engine3()
    drive(src, scans, range(6), 6)
    rows, _ = src.export_states(range(6))
    blobs = host_rows(src, rows, range(6))
    for s in range(6):                        # device row -> host import
        a.import_state(s, blobs[s])
    stride = rows.shape[1]
    dev = torch.full((6, stride), SENT, dtype=torch.uint8, device="cuda")
    for s in range(6):                        # host export -> device row -> device import
        blob = np.frombuffer(src.export_state(s), np.uint8)
        dev[s, :len(blob)] = torch.from_numpy(blob.copy()).cuda()
    assert b.import_states(dev, range(6)).cpu().tolist() == [OK] * 6
    torch.cuda.synchronize()
    for s in range(6):
        assert stream(a, s) == stream(src, s) == stream(b, s), f"stream {s}"


def test_rejected_entries_leave_streams_unchanged(scans):
    import torch
    src, dst = engine3(), engine3()
    drive(src, scans, range(6), 4)
    drive(dst, scans, range(6), 3, seed=2)
    rows, _ = src.export_states([0, 1, 2, 3, 4, 5, 0, 1])
    before = [stream(dst, s) for s in range(6)]
    rows[1, 0] ^= 1                            # magic
    rows[2, 4] ^= 1                            # version
    rows[3, 8] ^= 1                            # hcap
    rows[4, 12] ^= 16                          # state size
    ids = [0, 1, 2, 3, 4, -1, 7, 0]           # stream 5 skipped, 7 out of range, stream 0 twice
    st = dst.import_states(rows, ids).cpu().tolist()
    torch.cuda.synchronize()
    assert st == [OK, BLOB_MISMATCH, BLOB_MISMATCH, BLOB_MISMATCH, BLOB_MISMATCH, SKIPPED, OUT_OF_RANGE, DUPLICATE]
    assert stream(dst, 0) == stream(src, 0)
    for s in range(1, 6):
        assert stream(dst, s) == before[s], f"stream {s} changed"
    # stream 0's row (set 0) imported into stream 4 (set 1, another history capacity)
    r0, _ = src.export_states([0])
    assert dst.import_states(r0, [4]).cpu().tolist() == [BLOB_MISMATCH] and stream(dst, 4) == before[4]


def test_launch_counts_and_host_checks(scans):
    import torch
    e = engine3()
    lib, h = e.lib, e._h
    rows, _ = e.export_states(range(6))
    torch.cuda.synchronize()
    l0 = e.launch_count()
    e.export_states([0, 1])
    assert e.launch_count() - l0 == 1
    e.import_states(rows, [2, -1, 5])
    assert e.launch_count() - l0 == 3
    ids = torch.arange(6, dtype=torch.int32, device="cuda")
    size = e.state_blob_size()
    stride = rows.stride(0)
    ok = lambda n, p_ids, p_rows, st: (lib.pwpp_export_states_device(h, n, p_ids, p_rows, st, None, None),
                                       lib.pwpp_import_states_device(h, n, p_ids, p_rows, st, None, None))
    assert ok(0, None, None, stride) == (0, 0)
    assert e.launch_count() - l0 == 3          # n == 0 launches nothing
    for args in [(-1, ids.data_ptr(), rows.data_ptr(), stride), (65536, ids.data_ptr(), rows.data_ptr(), stride),
                 (2, None, rows.data_ptr(), stride), (2, ids.data_ptr(), None, stride),
                 (2, ids.data_ptr(), rows.data_ptr(), size - 16), (2, ids.data_ptr(), rows.data_ptr(), stride + 8),
                 (2, ids.data_ptr(), rows.data_ptr() + 8, stride)]:
        assert ok(*args) == (ERR_INVALID_ARG, ERR_INVALID_ARG), args
    assert e.launch_count() - l0 == 3


def test_snapshot_run_and_rollback_in_one_graph(scans):
    """One CUDA graph: export every stream (row i = stream i), run the bound call, import row i into the stream that entry i of
    the list names (-1: keep the tick; i itself: roll stream i back; another stream of the set: fork stream i's snapshot into
    it). The list is rewritten between replays. A twin driven by direct calls and pwpp_import_state agrees after each."""
    import torch
    sz = max(len(a) for a in scans)
    p = Pair([0, 1, 2, 3], NAMES, [sz] * 4, order=1)
    p.step(scans, 0, "eager run before the capture")
    ns = 4
    ids = torch.arange(ns, dtype=torch.int32, device="cuda")
    restore = torch.full((ns,), -1, dtype=torch.int32, device="cuda")
    rows = torch.empty((ns, (p.eng.state_blob_size() + 15) // 16 * 16), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cs = torch.cuda.current_stream().cuda_stream
        p.eng.export_states(ids, out=rows, stream=cs)
        p.eng.run_bound_call(cs)
        status = p.eng.import_states(rows, restore, stream=cs)
    plans = [[-1, -1, -1, -1], [-1, 1, -1, 3], [0, 1, 2, 3], [2, -1, -1, -1], [-1, -1, -1, -1], [3, 3, -1, 0]]
    for rep, plan in enumerate(plans):
        restore.copy_(torch.tensor(plan, dtype=torch.int32))
        sizes = p.load(scans, rep + 1)
        g.replay()
        torch.cuda.synchronize()
        snap = {s: p.twin.export_state(s) for s in range(ns)}
        p.run_twin(sizes)
        seen = set()
        want = []
        for i, s in enumerate(plan):              # row i holds stream i's snapshot: [2, -1, ...] forks stream 0 into stream 2
            if s < 0:
                want.append(SKIPPED)
            elif s in seen:
                want.append(DUPLICATE)
            else:
                seen.add(s)
                want.append(OK)
                p.twin.import_state(s, snap[i])
        assert status.cpu().tolist() == want, f"replay {rep}"
        p.check(sizes, f"replay {rep} with rollback of {plan}")


def test_clone(scans):
    import torch
    import pwpp_b200
    src = engine3()
    drive(src, scans, range(6), 3)
    src.estimate_host([no_plane_scan(scans[0]), scans[1], scans[2], scans[3]], streams=[4, 0, 5, 1])
    src.synchronize()
    c = src.clone()
    assert c.launch_count() == 0
    for f in range(4):
        assert outputs(c, f) == outputs(src, f), f"frame {f} of the last call on the clone"
        assert c.num_patches(f) == src.num_patches(f)
    for s in range(6):
        assert stream(c, s) == stream(src, s), f"stream {s} on the clone"
    assert c.time_us() == src.time_us()
    hi, hn, ho = src.host_index_lists()
    ci, cn, co = c.host_index_lists()
    assert np.array_equal(hi, ci) and np.array_equal(hn, cn) and np.array_equal(ho, co)
    di, dn = src.device_index_lists()
    ei, en = c.device_index_lists()
    assert ei.data_ptr() != di.data_ptr() and torch.equal(di, ei) and torch.equal(dn, en)
    for r in range(3):
        frames = [scans[(r + f) % 6] for f in range(6)]
        for e in (src, c):
            e.estimate_host(frames, streams=[5, 4, 3, 2, 1, 0])
        for f in range(6):
            assert outputs(c, f) == outputs(src, f), f"continuation {r} frame {f}"
        for s in range(6):
            assert stream(c, s) == stream(src, s)
    c.close()
    # refused while a call is bound; allowed again after the unbind
    sz = max(len(a) for a in scans)
    p = Pair([0, 1], NAMES[:2], [sz] * 2)
    p.step(scans, 0, "bound run")
    with pytest.raises(pwpp_b200.PwppError, match="unbind"):
        p.eng.clone()
    p.eng.unbind_call()
    d = p.eng.clone()
    for f in range(2):
        assert outputs(d, f) == outputs(p.eng, f)


def test_clone_on_another_device(scans):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device visible")
    src = engine3()
    drive(src, scans, range(6), 3)
    c = src.clone(device=1)
    for f in range(6):
        assert outputs(c, f) == outputs(src, f)
    for s in range(6):
        assert stream(c, s) == stream(src, s)
    for e in (src, c):
        e.estimate_host(scans[:6], streams=list(range(6)))
    for f in range(6):
        assert outputs(c, f) == outputs(src, f)


def test_dropin_copies(tmp_path, kitti):
    exe = os.path.join(REPO, "patchwork-plusplus_b200", "lib", "pwpp_copy_driver")
    assert os.path.exists(exe), "lib/pwpp_copy_driver was not built (patchwork-plusplus_b200/build.py)"
    paths = []
    for i in range(6):
        p = tmp_path / f"{i:06d}.bin"
        np.ascontiguousarray(kitti[i], np.float32).tofile(p)
        paths.append(str(p))
    out = subprocess.run([exe, "3"] + paths, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    rows = {}
    for line in out.stdout.splitlines():
        tok = line.split()
        if len(tok) > 2 and tok[0] in ("a", "b", "c", "fresh", "fresh_copy") and tok[1] != "empty":
            rows.setdefault(tok[1], {})[tok[0]] = tok[2:]
    assert set(rows) == {"copied", "frame3", "frame4", "frame5", "first"}
    for tag, by in rows.items():
        vals = list(by.values())
        assert len(vals) >= 2 and all(v == vals[0] for v in vals), f"{tag}: {by}"
    assert "fresh empty 0 0" in out.stdout
    assert out.stdout.count("INITIALIZATION COMPLETE") == 3, "copies print no banner"
