"""Record results of a bound call (pwpp_bind_record_results / pwpp_bound_record_results): the ground and non-ground clouds of
every frame as the sensor's own records, gathered on the GPU into fixed device buffers, also inside a captured CUDA graph.

Every run is compared with a twin context driven by pwpp_estimate_device_records with the same frames and sizes
(tests/test_gpu_bound_call.py's Pair): for every frame and part, the region's first count * point_step bytes equal the twin's
ground_records / nonground_records and the input records at the bound call's own index lists, the counts equal the twin's, and
the bytes after them keep the sentinel both buffers are filled with before the run."""
import hashlib

import numpy as np
import pytest

from test_gpu_bound_call import CASES, NAMES, Pair, engine
from test_gpu_records import LAYOUTS, records

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
ERR_INVALID_ARG = -1


@pytest.fixture(scope="module")
def scans(kitti):
    return list(kitti)


def fill(p):
    """Fills the enabled part buffers with the sentinel, done before the next run on any stream."""
    import torch
    g, ng, _, _ = p.eng.bound_record_results()
    for b in (g, ng):
        if b is not None:
            b.fill_(SENTINEL)
    torch.cuda.synchronize()


def check_records(p, sizes, what, parts=3):
    """The record results of the bound call's last run against the twin's last call (same sizes) and the input records."""
    import torch
    torch.cuda.synchronize()
    g, ng, off, cnt = p.eng.bound_record_results()
    assert (g is None) == (not parts & 1) and (ng is None) == (not parts & 2), f"{what}: views of the parts"
    bufs = [None if b is None else b.cpu().numpy() for b in (g, ng)]
    cnt = cnt.cpu().numpy()
    idx, poff, nground, _ = p.eng.bound_call_results()
    idx, poff, nground = idx.cpu().numpy(), poff.cpu().numpy(), nground.cpu().numpy()
    nf = len(p.streams)
    assert cnt.shape == (nf, 2)
    want_off = np.cumsum([0] + [(m * LAYOUTS[nm].itemsize + 15) // 16 * 16 for nm, m in zip(p.names, p.max_n)])
    assert np.array_equal(off, want_off), f"{what}: offsets"
    for f in range(nf):
        step = LAYOUTS[p.names[f]].itemsize
        want_cnt = [p.twin.num_ground(f), p.twin.num_nonground(f)]
        assert cnt[f].tolist() == want_cnt, f"{what}: frame {f} counts"
        assert int(nground[f]) == want_cnt[0]
        src = p.data[f].view(np.uint8).reshape(-1, step)[: sizes[f]]
        o = int(poff[f])
        lists = [idx[o: o + want_cnt[0]], idx[o + want_cnt[0]: o + sum(want_cnt)]]
        twin = [p.twin.ground_records(f), p.twin.nonground_records(f)]
        for z, buf in enumerate(bufs):
            if buf is None:
                continue
            k = want_cnt[z] * step
            region = buf[off[f]: off[f + 1]]
            assert np.array_equal(region[:k], np.ascontiguousarray(twin[z]).view(np.uint8).reshape(-1)), f"{what}: frame {f} part {z} vs the twin"
            assert np.array_equal(region[:k], src[lists[z]].reshape(-1)), f"{what}: frame {f} part {z} vs records[idx]"
            assert (region[k:] == SENTINEL).all(), f"{what}: frame {f} part {z}: a byte past the count was written"


def run_and_check(p, scans, seed, what, counts=None, parts=3):
    sizes = p.load(scans, seed, counts)
    fill(p)
    p.eng.run_bound_call()
    p.run_twin(sizes)
    check_records(p, sizes, what, parts)
    return sizes


RECORD_CASES = ["one_frame", "four_frames", "stream_table_with_repeats", "sixty_four_frames", "dense_capacities_small_counts"]


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
@pytest.mark.parametrize("case", RECORD_CASES)
def test_record_results_equal_the_twin(scans, case, order):
    """Two runs with state carried; layouts mixed within the call (16-byte float4, velodyne22, pcl_xyzi32, FLOAT64 xyz)."""
    streams, caps = CASES[case]
    sz = max(len(a) for a in scans)
    names = [NAMES[f % len(NAMES)] for f in range(len(streams))]
    p = Pair(streams, names, caps(sz), order)
    p.eng.bind_record_results()
    for run in range(2):
        run_and_check(p, scans, run, f"{case} run {run}")


@pytest.mark.parametrize("parts", [1, 2])
def test_one_part(scans, parts):
    """One part alone: the other view is None and both counts are still written."""
    sz = max(len(a) for a in scans)
    p = Pair([0, 1, 2, 3], NAMES, [sz + 50] * 4, order=1)
    p.eng.bind_record_results(ground=parts == 1, nonground=parts == 2)
    for run in range(2):
        run_and_check(p, scans, run, f"parts {parts} run {run}", parts=parts)


def digest(p):
    g, ng, _, cnt = p.eng.bound_record_results()
    return [hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest() for t in (g, ng, cnt)]


def test_graph_capture_and_replays(scans):
    """Record results enabled before the capture; 8 replays with new frames and counts (halved counts in one, an out-of-range
    count in another), each compared. A direct records call between two replays returns its own record results and leaves the
    bound buffers unchanged."""
    import torch
    sz = max(len(a) for a in scans)
    p = Pair([0, 1, 2, 3, 0], NAMES + ["velodyne22"], [sz + 100] * 5, order=1)
    p.eng.bind_record_results()
    run_and_check(p, scans, 0, "eager run before the capture")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        p.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    for rep in range(8):
        counts = None
        if rep == 5:
            counts = [len(scans[(f + rep + 1) % 6]) // 2 for f in range(5)]
        if rep == 6:
            counts = [len(scans[(f + rep + 1) % 6]) for f in range(5)]
            counts[2] = sz + 101
        sizes = p.load(scans, rep + 1, counts)
        fill(p)
        g.replay()
        torch.cuda.synchronize()
        p.run_twin(sizes)
        check_records(p, sizes, f"replay {rep}")
        if rep == 6:
            assert sizes[2] == 0 and p.eng.bound_record_results()[3][2].tolist() == [0, 0]
        if rep == 3:   # a direct records call of two frames on both contexts
            before = digest(p)
            data = [records(scans[k], LAYOUTS["velodyne22"], seed=k)[0] for k in (4, 5)]
            bufs = [torch.from_numpy(r.view(np.uint8).copy()).cuda() for r in data]
            lays = [p.lays[1]] * 2
            torch.cuda.synchronize()
            for e in (p.eng, p.twin):
                e.estimate_device_records([b.data_ptr() for b in bufs], [len(r) for r in data], lays, streams=[1, 3])
                e.synchronize()
            for f in range(2):
                assert np.array_equal(p.eng.ground_records(f), p.twin.ground_records(f)), f"direct call frame {f} ground"
                assert np.array_equal(p.eng.nonground_records(f), p.twin.nonground_records(f)), f"direct call frame {f} non-ground"
            torch.cuda.synchronize()
            assert digest(p) == before, "the direct call changed the bound record buffers"


def test_no_host_synchronisation(scans):
    """With record results on and a long sleep kernel ahead on the stream, run_bound_call and a graph replay return at once."""
    import torch
    sz = max(len(a) for a in scans)
    p = Pair([0, 1], ["xyzi16", "velodyne22"], [sz] * 2)
    p.eng.bind_record_results()
    run_and_check(p, scans, 0, "eager run")   # every kernel loaded before the timing-sensitive part
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda._sleep(2_000_000_000)
        p.eng.run_bound_call(st.cuda_stream)
        assert not st.query(), "run_bound_call waited for the stream"
    st.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        p.eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    with torch.cuda.stream(st):
        torch.cuda._sleep(2_000_000_000)
        g.replay()
        assert not st.query(), "the replay waited"
    st.synchronize()
    torch.cuda.synchronize()


def test_launch_count(scans):
    """One launch more per run with record results on, also for a call whose capacities are all 0."""
    import torch
    sz = max(len(a) for a in scans)
    for max_n in ([sz, sz], [0, 0]):
        p = Pair([0, 1], ["xyzi16", "pcl_xyzi32"], max_n)
        p.load(scans, 0)
        deltas = []
        for on in (False, True):
            if on:
                p.eng.bind_record_results()
            l0 = p.eng.launch_count()
            p.eng.run_bound_call()
            deltas.append(p.eng.launch_count() - l0)
        assert deltas[1] == deltas[0] + 1, (max_n, deltas)
        torch.cuda.synchronize()
        if max_n == [0, 0]:
            assert p.eng.bound_record_results()[3].cpu().numpy().tolist() == [[0, 0], [0, 0]]


def test_errors(scans):
    import pwpp_b200
    e = engine(2, 0)
    with pytest.raises(pwpp_b200.PwppError, match="no call is bound"):
        e.bind_record_results()
    with pytest.raises(pwpp_b200.PwppError, match="no call is bound"):
        e.bound_record_results()
    sz = max(len(a) for a in scans)
    p = Pair([0, 1], ["xyzi16", "velodyne22"], [sz, sz])
    for parts in (0, 4):
        assert p.eng.lib.pwpp_bind_record_results(p.eng._h, parts) == ERR_INVALID_ARG
    with pytest.raises(pwpp_b200.PwppError, match="not enabled"):
        p.eng.bound_record_results()
    p.eng.bind_record_results(nonground=False)
    with pytest.raises(pwpp_b200.PwppError, match="already enabled"):
        p.eng.bind_record_results()
    run_and_check(p, scans, 0, "run", parts=1)

    # the record results of direct calls still refuse the bound call
    with pytest.raises(pwpp_b200.PwppError, match="bound call"):
        p.eng.device_record_lists()
    with pytest.raises(pwpp_b200.PwppError, match="bound call"):
        p.eng.ground_records(0)

    # unbinding releases them; a later bind starts with them off
    p.eng.unbind_call()
    with pytest.raises(pwpp_b200.PwppError, match="no call is bound"):
        p.eng.bound_record_results()
    p.eng.bind_call(p.ptrs, p.max_n, p.lays, p.counts, streams=p.streams)
    with pytest.raises(pwpp_b200.PwppError, match="not enabled"):
        p.eng.bound_record_results()
    p.eng.bind_record_results()
    run_and_check(p, scans, 1, "run after rebinding")
