"""PWPP_ARITH_REFERENCE on the H100: every output bit for bit the reference build's arithmetic, with no degenerate-patch mask.
The yardstick is the oracle's literal fp32 statement (PWO_ARITH_REF32, pinned to oracle/_ref/libpwref_stable.so by
test_oracle_vs_reference.py): index lists in reference order, centers, normals, getHeight, every threshold and history row and
every patch record. Every call path that runs the fits is covered (batch, small calls, device, records, stream tables, three
parameter sets, a bound call replayed in a CUDA graph), and so are the mode's rules (frozen while bound, copied by a clone,
stream-state blobs that move between modes, switching back to double)."""
import numpy as np
import pytest

import oracle_py as O
from helpers import bits
from param_sets import PARAM_SETS
from test_gpu_records import LAYOUTS, records

pytestmark = pytest.mark.gpu
REF = 1


def _engine(params=None, num_streams=1, arith=REF, order=1, stream_set=None):
    import pwpp_b200
    e = pwpp_b200.Engine(params, device=0, num_streams=num_streams, stream_set=stream_set)
    e.set_output_order(order)
    e.set_arithmetic(arith)
    assert e.arithmetic() == arith
    return e


def oracle_runs(frames, params=None, sequence=None, reference=False):
    """Per frame the oracle (REF32, equal z in ascending index order: libpwref_stable.so's arithmetic) after that frame, or with
    reference=True the unmodified reference build libpwref.so (std::sort's order of equal z): lists, centers, normals, height,
    state, histories and (oracle only) the patch records; sequence: the stream of every frame."""
    sequence = list(range(len(frames))) if sequence is None else sequence
    orcs, out = {}, []
    for a, s in zip(frames, sequence):
        p = params(s) if callable(params) else params
        if s not in orcs:
            orcs[s] = O.Reference(p, stable_sort=False) if reference else O.Oracle(p, O.ARITH_REF32)
        o = orcs[s]
        o.estimate(a)
        out.append(dict(g=o.getGroundIndices(), ng=o.getNongroundIndices(), c=o.getCenters(), n=o.getNormals(), h=o.getHeight(),
                        st=o.state(), hist=[o.history(r, w) for r in range(4) for w in (0, 1)],
                        bins=None if reference else o.bin_results(), nbins=0 if reference else o.nbins))
    return out


needs_reference = pytest.mark.skipif(not O.have_reference_build(), reason="needs the reference build (oracle/_ref/libpwref.so)")


def quantised(a, step=0.01):
    """Centimetre-quantised z: equal z in almost every bin and inside every part of a patch."""
    a = a.copy()
    a[:, 2] = np.round(a[:, 2] / step) * step
    return a


def check_bins(want, got, what):
    for b in range(want["nbins"]):
        x, y = want["bins"][b], got[b]
        assert (x.n, x.n_ground, x.verdict, x.fitted) == (y.n, y.n_ground, y.verdict, y.fitted), f"{what}: bin {b} record"
        if x.fitted and x.n > 0:
            a1 = np.array(list(x.mean) + list(x.normal) + list(x.sv) + [x.d])
            a2 = np.array(list(y.mean) + list(y.normal) + list(y.sv) + [y.d])
            assert np.array_equal(bits(a1), bits(a2)), f"{what}: bin {b} plane"


def assert_frame(want, eng, f, what, bins=True, state=True, stream=None):
    """state: compare the state of frame f's stream (`stream`, by default f) too; the state getters take a stream id and read
    the state after the whole call."""
    s = f if stream is None else stream
    assert np.array_equal(want["g"], eng.ground_indices(f)), f"{what}: ground list"
    assert np.array_equal(want["ng"], eng.nonground_indices(f)), f"{what}: non-ground list"
    assert np.array_equal(bits(want["c"]), bits(eng.centers(f))), f"{what}: centers"
    assert np.array_equal(bits(want["n"]), bits(eng.normals(f))), f"{what}: normals"
    if bins and want["bins"] is not None:
        check_bins(want, eng.bin_results(f), what)
    if not state:
        return
    assert bits(np.float64(want["h"])) == bits(np.float64(eng.height(s))), f"{what}: height"
    sa, sb = want["st"], eng.state(s)
    for fld in ("elevation_thr", "flatness_thr"):
        assert np.array_equal(bits(np.array(getattr(sa, fld))), bits(np.array(getattr(sb, fld)))), f"{what}: {fld}"
    assert list(sa.n_elevation) == list(sb.n_elevation) and list(sa.n_flatness) == list(sb.n_flatness), f"{what}: history sizes"
    k = 0
    for r in range(4):
        for w in (0, 1):
            assert np.array_equal(bits(want["hist"][k]), bits(eng.history(s, r, w))), f"{what}: history {r}/{w}"
            k += 1


def assert_frames(want, eng, what, bins=True, sequence=None):
    """sequence: the stream of every frame; the state is compared at the last frame of each stream."""
    sequence = list(range(len(want))) if sequence is None else sequence
    for f, w in enumerate(want):
        assert_frame(w, eng, f, f"{what} frame {f}", bins, state=sequence[f] not in sequence[f + 1:], stream=sequence[f])


def wall_frame():
    rng = np.random.default_rng(11)
    return np.r_[np.c_[4 + rng.random(6000) * 0.05, rng.random(6000) * 0.6, -1.7 + rng.random(6000) * 2.0, rng.random(6000)],
                 np.c_[3 + rng.random(6000) * 4, rng.random(6000) * 0.6, -1.7 + rng.normal(0, 0.02, 6000), rng.random(6000)]].astype(np.float32)


def edge_frame():
    from test_simt_ref32 import _edge_frame
    return _edge_frame()


@pytest.fixture(scope="module")
def frames(kitti):
    import synth
    q = synth.make_frame(20260922, 2).numpy()
    q[:, 2] = np.round(q[:, 2] / 0.01) * 0.01   # centimetre-quantised z: ties in every bin
    return list(kitti) + [synth.make_frame(20260922, f).numpy() for f in range(2)] + [q, wall_frame(), edge_frame()]


def test_batch_small_calls_and_the_graph_replay(frames):
    want = oracle_runs(frames)
    eng = _engine(num_streams=len(frames))
    eng.estimate_host(frames)
    assert_frames(want, eng, "batch")
    for f, a in enumerate(frames):   # one frame per call: the small-call kernels and their graph, replayed on the second call
        e = _engine()
        for rep in range(2):
            if rep:
                e.reset()
            e.estimate_host([a])
            assert_frame(want[f], e, 0, f"small call {f} rep {rep}")
    e = _engine(num_streams=4)
    e.estimate_host(frames[:4])
    assert_frames(want[:4], e, "4-frame call")


def test_fixture_sequence_and_parameter_sets(kitti):
    want = oracle_runs(list(kitti), sequence=[0] * 6)
    e = _engine()
    for f, a in enumerate(kitti):
        e.estimate_host([a])
        assert_frame(want[f], e, 0, f"sequence {f}")
    names = ["default", "ros", "no_rvpf_tgr"]
    mk = {n: (PARAM_SETS[n][0] if n != "default" else (lambda: None)) for n in names}
    sets = [mk[n]() for n in names]
    from pwpp_ctypes import default_params
    sets = [s if s is not None else default_params() for s in sets]
    fr = [np.ascontiguousarray(kitti[k][:, :3]) for k in range(6)]   # N x 3: every set reads xyz (the ROS set's input)
    stream_set = [0, 1, 2, 0, 1, 2]
    want = oracle_runs(fr, params=lambda s: sets[stream_set[s]])
    e = _engine(sets, num_streams=6, stream_set=stream_set)
    e.estimate_host(fr)
    assert_frames(want, e, "3 sets")


def test_bench_batch_and_dense_frame():
    """The first 64 frames of bench.py's synthetic batch and the dense frame: against the oracle in reference order and, under
    PWPP_ORDER_REFERENCE_EXACT, against the unmodified reference libpwref.so itself, every output bit for bit (0 label mismatches)."""
    import synth
    fr = [synth.make_frame(20260922, f).numpy() for f in range(64)]
    dense = synth.make_frame(20260922, 1, "dense1m").numpy()
    eng = _engine(num_streams=64)
    eng.estimate_host(fr)
    assert_frames(oracle_runs(fr), eng, "bench batch")
    e = _engine()
    e.estimate_host([dense])
    assert_frame(oracle_runs([dense])[0], e, 0, "dense")
    if O.have_reference_build():
        eng = _engine(num_streams=64, order=2)
        eng.estimate_host(fr)
        assert_frames(oracle_runs(fr, reference=True), eng, "bench batch vs libpwref.so")
        e = _engine(order=2)
        e.estimate_host([dense])
        assert_frame(oracle_runs([dense], reference=True)[0], e, 0, "dense vs libpwref.so")


@needs_reference
def test_exact_order_on_tie_heavy_scans_matches_the_unmodified_reference(frames, kitti):
    """PWPP_ORDER_REFERENCE_EXACT on centimetre-quantised z: the fits take equal z in std::sort's order, so every output equals
    libpwref.so's, through the batch path, one-frame calls and one stream over the six scans."""
    q = [quantised(a) for a in frames]
    want = oracle_runs(q, reference=True)
    eng = _engine(num_streams=len(q), order=2)
    eng.estimate_host(q)
    assert_frames(want, eng, "exact batch")
    for f, a in enumerate(q):
        e = _engine(order=2)
        e.estimate_host([a])
        assert_frame(want[f], e, 0, f"exact small call {f}")
    seq = [quantised(a) for a in kitti]
    want = oracle_runs(seq, sequence=[0] * 6, reference=True)
    e = _engine(order=2)
    for f, a in enumerate(seq):
        e.estimate_host([a])
        assert_frame(want[f], e, 0, f"exact sequence {f}")


def test_device_records_and_stream_table_paths(kitti):
    import torch
    fr = list(kitti)
    want = oracle_runs(fr)
    dev = _engine(num_streams=6)
    pts = torch.from_numpy(np.ascontiguousarray(np.concatenate(fr))).cuda()
    off = np.r_[0, np.cumsum([len(a) for a in fr])]
    dev.estimate_device(pts.data_ptr(), off)
    dev.synchronize()
    assert_frames(want, dev, "device")
    dt = LAYOUTS["velodyne22"]
    recs = [records(a, dt, seed=k)[0] for k, a in enumerate(fr)]
    eqs = [records(a, dt, seed=k)[1] for k, a in enumerate(fr)]
    host = _engine(num_streams=6)
    host.estimate_host_records(recs)
    assert_frames(oracle_runs(eqs), host, "host records")
    seq = [0, 1, 0, 2, 1, 0]
    want = oracle_runs(fr, sequence=seq)
    e = _engine(num_streams=3)
    e.estimate_host(fr, streams=seq)
    assert_frames(want, e, "direct call with repeated streams", sequence=seq)
    # a bound call over a device stream table (pwpp_bind_stream_table) with repeated streams, run twice: the streams carry on
    want = oracle_runs(fr + fr, sequence=seq + seq)
    b = _engine(num_streams=3)
    b.bind_call_packed(pts, torch.tensor(off, dtype=torch.int64).cuda(), [len(a) + 16 for a in fr], streams=seq)
    table = torch.tensor(seq, dtype=torch.int32).cuda()
    b.bind_stream_table(table)
    for rep in range(2):
        b.run_bound_call()
        torch.cuda.synchronize()
        b.bound_call_results()
        assert_frames(want[6 * rep:6 * rep + 6], b, f"stream table run {rep}", sequence=seq)
    b.unbind_call()


def test_bound_call_in_a_graph_and_the_rules(frames):
    import torch
    fr = frames[:6]
    pts = torch.from_numpy(np.ascontiguousarray(np.concatenate(fr))).cuda()
    off = torch.tensor(np.r_[0, np.cumsum([len(a) for a in fr])], dtype=torch.int64).cuda()
    eng = _engine(num_streams=len(fr))
    eng.bind_call_packed(pts, off, [len(a) + 16 for a in fr])
    import pwpp_b200
    with pytest.raises(pwpp_b200.PwppError):
        eng.set_arithmetic(0)   # frozen while bound
    assert eng.arithmetic() == REF
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    orcs = [O.Oracle(arith=O.ARITH_REF32) for _ in fr]
    for rep in range(2):
        g.replay()
        torch.cuda.synchronize()
        eng.bound_call_results()
        for f, a in enumerate(fr):
            orcs[f].estimate(a)
            assert np.array_equal(orcs[f].getGroundIndices(), eng.ground_indices(f)), f"replay {rep} frame {f}"
            assert np.array_equal(orcs[f].getNongroundIndices(), eng.nonground_indices(f)), f"replay {rep} frame {f}"
            assert np.array_equal(bits(orcs[f].getNormals()), bits(eng.normals(f))), f"replay {rep} frame {f}"
            assert orcs[f].getHeight() == eng.height(f)
    eng.unbind_call()
    # a clone keeps the mode
    src = _engine()
    src.estimate_host([fr[0]])
    c = src.clone()
    assert c.arithmetic() == REF
    want = oracle_runs([fr[0], fr[1]], sequence=[0, 0])
    c.estimate_host([fr[1]])
    assert_frame(want[1], c, 0, "clone")


def test_blobs_move_between_modes_and_switching_back(kitti):
    fr = list(kitti)
    want = oracle_runs(fr, sequence=[0] * 6)

    def same(x, y, what):
        assert np.array_equal(x.ground_indices(0), y.ground_indices(0)) and np.array_equal(x.nonground_indices(0), y.nonground_indices(0)), what
        assert np.array_equal(bits(x.normals(0)), bits(y.normals(0))) and np.array_equal(bits(x.centers(0)), bits(y.centers(0))), what
        assert x.export_state(0) == y.export_state(0), f"{what}: state"
    # a reference-mode state continues in double mode: in a double-mode context that imported its blob, and in its own
    # context switched to double
    a = _engine()
    for f in range(3):
        a.estimate_host([fr[f]])
        assert_frame(want[f], a, 0, f"reference mode frame {f}")
    c = _engine(arith=0)
    c.import_state(0, a.export_state(0))
    a.set_arithmetic(0)
    for f in range(3, 6):
        a.estimate_host([fr[f]]); c.estimate_host([fr[f]])
        same(a, c, f"reference-mode blob, double frame {f}")
    # a double-mode state continues in reference mode the same two ways
    d = _engine(arith=0)
    for f in range(3):
        d.estimate_host([fr[f]])
    r = _engine()
    r.import_state(0, d.export_state(0))
    d.set_arithmetic(REF)
    for f in range(3, 6):
        d.estimate_host([fr[f]]); r.estimate_host([fr[f]])
        same(d, r, f"double-mode blob, reference frame {f}")
    # a reference-mode blob imported into a context created in double mode and switched gives the oracle's sequence
    a2 = _engine()
    for f in range(3):
        a2.estimate_host([fr[f]])
    b = _engine(arith=0)
    b.import_state(0, a2.export_state(0))
    b.set_arithmetic(REF)
    for f in range(3, 6):
        b.estimate_host([fr[f]])
        assert_frame(want[f], b, 0, f"blob from reference mode, frame {f}")
    # switching back gives the results of a context that never left double, launch for launch
    never = _engine(num_streams=6, arith=0)
    never.estimate_host(fr)
    sw = _engine(num_streams=6)
    sw.estimate_host(fr)
    sw.set_arithmetic(0)
    sw.reset()
    l0 = sw.launch_count()
    sw.estimate_host(fr)
    n0 = never.launch_count()
    never.reset()
    never.estimate_host(fr)
    assert sw.launch_count() - l0 == never.launch_count() - n0
    for f in range(6):
        assert np.array_equal(never.ground_indices(f), sw.ground_indices(f)) and np.array_equal(never.nonground_indices(f), sw.nonground_indices(f))
        assert np.array_equal(bits(never.normals(f)), bits(sw.normals(f))) and never.export_state(f) == sw.export_state(f)
