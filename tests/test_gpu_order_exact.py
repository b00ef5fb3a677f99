"""PWPP_ORDER_REFERENCE_EXACT on the H100: the ground / non-ground index LISTS equal those of the unmodified reference build
(oracle/_ref/libpwref.so, whose std::sort is libstdc++'s) element for element, through every path that runs the fix-up — the
batch path, the small-call path (<= 4 frames), a stream table with repeated streams, three parameter sets, both records entry
points and a bound call replayed in a CUDA graph — and every output built on the lists follows them row for row. A frame whose
label SETS differ from the reference's (an fp32-vs-double flip, DESIGN.md section 3) cannot have equal lists and is skipped;
all but two frames of every group must be compared."""
import numpy as np
import pytest

import oracle_py as O
from helpers import CheckedReference
from param_sets import PARAM_SETS
from test_gpu_records import LAYOUTS, records

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not O.have_reference_build(), reason="needs the reference build (oracle/_ref/libpwref.so)")]
EXACT = 2


def _engine(params=None, num_streams=1, order=EXACT):
    import pwpp_b200
    e = pwpp_b200.Engine(params, device=0, num_streams=num_streams)
    e.set_output_order(order)
    return e


def wall_frame():
    rng = np.random.default_rng(11)
    return np.r_[np.c_[4 + rng.random(6000) * 0.05, rng.random(6000) * 0.6, -1.7 + rng.random(6000) * 2.0, rng.random(6000)],
                 np.c_[3 + rng.random(6000) * 4, rng.random(6000) * 0.6, -1.7 + rng.normal(0, 0.02, 6000), rng.random(6000)]].astype(np.float32)


@pytest.fixture(scope="module")
def frames(kitti):
    import synth
    q = synth.make_frame(20260922, 2).numpy()
    q[:, 2] = np.round(q[:, 2] / 0.01) * 0.01   # centimetre-quantised z: thousands of ties per bin
    return list(kitti) + [synth.make_frame(20260922, f).numpy() for f in range(2)] + [q, wall_frame()]


def reference_lists(frames, params=None, sequence=None):
    """The unmodified reference's lists of every frame; sequence: the stream of every frame (frames of one stream in order)."""
    sequence = list(range(len(frames))) if sequence is None else sequence
    refs, out = {}, []
    for a, s in zip(frames, sequence):
        if s not in refs:
            refs[s] = CheckedReference(params, stable_sort=False)
        refs[s].estimate(a)
        out.append((refs[s].getGroundIndices(), refs[s].getNongroundIndices()))
    return out


def check_lists(want, got, what, min_compared=None):
    compared = 0
    for f, ((g_r, n_r), (g_e, n_e)) in enumerate(zip(want, got)):
        if not (np.array_equal(np.sort(g_r), np.sort(g_e)) and np.array_equal(np.sort(n_r), np.sort(n_e))):
            continue
        assert np.array_equal(g_r, g_e), f"{what} frame {f}: ground list differs (first at {np.nonzero(g_r != g_e)[0][:3]})"
        assert np.array_equal(n_r, n_e), f"{what} frame {f}: non-ground list differs"
        compared += 1
    need = len(want) - 2 if min_compared is None else min_compared
    assert compared >= need, f"{what}: only {compared} of {len(want)} frames compared"


def engine_lists(eng, nf):
    return [(eng.ground_indices(f), eng.nonground_indices(f)) for f in range(nf)]


def test_batch_and_small_call_paths(frames):
    import synth
    dense = synth.make_frame(20260922, 1, "dense1m").numpy()
    want = reference_lists(frames)
    eng = _engine(num_streams=len(frames))
    eng.estimate_host(frames)
    check_lists(want, engine_lists(eng, len(frames)), "batch")
    for f, a in enumerate(frames):   # one frame per call: the small-call kernels, the reference's own pattern
        e = _engine()
        e.estimate_host([a])
        check_lists([want[f]], engine_lists(e, 1), f"small call {f}")
    e = _engine(num_streams=4)
    e.estimate_host(frames[:4])
    check_lists(want[:4], engine_lists(e, 4), "4-frame call")
    e = _engine()
    e.estimate_host([dense])
    check_lists(reference_lists([dense]), engine_lists(e, 1), "dense frame")
    counts = eng.order_exact_counts()
    assert counts[0] > 0, counts


def test_stream_table_with_repeated_streams(kitti):
    seq = [0, 1, 0, 2, 1, 0]
    fr = [kitti[k] for k in range(6)]
    want = reference_lists(fr, sequence=seq)
    eng = _engine(num_streams=3)
    eng.estimate_host(fr, streams=seq)
    check_lists(want, engine_lists(eng, len(fr)), "repeated streams")


@pytest.mark.parametrize("pname", ["ros", "no_rvpf_tgr", "default"])
def test_parameter_sets(kitti, pname):
    if pname == "default":
        mk, cols = (lambda: None), 4
    else:
        mk, cols = PARAM_SETS[pname]
    fr = [np.ascontiguousarray(a[:, :cols]) for a in kitti]
    want = reference_lists(fr, mk())
    eng = _engine(mk(), num_streams=len(fr))
    eng.estimate_host(fr)
    # the ROS launch-file parameters leave patches of a few points whose planes are numerically undefined in fp32 and in double
    # alike (test_gpu_reference.py): their labels differ from the reference's in all fixtures but one
    check_lists(want, engine_lists(eng, len(fr)), pname, min_compared=1 if pname == "ros" else None)


def test_records_entry_points_and_outputs_follow_the_lists(kitti):
    import torch
    dt = LAYOUTS["velodyne22"]
    recs = [records(a, dt, seed=k)[0] for k, a in enumerate(kitti)]
    eqs = [records(a, dt, seed=k)[1] for k, a in enumerate(kitti)]
    want = reference_lists(eqs)
    host = _engine(num_streams=6)
    host.estimate_host_records(recs)
    check_lists(want, engine_lists(host, 6), "host records")
    dev = _engine(num_streams=6)
    bufs = [torch.from_numpy(r.view(np.uint8).copy()).cuda() for r in recs]
    from pwpp_b200 import layout_from_dtype
    dev.estimate_device_records([b.data_ptr() for b in bufs], [len(r) for r in recs], [layout_from_dtype(dt)] * 6, dtypes=[dt] * 6)
    dev.synchronize()
    check_lists(want, engine_lists(dev, 6), "device records")
    for f in range(6):   # records and xyz rows in list order
        g, n = host.ground_indices(f), host.nonground_indices(f)
        assert host.ground_records(f).tobytes() == recs[f][g].tobytes(), f"frame {f}: ground records"
        assert host.nonground_records(f).tobytes() == recs[f][n].tobytes(), f"frame {f}: non-ground records"
        assert np.array_equal(host.ground_xyz(f), eqs[f][g, :3]) and np.array_equal(host.nonground_xyz(f), eqs[f][n, :3]), f"frame {f}: xyz"


def test_bound_call_in_a_graph_equals_the_direct_call(frames):
    import torch
    fr = frames[:6]
    direct = _engine(num_streams=len(fr))   # a replay advances every stream like one direct call
    pts = torch.from_numpy(np.ascontiguousarray(np.concatenate(fr))).cuda()
    off = torch.tensor(np.r_[0, np.cumsum([len(a) for a in fr])], dtype=torch.int64).cuda()
    eng = _engine(num_streams=len(fr))
    eng.bind_call_packed(pts, off, [len(a) + 16 for a in fr])
    eng.bind_packed_xyz()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            eng.run_bound_call(torch.cuda.current_stream().cuda_stream)
    for rep in range(2):
        direct.estimate_host(fr)
        want = engine_lists(direct, len(fr))
        g.replay()
        torch.cuda.synchronize()
        eng.bound_call_results()
        got = engine_lists(eng, len(fr))
        for f, ((g_d, n_d), (g_b, n_b)) in enumerate(zip(want, got)):
            assert np.array_equal(g_d, g_b) and np.array_equal(n_d, n_b), f"replay {rep} frame {f}: lists"
        px = eng.bound_packed_xyz()
        go, no = px["ground_offsets"].cpu().numpy(), px["nonground_offsets"].cpu().numpy()
        gx, nx = px["ground"].cpu().numpy(), px["nonground"].cpu().numpy()
        for f, a in enumerate(fr):
            assert np.array_equal(gx[go[f]:go[f + 1]], a[want[f][0], :3]), f"replay {rep} frame {f}: packed ground xyz"
            assert np.array_equal(nx[no[f]:no[f + 1]], a[want[f][1], :3]), f"replay {rep} frame {f}: packed non-ground xyz"
    eng.unbind_call()


def test_switching_back_gives_the_reference_order_unchanged(frames):
    fr = frames[:4]
    plain = _engine(num_streams=4, order=1)
    plain.estimate_host(fr)
    eng = _engine(num_streams=4)
    eng.estimate_host(fr)
    exact = engine_lists(eng, 4)
    eng.set_output_order(1)
    eng.reset()
    eng.estimate_host(fr)
    differ = 0
    for f, (g_x, _) in enumerate(exact):
        assert np.array_equal(eng.ground_indices(f), plain.ground_indices(f)) and np.array_equal(eng.nonground_indices(f), plain.nonground_indices(f))
        differ += not np.array_equal(g_x, plain.ground_indices(f))
    assert differ > 0   # the fixtures hold ties inside one part
