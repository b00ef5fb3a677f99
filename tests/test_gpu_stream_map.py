"""The stream table of pwpp_estimate_host_streams / pwpp_estimate_device_streams on the GPU: frame f of a call advances stream
streams[f] (any subset, any order, repeats in call order). Results are indexed by call position, state by stream id."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_py as O
from helpers import assert_state_close
from test_gpu_parity import compare_frame

pytestmark = pytest.mark.gpu


def _engine(num_streams, order=0):
    import pwpp_b200
    eng = pwpp_b200.Engine(device=0, num_streams=num_streams)
    eng.set_output_order(order)
    return eng


def _outputs(eng, f):
    """Everything the call produced for call position f, as bytes."""
    parts = [eng.ground_indices(f), eng.nonground_indices(f), eng.centers(f), eng.normals(f), eng.bin_ids(f)]
    return b"|".join(np.ascontiguousarray(p).tobytes() for p in parts) + bytes(eng.bin_results(f))


def _stream(eng, s):
    """State, histories and the exported blob of stream s, as bytes."""
    parts = [bytes(eng.state(s))] + [eng.history(s, r, w).tobytes() for r in range(4) for w in (0, 1)]
    return b"|".join(parts) + eng.export_state(s)


def _run(eng, frames, streams, device):
    if not device:
        eng.estimate_host(frames, streams=streams)
        return
    import torch
    pts = torch.from_numpy(np.concatenate(frames)).cuda()
    offs = np.cumsum([0] + [len(a) for a in frames]).astype(np.int64)
    torch.cuda.synchronize()
    eng.estimate_device(pts.data_ptr(), offs, streams=streams)
    eng.synchronize()


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("nf", [2, 6], ids=["small_call", "batch"])
@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
def test_identity_table_equals_the_old_entry_points(kitti, device, nf, order):
    old, new = _engine(nf, order), _engine(nf, order)
    for c in range(2):   # the second call carries the state of the first
        frames = [kitti[(c + f) % 6] for f in range(nf)]
        _run(old, frames, None, device)
        _run(new, frames, list(range(nf)), device)
        for f in range(nf):
            assert _outputs(old, f) == _outputs(new, f), f"call {c} frame {f}"
            assert _stream(old, f) == _stream(new, f), f"call {c} stream {f}"


def test_fixed_permutation_equals_the_old_entry_point(kitti):
    """Six calls with the streams named in the order 3, 0, 4, 1, 2: the same frames reach the same streams as with the identity
    table, through the same batch kernels, so every output and every stream is bit-identical."""
    perm = [3, 0, 4, 1, 2]
    old, new = _engine(5), _engine(5)
    for c in range(6):
        frames = [kitti[(c + s) % 6] for s in range(5)]   # frames[s] belongs to stream s
        old.estimate_host(frames)
        new.estimate_host([frames[s] for s in perm], streams=perm)
        for f, s in enumerate(perm):
            assert _outputs(new, f) == _outputs(old, s), f"call {c}: position {f} (stream {s})"
        for s in range(5):
            assert _stream(new, s) == _stream(old, s), f"call {c}: stream {s}"


def test_irregular_schedule_against_one_oracle_per_stream(kitti):
    """Five streams, twelve calls: random subsets in random order, one call naming a stream three times, an empty frame, an
    N x 3 call. Every frame against the CANON64 oracle of its stream; streams a call does not name keep their blob byte for byte.
    The N x 3 call carries synthetic scans: without RNR the fixture scans leave a few planes fitted to fewer than 3 points,
    which the algorithm leaves numerically undefined (and with them, through the ring statistics of TGR, their neighbours).
    No frame of this schedule has such a plane, so every comparison is the full one."""
    import synth
    rng = np.random.default_rng(2024)
    eng = _engine(5)
    orcs = [O.Oracle(arith=O.ARITH_CANON64) for _ in range(5)]
    for c in range(12):
        if c == 3:
            streams = [2, 0, 2, 4, 2]
        else:
            streams = [int(s) for s in rng.permutation(5)[:int(rng.integers(1, 6))]]
        frames = [kitti[int(rng.integers(0, 6))] for _ in streams]
        if c == 5:
            frames[0] = np.zeros((0, 4), np.float32)
        if c == 11:
            frames = [np.ascontiguousarray(synth.make_frame(12, f).numpy()[:, :3]) for f in range(len(streams))]
        before = {s: eng.export_state(s) for s in range(5) if s not in streams}
        eng.estimate_host(frames, streams=streams)
        for f, (s, a) in enumerate(zip(streams, frames)):
            orcs[s].estimate(a)
            assert compare_frame(eng, f, orcs[s], a, f"call {c} position {f} stream {s}") == 0
        for s in set(streams):
            assert_state_close(orcs[s].state(), eng.state(s), f"call {c} stream {s}")
            for r in range(4):
                for w in (0, 1):
                    assert np.allclose(eng.history(s, r, w), orcs[s].history(r, w), rtol=1e-6, atol=1e-9), f"call {c} stream {s} history"
        for s, blob in before.items():
            assert eng.export_state(s) == blob, f"call {c}: stream {s} was not named but changed"


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
def test_repeats_in_one_call_equal_separate_calls(kitti, order):
    """K frames of one stream in one call are K runs of one frame each: the same small-call kernels as K one-frame calls."""
    frames = [kitti[1], kitti[4], kitti[2], kitti[4]]
    one = _engine(2, order)
    one.estimate_host(frames, streams=[1] * len(frames))
    sep = _engine(2, order)
    for f, a in enumerate(frames):
        sep.estimate_host([a], streams=[1])
        assert _outputs(one, f) == _outputs(sep, 0), f"frame {f}"
    assert _stream(one, 1) == _stream(sep, 1) and _stream(one, 0) == _stream(sep, 0)


def test_bad_input_changes_nothing(kitti):
    import pwpp_b200
    eng = _engine(3)
    eng.estimate_host(kitti[:3])
    blobs = [eng.export_state(s) for s in range(3)]
    a = kitti[3]
    for streams in ([3], [0, -1], [2, 0, 1, 7]):
        with pytest.raises(pwpp_b200.PwppError, match="stream id"):
            eng.estimate_host([a] * len(streams), streams=streams)
    import torch
    pts = torch.from_numpy(a).cuda()
    with pytest.raises(pwpp_b200.PwppError, match="stream id"):
        eng.estimate_device(pts.data_ptr(), [0, len(a)], streams=[5])
    lib = eng.lib
    ptrs = (C.c_void_p * 1)(a.ctypes.data)
    ns = (C.c_int64 * 1)(len(a))
    ids = (C.c_int32 * 1)(0)
    assert lib.pwpp_estimate_host_streams(eng._h, 1, None, ptrs, ns, 4, 4, 1) == -1 and b"NULL" in lib.pwpp_last_error()
    assert lib.pwpp_estimate_host_streams(eng._h, 0, ids, ptrs, ns, 4, 4, 1) == -1
    assert lib.pwpp_estimate_host_streams(eng._h, 65536, ids, ptrs, ns, 4, 4, 1) == -1
    offs = (C.c_int64 * 2)(0, len(a))
    assert lib.pwpp_estimate_device_streams(eng._h, 1, None, C.c_void_p(pts.data_ptr()), offs, 1, None) == -1
    for s in range(3):
        assert eng.export_state(s) == blobs[s], f"stream {s} changed after a refused call"
    # the results of the last good call are still there
    ref = _engine(3); ref.estimate_host(kitti[:3])
    assert _outputs(eng, 2) == _outputs(ref, 2)


def _sequence_exe():
    here = os.path.dirname(os.path.abspath(__file__))
    exe = os.path.join(os.path.dirname(here), "patchwork-plusplus_b200", "lib", "pwpp_sequence")
    if not os.path.exists(exe):
        import build as pw_build
        pw_build.build_examples()
    return exe


def _lines(args, multi):
    out = subprocess.run([_sequence_exe(), *args], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    rows = [l.split() for l in out.stdout.splitlines() if "points" in l.split()[1:3]]
    if multi:   # stream, name, points, ground, non-ground, patches, height
        return [(int(t[0]), t[1], int(t[3]), int(t[5]), int(t[7]), int(t[9]), t[11]) for t in rows]
    return [(0, t[0], int(t[2]), int(t[4]), int(t[6]), int(t[8]), t[10]) for t in rows]


def test_multi_directory_runner_matches_single_directory_runs(tmp_path, kitti):
    lengths = [3, 5, 2]
    dirs = []
    for d, m in enumerate(lengths):
        p = tmp_path / f"seq{d}"
        p.mkdir()
        for t in range(m):
            np.ascontiguousarray(kitti[(2 * d + t) % 6]).tofile(p / f"{t:06d}.bin")
        dirs.append(str(p))
    multi = _lines(dirs, True)
    assert len(multi) == sum(lengths)
    for d in range(3):
        single = _lines([dirs[d]], False)
        mine = [r[1:] for r in multi if r[0] == d]
        assert mine == [r[1:] for r in single], f"directory {d}"
    # one directory, four scans per call: the same counts; heights where the stream's state is reported (its last frame of a call)
    default = _lines([dirs[1]], False)
    batched = _lines([dirs[1], "--frames-per-call", "4"], True)
    assert [r[1:6] for r in batched] == [r[1:6] for r in default]
    assert [r[6] for r in batched] == ["-", "-", "-", default[3][6], default[4][6]]
