"""The kernels of a bound call's getter results (csrc/pwpp_getters.cuh) on the CPU and on the H100, from one case list.

k_gather_xyz_parts writes each frame's ground and non-ground lists as float32 xyz rows to the start of the frame's rows in one
buffer per part (rows laid out from the capacities) and both counts of every frame; every case fills both buffers with a
sentinel, compares the rows bit for bit with numpy's pts[idx, :3] and checks that no row past a count changed. k_bound_states
converts, after each run of a call, the state of every frame's bound stream into a pwpp_state row; the cases walk run tables
with repeated streams and skipped, reset and invalid-action frames, whose run stream table names a scratch slot with a different
state, and compare each run's rows with numpy. The "simt" backend runs the kernels through the SIMT stand-in
(tests/simt/simt_bound_getters.cpp); the "device" backend runs them as compiled for sm_90a (tests/gpu_bound_getters_probe.cu,
built by patchwork-plusplus_b200/build.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_bound_getters.so")
PROBE = os.path.join(REPO, "patchwork-plusplus_b200", "lib", "libpwpp_bound_getters_probe.so")
XYZ_ARGS = [C.c_int] + [C.c_void_p] * 5 + [C.c_int] + [C.c_void_p] * 4
STATE_ARGS = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
SENTINEL = np.float32(-7.25e33)
TILE = 1024   # points of one CTA of k_gather_xyz_parts
PATCHES = 7   # the count row between num_ground and num_dropped: the kernel must not read it
# pwpp_state (include/pwpp.h) and the engine's StreamState (csrc/pwpp_gle.cuh)
PWPP_STATE = np.dtype([("sensor_height", "<f8"), ("elevation_thr", "<f8", 4), ("flatness_thr", "<f8", 4), ("n_elevation", "<i4", 4),
                       ("n_flatness", "<i4", 4)])
STREAM_STATE = np.dtype([("sensor_height", "<f8"), ("elevation_thr", "<f8", 4), ("flatness_thr", "<f8", 4), ("n_elev", "<i4", 4),
                         ("n_flat", "<i4", 4), ("stale", "<f8", 9)])
SKIP, RESET, INVALID = 1, 2, 7


def _bind(L, prefix):
    getattr(L, prefix + "gather_xyz_parts").argtypes = XYZ_ARGS
    getattr(L, prefix + "gather_xyz_parts").restype = C.c_int
    getattr(L, prefix + "bound_states").argtypes = STATE_ARGS
    getattr(L, prefix + "bound_states").restype = C.c_int
    assert getattr(L, prefix + "stream_state_size")() == STREAM_STATE.itemsize
    return L


@pytest.fixture(scope="module")
def lib():
    """Same compile line as test_records_parts_backends.py's library."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_bound_getters.cpp", "simt_records.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_bound_getters.cpp")])
    return _bind(C.CDLL(LIB), "simt_")


@pytest.fixture(scope="module")
def probe():
    assert os.path.exists(PROBE), "lib/libpwpp_bound_getters_probe.so was not built (patchwork-plusplus_b200/build.py)"
    return _bind(C.CDLL(PROBE), "probe_")


def _ptr(a):
    return None if a is None else a.ctypes.data


# ---- the xyz gather ---------------------------------------------------------------------------------------------------------

class XyzFrame:
    """n float4 points (random bits in x, y, z, w: NaNs and infinities included), a ground list of ng and a non-ground list of nn
    distinct indices, the rest dropped."""
    def __init__(self, rng, n, ng, nn):
        assert ng + nn <= n
        self.n, self.ng, self.nn = n, ng, nn
        self.pts = rng.integers(0, 2**32, size=(n, 4), dtype=np.uint64).astype(np.uint32).view(np.float32)
        perm = rng.permutation(n).astype(np.int32)
        self.ground, self.nonground = perm[:ng], perm[ng:ng + nn]


def gather_xyz(prefix, L, frames, caps, parts):
    nf = len(frames)
    pts = np.concatenate([fr.pts for fr in frames] + [np.zeros((1, 4), np.float32)]).astype(np.float32)
    idx = np.zeros(max(sum(fr.n for fr in frames), 1), np.int32)   # the slots of dropped points hold 0: the kernel never reads them
    counts = np.zeros(3 * nf, np.int32)
    p = 0
    for f, fr in enumerate(frames):
        idx[p:p + fr.ng] = fr.ground
        idx[p + fr.ng:p + fr.ng + fr.nn] = fr.nonground
        p += fr.n
        counts[f], counts[nf + f], counts[2 * nf + f] = fr.ng, PATCHES, fr.n - fr.ng - fr.nn
    rows = int(sum(caps))
    bufs = [np.full((rows + 1, 3), SENTINEL, np.float32) if parts & bit else None for bit in (1, 2)]
    off = np.zeros(nf + 1, np.int64)
    cnt = np.full(2 * nf, -3, np.int32)
    n, cap = np.array([fr.n for fr in frames], np.int64), np.array(caps, np.int64)   # (every array is held by a name while the call runs)
    rc = getattr(L, prefix + "gather_xyz_parts")(nf, pts.ctypes.data, n.ctypes.data, cap.ctypes.data, idx.ctypes.data, counts.ctypes.data, parts,
                                                 _ptr(bufs[0]), _ptr(bufs[1]), off.ctypes.data, cnt.ctypes.data)
    assert rc == 0
    assert off.tolist() == np.cumsum([0] + list(caps)).tolist()
    assert cnt.tolist() == [c for fr in frames for c in (fr.ng, fr.nn)], "counts"
    for z, buf in enumerate(bufs):
        if buf is None:
            continue
        touched = np.zeros(len(buf), bool)
        for f, fr in enumerate(frames):
            lst = fr.nonground if z else fr.ground
            o = int(off[f])
            want = fr.pts[lst, :3]
            assert np.array_equal(buf[o:o + len(lst)].view(np.uint32), want.view(np.uint32)), f"part {z} frame {f}: rows differ"
            touched[o:o + len(lst)] = True
        assert (buf[~touched].view(np.uint32) == SENTINEL.view(np.uint32)).all(), f"part {z}: a row past a count was written"


def xyz_cases():
    """name -> build(rng) -> (frames, capacities)."""
    def sizes(rng):   # 0, 1 and tile-boundary list lengths, each list on its own
        fr, caps = [XyzFrame(rng, 0, 0, 0), XyzFrame(rng, 1, 1, 0), XyzFrame(rng, 1, 0, 1), XyzFrame(rng, 3, 1, 1)], [0, 1, 5, 3]
        for k, m in enumerate(t * TILE + d for t in (1, 2) for d in (-1, 0, 1)):
            other = (37 * k + 1) % (TILE // 2)
            ng, nn = (m, other) if k % 2 else (other, m)
            fr.append(XyzFrame(rng, ng + nn + k, ng, nn))
            caps.append(ng + nn + k + 3 * k)
        return fr, caps

    def empty_frames(rng):   # frames a skip or an out-of-range count left empty: count 0 under a large capacity
        return [XyzFrame(rng, 0, 0, 0), XyzFrame(rng, 500, 200, 250), XyzFrame(rng, 0, 0, 0), XyzFrame(rng, 0, 0, 0)], [4000, 600, 1, 9000]

    def counts_far_below(rng):   # most CTAs of the grid find no rows
        return [XyzFrame(rng, 400, 150, 200), XyzFrame(rng, 90, 30, 60), XyzFrame(rng, 33, 1, 31)], [20000, 9000, 4000]

    def many(rng):   # KITTI-sized and small frames in one launch
        fr = [XyzFrame(rng, 120000, 55000, 60000), XyzFrame(rng, 5000, 2000, 2900)] + [XyzFrame(rng, 700 + 31 * k, 300, 350) for k in range(30)]
        return fr, [f.n + 17 * k for k, f in enumerate(fr)]
    return {"sizes": sizes, "empty_frames": empty_frames, "counts_far_below": counts_far_below, "many": many}


XYZ_CASES = xyz_cases()
XYZ_RUNS = [(name, parts) for name in XYZ_CASES for parts in (1, 2, 3)]


def run_xyz(prefix, L, name, parts):
    rng = np.random.default_rng(sum(map(ord, name)))
    frames, caps = XYZ_CASES[name](rng)
    gather_xyz(prefix, L, frames, caps, parts)


# ---- the state snapshot -------------------------------------------------------------------------------------------------------

def run_tables(rng, streams, num_streams):
    """The run split of a call (split_runs, csrc/pwpp_capi.cu) and a random state array with a scratch slot per frame of the
    longest run."""
    nf = len(streams)
    runs, last = [0], {}
    for f, s in enumerate(streams):
        if last.get(s, -1) >= runs[-1]:
            runs.append(f)
        last[s] = f
    runs.append(nf)
    slots = num_streams + max(runs[r + 1] - runs[r] for r in range(len(runs) - 1))
    states = np.zeros(slots, STREAM_STATE)
    states.view(np.uint8)[:] = rng.integers(0, 256, size=states.nbytes, dtype=np.uint8)
    return runs, states


def snapshot_case(prefix, L, rng, streams, actions, num_streams):
    """Walks the runs as pwpp_run_bound_call does: before each run's snapshot the run's streams get new states (what k_gle would
    have written: a skipped frame's real stream keeps its state, its scratch slot changes); each run's rows must be its frames'
    real streams, and no other row may change."""
    nf = len(streams)
    b_stream = np.array(streams, np.int32)
    runs, states = run_tables(rng, streams, num_streams)
    raw = states.view(np.uint8).reshape(len(states), -1)
    out = np.zeros(nf, PWPP_STATE)
    out.view(np.uint8)[:] = 0xA5
    for r in range(len(runs) - 1):
        f0, f1 = runs[r], runs[r + 1]
        for f in range(f0, f1):
            scratch = num_streams + (f - f0)
            raw[scratch] = rng.integers(0, 256, STREAM_STATE.itemsize, dtype=np.uint8)   # where a skipped frame's empty update went
            if actions[f] in (0, RESET):   # the frame ran (after a reset): k_gle moved its real stream
                raw[streams[f]] = rng.integers(0, 256, STREAM_STATE.itemsize, dtype=np.uint8)
        before = out.copy()
        assert getattr(L, prefix + "bound_states")(f0, f1, b_stream.ctypes.data, states.ctypes.data, len(states), out.ctypes.data) == 0
        for f in range(nf):
            if f0 <= f < f1:
                src = states[streams[f]]   # the real stream, also for a skipped frame
                for k in ("sensor_height", "elevation_thr", "flatness_thr"):
                    assert np.array_equal(np.atleast_1d(out[f][k]).view(np.uint64), np.atleast_1d(src[k]).view(np.uint64)), (r, f, k)
                assert np.array_equal(out[f]["n_elevation"], src["n_elev"]) and np.array_equal(out[f]["n_flatness"], src["n_flat"]), (r, f)
                scratch = states[num_streams + (f - f0)]
                assert actions[f] in (0, RESET) or not np.array_equal(out[f]["flatness_thr"], scratch["flatness_thr"]), "read the scratch slot"
            else:
                assert out[f].tobytes() == before[f].tobytes(), f"run {r} wrote frame {f}'s row"


def state_cases():
    """name -> (streams, actions, num_streams)"""
    rng = np.random.default_rng(11)
    big = rng.permutation(300).tolist()
    return {
        "one_frame": ([0], [0], 1),
        "sixteen_sensors": (list(range(16)), [0, SKIP, RESET, INVALID] * 4, 16),
        "backlog": ([0, 1, 2, 3, 1, 4, 1], [0, 0, SKIP, 0, RESET, 0, SKIP], 5),
        "repeated_streams": ([2, 2, 2, 0, 0, 1], [SKIP, 0, RESET, INVALID, 0, 0], 3),
        "three_hundred": (big, rng.choice([0, 0, 0, SKIP, RESET, INVALID, -5], 300).tolist(), 300),
    }


STATE_CASES = state_cases()


def run_states(prefix, L, name):
    streams, actions, ns = STATE_CASES[name]
    snapshot_case(prefix, L, np.random.default_rng(sum(map(ord, name))), streams, actions, ns)


@pytest.mark.parametrize("name,parts", XYZ_RUNS, ids=[f"{n}-parts{p}" for n, p in XYZ_RUNS])
def test_xyz_simt(lib, name, parts):
    run_xyz("simt_", lib, name, parts)


@pytest.mark.parametrize("name", list(STATE_CASES))
def test_states_simt(lib, name):
    run_states("simt_", lib, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name,parts", XYZ_RUNS, ids=[f"{n}-parts{p}" for n, p in XYZ_RUNS])
def test_xyz_device(probe, name, parts):
    run_xyz("probe_", probe, name, parts)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(STATE_CASES))
def test_states_device(probe, name):
    run_states("probe_", probe, name)


def test_bad_arguments_launch_nothing(lib):
    buf = np.full((16, 3), SENTINEL, np.float32)
    cnt = np.full(2, -3, np.int32)
    pts = np.zeros((10, 4), np.float32)
    for n, cap, nd, parts in ((10, 9, 0, 3), (10, 10, 11, 3), (10, 10, -1, 3), (-1, 10, 0, 3), (10, 10, 0, 0), (10, 10, 0, 4)):
        args = [np.array([n], np.int64), np.array([cap], np.int64), np.zeros(10, np.int32), np.array([0, 0, nd], np.int32)]
        off = np.zeros(2, np.int64)
        rc = lib.simt_gather_xyz_parts(1, pts.ctypes.data, *[a.ctypes.data for a in args], parts, buf.ctypes.data, buf.ctypes.data,
                                       off.ctypes.data, cnt.ctypes.data)
        assert rc == -1 and (buf.view(np.uint32) == SENTINEL.view(np.uint32)).all() and (cnt == -3).all()
