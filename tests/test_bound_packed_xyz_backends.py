"""The kernels of a bound call's packed xyz results (csrc/pwpp_getters.cuh, k_bound_xyz_offsets then k_gather_xyz_packed) on the
CPU and on the H100, from one case list.

k_bound_xyz_offsets scans every frame's ground count and non-ground list length into one int64 offsets array per part;
k_gather_xyz_packed then writes each frame's lists as float32 xyz rows back to back from those offsets. Every case fills both
buffers with a sentinel and the offsets with garbage, checks the offsets against numpy's scan, the rows bit for bit against the
concatenation of pts[idx, :3] over the frames, and that no row past a total changed. The cases are those of
test_bound_getters_backends.py (list lengths of 0, 1 and tile boundaries, empty frames under large capacities, capacities far
above the counts, KITTI-sized and small frames together) plus 1025 frames, so that the offsets kernel's threads own slices of
several frames. The "simt" backend runs the kernels through the SIMT stand-in (tests/simt/simt_bound_packed.cpp); the "device"
backend runs them as compiled for sm_90a (tests/gpu_bound_packed_probe.cu, built by patchwork-plusplus_b200/build.py)."""
import ctypes as C
import os

import numpy as np
import pytest

from test_bound_getters_backends import PATCHES, SENTINEL, XYZ_CASES, XyzFrame
from test_simt_bound_packed import build_lib

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
PROBE = os.path.join(REPO, "patchwork-plusplus_b200", "lib", "libpwpp_bound_packed_probe.so")
ARGS = [C.c_int] + [C.c_void_p] * 5 + [C.c_int] + [C.c_void_p] * 4


def _bind(L, prefix):
    getattr(L, prefix + "packed_xyz").argtypes = ARGS
    getattr(L, prefix + "packed_xyz").restype = C.c_int
    return L


@pytest.fixture(scope="module")
def lib():
    return _bind(build_lib(), "simt_")


@pytest.fixture(scope="module")
def probe():
    assert os.path.exists(PROBE), "lib/libpwpp_bound_packed_probe.so was not built (patchwork-plusplus_b200/build.py)"
    return _bind(C.CDLL(PROBE), "probe_")


def _ptr(a):
    return None if a is None else a.ctypes.data


def packed_xyz(prefix, L, frames, caps, parts):
    nf = len(frames)
    pts = np.concatenate([fr.pts for fr in frames] + [np.zeros((1, 4), np.float32)]).astype(np.float32)
    idx = np.zeros(max(sum(fr.n for fr in frames), 1), np.int32)
    counts = np.zeros(3 * nf, np.int32)
    p = 0
    for f, fr in enumerate(frames):
        idx[p:p + fr.ng] = fr.ground
        idx[p + fr.ng:p + fr.ng + fr.nn] = fr.nonground
        p += fr.n
        counts[f], counts[nf + f], counts[2 * nf + f] = fr.ng, PATCHES, fr.n - fr.ng - fr.nn
    rows = int(sum(caps))
    bufs = [np.full((rows + 1, 3), SENTINEL, np.float32) if parts & bit else None for bit in (1, 2)]
    offs = [np.full(nf + 1, -5, np.int64) for _ in range(2)]
    n, cap = np.array([fr.n for fr in frames], np.int64), np.array(caps, np.int64)
    rc = getattr(L, prefix + "packed_xyz")(nf, pts.ctypes.data, n.ctypes.data, cap.ctypes.data, idx.ctypes.data, counts.ctypes.data, parts,
                                           _ptr(bufs[0]), _ptr(bufs[1]), offs[0].ctypes.data, offs[1].ctypes.data)
    assert rc == 0
    for z in range(2):
        want_off = np.concatenate([[0], np.cumsum([fr.nn if z else fr.ng for fr in frames])])
        assert offs[z].tolist() == want_off.tolist(), f"part {z}: offsets"
        buf = bufs[z]
        if buf is None:
            continue
        want = np.concatenate([fr.pts[fr.nonground if z else fr.ground, :3] for fr in frames] + [np.zeros((0, 3), np.float32)])
        total = int(want_off[-1])
        assert np.array_equal(buf[:total].view(np.uint32), want.view(np.uint32)), f"part {z}: rows differ"
        assert (buf[total:].view(np.uint32) == SENTINEL.view(np.uint32)).all(), f"part {z}: a row past the total was written"


def _many_frames(rng):
    fr = [XyzFrame(rng, k % 40, (k % 40) // 3, (k % 40) // 2) for k in range(1025)]
    return fr, [f.n + (k % 5) for k, f in enumerate(fr)]


CASES = dict(XYZ_CASES, many_frames=_many_frames)
RUNS = [(name, parts) for name in CASES for parts in (1, 2, 3)]


def run(prefix, L, name, parts):
    rng = np.random.default_rng(sum(map(ord, name)))
    frames, caps = CASES[name](rng)
    packed_xyz(prefix, L, frames, caps, parts)


@pytest.mark.parametrize("name,parts", RUNS, ids=[f"{n}-parts{p}" for n, p in RUNS])
def test_packed_xyz_simt(lib, name, parts):
    run("simt_", lib, name, parts)


@pytest.mark.gpu
@pytest.mark.parametrize("name,parts", RUNS, ids=[f"{n}-parts{p}" for n, p in RUNS])
def test_packed_xyz_device(probe, name, parts):
    run("probe_", probe, name, parts)
