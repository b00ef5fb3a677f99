"""The record unpack kernel (csrc/pwpp_records.cuh) on the GPU, value by value, and at its tile and launch-range edges on both
the CPU and the GPU.

tests/test_simt_records.py checks k_unpack_records bit for bit against numpy through the SIMT stand-in, where every conversion
is a host cast. TestDevice runs the same test functions on the H100: its `lib` fixture serves their simt_unpack_records calls
with the kernel as compiled for sm_90a (tests/gpu_records_probe.cu, built by patchwork-plusplus_b200/build.py), so the
device's __int2float_rn / __uint2float_rn / __double2float_rn / __hiloint2double, the non-allocating 16-byte load and the
FLOAT64 NaN branch of rec_f64 are what numpy is compared with. Each frame is copied to the device at the same distance from a
16-byte boundary as its host array, with 64 bytes of slack on both sides, and dst carries PAD sentinel rows after the call's
points that must stay untouched.

The cases below test_simt_records.py's run on both backends (the SIMT one through tests/simt/simt_records_range.cpp): frames
of k * tile - 1, k * tile and k * tile + 1 records for every step, and launches over a frame range [f0, f1) of a call, as the
host chunk path issues them, into a sentinel-filled dst: every word outside the range's frames must keep its sentinel."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import test_simt_records as R
from pwpp_ctypes import PwppPointLayout

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
SIMT_LIB = os.path.join(HERE, "_build", "libpwpp_simt_records_range.so")
PROBE = os.path.join(REPO, "patchwork-plusplus_b200", "lib", "libpwpp_records_probe.so")
SENTINEL = 0x7FBADBAD   # dst words before a launch: a signalling NaN, which no conversion of the kernel produces
PAD = 40                # float4 rows of dst after the call's points
ARGS = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]


@pytest.fixture(scope="module")
def probe():
    assert os.path.exists(PROBE), "lib/libpwpp_records_probe.so was not built (patchwork-plusplus_b200/build.py)"
    L = C.CDLL(PROBE)
    L.probe_unpack_records.argtypes = ARGS
    L.probe_unpack_records.restype = C.c_int
    return L


@pytest.fixture(scope="module")
def simt_range():
    """Same compile line as test_simt_records.py's library."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_records_range.cpp", "simt_records.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(SIMT_LIB) or any(os.path.getmtime(d) > os.path.getmtime(SIMT_LIB) for d in deps):
        os.makedirs(os.path.dirname(SIMT_LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", SIMT_LIB, os.path.join(HERE, "simt", "simt_records_range.cpp")])
    L = C.CDLL(SIMT_LIB)
    L.simt_unpack_records_range.argtypes = ARGS
    L.simt_unpack_records_range.restype = C.c_int
    return L


def device_launch(probe, nf, ptrs, ns, lays, dst, f0, f1):
    """probe_unpack_records on device copies of the host frames at ptrs (n[f] * point_step bytes each) and of dst (rows of
    float4, updated in place). Returns the status."""
    import torch
    keep, d_ptrs = [], []
    for f in range(nf):
        nbytes = max(0, ns[f] * lays[f].point_step) if ptrs[f] else 0
        mis = ptrs[f] % 16 if nbytes else 0
        t = torch.zeros(64 + mis + nbytes + 64, dtype=torch.uint8, device="cuda")   # (base: 512-byte aligned)
        if nbytes:
            t[64 + mis:64 + mis + nbytes] = torch.frombuffer(bytearray(C.string_at(ptrs[f], nbytes)), dtype=torch.uint8)
        keep.append(t)
        d_ptrs.append(t.data_ptr() + 64 + mis if ptrs[f] else None)
    d_dst = torch.from_numpy(dst.view(np.int32)).cuda()
    torch.cuda.synchronize()
    rc = probe.probe_unpack_records(nf, (C.c_void_p * nf)(*d_ptrs), ns, lays, d_dst.data_ptr(), f0, f1)   # (synchronous)
    dst[:] = d_dst.cpu().numpy().view(np.uint32)
    return rc


class DeviceLib:
    """simt_unpack_records (tests/simt/simt_records.cpp) served by the GPU: the same arguments, host frames and host dst, one
    probe launch over the whole call into a device dst with PAD sentinel rows after the call's points."""

    def __init__(self, probe):
        self.probe = probe

    def simt_unpack_records(self, nf, ptr, ns, lays, out):
        total = sum(max(0, ns[f]) for f in range(nf))
        rows = max(total, 1)
        dst = np.full((rows + PAD, 4), SENTINEL, np.uint32)
        C.memmove(dst.ctypes.data, out, rows * 16)
        rc = device_launch(self.probe, nf, [ptr[f] or 0 for f in range(nf)], ns, lays, dst, 0, nf)
        assert (dst[rows:] == SENTINEL).all(), "a word after the call's points was written"
        C.memmove(out, dst.ctypes.data, rows * 16)
        return rc


@pytest.mark.gpu
class TestDevice:
    """test_simt_records.py's value cases on the H100 (not its guard-page placements, which only the CPU can arrange, nor the
    host-only layout checks)."""

    @pytest.fixture
    def lib(self, probe):
        return DeviceLib(probe)

    test_every_intensity_datatype = staticmethod(R.test_every_intensity_datatype)
    test_xyz_datatypes_with_non_finite_values_and_signed_zeros = staticmethod(R.test_xyz_datatypes_with_non_finite_values_and_signed_zeros)
    test_record_steps_over_several_tiles = staticmethod(R.test_record_steps_over_several_tiles)
    test_every_source_alignment = staticmethod(R.test_every_source_alignment)
    test_small_and_empty_frames_in_a_mixed_layout_call = staticmethod(R.test_small_and_empty_frames_in_a_mixed_layout_call)


@pytest.fixture(params=["simt", pytest.param("device", marks=pytest.mark.gpu)])
def unpack_range(request):
    """unpack_range(frames, layouts, f0, f1) -> (status, the call's sum(n) float4 points): one launch over the frames [f0, f1),
    dst filled with SENTINEL; the PAD rows after the call's points must keep it."""
    if request.param == "simt":
        lib = request.getfixturevalue("simt_range")
        launch = lambda nf, ptrs, ns, lays, dst, f0, f1: lib.simt_unpack_records_range(nf, (C.c_void_p * nf)(*ptrs), ns, lays, dst.ctypes.data, f0, f1)  # noqa: E731
    else:
        probe = request.getfixturevalue("probe")
        launch = lambda nf, ptrs, ns, lays, dst, f0, f1: device_launch(probe, nf, ptrs, ns, lays, dst, f0, f1)  # noqa: E731

    def run(frames, layouts, f0, f1):
        nf = len(frames)
        n = [len(r) // lay.point_step for r, lay in zip(frames, layouts)]
        dst = np.full((sum(n) + PAD, 4), SENTINEL, np.uint32)
        rc = launch(nf, [r.ctypes.data for r in frames], (C.c_int64 * nf)(*n), (PwppPointLayout * nf)(*layouts), dst, f0, f1)
        assert (dst[sum(n):] == SENTINEL).all(), "a word after the call's points was written"
        return rc, dst[:sum(n)].view(np.float32)
    return run


def tile_pts(step):
    """Records per CTA of k_unpack_records (rec_tile_pts: REC_TILE_BYTES = 16384 bytes, at most REC_MAX_TILE_PTS = 1024)."""
    return min(16384 // step, 1024)


@pytest.mark.parametrize("step", sorted(R.STEP_LAYOUTS))
def test_frames_at_tile_boundaries(unpack_range, step):
    """Frames of k * tile - 1, k * tile and k * tile + 1 records (k = 1, 2) in one call: a last tile one record short, full, or
    holding a single record, beside frames that need one tile more or less (CTAs past a shorter frame's end return early)."""
    rng = np.random.default_rng(300 + step)
    lay = R.layout(step, *R.STEP_LAYOUTS[step])
    tp = tile_pts(step)
    sizes = [k * tp + d for k in (1, 2) for d in (-1, 0, 1)]
    frames, want = [], []
    for f, n in enumerate(sizes):
        raw, w = R.make_frame(rng, n, lay)
        frames.append(R.aligned_copy(raw, (5 * f) % 16))
        want.append(w)
    rc, got = unpack_range(frames, [lay] * len(sizes), 0, len(sizes))
    assert rc == 0
    R.assert_bits(got, np.concatenate(want), f"step {step}, tile {tp}, sizes {sizes}")


def test_launch_range_writes_only_its_frames(unpack_range):
    """One launch over the frames [f0, f1) of a call, as the host path issues one per pipeline chunk (f0 > 0: the offsets into
    dst are absolute): the range's points land at their offsets, and every other word of dst keeps its sentinel."""
    rng = np.random.default_rng(11)
    sizes = [5, 1100, 0, 31, 2600, 1, 700]
    steps = [22, 13, 16, 48, 17, 1024, 12]
    frames, layouts, want = [], [], []
    for f, (n, step) in enumerate(zip(sizes, steps)):
        lay = R.layout(step, *R.STEP_LAYOUTS[step])
        raw, w = R.make_frame(rng, n, lay)
        frames.append(R.aligned_copy(raw, (7 * f + 1) % 16))
        layouts.append(lay)
        want.append(w)
    want = np.concatenate(want)
    off = np.cumsum([0] + sizes)
    for f0, f1 in [(0, 2), (1, 4), (3, 7), (2, 3), (5, 6), (6, 7), (0, 7)]:
        rc, got = unpack_range(frames, layouts, f0, f1)
        assert rc == 0
        lo, hi = off[f0], off[f1]
        R.assert_bits(got[lo:hi], want[lo:hi], f"frames [{f0}, {f1})")
        g = got.view(np.uint32)
        assert (g[:lo] == SENTINEL).all() and (g[hi:] == SENTINEL).all(), f"frames [{f0}, {f1}): a word outside the range was written"
