"""The record unpack kernel of pwpp_estimate_host_records / pwpp_estimate_device_records (csrc/pwpp_records.cuh), executed on
the CPU by the SIMT stand-in (tests/simt/simt_records.cpp): sensor records of any PointCloud2 layout in, packed float4
{x, y, z, intensity} out, compared bit for bit with numpy's astype(np.float32) of the same fields (NaN intensity for a frame
without an intensity field). Also the host-side layout checks (csrc/pwpp_host.hpp: check_record_layouts) for every error class."""
import ctypes as C
import mmap
import os
import subprocess

import numpy as np
import pytest

from pwpp_ctypes import PwppPointLayout

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_records.so")

INT8, UINT8, INT16, UINT16, INT32, UINT32, FLOAT32, FLOAT64 = range(1, 9)
DT = {INT8: np.int8, UINT8: np.uint8, INT16: np.int16, UINT16: np.uint16, INT32: np.int32, UINT32: np.uint32, FLOAT32: np.float32,
      FLOAT64: np.float64}
NAN_BITS = 0x7FC00000   # intensity of a frame without an intensity field


@pytest.fixture(scope="module")
def lib():
    """Same compile line as the twin (tests/conftest.py: build_simt)."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_records.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_records.cpp")])
    L = C.CDLL(LIB)
    L.simt_unpack_records.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.simt_unpack_records.restype = C.c_int
    L.simt_check_record_layouts.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int]
    L.simt_check_record_layouts.restype = C.c_int
    return L


def layout(step, offsets, types):
    lay = PwppPointLayout()
    lay.point_step = step
    lay.offset[:] = list(offsets) + [-1] * (4 - len(offsets))
    lay.datatype[:] = list(types) + [0] * (4 - len(types))
    return lay


def field_values(rng, code, n):
    """n values of a datatype, the type's edge cases first (extremes, values that round, non-finite values, signed zeros)."""
    t = np.dtype(DT[code])
    if t.kind in "iu":
        info = np.iinfo(t)
        v = rng.integers(info.min, info.max, n, dtype=t, endpoint=True)
        edges = [info.min, info.max, 0, 1, info.max - 1]
        if t.itemsize == 4:
            edges += [(1 << 24) + 1, (1 << 24) + 3, (1 << 30) + 65, 2147483647 - 64]   # need rounding to float
    else:
        v = (rng.standard_normal(n) * 40).astype(t)
        edges = [np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, np.finfo(t).tiny, -np.finfo(t).max]
        if t == np.float64:
            edges += [1e300, -1e-320, 3.4028235677973366e38, 1.0000000596046448, 1 + 2.0 ** -24, 5e-46]
    e = np.array(edges[:n], dtype=t) if t.kind == "f" else np.array([x for x in edges if info.min <= x <= info.max][:n], dtype=t)
    v[:len(e)] = e
    if t == np.float64 and n > 10:   # NaNs with payloads and both signs
        v.view(np.uint64)[8:10] = [0x7FF0000000000001, 0xFFFA5A5A5A5A5A5A]
    return v


def make_frame(rng, n, lay):
    """Records of the layout (filler bytes between the fields) and the float4 points numpy makes of them."""
    step = lay.point_step
    raw = rng.integers(0, 256, n * step, dtype=np.uint8)
    rec = raw.reshape(n, step)
    want = np.empty((n, 4), np.float32)
    for c in range(4):
        if c == 3 and lay.offset[3] < 0:
            want[:, 3] = np.array([NAN_BITS], np.uint32).view(np.float32)[0]
            continue
        t = np.dtype(DT[lay.datatype[c]]).newbyteorder("<")
        v = field_values(rng, lay.datatype[c], n).astype(t)
        rec[:, lay.offset[c]:lay.offset[c] + t.itemsize] = v.view(np.uint8).reshape(n, t.itemsize)
        with np.errstate(over="ignore", invalid="ignore"):   # (FLOAT64 beyond the float range becomes inf, as it should)
            want[:, c] = v.astype(np.float32)
    return raw, want


def aligned_copy(raw, misalign):
    """raw at an address misalign bytes past a 16-byte boundary (the array object keeps the memory alive)."""
    base = np.empty(len(raw) + 64, np.uint8)
    start = (-base.ctypes.data) % 16 + misalign
    view = base[start:start + len(raw)]
    view[:] = raw
    assert len(raw) == 0 or view.ctypes.data % 16 == misalign
    return view


def unpack(lib, frames, layouts, ptrs=None):
    nf = len(frames)
    ns = (C.c_int64 * nf)(*[len(r) // lay.point_step for r, lay in zip(frames, layouts)])
    ptr = (C.c_void_p * nf)(*(ptrs if ptrs is not None else [r.ctypes.data for r in frames]))
    lays = (PwppPointLayout * nf)(*layouts)
    out = np.full((max(sum(ns), 1), 4), -7.0, np.float32)
    rc = lib.simt_unpack_records(nf, ptr, ns, lays, out.ctypes.data)
    return rc, out[:sum(ns)]


def assert_bits(got, want, what):
    g, w = got.view(np.uint32), want.view(np.uint32)
    bad = np.argwhere(g != w)
    assert bad.size == 0, f"{what}: {len(bad)} words differ, first at {tuple(bad[0])}: got {g[tuple(bad[0])]:#010x} want {w[tuple(bad[0])]:#010x}"


@pytest.mark.parametrize("code", list(DT), ids=[np.dtype(DT[c]).name for c in DT])
def test_every_intensity_datatype(lib, code):
    """Intensity of each of the eight datatypes at an odd offset of a 32-byte record (PCL-like)."""
    rng = np.random.default_rng(code)
    lay = layout(32, [0, 4, 8, 17], [FLOAT32] * 3 + [code])
    raw, want = make_frame(rng, 700, lay)
    rc, got = unpack(lib, [raw], [lay])
    assert rc == 0
    assert_bits(got, want, f"intensity {np.dtype(DT[code]).name}")


@pytest.mark.parametrize("xyz", [FLOAT32, FLOAT64], ids=["float32", "float64"])
def test_xyz_datatypes_with_non_finite_values_and_signed_zeros(lib, xyz):
    """x / y / z as FLOAT32 or FLOAT64 at unaligned offsets, fields out of order; every value class: NaN with payloads, +-inf,
    +-0, subnormals, values that round (FLOAT64) or overflow to inf."""
    rng = np.random.default_rng(10 + xyz)
    w = np.dtype(DT[xyz]).itemsize
    lay = layout(3 * w + 7, [2 * w + 5, 1, w + 3, 0], [xyz, xyz, xyz, UINT8])
    raw, want = make_frame(rng, 300, lay)
    rc, got = unpack(lib, [raw], [lay])
    assert rc == 0
    assert np.isnan(got[:, :3]).any() and np.isinf(got[:, :3]).any() and (np.signbit(got[:, :3]) & (got[:, :3] == 0)).any()
    assert_bits(got, want, f"xyz {np.dtype(DT[xyz]).name}")


STEP_LAYOUTS = {
    12: ([0, 4, 8], [FLOAT32] * 3),                                   # x, y, z only (the reference node's record)
    13: ([0, 4, 8, 12], [FLOAT32] * 3 + [UINT8]),
    16: ([0, 4, 8, 12], [FLOAT32] * 4),
    17: ([1, 5, 9, 13], [FLOAT32] * 3 + [INT32]),
    22: ([0, 4, 8, 12], [FLOAT32] * 4),                               # x, y, z, intensity, ring u16, time f32 (Velodyne-style)
    32: ([0, 4, 8, 16], [FLOAT32] * 4),                               # PCL PointXYZI
    48: ([0, 8, 24, 41], [FLOAT64] * 3 + [UINT16]),
    1024: ([1000, 1004, 1008, 1013], [FLOAT32] * 3 + [FLOAT64]),
}


@pytest.mark.parametrize("step", sorted(STEP_LAYOUTS))
def test_record_steps_over_several_tiles(lib, step):
    """Each step with a frame spanning several tiles of the kernel (tiles are whole records: 16 KB, at most 1024 points)."""
    rng = np.random.default_rng(step)
    lay = layout(step, *STEP_LAYOUTS[step])
    n = 2600 if step < 1024 else 70
    raw, want = make_frame(rng, n, lay)
    rc, got = unpack(lib, [aligned_copy(raw, 0)], [lay])
    assert rc == 0
    assert_bits(got, want, f"step {step}")


@pytest.mark.parametrize("step", [12, 13, 16, 17, 22, 48])
def test_every_source_alignment(lib, step):
    """The frame's first byte 0 to 15 bytes past a 16-byte boundary: the vector loads of the aligned body and the byte loads of
    the head and tail meet at a different place every time."""
    rng = np.random.default_rng(100 + step)
    lay = layout(step, *STEP_LAYOUTS[step])
    raw, want = make_frame(rng, 1500, lay)
    for mis in range(16):
        rc, got = unpack(lib, [aligned_copy(raw, mis)], [lay])
        assert rc == 0
        assert_bits(got, want, f"step {step}, source at 16k + {mis}")


def test_small_and_empty_frames_in_a_mixed_layout_call(lib):
    """One launch over frames of 0, 1, 2 and 31 points and larger ones, every frame with its own layout (with and without
    intensity, every alignment): frame f's points land at its offset of the output, and only there."""
    rng = np.random.default_rng(7)
    sizes = [0, 1, 2, 31, 1100, 0, 2600, 5, 31]
    steps = [16, 22, 12, 13, 17, 32, 48, 1024, 22]
    frames, layouts, want = [], [], []
    for f, (n, step) in enumerate(zip(sizes, steps)):
        lay = layout(step, *STEP_LAYOUTS[step])
        raw, w = make_frame(rng, n, lay)
        frames.append(aligned_copy(raw, (3 * f) % 16))
        layouts.append(lay)
        want.append(w)
    rc, got = unpack(lib, frames, layouts)
    assert rc == 0
    assert_bits(got, np.concatenate(want), "mixed call")
    assert np.isnan(got[sum(sizes[:2]):sum(sizes[:3]), 3]).all()   # the 12-byte frame has no intensity


@pytest.mark.parametrize("step", [13, 16, 22, 48])
def test_no_read_outside_the_frame(lib, step):
    """Frames placed so that the page after their last byte (and, in the second placement, the page before their first byte) is
    PROT_NONE: any read outside [frames[f], frames[f] + n[f] * step) faults."""
    rng = np.random.default_rng(200 + step)
    lay = layout(step, *STEP_LAYOUTS[step])
    page = mmap.PAGESIZE
    libc = C.CDLL(None, use_errno=True)
    libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    for n in (1, 2, 31, 1500):
        raw, want = make_frame(rng, n, lay)
        data_pages = (len(raw) + page - 1) // page + 1
        m = mmap.mmap(-1, (data_pages + 2) * page)
        base = C.addressof(C.c_char.from_buffer(m))
        assert libc.mprotect(base, page, 0) == 0 and libc.mprotect(base + (data_pages + 1) * page, page, 0) == 0
        for start in (base + (data_pages + 1) * page - len(raw), base + page):   # flush against the guard after / before
            C.memmove(start, raw.ctypes.data, len(raw))
            rc, got = unpack(lib, [raw], [lay], ptrs=[start])
            assert rc == 0
            assert_bits(got, want, f"step {step}, {n} points against a guard page")
        libc.mprotect(base, (data_pages + 2) * page, mmap.PROT_READ | mmap.PROT_WRITE)


def check(lib, frames, ns, layouts):
    nf = len(layouts) if layouts is not None else len(ns)
    msg = C.create_string_buffer(512)
    ptr = (C.c_void_p * nf)(*frames) if frames is not None else None
    n = (C.c_int64 * nf)(*ns) if ns is not None else None
    lays = (PwppPointLayout * nf)(*layouts) if layouts is not None else None
    rc = lib.simt_check_record_layouts(nf, ptr, n, lays, msg, 512)
    return rc, msg.value.decode()


def test_layout_validation_for_every_error_class(lib):
    INVALID, UNSUPPORTED = -1, -4
    good = layout(22, [0, 4, 8, 12], [FLOAT32] * 4)
    buf = np.zeros(22 * 10, np.uint8)
    p = buf.ctypes.data
    assert check(lib, [p, p], [10, 0], [good, layout(12, [0, 4, 8], [FLOAT32] * 3)]) == (0, "")
    assert check(lib, [p, None], [10, 0], [good, good])[0] == 0                  # a NULL pointer of an empty frame is fine
    cases = [
        (None, [10], [good], INVALID, "NULL"),
        ([p], None, [good], INVALID, "NULL"),
        ([p], [10], None, INVALID, "NULL"),
        ([p, None], [10, 3], [good, good], INVALID, "frame 1: frame pointer is NULL"),
        ([p, p], [10, -1], [good, good], INVALID, "frame 1: n < 0"),
        ([p], [1], [layout(0, [0, 4, 8], [FLOAT32] * 3)], INVALID, "frame 0: point_step 0"),
        ([p], [1], [layout(1025, [0, 4, 8], [FLOAT32] * 3)], UNSUPPORTED, "PWPP_MAX_POINT_STEP"),
        ([p], [1], [layout(16, [0, 4, 8, 12], [FLOAT32] * 3 + [9])], INVALID, "frame 0: field intensity: unknown datatype 9"),
        ([p], [1], [layout(16, [0, 4, 8, 12], [FLOAT32] * 3 + [0])], INVALID, "field intensity: unknown datatype 0"),
        ([p], [1], [layout(16, [0, 4, 8], [FLOAT32, 0, FLOAT32])], INVALID, "field y: unknown datatype 0"),
        ([p], [1], [layout(16, [0, 4, 8], [FLOAT32, FLOAT32, INT32])], UNSUPPORTED, "field z: x, y and z must be FLOAT32 or FLOAT64"),
        ([p], [1], [layout(16, [0, 4, 8], [UINT16, FLOAT32, FLOAT32])], UNSUPPORTED, "field x:"),
        ([p], [1], [layout(16, [0, 4, 13], [FLOAT32] * 3)], INVALID, "field z: bytes [13, 17) do not fit inside point_step 16"),
        ([p], [1], [layout(16, [-1, 4, 8], [FLOAT32] * 3)], INVALID, "field x: bytes [-1, 3)"),
        ([p], [1], [layout(16, [0, 4, 8, 9], [FLOAT32] * 3 + [FLOAT64])], INVALID, "field intensity: bytes [9, 17)"),
        ([p, p], [1, 1], [good, layout(15, [0, 8, 4], [FLOAT32, FLOAT64, FLOAT32])], INVALID, "frame 1: field y: bytes [8, 16) do not fit inside point_step 15"),
    ]
    for frames, ns, layouts, status, text in cases:
        rc, msg = check(lib, frames, ns, layouts) if layouts is not None else (None, None)
        if layouts is None:
            nf = len(ns)
            rc = lib.simt_check_record_layouts(nf, (C.c_void_p * nf)(*frames), (C.c_int64 * nf)(*ns), None, C.create_string_buffer(64), 64)
            msg = "NULL"
        assert rc == status and text in msg, (text, rc, msg)
    # a failing layout launches nothing: the output is untouched
    rc, out = unpack(lib, [buf], [layout(1025, [0, 4, 8], [FLOAT32] * 3)])
    assert rc == UNSUPPORTED and (out == -7.0).all()
