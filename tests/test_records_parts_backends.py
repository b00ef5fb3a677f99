"""The record gather of a bound call's record results (csrc/pwpp_records.cuh, k_gather_record_parts) on the CPU and on the H100,
from one case list, compared byte for byte with numpy's records[idx_part].

The kernel writes each frame's ground list and non-ground list as whole records to the start of the frame's region in one buffer
per part; the regions are laid out from the capacities (max_n), not the sizes, and it writes both counts of every frame. Every
case fills both buffers with a sentinel byte and checks each region's records, that no other byte changed, the region offsets and
the counts. The "simt" backend runs the kernel through the SIMT stand-in (tests/simt/simt_records_parts.cpp); the "device" backend
runs it as compiled for sm_90a (tests/gpu_records_parts_probe.cu, built by patchwork-plusplus_b200/build.py), each frame copied to
the device at the same distance from a 16-byte boundary as its host array. The guard-page placements, which show that no byte
outside a frame is read, can only be arranged on the CPU."""
import ctypes as C
import mmap
import os
import subprocess

import numpy as np
import pytest

from test_simt_records_gather import SENTINEL, Frame, tile_pts

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_records_parts.so")
PROBE = os.path.join(REPO, "patchwork-plusplus_b200", "lib", "libpwpp_records_parts_probe.so")
ARGS = [C.c_int] + [C.c_void_p] * 6 + [C.c_int] + [C.c_void_p] * 4
STEPS = [1, 2, 3, 4, 13, 16, 22, 32, 48, 1024]
PATCHES = 7   # the count row between num_ground and num_dropped: the kernel must not read it


@pytest.fixture(scope="module")
def lib():
    """Same compile line as test_simt_records_gather.py's library."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_records_parts.cpp", "simt_records.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_records_parts.cpp")])
    L = C.CDLL(LIB)
    L.simt_gather_record_parts.argtypes = ARGS
    L.simt_gather_record_parts.restype = C.c_int
    return L


@pytest.fixture(scope="module")
def probe():
    assert os.path.exists(PROBE), "lib/libpwpp_records_parts_probe.so was not built (patchwork-plusplus_b200/build.py)"
    L = C.CDLL(PROBE)
    L.probe_gather_record_parts.argtypes = ARGS
    L.probe_gather_record_parts.restype = C.c_int
    return L


def simt_launch(lib):
    def launch(nf, ptrs, n, cap, step, idx, counts, parts, ground, nonground, off, cnt):
        return lib.simt_gather_record_parts(nf, ptrs, n.ctypes.data, cap.ctypes.data, step.ctypes.data, idx.ctypes.data, counts.ctypes.data, parts,
                                            None if ground is None else ground.ctypes.data, None if nonground is None else nonground.ctypes.data,
                                            off.ctypes.data, cnt.ctypes.data)
    return launch


def device_launch(probe):
    def launch(nf, ptrs, n, cap, step, idx, counts, parts, ground, nonground, off, cnt):
        import torch
        keep, d_ptrs = [], []
        for f in range(nf):
            nbytes = int(n[f]) * int(step[f])
            mis = ptrs[f] % 16 if nbytes else 0
            t = torch.zeros(64 + mis + nbytes + 64, dtype=torch.uint8, device="cuda")   # (base: 512-byte aligned)
            if nbytes:
                t[64 + mis:64 + mis + nbytes] = torch.frombuffer(bytearray(C.string_at(ptrs[f], nbytes)), dtype=torch.uint8)
            keep.append(t)
            d_ptrs.append(t.data_ptr() + 64 + mis)
        d_bufs = [None if b is None else torch.from_numpy(b.copy()).cuda() for b in (ground, nonground)]   # (fresh allocations: 16-byte aligned)
        torch.cuda.synchronize()
        rc = probe.probe_gather_record_parts(nf, (C.c_void_p * nf)(*d_ptrs), n.ctypes.data, cap.ctypes.data, step.ctypes.data, idx.ctypes.data,
                                             counts.ctypes.data, parts, *[None if d is None else d.data_ptr() for d in d_bufs],
                                             off.ctypes.data, cnt.ctypes.data)   # (synchronous)
        for b, d in zip((ground, nonground), d_bufs):
            if b is not None:
                b[:] = d.cpu().numpy()
        return rc
    return launch


def sentinel_buffer(nbytes):
    """nbytes of SENTINEL, 16-byte aligned, 64 bytes of slack after them."""
    raw = np.full(nbytes + 64 + 16, SENTINEL, np.uint8)
    return raw[(-raw.ctypes.data) % 16:][:nbytes + 64]


def gather_parts(launch, frames, caps, parts, ptrs=None):
    """One launch over the call; checks the offsets, the counts, every region of every enabled part and that no other byte of
    either buffer was written; returns the status."""
    nf = len(frames)
    idx = np.zeros(max(sum(fr.n for fr in frames), 1), np.int32)   # the slots of dropped points hold 0: the kernel never reads them
    counts = np.zeros(3 * nf, np.int32)
    p = 0
    for f, fr in enumerate(frames):
        idx[p:p + fr.ng] = fr.ground
        idx[p + fr.ng:p + fr.ng + fr.nn] = fr.nonground
        p += fr.n
        counts[f], counts[nf + f], counts[2 * nf + f] = fr.ng, PATCHES, fr.n - fr.ng - fr.nn
    want_off = np.cumsum([0] + [(c * fr.step + 15) // 16 * 16 for fr, c in zip(frames, caps)])
    bufs = [sentinel_buffer(int(want_off[-1])) if parts & bit else None for bit in (1, 2)]
    off = np.zeros(nf + 1, np.int64)
    cnt = np.full(2 * nf, -3, np.int32)
    rc = launch(nf, (C.c_void_p * nf)(*(ptrs if ptrs is not None else [fr.raw.ctypes.data for fr in frames])),
                np.array([fr.n for fr in frames], np.int64), np.array(caps, np.int64), np.array([fr.step for fr in frames], np.int32), idx, counts,
                parts, bufs[0], bufs[1], off, cnt)
    if rc != 0:
        return rc
    assert (off == want_off).all(), (off, want_off)
    assert cnt.tolist() == [c for fr in frames for c in (fr.ng, fr.nn)], "counts"
    for z, buf in enumerate(bufs):
        if buf is None:
            continue
        touched = np.zeros(len(buf), bool)
        for f, fr in enumerate(frames):
            lst = fr.nonground if z else fr.ground
            o, m = int(off[f]), len(lst) * fr.step
            assert np.array_equal(buf[o:o + m], fr.want(lst)), f"part {z} frame {f} (step {fr.step}, {fr.n} records): records differ"
            touched[o:o + m] = True
        assert (buf[~touched] == SENTINEL).all(), f"part {z}: a byte outside the records was written, first at {np.argmax((buf != SENTINEL) & ~touched)}"
    return 0


# ---- the cases (both backends): build(rng) -> (frames, capacities) ---------------------------------------------------------------

def case_steps(step):
    """One frame of about 2.5 tiles with dropped points (capacity a tile more), one with none (capacity = size)."""
    def build(rng):
        tp = tile_pts(step)
        n = 5 * tp // 2 + 3
        return [Frame(rng, n, step, n // 3, n - n // 3 - 7, mis=3), Frame(rng, n, step, n // 2, n - n // 2, mis=12)], [n + tp, n]
    return build


def case_alignments(step):
    """Sixteen frames, frame k starting k bytes past a 16-byte boundary; capacities vary, so region alignments vary too."""
    def build(rng):
        fr = [Frame(rng, 300 + 7 * k, step, 100 + k, 180, mis=k) for k in range(16)]
        return fr, [f.n + 5 * k for k, f in enumerate(fr)]
    return build


def case_tile_boundaries(step):
    """Ground and non-ground lengths at k * tile - 1, k * tile and k * tile + 1 (k = 1, 2), each list on its own."""
    def build(rng):
        tp = tile_pts(step)
        out, caps = [], []
        for f, m in enumerate(k * tp + d for k in (1, 2) for d in (-1, 0, 1)):
            other = (7 * f + 1) % (tp // 2 + 1)
            ng, nn = (m, other) if f % 2 else (other, m)
            drop = 0 if f % 3 else 2 + f
            out.append(Frame(rng, ng + nn + drop, step, ng, nn, mis=(5 * f) % 16))
            caps.append(ng + nn + drop + f)
        return out, caps
    return build


def case_empty_and_one_sided():
    """Empty frames (capacity 0 and capacity 700), all points dropped, ng = 0, nn = 0, single records."""
    def build(rng):
        fr = [Frame(rng, 0, 22, 0, 0), Frame(rng, 0, 16, 0, 0), Frame(rng, 40, 22, 0, 0, mis=3), Frame(rng, 1500, 22, 1500, 0, mis=1),
              Frame(rng, 1500, 22, 0, 1500, mis=7), Frame(rng, 1, 13, 1, 0, mis=15), Frame(rng, 1, 13, 0, 1, mis=2),
              Frame(rng, 2, 1024, 0, 1, mis=9)]
        return fr, [0, 700, 40, 1600, 1500, 1, 90, 3]
    return build


def case_counts_far_below_capacities():
    """Sizes of 1/20 of the capacities or less: most CTAs of the grid have no records."""
    def build(rng):
        fr = [Frame(rng, 400, 16, 150, 200, mis=1), Frame(rng, 90, 22, 30, 60, mis=6), Frame(rng, 0, 32, 0, 0), Frame(rng, 33, 48, 1, 31, mis=11)]
        return fr, [20000, 9000, 5000, 4000]
    return build


def case_mixed_layouts():
    """Every step of STEPS plus 5, 7, 12 and 17 in one launch."""
    def build(rng):
        steps = STEPS + [5, 7, 12, 17]
        fr = [Frame(rng, 900 + 37 * f, s, 300 + f, 500, mis=(3 * f + 1) % 16) for f, s in enumerate(steps)]
        return fr, [f.n + 100 * k for k, f in enumerate(fr)]
    return build


CASES = {**{f"steps_{s}": case_steps(s) for s in STEPS},
         **{f"alignments_{s}": case_alignments(s) for s in (13, 16, 22, 48)},
         **{f"tile_boundaries_{s}": case_tile_boundaries(s) for s in (1, 3, 13, 16, 22, 48, 1024)},
         "empty_and_one_sided": case_empty_and_one_sided(), "counts_far_below_capacities": case_counts_far_below_capacities(),
         "mixed_layouts": case_mixed_layouts()}
# every case with both parts; the parts alone on the cases that hold every kind of list
RUNS = [(name, 3) for name in CASES] + [(name, parts) for name in ("empty_and_one_sided", "mixed_layouts", "steps_22") for parts in (1, 2)]


def run_case(launch, name, parts):
    rng = np.random.default_rng(sum(map(ord, name)))
    frames, caps = CASES[name](rng)
    assert gather_parts(launch, frames, caps, parts) == 0


@pytest.mark.parametrize("name,parts", RUNS, ids=[f"{n}-parts{p}" for n, p in RUNS])
class TestSimt:
    def test_case(self, lib, name, parts):
        run_case(simt_launch(lib), name, parts)


@pytest.mark.gpu
@pytest.mark.parametrize("name,parts", RUNS, ids=[f"{n}-parts{p}" for n, p in RUNS])
class TestDevice:
    def test_case(self, probe, name, parts):
        run_case(device_launch(probe), name, parts)


def test_bad_arguments_launch_nothing(lib):
    rng = np.random.default_rng(1)
    fr = Frame(rng, 10, 16, 5, 5)
    for step, nd, cap, parts in ((0, 0, 10, 3), (1025, 0, 10, 3), (16, 11, 10, 3), (16, -1, 10, 3), (16, 0, 9, 3), (16, 0, 10, 0), (16, 0, 10, 4)):
        buf = np.full(256, SENTINEL, np.uint8)
        cnt = np.full(2, -3, np.int32)
        args = [np.array([10], np.int64), np.array([cap], np.int64), np.array([step], np.int32), np.zeros(10, np.int32), np.array([0, 0, nd], np.int32)]
        off = np.zeros(2, np.int64)   # (every array is held by a name while the call runs)
        rc = lib.simt_gather_record_parts(1, (C.c_void_p * 1)(fr.raw.ctypes.data), *[a.ctypes.data for a in args], parts,
                                          buf.ctypes.data, buf.ctypes.data, off.ctypes.data, cnt.ctypes.data)
        assert rc == -1 and (buf == SENTINEL).all() and (cnt == -3).all()


@pytest.mark.parametrize("step", [1, 3, 13, 16, 22, 48, 1024])
def test_no_read_outside_the_frame(lib, step):
    """Frames placed so that the page after their last byte (and, in the second placement, the page before their first byte) is
    PROT_NONE, with the frame's first and last records in the lists and a capacity far past the size: any read outside
    [frames[f], frames[f] + n[f] * step) faults."""
    rng = np.random.default_rng(500 + step)
    page = mmap.PAGESIZE
    libc = C.CDLL(None, use_errno=True)
    libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    for n in (1, 2, 31, 1500):
        fr = Frame(rng, n, step, n // 2, n - n // 2)
        data_pages = (len(fr.raw) + page - 1) // page + 1
        m = mmap.mmap(-1, (data_pages + 2) * page)
        base = C.addressof(C.c_char.from_buffer(m))
        assert libc.mprotect(base, page, 0) == 0 and libc.mprotect(base + (data_pages + 1) * page, page, 0) == 0
        for start in (base + (data_pages + 1) * page - len(fr.raw), base + page):   # flush against the guard after / before
            C.memmove(start, fr.raw.ctypes.data, len(fr.raw))
            assert gather_parts(simt_launch(lib), [fr], [3 * n + 5], 3, ptrs=[start]) == 0, f"step {step}, {n} records against a guard page"
        libc.mprotect(base, (data_pages + 2) * page, mmap.PROT_READ | mmap.PROT_WRITE)
