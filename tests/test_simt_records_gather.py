"""The record gather kernel of the record results (csrc/pwpp_records.cuh, k_gather_records), executed on the CPU by the SIMT
stand-in (tests/simt/simt_records_gather.cpp) and compared byte for byte with numpy's records[idx].

For every frame of a call the kernel writes its index lists (ground, then non-ground; dropped points are in neither) as whole
records, to a 16-byte-aligned region of its own. Every case fills dst with a sentinel byte and checks that each region holds
exactly records[lists] and that no byte outside the regions' records changed. The value cases (CASES) also run on the H100 in
tests/test_records_gather_backends.py; the guard-page placements below, which show that no byte outside a frame is read,
can only be arranged on the CPU."""
import ctypes as C
import mmap
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_records_gather.so")
SENTINEL = 0xA5       # dst bytes before a launch
ARGS = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
STEPS = [12, 13, 16, 17, 22, 32, 48, 1024]


@pytest.fixture(scope="module")
def lib():
    """Same compile line as test_simt_records.py's library."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_records_gather.cpp", "simt_records.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_records_gather.cpp")])
    L = C.CDLL(LIB)
    L.simt_gather_records.argtypes = ARGS
    L.simt_gather_records.restype = C.c_int
    return L


def tile_pts(step):
    """Records per CTA (rec_tile_pts: 16384 bytes of whole records, at most 1024)."""
    return min(16384 // step, 1024)


def aligned_copy(raw, misalign):
    """raw at an address misalign bytes past a 16-byte boundary (the array object keeps the memory alive)."""
    base = np.empty(len(raw) + 64, np.uint8)
    start = (-base.ctypes.data) % 16 + misalign
    view = base[start:start + len(raw)]
    view[:] = raw
    return view


class Frame:
    """n random records of `step` bytes at `mis` bytes past a 16-byte boundary, with a ground list of ng and a non-ground list of
    nn distinct indices (n - ng - nn dropped), in random order (the reference order scatters sources inside a bin)."""

    def __init__(self, rng, n, step, ng, nn, mis=0):
        assert ng + nn <= n
        self.n, self.step, self.ng, self.nn = n, step, ng, nn
        self.raw = aligned_copy(rng.integers(0, 256, n * step, dtype=np.uint8), mis)
        pick = rng.permutation(n)[:ng + nn].astype(np.int32)
        self.ground, self.nonground = pick[:ng], pick[ng:]

    def want(self, lst):
        return self.raw.reshape(self.n, self.step)[lst].ravel() if self.n else np.empty(0, np.uint8)


def gather(launch, frames, ptrs=None):
    """Runs one launch over the call; checks every region and every byte outside the regions' records; returns the status."""
    nf = len(frames)
    idx = np.zeros(max(sum(fr.n for fr in frames), 1), np.int32)   # the slots of dropped points hold 0: the kernel never reads them
    p = 0
    for fr in frames:
        idx[p:p + fr.ng] = fr.ground
        idx[p + fr.ng:p + fr.ng + fr.nn] = fr.nonground
        p += fr.n
    want_off = np.cumsum([0] + [(fr.n * fr.step + 15) // 16 * 16 for fr in frames])
    dst = np.full(int(want_off[-1]) + 64 + 16, SENTINEL, np.uint8)
    dst = dst[(-dst.ctypes.data) % 16:][:int(want_off[-1]) + 64]   # 16-byte aligned, 64 bytes of slack after the last region
    dst[:] = SENTINEL
    rec_off = np.zeros(nf + 1, np.int64)
    rc = launch(nf, (C.c_void_p * nf)(*(ptrs if ptrs is not None else [fr.raw.ctypes.data for fr in frames])),
                np.array([fr.n for fr in frames], np.int64), np.array([fr.step for fr in frames], np.int32), idx,
                np.array([fr.n - fr.ng - fr.nn for fr in frames], np.int32), dst, rec_off)
    if rc != 0:
        return rc
    assert (rec_off == want_off).all(), (rec_off, want_off)
    touched = np.zeros(len(dst), bool)
    for f, fr in enumerate(frames):
        o, s = int(rec_off[f]), fr.step
        g = dst[o:o + fr.ng * s]
        ng_bytes = dst[o + fr.ng * s:o + (fr.ng + fr.nn) * s]
        assert np.array_equal(g, fr.want(fr.ground)), f"frame {f} (step {s}, {fr.n} records): ground records differ"
        assert np.array_equal(ng_bytes, fr.want(fr.nonground)), f"frame {f} (step {s}, {fr.n} records): non-ground records differ"
        touched[o:o + (fr.ng + fr.nn) * s] = True
    assert (dst[~touched] == SENTINEL).all(), f"a byte outside the regions' records was written, first at {np.argmax((dst != SENTINEL) & ~touched)}"
    return 0


def simt_launch(lib):
    return lambda nf, ptrs, n, step, idx, nd, dst, off: lib.simt_gather_records(nf, ptrs, n.ctypes.data, step.ctypes.data, idx.ctypes.data,
                                                                                nd.ctypes.data, dst.ctypes.data, off.ctypes.data)


# ---- the value cases (both backends) -------------------------------------------------------------------------------------------

def case_steps(step):
    """One frame of about 2.5 tiles with dropped points, then one with none."""
    def build(rng):
        tp = tile_pts(step)
        n = 5 * tp // 2 + 3
        return [Frame(rng, n, step, n // 3, n - n // 3 - 7), Frame(rng, n, step, n // 2, n - n // 2)]
    return build


def case_alignments(step):
    """Sixteen frames in one call, frame k starting k bytes past a 16-byte boundary (sizes vary, so the output alignment varies too)."""
    def build(rng):
        return [Frame(rng, 300 + 7 * k, step, 100 + k, 180, mis=k) for k in range(16)]
    return build


def case_tile_boundaries(step):
    """ng + nn at k * tile - 1, k * tile and k * tile + 1 (k = 1, 2), with and without dropped points after them."""
    def build(rng):
        tp = tile_pts(step)
        out = []
        for f, m in enumerate(k * tp + d for k in (1, 2) for d in (-1, 0, 1)):
            drop = 0 if f % 2 else 1 + f
            out.append(Frame(rng, m + drop, step, m // 3, m - m // 3, mis=(5 * f) % 16))
        return out
    return build


def case_empty_and_one_sided():
    """Empty frames, frames whose points are all dropped, all ground, all non-ground, single records."""
    def build(rng):
        return [Frame(rng, 0, 22, 0, 0), Frame(rng, 40, 22, 0, 0, mis=3), Frame(rng, 1500, 22, 1500, 0, mis=1),
                Frame(rng, 1500, 22, 0, 1500, mis=7), Frame(rng, 1, 13, 1, 0, mis=15), Frame(rng, 1, 13, 0, 1, mis=2),
                Frame(rng, 0, 1024, 0, 0), Frame(rng, 2, 1024, 0, 1, mis=9)]
    return build


def case_mixed_layouts():
    """Every step of STEPS plus steps 1, 2, 3, 5 and 7 (a word of output spans up to four records) in one launch."""
    def build(rng):
        steps = STEPS + [1, 2, 3, 5, 7]
        return [Frame(rng, 900 + 37 * f, s, 300 + f, 500, mis=(3 * f + 1) % 16) for f, s in enumerate(steps)]
    return build


CASES = {**{f"steps_{s}": case_steps(s) for s in STEPS},
         **{f"alignments_{s}": case_alignments(s) for s in (12, 13, 16, 17, 22, 48)},
         **{f"tile_boundaries_{s}": case_tile_boundaries(s) for s in STEPS},
         "empty_and_one_sided": case_empty_and_one_sided(), "mixed_layouts": case_mixed_layouts()}


def run_case(launch, name):
    rng = np.random.default_rng(sum(map(ord, name)))
    assert gather(launch, CASES[name](rng)) == 0


def test_bad_step_or_count_launches_nothing(lib):
    rng = np.random.default_rng(1)
    fr = Frame(rng, 10, 16, 5, 5)
    for step, nd in ((0, 0), (1025, 0), (16, 11), (16, -1)):
        dst = np.full(256, SENTINEL, np.uint8)
        rc = lib.simt_gather_records(1, (C.c_void_p * 1)(fr.raw.ctypes.data), np.array([10], np.int64).ctypes.data, np.array([step], np.int32).ctypes.data,
                                     np.zeros(10, np.int32).ctypes.data, np.array([nd], np.int32).ctypes.data, dst.ctypes.data,
                                     np.zeros(2, np.int64).ctypes.data)
        assert rc == -1 and (dst == SENTINEL).all()


@pytest.mark.parametrize("step", [1, 3, 13, 16, 22, 48, 1024])
def test_no_read_outside_the_frame(lib, step):
    """Frames placed so that the page after their last byte (and, in the second placement, the page before their first byte) is
    PROT_NONE, with the frame's first and last records in the lists: any read outside [frames[f], frames[f] + n[f] * step) faults."""
    rng = np.random.default_rng(400 + step)
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
            assert gather(simt_launch(lib), [fr], ptrs=[start]) == 0, f"step {step}, {n} records against a guard page"
        libc.mprotect(base, (data_pages + 2) * page, mmap.PROT_READ | mmap.PROT_WRITE)
