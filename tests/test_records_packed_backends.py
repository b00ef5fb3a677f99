"""The packed record gather of a bound call's packed records (csrc/pwpp_getters.cuh, k_bound_xyz_offsets, then
csrc/pwpp_records.cuh, k_gather_record_packed) on the CPU and on the H100, from one case list, compared byte for byte with
numpy's concatenation of records[idx_part] over the frames.

k_bound_xyz_offsets scans every frame's ground count and non-ground list length into one int64 offsets array per part (in
records); k_gather_record_packed then writes each frame's list of a part as whole records of the call's one point_step at byte
off[f] * step of the part's buffer, with no padding, so neighbouring frames share 16-byte words. Every case fills both buffers
with a sentinel byte and checks the offsets, the whole buffer up to the total against numpy, and that no byte past the total
changed. The "simt" backend runs the kernels through the SIMT stand-in (tests/simt/simt_records_packed.cpp); the "device"
backend runs them as compiled for sm_90a (tests/gpu_records_packed_probe.cu, built by patchwork-plusplus_b200/build.py), each
frame copied to the device at the same distance from a 16-byte boundary as its host array, and each buffer at the same distance
from one as the host buffer. The guard-page placements, which show that no byte outside a frame is read and none past the end
of the buffer written, can only be arranged on the CPU."""
import ctypes as C
import mmap
import os
import subprocess

import numpy as np
import pytest

from test_simt_records_gather import SENTINEL, Frame, tile_pts

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_records_packed.so")
PROBE = os.path.join(REPO, "patchwork-plusplus_b200", "lib", "libpwpp_records_packed_probe.so")
ARGS = [C.c_int] + [C.c_void_p] * 3 + [C.c_int32] + [C.c_void_p] * 2 + [C.c_int] + [C.c_void_p] * 4
STEPS = [1, 2, 3, 4, 13, 16, 22, 32, 48, 1024]
PATCHES = 7   # the count row between num_ground and num_dropped: the kernels must not read it


@pytest.fixture(scope="module")
def lib():
    """Same compile line as test_simt_records_gather.py's library."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_records_packed.cpp", "simt_records.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_records_packed.cpp")])
    L = C.CDLL(LIB)
    L.simt_gather_record_packed.argtypes = ARGS
    L.simt_gather_record_packed.restype = C.c_int
    return L


@pytest.fixture(scope="module")
def probe():
    assert os.path.exists(PROBE), "lib/libpwpp_records_packed_probe.so was not built (patchwork-plusplus_b200/build.py)"
    L = C.CDLL(PROBE)
    L.probe_gather_record_packed.argtypes = ARGS
    L.probe_gather_record_packed.restype = C.c_int
    return L


def simt_launch(lib):
    def launch(nf, ptrs, n, cap, step, idx, counts, parts, ground, nonground, g_off, ng_off):
        return lib.simt_gather_record_packed(nf, ptrs, n.ctypes.data, cap.ctypes.data, step, idx.ctypes.data, counts.ctypes.data, parts,
                                             None if ground is None else ground.ctypes.data,
                                             None if nonground is None else nonground.ctypes.data, g_off.ctypes.data, ng_off.ctypes.data)
    return launch


def device_launch(probe):
    def launch(nf, ptrs, n, cap, step, idx, counts, parts, ground, nonground, g_off, ng_off):
        import torch
        keep, d_ptrs = [], []
        for f in range(nf):
            nbytes = int(n[f]) * step
            mis = ptrs[f] % 16 if nbytes else 0
            t = torch.zeros(64 + mis + nbytes + 64, dtype=torch.uint8, device="cuda")   # (base: 512-byte aligned)
            if nbytes:
                t[64 + mis:64 + mis + nbytes] = torch.frombuffer(bytearray(C.string_at(ptrs[f], nbytes)), dtype=torch.uint8)
            keep.append(t)
            d_ptrs.append(t.data_ptr() + 64 + mis)
        d_bufs = []
        for b in (ground, nonground):   # each at its host buffer's distance from a 16-byte boundary
            if b is None:
                d_bufs.append(None)
                continue
            mis = b.ctypes.data % 16
            t = torch.empty(mis + len(b), dtype=torch.uint8, device="cuda")
            t[mis:] = torch.from_numpy(b.copy()).cuda()
            d_bufs.append((t, mis))
        torch.cuda.synchronize()
        rc = probe.probe_gather_record_packed(nf, (C.c_void_p * nf)(*d_ptrs), n.ctypes.data, cap.ctypes.data, step, idx.ctypes.data,
                                              counts.ctypes.data, parts, *[None if d is None else d[0].data_ptr() + d[1] for d in d_bufs],
                                              g_off.ctypes.data, ng_off.ctypes.data)   # (synchronous)
        for b, d in zip((ground, nonground), d_bufs):
            if b is not None:
                b[:] = d[0][d[1]:].cpu().numpy()
        return rc
    return launch


def sentinel_buffer(nbytes, mis=0):
    """nbytes of SENTINEL at mis bytes past a 16-byte boundary, 64 bytes of slack after them."""
    raw = np.full(nbytes + 64 + 32, SENTINEL, np.uint8)
    return raw[(-raw.ctypes.data) % 16 + mis:][:nbytes + 64]


def gather_packed(launch, frames, caps, parts, ptrs=None, dst_mis=0, bufs=None):
    """One launch pair over the call; checks both offsets arrays, every enabled part's buffer up to its total against numpy's
    concatenation of records[list] over the frames, and that no byte past the total changed; returns the status. bufs, when
    given, are the two destination arrays."""
    nf = len(frames)
    step = frames[0].step
    assert all(fr.step == step for fr in frames)
    idx = np.zeros(max(sum(fr.n for fr in frames), 1), np.int32)   # the slots of dropped points hold 0: the kernel never reads them
    counts = np.zeros(3 * nf, np.int32)
    p = 0
    for f, fr in enumerate(frames):
        idx[p:p + fr.ng] = fr.ground
        idx[p + fr.ng:p + fr.ng + fr.nn] = fr.nonground
        p += fr.n
        counts[f], counts[nf + f], counts[2 * nf + f] = fr.ng, PATCHES, fr.n - fr.ng - fr.nn
    want_off = [np.cumsum([0] + [fr.ng for fr in frames]), np.cumsum([0] + [fr.nn for fr in frames])]
    if bufs is None:
        bufs = [sentinel_buffer(int(sum(caps)) * step, dst_mis) if parts & bit else None for bit in (1, 2)]
    offs = [np.full(nf + 1, -5, np.int64), np.full(nf + 1, -5, np.int64)]
    rc = launch(nf, (C.c_void_p * nf)(*(ptrs if ptrs is not None else [fr.raw.ctypes.data for fr in frames])),
                np.array([fr.n for fr in frames], np.int64), np.array(caps, np.int64), step, idx, counts, parts, bufs[0], bufs[1], offs[0], offs[1])
    if rc != 0:
        return rc
    for z in (0, 1):   # the scan writes both arrays whichever parts run
        assert (offs[z] == want_off[z]).all(), (z, offs[z], want_off[z])
    for z, buf in enumerate(bufs):
        if buf is None:
            continue
        want = np.concatenate([fr.want(fr.nonground if z else fr.ground) for fr in frames] + [np.empty(0, np.uint8)])
        total = int(want_off[z][-1]) * step
        assert len(want) == total
        got = buf[:total]
        if not np.array_equal(got, want):
            first = int(np.argmax(got != want))
            f = int(np.searchsorted(want_off[z], first // step, side="right")) - 1
            raise AssertionError(f"part {z}: byte {first} differs (record {first // step}, frame {f}, step {step})")
        assert (buf[total:] == SENTINEL).all(), f"part {z}: a byte past the total was written, first at {total + np.argmax(buf[total:] != SENTINEL)}"
    return 0


# ---- the cases (both backends): build(rng) -> (frames, capacities, destination misalignment) ----------------------------------

def case_steps(step):
    """One frame of about 2.5 tiles with dropped points (capacity a tile more), one with none (capacity = size)."""
    def build(rng):
        tp = tile_pts(step)
        n = 5 * tp // 2 + 3
        return [Frame(rng, n, step, n // 3, n - n // 3 - 7, mis=3), Frame(rng, n, step, n // 2, n - n // 2, mis=12)], [n + tp, n], 0
    return build


def case_alignments(step):
    """Sixteen frames, frame k starting k bytes past a 16-byte boundary; list lengths vary, so destination alignments vary too."""
    def build(rng):
        fr = [Frame(rng, 300 + 7 * k, step, 100 + k, 180 + 3 * k, mis=k) for k in range(16)]
        return fr, [f.n + 5 * k for k, f in enumerate(fr)], 5
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
        return out, caps, 0
    return build


def case_empty_and_one_sided(step):
    """Empty frames (capacity 0 and capacity 700), all points dropped, ng = 0, nn = 0, single records."""
    def build(rng):
        fr = [Frame(rng, 0, step, 0, 0), Frame(rng, 0, step, 0, 0), Frame(rng, 40, step, 0, 0, mis=3), Frame(rng, 1500, step, 1500, 0, mis=1),
              Frame(rng, 1500, step, 0, 1500, mis=7), Frame(rng, 1, step, 1, 0, mis=15), Frame(rng, 1, step, 0, 1, mis=2),
              Frame(rng, 2, step, 0, 1, mis=9)]
        return fr, [0, 700, 40, 1600, 1500, 1, 90, 3], 0
    return build


def case_counts_far_below_capacities(step):
    """Sizes of 1/20 of the capacities or less: most CTAs of the grid have no records."""
    def build(rng):
        fr = [Frame(rng, 400, step, 150, 200, mis=1), Frame(rng, 90, step, 30, 60, mis=6), Frame(rng, 0, step, 0, 0), Frame(rng, 33, step, 1, 31, mis=11)]
        return fr, [20000, 9000, 5000, 4000], 0
    return build


def case_word_boundaries(step):
    """Forty frames whose lists hold 1 to 17 records, so that frame boundaries fall at every byte of a 16-byte word (step 13
    and 22 are coprime with 16), the destination starting at every distance from a word in turn."""
    def build(rng):
        fr = []
        for f in range(40):
            ng, nn = 1 + (3 * f) % 17, 1 + (5 * f + 2) % 17
            fr.append(Frame(rng, ng + nn + f % 3, step, ng, nn, mis=(7 * f) % 16))
        return fr, [x.n + 4 for x in fr], 11
    return build


def case_zero_length_between(step):
    """Empty lists between non-empty ones: frames of size 0, frames whose points are all dropped and one-sided frames alternate
    with frames that hold records, so several frames start at the same offset."""
    def build(rng):
        fr = []
        for f in range(24):
            kind = f % 4
            if kind == 0:
                fr.append(Frame(rng, 37 + f, step, 11 + f, 19, mis=f % 16))
            elif kind == 1:
                fr.append(Frame(rng, 0, step, 0, 0))
            elif kind == 2:
                fr.append(Frame(rng, 9, step, 0, 0, mis=3))
            else:
                fr.append(Frame(rng, 5 + f, step, 5 + f, 0, mis=9) if f % 8 == 3 else Frame(rng, 6 + f, step, 0, 6 + f, mis=4))
        return fr, [x.n + 3 * f for f, x in enumerate(fr)], 3
    return build


def case_many_frames(step):
    """1025 frames (more than one frame per thread of the offsets scan) of 0 to 40 records."""
    def build(rng):
        fr = []
        for f in range(1025):
            n = int(rng.integers(0, 41))
            ng = int(rng.integers(0, n + 1))
            nn = int(rng.integers(0, n - ng + 1))
            fr.append(Frame(rng, n, step, ng, nn, mis=f % 16))
        return fr, [x.n + (f % 5) for f, x in enumerate(fr)], 7
    return build


CASES = {**{f"steps_{s}": case_steps(s) for s in STEPS},
         **{f"alignments_{s}": case_alignments(s) for s in (13, 16, 22, 48)},
         **{f"tile_boundaries_{s}": case_tile_boundaries(s) for s in (1, 3, 13, 16, 22, 48, 1024)},
         **{f"empty_and_one_sided_{s}": case_empty_and_one_sided(s) for s in (13, 22, 1024)},
         **{f"counts_far_below_capacities_{s}": case_counts_far_below_capacities(s) for s in (16, 22, 32, 48)},
         **{f"word_boundaries_{s}": case_word_boundaries(s) for s in (13, 22)},
         **{f"zero_length_between_{s}": case_zero_length_between(s) for s in (13, 22)},
         **{f"many_frames_{s}": case_many_frames(s) for s in (13, 22)}}
# every case with both parts; the parts alone on the cases that hold every kind of list
RUNS = [(name, 3) for name in CASES] + [(name, parts) for name in ("empty_and_one_sided_22", "zero_length_between_13", "word_boundaries_22", "steps_22")
                                        for parts in (1, 2)]


def run_case(launch, name, parts):
    rng = np.random.default_rng(sum(map(ord, name)))
    frames, caps, dst_mis = CASES[name](rng)
    assert gather_packed(launch, frames, caps, parts, dst_mis=dst_mis) == 0


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
        off = np.full(2, -5, np.int64)
        args = [np.array([10], np.int64), np.array([cap], np.int64)]
        tail = [np.zeros(10, np.int32), np.array([0, 0, nd], np.int32)]   # (every array is held by a name while the call runs)
        rc = lib.simt_gather_record_packed(1, (C.c_void_p * 1)(fr.raw.ctypes.data), *[a.ctypes.data for a in args], step,
                                           *[a.ctypes.data for a in tail], parts, buf.ctypes.data, buf.ctypes.data, off.ctypes.data, off.ctypes.data)
        assert rc == -1 and (buf == SENTINEL).all() and (off == -5).all()


@pytest.mark.parametrize("step", [1, 3, 13, 16, 22, 48, 1024])
def test_no_access_outside_the_frames_and_the_buffer(lib, step):
    """Two frames placed so that the page after the last byte of each (and, in the second placement, the page before its first
    byte) is PROT_NONE, with every frame's first and last records in the lists and a capacity far past the size; and both
    destination buffers ending flush against a PROT_NONE page, every record of every frame in a list, so the packed total is
    the buffer's end: any read outside [frames[f], frames[f] + n[f] * step) or write past the buffer faults."""
    rng = np.random.default_rng(700 + step)
    page = mmap.PAGESIZE
    libc = C.CDLL(None, use_errno=True)
    libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    maps = []

    def guarded(nbytes):
        """(base of the data pages, mapping): nbytes of room between two PROT_NONE pages."""
        data_pages = (nbytes + page - 1) // page + 1
        m = mmap.mmap(-1, (data_pages + 2) * page)
        base = C.addressof(C.c_char.from_buffer(m))
        assert libc.mprotect(base, page, 0) == 0 and libc.mprotect(base + (data_pages + 1) * page, page, 0) == 0
        maps.append((m, base, data_pages))
        return base, data_pages

    for n in (1, 2, 31, 1500):
        frames = [Frame(rng, n, step, n // 2, n - n // 2), Frame(rng, n + 3, step, n - n // 3, n // 3 + 3)]
        srcs = [guarded(len(fr.raw)) for fr in frames]
        # the destination: exactly the packed total of each part, ending at the guard page after it
        dst = []
        for z in (0, 1):
            total = sum(len(fr.nonground if z else fr.ground) for fr in frames) * step
            base, data_pages = guarded(total)
            end = base + (data_pages + 1) * page
            dst.append(np.ctypeslib.as_array((C.c_ubyte * total).from_address(end - total)) if total else np.empty(0, np.uint8))
        for before in (False, True):   # flush against the guard after / before
            ptrs = []
            for fr, (base, data_pages) in zip(frames, srcs):
                start = base + page if before else base + (data_pages + 1) * page - len(fr.raw)
                C.memmove(start, fr.raw.ctypes.data, len(fr.raw))
                ptrs.append(start)
            for d in dst:
                d[:] = SENTINEL
            assert gather_packed(simt_launch(lib), frames, [3 * n + 5, 3 * n + 9], 3, ptrs=ptrs, bufs=dst) == 0, \
                f"step {step}, {n} records against a guard page"
        # the whole buffers with sentinel slack, from the same frames
        assert gather_packed(simt_launch(lib), frames, [3 * n + 5, 3 * n + 9], 3, ptrs=ptrs) == 0
    for m, base, data_pages in maps:
        libc.mprotect(base, (data_pages + 2) * page, mmap.PROT_READ | mmap.PROT_WRITE)
