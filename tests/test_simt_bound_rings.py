"""The frame-table kernels of ring-bound calls (csrc/pwpp_records.cuh, k_bound_table_rings and k_bound_table_rings_actions),
executed on the CPU by the SIMT stand-in (tests/simt/simt_bound_rings.cpp) and compared word for word with numpy; then the record
unpack and the part gather of the run, which read the run's record table the table kernel wrote, over rings placed flush
against guard pages.

A frame that runs reads its slot once (the run's copy holds it), takes its count from its ring's slot entry, and its run record
table entry points at base + slot * slot_stride. A slot outside [0, num_slots) gives PWPP_SLOT_OUT_OF_RANGE and an empty frame;
a skipped frame reads neither slot nor count (copy -1). Both kinds keep src = base with n = 0. Every output array is filled with
a sentinel first and the words after its table must keep it."""
import ctypes as C
import mmap
import os
import subprocess

import numpy as np
import pytest

from test_simt_bound_actions import ACTION_MENU, I32_MAX, I32_MIN, INVALID, OUT_OF_RANGE, PAD, RESET, RUN, SENT32, SENT64, SKIP, SKIPPED, \
    bind_tables, check_states

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_bound_rings.so")
CHUNK_PTS = 4096
SLOT_OUT_OF_RANGE = 4   # PWPP_SLOT_OUT_OF_RANGE
SENT_BYTE = 0xA5


@pytest.fixture(scope="module")
def lib():
    """Same compile line as test_simt_bound_actions.py's library."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_bound_rings.cpp", "simt_records.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_bound_rings.cpp")])
    L = C.CDLL(LIB)
    L.simt_stream_state_bytes.restype = C.c_int
    L.simt_record_frame_bytes.restype = C.c_int
    L.simt_bound_table_rings.argtypes = [C.c_int] + [C.c_void_p] * 22
    L.simt_bound_table_rings.restype = None
    L.simt_unpack_run.argtypes = [C.c_int] + [C.c_void_p] * 4
    L.simt_unpack_run.restype = None
    L.simt_gather_parts_run.argtypes = [C.c_int] + [C.c_void_p] * 9
    L.simt_gather_parts_run.restype = None
    assert L.simt_record_frame_bytes() == 48
    return L


def layout(step):
    """x, y, z FLOAT32 at 0, 4, 8 and an intensity that converts exactly: UINT8 at 12 (step 13), FLOAT32 at 12 (16) or 16 (22)."""
    from pwpp_ctypes import PwppPointLayout
    lay = PwppPointLayout()
    lay.point_step = step
    ioff, itype = {13: (12, 2), 16: (12, 7), 22: (16, 7)}[step]
    for c, (o, t) in enumerate([(0, 7), (4, 7), (8, 7), (ioff, itype)]):
        lay.offset[c], lay.datatype[c] = o, t
    return lay


class Rings:
    """Ring r: num_slots[r] slots of int64 counts; frame f names ring ring_of[f]."""

    def __init__(self, bases, strides, counts, ring_of, steps):
        self.bases, self.strides = [int(b) for b in bases], [int(s) for s in strides]
        self.counts = [np.ascontiguousarray(c, np.int64) for c in counts]
        self.ring_of = np.asarray(ring_of)
        self.steps = list(steps)


def run_table(lib, rings, max_n, streams, sets, slots, actions, num_streams):
    """One ring table launch; checks every output word against the numpy model and returns (pt_off, status, the run's record
    table as nframes rows of 48 bytes)."""
    nf = len(max_n)
    max_n = np.ascontiguousarray(max_n, np.int64)
    streams, sets = np.ascontiguousarray(streams, np.int32), np.ascontiguousarray(sets, np.int32)
    slots = np.ascontiguousarray(slots, np.int32)
    ro = rings.ring_of
    f_bases = np.array([rings.bases[r] for r in ro], np.uint64)
    f_strides = np.array([rings.strides[r] for r in ro], np.int64)
    f_slots_n = np.array([len(rings.counts[r]) for r in ro], np.int32)
    f_counts = (C.c_void_p * nf)(*[rings.counts[r].ctypes.data for r in ro])
    lays = [layout(rings.steps[f]) for f in range(nf)]
    from pwpp_ctypes import PwppPointLayout
    lay_arr = (PwppPointLayout * nf)(*lays)
    runs, scratch, dep = bind_tables(streams.tolist(), num_streams)
    sb = lib.simt_stream_state_bytes()
    nslots = num_streams + (max(np.diff(runs)) if nf else 0)
    init = np.ascontiguousarray(((np.arange(nslots)[:, None] * 7 + np.arange(sb)[None, :]) % 251 + 1).astype(np.uint8))
    states = np.full((nslots + PAD, sb), 0x5A, np.uint8)
    out = [np.full(nf + 1 + PAD, SENT64, np.int64), np.full(nf + 1 + PAD, SENT32, np.int32)] + [np.full(nf + PAD, SENT32, np.int32) for _ in range(5)]
    brun = np.full((nf + PAD) * 48, 0x5A, np.uint8)
    acts = None if actions is None else np.ascontiguousarray(actions, np.int32)
    lib.simt_bound_table_rings(nf, max_n.ctypes.data, streams.ctypes.data, sets.ctypes.data, *[o.ctypes.data for o in out[:5]],
                               None if acts is None else acts.ctypes.data, out[5].ctypes.data, scratch.ctypes.data, dep.ctypes.data,
                               init.ctypes.data, states.ctypes.data, slots.ctypes.data, out[6].ctypes.data, (C.c_void_p * nf)(*f_bases.tolist()),
                               f_counts, f_strides.ctypes.data, f_slots_n.ctypes.data, lay_arr, brun.ctypes.data)
    # the model
    runs_ = np.ones(nf, bool) if acts is None else (acts == RUN) | (acts == RESET)
    slot_ok = runs_ & (slots >= 0) & (slots < f_slots_n)
    c = np.array([rings.counts[ro[f]][slots[f]] if slot_ok[f] else -1 for f in range(nf)], np.int64)
    ok = slot_ok & (c >= 0) & (c <= max_n)
    n = np.where(ok, c, 0)
    pt_off = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    chunk_off = np.concatenate([[0], np.cumsum((n + CHUNK_PTS - 1) // CHUNK_PTS)]).astype(np.int32)
    if acts is None:
        skip_st = np.zeros(nf, np.int32)
    else:
        skip_st = np.where(acts == SKIP, SKIPPED, INVALID)
    status = np.where(runs_, np.where(ok, 0, np.where(slot_ok, OUT_OF_RANGE, SLOT_OUT_OF_RANGE)), skip_st).astype(np.int32)
    stream = np.where(runs_, streams, scratch).astype(np.int32)
    slot_copy = np.where(runs_, slots, -1).astype(np.int32)
    want = [pt_off, chunk_off, stream, sets, status]
    names = ["pt_off", "chunk_off", "stream", "pset", "status"]
    if acts is not None:
        want.append(acts)
        names.append("act")
    for name, o, w in zip(names, out, want):
        assert np.array_equal(o[:len(w)], w), f"{name}: first mismatch at {np.flatnonzero(o[:len(w)] != w)[:5]}"
        assert np.all(o[len(w):] == (SENT64 if o.dtype == np.int64 else SENT32)), f"{name}: a word after the table changed"
    if acts is None:
        assert np.all(out[5] == SENT32), "act was written without actions"
    assert np.array_equal(out[6][:nf], slot_copy), f"slot copy: first mismatch at {np.flatnonzero(out[6][:nf] != slot_copy)[:5]}"
    assert np.all(out[6][nf:] == SENT32)
    # the run's record table: the bound entry with src moved to the slot
    rec = brun.reshape(-1, 48)
    src = rec[:nf, :8].copy().view(np.uint64).reshape(-1)
    want_src = np.where(slot_ok, f_bases + (np.where(slot_ok, slots, 0).astype(np.int64) * f_strides).astype(np.uint64), f_bases)
    assert np.array_equal(src, want_src), f"brun src: first mismatch at {np.flatnonzero(src != want_src)[:5]}"
    step = rec[:nf, 8:12].copy().view(np.int32).reshape(-1)
    assert step.tolist() == [rings.steps[f] for f in range(nf)], "brun step"
    assert np.all(rec[nf:] == 0x5A), "a record after the table changed"
    reset = np.zeros(nslots + PAD, bool)
    if acts is not None:
        reset[np.unique(streams[(acts == RESET) & (dep == 0)])] = True
    check_states(states, init, reset, "ring table")
    return pt_off, status, rec[:nf].copy()


SLOT_MENU = lambda S: [0, 1 % S, S - 1, -1, S, I32_MAX, I32_MIN]   # noqa: E731


def random_rings(rng, nf, steps=(13, 16, 22)):
    """max(1, nf // 3) rings of 1 to 5 slots (frames share them: frame f names ring f % nrings), counts in and out of range of
    every frame's capacity, fake bases (the table kernel only forms addresses)."""
    nr = max(1, nf // 3)
    max_n = rng.integers(1, 20000, nf)
    step_r = rng.choice(steps, nr)
    ro = np.arange(nf) % nr
    cap_r = [max(max_n[ro == r]) for r in range(nr)]
    num_slots = rng.integers(1, 6, nr)
    counts = []
    for r in range(nr):
        menu = [0, 1, 4095, 4096, 4097, cap_r[r], cap_r[r] + 1, -1, -2 ** 63, 2 ** 63 - 1]
        counts.append(np.array([menu[k] if rng.random() < 0.3 else rng.integers(0, cap_r[r] + 1) for k in rng.integers(0, len(menu), num_slots[r])], np.int64))
    strides = [cap_r[r] * step_r[r] + int(rng.integers(0, 100)) for r in range(nr)]
    bases = [0x7f0000000000 + (r << 32) + int(rng.integers(0, 16)) for r in range(nr)]
    return Rings(bases, strides, counts, ro, [int(step_r[r]) for r in ro]), max_n


@pytest.mark.parametrize("nf", [1, 1023, 1024, 1025, 3000])
@pytest.mark.parametrize("with_actions", [False, True], ids=["rings", "rings_actions"])
def test_slots_counts_and_actions(lib, nf, with_actions):
    """Slots in range, -1, num_slots and INT_MAX / INT_MIN, per-slot counts in and out of range, shared rings; with actions every
    action of the menu, a skipped frame's slot being garbage."""
    rng = np.random.default_rng(nf + 7 * with_actions)
    rings, max_n = random_rings(rng, nf)
    S = np.array([len(rings.counts[r]) for r in rings.ring_of])
    slots = np.array([SLOT_MENU(int(s))[k] if rng.random() < 0.4 else rng.integers(0, s) for s, k in zip(S, rng.integers(0, 7, nf))], np.int64)
    actions = None
    if with_actions:
        actions = np.array(ACTION_MENU * (nf // len(ACTION_MENU) + 1))[:nf] if nf > 7 else rng.choice(ACTION_MENU, nf)
        skipped = ~np.isin(actions, [RUN, RESET])
        slots = np.where(skipped, rng.choice([I32_MAX, I32_MIN, -1, 10 ** 6], nf), slots)
    num_streams = max(8, nf // 4) if nf > 5 else 3
    streams = rng.integers(0, num_streams, nf) if with_actions else rng.permutation(max(nf, 1))[:nf]
    run_table(lib, rings, max_n, streams, rng.integers(0, 8, nf), slots.astype(np.int32), actions,
              num_streams if with_actions else max(nf, 1))


@pytest.mark.parametrize("action", ACTION_MENU)
def test_one_action_everywhere(lib, action):
    """All frames on one action over rings whose slots and counts are all garbage for the skipped ones."""
    rng = np.random.default_rng(5)
    nf = 300
    rings, max_n = random_rings(rng, nf)
    slots = rng.choice([0, 1, -1, I32_MAX], nf).astype(np.int32)
    _, status, _ = run_table(lib, rings, max_n, rng.permutation(nf), np.arange(nf) % 4, slots, np.full(nf, action, np.int32), nf)
    if action not in (RUN, RESET):
        assert np.all(status == (SKIPPED if action == SKIP else INVALID))


def test_backlog_and_identity_shape(lib):
    """One sensor's backlog: its ring bound to two entries of one stream (second entry reads the next slot, or is skipped), next
    to one-slot rings of the identity shape {frame, max_n * step, counts + f, 1} with slot 0; RESET with an invalid slot resets."""
    counts_shared = np.array([100, 7, 5000, -3], np.int64)
    one = [np.array([c], np.int64) for c in (50, 0, 4097)]
    rings = Rings([0x1000, 0x900000, 0xA00000, 0xB00000], [5000 * 22 + 3, 100 * 16, 100 * 16, 5000 * 16],
                  [counts_shared] + one, [0, 1, 0, 2, 3], [22, 16, 22, 16, 16])
    max_n = np.array([5000, 100, 5000, 100, 5000])
    streams = [0, 1, 0, 2, 3]
    for slots, acts in (([0, 0, 1, 0, 0], [RUN] * 5), ([1, 0, 2, 0, 0], [RUN, RUN, SKIP, RUN, RUN]), ([2, 0, 3, 0, 0], [RUN, RESET, RUN, RUN, RUN]),
                        ([4, 0, -1, 1, 0], [RESET, RUN, RESET, RESET, RUN]), ([3, 0, 0, 0, 0], None)):
        _, status, _ = run_table(lib, rings, max_n, streams, [0] * 5, slots, None if acts is None else np.array(acts), 4)
        assert status[3] == (SLOT_OUT_OF_RANGE if slots[3] else 0)


# ---- the unpack and the part gather of the run, over rings flush against guard pages -------------------------------------------

def make_records(rng, n, step):
    raw = rng.integers(0, 256, (n, step), dtype=np.uint8)
    xyz = rng.uniform(-50, 50, (n, 3)).astype(np.float32)
    raw[:, 0:12] = xyz.view(np.uint8).reshape(n, 12)
    if step == 13:
        inten = raw[:, 12].astype(np.float32)
    else:
        o = 12 if step == 16 else 16
        iv = rng.uniform(0, 1, n).astype(np.float32)
        raw[:, o:o + 4] = iv.view(np.uint8).reshape(n, 4)
        inten = iv
    pts = np.concatenate([xyz, inten[:, None]], axis=1)
    return raw, pts


@pytest.mark.parametrize("step", [13, 16, 22])
@pytest.mark.parametrize("pad", [0, 5])
def test_unpack_and_gather_through_the_run_table(lib, step, pad):
    """A 3-slot ring placed with its extent [base, base + 2 * stride + max_n * step) flush against a PROT_NONE page after it, then
    with base right after a PROT_NONE page; five frames name it (slots 0 and 2 at full capacity, so the extent's first and last
    bytes are read, slot 1, an invalid slot and an out-of-range count), next to a valid frame of its own one-slot ring. The
    unpack through the run's table must give each frame the points of its slot, the gather the records of its lists: any read
    outside the ring faults."""
    rng = np.random.default_rng(step * 10 + pad)
    page = mmap.PAGESIZE
    libc = C.CDLL(None, use_errno=True)
    libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    max_n = 300
    stride = max_n * step + pad
    extent = 2 * stride + max_n * step
    slot_n = [max_n, 123, max_n]
    recs = [make_records(rng, slot_n[s], step) for s in range(3)]
    ring_img = np.full(extent, SENT_BYTE, np.uint8)
    for s in range(3):
        ring_img[s * stride: s * stride + slot_n[s] * step] = recs[s][0].reshape(-1)
    other_raw, other_pts = make_records(rng, 77, step)
    data_pages = (extent + page - 1) // page + 1
    m = mmap.mmap(-1, (data_pages + 2) * page)
    base0 = C.addressof(C.c_char.from_buffer(m))
    assert libc.mprotect(base0, page, 0) == 0 and libc.mprotect(base0 + (data_pages + 1) * page, page, 0) == 0
    counts_main = np.array(slot_n, np.int64)
    counts_oor = np.array([max_n + 1, 5, 6], np.int64)   # (a ring of the same slots whose slot 0 count is out of range)
    counts_other = np.array([77], np.int64)
    slots = np.array([0, 2, 1, 3, 0, 0], np.int32)
    try:
        for start in (base0 + (data_pages + 1) * page - extent, base0 + page):   # flush against the guard after / before
            C.memmove(start, ring_img.ctypes.data, extent)
            rings = Rings([start, start, other_raw.ctypes.data], [stride, stride, 77 * step], [counts_main, counts_oor, counts_other],
                          [0, 0, 0, 0, 1, 2], [step] * 6)
            mx = np.array([max_n] * 5 + [77], np.int64)
            pt_off, status, brun = run_table(lib, rings, mx, np.arange(6), np.zeros(6), slots, None, 6)
            assert status.tolist() == [0, 0, 0, SLOT_OUT_OF_RANGE, OUT_OF_RANGE, 0]
            srcs = [recs[0], recs[2], recs[1], None, None, (other_raw, other_pts)]
            brun = np.ascontiguousarray(brun)
            dst = np.full((int(pt_off[-1]) + 1, 4), np.nan, np.float32)
            lib.simt_unpack_run(6, brun.ctypes.data, mx.ctypes.data, pt_off.ctypes.data, dst.ctypes.data)
            for f, sr in enumerate(srcs):
                got = dst[pt_off[f]:pt_off[f + 1]]
                want = np.zeros((0, 4), np.float32) if sr is None else sr[1]
                assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"frame {f}: unpacked points"
            # index lists: a permutation of each frame's records, the ground list first, some points dropped
            nfr = np.diff(pt_off)
            idx = np.zeros(max(int(pt_off[-1]), 1), np.int32)
            counts = np.zeros(18, np.int32)
            lists = []
            for f in range(6):
                n = int(nfr[f])
                perm = rng.permutation(n).astype(np.int32)
                if n:   # the first and the last record of the slot are in the lists
                    perm = np.concatenate([[0, n - 1] if n > 1 else [0], perm[(perm != 0) & (perm != n - 1)]]).astype(np.int32)
                ng, nd = n // 3, min(n // 10, max(n - 2, 0))
                idx[pt_off[f]:pt_off[f] + n] = perm
                counts[f], counts[6 + f], counts[12 + f] = ng, 9, nd
                lists.append((perm[:ng], perm[ng:n - nd]))
            region = [(c * step + 15) // 16 * 16 for c in mx]
            total = int(sum(region))
            bufs = [np.full(total + 64, SENT_BYTE, np.uint8) for _ in range(2)]
            part_off = np.zeros(7, np.int64)
            part_cnt = np.full(12, -3, np.int32)
            lib.simt_gather_parts_run(6, brun.ctypes.data, mx.ctypes.data, pt_off.ctypes.data, counts.ctypes.data, idx.ctypes.data,
                                      bufs[0].ctypes.data, bufs[1].ctypes.data, part_off.ctypes.data, part_cnt.ctypes.data)
            assert part_off.tolist() == np.concatenate([[0], np.cumsum(region)]).tolist()
            for f, sr in enumerate(srcs):
                raw = np.zeros((0, step), np.uint8) if sr is None else sr[0]
                assert part_cnt[2 * f: 2 * f + 2].tolist() == [len(lists[f][0]), len(lists[f][1])], f"frame {f}: counts"
                for z in range(2):
                    want = raw[lists[f][z]].reshape(-1)
                    o = int(part_off[f])
                    assert np.array_equal(bufs[z][o:o + len(want)], want), f"frame {f} part {z}: records"
                    assert np.all(bufs[z][o + len(want):int(part_off[f + 1])] == SENT_BYTE), f"frame {f} part {z}: past the records"
    finally:
        libc.mprotect(base0, (data_pages + 2) * page, mmap.PROT_READ | mmap.PROT_WRITE)
