"""The device state copies (csrc/pwpp_state_copy.cuh: k_state_export, k_state_import_claim + k_state_import), executed on the
CPU by the SIMT stand-in (tests/simt/simt_state_copy.cpp) and compared byte for byte with rows and states built in numpy.

A ctx's state buffers are modelled here as raw bytes: num_streams 176-byte StreamStates and 8 history rows of hist_stride
doubles per stream, of which stream s uses the first hcap[s] (its set's capacity). Export writes row i of the blob buffer from
stream streams[i]: the 16-byte header {magic "PWST", ABI version, hcap, 176}, the state and the eight history rows back to back.
Import is the reverse with a status per entry: SKIPPED (id < 0), OUT_OF_RANGE (id >= num_streams), DUPLICATE (an earlier entry
names the stream; the first one wins), BLOB_MISMATCH (header not for that stream; stream untouched) or OK. Every buffer carries
random bits and every blob row a sentinel tail past its stream's size, which the copies must leave alone. The claim table must
hold -1 everywhere after every import. tests/test_state_copy_backends.py runs the same cases on the H100."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_state_copy.so")
MAGIC, VERSION, STATE_BYTES = 0x50575354, 1, 176
OK, SKIPPED, OUT_OF_RANGE, BLOB_MISMATCH, DUPLICATE = 0, 1, 2, 3, 4
SENT = 0xA5
SIG = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_longlong]


def build_lib():
    """Same compile line as the other SIMT libraries (test_simt_bound_table.py)."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_state_copy.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_state_copy.cpp")])
    return LIB


class Backend:
    """export(...) / import_(...) over host arrays, through the library's <prefix>_state_export / <prefix>_state_import."""

    def __init__(self, path, prefix):
        L = C.CDLL(path)
        self.exp, self.imp = getattr(L, prefix + "_state_export"), getattr(L, prefix + "_state_import")
        self.exp.argtypes = SIG + [C.c_void_p]
        self.imp.argtypes = SIG + [C.c_void_p, C.c_void_p]
        self.exp.restype = self.imp.restype = C.c_int if prefix == "probe" else None
        self.checked = prefix == "probe"

    def export(self, ctx, streams, blobs, stride, status):
        rc = self.exp(len(streams), streams.ctypes.data, ctx.states.ctypes.data, ctx.hist.ctypes.data, ctx.stride, ctx.hcap.ctypes.data,
                      ctx.ns, blobs.ctypes.data, stride, None if status is None else status.ctypes.data)
        assert not self.checked or rc == 0

    def import_(self, ctx, streams, blobs, stride, status):
        rc = self.imp(len(streams), streams.ctypes.data, ctx.states.ctypes.data, ctx.hist.ctypes.data, ctx.stride, ctx.hcap.ctypes.data,
                      ctx.ns, blobs.ctypes.data, stride, ctx.claim.ctypes.data, None if status is None else status.ctypes.data)
        assert not self.checked or rc == 0


@pytest.fixture(scope="module")
def backend():
    return Backend(build_lib(), "simt")


class Ctx:
    """The state buffers of a ctx with streams on sets of the given history capacities, filled with random bits."""

    def __init__(self, rng, stream_hcap):
        self.hcap = np.ascontiguousarray(stream_hcap, np.int32)
        self.ns = len(self.hcap)
        self.stride = int(self.hcap.max())
        self.states = rng.integers(0, 256, (self.ns, STATE_BYTES), dtype=np.uint8)
        self.hist = rng.integers(0, 256, (self.ns, 8, self.stride * 8), dtype=np.uint8).view(np.float64)
        self.claim = np.full(self.ns, -1, np.int32)

    def copy(self):
        c = Ctx.__new__(Ctx)
        c.__dict__.update({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in self.__dict__.items()})
        return c

    def blob(self, s):
        h = int(self.hcap[s])
        head = np.array([MAGIC, VERSION, h, STATE_BYTES], np.uint32).view(np.uint8)
        return np.concatenate([head, self.states[s], self.hist[s, :, :h].copy().view(np.uint8).ravel()])


def blob_stride(ctx, extra=0):
    return (16 + STATE_BYTES + 64 * ctx.stride + extra + 15) // 16 * 16


def export_expected(ctx, streams, stride):
    rows = np.full((len(streams), stride), SENT, np.uint8)
    status = np.zeros(len(streams), np.int32)
    for i, s in enumerate(streams):
        if s < 0:
            status[i] = SKIPPED
        elif s >= ctx.ns:
            status[i] = OUT_OF_RANGE
        else:
            b = ctx.blob(s)
            rows[i, :len(b)] = b
    return rows, status


def import_expected(ctx, streams, rows):
    """The ctx after the import, and the statuses."""
    want = ctx.copy()
    status = np.zeros(len(streams), np.int32)
    seen = set()
    for i, s in enumerate(streams):
        if s < 0:
            status[i] = SKIPPED
            continue
        if s >= ctx.ns:
            status[i] = OUT_OF_RANGE
            continue
        if s in seen:
            status[i] = DUPLICATE
            continue
        seen.add(s)
        head = rows[i, :16].view(np.uint32)
        if head[0] != MAGIC or head[1] != VERSION or head[2] != ctx.hcap[s] or head[3] != STATE_BYTES:
            status[i] = BLOB_MISMATCH
            continue
        h = int(ctx.hcap[s])
        want.states[s] = rows[i, 16:16 + STATE_BYTES]
        want.hist[s, :, :h] = rows[i, 16 + STATE_BYTES:16 + STATE_BYTES + 64 * h].copy().view(np.float64).reshape(8, h)
    return want, status


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def run_export(backend, ctx, streams, stride, with_status=True):
    streams = np.ascontiguousarray(streams, np.int32)
    rows = np.full((len(streams), stride), SENT, np.uint8)
    status = np.full(len(streams), -7, np.int32) if with_status else None
    before = ctx.copy()
    backend.export(ctx, streams, rows, stride, status)
    want_rows, want_status = export_expected(ctx, streams, stride)
    for i in range(len(streams)):
        assert np.array_equal(rows[i], want_rows[i]), f"row {i} (stream {streams[i]}): first difference at byte {np.flatnonzero(rows[i] != want_rows[i])[:4]}"
    if with_status:
        assert np.array_equal(status, want_status), f"export status {status[:16]} != {want_status[:16]}"
    assert same_bits(ctx.states, before.states) and same_bits(ctx.hist, before.hist), "export changed the ctx"
    return rows


def run_import(backend, ctx, streams, rows, stride, with_status=True):
    streams = np.ascontiguousarray(streams, np.int32)
    rows = np.ascontiguousarray(rows)
    want, want_status = import_expected(ctx, streams, rows)
    status = np.full(len(streams), -7, np.int32) if with_status else None
    backend.import_(ctx, streams, rows, stride, status)
    if with_status:
        assert np.array_equal(status, want_status), f"import status {status[:16]} != {want_status[:16]}"
    for s in range(ctx.ns):
        assert same_bits(ctx.states[s], want.states[s]), f"state of stream {s}"
        assert same_bits(ctx.hist[s], want.hist[s]), f"histories of stream {s} (their tails past hcap included)"
    assert np.all(ctx.claim == -1), f"claim table not back at -1: {np.flatnonzero(ctx.claim != -1)[:8]}"
    return want_status


# history capacities of three sets: the default 1280 with an even stride, and an odd largest capacity (odd row stride, so no
# history word is one aligned 16-byte word of the ctx's rows)
HCAPS = {"even": (1280, 300, 12), "odd": (283, 97, 12)}


def three_set_ctx(rng, kind, ns):
    return Ctx(rng, np.array(HCAPS[kind])[np.arange(ns) % 3])


@pytest.mark.parametrize("kind", list(HCAPS))
@pytest.mark.parametrize("extra", [0, 48])
def test_export_every_stream_of_three_sets(backend, kind, extra):
    rng = np.random.default_rng(1)
    ctx = three_set_ctx(rng, kind, 7)
    stride = blob_stride(ctx, extra)
    run_export(backend, ctx, rng.permutation(ctx.ns), stride)


@pytest.mark.parametrize("kind", list(HCAPS))
def test_roundtrip_into_other_streams(backend, kind):
    """Export streams, import each row into another stream of the same set: the states and histories move, tails stay."""
    rng = np.random.default_rng(2)
    ctx = three_set_ctx(rng, kind, 9)
    stride = blob_stride(ctx, 32)
    src = np.arange(9)
    rows = run_export(backend, ctx, src, stride)
    dst = (src + 3) % 9                       # same set: stream s + 3 has the set of s
    st = run_import(backend, ctx, dst, rows, stride)
    assert np.all(st == OK)


def test_negative_and_out_of_range_ids(backend):
    rng = np.random.default_rng(3)
    ctx = three_set_ctx(rng, "even", 6)
    stride = blob_stride(ctx, 16)
    streams = np.array([0, -1, 6, 5, -2147483648, 2147483647, 2, 100], np.int32)
    rows = run_export(backend, ctx, streams, stride)
    other = three_set_ctx(np.random.default_rng(30), "even", 6)
    run_import(backend, other, streams, rows, stride)


@pytest.mark.parametrize("field", ["magic", "version", "hcap", "state_bytes"])
def test_corrupted_headers_leave_the_stream_untouched(backend, field):
    rng = np.random.default_rng(4)
    ctx = three_set_ctx(rng, "odd", 6)
    stride = blob_stride(ctx, 16)
    rows = run_export(backend, ctx, np.arange(6), stride)
    bad = {"magic": (0, MAGIC ^ 1), "version": (1, VERSION + 1), "hcap": (2, 0), "state_bytes": (3, STATE_BYTES - 16)}[field]
    for s in (1, 4):
        h = rows[s, :16].view(np.uint32)
        h[bad[0]] = bad[1] if field != "hcap" else int(ctx.hcap[(s + 1) % 6])   # a capacity of another set
    target = three_set_ctx(np.random.default_rng(40), "odd", 6)
    st = run_import(backend, target, np.arange(6), rows, stride)
    assert list(np.flatnonzero(st == BLOB_MISMATCH)) == [1, 4]


def test_duplicates_first_wins_across_two_calls(backend):
    """Several entries per stream, the first of them sometimes with a bad header (it still wins); then a second call that
    reuses the same claim table."""
    rng = np.random.default_rng(5)
    ctx = three_set_ctx(rng, "even", 6)
    stride = blob_stride(ctx, 0)
    pool = three_set_ctx(np.random.default_rng(50), "even", 6)
    rows = run_export(backend, pool, np.array([0, 3, 1, 4, 2, 5, 0, 3, 1, 4, 2, 5]), stride)
    rows[2, 0] ^= 0xFF                        # entry 2 (stream 1 below) fails its header check and still wins stream 1
    streams = np.array([0, 0, 1, 1, 2, 3, 3, 3, 4, -1, 5, 5], np.int32)
    st = run_import(backend, ctx, streams, rows, stride)
    assert list(np.flatnonzero(st == DUPLICATE)) == [1, 3, 6, 7, 11] and st[2] == BLOB_MISMATCH, st
    st = run_import(backend, ctx, streams[::-1].copy(), rows[::-1].copy(), stride)
    assert list(np.flatnonzero(st == DUPLICATE)) == [1, 5, 6, 9, 11] and st[9] == DUPLICATE, st


@pytest.mark.parametrize("n", [1, 64, 1025])
def test_list_lengths(backend, n):
    """n entries over fewer streams (so 1025 holds many duplicates), random ids with some skipped and out of range; export
    with and without a status buffer, then import a shuffled list."""
    rng = np.random.default_rng(n)
    ns = 64 if n > 1 else 3
    ctx = Ctx(rng, np.array([40, 17, 6])[np.arange(ns) % 3])
    stride = blob_stride(ctx, 16)
    streams = rng.integers(-2, ns + 2, n).astype(np.int32)
    rows = run_export(backend, ctx, streams, stride, with_status=(n != 64))
    target = Ctx(np.random.default_rng(n + 1), ctx.hcap)
    run_import(backend, target, streams, rows, stride)
    perm = rng.permutation(n)
    run_import(backend, target, streams[perm], rows[perm], stride, with_status=(n != 1025))
