"""The reference arithmetic (pwpp_set_arithmetic(ctx, PWPP_ARITH_REFERENCE)) on the SIMT twin: the kernels themselves, run on
the CPU through the launch sequence of that mode (tests/simt/simt_ref32.cpp). Every output is compared BIT FOR BIT with the
oracle's literal fp32 statement (PWO_ARITH_REF32, itself pinned to oracle/_ref/libpwref_stable.so by test_oracle_vs_reference.py)
and, where the reference build exists, with libpwref_stable.so directly: index lists in reference order, centers, normals,
getHeight, every threshold and history row and every patch record. No patch is excluded as degenerate."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_py as O
from helpers import SimtTwin, bits
from param_sets import PARAM_SETS
from pwpp_ctypes import PwppParams, default_params

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libpwpp_simt_ref32.so")


def build_lib():
    """tests/simt/simt_ref32.cpp with the twin's compile line (tests/conftest.py: build_simt)."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    deps = [os.path.join(HERE, "simt", f) for f in ("simt_ref32.cpp", "simt_order_exact.cpp", "simt_twin.cpp", "cuda_runtime.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))] + [os.path.join(REPO, "include", "pwpp.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, os.path.join(HERE, "simt", "simt_ref32.cpp")])
    return LIB


class Ref32Twin(SimtTwin):
    """helpers.SimtTwin on libpwpp_simt_ref32.so, estimating through simt_estimate_ref32_multi (reference order by default)."""

    def __init__(self, params=None, num_streams=1, order=1):
        lib = C.CDLL(build_lib())
        self._bind(lib, "simt_")
        lib.simt_create.argtypes = [C.POINTER(PwppParams), C.c_int]; lib.simt_create.restype = C.c_void_p
        lib.simt_bin_ids.argtypes = [C.c_void_p, C.c_void_p]
        lib.simt_bin_results.argtypes = [C.c_void_p, C.c_void_p]
        lib.simt_num_bins.argtypes = [C.c_void_p]
        lib.simt_select.argtypes = [C.c_void_p, C.c_int]
        lib.simt_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        lib.simt_queue_sizes.argtypes = [C.c_void_p]; lib.simt_queue_sizes.restype = C.c_char_p
        lib.simt_estimate_ref32_multi.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
        self._lib = lib
        self.params = params if params is not None else default_params()
        self._h = lib.simt_create(C.byref(self.params), num_streams)
        self.nbins = lib.simt_num_bins(self._h)
        self._ns = [0] * num_streams
        assert lib.simt_set_option(self._h, b"order", order) == 0

    def estimate(self, pts):
        self.estimate_multi([pts])

    def estimate_multi(self, frames):
        frames = [np.ascontiguousarray(a, dtype=np.float32) for a in frames]
        ptrs = (C.c_void_p * len(frames))(*[a.ctypes.data for a in frames])
        ns = (C.c_int64 * len(frames))(*[a.shape[0] for a in frames])
        self._lib.simt_estimate_ref32_multi(self._h, len(frames), ptrs, ns, frames[0].shape[1])
        self._ns[:len(frames)] = [a.shape[0] for a in frames]
        self.select(0)


BIN_FIELDS = ("n", "n_ground", "verdict", "fitted")


def assert_ref32_equal(orc, tw, what, bins=True):
    """Every output of the twin bit for bit that of the oracle (REF32) or of a reference build."""
    for name in ("getGroundIndices", "getNongroundIndices", "getCenters", "getNormals"):
        x, y = getattr(orc, name)(), getattr(tw, name)()
        assert x.shape == y.shape and np.array_equal(bits(x), bits(y)), f"{what} {name} differs"
    sa, sb = orc.state(), tw.state()
    assert bits(np.float64(sa.sensor_height)) == bits(np.float64(sb.sensor_height)), f"{what} sensor_height"
    for fld in ("elevation_thr", "flatness_thr"):
        assert np.array_equal(bits(np.array(getattr(sa, fld))), bits(np.array(getattr(sb, fld)))), f"{what} {fld}"
    assert list(sa.n_elevation) == list(sb.n_elevation) and list(sa.n_flatness) == list(sb.n_flatness), f"{what} history sizes"
    for r in range(4):
        for w in (0, 1):
            assert np.array_equal(bits(orc.history(r, w)), bits(tw.history(r, w))), f"{what} history ring {r} kind {w}"
    if not bins:
        return
    ba, bb = orc.bin_results(), tw.bin_results()
    for b in range(orc.nbins):
        x, y = ba[b], bb[b]
        assert tuple(getattr(x, k) for k in BIN_FIELDS) == tuple(getattr(y, k) for k in BIN_FIELDS), f"{what} bin {b} record"
        if x.fitted and x.n > 0:
            got = np.array(list(y.mean) + list(y.normal) + list(y.sv) + [y.d])
            want = np.array(list(x.mean) + list(x.normal) + list(x.sv) + [x.d])
            assert np.array_equal(bits(got), bits(want)), f"{what} bin {b} plane {got} vs {want}"


def test_fixture_sequence_default(kitti):
    """One stream over the six fixture scans, fresh state then carried: A-GLE, TGR and the thresholds in the reference arithmetic."""
    orc, tw = O.Oracle(arith=O.ARITH_REF32), Ref32Twin()
    for f, a in enumerate(kitti):
        orc.estimate(a); tw.estimate(a)
        assert np.array_equal(orc.bin_ids(), tw.bin_ids())
        assert_ref32_equal(orc, tw, f"seq/{f}")
    if O.have_reference_build():
        ref, tw2 = O.Reference(stable_sort=True), Ref32Twin()
        for f, a in enumerate(kitti[:3]):
            ref.estimate(a); tw2.estimate(a)
            assert_ref32_equal(ref, tw2, f"libpwref_stable/{f}", bins=False)


@pytest.mark.parametrize("pname", ["ros", "no_rvpf_tgr"])
def test_fixture_other_parameter_sets(kitti, pname):
    """The ROS launch set (N x 3, num_min_pts = 0: every 1-4-point patch is fitted) and no-R-VPF/no-TGR, no degenerate mask."""
    mk, cols = PARAM_SETS[pname]
    orc, tw = O.Oracle(mk(), O.ARITH_REF32), Ref32Twin(mk())
    for f in (0, 4):
        a = kitti[f][:, :cols]
        orc.estimate(a); tw.estimate(a)
        assert_ref32_equal(orc, tw, f"{pname}/{f}")


def _edge_frame():
    """Patches of 1, 2, 3, 9 and 10 points, a collinear and an exactly vertical patch, a zone-0 wall and a 20 000-point bin."""
    rng = np.random.default_rng(7)
    pts = []

    def polar(r, th, z):
        return [r * np.cos(th), r * np.sin(th), z, 0.1]
    for k, n in enumerate((1, 2, 3, 9, 10)):
        for i in range(n):
            pts.append(polar(20.0 + 0.01 * i, 0.3 + 0.2 * k, -1.7 + 0.01 * i))
    for i in range(12):   # collinear along x
        pts.append([30.0 + 0.05 * i, 5.0, -1.7, 0.1])
    for i in range(12):   # vertical: equal x, y
        pts.append([-25.0, 3.0, -1.7 + 0.1 * i, 0.1])
    for i in range(300):   # a wall in zone 0
        pts.append([4.0, -1.0 + 0.01 * (i % 100), -1.7 + 0.02 * (i // 100) + 0.5 * rng.random(), 0.1])
    th = rng.uniform(1.0, 1.02, 20000); r = rng.uniform(50.0, 50.5, 20000)
    big = np.stack([r * np.cos(th), r * np.sin(th), -1.7 + 0.02 * rng.standard_normal(20000), np.full(20000, 0.1)], 1)
    return np.concatenate([np.array(pts), big]).astype(np.float32)


def test_edge_cases():
    a = _edge_frame()
    for pname in ("default", "ros"):
        mk, cols = PARAM_SETS[pname]
        orc, tw = O.Oracle(mk(), O.ARITH_REF32), Ref32Twin(mk())
        orc.estimate(a[:, :cols]); tw.estimate(a[:, :cols])
        assert tw.queue_sizes().endswith("X=1"), tw.queue_sizes()
        assert_ref32_equal(orc, tw, f"edges/{pname}")


def test_synthetic_frames():
    import synth
    orc, tw = O.Oracle(arith=O.ARITH_REF32), Ref32Twin()
    for f in range(2):
        a = synth.make_frame(1, f).numpy()
        orc.estimate(a); tw.estimate(a)
        assert_ref32_equal(orc, tw, f"synth/{f}")


def quantised(a, step=0.01):
    """Centimetre-quantised z: equal z in almost every bin, and ties inside every part of a patch."""
    a = a.copy()
    a[:, 2] = np.round(a[:, 2] / step) * step
    return a


@pytest.mark.skipif(not O.have_reference_build(), reason="needs the reference build (oracle/_ref/libpwref.so)")
def test_exact_order_matches_the_unmodified_reference(kitti):
    """PWPP_ORDER_REFERENCE_EXACT: the fits sum equal z in libstdc++ std::sort's order, so every output equals libpwref.so's (the
    unmodified reference) bit for bit on tie-heavy scans: the six fixture scans quantised as one stream, a synthetic frame and the
    edge frame with the default parameter set, the synthetic frame with the ROS set."""
    import synth
    ref, tw = O.Reference(stable_sort=False), Ref32Twin(order=2)
    for f, a in enumerate(kitti):
        q = quantised(a)
        ref.estimate(q); tw.estimate(q)
        assert_ref32_equal(ref, tw, f"exact seq/{f}", bins=False)
    # (the edge frame leaves the first bins empty: with num_min_pts = 0 the reference build then reads an empty plane, which is
    # undefined behaviour there, so the ROS set takes the synthetic frame only)
    for pname, inputs in (("default", (synth.make_frame(20260922, 2).numpy(), _edge_frame())), ("ros", (synth.make_frame(20260922, 2).numpy(),))):
        mk, cols = PARAM_SETS[pname]
        for k, a in enumerate(inputs):
            q = np.ascontiguousarray(quantised(a)[:, :cols])
            ref, tw = O.Reference(mk(), stable_sort=False), Ref32Twin(mk(), order=2)
            ref.estimate(q); tw.estimate(q)
            assert_ref32_equal(ref, tw, f"exact {pname}/{k}", bins=False)


@pytest.fixture(scope="module")
def oracle_jsvd(tmp_path_factory):
    """oracle/pwpp_oracle.c's jsvd3f, exported from a test-only wrapper around the oracle source."""
    d = tmp_path_factory.mktemp("jsvd")
    src = d / "jsvd.c"
    src.write_text(f'#include "{os.path.join(REPO, "oracle", "pwpp_oracle.c")}"\n'
                   "void oracle_jsvd3f(const float* c, float* s, float* u) { jsvd3f(c, s, u); }\n")
    so = d / "libjsvd.so"
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(REPO, "include"), "-o", str(so), str(src), "-lm"])
    return C.CDLL(str(so)).oracle_jsvd3f


def test_jacobi_matches_the_oracle(oracle_jsvd):
    """The product's fp32 Jacobi SVD against the oracle's jsvd3f, bit for bit: random symmetric and general, rank-deficient."""
    prod = C.CDLL(build_lib()).simt_jsvd3f
    rng = np.random.default_rng(3)
    mats = []
    for _ in range(3000):
        m = rng.standard_normal((3, 3)).astype(np.float32)
        mats += [m, m + m.T, m @ m.T]
        v = rng.standard_normal(3).astype(np.float32)
        mats += [np.outer(v, v).astype(np.float32), np.outer(v, rng.standard_normal(3)).astype(np.float32)]
        u = rng.standard_normal((3, 2)).astype(np.float32)
        mats.append((u @ u.T).astype(np.float32))
    mats += [np.zeros((3, 3), np.float32), np.eye(3, dtype=np.float32), np.full((3, 3), np.nan, np.float32), np.diag([0, 1, 0]).astype(np.float32)]
    for m in mats:
        cm = np.ascontiguousarray(m.T, dtype=np.float32).ravel()   # column-major
        s1, u1, s2, u2 = (np.zeros(k, np.float32) for k in (3, 9, 3, 9))
        oracle_jsvd(cm.ctypes.data, s1.ctypes.data, u1.ctypes.data)
        prod(cm.ctypes.data, s2.ctypes.data, u2.ctypes.data)
        assert np.array_equal(bits(s1), bits(s2)) and np.array_equal(bits(u1), bits(u2)), m
