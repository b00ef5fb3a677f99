"""Class L1 (513–2048 points per patch): k_fit_warp<true, ..., SOA> stages each patch's x, y and z in its warp's shared memory
and runs every pass from there. It runs on the CPU through the SIMT twin's launch sequence (tests/simt/simt_twin.cpp, built
here with the library's class-L1 launch in place of the streamed kernel the twin launches) and is compared with the oracle
(CANON64): patches at both class limits and at the 1024 mid-point, tie-heavy selections, an R-VPF wall in zone 0, one CTA
draining every patch so that each warp reuses its staging region for patches of different sizes, and the fixture scans."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_py as O
from helpers import SimtTwin, assert_bins_close, assert_sets_equal, assert_state_close
from param_sets import PARAM_SETS
from pwpp_ctypes import PwppParams, default_params

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
SRC = os.path.join(HERE, "_build", "simt_twin_l1.cpp")
LIB = os.path.join(HERE, "_build", "libpwpp_simt_l1.so")
# the twin's class-L1 launch and the library's (csrc/pwpp_capi.cu: ctx->fit[2])
TWIN_L1 = 'simt::launch("k_fit_warp<false,2,2,pls>", pg, FITW_WARPS * 32, 0, [&] { k_fit_warp<false, 2, 2, 2, 3, false, true>(FIT_ARGS); });'
LIB_L1 = 'simt::launch("k_fit_warp<true,2,2,fuse,soa>", pg, FITW_WARPS * 32, FITW_SMEM_L1, [&] { k_fit_warp<true, 2, 2, 2, 1, true, false, true>(FIT_ARGS); });'


def build_lib():
    """simt_twin.cpp with LIB_L1 for TWIN_L1, compiled with the twin's compile line (tests/conftest.py: build_simt)."""
    csrc = os.path.join(REPO, "patchwork-plusplus_b200", "csrc")
    twin = os.path.join(HERE, "simt", "simt_twin.cpp")
    deps = [twin, os.path.join(HERE, "simt", "cuda_runtime.h"), os.path.abspath(__file__), os.path.join(REPO, "include", "pwpp.h")] + \
           [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        src = open(twin).read()
        assert src.count(TWIN_L1) == 1, "the twin's class-L1 launch changed"
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        with open(SRC, "w") as f:
            f.write(src.replace(TWIN_L1, LIB_L1))
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(HERE, "simt"),
                               "-I" + os.path.join(REPO, "include"), "-I" + csrc, "-o", LIB, SRC])
    return LIB


class L1Twin(SimtTwin):
    """helpers.SimtTwin on libpwpp_simt_l1.so."""

    def __init__(self, params=None, num_streams=1, **options):
        lib = C.CDLL(build_lib())
        self._bind(lib, "simt_")
        lib.simt_create.argtypes = [C.POINTER(PwppParams), C.c_int]; lib.simt_create.restype = C.c_void_p
        lib.simt_bin_ids.argtypes = [C.c_void_p, C.c_void_p]
        lib.simt_bin_results.argtypes = [C.c_void_p, C.c_void_p]
        lib.simt_num_bins.argtypes = [C.c_void_p]
        lib.simt_select.argtypes = [C.c_void_p, C.c_int]
        lib.simt_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        lib.simt_queue_sizes.argtypes = [C.c_void_p]; lib.simt_queue_sizes.restype = C.c_char_p
        lib.simt_estimate_multi.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
        self._lib = lib
        self.params = params if params is not None else default_params()
        self._h = lib.simt_create(C.byref(self.params), num_streams)
        self.nbins = lib.simt_num_bins(self._h)
        self._ns = [0] * num_streams
        for k, v in options.items():
            assert lib.simt_set_option(self._h, k.encode(), int(v)) == 0, k


def _one_bin(rng, n, z):
    """n points of one zone-0 bin (x in [5, 5.5], y in [0, 0.5]) with heights z."""
    return np.c_[5 + rng.random(n) * 0.5, rng.random(n) * 0.5, z, rng.random(n)].astype(np.float32)


def _cases():
    rng = np.random.default_rng(21)
    noisy = lambda n: _one_bin(rng, n, -1.7 + rng.normal(0, 0.02, n))  # noqa: E731
    wall = np.r_[np.c_[4 + rng.random(700) * 0.05, rng.random(700) * 0.6, -1.7 + rng.random(700) * 2.0, rng.random(700)],
                 np.c_[3 + rng.random(1200) * 4, rng.random(1200) * 0.6, -1.7 + rng.normal(0, 0.02, 1200), rng.random(1200)]]
    return {
        "n513": noisy(513),
        "n1024": noisy(1024),
        "n1025": noisy(1025),
        "n2048": noisy(2048),
        "flat_2048": _one_bin(rng, 2048, np.full(2048, -1.723)),
        "two_level_1500": _one_bin(rng, 1500, np.where(rng.random(1500) < 0.6, -1.75, -1.70)),
        "mm_quantised_1800": _one_bin(rng, 1800, np.round(-1.7 + rng.normal(0, 0.02, 1800), 3)),
        "wall_zone0_1900": wall.astype(np.float32),
    }


def _check(orc, tw, a, what):
    assert np.array_equal(orc.bin_ids(), tw.bin_ids()), f"{what}: polar bin ids differ"
    assert_sets_equal(orc.getGroundIndices(), orc.getNongroundIndices(), tw.getGroundIndices(), tw.getNongroundIndices(), len(a), what)
    assert_bins_close(orc.bin_results(), tw.bin_results(), orc.nbins, what)
    assert_state_close(orc.state(), tw.state(), what)


@pytest.mark.parametrize("opts", [dict(), dict(order=1), dict(persistent_ctas=1)])
def test_class_l1_patches(opts):
    cases = _cases()
    names = list(cases)
    tw = L1Twin(num_streams=len(names), **opts)
    tw.estimate_multi([cases[k] for k in names])
    l1 = 0
    for f, k in enumerate(names):
        orc = O.Oracle(arith=O.ARITH_CANON64)
        orc.estimate(cases[k])
        sizes = np.array([orc.bin_results()[b].n for b in range(orc.nbins)])
        assert sizes.max() == len(cases[k]), f"{k}: not one patch"
        l1 += int(((sizes > 512) & (sizes <= 2048)).sum())
        tw.select(f)
        _check(orc, tw, cases[k], f"l1/{k}/{opts}")
    assert f"L1={l1} " in tw.queue_sizes() + " ", tw.queue_sizes()


def test_fixture_scans():
    """The six fixture scans as one stream (patches of every class, the temporal state carried), then frames 0 and 4 under the
    ROS and no-R-VPF/no-TGR parameter sets."""
    kitti = [np.ascontiguousarray(np.load(os.path.join(HERE, "golden", f"kitti_{k:06d}.npz"))["xyzi_t"].T) for k in range(6)]
    orc, tw = O.Oracle(arith=O.ARITH_CANON64), L1Twin()
    for f, a in enumerate(kitti):
        orc.estimate(a); tw.estimate(a)
        _check(orc, tw, a, f"seq/{f}")
    assert "L1=0 " not in tw.queue_sizes() + " "
    for pname in ("ros", "no_rvpf_tgr"):
        mk, cols = PARAM_SETS[pname]
        for f in (0, 4):
            a = kitti[f][:, :cols]
            orc, tw = O.Oracle(mk(), O.ARITH_CANON64), L1Twin(mk())
            orc.estimate(a); tw.estimate(a)
            g_o, ng_o, g_t, ng_t = orc.getGroundIndices(), orc.getNongroundIndices(), tw.getGroundIndices(), tw.getNongroundIndices()
            big = np.array([orc.bin_results()[b].n > 512 for b in range(orc.nbins)] + [False] * 3)[orc.bin_ids()]
            mo = np.zeros(len(a), bool); mo[g_o] = True
            mt = np.zeros(len(a), bool); mt[g_t] = True
            assert len(g_o) + len(ng_o) == len(g_t) + len(ng_t)
            assert np.array_equal(mo[big], mt[big]), f"{pname}/{f}: labels of the patches above 512 points differ"
