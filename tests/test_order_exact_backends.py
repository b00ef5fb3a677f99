"""The libstdc++ tie fix-up alone (csrc/pwpp_order_exact.cuh: k_order_exact_* after k_order_*), on the CPU and on the H100, against
std::sort itself.

Every case is a list of patches whose points are all ground, so a patch's list is its points sorted by z; the expected list is
what std::sort over {z, index} with `a.z < b.z` leaves, compiled here by g++ (the standard library, nothing of the reference).
The cases: every size from 0 to 600, the limits of the kernels and of the sort network (16/17, 512/513, 2048/2049, 8192/8193) and a
class-X patch; 1, 2, 3 and 17 distinct values; +-0, +-inf and NaN mixes; sorted, reversed and organ-pipe inputs; McIlroy's
adversary against this same std::sort, which drives the introsort loop to its depth limit — the fix-up's heap counter shows
that its heap branch ran. Groups: a patch whose points carry R-VPF and reject labels must come out as the stable partition of the
std::sort output by group. The "simt" backend runs the kernels through the SIMT stand-in (simt_order_exact in
tests/simt/simt_order_exact.cpp); the "device" backend as compiled for sm_90a (tests/gpu_order_exact_probe.cu, built by build.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
PROBE = os.path.join(REPO, "patchwork-plusplus_b200", "lib", "libpwpp_order_exact_probe.so")
ARGS = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
GROUND, REJECT = 255, 0

STD_SORT_SRC = r"""
#include <algorithm>
#include <cstdint>
#include <vector>
struct Pt { float z; int32_t idx; };
extern "C" long long std_sort_order(int n, const float* z, int32_t* out) {
  std::vector<Pt> v(n);
  for (int i = 0; i < n; ++i) v[i] = {z[i], i};
  long long cmp = 0;
  std::sort(v.begin(), v.end(), [&cmp](const Pt& a, const Pt& b) { ++cmp; return a.z < b.z; });
  for (int i = 0; i < n; ++i) out[i] = v[i].idx;
  return cmp;
}
// McIlroy, "A killer adversary for quicksort" (1999), against this std::sort: values are fixed as the sort compares them
extern "C" void antiqsort(int n, float* out) {
  std::vector<int> val(n, n - 1), ptr(n);
  int nsolid = 0, candidate = 0;
  const int gas = n - 1;
  for (int i = 0; i < n; ++i) ptr[i] = i;
  std::sort(ptr.begin(), ptr.end(), [&](int x, int y) {
    if (val[x] == gas && val[y] == gas) val[x == candidate ? x : y] = nsolid++;
    if (val[x] == gas) candidate = x;
    else if (val[y] == gas) candidate = y;
    return val[x] < val[y];
  });
  for (int i = 0; i < n; ++i) out[i] = (float) val[i];
}
"""


@pytest.fixture(scope="module")
def std(tmp_path_factory):
    d = tmp_path_factory.mktemp("stdsort")
    src, so = d / "std_sort.cpp", d / "libstd_sort.so"
    src.write_text(STD_SORT_SRC)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.std_sort_order.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
    L.std_sort_order.restype = C.c_longlong
    L.antiqsort.argtypes = [C.c_int, C.c_void_p]
    return L


@pytest.fixture(scope="module", params=["simt", pytest.param("device", marks=pytest.mark.gpu)])
def backend(request):
    if request.param == "simt":
        from test_order_exact import build_lib
        L, fn = C.CDLL(build_lib()), "simt_order_exact"
    else:
        assert os.path.exists(PROBE), "lib/libpwpp_order_exact_probe.so was not built (patchwork-plusplus_b200/build.py)"
        L, fn = C.CDLL(PROBE), "probe_order_exact"
    f = getattr(L, fn)
    f.argtypes = ARGS
    f.restype = C.c_int
    return f


def run(fn, patches, labels=None):
    """Every patch through both stages in one call: (lists, counters)."""
    sizes = np.array([len(p) for p in patches], np.int64)
    z = np.ascontiguousarray(np.concatenate([np.asarray(p, np.float32) for p in patches] + [np.zeros(1, np.float32)]))
    lab = None if labels is None else np.ascontiguousarray(np.concatenate(list(labels) + [np.zeros(1, np.uint8)]).astype(np.uint8))
    out = np.full(max(int(sizes.sum()), 1), -1, np.int32)
    counts = np.zeros(3, np.uint64)
    assert fn(len(patches), z.ctypes.data, sizes.ctypes.data, None if lab is None else lab.ctypes.data, out.ctypes.data, counts.ctypes.data) == 0
    lists, o = [], 0
    for n in sizes:
        lists.append(out[o:o + n].copy())
        o += n
    return lists, counts


def want(std, z):
    z = np.ascontiguousarray(z, np.float32)
    out = np.zeros(max(len(z), 1), np.int32)
    std.std_sort_order(len(z), z.ctypes.data, out.ctypes.data)
    return out[:len(z)]


def check(std, fn, patches, what):
    lists, counts = run(fn, patches)
    for k, (p, got) in enumerate(zip(patches, lists)):
        w = want(std, p)
        assert np.array_equal(got, w), f"{what}: patch {k} (n={len(p)}) first difference at {np.nonzero(got != w)[0][:3]}"
    return counts


def test_every_size_to_600(std, backend):
    rng = np.random.default_rng(1)
    patches = [rng.integers(0, 1 + n // 8, n).astype(np.float32) * 0.01 for n in range(601)]
    counts = check(std, backend, patches, "sizes 0..600")
    assert counts[0] > 500, counts   # nearly all of them hold ties and took the simulation


@pytest.mark.parametrize("n", [16, 17, 512, 513, 2048, 2049, 4096, 4097, 8192, 8193, 20000])
@pytest.mark.parametrize("distinct", [1, 2, 3, 17, 1000])
def test_class_limits_and_distinct_values(std, backend, n, distinct):
    rng = np.random.default_rng(n * 31 + distinct)
    vals = np.sort(rng.normal(-1.7, 0.2, distinct)).astype(np.float32)
    check(std, backend, [vals[rng.integers(0, distinct, n)]], f"n={n} distinct={distinct}")


def test_signed_zero_infinity_nan(std, backend):
    rng = np.random.default_rng(7)
    pool = np.array([0.0, -0.0, np.inf, -np.inf, 1.5, -1.5], np.float32)
    patches = [pool[rng.integers(0, len(pool), n)] for n in (5, 40, 300, 1500, 3000, 9000)]
    with_nan = []
    for n in (20, 100, 700, 2100, 5000):
        a = pool[rng.integers(0, len(pool), n)].copy()
        a[rng.integers(0, n, max(1, n // 50))] = np.nan
        with_nan.append(a)
    counts = check(std, backend, patches + with_nan, "+-0 / +-inf / NaN")
    assert counts[2] == len(with_nan), counts


@pytest.mark.parametrize("shape", ["sorted", "reversed", "organ"])
def test_presorted_shapes(std, backend, shape):
    patches = []
    for n in (33, 500, 1800, 4000, 8000, 12000):
        a = (np.arange(n) // 3).astype(np.float32)   # ties of three
        if shape == "reversed":
            a = a[::-1].copy()
        elif shape == "organ":
            a = np.r_[a[: n // 2], a[: n - n // 2][::-1]].astype(np.float32)
        patches.append(a)
    check(std, backend, patches, shape)


def test_mcilroy_adversary_reaches_the_heap_branch(std, backend):
    """The adversary fixes all n values distinct. Merging two adjacent values changes only the compares between those two points,
    so the sort still walks into its depth limit; halving every value ties them all in pairs. Both must take the heap branch."""
    patches, tied = [], 0
    for n in (64, 500, 4096, 8193):
        a = np.zeros(n, np.float32)
        std.antiqsort(n, a.ctypes.data)
        assert len(np.unique(a)) == n
        patches += [a, np.minimum(a, n - 2), np.floor(a / 2)]
        tied += 2
    counts = check(std, backend, patches, "antiqsort")
    assert counts[0] == tied and counts[1] >= tied, f"every tied adversary input must reach the depth limit: {counts}"


def test_groups_are_the_stable_partition_of_the_sort(std, backend):
    rng = np.random.default_rng(3)
    patches, labels = [], []
    for n in (50, 400, 1500, 3000, 7000, 10000):
        patches.append((rng.integers(0, 12, n) * 0.05).astype(np.float32))
        labels.append(rng.choice(np.array([GROUND, 1, 2, 3, REJECT], np.uint8), n))
    lists, _ = run(backend, patches, labels)
    grp = lambda lab: np.where(lab == GROUND, 0, np.where(lab == REJECT, 9, lab))
    for p, lab, got in zip(patches, labels, lists):
        w = want(std, p)
        g = grp(lab)[w]
        expect = w[np.argsort(g, kind="stable")]
        assert np.array_equal(got, expect), f"n={len(p)}"
