"""The device kernels at their edges, against the oracle (CANON64) through the C-ABI.

1. Polar binning on and beside every decision boundary of four geometries (ring, zone and range limits, sector limits,
   the RNR predicate), through all three front ends a call can take: the stand-alone kernels of a one-frame call
   (k_bin_hist / k_scatter), the cluster kernel of a batch (k_front_cluster<FAST, ..., 256>) and its dense variant
   (k_front_cluster<FAST, ..., 512>). FAST is the fp32 filter of bin_of_point where build_geometry allows it, the exact
   double path otherwise. Bin ids must equal the oracle's bit for bit, except on the libm-defined band: the points whose
   bin changes when a double atan2 moves by at most 4 ulp from the exact angle (CUDA's and glibc's atan2 are both
   within that of the exact value, but neither is correctly rounded). There the device's bin must be one of the bins
   those angles give, i.e. the oracle's bin or the adjacent sector of the same ring.
2. Every fit and sort kernel at its size limits: patches on both sides of every class limit and of the sort network's
   limits, tie-heavy and signed-zero z, the class-X selections that overflow k_fit_big's candidate buffer and a zone-0
   wall, through a batch call, one-frame calls (called twice, so the second call replays the small-call graph) and a
   stream-table call that mixes both kernel sets, in both output orders.

Each case asserts the conditions under which launch_range_impl (csrc/pwpp_capi.cu) picks the kernels it is meant to
reach, so that a change of those rules cannot move it silently onto another kernel.
"""
import os
import re

import numpy as np
import pytest

import oracle_py as O
from pwpp_ctypes import default_params
from test_gpu_parity import compare_frame

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "patchwork-plusplus_b200", "csrc")
LD = np.longdouble
PI_LD = np.arctan2(LD(0), LD(-1))
ULPS = 4              # half-width of the libm-defined band, in ulps of the double angle
DENSE_MEAN = 400_000  # launch_range_impl: mean points per frame above which the front end takes 512 threads per CTA
HOST_CHUNK_PTS = 4 << 20   # pwpp_estimate_host: points per pipeline chunk
CLASS_MAX = (64, 512, 2048, 4096, 8192)   # S, M, L1, L2, L3; X above (csrc/pwpp_fit.cuh)
CLASS_NAMES = ("S", "M", "L1", "L2", "L3", "X")


def _tuning(name):
    with open(os.path.join(CSRC, "pwpp_tuning.h")) as fh:
        return int(re.search(rf"#define {name}\s+(\d+)", fh.read()).group(1))


def _assert_default_switches():
    """The kernels a call takes depend on these switches: the cases below assume the compiled-in defaults."""
    for k in ("PWPP_FRONT", "PWPP_FIT_PATCH", "PWPP_SMALL_CALL", "PWPP_GRAPH", "PWPP_SERIAL_FIT", "PWPP_SUBBATCH_POINTS"):
        assert k not in os.environ, f"{k} is set: the kernel selection asserted here assumes the defaults"
    assert _tuning("PWPP_FRONT_DEFAULT") == 1 and _tuning("PWPP_FIT_PATCH_DEFAULT") == 0
    return _tuning("PWPP_SMALL_CALL_DEFAULT")


def _assert_one_launch_range(frames):
    """pwpp_estimate_host cuts a call into pipeline chunks of ~4M points; a case that names a kernel of a call shape needs
    the whole call in one chunk (a call split into ranges of <= PWPP_SMALL_CALL frames would take the small-call kernels)."""
    nf, total = len(frames), sum(len(a) for a in frames)
    if nf > 1:
        assert min(nf, max(1, HOST_CHUNK_PTS // max(1, total // nf))) == nf


# ---- geometry (build_geometry, csrc/pwpp_host.hpp) -----------------------------------------------------------------------
class Geom:
    def __init__(self, p):
        mn, mx = p.min_range, p.max_range
        self.mins = [mn, (7 * mn + mx) / 8.0, (3 * mn + mx) / 4.0, (mn + mx) / 2.0]
        bounds = self.mins + [mx]
        self.nr = [int(v) for v in p.num_rings_each_zone]
        self.ns = [int(v) for v in p.num_sectors_each_zone]
        self.rs = [(bounds[k + 1] - bounds[k]) / self.nr[k] for k in range(4)]
        self.ss = [2 * np.pi / n for n in self.ns]
        self.base = np.cumsum([0] + [self.nr[k] * self.ns[k] for k in range(4)])
        self.nbins = int(self.base[4])
        self.min_range, self.max_range = mn, mx
        self.fast = mx <= 250.0 and all(r >= 1.5 for r in self.rs) and all(n <= 128 for n in self.ns)
        self.nbp = (self.nbins + 3 + 31) // 32 * 32

    def front_smem(self, nthreads):   # front_cluster_smem_bytes (csrc/pwpp_front.cuh)
        w = nthreads // 32
        return w * 2 * 128 * 16 + (w + 1) * self.nbp * 4 + (((self.nbp + 1) * 4 + 15) & ~15) + w * 2 * 8 + 3 * 6 * 4

    def ring_bounds(self):
        rb = []
        for k in range(4):
            rb += [self.mins[k] + i * self.rs[k] for i in range(self.nr[k])]
        return rb + [self.max_range]

    def bin_of(self, zone, ring, sector):
        return int(self.base[zone]) + ring * self.ns[zone] + sector


def _steps(d, n):
    """d moved by n ulps (n may be negative)."""
    out = d.copy()
    for _ in range(abs(n)):
        out = np.nextafter(out, np.inf if n > 0 else -np.inf)
    return out


def _model_bins(pts, p, g):
    """bin_of_point_exact / rnr_hit in numpy, for every double the atan2 calls may return within ULPS of the exact angle.
    Returns (candidates, rnr): polar bin per candidate angle [n, 2 ULPS + 1] (column ULPS: the correctly rounded angle) and
    the RNR verdict per candidate vertical angle [n, 2 ULPS + 1]. Everything but atan2 is correctly rounded IEEE double
    (or float, as in the code), so it is the same on both sides."""
    n = len(pts)
    x, y, z = (pts[:, i].astype(np.float64) for i in range(3))
    r = np.sqrt(x * x + y * y)
    inr = (r <= g.max_range) & (r > g.min_range) & np.isfinite(z)
    k = np.where(r < g.mins[1], 0, np.where(r < g.mins[2], 1, np.where(r < g.mins[3], 2, 3)))
    mins, rs = np.array(g.mins)[k], np.array(g.rs)[k]
    nr, ns, ss, base = np.array(g.nr)[k], np.array(g.ns)[k], np.array(g.ss)[k], g.base[k]
    with np.errstate(invalid="ignore"):
        ring = np.minimum(np.nan_to_num((r - mins) / rs, nan=0.0, posinf=0.0, neginf=0.0).astype(np.int64), nr - 1)
    theta = np.arctan2(pts[:, 1].astype(LD), pts[:, 0].astype(LD)).astype(np.float64)
    exact = (pts[:, 1] == 0) & (pts[:, 0] > 0)   # atan2(+-0, x > 0) is +-0 exactly (C99 F.9.1.4, and CUDA's atan2)
    cand = np.empty((n, 2 * ULPS + 1), np.int64)
    rnr = np.zeros((n, 2 * ULPS + 1), bool)
    use_rnr = bool(p.enable_RNR) and pts.shape[1] >= 4
    if use_rnr:
        xf, yf = pts[:, 0], pts[:, 1]
        rf = np.sqrt(xf * xf + yf * yf)   # float32, as S:387
        pre = (pts[:, 3].astype(np.float64) < p.RNR_intensity_thr) & (z < -p.sensor_height - 0.8)
        vang = np.arctan2(pts[:, 2].astype(LD), rf.astype(LD)).astype(np.float64)
    for j in range(-ULPS, ULPS + 1):
        t = np.where(exact, theta, _steps(theta, j))
        t = np.where(t > 0, t, 2 * np.pi + t)
        sec = np.minimum((t / ss).astype(np.int64), ns - 1)
        cand[:, j + ULPS] = np.where(inr, base + ring * ns + sec, g.nbins + 1)
        if use_rnr:
            rnr[:, j + ULPS] = pre & ((_steps(vang, j) * 180.0) / np.pi < p.RNR_ver_angle_thr)
    return cand, rnr


def _check_bins(ids_dev, ids_orc, cand, rnr, nb, what):
    """Bit-exact outside the libm-defined band; inside it, one of the bins the band's angles give. Returns (band, differ)."""
    any_r, all_r = rnr.any(1), rnr.all(1)
    polar_vary = (cand != cand[:, :1]).any(1)
    band = (any_r & ~all_r) | (~all_r & polar_vary)
    model = np.where(rnr[:, ULPS], nb, cand[:, ULPS])
    # the model itself: equal to the oracle wherever the band's angles agree
    assert np.array_equal(model[~band], ids_orc[~band]), f"{what}: the numpy model disagrees with the oracle outside the band"
    out = ~band & (ids_dev != ids_orc)
    assert not out.any(), f"{what}: {int(out.sum())} bin ids differ outside the libm-defined band (first {np.nonzero(out)[0][:5]})"

    def allowed(ids):
        return (any_r & (ids == nb)) | (~all_r & (cand == ids[:, None].astype(np.int64)).any(1))
    assert allowed(ids_orc)[band].all(), f"{what}: the oracle's bin is not among the band's bins"
    ok = allowed(ids_dev)
    assert ok[band].all(), f"{what}: {int((~ok & band).sum())} band points in a bin no angle within {ULPS} ulp gives"
    # (4 ulp of an angle is far less than a sector: the bins a band point may take are one sector apart in one ring)
    return int(band.sum()), int((band & (ids_dev != ids_orc)).sum())


# ---- boundary point generator -------------------------------------------------------------------------------------------
RADIAL_OFFSETS = (0.0, 1e-7, -1e-7, 1e-5, -1e-5, 1.5e-4, -1.5e-4, 1.9e-4, -1.9e-4, 2.1e-4, -2.1e-4, 3e-4, -3e-4)
ANGULAR_OFFSETS = (0.0, 1e-8, -1e-8, 1e-6, -1e-6)


def _polar(r, th):
    r, th = np.asarray(r, np.float64), np.asarray(th, np.float64)
    return np.c_[r * np.cos(th), r * np.sin(th)].astype(np.float32)


def _toward(sign):
    """float32 +-inf per element (nextafter must step in float32, not in the double a mixed-type call would promote to)."""
    return np.where(sign > 0, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32)


def _nudge_radius(xy, s):
    """Both coordinates one float ulp away from (s = +1) or towards (s = -1) the origin."""
    return np.c_[np.nextafter(xy[:, 0], _toward(np.where(xy[:, 0] >= 0, s, -s))),
                 np.nextafter(xy[:, 1], _toward(np.where(xy[:, 1] >= 0, s, -s)))].astype(np.float32)


def _nudge_angle(xy, s):
    """One coordinate one float ulp in the direction that turns the point by s (counter-clockwise for s = +1)."""
    x, y = xy[:, 0].copy(), xy[:, 1].copy()
    wide = np.abs(x) >= np.abs(y)
    y = np.where(wide, np.nextafter(y, _toward(np.where(x >= 0, s, -s))), y)
    x = np.where(wide, x, np.nextafter(x, _toward(np.where(y >= 0, -s, s))))
    return np.c_[x, y].astype(np.float32)


def _lattice_walk(g, width=256):
    """For every sector boundary k * sector_size of every zone, at the middle of the zone's first ring: walk `width` floats
    of the larger coordinate and take, for each, the two floats of the other coordinate around the boundary ray; keep the
    two pairs whose exact angle lies closest to the boundary. These are where a last-ulp atan2 difference moves a bin."""
    out = []
    for k in range(4):
        r = g.mins[k] + 0.5 * g.rs[k]
        for s in range(g.ns[k]):
            phi = LD(s) * LD(g.ss[k])
            c, sn = np.cos(phi), np.sin(phi)
            wide = abs(c) >= abs(sn)
            a0 = np.float32(r * (c if wide else sn))
            a = np.array([a0], np.float32)
            walk = [a0]
            lo = hi = a
            for _ in range(width // 2):
                lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
                walk += [lo[0], hi[0]]
            a = np.array(walk, np.float32)
            b_ideal = a.astype(LD) * (sn / c if wide else c / sn)
            b1 = b_ideal.astype(np.float32)
            b = np.r_[b1, np.nextafter(b1, _toward(np.where(b_ideal > b1.astype(LD), 1, -1)))]
            aa = np.r_[a, a]
            xy = np.c_[aa, b] if wide else np.c_[b, aa]
            ang = np.arctan2(xy[:, 1].astype(LD), xy[:, 0].astype(LD))
            ang = np.where(ang < 0, ang + 2 * PI_LD, ang)
            dist = np.abs(ang - phi)
            if s == 0:
                dist = np.minimum(dist, np.abs(ang - 2 * PI_LD))
            out.append(xy[np.argsort(dist)[:2]])
    return np.concatenate(out).astype(np.float32)


def _exact_rays(g):
    """Points on the axes and the diagonals (signed zeros included): the sector boundaries that are representable angles."""
    pts = []
    for k in range(4):
        a = np.float32((g.mins[k] + 0.5 * g.rs[k]) / np.sqrt(2.0))
        b = np.float32(g.mins[k] + 0.5 * g.rs[k])
        pts += [[a, a], [-a, a], [-a, -a], [a, -a], [b, 0.0], [b, -0.0], [-b, 0.0], [-b, -0.0], [0.0, b], [-0.0, b], [0.0, -b], [-0.0, -b]]
    return np.array(pts, np.float32)


def _rnr_points(p, rng):
    """Intensity straddling RNR_intensity_thr, z straddling -sensor_height - 0.8, vertical angle straddling RNR_ver_angle_thr
    (at random azimuths, so that no bin holds a stack of them)."""
    f = np.float32
    it0 = f(p.RNR_intensity_thr)
    its = [np.nextafter(it0, f(-1)), it0, np.nextafter(it0, f(1)), f(0.05)]
    z0 = f(-p.sensor_height - 0.8)
    zs = [np.nextafter(z0, f(-9)), z0, np.nextafter(z0, f(9)), z0 - f(1e-5), z0 + f(1e-5), f(-3.0), f(-2.9)]
    out = []
    tan = np.tan(np.deg2rad(-p.RNR_ver_angle_thr))
    for z in zs:
        r0 = f(-float(z) / tan)
        rr = [r0]
        lo = hi = np.array([r0], f)
        for _ in range(3):
            lo, hi = np.nextafter(lo, f(0)), np.nextafter(hi, f(1e9))
            rr += [lo[0], hi[0]]
        rr += [r0 * f(1 + 1e-5), r0 * f(1 - 1e-5), r0 * f(1.001), r0 * f(0.999)]
        for r in rr:
            for it in its:
                for _ in range(2):
                    xy = _polar([r], [rng.uniform(0, 2 * np.pi)])[0]
                    out.append([xy[0], xy[1], z, it])
    return np.array(out, np.float32)


def _boundary_points(g, p, rng):
    """Points on and beside every decision boundary (z ~ ground, intensity 0.5), then the RNR points, then the points whose
    exact angle is closest to a sector boundary (last: they are the ones that may lie in the band)."""
    parts = []
    angles = (np.arange(24) + 0.37) * (2 * np.pi / 24)
    for rb in g.ring_bounds():          # ring, zone and range limits
        for dr in RADIAL_OFFSETS:
            parts.append(_polar(np.full(len(angles), rb + dr), angles))
        on = _polar(np.full(len(angles), rb), angles)
        parts += [_nudge_radius(on, 1), _nudge_radius(on, -1)]
    for k in range(4):                  # sector limits at every ring's middle
        for ring in range(g.nr[k]):
            r = g.mins[k] + (ring + 0.5) * g.rs[k]
            th = np.arange(g.ns[k]) * g.ss[k]
            for dth in ANGULAR_OFFSETS + (1.9e-4 * g.ss[k], -1.9e-4 * g.ss[k], 2.1e-4 * g.ss[k], -2.1e-4 * g.ss[k]):
                parts.append(_polar(np.full(len(th), r), th + dth))
            on = _polar(np.full(len(th), r), th)
            parts += [_nudge_angle(on, 1), _nudge_angle(on, -1)]
    xy = np.concatenate(parts)
    body = np.c_[xy, -1.7 + rng.normal(0, 0.02, len(xy)), np.full(len(xy), 0.5)].astype(np.float32)
    tail = np.concatenate([_exact_rays(g), _lattice_walk(g)])
    tail = np.c_[tail, -1.7 + rng.normal(0, 0.02, len(tail)), np.full(len(tail), 0.5)].astype(np.float32)
    return np.concatenate([body, _rnr_points(p, rng), tail])


def _cloud(g, n, rng):
    """Scattered ground points over the whole range (every bin gets a well-conditioned plane)."""
    r = rng.uniform(g.min_range + 0.01, g.max_range - 0.01, n)
    th = rng.uniform(0, 2 * np.pi, n)
    return np.c_[_polar(r, th), -1.7 + rng.normal(0, 0.03, n), rng.uniform(0.3, 1.0, n)].astype(np.float32)


def _geometries():
    def mk(max_range=None, min_range=None, rings=None, sectors=None):
        p = default_params()
        if max_range is not None:
            p.max_range = max_range
        if min_range is not None:
            p.min_range = min_range
        if rings is not None:
            p.num_rings_each_zone[:] = rings
        if sectors is not None:
            p.num_sectors_each_zone[:] = sectors
        return p
    return {
        "default": (mk(), True),
        "range250_128sectors": (mk(max_range=250.0, sectors=[16, 32, 128, 32]), True),
        "narrow_rings": (mk(min_range=5.0, max_range=40.0, rings=[5, 1, 2, 3], sectors=[32, 54, 32, 32]), False),
        "129sectors": (mk(sectors=[16, 32, 129, 32]), False),
    }


GEOMETRIES = _geometries()


@pytest.mark.parametrize("gname", list(GEOMETRIES))
def test_binning_at_every_decision_boundary(gname):
    import pwpp_b200
    small = _assert_default_switches()
    p, fast = GEOMETRIES[gname]
    g = Geom(p)
    assert g.fast == fast, f"{gname}: build_geometry would bin with the {'fp32 filter' if g.fast else 'exact path'}"
    # pwpp_create keeps the cluster front end, and its dense variant, only where their shared memory fits in 220 KB
    assert g.front_smem(256) <= 220 * 1024 and g.front_smem(512) <= 220 * 1024
    rng = np.random.default_rng(20261016)
    pts = _boundary_points(g, p, rng)
    shapes = {
        # one frame: k_bin_hist<FAST> + k_bin_scan + k_scatter
        "one_frame": [np.concatenate([pts, _cloud(g, 40_000, rng)])],
        # six frames: k_front_cluster<FAST, 4096, 256>
        "batch6": [np.concatenate([part, _cloud(g, 40_000, rng)]) for part in np.array_split(pts, 6)],
        # five frames of > 400k points: k_front_cluster<FAST, 4096, 512>
        "dense5": [np.concatenate([part, _cloud(g, 410_000 - len(part), rng)]) for part in np.array_split(pts, 5)],
    }
    assert len(shapes["one_frame"]) <= small
    assert len(shapes["batch6"]) > small and np.mean([len(a) for a in shapes["batch6"]]) <= DENSE_MEAN
    assert len(shapes["dense5"]) > small and np.mean([len(a) for a in shapes["dense5"]]) > DENSE_MEAN
    for shape, frames in shapes.items():
        _assert_one_launch_range(frames)
        eng = pwpp_b200.Engine(p, device=0, num_streams=len(frames))
        assert eng.nbins == g.nbins
        eng.estimate_host(frames)
        band_n = differ_n = compared = 0
        for f, a in enumerate(frames):
            orc = O.Oracle(p, O.ARITH_CANON64)
            orc.estimate(a)
            ids_o, ids_e = orc.bin_ids(), eng.bin_ids(f)
            cand, rnr = _model_bins(a, p, g)
            b, d = _check_bins(ids_e, ids_o, cand, rnr, g.nbins, f"{gname}/{shape}/{f}")
            band_n += b
            differ_n += d
            if d == 0:   # bins identical (in particular every frame without a band point): the whole frame
                compare_frame(eng, f, orc, a, f"{gname}/{shape}/{f}")
                compared += 1
        assert compared == len(frames) or differ_n > 0
        line = f"binning {gname} ({'fp32 filter' if fast else 'exact'}) {shape}: {sum(len(a) for a in frames)} points, " \
               f"{band_n} in the libm-defined band, {differ_n} of them binned differently from the oracle; {compared}/{len(frames)} frames fully compared"
        print(line)
        eng.close()


# ---- fit and sort kernels at their size limits -------------------------------------------------------------------------
def _class_of(n):
    for c, m in enumerate(CLASS_MAX):
        if n <= m:
            return c
    return 5


def _patch(g, zone, ring, sector, n, z, rng):
    r = g.mins[zone] + (ring + 0.2 + 0.6 * rng.random(n)) * g.rs[zone]
    th = (sector + 0.2 + 0.6 * rng.random(n)) * g.ss[zone]
    return np.c_[_polar(r, th), z, rng.uniform(0.3, 1.0, n)].astype(np.float32)


def _patch_frames():
    """Ten frames of one or a few patches each (distinct bins), padded with points inside min_range (out of range) to frame
    sizes on and beside multiples of k_emit's tiles (1024 positions per warp, 8192 per CTA). Returns [(frame, [(bin, n)])]."""
    rng = np.random.default_rng(7)
    g = Geom(default_params())

    def gauss(n): return -1.7 + rng.normal(0, 0.03, n)
    def cm(n): return np.round((-1.7 + rng.normal(0, 0.05, n)) / 0.01) * 0.01     # thousands of exact ties
    def signed_zero(n):    # a ground plane at z = 0: ~a third of the points are +0.0 or -0.0
        v = np.round(rng.normal(0, 0.02, n) / 0.01) * 0.01
        v[v == 0] = np.where(rng.random(int((v == 0).sum())) < 0.5, -0.0, 0.0)
        return v
    def flat(n): return np.full(n, -1.723)
    def two_level(n): return np.where(rng.random(n) < 0.6, -1.75, -1.70)

    layout = [   # (target frame size, [(n, shape)])
        (1023, [(15, gauss), (16, gauss), (17, gauss), (31, gauss), (33, gauss), (64, gauss), (65, gauss), (255, gauss), (256, gauss), (257, gauss)]),
        (2049, [(511, gauss), (512, gauss), (513, gauss), (64, cm), (65, cm), (17, signed_zero)]),
        (8191, [(1023, gauss), (1025, gauss), (2048, gauss), (2049, gauss), (257, signed_zero), (512, cm), (513, cm)]),
        (8193, [(4096, gauss), (4097, gauss)]),
        (8192, [(8192, gauss)]),
        (16385, [(8193, gauss), (2049, cm), (4096, signed_zero)]),
        (16384, [(12000, gauss), (4097, cm)]),
        (24578, [(16385, gauss), (8193, cm)]),
        (32769, [(20000, gauss), (12000, cm)]),
        (32768, [(9000, flat), (9000, two_level), (1025, signed_zero)]),
    ]
    frames = []
    for f, (target, specs) in enumerate(layout):
        parts, placed, used = [], [], set()
        for j, (n, shape) in enumerate(specs):
            zone = (j + f) % 4
            ring = (j // 4 + f) % g.nr[zone]
            sector = (3 * j + 5 * f + 1) % g.ns[zone]
            b = g.bin_of(zone, ring, sector)
            assert b not in used and b != 0
            used.add(b)
            parts.append(_patch(g, zone, ring, sector, n, shape(n), rng))
            placed.append((b, n))
        if f == len(layout) - 1:   # a zone-0 wall: R-VPF removes points over several iterations (bin 0)
            wall = np.r_[np.c_[4 + rng.random(6000) * 0.05, rng.random(6000) * 0.6, -1.7 + rng.random(6000) * 2.0, rng.random(6000)],
                         np.c_[3 + rng.random(6000) * 4, rng.random(6000) * 0.6, -1.7 + rng.normal(0, 0.02, 6000), rng.random(6000)]]
            parts.append(wall.astype(np.float32))
            placed.append((0, 12000))
        n_pad = target - sum(len(q) for q in parts)
        assert n_pad >= 0
        rad = rng.uniform(0.3, 2.5, n_pad)
        parts.append(np.c_[_polar(rad, rng.uniform(0, 2 * np.pi, n_pad)), -1.7 + rng.normal(0, 0.03, n_pad), rng.random(n_pad)].astype(np.float32))
        a = np.concatenate(parts)
        a = a[rng.permutation(len(a))]   # patches interleaved in input order: the stable scatter and the sorts see mixed indices
        frames.append((np.ascontiguousarray(a), placed))
    return frames


@pytest.fixture(scope="module")
def patch_case():
    frames = _patch_frames()
    fresh = []
    for a, _ in frames:
        o = O.Oracle(arith=O.ARITH_CANON64)
        o.estimate(a)
        fresh.append(o)
    return frames, fresh


def _assert_bin_order(ge, go, ids, what):
    """Native order (test_emission_order_is_bin_major): the oracle's sequence of bins, each bin's indices ascending."""
    def runs(idx):
        b = ids[idx]
        cut = np.nonzero(np.diff(b))[0] + 1
        return [np.sort(x) for x in np.split(idx, cut)], (list(b[np.r_[0, cut]]) if len(idx) else [])
    re_, be_ = runs(ge)
    ro_, bo_ = runs(go)
    assert be_ == bo_, f"{what}: bins in another order"
    assert all(np.array_equal(x, y) for x, y in zip(re_, ro_)), f"{what}: a bin holds other points"
    return [x for x in np.split(ge, np.nonzero(np.diff(ids[ge]))[0] + 1)]


def _check_patch_frame(eng, f, orc, a, placed, order, what, counts):
    nd = compare_frame(eng, f, orc, a, what)
    assert nd == 0, f"{what}: {nd} degenerate patches"
    be, bo = eng.bin_results(f), orc.bin_results()
    for b, n in placed:
        assert be[b].n == n and bo[b].n == n, f"{what}: bin {b} holds {be[b].n} points, {n} intended"
    g_e, ng_e = eng.ground_indices(f), eng.nonground_indices(f)
    g_o, ng_o = orc.getGroundIndices(), orc.getNongroundIndices()
    if order:   # reference order: the oracle sorts each bin stably, so its lists are the reference's lists with stable ties
        assert np.array_equal(g_e, g_o), f"{what}: ground list differs from the oracle's"
        assert np.array_equal(ng_e, ng_o), f"{what}: non-ground list differs from the oracle's"
    else:
        ids = orc.bin_ids().astype(np.int64)
        for x in _assert_bin_order(g_e, g_o, ids, what + "/ground"):
            assert (np.diff(x) > 0).all(), f"{what}: ground indices of a bin not ascending"
        for x in _assert_bin_order(ng_e, ng_o, ids, what + "/nonground"):
            assert int((np.diff(x) <= 0).sum()) <= 1, f"{what}: non-ground indices of a bin not in two ascending pieces"
    for b in range(orc.nbins):
        if bo[b].fitted and bo[b].n > 0:
            counts[_class_of(bo[b].n)] += 1


@pytest.mark.parametrize("order", [0, 1], ids=["bin_order", "reference_order"])
def test_fit_and_sort_kernels_at_size_limits(patch_case, order):
    """Batch call (k_fit_resident, k_fit_warp<true/false>, k_fit_cta<4096/8192>, k_fit_big), one-frame calls (k_fit_patch
    <4,4,2> / <8,2,3> / <16,1,4> above 512 points; each frame twice, the second call replaying the captured graph) and one
    call that names stream 0 twice (a batch run, then a one-frame run). In reference order also k_order_warp,
    k_order_cta<128,2> / <256,3> / <512,4> and <512,5>, whose patches above 8192 keys sort in global memory."""
    import pwpp_b200
    small = _assert_default_switches()
    frames, fresh = patch_case
    pts = [a for a, _ in frames]
    nf = len(frames)
    assert nf > small   # the batch kernel set
    _assert_one_launch_range(pts)
    counts = {path: [0] * 6 for path in ("batch", "one_frame", "one_frame_replay", "mixed")}
    # sizes on both sides of every limit reach their classes (and, in reference order, their sorts)
    sizes = sorted({n for _, pl in frames for _, n in pl})
    for lim in CLASS_MAX:
        assert lim in sizes and lim + 1 in sizes
    assert all(n in sizes for n in (15, 16, 17, 31, 33, 255, 256, 257, 511, 512, 513, 1023, 1025, 12000, 16385, 20000))

    eng = pwpp_b200.Engine(num_streams=nf)
    eng.set_output_order(order)
    eng.estimate_host(pts)
    for f, (a, placed) in enumerate(frames):
        _check_patch_frame(eng, f, fresh[f], a, placed, order, f"batch/{f}", counts["batch"])
    eng.close()

    eng = pwpp_b200.Engine()
    eng.set_output_order(order)
    for f, (a, placed) in enumerate(frames):
        for call, path in enumerate(("one_frame", "one_frame_replay")):
            # the same frame twice from the same state: the second call's graph key (frames, frames of the call, intensity,
            # grid size, buffer generation, input buffer) equals the first's, so it replays the graph the first captured
            eng.reset()
            eng.estimate_host([a])
            _check_patch_frame(eng, 0, fresh[f], a, placed, order, f"{path}/{f}", counts[path])
    eng.close()

    # streams 0..nf-2, then stream 0 again: a run of nf-1 frames (batch kernels), then a run of one frame (small-call kernels)
    streams = list(range(nf - 1)) + [0]
    assert nf - 1 > small
    eng = pwpp_b200.Engine(num_streams=nf)
    eng.set_output_order(order)
    eng.estimate_host(pts, streams=streams)
    for f in range(nf - 1):
        _check_patch_frame(eng, f, fresh[f], pts[f], frames[f][1], order, f"mixed/{f}", counts["mixed"])
    seq = O.Oracle(arith=O.ARITH_CANON64)
    seq.estimate(pts[0])
    seq.estimate(pts[nf - 1])
    _check_patch_frame(eng, nf - 1, seq, pts[nf - 1], frames[nf - 1][1], order, "mixed/second frame of stream 0", counts["mixed"])
    eng.close()

    mode = ("bin", "reference")[order]
    for path, c in counts.items():
        print(f"fit/sort {mode} order, {path}: fully compared patches per class " + ", ".join(f"{CLASS_NAMES[i]} {c[i]}" for i in range(6)))
        # every class from S to X received patches, on every path
        assert all(v > 0 for v in c), (path, c)
    assert counts["batch"] == counts["one_frame"] == counts["one_frame_replay"]
