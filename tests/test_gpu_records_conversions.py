"""Field values through the real records entry points (pwpp_estimate_host_records and pwpp_estimate_device_records) on the GPU.

- xyz: FLOAT64 x, y, z at float rounding edges (exact ties, one double ulp either side of a tie, values that become float
  subnormals or -0). The xyz getters must return numpy's astype(np.float32) of them bit for bit, and a non-finite coordinate
  or one beyond the float range must send its point to the out-of-range pseudo-bin.
- intensity in the sensor's own units around RNR_intensity_thr: eight parameter sets in one context, one stream each, with
  thresholds from 0.2 to 2^32 - 0.5, among them thresholds whose nearest float lies below them. Every integer datatype, FLOAT32
  and FLOAT64 carries values around each threshold. The bin ids carry the RNR verdict (the RNR pseudo-bin) and must equal the
  CANON64 oracle's, run with the stream's set on the numpy-converted N x 4 array, in a fresh call and in a second call."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

INT8, UINT8, INT16, UINT16, INT32, UINT32, FLOAT32, FLOAT64 = range(1, 9)
DT = {INT8: np.int8, UINT8: np.uint8, INT16: np.int16, UINT16: np.uint16, INT32: np.int32, UINT32: np.uint32, FLOAT32: np.float32,
      FLOAT64: np.float64}
RNR_THRESHOLDS = [0.2, 13107.0, 32767.5, 32768.001, 40000.001, 70000.003, 2.0 ** 24 + 3, 4294967295.5]


def run(eng, path, recs, streams=None):
    """One records call of the structured arrays recs through the host or the device entry point."""
    if path == "host":
        eng.estimate_host_records(recs, streams=streams)
        return
    import torch
    import pwpp_b200
    bufs = [torch.from_numpy(r.view(np.uint8).copy()).cuda() for r in recs]
    torch.cuda.synchronize()
    eng.estimate_device_records([b.data_ptr() for b in bufs], [len(r) for r in recs], [pwpp_b200.layout_from_dtype(r.dtype) for r in recs],
                                streams=streams)
    eng.synchronize()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def ties(rng, lo, hi, n):
    """Doubles exactly halfway between two adjacent floats of [lo, hi) (half of them above a float with an even significand,
    so both directions of round-half-even occur), and the doubles one ulp below and above each."""
    f = rng.uniform(lo, hi, n).astype(np.float32)
    t = (f.astype(np.float64) + np.nextafter(f, np.float32(np.inf)).astype(np.float64)) / 2   # exact in double
    return np.concatenate([t, np.nextafter(t, -np.inf), np.nextafter(t, np.inf)])


XYZ_DT = np.dtype({"names": ["intensity", "x", "y", "z"], "formats": ["<f4", "<f8", "<f8", "<f8"], "offsets": [0, 4, 12, 20], "itemsize": 28})


def xyz_frame(rng):
    """In-range points at rounding edges, then points with one non-finite or huge coordinate (their indices returned)."""
    n = 1500
    x, y, z = ties(rng, 3.0, 60.0, n), ties(rng, -30.0, 30.0, n), ties(rng, -2.2, 0.4, n)
    rng.shuffle(x); rng.shuffle(y)
    tiny = [2.0 ** -150, -(2.0 ** -150), 3 * 2.0 ** -150, 1.5 * 2.0 ** -149, 1e-40, -1e-40, 1e-45, 7e-46, -7e-46, 1e-50, -1e-50,
            -0.0, 0.0, 2.0 ** -126 * (1 - 2.0 ** -25), -(2.0 ** -126) * (1 - 2.0 ** -24)]   # float subnormals, ties, -0, FLT_MIN
    m = len(tiny)
    x = np.r_[x, ties(rng, 5.0, 9.0, m)[:m], np.full(m, 11.0)]
    y = np.r_[y, tiny, ties(rng, 1.0, 2.0, m)[:m]]
    z = np.r_[z, np.full(m, -1.7), tiny]
    nan_p, nan_n = np.array([0x7FF0000000000001, 0xFFFA5A5A5A5A5A5A], np.uint64).view(np.float64)
    bad = [(nan_p, 4.0, -1.7), (np.inf, 4.0, -1.7), (-np.inf, 4.0, -1.7), (1e300, 4.0, -1.7), (-1e300, 4.0, -1.7), (6.0, nan_n, -1.7),
           (6.0, 1e300, -1.7), (6.0, -np.inf, -1.7), (6.0, 3.5e38, -1.7), (6.0, 4.0, nan_p), (6.0, 4.0, np.inf), (6.0, 4.0, -np.inf),
           (6.0, 4.0, 1e300), (6.0, 4.0, -1e300), (6.0, 4.0, 3.4028235677973366e38 * 1.0000001)]
    k = len(x)
    x, y, z = np.r_[x, [b[0] for b in bad]], np.r_[y, [b[1] for b in bad]], np.r_[z, [b[2] for b in bad]]
    r = np.zeros(len(x), XYZ_DT)
    r["x"], r["y"], r["z"], r["intensity"] = x, y, z, 1.0   # (intensity above RNR_intensity_thr: no reflected noise)
    return r, np.arange(k, len(x))


@pytest.mark.parametrize("path", ["host", "device"])
def test_float64_xyz_rounding_edges_and_non_finite_coordinates(path):
    import oracle_py as O
    import pwpp_b200
    rng = np.random.default_rng(21)
    eng = pwpp_b200.Engine(device=0, num_streams=1)
    orc = O.Oracle(arith=O.ARITH_CANON64)
    for call in range(2):
        r, bad = xyz_frame(rng)
        with np.errstate(over="ignore", invalid="ignore"):
            eq = np.ascontiguousarray(np.stack([r[c].astype(np.float32) for c in ("x", "y", "z", "intensity")], axis=1))
        assert (eq[:len(r) - len(bad), :3].view(np.uint32) & 0x7F800000 == 0).any()   # subnormals and zeros among the in-range points
        drop = eq[:, 2] == np.finfo(np.float32).tiny   # a z that rounds to FLT_MIN: the point leaves both lists (S:591)
        assert drop.sum() == 1
        run(eng, path, [r])
        gi, ni = eng.ground_indices(0), eng.nonground_indices(0)
        assert len(gi) + len(ni) == len(r) - 1 and not drop[gi].any() and not drop[ni].any()
        for what, idx, got in (("ground", gi, eng.ground_xyz(0)), ("non-ground", ni, eng.nonground_xyz(0))):
            want = eq[idx, :3]
            diff = np.argwhere(bits(got) != bits(want))
            assert diff.size == 0, f"call {call}: {what} point {idx[diff[0][0]]}: got {got[tuple(diff[0])]!r} want {want[tuple(diff[0])]!r}"
        ids = eng.bin_ids(0)
        assert (ids[bad] == eng.nbins + 1).all(), f"call {call}: non-finite or huge coordinates outside the out-of-range pseudo-bin"
        orc.estimate(eq)
        assert np.array_equal(ids, orc.bin_ids()), f"call {call}: bin ids differ from the oracle"


def intensities(code, thr):
    """Values of a datatype around thr: for integers the ones from floor(thr) - 2 to ceil(thr) + 2, for floats the floats within
    4 ulp of thr (and, FLOAT64, thr itself, its neighbouring doubles and the halfway points to the neighbouring floats), plus
    the type's extremes, integers that round to float (2^24 + 1, 2^24 + 3, 2^32 - 1, ...), and non-finite values."""
    t = np.dtype(DT[code])
    rounding = [2 ** 24 + 1, 2 ** 24 + 2, 2 ** 24 + 3, 2 ** 24 + 5, 2 ** 31 - 1, 2 ** 31 - 65, 2 ** 31 + 129, 2 ** 32 - 1, 2 ** 32 - 129,
                32767, 32768, 40000, 40001, 65535, 70000, 70003, 13107, 255, 127, 0, 1]
    if t.kind in "iu":
        info = np.iinfo(t)
        v = [np.floor(thr) + d for d in range(-2, 1)] + [np.ceil(thr) + d for d in range(0, 3)] + rounding + [info.min, info.max, -1, -2 ** 24 - 3]
        return np.unique(np.array([int(a) for a in v if info.min <= a <= info.max], dtype=t))
    f = np.float32(thr)
    near = [f]
    lo = hi = f
    for _ in range(4):
        lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
        near += [lo, hi]
    near = np.sort(np.array(near, np.float32))
    special = [np.nan, np.inf, -np.inf, -0.0, -1.0, float(np.finfo(np.float32).max)]
    if t == np.float32:
        return np.r_[near, np.array(rounding + special, np.float32)]
    half = (near[:-1].astype(np.float64) + near[1:].astype(np.float64)) / 2   # halfway between neighbouring floats
    return np.r_[near.astype(np.float64), half, [thr, np.nextafter(thr, -np.inf), np.nextafter(thr, np.inf)], np.array(rounding, np.float64),
                 special, [1e300, -1e300]]


def rnr_frame(rng, code, thr):
    """Each intensity value on three points in RNR geometry: 3 to 8 m out and 4.5 m down, far below -sensor_height - 0.8 and
    steeper than RNR_ver_angle_thr, so the intensity alone decides the verdict."""
    v = np.repeat(intensities(code, thr), 3)
    rng.shuffle(v)
    dt = np.dtype({"names": ["x", "y", "z", "intensity"], "formats": ["<f4", "<f4", "<f4", np.dtype(DT[code]).newbyteorder("<")],
                   "offsets": [0, 4, 8, 13], "itemsize": 24})
    r = np.zeros(len(v), dt)
    r["x"], r["y"], r["z"], r["intensity"] = rng.uniform(3, 8, len(v)), rng.uniform(-2, 2, len(v)), -4.5, v
    with np.errstate(over="ignore", invalid="ignore"):
        eq = np.ascontiguousarray(np.stack([r[c].astype(np.float32) for c in ("x", "y", "z", "intensity")], axis=1))
    return r, eq


@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("code", list(DT), ids=[np.dtype(DT[c]).name for c in DT])
def test_intensity_around_rnr_threshold_of_every_set(code, path):
    import oracle_py as O
    import pwpp_b200
    sets = []
    for thr in RNR_THRESHOLDS:
        p = pwpp_b200.default_params()
        p.RNR_intensity_thr = thr
        sets.append(p)
    eng = pwpp_b200.Engine(params=sets, stream_set=list(range(8)), num_streams=8)
    orcs = [O.Oracle(p, O.ARITH_CANON64) for p in sets]
    rng = np.random.default_rng(code)
    data = [rnr_frame(rng, code, thr) for thr in RNR_THRESHOLDS]
    streams = [3, 0, 7, 5, 1, 6, 2, 4]
    hits = 0
    for call in ("fresh", "second"):
        run(eng, path, [data[s][0] for s in streams], streams=streams)
        for f, s in enumerate(streams):
            orcs[s].estimate(data[s][1])
            want = orcs[s].bin_ids()
            got = eng.bin_ids(f)
            bad = np.nonzero(got != want)[0]
            assert bad.size == 0, (f"{call} call, threshold {RNR_THRESHOLDS[s]!r}: {bad.size} bin ids differ from the oracle, first "
                                   f"intensity {data[s][1][bad[0], 3]!r}: got bin {got[bad[0]]}, oracle {want[bad[0]]} (RNR pseudo-bin {orcs[s].nbins})")
            hits += int((want == orcs[s].nbins).sum())
    assert hits > 0
