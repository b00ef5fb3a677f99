"""RNR's intensity test (rnr_hit, csrc/pwpp_math.cuh) with RNR_intensity_thr in a sensor's raw units, on the CPU: the twin
(tests/host_twin.cu) and the kernels through the SIMT stand-in, against the oracle (CANON64)."""
import numpy as np
import pytest

import oracle_py as O
from helpers import SimtTwin, Twin


@pytest.mark.parametrize("thr", [0.2, 13107.0, 32767.5, 32768.001, 40000.001, 70000.003, 2.0 ** 24 + 3, 4294967295.5])
def test_rnr_intensity_threshold_in_sensor_units(thr):
    """Intensities in a sensor's raw units (UINT16 / UINT32 counts) with RNR_intensity_thr in the same units: points in RNR
    geometry (3 to 8 m out, 4.5 m down) whose intensity is every float within 4 ulp of the threshold, or an integer next to it.
    rnr_hit must mark exactly the points with (double) intensity < RNR_intensity_thr, like the oracle. Regression: its fp32
    pre-filter `intensity < (float) thr + 1e-3f` rejected 40000 against 40000.001, where (float) thr rounds down and the 1e-3
    is absorbed (also 32768.001 and 70000.003)."""
    from pwpp_ctypes import default_params
    p = default_params()
    p.RNR_intensity_thr = thr
    f = np.float32(thr)
    its = [f]
    lo = hi = f
    for _ in range(4):
        lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
        its += [lo, hi]
    its += [np.float32(v) for v in (np.floor(thr) - 1, np.floor(thr), np.ceil(thr), np.ceil(thr) + 1, 0.0, np.nan)]
    rng = np.random.default_rng(int(thr) % 1000)
    it = np.repeat(np.array(its, np.float32), 4)
    a = np.stack([rng.uniform(3, 8, len(it)), rng.uniform(-2, 2, len(it)), np.full(len(it), -4.5), it], axis=1).astype(np.float32)
    orc = O.Oracle(p, O.ARITH_CANON64)
    orc.estimate(a)
    want = orc.bin_ids()
    rnr = want == orc.nbins
    assert np.array_equal(rnr, a[:, 3].astype(np.float64) < thr)   # (the geometry leaves the verdict to the intensity)
    for impl in (Twin(p), SimtTwin(p)):
        impl.estimate(a)
        got = impl.bin_ids()
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, f"{type(impl).__name__}: intensity {a[bad[0], 3]!r} against {thr!r}: bin {got[bad[0]]}, oracle {want[bad[0]]}"
