"""ctypes mirrors of the PODs in include/pwpp.h (shared by the product wrapper and the test oracles)."""
import ctypes as C

NUM_ZONES = 4


class PwppParams(C.Structure):
    """Mirror of `pwpp_params` (include/pwpp.h), itself a POD mirror of patchwork::Params
    (reference cpp/patchworkpp/include/patchwork/patchworkpp.h:42-112)."""
    _fields_ = [
        ("verbose", C.c_int32), ("enable_RNR", C.c_int32), ("enable_RVPF", C.c_int32), ("enable_TGR", C.c_int32),
        ("num_iter", C.c_int32), ("num_lpr", C.c_int32), ("num_min_pts", C.c_int32), ("num_zones", C.c_int32),
        ("num_rings_of_interest", C.c_int32), ("max_flatness_storage", C.c_int32),
        ("max_elevation_storage", C.c_int32), ("_pad0", C.c_int32),
        ("RNR_ver_angle_thr", C.c_double), ("RNR_intensity_thr", C.c_double), ("sensor_height", C.c_double),
        ("th_seeds", C.c_double), ("th_dist", C.c_double), ("th_seeds_v", C.c_double), ("th_dist_v", C.c_double),
        ("max_range", C.c_double), ("min_range", C.c_double), ("uprightness_thr", C.c_double),
        ("adaptive_seed_selection_margin", C.c_double), ("intensity_thr", C.c_double),
        ("num_sectors_each_zone", C.c_int32 * 4), ("num_rings_each_zone", C.c_int32 * 4),
        ("elevation_thr", C.c_double * 4), ("flatness_thr", C.c_double * 4),
    ]


def default_params() -> PwppParams:
    """Reference defaults, patchworkpp.h:79-111."""
    p = PwppParams()
    p.verbose = 0; p.enable_RNR = 1; p.enable_RVPF = 1; p.enable_TGR = 1
    p.num_iter = 3; p.num_lpr = 20; p.num_min_pts = 10; p.num_zones = 4; p.num_rings_of_interest = 4
    p.max_flatness_storage = 1000; p.max_elevation_storage = 1000
    p.RNR_ver_angle_thr = -15.0; p.RNR_intensity_thr = 0.2; p.sensor_height = 1.723
    p.th_seeds = 0.125; p.th_dist = 0.125; p.th_seeds_v = 0.25; p.th_dist_v = 0.1
    p.max_range = 80.0; p.min_range = 2.7; p.uprightness_thr = 0.707
    p.adaptive_seed_selection_margin = -1.2; p.intensity_thr = 0.0
    p.num_sectors_each_zone[:] = [16, 32, 54, 32]
    p.num_rings_each_zone[:] = [2, 4, 4, 4]
    p.elevation_thr[:] = [0.0] * 4
    p.flatness_thr[:] = [0.0] * 4
    return p


class PwppState(C.Structure):
    _fields_ = [("sensor_height", C.c_double), ("elevation_thr", C.c_double * 4), ("flatness_thr", C.c_double * 4),
                ("n_elevation", C.c_int32 * 4), ("n_flatness", C.c_int32 * 4)]


class PwppBinResult(C.Structure):
    _fields_ = [("mean", C.c_double * 3), ("normal", C.c_double * 3), ("sv", C.c_double * 3), ("d", C.c_double),
                ("n", C.c_int32), ("n_ground", C.c_int32), ("verdict", C.c_int32), ("fitted", C.c_int32)]


class PwppPointLayout(C.Structure):
    """Mirror of `pwpp_point_layout` (include/pwpp.h): the record layout of a frame for pwpp_estimate_*_records."""
    _fields_ = [("point_step", C.c_int32), ("offset", C.c_int32 * 4), ("datatype", C.c_int32 * 4)]


class PwppScanRing(C.Structure):
    """Mirror of `pwpp_scan_ring` (include/pwpp.h): a ring of scan slots in device memory for pwpp_bind_call_rings."""
    _fields_ = [("base", C.c_void_p), ("slot_stride", C.c_int64), ("d_counts", C.c_void_p), ("num_slots", C.c_int32), ("_pad", C.c_int32)]


class PwppBoundGetters(C.Structure):
    """Mirror of `pwpp_bound_getters` (include/pwpp.h): the fixed device pointers of a bound call's getter results."""
    _fields_ = [("ground_xyz", C.c_void_p), ("nonground_xyz", C.c_void_p), ("h_row_off", C.c_void_p), ("xyz_counts", C.c_void_p),
                ("centers", C.c_void_p), ("normals", C.c_void_p), ("num_patches", C.c_void_p), ("patch_row_stride", C.c_int64),
                ("states", C.c_void_p)]
