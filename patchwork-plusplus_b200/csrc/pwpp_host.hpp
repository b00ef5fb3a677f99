// pwpp_host.hpp — host-side helpers shared by the C-ABI implementation and the CPU twin used in tests.
#pragma once
#include <cstring>
#include <string>

#include "pwpp.h"
#include "pwpp_gle.cuh"
#include "pwpp_math.cuh"

namespace pwpp {

inline void build_geometry(const pwpp_params& p, Geometry& g, AlgoParams& ap, bool& fast) {
  // reference ctor, patchworkpp.h:122-134
  const double z2 = (7 * p.min_range + p.max_range) / 8.0;
  const double z3 = (3 * p.min_range + p.max_range) / 4.0;
  const double z4 = (p.min_range + p.max_range) / 2.0;
  g.min_ranges[0] = p.min_range; g.min_ranges[1] = z2; g.min_ranges[2] = z3; g.min_ranges[3] = z4;
  g.ring_sizes[0] = (z2 - p.min_range) / p.num_rings_each_zone[0];
  g.ring_sizes[1] = (z3 - z2) / p.num_rings_each_zone[1];
  g.ring_sizes[2] = (z4 - z3) / p.num_rings_each_zone[2];
  g.ring_sizes[3] = (p.max_range - z4) / p.num_rings_each_zone[3];
  g.max_range = p.max_range; g.min_range = p.min_range;
  g.bin_base[0] = 0; g.concentric_base[0] = 0;
  fast = p.max_range <= 250.0;
  for (int k = 0; k < 4; ++k) {
    g.sector_sizes[k] = 2 * PW_PI / p.num_sectors_each_zone[k];
    g.num_rings[k] = p.num_rings_each_zone[k];
    g.num_sectors[k] = p.num_sectors_each_zone[k];
    g.bin_base[k + 1] = g.bin_base[k] + g.num_rings[k] * g.num_sectors[k];
    g.concentric_base[k + 1] = g.concentric_base[k] + g.num_rings[k];
    g.f_min_ranges[k] = (float) g.min_ranges[k];
    g.f_ring_sizes[k] = (float) g.ring_sizes[k];
    g.f_sector_sizes[k] = (float) g.sector_sizes[k];
    g.f_inv_ring[k] = (float) (1.0 / g.ring_sizes[k]);
    g.f_inv_sector[k] = (float) (1.0 / g.sector_sizes[k]);
    // the fp32 filter of bin_of_point() needs decision cells much wider than the float error, and rings of at least
    // GUARD_R / GUARD_U = 1 m: its range test rejects only points more than GUARD_R (2e-4 m) outside (min_range, max_range]
    // and leaves the rest to the ring-coordinate guard of GUARD_U (2e-4) RING WIDTHS, so with rings narrower than 1 m a
    // point 1.9e-4 m inside the rejected side of min_range / max_range was binned instead of dropped (found by the random
    // parameter sets of tests/test_simt_kernels.py: ring width 0.875 m). Such geometries take the exact double path.
    if (!(g.ring_sizes[k] >= 1.5) || g.num_sectors[k] > 128) fast = false;
  }
  g.f_max_range = (float) g.max_range;
  g.nbins = g.bin_base[4];
  ap.RNR_ver_angle_thr = p.RNR_ver_angle_thr; ap.RNR_intensity_thr = p.RNR_intensity_thr;
  ap.f_RNR_intensity_thr = float_ru(p.RNR_intensity_thr);
  ap.th_seeds = p.th_seeds; ap.th_seeds_v = p.th_seeds_v; ap.th_dist = p.th_dist; ap.th_dist_v = p.th_dist_v;
  ap.uprightness_thr = p.uprightness_thr; ap.adaptive_seed_selection_margin = p.adaptive_seed_selection_margin;
  ap.num_iter = p.num_iter; ap.num_lpr = p.num_lpr; ap.num_min_pts = p.num_min_pts; ap.num_rings_of_interest = p.num_rings_of_interest;
  ap.enable_RNR = p.enable_RNR; ap.enable_RVPF = p.enable_RVPF; ap.enable_TGR = p.enable_TGR;
  ap.max_flatness_storage = p.max_flatness_storage; ap.max_elevation_storage = p.max_elevation_storage;
}

inline void init_state(const pwpp_params& p, StreamState& s) {
  std::memset(&s, 0, sizeof(s));
  s.sensor_height = p.sensor_height;
  for (int i = 0; i < 4; ++i) { s.elevation_thr[i] = p.elevation_thr[i]; s.flatness_thr[i] = p.flatness_thr[i]; }
}

// bytes of a PWPP_FIELD_* datatype, 0 for an unknown code
inline int field_bytes(int32_t datatype) {
  static const int bytes[9] = {0, 1, 1, 2, 2, 4, 4, 4, 8};
  return datatype >= 1 && datatype <= 8 ? bytes[datatype] : 0;
}

// The checks of pwpp_estimate_*_records on the frames, sizes and layouts of a call (include/pwpp.h), before anything is
// allocated or launched: PWPP_OK, or the status with *msg naming the frame and the field.
inline int check_record_layouts(int nframes, const void* const* frames, const int64_t* n, const pwpp_point_layout* layouts, std::string* msg) {
  static const char* names[4] = {"x", "y", "z", "intensity"};
  if (!frames || !n || !layouts) { *msg = "frames, n or layouts is NULL"; return PWPP_ERR_INVALID_ARG; }
  for (int f = 0; f < nframes; ++f) {
    const std::string fr = "frame " + std::to_string(f) + ": ";
    if (n[f] < 0) { *msg = fr + "n < 0"; return PWPP_ERR_INVALID_ARG; }
    if (n[f] > 0 && !frames[f]) { *msg = fr + "frame pointer is NULL"; return PWPP_ERR_INVALID_ARG; }
    const pwpp_point_layout& L = layouts[f];
    if (L.point_step < 1) { *msg = fr + "point_step " + std::to_string(L.point_step) + " < 1"; return PWPP_ERR_INVALID_ARG; }
    if (L.point_step > PWPP_MAX_POINT_STEP) {
      *msg = fr + "point_step " + std::to_string(L.point_step) + " > PWPP_MAX_POINT_STEP (" + std::to_string(PWPP_MAX_POINT_STEP) + ")";
      return PWPP_ERR_UNSUPPORTED;
    }
    for (int c = 0; c < 4; ++c) {
      if (c == 3 && L.offset[3] < 0) break;   // no intensity field
      const std::string fl = fr + "field " + names[c] + ": ";
      const int nb = field_bytes(L.datatype[c]);
      if (nb == 0) { *msg = fl + "unknown datatype " + std::to_string(L.datatype[c]); return PWPP_ERR_INVALID_ARG; }
      if (c < 3 && L.datatype[c] != PWPP_FIELD_FLOAT32 && L.datatype[c] != PWPP_FIELD_FLOAT64) {
        *msg = fl + "x, y and z must be FLOAT32 or FLOAT64, got datatype " + std::to_string(L.datatype[c]);
        return PWPP_ERR_UNSUPPORTED;
      }
      if (L.offset[c] < 0 || (int64_t) L.offset[c] + nb > L.point_step) {
        *msg = fl + "bytes [" + std::to_string(L.offset[c]) + ", " + std::to_string((int64_t) L.offset[c] + nb) + ") do not fit inside point_step " +
               std::to_string(L.point_step);
        return PWPP_ERR_INVALID_ARG;
      }
    }
  }
  return PWPP_OK;
}


}  // namespace pwpp
