// simt_bound_getters.cpp — TEST-ONLY: the kernels of a bound call's getter results (csrc/pwpp_getters.cuh, k_gather_xyz_parts
// and k_bound_states) executed on the CPU by the SIMT stand-in (tests/test_bound_getters_backends.py; the device twin of these
// entry points is tests/gpu_bound_getters_probe.cu).
#include "simt_records.cpp"

#include "pwpp_getters.cuh"

extern "C" {

int simt_stream_state_size() { return (int) sizeof(pwpp::StreamState); }

// One k_gather_xyz_parts launch over a call of nframes frames, as pwpp_capi.cu's pwpp_run_bound_call issues it: frame f's n[f]
// float4 points start at pts + 4 p_f (p_f = n[0] + ... + n[f - 1]), its capacity is max_n[f] >= n[f]; its index lists are
// idx[p_f, p_f + ng + nn) (ground list, then non-ground list), counts the call's count rows [3][nframes] (num_ground,
// num_patches, num_dropped). parts: 1 ground, 2 non-ground, 3 both. row_off receives the nframes + 1 row offsets (the prefix
// sum of the capacities); ground / nonground (NULL for a part that is not gathered) must hold 3 row_off[nframes] floats;
// xyz_cnt receives [nframes][2] counts. Returns PWPP_ERR_INVALID_ARG for a bad size or count and launches nothing.
int simt_gather_xyz_parts(int nframes, const float* pts, const int64_t* n, const int64_t* max_n, const int32_t* idx, const int32_t* counts, int parts,
                          float* ground, float* nonground, int64_t* row_off, int32_t* xyz_cnt) {
  if (nframes < 1 || parts < 1 || parts > 3) return PWPP_ERR_INVALID_ARG;
  std::vector<long long> off(nframes + 1, 0), cap(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) {
    const int ng = counts[f], nd = counts[2 * nframes + f];
    if (n[f] < 0 || n[f] > max_n[f] || ng < 0 || nd < 0 || ng + nd > n[f]) return PWPP_ERR_INVALID_ARG;
    off[f + 1] = off[f] + n[f];
    cap[f + 1] = cap[f] + max_n[f];
  }
  for (int f = 0; f <= nframes; ++f) row_off[f] = cap[f];
  const long long gx = pwpp::xyz_parts_grid_x(cap.data(), nframes);
  const int first = parts == PWPP_GETTER_NONGROUND_XYZ ? 1 : 0, nparts = parts == 3 ? 2 : 1;
  const float4* p = reinterpret_cast<const float4*>(pts);
  simt::launch("k_gather_xyz_parts", dim3((unsigned) gx, (unsigned) nframes, (unsigned) nparts), pwpp::XYZ_THREADS, 0,
               [&] { pwpp::k_gather_xyz_parts(p, off.data(), counts, nframes, idx, cap.data(), first, ground, nonground, xyz_cnt); });
  return PWPP_OK;
}

// One k_bound_states launch over frames [f0, f1) of a run, as pwpp_run_bound_call issues it after the run: b_stream is the bound
// stream table, states the ctx's num_slots state slots (simt_stream_state_size() bytes each), out the pwpp_state rows of the call.
int simt_bound_states(int f0, int f1, const int32_t* b_stream, const void* states, int num_slots, pwpp_state* out) {
  if (f0 < 0 || f1 <= f0 || num_slots < 1) return PWPP_ERR_INVALID_ARG;
  const pwpp::StreamState* s = static_cast<const pwpp::StreamState*>(states);
  simt::launch("k_bound_states", dim3((unsigned) ((f1 - f0 + pwpp::BS_THREADS - 1) / pwpp::BS_THREADS)), pwpp::BS_THREADS, 0,
               [&] { pwpp::k_bound_states(f0, f1, b_stream, s, out); });
  return PWPP_OK;
}

}  // extern "C"
