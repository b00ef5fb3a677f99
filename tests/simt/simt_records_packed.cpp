// simt_records_packed.cpp — TEST-ONLY: the packed record gather of a bound call's packed records (csrc/pwpp_getters.cuh,
// k_bound_xyz_offsets, then csrc/pwpp_records.cuh, k_gather_record_packed) executed on the CPU by the SIMT stand-in
// (tests/test_records_packed_backends.py; the device twin of this entry point is tests/gpu_records_packed_probe.cu).
#include "simt_records.cpp"

#include "pwpp_getters.cuh"

extern "C" {

// The two launches of packed records, as pwpp_run_bound_call issues them after the last run: k_bound_xyz_offsets, then
// k_gather_record_packed with the grid sized from the capacities max_n. Frame f's n[f] records of step bytes (the same step
// for every frame) start at frames[f] (host memory here, any alignment), its capacity is max_n[f] >= n[f]; its index lists are
// idx[p_f, p_f + ng + nn) with p_f = n[0] + ... + n[f - 1] (ground list, then non-ground list), counts the call's count rows
// [3][nframes] (num_ground, num_patches, num_dropped). parts: 1 ground, 2 non-ground, 3 both. g_off / ng_off receive nframes + 1
// record offsets each; ground / nonground (any alignment, NULL for a part that is not gathered) receive the packed records.
// Returns PWPP_ERR_INVALID_ARG for a bad step, size or count and launches nothing.
int simt_gather_record_packed(int nframes, const void* const* frames, const int64_t* n, const int64_t* max_n, int32_t step, const int32_t* idx,
                              const int32_t* counts, int parts, unsigned char* ground, unsigned char* nonground, int64_t* g_off, int64_t* ng_off) {
  if (nframes < 1 || parts < 1 || parts > 3 || step < 1 || step > PWPP_MAX_POINT_STEP) return PWPP_ERR_INVALID_ARG;
  std::vector<pwpp::RecordFrame> recs(nframes);
  std::vector<long long> off(nframes + 1, 0), cap(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) {
    const int ng = counts[f], nd = counts[2 * nframes + f];
    if (n[f] < 0 || n[f] > max_n[f] || ng < 0 || nd < 0 || ng + nd > n[f]) return PWPP_ERR_INVALID_ARG;
    recs[f] = pwpp::RecordFrame{};
    recs[f].src = static_cast<const unsigned char*>(frames[f]);
    recs[f].step = step;
    off[f + 1] = off[f] + n[f];
    cap[f + 1] = cap[f] + max_n[f];
  }
  const long long gx = pwpp::rec_parts_grid_x(cap.data(), recs.data(), nframes);
  const int first = parts == PWPP_PART_NONGROUND ? 1 : 0, nparts = parts == 3 ? 2 : 1;
  auto go = reinterpret_cast<long long*>(g_off);
  auto no = reinterpret_cast<long long*>(ng_off);
  simt::launch("k_bound_xyz_offsets", dim3(1), pwpp::BT_THREADS, 0, [&] { pwpp::k_bound_xyz_offsets(nframes, off.data(), counts, go, no); });
  simt::launch("k_gather_record_packed", dim3((unsigned) gx, (unsigned) nframes, (unsigned) nparts), pwpp::REC_THREADS, 0,
               [&] { pwpp::k_gather_record_packed(recs.data(), off.data(), counts, nframes, idx, go, no, first, ground, nonground); });
  return PWPP_OK;
}

}  // extern "C"
