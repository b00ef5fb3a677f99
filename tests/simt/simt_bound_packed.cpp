// simt_bound_packed.cpp — TEST-ONLY: the frame-table kernels of packed bound calls (csrc/pwpp_records.cuh, k_bound_table_packed
// and k_bound_table_packed_actions) and the kernels of packed xyz results (csrc/pwpp_getters.cuh, k_bound_xyz_offsets and
// k_gather_xyz_packed), executed on the CPU by the SIMT stand-in (tests/test_simt_bound_packed.py,
// tests/test_bound_packed_xyz_backends.py; the device twin of the xyz entry point is tests/gpu_bound_packed_probe.cu).
#include "simt_records.cpp"

#include "pwpp_getters.cuh"

extern "C" {

int simt_stream_state_bytes() { return (int) sizeof(pwpp::StreamState); }
int simt_record_frame_bytes() { return (int) sizeof(pwpp::RecordFrame); }

// One packed table launch over nframes frames, as pwpp_run_bound_call issues it (host memory here): k_bound_table_packed_actions
// when actions is not NULL (act, scratch, dep, init and states as for simt_bound_table_actions), k_bound_table_packed otherwise.
// The buffer holds capacity records of layout at base; offsets holds nframes + 1 entries; brun (nframes RecordFrames) receives
// the run's record table.
void simt_bound_table_packed(int nframes, const int64_t* max_n, const int32_t* b_stream, const int32_t* b_pset, int64_t* pt_off, int32_t* chunk_off,
                             int32_t* stream, int32_t* pset, int32_t* status, const int32_t* actions, int32_t* act, const int32_t* scratch,
                             const int32_t* dep, const void* init, void* states, const void* base, const pwpp_point_layout* layout, int64_t capacity,
                             const int64_t* offsets, void* brun) {
  std::vector<pwpp::RecordFrame> brec(nframes, pwpp::record_frame(*layout, base));
  const pwpp::BoundPacked P{reinterpret_cast<const long long*>(offsets), (long long) capacity, brec.data(), static_cast<pwpp::RecordFrame*>(brun)};
  const auto mx = reinterpret_cast<const long long*>(max_n);
  const auto po = reinterpret_cast<long long*>(pt_off);
  if (actions) {
    const pwpp::BoundActions A{actions, act, scratch, dep, static_cast<const pwpp::StreamState*>(init), static_cast<pwpp::StreamState*>(states)};
    simt::launch("k_bound_table_packed_actions", dim3(1), pwpp::BT_THREADS, 0,
                 [&] { pwpp::k_bound_table_packed_actions(nframes, mx, b_stream, b_pset, po, chunk_off, stream, pset, status, A, P); });
  } else {
    simt::launch("k_bound_table_packed", dim3(1), pwpp::BT_THREADS, 0,
                 [&] { pwpp::k_bound_table_packed(nframes, mx, b_stream, b_pset, po, chunk_off, stream, pset, status, P); });
  }
}

// The bound call's unpack over the run's record table brun and point offsets pt_off (the table kernel's), with the grid sized
// from the capacities max_n as pwpp_run_bound_call sizes it. dst receives pt_off[nframes] float4 points.
void simt_unpack_run(int nframes, const void* brun, const int64_t* max_n, const int64_t* pt_off, float* dst) {
  const auto* recs = static_cast<const pwpp::RecordFrame*>(brun);
  std::vector<long long> cap(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) cap[f + 1] = cap[f] + max_n[f];
  if (cap[nframes] == 0) return;
  const long long gx = pwpp::rec_grid_x(cap.data(), recs, nframes);
  simt::launch("k_unpack_records", dim3((unsigned) gx, (unsigned) nframes), pwpp::REC_THREADS, 0, [&] {
    pwpp::k_unpack_records(recs, reinterpret_cast<const long long*>(pt_off), reinterpret_cast<float4*>(dst));
  });
}

// The two launches of packed xyz results, as pwpp_run_bound_call issues them after the last run: k_bound_xyz_offsets, then
// k_gather_xyz_packed with the grid sized from the capacities max_n. Frame f's n[f] float4 points start at pts + 4 p_f (p_f =
// n[0] + ... + n[f - 1]), its index lists are idx[p_f, p_f + ng + nn) (ground, then non-ground), counts the call's count rows
// [3][nframes]. parts: 1 ground, 2 non-ground, 3 both. g_off / ng_off receive nframes + 1 row offsets each; ground / nonground
// (NULL for a part that is not gathered) hold the packed rows. Returns PWPP_ERR_INVALID_ARG for a bad size or count and
// launches nothing.
int simt_packed_xyz(int nframes, const float* pts, const int64_t* n, const int64_t* max_n, const int32_t* idx, const int32_t* counts, int parts,
                    float* ground, float* nonground, int64_t* g_off, int64_t* ng_off) {
  if (nframes < 1 || parts < 1 || parts > 3) return PWPP_ERR_INVALID_ARG;
  std::vector<long long> off(nframes + 1, 0), cap(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) {
    const int ng = counts[f], nd = counts[2 * nframes + f];
    if (n[f] < 0 || n[f] > max_n[f] || ng < 0 || nd < 0 || ng + nd > n[f]) return PWPP_ERR_INVALID_ARG;
    off[f + 1] = off[f] + n[f];
    cap[f + 1] = cap[f] + max_n[f];
  }
  const long long gx = pwpp::xyz_parts_grid_x(cap.data(), nframes);
  const int first = parts == PWPP_PART_NONGROUND ? 1 : 0, nparts = parts == 3 ? 2 : 1;
  auto go = reinterpret_cast<long long*>(g_off);
  auto no = reinterpret_cast<long long*>(ng_off);
  simt::launch("k_bound_xyz_offsets", dim3(1), pwpp::BT_THREADS, 0, [&] { pwpp::k_bound_xyz_offsets(nframes, off.data(), counts, go, no); });
  const float4* p = reinterpret_cast<const float4*>(pts);
  simt::launch("k_gather_xyz_packed", dim3((unsigned) gx, (unsigned) nframes, (unsigned) nparts), pwpp::XYZ_THREADS, 0,
               [&] { pwpp::k_gather_xyz_packed(p, off.data(), counts, nframes, idx, go, no, first, ground, nonground); });
  return PWPP_OK;
}

}  // extern "C"
