// simt_records_parts.cpp — TEST-ONLY: the record gather of a bound call's record results (csrc/pwpp_records.cuh,
// k_gather_record_parts) executed on the CPU by the SIMT stand-in (tests/test_records_parts_backends.py; the device twin of
// this entry point is tests/gpu_records_parts_probe.cu).
#include "simt_records.cpp"

extern "C" {

// One k_gather_record_parts launch over a call of nframes frames, as pwpp_capi.cu's pwpp_run_bound_call issues it: frame f's
// n[f] records of step[f] bytes start at frames[f] (host memory here, any alignment), its capacity is max_n[f] >= n[f]; its
// index lists are idx[p_f, p_f + ng + nn) with p_f = n[0] + ... + n[f - 1] (ground list, then non-ground list), counts the
// call's count rows [3][nframes] (num_ground, num_patches, num_dropped). parts: 1 ground, 2 non-ground, 3 both. part_off
// receives the nframes + 1 region offsets (from the capacities); ground / nonground (16-byte aligned, NULL for a part that is
// not gathered) must hold part_off[nframes] bytes; part_cnt receives [nframes][2] counts. Returns PWPP_ERR_INVALID_ARG for a
// bad step, size or count and launches nothing.
int simt_gather_record_parts(int nframes, const void* const* frames, const int64_t* n, const int64_t* max_n, const int32_t* step, const int32_t* idx,
                             const int32_t* counts, int parts, unsigned char* ground, unsigned char* nonground, int64_t* part_off, int32_t* part_cnt) {
  if (nframes < 1 || parts < 1 || parts > 3) return PWPP_ERR_INVALID_ARG;
  std::vector<pwpp::RecordFrame> recs(nframes);
  std::vector<long long> off(nframes + 1, 0), cap(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) {
    const int ng = counts[f], nd = counts[2 * nframes + f];
    if (step[f] < 1 || step[f] > PWPP_MAX_POINT_STEP || n[f] < 0 || n[f] > max_n[f] || ng < 0 || nd < 0 || ng + nd > n[f]) return PWPP_ERR_INVALID_ARG;
    recs[f] = pwpp::RecordFrame{};
    recs[f].src = static_cast<const unsigned char*>(frames[f]);
    recs[f].step = step[f];
    off[f + 1] = off[f] + n[f];
    cap[f + 1] = cap[f] + max_n[f];
  }
  std::vector<long long> poff(nframes + 1);
  pwpp::rec_out_offsets(cap.data(), recs.data(), nframes, poff.data());
  for (int f = 0; f <= nframes; ++f) part_off[f] = poff[f];
  const long long gx = pwpp::rec_parts_grid_x(cap.data(), recs.data(), nframes);
  const int first = parts == PWPP_PART_NONGROUND ? 1 : 0, nparts = parts == 3 ? 2 : 1;
  simt::launch("k_gather_record_parts", dim3((unsigned) gx, (unsigned) nframes, (unsigned) nparts), pwpp::REC_THREADS, 0,
               [&] { pwpp::k_gather_record_parts(recs.data(), off.data(), counts, nframes, idx, poff.data(), first, ground, nonground, part_cnt); });
  return PWPP_OK;
}

}  // extern "C"
