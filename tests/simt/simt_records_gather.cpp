// simt_records_gather.cpp — TEST-ONLY: the record gather kernel of the record results (csrc/pwpp_records.cuh, k_gather_records)
// executed on the CPU by the SIMT stand-in (tests/test_simt_records_gather.py, tests/test_records_gather_backends.py; the
// device twin of this entry point is tests/gpu_records_gather_probe.cu).
#include "simt_records.cpp"

extern "C" {

// One k_gather_records launch over a call of nframes frames, as pwpp_capi.cu's gather_records issues it: frame f's n[f]
// records of step[f] bytes start at frames[f] (host memory here, any alignment); its index lists are idx[p_f, p_f + n[f] -
// nd[f]) with p_f = n[0] + ... + n[f - 1] (ground list, then non-ground list: the kernel does not tell them apart), nd[f] the
// dropped points. rec_off receives the nframes + 1 byte offsets of the output regions; dst (16-byte aligned) must hold
// rec_off[nframes] bytes. Returns PWPP_ERR_INVALID_ARG for a bad step or count and launches nothing.
int simt_gather_records(int nframes, const void* const* frames, const int64_t* n, const int32_t* step, const int32_t* idx, const int32_t* nd,
                        unsigned char* dst, int64_t* rec_off) {
  std::vector<pwpp::RecordFrame> recs(nframes);
  std::vector<long long> off(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) {
    if (step[f] < 1 || step[f] > PWPP_MAX_POINT_STEP || n[f] < 0 || nd[f] < 0 || nd[f] > n[f]) return PWPP_ERR_INVALID_ARG;
    recs[f] = pwpp::RecordFrame{};
    recs[f].src = static_cast<const unsigned char*>(frames[f]);
    recs[f].step = step[f];
    off[f + 1] = off[f] + n[f];
  }
  std::vector<long long> roff(nframes + 1);
  pwpp::rec_out_offsets(off.data(), recs.data(), nframes, roff.data());
  for (int f = 0; f <= nframes; ++f) rec_off[f] = roff[f];
  if (off[nframes] == 0) return PWPP_OK;
  const long long gx = pwpp::rec_grid_x(off.data(), recs.data(), nframes);
  simt::launch("k_gather_records", dim3((unsigned) gx, (unsigned) nframes), pwpp::REC_THREADS, 0,
               [&] { pwpp::k_gather_records(recs.data(), off.data(), roff.data(), nd, idx, dst); });
  return PWPP_OK;
}

}  // extern "C"
