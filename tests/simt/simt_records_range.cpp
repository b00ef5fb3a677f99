// simt_records_range.cpp — TEST-ONLY: simt_records.cpp plus a k_unpack_records launch over a frame range of a call, as the host
// chunk path of pwpp_estimate_host_records issues one per pipeline chunk (tests/test_records_unpack_backends.py; the device
// twin of this entry point is tests/gpu_records_probe.cu).
#include "simt_records.cpp"

extern "C" {

// One launch over the frames [f0, f1) of a call of nframes frames (host memory here). Frame f's points go to dst from the
// absolute offset n[0] + ... + n[f - 1]; nothing else of dst is written. Returns the status of check_record_layouts, or
// PWPP_ERR_INVALID_ARG for a bad range.
int simt_unpack_records_range(int nframes, const void* const* frames, const int64_t* n, const pwpp_point_layout* layouts, float* dst, int f0,
                              int f1) {
  std::string msg;
  const int rc = pwpp::check_record_layouts(nframes, frames, n, layouts, &msg);
  if (rc) return rc;
  if (f0 < 0 || f1 > nframes || f0 > f1) return PWPP_ERR_INVALID_ARG;
  std::vector<pwpp::RecordFrame> recs(nframes);
  std::vector<long long> off(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) {
    recs[f] = pwpp::record_frame(layouts[f], frames[f]);
    off[f + 1] = off[f] + n[f];
  }
  if (off[f1] == off[f0]) return PWPP_OK;
  const long long gx = pwpp::rec_grid_x(off.data() + f0, recs.data() + f0, f1 - f0);
  float4* out = reinterpret_cast<float4*>(dst);
  simt::launch("k_unpack_records", dim3((unsigned) gx, (unsigned) (f1 - f0)), pwpp::REC_THREADS, 0,
               [&] { pwpp::k_unpack_records(recs.data() + f0, off.data() + f0, out); });
  return PWPP_OK;
}

}  // extern "C"
