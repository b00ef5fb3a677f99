// simt_records.cpp — TEST-ONLY: the record unpack kernel (csrc/pwpp_records.cuh) executed on the CPU by the SIMT stand-in, plus
// the host-side layout checks of pwpp_estimate_*_records (csrc/pwpp_host.hpp). tests/test_simt_records.py compares the
// unpacked float4 points bit for bit with numpy's conversion. Built with plain g++ like the twin (simt_twin.cpp, included whole
// for the stand-in's runtime).
#include "simt_twin.cpp"

#include "pwpp_records.cuh"

extern "C" {

// One k_unpack_records launch over nframes frames, as pwpp_capi.cu issues it: frame f's n[f] records start at frames[f]
// (host memory here), layouts as in include/pwpp.h (validated first: the status of check_record_layouts is returned and
// nothing runs when it fails). dst receives sum(n) float4 points, frame after frame.
int simt_unpack_records(int nframes, const void* const* frames, const int64_t* n, const pwpp_point_layout* layouts, float* dst) {
  std::string msg;
  const int rc = pwpp::check_record_layouts(nframes, frames, n, layouts, &msg);
  if (rc) return rc;
  std::vector<pwpp::RecordFrame> recs(nframes);
  std::vector<long long> off(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) {
    const pwpp_point_layout& L = layouts[f];
    pwpp::RecordFrame& r = recs[f];
    r = pwpp::RecordFrame{};
    r.src = static_cast<const unsigned char*>(frames[f]);
    r.step = L.point_step;
    for (int c = 0; c < 4; ++c) { r.off[c] = L.offset[c]; r.type[c] = L.datatype[c]; }
    if (L.offset[3] < 0) { r.off[3] = 0; r.type[3] = 0; }
    off[f + 1] = off[f] + n[f];
  }
  if (off[nframes] == 0) return 0;
  const long long gx = pwpp::rec_grid_x(off.data(), recs.data(), nframes);
  float4* out = reinterpret_cast<float4*>(dst);
  simt::launch("k_unpack_records", dim3((unsigned) gx, (unsigned) nframes), pwpp::REC_THREADS, 0,
               [&] { pwpp::k_unpack_records(recs.data(), off.data(), out); });
  return 0;
}

// The layout checks alone; msg receives the message (at most cap bytes, NUL-terminated).
int simt_check_record_layouts(int nframes, const void* const* frames, const int64_t* n, const pwpp_point_layout* layouts, char* msg, int cap) {
  std::string m;
  const int rc = pwpp::check_record_layouts(nframes, frames, n, layouts, &m);
  std::snprintf(msg, (size_t) cap, "%s", m.c_str());
  return rc;
}

}  // extern "C"
