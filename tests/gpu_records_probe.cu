// gpu_records_probe.cu — TEST-ONLY: the record unpack kernel (csrc/pwpp_records.cuh) compiled for sm_90a and launched the way
// pwpp_capi.cu's unpack_records launches it, so that tests/test_records_unpack_backends.py runs the cases of
// tests/test_simt_records.py on the GPU as well as through the SIMT stand-in (tests/simt/simt_records.cpp). Built by patchwork-plusplus_b200/build.py (build_examples) with the core
// library's nvcc line, so the device conversions, the non-allocating vector load and the NaN branch of rec_f64 are the ones
// the product runs.
#include <string>
#include <vector>

#include "pwpp_host.hpp"
#include "pwpp_records.cuh"

extern "C" {

// simt_unpack_records_range (tests/simt/simt_records_range.cpp) with the frames and dst in device memory: check_record_layouts, then one k_unpack_records launch over
// the frames [f0, f1) of a call of nframes frames. Frame f's n[f] records start at frames[f]; its points go to dst from the
// absolute offset n[0] + ... + n[f - 1], as on the host chunk path, and nothing else of dst is written. Synchronous: returns
// the layout status, PWPP_ERR_INVALID_ARG for a bad range, PWPP_ERR_CUDA for a CUDA error.
int probe_unpack_records(int nframes, const void* const* frames, const int64_t* n, const pwpp_point_layout* layouts, float* dst, int f0, int f1) {
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
  pwpp::RecordFrame* d_rec = nullptr;
  long long* d_off = nullptr;
  cudaError_t e = cudaMalloc(&d_rec, recs.size() * sizeof(pwpp::RecordFrame));
  if (e == cudaSuccess) e = cudaMalloc(&d_off, off.size() * sizeof(long long));
  if (e == cudaSuccess) e = cudaMemcpy(d_rec, recs.data(), recs.size() * sizeof(pwpp::RecordFrame), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_off, off.data(), off.size() * sizeof(long long), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    pwpp::k_unpack_records<<<dim3((unsigned) gx, (unsigned) (f1 - f0)), pwpp::REC_THREADS>>>(d_rec + f0, d_off + f0, reinterpret_cast<float4*>(dst));
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  cudaFree(d_rec);
  cudaFree(d_off);
  return e == cudaSuccess ? PWPP_OK : PWPP_ERR_CUDA;
}

}  // extern "C"
