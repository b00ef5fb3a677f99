// gpu_records_gather_probe.cu — TEST-ONLY: the record gather kernel (csrc/pwpp_records.cuh, k_gather_records) compiled for
// sm_90a and launched the way pwpp_capi.cu's gather_records launches it, so that tests/test_records_gather_backends.py runs
// its cases on the GPU as well as through the SIMT stand-in (tests/simt/simt_records_gather.cpp). Built by
// patchwork-plusplus_b200/build.py (build_examples) with the core library's nvcc line.
#include <vector>

#include "pwpp_records.cuh"

extern "C" {

// simt_gather_records (tests/simt/simt_records_gather.cpp) with the frames and dst in device memory; n, step, idx, nd and
// rec_off are host arrays. Synchronous: returns PWPP_ERR_INVALID_ARG for a bad step or count, PWPP_ERR_CUDA for a CUDA error.
int probe_gather_records(int nframes, const void* const* frames, const int64_t* n, const int32_t* step, const int32_t* idx, const int32_t* nd,
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
  pwpp::RecordFrame* d_rec = nullptr;
  long long *d_off = nullptr, *d_roff = nullptr;
  int *d_idx = nullptr, *d_nd = nullptr;
  cudaError_t e = cudaMalloc(&d_rec, recs.size() * sizeof(pwpp::RecordFrame));
  if (e == cudaSuccess) e = cudaMalloc(&d_off, off.size() * sizeof(long long));
  if (e == cudaSuccess) e = cudaMalloc(&d_roff, roff.size() * sizeof(long long));
  if (e == cudaSuccess) e = cudaMalloc(&d_idx, (size_t) off[nframes] * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&d_nd, (size_t) nframes * sizeof(int));
  if (e == cudaSuccess) e = cudaMemcpy(d_rec, recs.data(), recs.size() * sizeof(pwpp::RecordFrame), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_off, off.data(), off.size() * sizeof(long long), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_roff, roff.data(), roff.size() * sizeof(long long), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_idx, idx, (size_t) off[nframes] * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_nd, nd, (size_t) nframes * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    pwpp::k_gather_records<<<dim3((unsigned) gx, (unsigned) nframes), pwpp::REC_THREADS>>>(d_rec, d_off, d_roff, d_nd, d_idx, dst);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  cudaFree(d_rec);
  cudaFree(d_off);
  cudaFree(d_roff);
  cudaFree(d_idx);
  cudaFree(d_nd);
  return e == cudaSuccess ? PWPP_OK : PWPP_ERR_CUDA;
}

}  // extern "C"
