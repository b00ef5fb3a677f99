// gpu_records_packed_probe.cu — TEST-ONLY: the packed record gather of a bound call's packed records (csrc/pwpp_getters.cuh,
// k_bound_xyz_offsets, then csrc/pwpp_records.cuh, k_gather_record_packed) compiled for sm_90a and launched the way
// pwpp_capi.cu's pwpp_run_bound_call launches them, so that tests/test_records_packed_backends.py runs its cases on the GPU as
// well as through the SIMT stand-in (tests/simt/simt_records_packed.cpp). Built by patchwork-plusplus_b200/build.py
// (build_examples) with the core library's nvcc line.
#include <vector>

#include "pwpp_getters.cuh"

extern "C" {

// simt_gather_record_packed (tests/simt/simt_records_packed.cpp) with the frames, ground and nonground in device memory; n,
// max_n, idx, counts, g_off and ng_off are host arrays. Synchronous: returns PWPP_ERR_INVALID_ARG for a bad step, size or
// count, PWPP_ERR_CUDA for a CUDA error.
int probe_gather_record_packed(int nframes, const void* const* frames, const int64_t* n, const int64_t* max_n, int32_t step, const int32_t* idx,
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
  const size_t nidx = (size_t) std::max<long long>(off[nframes], 1);
  pwpp::RecordFrame* d_rec = nullptr;
  long long *d_off = nullptr, *d_go = nullptr, *d_no = nullptr;
  int *d_idx = nullptr, *d_counts = nullptr;
  cudaError_t e = cudaMalloc(&d_rec, recs.size() * sizeof(pwpp::RecordFrame));
  if (e == cudaSuccess) e = cudaMalloc(&d_off, off.size() * sizeof(long long));
  if (e == cudaSuccess) e = cudaMalloc(&d_go, off.size() * sizeof(long long));
  if (e == cudaSuccess) e = cudaMalloc(&d_no, off.size() * sizeof(long long));
  if (e == cudaSuccess) e = cudaMalloc(&d_idx, nidx * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&d_counts, (size_t) 3 * nframes * sizeof(int));
  if (e == cudaSuccess) e = cudaMemcpy(d_rec, recs.data(), recs.size() * sizeof(pwpp::RecordFrame), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_off, off.data(), off.size() * sizeof(long long), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && off[nframes] > 0) e = cudaMemcpy(d_idx, idx, (size_t) off[nframes] * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_counts, counts, (size_t) 3 * nframes * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    pwpp::k_bound_xyz_offsets<<<1, pwpp::BT_THREADS>>>(nframes, d_off, d_counts, d_go, d_no);
    pwpp::k_gather_record_packed<<<dim3((unsigned) gx, (unsigned) nframes, (unsigned) nparts), pwpp::REC_THREADS>>>(
        d_rec, d_off, d_counts, nframes, d_idx, d_go, d_no, first, ground, nonground);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(g_off, d_go, off.size() * sizeof(long long), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess) e = cudaMemcpy(ng_off, d_no, off.size() * sizeof(long long), cudaMemcpyDeviceToHost);
  cudaFree(d_rec);
  cudaFree(d_off);
  cudaFree(d_go);
  cudaFree(d_no);
  cudaFree(d_idx);
  cudaFree(d_counts);
  return e == cudaSuccess ? PWPP_OK : PWPP_ERR_CUDA;
}

}  // extern "C"
