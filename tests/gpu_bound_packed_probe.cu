// gpu_bound_packed_probe.cu — TEST-ONLY: the kernels of a bound call's packed xyz results (csrc/pwpp_getters.cuh,
// k_bound_xyz_offsets and k_gather_xyz_packed) compiled for sm_90a and launched the way pwpp_capi.cu's pwpp_run_bound_call
// launches them, so that tests/test_bound_packed_xyz_backends.py runs its cases on the GPU as well as through the SIMT stand-in
// (tests/simt/simt_bound_packed.cpp). Built by patchwork-plusplus_b200/build.py (build_examples) with the core library's nvcc line.
#include <vector>

#include "pwpp_getters.cuh"

namespace {
template <typename T>
cudaError_t upload(T** d, const T* h, size_t n) {
  cudaError_t e = cudaMalloc(d, (n ? n : 1) * sizeof(T));
  if (e == cudaSuccess && n) e = cudaMemcpy(*d, h, n * sizeof(T), cudaMemcpyHostToDevice);
  return e;
}
}  // namespace

extern "C" {

// simt_packed_xyz (tests/simt/simt_bound_packed.cpp) with every array a host array: the points, lists, counts, offsets and both
// output buffers (sum(max_n) rows each) are copied to the device and back. Synchronous: PWPP_ERR_INVALID_ARG for a bad size or
// count, PWPP_ERR_CUDA for a CUDA error.
int probe_packed_xyz(int nframes, const float* pts, const int64_t* n, const int64_t* max_n, const int32_t* idx, const int32_t* counts, int parts,
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
  const size_t rows = (size_t) cap[nframes];
  float4* d_pts = nullptr;
  long long *d_off = nullptr, *d_go = nullptr, *d_no = nullptr;
  int *d_idx = nullptr, *d_counts = nullptr;
  float *d_g = nullptr, *d_n = nullptr;
  cudaError_t e = upload(&d_pts, reinterpret_cast<const float4*>(pts), (size_t) off[nframes]);
  if (e == cudaSuccess) e = upload(&d_off, off.data(), off.size());
  if (e == cudaSuccess) e = upload(&d_idx, idx, (size_t) off[nframes]);
  if (e == cudaSuccess) e = upload(&d_counts, counts, (size_t) 3 * nframes);
  if (e == cudaSuccess) e = upload(&d_go, reinterpret_cast<const long long*>(g_off), (size_t) nframes + 1);
  if (e == cudaSuccess) e = upload(&d_no, reinterpret_cast<const long long*>(ng_off), (size_t) nframes + 1);
  if (e == cudaSuccess && ground) e = upload(&d_g, ground, 3 * rows);
  if (e == cudaSuccess && nonground) e = upload(&d_n, nonground, 3 * rows);
  if (e == cudaSuccess) {
    pwpp::k_bound_xyz_offsets<<<1, pwpp::BT_THREADS>>>(nframes, d_off, d_counts, d_go, d_no);
    pwpp::k_gather_xyz_packed<<<dim3((unsigned) gx, (unsigned) nframes, (unsigned) nparts), pwpp::XYZ_THREADS>>>(d_pts, d_off, d_counts, nframes, d_idx,
                                                                                                              d_go, d_no, first, d_g, d_n);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(g_off, d_go, (size_t) (nframes + 1) * sizeof(long long), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess) e = cudaMemcpy(ng_off, d_no, (size_t) (nframes + 1) * sizeof(long long), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && ground && rows) e = cudaMemcpy(ground, d_g, 3 * rows * sizeof(float), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && nonground && rows) e = cudaMemcpy(nonground, d_n, 3 * rows * sizeof(float), cudaMemcpyDeviceToHost);
  cudaFree(d_pts);
  cudaFree(d_off);
  cudaFree(d_idx);
  cudaFree(d_counts);
  cudaFree(d_go);
  cudaFree(d_no);
  cudaFree(d_g);
  cudaFree(d_n);
  return e == cudaSuccess ? PWPP_OK : PWPP_ERR_CUDA;
}

}  // extern "C"
