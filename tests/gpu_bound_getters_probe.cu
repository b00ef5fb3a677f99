// gpu_bound_getters_probe.cu — TEST-ONLY: the kernels of a bound call's getter results (csrc/pwpp_getters.cuh) compiled for
// sm_90a and launched the way pwpp_capi.cu's pwpp_run_bound_call launches them, so that tests/test_bound_getters_backends.py runs
// its cases on the GPU as well as through the SIMT stand-in (tests/simt/simt_bound_getters.cpp). Built by
// patchwork-plusplus_b200/build.py (build_examples) with the core library's nvcc line.
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

int probe_stream_state_size() { return (int) sizeof(pwpp::StreamState); }

// simt_gather_xyz_parts (tests/simt/simt_bound_getters.cpp) with every array a host array: the points, lists, counts and both
// output buffers are copied to the device and back. Synchronous: PWPP_ERR_INVALID_ARG for a bad size or count, PWPP_ERR_CUDA
// for a CUDA error.
int probe_gather_xyz_parts(int nframes, const float* pts, const int64_t* n, const int64_t* max_n, const int32_t* idx, const int32_t* counts, int parts,
                           float* ground, float* nonground, int64_t* row_off, int32_t* xyz_cnt) {
  if (nframes < 1 || parts < 1 || parts > 3) return PWPP_ERR_INVALID_ARG;
  std::vector<long long> off(nframes + 1, 0), cap(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) {
    const int ng = counts[f], nd = counts[2 * nframes + f];
    if (n[f] < 0 || n[f] > max_n[f] || ng < 0 || nd < 0 || ng + nd > n[f]) return PWPP_ERR_INVALID_ARG;
    off[f + 1] = off[f] + n[f];
    cap[f + 1] = cap[f] + max_n[f];
  }
  for (int f = 0; f <= nframes; ++f) row_off[f] = cap[f];
  const long long gx = pwpp::xyz_parts_grid_x(cap.data(), nframes);
  const int first = parts == PWPP_GETTER_NONGROUND_XYZ ? 1 : 0, nparts = parts == 3 ? 2 : 1;
  const size_t rows = (size_t) cap[nframes];
  float4* d_pts = nullptr;
  long long *d_off = nullptr, *d_cap = nullptr;
  int *d_idx = nullptr, *d_counts = nullptr, *d_cnt = nullptr;
  float *d_g = nullptr, *d_n = nullptr;
  cudaError_t e = upload(&d_pts, reinterpret_cast<const float4*>(pts), (size_t) off[nframes]);
  if (e == cudaSuccess) e = upload(&d_off, off.data(), off.size());
  if (e == cudaSuccess) e = upload(&d_cap, cap.data(), cap.size());
  if (e == cudaSuccess) e = upload(&d_idx, idx, (size_t) off[nframes]);
  if (e == cudaSuccess) e = upload(&d_counts, counts, (size_t) 3 * nframes);
  if (e == cudaSuccess) e = upload(&d_cnt, xyz_cnt, (size_t) 2 * nframes);
  if (e == cudaSuccess && ground) e = upload(&d_g, ground, 3 * rows);
  if (e == cudaSuccess && nonground) e = upload(&d_n, nonground, 3 * rows);
  if (e == cudaSuccess) {
    pwpp::k_gather_xyz_parts<<<dim3((unsigned) gx, (unsigned) nframes, (unsigned) nparts), pwpp::XYZ_THREADS>>>(d_pts, d_off, d_counts, nframes, d_idx, d_cap,
                                                                                                             first, d_g, d_n, d_cnt);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(xyz_cnt, d_cnt, (size_t) 2 * nframes * sizeof(int), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && ground && rows) e = cudaMemcpy(ground, d_g, 3 * rows * sizeof(float), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && nonground && rows) e = cudaMemcpy(nonground, d_n, 3 * rows * sizeof(float), cudaMemcpyDeviceToHost);
  cudaFree(d_pts);
  cudaFree(d_off);
  cudaFree(d_cap);
  cudaFree(d_idx);
  cudaFree(d_counts);
  cudaFree(d_cnt);
  cudaFree(d_g);
  cudaFree(d_n);
  return e == cudaSuccess ? PWPP_OK : PWPP_ERR_CUDA;
}

// simt_bound_states with host arrays: states holds num_slots StreamState slots; out holds f1 rows (rows [f0, f1) are written,
// the others come back as they went in). Synchronous.
int probe_bound_states(int f0, int f1, const int32_t* b_stream, const void* states, int num_slots, pwpp_state* out) {
  if (f0 < 0 || f1 <= f0 || num_slots < 1) return PWPP_ERR_INVALID_ARG;
  int* d_bs = nullptr;
  pwpp::StreamState* d_st = nullptr;
  pwpp_state* d_out = nullptr;
  cudaError_t e = upload(&d_bs, b_stream, (size_t) f1);
  if (e == cudaSuccess) e = upload(&d_st, static_cast<const pwpp::StreamState*>(states), (size_t) num_slots);
  if (e == cudaSuccess) e = upload(&d_out, out, (size_t) f1);
  if (e == cudaSuccess) {
    pwpp::k_bound_states<<<(f1 - f0 + pwpp::BS_THREADS - 1) / pwpp::BS_THREADS, pwpp::BS_THREADS>>>(f0, f1, d_bs, d_st, d_out);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(out, d_out, (size_t) f1 * sizeof(pwpp_state), cudaMemcpyDeviceToHost);
  cudaFree(d_bs);
  cudaFree(d_st);
  cudaFree(d_out);
  return e == cudaSuccess ? PWPP_OK : PWPP_ERR_CUDA;
}

}  // extern "C"
