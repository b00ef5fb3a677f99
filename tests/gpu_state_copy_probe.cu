// gpu_state_copy_probe.cu — TEST-ONLY: the device state copies (csrc/pwpp_state_copy.cuh) compiled for sm_90a and launched the
// way pwpp_export_states_device / pwpp_import_states_device launch them, over host copies of a ctx's state buffers, so that
// tests/test_state_copy_backends.py runs the cases of tests/test_simt_state_copy.py on the GPU as well as through the SIMT
// stand-in. Built by patchwork-plusplus_b200/build.py (build_examples) with the core library's nvcc line.
#include <vector>

#include "pwpp.h"
#include "pwpp_state_copy.cuh"

using namespace pwpp;

namespace {

// the host arrays of one call on the device and back: states[ns], hist[ns][8][stride] doubles, hcap[ns], blobs[n][blob_stride],
// claim[ns] (import), status[n] (NULL: none)
struct Dev {
  int *streams = nullptr, *hcap = nullptr, *claim = nullptr, *status = nullptr;
  StreamState* states = nullptr;
  double* hist = nullptr;
  unsigned char* blobs = nullptr;
  cudaError_t e = cudaSuccess;
  template <typename T>
  void up(T** d, const void* h, size_t bytes) {
    if (e == cudaSuccess) e = cudaMalloc(d, bytes ? bytes : 16);
    if (e == cudaSuccess && h && bytes) e = cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice);
  }
  void down(void* h, const void* d, size_t bytes) {
    if (e == cudaSuccess && h && bytes) e = cudaMemcpy(h, d, bytes, cudaMemcpyDeviceToHost);
  }
  ~Dev() { cudaFree(streams); cudaFree(hcap); cudaFree(claim); cudaFree(status); cudaFree(states); cudaFree(hist); cudaFree(blobs); }
};

}  // namespace

extern "C" {

int probe_state_export(int n, const int32_t* streams, void* states, double* hist, int hist_stride, const int32_t* hcap, int num_streams, void* blobs,
                       int64_t blob_stride, int32_t* status) {
  if (n <= 0) return PWPP_OK;
  Dev d;
  const size_t sb = (size_t) num_streams * sizeof(StreamState), hb = (size_t) num_streams * 8 * hist_stride * sizeof(double), bb = (size_t) n * blob_stride;
  d.up(&d.streams, streams, (size_t) n * sizeof(int));
  d.up(&d.hcap, hcap, (size_t) num_streams * sizeof(int));
  d.up(&d.states, states, sb);
  d.up(&d.hist, hist, hb);
  d.up(&d.blobs, blobs, bb);
  if (status) d.up(&d.status, status, (size_t) n * sizeof(int));
  if (d.e == cudaSuccess) {
    k_state_export<<<n, SC_THREADS>>>(d.streams, StateStore{d.states, reinterpret_cast<long long*>(d.hist), hist_stride, d.hcap, num_streams}, d.blobs,
                                      blob_stride, status ? d.status : nullptr);
    d.e = cudaGetLastError();
  }
  if (d.e == cudaSuccess) d.e = cudaDeviceSynchronize();
  d.down(blobs, d.blobs, bb);
  d.down(states, d.states, sb);
  d.down(hist, d.hist, hb);
  if (status) d.down(status, d.status, (size_t) n * sizeof(int));
  return d.e == cudaSuccess ? PWPP_OK : PWPP_ERR_CUDA;
}

int probe_state_import(int n, const int32_t* streams, void* states, double* hist, int hist_stride, const int32_t* hcap, int num_streams, const void* blobs,
                       int64_t blob_stride, int32_t* claim, int32_t* status) {
  if (n <= 0) return PWPP_OK;
  Dev d;
  const size_t sb = (size_t) num_streams * sizeof(StreamState), hb = (size_t) num_streams * 8 * hist_stride * sizeof(double), bb = (size_t) n * blob_stride;
  d.up(&d.streams, streams, (size_t) n * sizeof(int));
  d.up(&d.hcap, hcap, (size_t) num_streams * sizeof(int));
  d.up(&d.claim, claim, (size_t) num_streams * sizeof(int));
  d.up(&d.states, states, sb);
  d.up(&d.hist, hist, hb);
  d.up(&d.blobs, blobs, bb);
  if (status) d.up(&d.status, status, (size_t) n * sizeof(int));
  if (d.e == cudaSuccess) {
    const StateStore st{d.states, reinterpret_cast<long long*>(d.hist), hist_stride, d.hcap, num_streams};
    k_state_import_claim<<<(n + SC_CLAIM_THREADS - 1) / SC_CLAIM_THREADS, SC_CLAIM_THREADS>>>(n, d.streams, num_streams, d.claim);
    k_state_import<<<n, SC_THREADS>>>(d.streams, st, d.blobs, blob_stride, d.claim, status ? d.status : nullptr);
    d.e = cudaGetLastError();
  }
  if (d.e == cudaSuccess) d.e = cudaDeviceSynchronize();
  d.down(states, d.states, sb);
  d.down(hist, d.hist, hb);
  d.down(claim, d.claim, (size_t) num_streams * sizeof(int));
  if (status) d.down(status, d.status, (size_t) n * sizeof(int));
  return d.e == cudaSuccess ? PWPP_OK : PWPP_ERR_CUDA;
}

}  // extern "C"
