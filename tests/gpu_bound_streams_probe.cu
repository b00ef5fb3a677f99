// gpu_bound_streams_probe.cu — TEST-ONLY: the kernels of bound calls with a stream table (csrc/pwpp_records.cuh,
// k_bound_table_streams, k_bound_table_rings_streams, k_bound_table_packed_streams, k_bound_reset; csrc/pwpp_getters.cuh,
// k_bound_states_streams) compiled for sm_90a and launched the way pwpp_capi.cu's pwpp_run_bound_call launches them, so that
// tests/test_bound_streams_backends.py runs the cases of tests/test_simt_bound_streams.py on the GPU as well as through the SIMT
// stand-in (tests/simt/simt_bound_streams.cpp). The entry points take the SIMT driver's arguments with every array in device
// memory; each launch is followed by a synchronise, and the return value is PWPP_OK or PWPP_ERR_CUDA. Built by
// patchwork-plusplus_b200/build.py (build_examples) with the core library's nvcc line.
#include <algorithm>
#include <vector>

#include "pwpp_getters.cuh"

namespace {
int done(cudaError_t e) {
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  return e == cudaSuccess ? PWPP_OK : PWPP_ERR_CUDA;
}
}  // namespace

extern "C" {

int probe_stream_state_bytes() { return (int) sizeof(pwpp::StreamState); }
int probe_pwpp_state_bytes() { return (int) sizeof(pwpp_state); }

// simt_bound_table_streams with device arrays. max_n is read back to the host for the ring stride, as the SIMT driver computes
// it; the bound record table and the rings are built on the host and uploaded.
int probe_bound_table_streams(int kind, int nframes, const int64_t* counts, const int64_t* max_n, const int32_t* b_pset, int64_t* pt_off,
                              int32_t* chunk_off, int32_t* stream, int32_t* pset, int32_t* status, const int32_t* actions, int32_t* act,
                              const int32_t* scratch, const int32_t* dep, const void* init, void* states, const int32_t* streams, int32_t* read,
                              int32_t* claim, const int32_t* set_of, const int32_t* runs, int nruns, int num_streams, const int32_t* slots,
                              int32_t* slot, int num_slots, const int64_t* ring_counts, const void* base, int64_t capacity, const int64_t* offsets,
                              void* brun) {
  pwpp_point_layout L{};
  L.point_step = 16;
  for (int c = 0; c < 4; ++c) { L.offset[c] = 4 * c; L.datatype[c] = PWPP_FIELD_FLOAT32; }
  std::vector<long long> mxh(nframes);
  cudaError_t e = cudaMemcpy(mxh.data(), max_n, (size_t) nframes * sizeof(long long), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) return PWPP_ERR_CUDA;
  long long mx = 1;
  for (long long m : mxh) mx = std::max(mx, m);
  const std::vector<pwpp::RecordFrame> brec(nframes, pwpp::record_frame(L, base));
  const std::vector<pwpp::BoundRing> ring(nframes, pwpp::BoundRing{reinterpret_cast<const long long*>(ring_counts), mx * 16, num_slots, 0});
  pwpp::RecordFrame* d_brec = nullptr;
  pwpp::BoundRing* d_ring = nullptr;
  e = cudaMalloc(&d_brec, (size_t) nframes * sizeof(pwpp::RecordFrame));
  if (e == cudaSuccess) e = cudaMalloc(&d_ring, (size_t) nframes * sizeof(pwpp::BoundRing));
  if (e == cudaSuccess) e = cudaMemcpy(d_brec, brec.data(), (size_t) nframes * sizeof(pwpp::RecordFrame), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_ring, ring.data(), (size_t) nframes * sizeof(pwpp::BoundRing), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    const pwpp::BoundActions A{actions, act, scratch, dep, static_cast<const pwpp::StreamState*>(init), static_cast<pwpp::StreamState*>(states)};
    const pwpp::BoundStreams T{streams, read, claim, set_of, runs, nruns, num_streams};
    const auto cn = reinterpret_cast<const long long*>(counts);
    const auto mn = reinterpret_cast<const long long*>(max_n);
    const auto po = reinterpret_cast<long long*>(pt_off);
    auto* run = static_cast<pwpp::RecordFrame*>(brun);
    if (kind == 1) {
      const pwpp::BoundRings G{slots, slot, d_ring, d_brec, run};
      pwpp::k_bound_table_rings_streams<<<1, pwpp::BT_THREADS>>>(nframes, mn, b_pset, po, chunk_off, stream, pset, status, A, G, T);
    } else if (kind == 2) {
      const pwpp::BoundPacked P{reinterpret_cast<const long long*>(offsets), (long long) capacity, d_brec, run};
      pwpp::k_bound_table_packed_streams<<<1, pwpp::BT_THREADS>>>(nframes, mn, b_pset, po, chunk_off, stream, pset, status, A, P, T);
    } else {
      pwpp::k_bound_table_streams<<<1, pwpp::BT_THREADS>>>(nframes, cn, mn, b_pset, po, chunk_off, stream, pset, status, A, T);
    }
  }
  const int rc = done(e);
  cudaFree(d_brec);
  cudaFree(d_ring);
  return rc;
}

int probe_bound_reset(int f0, int f1, const int32_t* act, const int32_t* dep, const int32_t* read, const void* init, void* states) {
  pwpp::k_bound_reset<<<1, pwpp::BR_THREADS>>>(f0, f1, act, dep, read, static_cast<const pwpp::StreamState*>(init), static_cast<pwpp::StreamState*>(states));
  return done(cudaSuccess);
}

int probe_bound_states_streams(int f0, int f1, const int32_t* read, int num_streams, const void* states, void* out) {
  const int len = f1 - f0;
  pwpp::k_bound_states_streams<<<(len + pwpp::BS_THREADS - 1) / pwpp::BS_THREADS, pwpp::BS_THREADS>>>(
      f0, f1, read, num_streams, static_cast<const pwpp::StreamState*>(states), static_cast<pwpp_state*>(out));
  return done(cudaSuccess);
}

}  // extern "C"
