// simt_state_copy.cpp — TEST-ONLY: the device state copies (csrc/pwpp_state_copy.cuh: k_state_export, k_state_import_claim,
// k_state_import) executed on the CPU by the SIMT stand-in, launched as pwpp_export_states_device / pwpp_import_states_device
// launch them (tests/test_simt_state_copy.py builds the expected rows and states in numpy).
#include "simt_twin.cpp"

// the device's unsigned atomicMin (the stand-in declares the signed one only; one OS thread: a plain read-modify-write)
static inline unsigned atomicMin(unsigned* p, unsigned v) { const unsigned o = *p; if (v < o) *p = v; return o; }

#include "pwpp_state_copy.cuh"

extern "C" {

// The ctx's state buffers in host memory: states[num_streams] StreamStates (176 bytes each), hist[num_streams][8][hist_stride]
// doubles, hcap[num_streams]. blobs: n rows of blob_stride bytes. status may be NULL.
void simt_state_export(int n, const int32_t* streams, void* states, double* hist, int hist_stride, const int32_t* hcap, int num_streams, void* blobs,
                       int64_t blob_stride, int32_t* status) {
  const pwpp::StateStore st{static_cast<pwpp::StreamState*>(states), reinterpret_cast<long long*>(hist), hist_stride, hcap, num_streams};
  if (n <= 0) return;
  simt::launch("k_state_export", dim3((unsigned) n), pwpp::SC_THREADS, 0, [&] {
    pwpp::k_state_export(streams, st, static_cast<unsigned char*>(blobs), blob_stride, status);
  });
}

// claim: the ctx's claim table, int32[num_streams], -1 between calls.
void simt_state_import(int n, const int32_t* streams, void* states, double* hist, int hist_stride, const int32_t* hcap, int num_streams, const void* blobs,
                       int64_t blob_stride, int32_t* claim, int32_t* status) {
  const pwpp::StateStore st{static_cast<pwpp::StreamState*>(states), reinterpret_cast<long long*>(hist), hist_stride, hcap, num_streams};
  if (n <= 0) return;
  simt::launch("k_state_import_claim", dim3((unsigned) ((n + pwpp::SC_CLAIM_THREADS - 1) / pwpp::SC_CLAIM_THREADS)), pwpp::SC_CLAIM_THREADS, 0,
               [&] { pwpp::k_state_import_claim(n, streams, num_streams, claim); });
  simt::launch("k_state_import", dim3((unsigned) n), pwpp::SC_THREADS, 0, [&] {
    pwpp::k_state_import(streams, st, static_cast<const unsigned char*>(blobs), blob_stride, claim, status);
  });
}

}  // extern "C"
