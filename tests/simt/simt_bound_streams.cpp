// simt_bound_streams.cpp — TEST-ONLY: the frame-table kernels of bound calls with a stream table (csrc/pwpp_records.cuh,
// k_bound_table_streams, k_bound_table_rings_streams and k_bound_table_packed_streams), the reset kernel before a later run
// (k_bound_reset) and the state rows (csrc/pwpp_getters.cuh, k_bound_states_streams), executed on the CPU by the SIMT stand-in
// (tests/test_simt_bound_streams.py).
#include "simt_records.cpp"

#include "pwpp_getters.cuh"

extern "C" {

int simt_stream_state_bytes() { return (int) sizeof(pwpp::StreamState); }
int simt_pwpp_state_bytes() { return (int) sizeof(pwpp_state); }

// One table launch over nframes frames, as pwpp_run_bound_call issues it with a stream table (host memory here). kind 0: counts
// from counts[f]; kind 1: every frame reads slots[f] of one ring of num_slots slots (counts ring_counts, stride max(max_n) *
// 16 bytes, base); kind 2: a packed buffer of capacity 16-byte records at base with offsets[nframes + 1]. actions may be NULL
// (then act and dep are too). brun (kind 1 and 2) receives the run's record table.
void simt_bound_table_streams(int kind, int nframes, const int64_t* counts, const int64_t* max_n, const int32_t* b_pset, int64_t* pt_off,
                              int32_t* chunk_off, int32_t* stream, int32_t* pset, int32_t* status, const int32_t* actions, int32_t* act,
                              const int32_t* scratch, const int32_t* dep, const void* init, void* states, const int32_t* streams, int32_t* read,
                              int32_t* claim, const int32_t* set_of, const int32_t* runs, int nruns, int num_streams, const int32_t* slots,
                              int32_t* slot, int num_slots, const int64_t* ring_counts, const void* base, int64_t capacity, const int64_t* offsets,
                              void* brun) {
  pwpp_point_layout L{};
  L.point_step = 16;
  for (int c = 0; c < 4; ++c) { L.offset[c] = 4 * c; L.datatype[c] = PWPP_FIELD_FLOAT32; }
  std::vector<pwpp::RecordFrame> brec(nframes, pwpp::record_frame(L, base));
  long long mx = 1;
  for (int f = 0; f < nframes; ++f) mx = std::max<long long>(mx, max_n[f]);
  std::vector<pwpp::BoundRing> ring(nframes, pwpp::BoundRing{reinterpret_cast<const long long*>(ring_counts), mx * 16, num_slots, 0});
  const pwpp::BoundActions A{actions, act, scratch, dep, static_cast<const pwpp::StreamState*>(init), static_cast<pwpp::StreamState*>(states)};
  const pwpp::BoundStreams T{streams, read, claim, set_of, runs, nruns, num_streams};
  const auto cn = reinterpret_cast<const long long*>(counts);
  const auto mn = reinterpret_cast<const long long*>(max_n);
  const auto po = reinterpret_cast<long long*>(pt_off);
  auto* run = static_cast<pwpp::RecordFrame*>(brun);
  if (kind == 1) {
    const pwpp::BoundRings G{slots, slot, ring.data(), brec.data(), run};
    simt::launch("k_bound_table_rings_streams", dim3(1), pwpp::BT_THREADS, 0,
                 [&] { pwpp::k_bound_table_rings_streams(nframes, mn, b_pset, po, chunk_off, stream, pset, status, A, G, T); });
  } else if (kind == 2) {
    const pwpp::BoundPacked P{reinterpret_cast<const long long*>(offsets), (long long) capacity, brec.data(), run};
    simt::launch("k_bound_table_packed_streams", dim3(1), pwpp::BT_THREADS, 0,
                 [&] { pwpp::k_bound_table_packed_streams(nframes, mn, b_pset, po, chunk_off, stream, pset, status, A, P, T); });
  } else {
    simt::launch("k_bound_table_streams", dim3(1), pwpp::BT_THREADS, 0,
                 [&] { pwpp::k_bound_table_streams(nframes, cn, mn, b_pset, po, chunk_off, stream, pset, status, A, T); });
  }
}

// One k_bound_reset launch over the run [f0, f1), reading the run's copy of the streams.
void simt_bound_reset(int f0, int f1, const int32_t* act, const int32_t* dep, const int32_t* read, const void* init, void* states) {
  simt::launch("k_bound_reset", dim3(1), pwpp::BR_THREADS, 0, [&] {
    pwpp::k_bound_reset(f0, f1, act, dep, read, static_cast<const pwpp::StreamState*>(init), static_cast<pwpp::StreamState*>(states));
  });
}

// One k_bound_states_streams launch over the run [f0, f1).
void simt_bound_states_streams(int f0, int f1, const int32_t* read, int num_streams, const void* states, void* out) {
  const int len = f1 - f0;
  simt::launch("k_bound_states_streams", dim3((unsigned) ((len + pwpp::BS_THREADS - 1) / pwpp::BS_THREADS)), pwpp::BS_THREADS, 0, [&] {
    pwpp::k_bound_states_streams(f0, f1, read, num_streams, static_cast<const pwpp::StreamState*>(states), static_cast<pwpp_state*>(out));
  });
}

}  // extern "C"
