// simt_bound_actions.cpp — TEST-ONLY: the frame-table kernel of bound calls with actions (csrc/pwpp_records.cuh,
// k_bound_table_actions) and the reset kernel that runs before a dependent run (k_bound_reset), executed on the CPU by the
// SIMT stand-in (tests/test_simt_bound_actions.py).
#include "simt_records.cpp"

extern "C" {

int simt_stream_state_bytes() { return (int) sizeof(pwpp::StreamState); }

// One k_bound_table_actions launch over nframes frames, as pwpp_run_bound_call issues it (host memory here). The outputs of
// k_bound_table, plus act[0..nframes) (the copy of actions) and the constructor states init[s] copied into states[s] for the
// RESET frames with dep[f] == 0.
void simt_bound_table_actions(int nframes, const int64_t* counts, const int64_t* max_n, const int32_t* b_stream, const int32_t* b_pset,
                              int64_t* pt_off, int32_t* chunk_off, int32_t* stream, int32_t* pset, int32_t* status, const int32_t* actions,
                              int32_t* act, const int32_t* scratch, const int32_t* dep, const void* init, void* states) {
  const pwpp::BoundActions A{actions, act, scratch, dep, static_cast<const pwpp::StreamState*>(init), static_cast<pwpp::StreamState*>(states)};
  simt::launch("k_bound_table_actions", dim3(1), pwpp::BT_THREADS, 0, [&] {
    pwpp::k_bound_table_actions(nframes, reinterpret_cast<const long long*>(counts), reinterpret_cast<const long long*>(max_n), b_stream, b_pset,
                                reinterpret_cast<long long*>(pt_off), chunk_off, stream, pset, status, A);
  });
}

// One k_bound_reset launch over the run [f0, f1).
void simt_bound_reset(int f0, int f1, const int32_t* act, const int32_t* dep, const int32_t* b_stream, const void* init, void* states) {
  simt::launch("k_bound_reset", dim3(1), pwpp::BR_THREADS, 0, [&] {
    pwpp::k_bound_reset(f0, f1, act, dep, b_stream, static_cast<const pwpp::StreamState*>(init), static_cast<pwpp::StreamState*>(states));
  });
}

}  // extern "C"
