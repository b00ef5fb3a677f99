// simt_bound_table.cpp — TEST-ONLY: the frame-table kernel of bound calls (csrc/pwpp_records.cuh, k_bound_table) executed on the
// CPU by the SIMT stand-in (tests/test_simt_bound_table.py).
#include "simt_records.cpp"

extern "C" {

// One k_bound_table launch over nframes frames, as pwpp_run_bound_call issues it (host memory here): counts and max_n are
// int64[nframes], b_stream / b_pset the bound call's tables. The kernel writes pt_off[0..nframes], chunk_off[0..nframes] and
// stream, pset, status[0..nframes).
void simt_bound_table(int nframes, const int64_t* counts, const int64_t* max_n, const int32_t* b_stream, const int32_t* b_pset, int64_t* pt_off,
                      int32_t* chunk_off, int32_t* stream, int32_t* pset, int32_t* status) {
  simt::launch("k_bound_table", dim3(1), pwpp::BT_THREADS, 0, [&] {
    pwpp::k_bound_table(nframes, reinterpret_cast<const long long*>(counts), reinterpret_cast<const long long*>(max_n), b_stream, b_pset,
                        reinterpret_cast<long long*>(pt_off), chunk_off, stream, pset, status);
  });
}

}  // extern "C"
