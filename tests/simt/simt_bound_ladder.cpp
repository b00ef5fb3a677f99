// simt_bound_ladder.cpp — TEST-ONLY: the width selector of bound calls with a width ladder (csrc/pwpp_ladder.cuh,
// k_ladder_select) executed on the CPU by the SIMT stand-in (tests/test_simt_bound_ladder.py).
#include "simt_twin.cpp"

// The stand-in of the device API pwpp_ladder.cuh calls (tests/simt/cuda_runtime.h has no graph types): cudaGraphSetConditional
// records the handle and value it was given.
typedef unsigned long long cudaGraphConditionalHandle;
namespace simt {
struct CondSet {
  cudaGraphConditionalHandle handle = 0;
  unsigned value = 0;
  int calls = 0;
};
static CondSet g_cond;
}  // namespace simt
static inline void cudaGraphSetConditional(cudaGraphConditionalHandle handle, unsigned value) {
  simt::g_cond.handle = handle;
  simt::g_cond.value = value;
  ++simt::g_cond.calls;
}

#include "pwpp_ladder.cuh"

extern "C" {

// One k_ladder_select launch over the status array of nframes positions with the ladder widths[0 .. nwidths) (nframes last), as
// pwpp_run_bound_call issues it. *width receives what the kernel wrote to d_width; *index the value it gave
// cudaGraphSetConditional, -1 when it made no such call or named another handle. Returns PWPP_OK.
int simt_ladder_select(int nframes, const int32_t* status, const int32_t* widths, int nwidths, int32_t* width, int32_t* index) {
  pwpp::LadderWidths lw{};
  lw.n = nwidths;
  for (int i = 0; i < nwidths; ++i) lw.w[i] = widths[i];
  const cudaGraphConditionalHandle h = 0x5eed0000ull + (unsigned) nframes;
  simt::CondSet& c = simt::g_cond;
  c = simt::CondSet{};
  simt::launch("k_ladder_select", dim3(1), pwpp::LS_THREADS, 0, [&] { pwpp::k_ladder_select(nframes, status, lw, width, h); });
  *index = (c.calls == 1 && c.handle == h) ? (int32_t) c.value : -1;
  return PWPP_OK;
}

}  // extern "C"
