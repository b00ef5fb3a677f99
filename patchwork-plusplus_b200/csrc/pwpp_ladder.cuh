// pwpp_ladder.cuh — the width selector of a bound call with a width ladder (pwpp_bind_width_ladder, include/pwpp.h).
//
// A run of such a call is the table kernel, k_ladder_select, then a SWITCH node of the caller's CUDA graph whose body i is the
// call's launch sequence cut at widths.w[i]. k_ladder_select reads the status array the table kernel just wrote, finds L = 1 +
// the last position that runs (0 when none runs) and picks the smallest width w >= max(L, 1); widths.w is strictly increasing
// and its last entry is the call's nframes, so there always is one. It writes w to *d_width and sets the SWITCH node's value to
// w's index. One CTA: each thread takes positions tid, tid + LS_THREADS, ..., then a warp and a CTA max reduce the last one.
#pragma once
#include "pwpp.h"

namespace pwpp {

constexpr int LS_THREADS = 256;

struct LadderWidths {
  int n;                               // 1 .. PWPP_MAX_LADDER_WIDTHS
  int w[PWPP_MAX_LADDER_WIDTHS];       // strictly increasing, w[n - 1] = nframes
};

// A position runs unless the table kernel rejected it: every other status (0 and the three out-of-range codes) is a frame whose
// stream state advances.
__device__ __forceinline__ bool ladder_position_runs(int status) {
  return status != PWPP_FRAME_SKIPPED && status != PWPP_ACTION_INVALID && status != PWPP_STREAM_OUT_OF_RANGE &&
         status != PWPP_STREAM_DUPLICATE;
}

__global__ void __launch_bounds__(LS_THREADS) k_ladder_select(int nf, const int* __restrict__ status, LadderWidths widths,
                                                              int* __restrict__ d_width, cudaGraphConditionalHandle handle) {
  __shared__ int s_last[LS_THREADS / 32];
  const int tid = (int) threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int last = -1;
  for (int f = tid; f < nf; f += LS_THREADS)
    if (ladder_position_runs(status[f])) last = f;
  last = __reduce_max_sync(0xffffffffu, last);
  if (lane == 0) s_last[warp] = last;
  __syncthreads();
  if (tid != 0) return;
  for (int k = 1; k < LS_THREADS / 32; ++k) last = max(last, s_last[k]);
  const int need = max(last + 1, 1);
  int i = 0;
  while (i + 1 < widths.n && widths.w[i] < need) ++i;
  *d_width = widths.w[i];
  cudaGraphSetConditional(handle, (unsigned) i);
}

}  // namespace pwpp
