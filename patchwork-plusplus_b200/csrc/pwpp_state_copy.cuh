// pwpp_state_copy.cuh — stream state on the GPU (pwpp_export_states_device / pwpp_import_states_device, include/pwpp.h): the
// complete state of a list of streams copied between the ctx's state buffers and rows of a caller's blob buffer, inside the
// caller's stream order and so inside a CUDA graph.
//
// A blob row is byte for byte what pwpp_export_state writes: the 16-byte header, the StreamState (the carried plane included)
// and the stream's eight history rows of its set's capacity hcap, back to back (192 + 64 hcap bytes, a multiple of 16). The
// kernels move it in 16-byte words: the header and the state are whole words, and a history word is two doubles, which sit in
// one 16-byte word of the ctx's history rows only when hcap and the row stride are even; otherwise they are moved as two
// 8-byte words. One CTA per list entry; its first thread reads the stream id once, so a list rewritten during the launch
// never splits one entry between two streams.
//
// Import runs in two launches so that two entries naming one stream are resolved without a race: k_state_import_claim
// leaves in claim[s] the smallest entry index naming stream s (an unsigned atomicMin over a table that holds -1, the largest
// unsigned value, between calls); in k_state_import only that entry copies, and it puts -1 back after reading its claim.
// Any other entry naming s reads either the winner's index or, after the reset, -1: never its own index.
#pragma once
#include "pwpp_gle.cuh"
#include "pwpp.h"

namespace pwpp {

struct StateBlobHeader { uint32_t magic, version; int32_t hcap, state_bytes; };
constexpr uint32_t STATE_BLOB_MAGIC = 0x50575354u;  // "PWST"
constexpr int SC_THREADS = 512;
constexpr int SC_UNROLL = 4;                         // 16-byte words a thread has in flight
constexpr int SC_HEAD_WORDS = (int) ((sizeof(StateBlobHeader) + sizeof(StreamState)) / 16);   // header + state: 12 words
constexpr int SC_CLAIM_THREADS = 256;
static_assert(sizeof(StateBlobHeader) == 16 && sizeof(StreamState) % 16 == 0, "blob header and state are whole 16-byte words");

// where the streams' state lives: num_streams StreamStates and 2 x 4 history rows of hist_stride doubles per stream, of which
// stream s uses the first hcap[s]
struct StateStore {
  StreamState* states;
  long long* hist;            // the doubles of the history rows, moved as bits
  int hist_stride;
  const int* hcap;            // [num_streams]
  int num_streams;
};

inline size_t state_blob_bytes(int hcap) { return sizeof(StateBlobHeader) + sizeof(StreamState) + (size_t) 2 * 4 * hcap * sizeof(double); }

__device__ __forceinline__ int4 sc_pack(long long a, long long b) {
  return make_int4((int) (unsigned) a, (int) (a >> 32), (int) (unsigned) b, (int) (b >> 32));
}
__device__ __forceinline__ long long sc_lo(const int4& v) { return (long long) (unsigned) v.x | ((long long) v.y << 32); }
__device__ __forceinline__ long long sc_hi(const int4& v) { return (long long) (unsigned) v.z | ((long long) v.w << 32); }

// history word w (>= SC_HEAD_WORDS) of a blob row: the positions of its two doubles in the stream's history rows
__device__ __forceinline__ void sc_hist_pos(int w, int hcap, int hist_stride, long long& p0, long long& p1) {
  const int k = 2 * (w - SC_HEAD_WORDS);
  const int r0 = k / hcap, c0 = k - r0 * hcap;
  const int r1 = (k + 1) / hcap, c1 = k + 1 - r1 * hcap;
  p0 = (long long) r0 * hist_stride + c0;
  p1 = (long long) r1 * hist_stride + c1;
}

// Entry i = blockIdx.x: stream s = streams[i] into blob row i. status[i] (when status != NULL): PWPP_STATE_OK, or
// PWPP_STATE_SKIPPED (s < 0) / PWPP_STATE_OUT_OF_RANGE (s >= num_streams), and then the row is not written. Bytes of the row
// past the stream's blob size are never written.
__global__ void __launch_bounds__(SC_THREADS) k_state_export(const int* __restrict__ streams, StateStore st, unsigned char* __restrict__ blobs,
                                                             long long blob_stride, int* __restrict__ status) {
  __shared__ int s_stream;
  const int i = blockIdx.x;
  if (threadIdx.x == 0) {
    const int s = streams[i];
    const int code = s < 0 ? PWPP_STATE_SKIPPED : (s >= st.num_streams ? PWPP_STATE_OUT_OF_RANGE : PWPP_STATE_OK);
    if (status) status[i] = code;
    s_stream = code == PWPP_STATE_OK ? s : -1;
  }
  __syncthreads();
  const int s = s_stream;
  if (s < 0) return;
  const int hcap = st.hcap[s], stride = st.hist_stride;
  const int words = SC_HEAD_WORDS + 4 * hcap;
  const bool paired = ((hcap | stride) & 1) == 0;
  const int4* state = reinterpret_cast<const int4*>(st.states + s);
  const long long* hist = st.hist + (long long) s * 8 * stride;
  int4* row = reinterpret_cast<int4*>(blobs + (long long) i * blob_stride);
  for (int w0 = threadIdx.x; w0 < words; w0 += SC_THREADS * SC_UNROLL) {
    int4 v[SC_UNROLL];
#pragma unroll
    for (int u = 0; u < SC_UNROLL; ++u) {
      const int w = w0 + u * SC_THREADS;
      if (w >= words) break;
      if (w == 0) {
        v[u] = make_int4((int) STATE_BLOB_MAGIC, PWPP_ABI_VERSION, hcap, (int) sizeof(StreamState));
      } else if (w < SC_HEAD_WORDS) {
        v[u] = state[w - 1];
      } else {
        long long p0, p1;
        sc_hist_pos(w, hcap, stride, p0, p1);
        v[u] = paired ? *reinterpret_cast<const int4*>(hist + p0) : sc_pack(hist[p0], hist[p1]);
      }
    }
#pragma unroll
    for (int u = 0; u < SC_UNROLL; ++u) {
      const int w = w0 + u * SC_THREADS;
      if (w >= words) break;
      row[w] = v[u];
    }
  }
}

// First import launch: one thread per entry; claim[s] becomes the smallest index of the entries naming stream s.
__global__ void __launch_bounds__(SC_CLAIM_THREADS) k_state_import_claim(int n, const int* __restrict__ streams, int num_streams, int* __restrict__ claim) {
  const int i = blockIdx.x * SC_CLAIM_THREADS + threadIdx.x;
  if (i >= n) return;
  const int s = streams[i];
  if (s >= 0 && s < num_streams) atomicMin(reinterpret_cast<unsigned*>(claim + s), (unsigned) i);
}

// Second import launch, entry i = blockIdx.x: blob row i into stream s = streams[i] when entry i holds the claim of s and the
// row's header is one pwpp_import_state accepts for s (magic, PWPP_ABI_VERSION, the hcap of s's set, sizeof(StreamState)).
// status[i] (when status != NULL): PWPP_STATE_OK, PWPP_STATE_SKIPPED (s < 0, nothing read), PWPP_STATE_OUT_OF_RANGE
// (s >= num_streams), PWPP_STATE_DUPLICATE (an earlier entry names s) or PWPP_STATE_BLOB_MISMATCH (s untouched).
__global__ void __launch_bounds__(SC_THREADS) k_state_import(const int* __restrict__ streams, StateStore st, const unsigned char* __restrict__ blobs,
                                                             long long blob_stride, int* __restrict__ claim, int* __restrict__ status) {
  __shared__ int s_stream;
  const int i = blockIdx.x;
  const int4* row = reinterpret_cast<const int4*>(blobs + (long long) i * blob_stride);
  if (threadIdx.x == 0) {
    const int s = streams[i];
    int code = PWPP_STATE_OK;
    if (s < 0) {
      code = PWPP_STATE_SKIPPED;
    } else if (s >= st.num_streams) {
      code = PWPP_STATE_OUT_OF_RANGE;
    } else if (*(volatile int*) (claim + s) != i) {
      code = PWPP_STATE_DUPLICATE;
    } else {
      claim[s] = -1;
      const int4 h = row[0];
      if ((unsigned) h.x != STATE_BLOB_MAGIC || h.y != PWPP_ABI_VERSION || h.z != st.hcap[s] || h.w != (int) sizeof(StreamState))
        code = PWPP_STATE_BLOB_MISMATCH;
    }
    if (status) status[i] = code;
    s_stream = code == PWPP_STATE_OK ? s : -1;
  }
  __syncthreads();
  const int s = s_stream;
  if (s < 0) return;
  const int hcap = st.hcap[s], stride = st.hist_stride;
  const int words = SC_HEAD_WORDS + 4 * hcap;
  const bool paired = ((hcap | stride) & 1) == 0;
  int4* state = reinterpret_cast<int4*>(st.states + s);
  long long* hist = st.hist + (long long) s * 8 * stride;
  for (int w0 = 1 + (int) threadIdx.x; w0 < words; w0 += SC_THREADS * SC_UNROLL) {
    int4 v[SC_UNROLL];
#pragma unroll
    for (int u = 0; u < SC_UNROLL; ++u) {
      const int w = w0 + u * SC_THREADS;
      if (w >= words) break;
      v[u] = row[w];
    }
#pragma unroll
    for (int u = 0; u < SC_UNROLL; ++u) {
      const int w = w0 + u * SC_THREADS;
      if (w >= words) break;
      if (w < SC_HEAD_WORDS) {
        state[w - 1] = v[u];
      } else {
        long long p0, p1;
        sc_hist_pos(w, hcap, stride, p0, p1);
        if (paired) {
          *reinterpret_cast<int4*>(hist + p0) = v[u];
        } else {
          hist[p0] = sc_lo(v[u]);
          hist[p1] = sc_hi(v[u]);
        }
      }
    }
  }
}

}  // namespace pwpp
