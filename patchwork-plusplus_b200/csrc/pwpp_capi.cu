// pwpp_capi.cu — implementation of the C-ABI declared in include/pwpp.h (libpwpp_b200.so).
// Host side only orchestrates: every stage of estimateGround() runs in the kernels of pwpp_kernels.cuh.
// There is no CPU fallback; without a CUDA device pwpp_create() fails with PWPP_ERR_NO_DEVICE.
#include <cuda_runtime.h>

#include <sched.h>

#include <algorithm>
#include <cctype>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "pwpp.h"
#include "pwpp_kernels.cuh"
#include "pwpp_records.cuh"
#include "pwpp_tuning.h"
#include "pwpp_host.hpp"

using namespace pwpp;

static_assert(sizeof(BinFit) == sizeof(pwpp_bin_result), "BinFit must mirror pwpp_bin_result");

namespace {

thread_local std::string g_last_error;

// integer experiment switch from the environment, clamped to [lo, hi]
int env_int(const char* name, int dflt, int lo, int hi) {
  const char* e = std::getenv(name);
  if (!e || !*e) return dflt;
  const long v = std::strtol(e, nullptr, 10);
  return (int) (v < lo ? lo : (v > hi ? hi : v));
}

int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

#define CU_TRY(expr)                                                                                         \
  do {                                                                                                       \
    cudaError_t _e = (expr);                                                                                 \
    if (_e != cudaSuccess) {                                                                                 \
      return fail(PWPP_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" + __FILE__ + ":" + std::to_string(__LINE__) + ")"); \
    }                                                                                                        \
  } while (0)

unsigned long long g_alloc_gen = 0;   // bumped whenever a device buffer moves: captured CUDA graphs hold the old pointers

// InGraphs = false: a buffer no captured launch sequence reads (its moves leave the graphs valid)
template <typename T, bool InGraphs = true>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;  // elements
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (InGraphs) ++g_alloc_gen;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = n + n / 8 + 64;
    cudaError_t e = cudaMalloc(&p, want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};
template <typename T>
struct PinBuf {
  T* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    size_t want = n + n / 8 + 64;
    cudaError_t e = cudaMallocHost(&p, want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

}  // namespace

// N x cols column-major (an Eigen::MatrixXf, reference patchworkpp.h:152) -> packed float4 {x, y, z, intensity | 0}
__global__ void k_repack_colmajor(const float* __restrict__ src, long long n, int cols, float4* __restrict__ dst) {
  const long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = make_float4(src[i], src[n + i], src[2 * n + i], cols == 4 ? src[3 * n + i] : 0.f);
}

// packed N x 3 rows on the device (the ROS node's conversion, reference ros/src/Utils.hpp:158-172) -> float4 {x, y, z, 0}
__global__ void k_pad_xyz(const float* __restrict__ src, long long n, float4* __restrict__ dst) {
  const long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = make_float4(src[3 * i], src[3 * i + 1], src[3 * i + 2], 0.f);
}

typedef void (*FitKernel)(const float4*, FrameTable, const StreamState*, GeometrySets, AlgoParamSets, int, const int*, WorkQueues, int*, BinFit*);
struct FitLaunch {
  FitKernel fn = nullptr;
  int grid = 0, threads = 0;
  size_t smem = 0;
};

constexpr int NUM_SIDE = 6;

struct pwpp_ctx {
  // parameter sets (pwpp_create: one) and the set of every stream; the kernels get the set records by value
  int num_sets = 1;
  GeometrySets gs;                          // gs.nbs: the largest bin count of the sets, stride of the per-frame bin arrays
  AlgoParamSets aps;
  bool set_fast[MAX_PARAM_SETS] = {};       // build_geometry: the fp32 binning filter is exact for the set's geometry
  int set_hcap[MAX_PARAM_SETS] = {};        // history row capacity of the set (history_cap)
  std::vector<int> stream_set;              // [num_streams]
  int device = 0;
  int num_streams = 0;
  int nbp = 0;          // padded number of bins incl. pseudo-bins, of the set with the most bins
  int hist_stride = 0;  // row stride of d_hist in doubles: the largest set_hcap
  // kernel-variant switches, read from the environment when the context is created (see pwpp_create)
  int sw_front = 1, sw_patch = 0, small_call_frames = 0;
  bool sw_serial_fit = false, front_dense_ok = false;
  cudaStream_t stream = nullptr, stream_h2d = nullptr, stream_d2h = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_begin = nullptr, ev_end = nullptr;
  bool call_times_valid = false;
  cudaEvent_t stage_ev[PWPP_NUM_STAGES + 1] = {};
  cudaStream_t side[NUM_SIDE] = {};       // one side stream per patch-size class: its fit kernel, then its sort (reference order)
  cudaEvent_t ev_fork = nullptr, ev_fit[NUM_SIDE] = {}, ev_join[NUM_SIDE] = {};
  bool profiling = false, stage_valid = false;
  long long launches = 0;

  // persistent per-stream state
  DevBuf<StreamState> d_states;
  DevBuf<StreamState> d_states_init;  // constructor state of every stream (reset source)
  DevBuf<double> d_hist;

  // per-call work buffers
  DevBuf<float4> d_in;            // host path only
  DevBuf<float> d_cm;             // host path: column-major frames as uploaded, repacked on the device
  DevBuf<long long> d_pt_off;     // [F+1]
  DevBuf<int> d_chunk_off;        // [F+1]
  DevBuf<int> d_stream;           // [F] stream of every frame of the call
  DevBuf<int> d_pset;             // [F] parameter set of every frame of the call
  DevBuf<unsigned short> d_bin_ids;
  DevBuf<unsigned short> d_chist;
  DevBuf<unsigned int> d_cbase;
  DevBuf<int> d_bin_off;          // [F][nbp+1]
  DevBuf<float4> d_sorted;
  DevBuf<int> d_part;
  DevBuf<BinFit> d_fits;          // [F][nbins]
  DevBuf<BinSeg> d_segs;          // [F][nbins+3]
  DevBuf<int4> d_wq_items[NUM_CLASSES];  // fit work queues
  DevBuf<int> d_wq_ctr;           // [2*NUM_CLASSES + ORD_NUM_HEADS]: counts, heads, the heads of the five k_order launches
  DevBuf<unsigned char> d_labels; // reference-order output only: what became of every point of a fitted patch
  int order_mode = 0;             // PWPP_ORDER_*
  FitLaunch fit[NUM_CLASSES];   // persistent fit kernel of every patch-size class (variant chosen in pwpp_create)
  FitLaunch fit_small[NUM_CLASSES];   // the same for calls of at most small_call_frames frames (one CTA per patch above 512 points)
  int max_sectors = 0;
  FitLaunch order_k[ORD_NUM_HEADS];   // k_order_cta<512, X>, <512, L3>, <256, L2>, <128, L1>, k_order_warp (same argument list as the fit kernels' type is not needed: launched by name)
  DevBuf<int> d_out_idx;
  DevBuf<int> d_counts;           // [3][F]: num_ground, num_patches, num_dropped (F = frames of the call)
  DevBuf<float> d_centers, d_normals;  // [F][nbins][3]
  DevBuf<float> d_xyz;            // gather scratch
  DevBuf<unsigned char> d_raw;    // pwpp_estimate_host_records: the frames' records as uploaded, unpacked on the device
  DevBuf<RecordFrame> d_rec;      // [F] record table of a records call
  // record results (pwpp_*_record_results), reserved by the first call that asks for them
  DevBuf<unsigned char, false> d_rec_out;   // every frame's ground and non-ground records, region f at rec_off[f]
  DevBuf<long long, false> d_rec_off;       // [F+1]

  PinBuf<float4> h_in;
  PinBuf<long long> h_pt_off_buf[2];      // double-buffered: a call never waits for the previous call's upload
  PinBuf<int> h_chunk_off_buf[2];
  PinBuf<int> h_stream_buf[2];
  PinBuf<int> h_pset_buf[2];
  PinBuf<RecordFrame> h_rec_buf[2];
  PinBuf<unsigned char> h_raw;            // page-locked staging of pageable records
  PinBuf<long long> h_rec_off;            // upload of rec_off; ev_rec_off marks when the copy has read it
  PinBuf<unsigned char> h_rec_out;        // host view of d_rec_out
  cudaEvent_t ev_rec_off = nullptr;
  cudaEvent_t tab_ev[2] = {nullptr, nullptr};
  int tab_cur = 0;
  std::vector<int> chunk_off;             // host copy of the current call's chunk table
  std::vector<int> frame_set;             // host copy of the current call's set table
  // Frames of one stream are sequentially dependent (k_gle of one frame writes what the next one reads), so a call is
  // launched as runs of consecutive frames with pairwise distinct streams: frames [runs[r], runs[r + 1]) are run r.
  std::vector<int> runs;
  std::vector<int> identity;              // [num_streams] 0, 1, 2, ...: the stream table of pwpp_estimate_host / _device
  std::vector<int> last_pos;              // [num_streams] scratch of the run split, -1 between calls
  PinBuf<int> h_out_idx;
  PinBuf<int> h_counts;
  PinBuf<float> h_centers, h_normals;

  // description of the last call
  int last_nframes = 0;
  long long last_total = 0;
  std::vector<long long> pt_off;  // host copy
  const float4* last_pts = nullptr;  // device pointer of the input of the last call
  bool counts_fetched = false, idx_fetched = false, patches_fetched = false;
  std::vector<RecordFrame> last_recs;     // record table of the last call when it took records (empty otherwise)
  std::vector<long long> rec_off;         // [F+1] byte offsets of the record result regions (set by the gather)
  bool rec_gathered = false, rec_fetched = false;
  double last_time_us = 0.0;
  cudaStream_t last_stream = nullptr;

  // small calls (the reference's one-frame-per-call pattern): the launch sequence replayed as a CUDA graph
  struct GraphKey { int nf, call_frames, has_intensity, chunks, fast; unsigned long long gen; const void* pts; };
  cudaGraphExec_t gexec[2] = {nullptr, nullptr};
  GraphKey gkey[2] = {};
  long long glaunches[2] = {0, 0};
  int sw_graph = 1;
};

namespace {

int validate_params(const pwpp_params* p) {
  if (!p) return fail(PWPP_ERR_INVALID_ARG, "params is NULL");
  if (p->num_zones != PWPP_NUM_ZONES) return fail(PWPP_ERR_UNSUPPORTED, "num_zones must be 4 (the reference hard-wires four zones, patchworkpp.h:127-134)");
  if (p->num_rings_of_interest < 0 || p->num_rings_of_interest > PWPP_MAX_RINGS_OF_INTEREST)
    return fail(PWPP_ERR_UNSUPPORTED, "num_rings_of_interest must be in [0,4] (patchworkpp.h:174-175 holds 4 histories)");
  if (p->num_min_pts < 0) return fail(PWPP_ERR_UNSUPPORTED, "num_min_pts must be >= 0");
  if (p->num_iter < 1 || p->num_iter > MAX_RVPF) return fail(PWPP_ERR_UNSUPPORTED, "num_iter must be in [1,8]");
  if (p->num_lpr < 1 || p->num_lpr > MAX_LPR) return fail(PWPP_ERR_UNSUPPORTED, "num_lpr must be in [1,64]");
  if (!(p->th_seeds > 0) || !(p->th_seeds_v > 0)) return fail(PWPP_ERR_UNSUPPORTED, "th_seeds and th_seeds_v must be > 0");
  if (!(p->max_range > p->min_range) || !(p->min_range >= 0)) return fail(PWPP_ERR_INVALID_ARG, "need 0 <= min_range < max_range");
  if (p->max_flatness_storage < 1 || p->max_elevation_storage < 1) return fail(PWPP_ERR_INVALID_ARG, "max_*_storage must be >= 1");
  long long nb = 0;
  for (int k = 0; k < 4; ++k) {
    if (p->num_rings_each_zone[k] < 1 || p->num_sectors_each_zone[k] < 1 || p->num_sectors_each_zone[k] > 1024)
      return fail(PWPP_ERR_UNSUPPORTED, "rings per zone must be >= 1 and sectors per zone in [1,1024]");
    nb += (long long) p->num_rings_each_zone[k] * p->num_sectors_each_zone[k];
  }
  if (nb + PW_NUM_PSEUDO > 4096) return fail(PWPP_ERR_UNSUPPORTED, "more than 4093 bins are not supported");
  return PWPP_OK;
}

// The dynamic shared-memory limit is an attribute of the kernel, shared by every context of the process: a context only ever
// raises it, so that a context whose geometry needs less (fewer bins, fewer sectors) does not break the launches of one that
// needs more.
template <typename F>
cudaError_t raise_smem_limit(F* fn, size_t bytes) {
  cudaFuncAttributes a;
  const cudaError_t e = cudaFuncGetAttributes(&a, (const void*) fn);
  if (e != cudaSuccess) return e;
  if ((size_t) a.maxDynamicSharedSizeBytes >= bytes) return cudaSuccess;
  return cudaFuncSetAttribute((const void*) fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) bytes);
}

int bind_device(pwpp_ctx* ctx) {
  CU_TRY(cudaSetDevice(ctx->device));
  return PWPP_OK;
}

// Checks the stream table of a call: 1 <= nframes <= 65535 (a grid dimension of the per-frame kernels), every id a stream of
// the ctx. Nothing is launched and no state changes when it fails.
int check_streams(const pwpp_ctx* ctx, int nframes, const int32_t* streams) {
  if (!streams) return fail(PWPP_ERR_INVALID_ARG, "streams is NULL");
  if (nframes < 1 || nframes > 65535) return fail(PWPP_ERR_INVALID_ARG, "nframes must be in [1, 65535]");
  for (int f = 0; f < nframes; ++f)
    if (streams[f] < 0 || streams[f] >= ctx->num_streams)
      return fail(PWPP_ERR_INVALID_ARG, "stream id " + std::to_string(streams[f]) + " of frame " + std::to_string(f) + " is outside [0, num_streams)");
  return PWPP_OK;
}

// Splits a call into maximal runs of consecutive frames whose streams are pairwise distinct (ctx->runs).
void split_runs(pwpp_ctx* ctx, int nframes, const int32_t* streams) {
  ctx->runs.assign(1, 0);
  for (int f = 0; f < nframes; ++f) {
    int& p = ctx->last_pos[streams[f]];
    if (p >= ctx->runs.back()) ctx->runs.push_back(f);   // the stream already has a frame in the current run
    p = f;
  }
  ctx->runs.push_back(nframes);
  for (int f = 0; f < nframes; ++f) ctx->last_pos[streams[f]] = -1;
}

// Sizes the work buffers for a call over nframes frames (ctx->pt_off filled), uploads the frame tables (points, chunks,
// stream of every frame and, for a records call, the record table) and splits the call into runs.
int prepare_call(pwpp_ctx* ctx, int nframes, const int32_t* streams, cudaStream_t s, const RecordFrame* recs = nullptr) {
  const long long total = ctx->pt_off[nframes];
  int total_chunks = 0;
  ctx->tab_cur ^= 1;
  const int tb = ctx->tab_cur;
  PinBuf<long long>& h_pt_off = ctx->h_pt_off_buf[tb];
  PinBuf<int>& h_chunk_off = ctx->h_chunk_off_buf[tb];
  PinBuf<int>& h_stream = ctx->h_stream_buf[tb];
  PinBuf<int>& h_pset = ctx->h_pset_buf[tb];
  CU_TRY(cudaEventSynchronize(ctx->tab_ev[tb]));   // upload issued two calls ago: long finished
  CU_TRY(h_pt_off.reserve(nframes + 1));
  CU_TRY(h_chunk_off.reserve(nframes + 1));
  CU_TRY(h_stream.reserve(nframes));
  CU_TRY(h_pset.reserve(nframes));
  std::memcpy(h_stream.p, streams, (size_t) nframes * sizeof(int));
  ctx->frame_set.resize(nframes);
  for (int f = 0; f < nframes; ++f) h_pset.p[f] = ctx->frame_set[f] = ctx->stream_set[streams[f]];
  split_runs(ctx, nframes, streams);
  ctx->chunk_off.assign(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) {
    const long long n = ctx->pt_off[f + 1] - ctx->pt_off[f];
    if (n < 0 || n > 0x7fffffffLL - CHUNK_PTS) return fail(PWPP_ERR_INVALID_ARG, "frame size out of range");
    h_pt_off.p[f] = ctx->pt_off[f];
    h_chunk_off.p[f] = total_chunks;
    ctx->chunk_off[f] = total_chunks;
    total_chunks += (int) ((n + CHUNK_PTS - 1) / CHUNK_PTS);
  }
  h_pt_off.p[nframes] = total;
  h_chunk_off.p[nframes] = total_chunks;
  ctx->chunk_off[nframes] = total_chunks;
  const int nb = ctx->gs.nbs, nbp = ctx->nbp, nb_all = nb + PW_NUM_PSEUDO;
  CU_TRY(ctx->d_pt_off.reserve(nframes + 1));
  CU_TRY(ctx->d_chunk_off.reserve(nframes + 1));
  CU_TRY(ctx->d_stream.reserve(nframes));
  CU_TRY(ctx->d_pset.reserve(nframes));
  CU_TRY(ctx->d_bin_ids.reserve((size_t) total));
  CU_TRY(ctx->d_chist.reserve((size_t) total_chunks * nbp));
  CU_TRY(ctx->d_cbase.reserve((size_t) total_chunks * nbp));
  CU_TRY(ctx->d_bin_off.reserve((size_t) nframes * (nbp + 1)));
  CU_TRY(ctx->d_sorted.reserve((size_t) total));
  CU_TRY(ctx->d_part.reserve((size_t) total));
  if (ctx->order_mode) CU_TRY(ctx->d_labels.reserve((size_t) total));
  CU_TRY(ctx->d_fits.reserve((size_t) nframes * nb));
  CU_TRY(ctx->d_segs.reserve((size_t) nframes * nb_all));
  for (int c = 0; c < NUM_CLASSES; ++c) CU_TRY(ctx->d_wq_items[c].reserve((size_t) nframes * nb));
  CU_TRY(ctx->d_out_idx.reserve((size_t) total));
  CU_TRY(ctx->d_counts.reserve((size_t) 3 * nframes));
  CU_TRY(ctx->d_centers.reserve((size_t) nframes * nb * 3));
  CU_TRY(ctx->d_normals.reserve((size_t) nframes * nb * 3));
  CU_TRY(cudaMemcpyAsync(ctx->d_pt_off.p, h_pt_off.p, (nframes + 1) * sizeof(long long), cudaMemcpyHostToDevice, s));
  CU_TRY(cudaMemcpyAsync(ctx->d_chunk_off.p, h_chunk_off.p, (nframes + 1) * sizeof(int), cudaMemcpyHostToDevice, s));
  CU_TRY(cudaMemcpyAsync(ctx->d_stream.p, h_stream.p, nframes * sizeof(int), cudaMemcpyHostToDevice, s));
  CU_TRY(cudaMemcpyAsync(ctx->d_pset.p, h_pset.p, nframes * sizeof(int), cudaMemcpyHostToDevice, s));
  if (recs) ctx->last_recs.assign(recs, recs + nframes);
  else ctx->last_recs.clear();
  ctx->rec_gathered = ctx->rec_fetched = false;
  if (recs) {
    PinBuf<RecordFrame>& h_rec = ctx->h_rec_buf[tb];
    CU_TRY(h_rec.reserve(nframes));
    CU_TRY(ctx->d_rec.reserve(nframes));
    std::memcpy(h_rec.p, recs, (size_t) nframes * sizeof(RecordFrame));
    CU_TRY(cudaMemcpyAsync(ctx->d_rec.p, h_rec.p, nframes * sizeof(RecordFrame), cudaMemcpyHostToDevice, s));
  }
  CU_TRY(cudaEventRecord(ctx->tab_ev[tb], s));
  ctx->last_nframes = nframes;
  ctx->last_total = total;
  ctx->counts_fetched = ctx->idx_fetched = ctx->patches_fetched = false;
  ctx->stage_valid = false;
  return PWPP_OK;
}

// The fp32 binning filter is used for a launch range only when build_geometry allows it for every set the range names;
// otherwise the range takes the exact kernel. Both bin exactly, so the bins are the same either way.
bool range_fast(const pwpp_ctx* ctx, int f0, int nf) {
  for (int f = f0; f < f0 + nf; ++f)
    if (!ctx->set_fast[ctx->frame_set[f]]) return false;
  return true;
}

// Launches the whole path for frames [f0, f0 + nf) of the prepared call on stream s; the range must not hold two frames of
// one stream (a run or part of one). A frame range is the same launch sequence over per-frame arrays offset by f0 (frame
// tables hold absolute point / chunk positions), which is what lets pwpp_estimate_host pipeline chunks of frames against
// their H2D / D2H copies. Stream state and histories are indexed by the stream table, never by the frame.
int launch_range_impl(pwpp_ctx* ctx, int f0, int nf, const float4* d_pts, int has_intensity, cudaStream_t s, bool prof, int chunks_override) {
  int max_chunks = 0;
  for (int f = f0; f < f0 + nf; ++f) max_chunks = std::max(max_chunks, ctx->chunk_off[f + 1] - ctx->chunk_off[f]);
  if (chunks_override > 0) max_chunks = chunks_override;   // graph capture: grids sized for a range of frame sizes (surplus CTAs exit at once)
  const int nb = ctx->gs.nbs, nbp = ctx->nbp, nb_all = nb + PW_NUM_PSEUDO;   // strides of the per-frame bin arrays (the largest set)
  const int nframes = nf;
  FrameTable ft{ctx->d_pt_off.p + f0, ctx->d_chunk_off.p + f0, ctx->d_stream.p + f0, ctx->d_pset.p + f0};
  const bool fast = range_fast(ctx, f0, nf);
  StreamState* states = ctx->d_states.p;
  double* hist = ctx->d_hist.p;
  int* bin_off = ctx->d_bin_off.p + (size_t) f0 * (nbp + 1);
  BinFit* fits = ctx->d_fits.p + (size_t) f0 * nb;
  BinSeg* segs = ctx->d_segs.p + (size_t) f0 * nb_all;
  float* centers = ctx->d_centers.p + (size_t) f0 * nb * 3;
  float* normals = ctx->d_normals.p + (size_t) f0 * nb * 3;
  CU_TRY(cudaMemsetAsync(ctx->d_wq_ctr.p, 0, (2 * NUM_CLASSES + ORD_NUM_HEADS) * sizeof(int), s));
  int stage = 0;
#define STAGE_MARK() do { if (prof) CU_TRY(cudaEventRecord(ctx->stage_ev[stage], s)); ++stage; } while (0)
  STAGE_MARK();
  WorkQueues wq;
  for (int c = 0; c < NUM_CLASSES; ++c) wq.items[c] = ctx->d_wq_items[c].p;
  wq.count = ctx->d_wq_ctr.p;
  wq.head = ctx->d_wq_ctr.p + NUM_CLASSES;
  wq.labels = ctx->order_mode ? ctx->d_labels.p : nullptr;
  // A call of a few frames (the reference's pattern is one frame per call) cannot fill the GPU with warp-sized work items: there the
  // latency of the longest patch counts, so patches above 512 points go to the CTA-per-patch kernels, and one frame's cloud is
  // binned by ~30 independent CTAs (the three stand-alone kernels) rather than by the 8 CTAs of one cluster: both shorten
  // the longest kernel of a one-frame call.
  const bool small_call = nframes <= ctx->small_call_frames;
  const FitLaunch* fitk = small_call ? ctx->fit_small : ctx->fit;
  if (ctx->sw_front && !small_call) {
    // one thread-block cluster per frame: binning, scan and stable scatter in one kernel (pwpp_front.cuh)
    if (nframes > 0) {
      // 64 warps per frame for KITTI-sized frames, 128 for dense ones (pwpp_front.cuh)
      const long long mean_front = (ctx->pt_off[f0 + nf] - ctx->pt_off[f0]) / std::max(nf, 1);
      const bool dense = mean_front > 400000 && ctx->front_dense_ok;
      const int nt = dense ? FC_THREADS_DENSE : FC_THREADS;
      const size_t sm_f = front_cluster_smem_bytes(nbp, nt);
      dim3 grid(FC_CS, nframes);
#define FC_ARGS d_pts, ft, states, ctx->gs, ctx->aps, has_intensity, nbp, nb, ctx->d_bin_ids.p, bin_off, wq, fits, ctx->d_sorted.p
      if (dense) {
        if (fast) k_front_cluster<true, CLS_L2_MAX, FC_THREADS_DENSE><<<grid, nt, sm_f, s>>>(FC_ARGS);
        else k_front_cluster<false, CLS_L2_MAX, FC_THREADS_DENSE><<<grid, nt, sm_f, s>>>(FC_ARGS);
      } else {
        if (fast) k_front_cluster<true, CLS_L2_MAX, FC_THREADS><<<grid, nt, sm_f, s>>>(FC_ARGS);
        else k_front_cluster<false, CLS_L2_MAX, FC_THREADS><<<grid, nt, sm_f, s>>>(FC_ARGS);
      }
#undef FC_ARGS
      ++ctx->launches;
    }
    STAGE_MARK(); STAGE_MARK(); STAGE_MARK();
  } else {
    // the three stand-alone kernels (PWPP_FRONT=0)
    if (max_chunks > 0) {
      dim3 grid(max_chunks, nframes);
      const size_t sm_h = nbp * sizeof(unsigned int);
#define HIST_ARGS d_pts, ft, states, ctx->gs, ctx->aps, has_intensity, nbp, ctx->d_bin_ids.p, ctx->d_chist.p
      if (!fast) k_bin_hist<false, 0><<<grid, CHUNK_THREADS, sm_h, s>>>(HIST_ARGS);
      else k_bin_hist<true, 2><<<grid, CHUNK_THREADS, sm_h, s>>>(HIST_ARGS);
#undef HIST_ARGS
      ++ctx->launches;
    }
    STAGE_MARK();
    k_bin_scan<CLS_L2_MAX><<<nframes, 512, (nbp + 1) * sizeof(int), s>>>(ft, nbp, nb, ctx->gs, ctx->aps, ctx->d_chist.p, ctx->d_cbase.p, bin_off, wq, fits);
    ++ctx->launches;
    STAGE_MARK();
    if (max_chunks > 0) {
      dim3 grid(max_chunks, nframes);
      const size_t sm_sc = (size_t) (CHUNK_THREADS / 32) * nbp * sizeof(unsigned int);
      k_scatter<false, 4><<<grid, CHUNK_THREADS, sm_sc, s>>>(d_pts, ft, nbp, ctx->d_bin_ids.p, ctx->d_cbase.p, ctx->d_sorted.p);
      ++ctx->launches;
    }
    STAGE_MARK();
  }
  // persistent fit kernels, one per patch-size class (queues were filled by k_bin_scan). The classes are independent:
  // unless per-stage timing is requested they run on side streams so that the tail of one class (few long patches
  // left) overlaps the start of the next.
#define FIT_ARGS ctx->d_sorted.p, ft, states, ctx->gs, ctx->aps, nbp, bin_off, wq, ctx->d_part.p, fits
  const bool serial_fit = ctx->sw_serial_fit;   // PWPP_SERIAL_FIT: diagnostic switch
  // persistent grids are sized for a full GPU; a small call (one frame per call is the reference's pattern) would launch hundreds
  // of CTAs per class that find their queue empty and, worse, keep the six classes from running side by side: cap the grid
  // by what the call can hold (a frame has at most a few hundred patches)
  auto launch_fit = [&](int c, cudaStream_t st) {
    const FitLaunch& k = fitk[c];
    if (!k.fn) return;
    const long long cap = (long long) nframes * (k.threads <= 128 ? 96 : 48);
    const int grid = (int) std::min<long long>(k.grid, std::max<long long>(1, cap));
    k.fn<<<grid, k.threads, k.smem, st>>>(FIT_ARGS);
    ++ctx->launches;
  };
  // reference emission order inside every fitted patch (pwpp_order.cuh): one launch per class (X, L3, L2, L1 with a CTA sized to the
  // class; M + S one warp per patch). A sort only permutes `part` inside the patches of its own class, so it runs on its class's
  // side stream right behind the fit kernel, beside the other classes' fits and beside k_gle (which only reads the patch records);
  // k_emit joins everything. On a one-frame call the sort of the largest patch and the ring walk of k_gle are
  // both pure latency.
  int* heads = ctx->d_wq_ctr.p + 2 * NUM_CLASSES;
  auto launch_order = [&](int q, cudaStream_t so) {   // q: 0 = X, 1 = L3, 2 = L2, 3 = L1, 4 = M + S
    const int grid = (int) std::min<long long>(ctx->order_k[q].grid, std::max<long long>(1, (long long) nframes * (q == 4 ? 64 : 32)));
    const int th = ctx->order_k[q].threads;
    const size_t sm = ctx->order_k[q].smem;
    switch (q) {
      case 0: k_order_cta<512, 5><<<grid, th, sm, so>>>(ctx->d_sorted.p, wq, heads + q, ctx->d_part.p); break;
      case 1: k_order_cta<512, 4><<<grid, th, sm, so>>>(ctx->d_sorted.p, wq, heads + q, ctx->d_part.p); break;
      case 2: k_order_cta<256, 3><<<grid, th, sm, so>>>(ctx->d_sorted.p, wq, heads + q, ctx->d_part.p); break;
      case 3: k_order_cta<128, 2><<<grid, th, sm, so>>>(ctx->d_sorted.p, wq, heads + q, ctx->d_part.p); break;
      default: k_order_warp<<<grid, th, 0, so>>>(ctx->d_sorted.p, wq, heads + q, ctx->d_part.p); break;
    }
    ++ctx->launches;
  };
  const bool aside = !(prof || serial_fit);
  if (!aside) {
    static const int order[NUM_CLASSES] = {0, 4, 3, 2, 1, 5};   // stage slots: S, L3, L2, L1, M, X
    for (int q = 0; q < NUM_CLASSES; ++q) { launch_fit(order[q], s); STAGE_MARK(); }
    if (ctx->order_mode) for (int q = 0; q < ORD_NUM_HEADS; ++q) launch_order(q, s);
  } else {
    // side stream of every class, longest patches first: L3, L2, L1, M, S, X
    static const int cls_of_side[NUM_SIDE] = {4, 3, 2, 1, 0, 5};
    static const int order_of_side[NUM_SIDE] = {1, 2, 3, 4, -1, 0};   // the sort that follows the fit on that stream (M + S: behind M)
    CU_TRY(cudaEventRecord(ctx->ev_fork, s));
    for (int q = 0; q < NUM_SIDE; ++q) {
      CU_TRY(cudaStreamWaitEvent(ctx->side[q], ctx->ev_fork, 0));
      launch_fit(cls_of_side[q], ctx->side[q]);
      CU_TRY(cudaEventRecord(ctx->ev_fit[q], ctx->side[q]));
    }
    if (ctx->order_mode) {
      for (int q = 0; q < NUM_SIDE; ++q) {
        if (order_of_side[q] < 0) continue;
        if (order_of_side[q] == 4) CU_TRY(cudaStreamWaitEvent(ctx->side[q], ctx->ev_fit[4], 0));   // the warp sort also covers class S (side 4)
        launch_order(order_of_side[q], ctx->side[q]);
        CU_TRY(cudaEventRecord(ctx->ev_join[q], ctx->side[q]));
      }
    }
    for (int q = 0; q < NUM_SIDE; ++q) CU_TRY(cudaStreamWaitEvent(s, ctx->ev_fit[q], 0));   // k_gle needs every fit, no sort
    stage += 6;
  }
#undef FIT_ARGS
  const int call_frames = ctx->last_nframes;   // the count rows are as long as the call
  int* d_ng = ctx->d_counts.p + f0;
  int* d_np = ctx->d_counts.p + call_frames + f0;
  int* d_nd = ctx->d_counts.p + 2 * call_frames + f0;
  {
    const size_t gle_smem = gle_smem_bytes(ctx->max_sectors);
    k_gle<<<nframes, 32, gle_smem, s>>>(ft, states, hist, ctx->hist_stride, ctx->gs, ctx->aps, nbp, ctx->max_sectors, bin_off, fits, segs, d_ng, d_np, centers, normals, d_nd);
    ++ctx->launches;
  }
  STAGE_MARK();
  if (aside && ctx->order_mode) for (int q = 0; q < NUM_SIDE; ++q) if (q != 4) CU_TRY(cudaStreamWaitEvent(s, ctx->ev_join[q], 0));
  if (max_chunks > 0) {
    const long long max_pts = (long long) max_chunks * CHUNK_PTS;   // upper bound of the largest frame of the range
    dim3 grid((unsigned) ((max_pts + (long long) EMIT_TILE * EMIT_WARPS - 1) / ((long long) EMIT_TILE * EMIT_WARPS)), nframes);
    k_emit<<<grid, EMIT_WARPS * 32, 0, s>>>(ft, ctx->gs, nbp, bin_off, fits, segs, ctx->d_part.p, ctx->d_sorted.p, ctx->d_out_idx.p);
    ++ctx->launches;
  }
  STAGE_MARK();
#undef STAGE_MARK
  if (prof) ctx->stage_valid = true;
  CU_TRY(cudaGetLastError());
  ctx->last_pts = d_pts;
  ctx->last_stream = s;
  return PWPP_OK;
}

// Small calls are launch-bound (ten kernels of a few microseconds each plus the fork / join events of the fit kernels): the
// sequence is captured once per (frames, frames of the call, intensity flag, grid size class, binning kernel, buffer generation)
// and replayed as one CUDA graph; it reads the frame tables (stream and set ids included) the current call uploaded. Only for the
// first range of calls whose input sits in the ctx's own upload buffer (the host entry point), so the captured pointers
// stay valid; PWPP_GRAPH=0 switches it off.
constexpr int GRAPH_MAX_FRAMES = 16;
int launch_range(pwpp_ctx* ctx, int f0, int nf, const float4* d_pts, int has_intensity, cudaStream_t s, bool prof) {
  if (prof || !ctx->sw_graph || nf > GRAPH_MAX_FRAMES || f0 != 0 || d_pts != ctx->d_in.p) return launch_range_impl(ctx, f0, nf, d_pts, has_intensity, s, prof, 0);
  int max_chunks = 0;
  for (int f = 0; f < nf; ++f) max_chunks = std::max(max_chunks, ctx->chunk_off[f + 1] - ctx->chunk_off[f]);
  const int capc = std::max(8, (max_chunks + 7) & ~7);
  const int slot = has_intensity ? 1 : 0;
  const pwpp_ctx::GraphKey key{nf, ctx->last_nframes, has_intensity, capc, range_fast(ctx, 0, nf) ? 1 : 0, g_alloc_gen, (const void*) d_pts};
  pwpp_ctx::GraphKey& have = ctx->gkey[slot];
  if (!ctx->gexec[slot] || have.nf != key.nf || have.call_frames != key.call_frames || have.chunks != key.chunks || have.fast != key.fast || have.gen != key.gen ||
      have.pts != key.pts) {
    if (ctx->gexec[slot]) { cudaGraphExecDestroy(ctx->gexec[slot]); ctx->gexec[slot] = nullptr; }
    const long long l0 = ctx->launches;
    CU_TRY(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    const int rc = launch_range_impl(ctx, 0, nf, d_pts, has_intensity, s, false, capc);
    cudaGraph_t graph = nullptr;
    const cudaError_t e = cudaStreamEndCapture(s, &graph);
    if (rc != PWPP_OK || e != cudaSuccess || !graph) {
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      ctx->sw_graph = 0;   // capture is not available here: fall back to plain launches for good
      ctx->launches = l0;
      return launch_range_impl(ctx, 0, nf, d_pts, has_intensity, s, false, 0);
    }
    const cudaError_t e2 = cudaGraphInstantiate(&ctx->gexec[slot], graph, 0);
    cudaGraphDestroy(graph);
    if (e2 != cudaSuccess) { ctx->gexec[slot] = nullptr; ctx->sw_graph = 0; ctx->launches = l0; cudaGetLastError(); return launch_range_impl(ctx, 0, nf, d_pts, has_intensity, s, false, 0); }
    ctx->glaunches[slot] = ctx->launches - l0;
    ctx->launches = l0;
    have = key;
  }
  CU_TRY(cudaGraphLaunch(ctx->gexec[slot], s));
  ctx->launches += ctx->glaunches[slot];
  ctx->last_pts = d_pts;
  ctx->last_stream = s;
  return PWPP_OK;
}

// Optional sub-batching of a big call (PWPP_SUBBATCH_POINTS=n: consecutive launch sequences of at most n points).
// Off by default: each persistent fit kernel already fills the GPU, so splitting a call only adds tails.
long long subbatch_points() {
  static long long v = [] {
    const char* e = std::getenv("PWPP_SUBBATCH_POINTS");
    return e ? std::atoll(e) : (1LL << 62);   // default: one sequence per call
  }();
  return v;
}

// Launches the frames [f0, f1) of the prepared call: one range per run they overlap (stream order serialises the runs).
// *r is the first run that may overlap; calls with increasing f0 pass the same cursor.
int launch_runs(pwpp_ctx* ctx, int f0, int f1, size_t* r, const float4* d_pts, int has_intensity, cudaStream_t s, bool prof) {
  const std::vector<int>& runs = ctx->runs;
  while (*r + 2 < runs.size() && runs[*r + 1] <= f0) ++*r;
  for (size_t q = *r; q + 1 < runs.size() && runs[q] < f1; ++q) {
    const int a = std::max(f0, runs[q]), b = std::min(f1, runs[q + 1]);
    if (a >= b) continue;
    const int rc = launch_range(ctx, a, b - a, d_pts, has_intensity, s, prof);
    if (rc) return rc;
  }
  return PWPP_OK;
}

// Launches the whole prepared call on stream s.
int launch_call(pwpp_ctx* ctx, int nframes, const float4* d_pts, int has_intensity, cudaStream_t s) {
  int rc = PWPP_OK;
  size_t r = 0;
  // per-stage timing covers one launch sequence: a call of several runs is launched, but not timed
  if (ctx->profiling) return launch_runs(ctx, 0, nframes, &r, d_pts, has_intensity, s, ctx->runs.size() == 2);
  const long long cap = subbatch_points();
  int f0 = 0;
  while (f0 < nframes) {
    int f1 = f0 + 1;
    while (f1 < nframes && ctx->pt_off[f1 + 1] - ctx->pt_off[f0] <= cap) ++f1;
    rc = launch_runs(ctx, f0, f1, &r, d_pts, has_intensity, s, false);
    if (rc) return rc;
    f0 = f1;
  }
  return PWPP_OK;
}

int run_path(pwpp_ctx* ctx, int nframes, const int32_t* streams, const float4* d_pts, int has_intensity, cudaStream_t s) {
  const int rc = prepare_call(ctx, nframes, streams, s);
  if (rc) return rc;
  return launch_call(ctx, nframes, d_pts, has_intensity, s);
}

int check_frame(pwpp_ctx* ctx, int f) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (f < 0 || f >= ctx->last_nframes) return fail(PWPP_ERR_INVALID_ARG, "frame index outside the last estimate call");
  return PWPP_OK;
}

int fetch_counts(pwpp_ctx* ctx) {
  if (ctx->counts_fetched) return PWPP_OK;
  int rc = bind_device(ctx);
  if (rc) return rc;
  CU_TRY(ctx->h_counts.reserve((size_t) 3 * ctx->last_nframes));
  CU_TRY(cudaMemcpyAsync(ctx->h_counts.p, ctx->d_counts.p, (size_t) 3 * ctx->last_nframes * sizeof(int), cudaMemcpyDeviceToHost, ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  ctx->counts_fetched = true;
  return PWPP_OK;
}
int fetch_indices(pwpp_ctx* ctx) {
  if (ctx->idx_fetched) return PWPP_OK;
  int rc = fetch_counts(ctx);
  if (rc) return rc;
  CU_TRY(ctx->h_out_idx.reserve((size_t) std::max<long long>(ctx->last_total, 1)));
  if (ctx->last_total > 0)
    CU_TRY(cudaMemcpyAsync(ctx->h_out_idx.p, ctx->d_out_idx.p, (size_t) ctx->last_total * sizeof(int), cudaMemcpyDeviceToHost, ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  ctx->idx_fetched = true;
  return PWPP_OK;
}
int fetch_patches(pwpp_ctx* ctx) {
  if (ctx->patches_fetched) return PWPP_OK;
  int rc = fetch_counts(ctx);
  if (rc) return rc;
  const size_t n = (size_t) ctx->last_nframes * ctx->gs.nbs * 3;
  CU_TRY(ctx->h_centers.reserve(n));
  CU_TRY(ctx->h_normals.reserve(n));
  CU_TRY(cudaMemcpyAsync(ctx->h_centers.p, ctx->d_centers.p, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->last_stream));
  CU_TRY(cudaMemcpyAsync(ctx->h_normals.p, ctx->d_normals.p, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  ctx->patches_fetched = true;
  return PWPP_OK;
}

inline int frame_n(const pwpp_ctx* ctx, int f) { return (int) (ctx->pt_off[f + 1] - ctx->pt_off[f]); }
// fetched count of frame f: q = 0 ground points, 1 patches, 2 dropped points
inline int count_of(const pwpp_ctx* ctx, int q, int f) { return ctx->h_counts.p[(size_t) q * ctx->last_nframes + f]; }

}  // namespace

extern "C" {

void pwpp_params_default(pwpp_params* p) {
  if (!p) return;
  std::memset(p, 0, sizeof(*p));
  p->verbose = 0; p->enable_RNR = 1; p->enable_RVPF = 1; p->enable_TGR = 1;            // patchworkpp.h:80-83
  p->num_iter = 3; p->num_lpr = 20; p->num_min_pts = 10; p->num_zones = 4; p->num_rings_of_interest = 4;  // :85-89
  p->RNR_ver_angle_thr = -15.0; p->RNR_intensity_thr = 0.2;                             // :91-92
  p->sensor_height = 1.723; p->th_seeds = 0.125; p->th_dist = 0.125; p->th_seeds_v = 0.25; p->th_dist_v = 0.1;  // :94-98
  p->max_range = 80.0; p->min_range = 2.7; p->uprightness_thr = 0.707; p->adaptive_seed_selection_margin = -1.2;  // :99-102
  p->intensity_thr = 0.0;
  const int sectors[4] = {16, 32, 54, 32}, rings[4] = {2, 4, 4, 4};                     // :104-105
  for (int k = 0; k < 4; ++k) { p->num_sectors_each_zone[k] = sectors[k]; p->num_rings_each_zone[k] = rings[k]; p->elevation_thr[k] = 0; p->flatness_thr[k] = 0; }
  p->max_flatness_storage = 1000; p->max_elevation_storage = 1000;                      // :107-108
}

const char* pwpp_last_error(void) { return g_last_error.c_str(); }
int pwpp_abi_version(void) { return PWPP_ABI_VERSION; }
int pwpp_num_bins(const pwpp_ctx* ctx) { return ctx ? ctx->gs.nbs : 0; }
int pwpp_stream_num_bins(const pwpp_ctx* ctx, int s) {
  if (!ctx || s < 0 || s >= ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "bad stream index");
  return ctx->gs.g[ctx->stream_set[s]].nbins;
}
int pwpp_stream_set(const pwpp_ctx* ctx, int s) {
  if (!ctx || s < 0 || s >= ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "bad stream index");
  return ctx->stream_set[s];
}

// The context of pwpp_create and pwpp_create_sets: sets and stream_set (NULL: every stream on set 0) are validated.
static int create_impl(const pwpp_params* sets, int num_sets, const int32_t* stream_set, int device, int num_streams, int64_t max_points_per_frame,
                       pwpp_ctx** out) {
  int rc = PWPP_OK;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(PWPP_ERR_NO_DEVICE, std::string("no CUDA device available (") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count 0") +
                                        "); this library has no CPU path");
  if (device < 0 || device >= ndev) return fail(PWPP_ERR_INVALID_ARG, "device index out of range");
  pwpp_ctx* ctx = new pwpp_ctx();
  ctx->device = device;
  ctx->num_streams = num_streams;
  ctx->identity.resize(num_streams);
  for (int i = 0; i < num_streams; ++i) ctx->identity[i] = i;
  ctx->last_pos.assign(num_streams, -1);
  ctx->stream_set.assign(num_streams, 0);
  if (stream_set) ctx->stream_set.assign(stream_set, stream_set + num_streams);
  ctx->num_sets = num_sets;
  ctx->gs.nbs = 0;
  int max_sectors = 0;
  for (int k = 0; k < num_sets; ++k) {
    build_geometry(sets[k], ctx->gs.g[k], ctx->aps.a[k], ctx->set_fast[k]);
    ctx->set_hcap[k] = history_cap(ctx->gs.g[k], ctx->aps.a[k]);
    ctx->gs.nbs = std::max(ctx->gs.nbs, ctx->gs.g[k].nbins);
    ctx->hist_stride = std::max(ctx->hist_stride, ctx->set_hcap[k]);
    for (int z = 0; z < 4; ++z) max_sectors = std::max(max_sectors, ctx->gs.g[k].num_sectors[z]);
  }
  ctx->sw_serial_fit = env_int("PWPP_SERIAL_FIT", 0, 0, 1) != 0;       // diagnostic: the fit kernels one after another on the call's stream
  ctx->sw_front = env_int("PWPP_FRONT", PWPP_FRONT_DEFAULT, 0, 1);        // 1: cluster-per-frame front end, 0: k_bin_hist + k_bin_scan + k_scatter
  ctx->sw_patch = env_int("PWPP_FIT_PATCH", PWPP_FIT_PATCH_DEFAULT, 0, 1);   // 1: patches above 512 points on k_fit_patch
  ctx->sw_graph = env_int("PWPP_GRAPH", 1, 0, 1);
  ctx->small_call_frames = env_int("PWPP_SMALL_CALL", PWPP_SMALL_CALL_DEFAULT, 0, 64);   // calls of at most this many frames take the small-call kernels (0: never)
  ctx->nbp = ((ctx->gs.nbs + PW_NUM_PSEUDO + 31) / 32) * 32;
  ctx->max_sectors = max_sectors;
#define CU_TRY_CTX(expr)                                                                                  \
  do {                                                                                                    \
    cudaError_t _e = (expr);                                                                              \
    if (_e != cudaSuccess) {                                                                              \
      std::string m = std::string(#expr) + ": " + cudaGetErrorString(_e);                                 \
      pwpp_destroy(ctx);                                                                                  \
      return fail(PWPP_ERR_CUDA, m);                                                                      \
    }                                                                                                     \
  } while (0)
  CU_TRY_CTX(cudaSetDevice(device));
  CU_TRY_CTX(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  CU_TRY_CTX(cudaStreamCreateWithFlags(&ctx->stream_h2d, cudaStreamNonBlocking));
  CU_TRY_CTX(cudaStreamCreateWithFlags(&ctx->stream_d2h, cudaStreamNonBlocking));
  CU_TRY_CTX(cudaEventCreate(&ctx->ev0));
  CU_TRY_CTX(cudaEventCreate(&ctx->ev1));
  CU_TRY_CTX(cudaEventCreate(&ctx->ev_begin));
  CU_TRY_CTX(cudaEventCreate(&ctx->ev_end));
  for (int i = 0; i <= PWPP_NUM_STAGES; ++i) CU_TRY_CTX(cudaEventCreate(&ctx->stage_ev[i]));
  for (int i = 0; i < 2; ++i) CU_TRY_CTX(cudaEventCreateWithFlags(&ctx->tab_ev[i], cudaEventDisableTiming));
  CU_TRY_CTX(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
  for (int q = 0; q < NUM_SIDE; ++q) {
    CU_TRY_CTX(cudaStreamCreateWithFlags(&ctx->side[q], cudaStreamNonBlocking));
    CU_TRY_CTX(cudaEventCreateWithFlags(&ctx->ev_fit[q], cudaEventDisableTiming));
    CU_TRY_CTX(cudaEventCreateWithFlags(&ctx->ev_join[q], cudaEventDisableTiming));
  }
  CU_TRY_CTX(ctx->d_states.reserve(num_streams));
  CU_TRY_CTX(ctx->d_states_init.reserve(num_streams));
  {
    std::vector<StreamState> v(num_streams);
    for (int i = 0; i < num_streams; ++i) init_state(sets[ctx->stream_set[i]], v[i]);   // the constructor state of the stream's set
    CU_TRY_CTX(cudaMemcpy(ctx->d_states_init.p, v.data(), v.size() * sizeof(StreamState), cudaMemcpyHostToDevice));
  }
  CU_TRY_CTX(ctx->d_hist.reserve((size_t) num_streams * 2 * 4 * ctx->hist_stride));
  CU_TRY_CTX(ctx->d_counts.reserve((size_t) 3 * num_streams));
  CU_TRY_CTX(ctx->d_wq_ctr.reserve(2 * NUM_CLASSES + ORD_NUM_HEADS));
  {
    cudaDeviceProp prop;
    CU_TRY_CTX(cudaGetDeviceProperties(&prop, device));
    // Fit kernel of every patch-size class:
    //   S  <= 64      k_fit_resident: 8 lanes x 8 register slots per patch
    //   M  <= 512     k_fit_warp, patch staged in shared memory, plane + moment sums in shared memory, 3 CTAs/SM
    //   L1 <= 2048    k_fit_warp streaming from L2, the same (4 CTAs/SM at 64 registers and a cp.async chunk ring were slower)
    //                 Both are instruction-fetch sensitive (125 KB of code each): the passes take TWO rows per batch, the LPR scans two
    //                 loads in flight (more rows per batch or more loads in flight were slower).
    //                 PWPP_FIT_PATCH=1 (and calls of <= 4 frames): k_fit_patch, one patch per CTA of 4 / 8 / 16 warps held in registers
    //   L2 <= 4096    k_fit_cta, plane in shared memory, 3 CTAs/SM
    //   L3 <= 8192    k_fit_cta, 2 CTAs/SM
    //   X  >  8192    k_fit_big (dense sensors)
    const size_t sm_m = FITW_WARPS * CLS_M_MAX * sizeof(float4), sm_l2 = 3 * 4096 * sizeof(float), sm_l3 = 3 * 8192 * sizeof(float);
    ctx->fit[0] = {k_fit_resident<8, 8, 0, 2>, 0, FIT_THREADS, 0};
    ctx->fit[1] = {k_fit_warp<true, 1, 1, 2, 3, false, true>, 0, FITW_WARPS * 32, sm_m};
    ctx->fit[2] = {k_fit_warp<false, 2, 2, 2, 3, false, true>, 0, FITW_WARPS * 32, 0};
    ctx->fit[3] = {k_fit_cta<4096, 3, 3, 8, true, true>, 0, FIT_THREADS, sm_l2};
    ctx->fit[4] = {k_fit_cta<8192, 4, 2, 8, true>, 0, FIT_THREADS, sm_l3};
    ctx->fit[5] = {k_fit_big<16, 1, true>, 0, 512, 0};
    if (ctx->sw_patch) {
      ctx->fit[2] = {k_fit_patch<4, 4, 2>, 0, 4 * 32, (size_t) 4 * FP_STG * sizeof(float4)};
      ctx->fit[3] = {k_fit_patch<8, 2, 3>, 0, 8 * 32, (size_t) 8 * FP_STG * sizeof(float4)};
      ctx->fit[4] = {k_fit_patch<16, 1, 4>, 0, 16 * 32, (size_t) 16 * FP_STG * sizeof(float4)};
    }
    for (int c = 0; c < NUM_CLASSES; ++c) ctx->fit_small[c] = ctx->fit[c];
    ctx->fit_small[2] = {k_fit_patch<4, 4, 2>, 0, 4 * 32, (size_t) 4 * FP_STG * sizeof(float4)};
    ctx->fit_small[3] = {k_fit_patch<8, 2, 3>, 0, 8 * 32, (size_t) 8 * FP_STG * sizeof(float4)};
    ctx->fit_small[4] = {k_fit_patch<16, 1, 4>, 0, 16 * 32, (size_t) 16 * FP_STG * sizeof(float4)};
    for (int c = 0; c < 2 * NUM_CLASSES; ++c) {
      FitLaunch& k = c < NUM_CLASSES ? ctx->fit[c] : ctx->fit_small[c - NUM_CLASSES];
      if (k.smem > 0) CU_TRY_CTX(raise_smem_limit(k.fn, k.smem));
      int per_sm = 1;
      CU_TRY_CTX(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k.fn, k.threads, k.smem));
      k.grid = std::max(1, per_sm) * prop.multiProcessorCount;
    }
    {
      typedef void (*OrdKernel)(const float4*, WorkQueues, int*, int*);
      const OrdKernel fn[ORD_NUM_HEADS] = {k_order_cta<512, 5>, k_order_cta<512, 4>, k_order_cta<256, 3>, k_order_cta<128, 2>, k_order_warp};
      const int th[ORD_NUM_HEADS] = {512, 512, 256, 128, ORD_WARP_THREADS};
      for (int q = 0; q < ORD_NUM_HEADS; ++q) {
        const size_t sm = q < 4 ? ord_cta_smem_bytes(th[q]) : 0;
        if (sm > 48 * 1024) CU_TRY_CTX(raise_smem_limit(fn[q], sm));
        int per_sm = 1;
        CU_TRY_CTX(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn[q], th[q], sm));
        ctx->order_k[q].grid = std::max(1, per_sm) * prop.multiProcessorCount;
        ctx->order_k[q].threads = th[q];
        ctx->order_k[q].smem = sm;
      }
    }
    const size_t gle_smem = gle_smem_bytes(max_sectors);
    if (gle_smem > 48 * 1024) CU_TRY_CTX(raise_smem_limit(k_gle, gle_smem));
  }
  {
    const size_t scat = (size_t) (CHUNK_THREADS / 32) * ctx->nbp * sizeof(unsigned int);
    if (scat > 48 * 1024) CU_TRY_CTX(raise_smem_limit(k_scatter<false, 4>, scat));
    const size_t sm_f = front_cluster_smem_bytes(ctx->nbp, FC_THREADS), sm_fd = front_cluster_smem_bytes(ctx->nbp, FC_THREADS_DENSE);
    if (sm_f > 220 * 1024) ctx->sw_front = 0;   // (thousands of bins: the per-warp count tables no longer fit next to the tiles)
    ctx->front_dense_ok = sm_fd <= 220 * 1024;
    if (ctx->sw_front) {
      CU_TRY_CTX(raise_smem_limit(k_front_cluster<true, CLS_L2_MAX, FC_THREADS>, sm_f));
      CU_TRY_CTX(raise_smem_limit(k_front_cluster<false, CLS_L2_MAX, FC_THREADS>, sm_f));
      if (ctx->front_dense_ok) {
        CU_TRY_CTX(raise_smem_limit(k_front_cluster<true, CLS_L2_MAX, FC_THREADS_DENSE>, sm_fd));
        CU_TRY_CTX(raise_smem_limit(k_front_cluster<false, CLS_L2_MAX, FC_THREADS_DENSE>, sm_fd));
      }
    }
  }
  *out = ctx;
  rc = pwpp_reset_all(ctx);
  if (rc) { pwpp_destroy(ctx); *out = nullptr; return rc; }
  CU_TRY_CTX(cudaStreamSynchronize(ctx->stream));   // the initial state is in place before any caller stream can read it
  if (max_points_per_frame > 0) {
    const size_t tot = (size_t) max_points_per_frame * num_streams;
    CU_TRY_CTX(ctx->d_bin_ids.reserve(tot));
    CU_TRY_CTX(ctx->d_sorted.reserve(tot));
    CU_TRY_CTX(ctx->d_part.reserve(tot));
    CU_TRY_CTX(ctx->d_out_idx.reserve(tot));
  }
#undef CU_TRY_CTX
  return PWPP_OK;
}

static int check_create_args(int num_streams, int64_t max_points_per_frame, pwpp_ctx** out) {
  if (!out) return fail(PWPP_ERR_INVALID_ARG, "out is NULL");
  *out = nullptr;
  if (num_streams < 1 || num_streams > 65535) return fail(PWPP_ERR_INVALID_ARG, "num_streams must be in [1,65535]");
  if (max_points_per_frame < 0) return fail(PWPP_ERR_INVALID_ARG, "max_points_per_frame < 0");
  return PWPP_OK;
}

int pwpp_create(const pwpp_params* params, int device, int num_streams, int64_t max_points_per_frame, pwpp_ctx** out) {
  if (!out) return fail(PWPP_ERR_INVALID_ARG, "out is NULL");
  *out = nullptr;
  int rc = validate_params(params);
  if (rc) return rc;
  rc = check_create_args(num_streams, max_points_per_frame, out);
  if (rc) return rc;
  return create_impl(params, 1, nullptr, device, num_streams, max_points_per_frame, out);
}

int pwpp_create_sets(const pwpp_params* sets, int num_sets, const int32_t* stream_set, int device, int num_streams, int64_t max_points_per_frame,
                     pwpp_ctx** out) {
  if (!out) return fail(PWPP_ERR_INVALID_ARG, "out is NULL");
  *out = nullptr;
  if (num_sets < 1 || num_sets > PWPP_MAX_PARAM_SETS)
    return fail(PWPP_ERR_INVALID_ARG, "num_sets must be in [1, " + std::to_string(PWPP_MAX_PARAM_SETS) + "], got " + std::to_string(num_sets));
  if (!sets) return fail(PWPP_ERR_INVALID_ARG, "sets is NULL");
  for (int k = 0; k < num_sets; ++k) {
    const int rc = validate_params(&sets[k]);
    if (rc) return fail(rc, "parameter set " + std::to_string(k) + ": " + g_last_error);
  }
  int rc = check_create_args(num_streams, max_points_per_frame, out);
  if (rc) return rc;
  if (!stream_set) return fail(PWPP_ERR_INVALID_ARG, "stream_set is NULL");
  for (int i = 0; i < num_streams; ++i)
    if (stream_set[i] < 0 || stream_set[i] >= num_sets)
      return fail(PWPP_ERR_INVALID_ARG, "stream " + std::to_string(i) + " names parameter set " + std::to_string(stream_set[i]) + ", outside [0, num_sets)");
  return create_impl(sets, num_sets, stream_set, device, num_streams, max_points_per_frame, out);
}

void pwpp_destroy(pwpp_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  for (int i = 0; i <= PWPP_NUM_STAGES; ++i) if (ctx->stage_ev[i]) cudaEventDestroy(ctx->stage_ev[i]);
  for (int i = 0; i < 2; ++i) if (ctx->gexec[i]) cudaGraphExecDestroy(ctx->gexec[i]);
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  for (int i = 0; i < 2; ++i) if (ctx->tab_ev[i]) cudaEventDestroy(ctx->tab_ev[i]);
  for (int q = 0; q < NUM_SIDE; ++q) { if (ctx->ev_fit[q]) cudaEventDestroy(ctx->ev_fit[q]); if (ctx->ev_join[q]) cudaEventDestroy(ctx->ev_join[q]); if (ctx->side[q]) cudaStreamDestroy(ctx->side[q]); }
  ctx->d_states.release(); ctx->d_states_init.release(); ctx->d_hist.release(); ctx->d_in.release(); ctx->d_cm.release(); ctx->d_pt_off.release(); ctx->d_chunk_off.release();
  ctx->d_stream.release(); ctx->d_pset.release();
  ctx->d_bin_ids.release(); ctx->d_chist.release(); ctx->d_cbase.release(); ctx->d_bin_off.release(); ctx->d_sorted.release();
  ctx->d_part.release(); ctx->d_labels.release(); ctx->d_fits.release(); ctx->d_segs.release(); ctx->d_wq_ctr.release();
  for (int c = 0; c < NUM_CLASSES; ++c) ctx->d_wq_items[c].release();
  ctx->d_out_idx.release(); ctx->d_counts.release();
  ctx->d_centers.release(); ctx->d_normals.release(); ctx->d_xyz.release();
  ctx->d_raw.release(); ctx->d_rec.release(); ctx->h_raw.release(); for (int i = 0; i < 2; ++i) ctx->h_rec_buf[i].release();
  ctx->d_rec_out.release(); ctx->d_rec_off.release(); ctx->h_rec_off.release(); ctx->h_rec_out.release();
  if (ctx->ev_rec_off) cudaEventDestroy(ctx->ev_rec_off);
  ctx->h_in.release(); for (int i = 0; i < 2; ++i) { ctx->h_pt_off_buf[i].release(); ctx->h_chunk_off_buf[i].release(); ctx->h_stream_buf[i].release(); ctx->h_pset_buf[i].release(); }
  ctx->h_out_idx.release(); ctx->h_counts.release();
  ctx->h_centers.release(); ctx->h_normals.release();
  if (ctx->ev0) cudaEventDestroy(ctx->ev0);
  if (ctx->ev1) cudaEventDestroy(ctx->ev1);
  if (ctx->ev_begin) cudaEventDestroy(ctx->ev_begin);
  if (ctx->ev_end) cudaEventDestroy(ctx->ev_end);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  if (ctx->stream_h2d) cudaStreamDestroy(ctx->stream_h2d);
  if (ctx->stream_d2h) cudaStreamDestroy(ctx->stream_d2h);
  delete ctx;
}

int pwpp_reset_stream(pwpp_ctx* ctx, int f) {
  if (!ctx || f < 0 || f >= ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "bad stream index");
  int rc = bind_device(ctx);
  if (rc) return rc;
  cudaStream_t s = ctx->last_stream ? ctx->last_stream : ctx->stream;
  CU_TRY(cudaMemcpyAsync(ctx->d_states.p + f, ctx->d_states_init.p + f, sizeof(StreamState), cudaMemcpyDeviceToDevice, s));
  return PWPP_OK;
}
int pwpp_reset_all(pwpp_ctx* ctx) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  int rc = bind_device(ctx);
  if (rc) return rc;
  cudaStream_t s = ctx->last_stream ? ctx->last_stream : ctx->stream;
  CU_TRY(cudaMemcpyAsync(ctx->d_states.p, ctx->d_states_init.p, (size_t) ctx->num_streams * sizeof(StreamState), cudaMemcpyDeviceToDevice, s));
  return PWPP_OK;
}

void* pwpp_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) { g_last_error = "cudaMallocHost failed"; return nullptr; }
  return p;
}
void pwpp_host_free(void* p) { if (p) cudaFreeHost(p); }

int pwpp_set_profiling(pwpp_ctx* ctx, int enabled) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  ctx->profiling = enabled != 0;
  ctx->stage_valid = false;
  return PWPP_OK;
}
int pwpp_stage_times_ms(pwpp_ctx* ctx, float* ms) {
  if (!ctx || !ms) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  if (!ctx->stage_valid) return fail(PWPP_ERR_INVALID_ARG, "no profiled estimate call yet (pwpp_set_profiling)");
  int rc = bind_device(ctx);
  if (rc) return rc;
  CU_TRY(cudaEventSynchronize(ctx->stage_ev[PWPP_NUM_STAGES]));
  for (int i = 0; i < PWPP_NUM_STAGES; ++i) CU_TRY(cudaEventElapsedTime(&ms[i], ctx->stage_ev[i], ctx->stage_ev[i + 1]));
  return PWPP_OK;
}
const char* pwpp_stage_name(int stage) {
  static const char* names[PWPP_NUM_STAGES] = {"k_bin_hist", "k_bin_scan", "k_scatter", "k_fit_S", "k_fit_L3", "k_fit_L2", "k_fit_L1", "k_fit_M", "k_fit_X", "k_gle", "k_emit"};
  return (stage >= 0 && stage < PWPP_NUM_STAGES) ? names[stage] : "";
}
int64_t pwpp_launch_count(const pwpp_ctx* ctx) { return ctx ? ctx->launches : 0; }

// The host path of pwpp_estimate_host and pwpp_estimate_host_streams (stream table checked by the caller).
static int estimate_host_impl(pwpp_ctx* ctx, int nframes, const int32_t* streams, const float* const* pts, const int64_t* n, int cols,
                              int64_t row_stride, int64_t col_stride) {
  if (!pts || !n) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  if (cols != 3 && cols != 4) return fail(PWPP_ERR_INVALID_ARG, "cols must be 3 or 4 (x,y,z[,intensity])");
  for (int f = 0; f < nframes; ++f)
    if (n[f] < 0 || (n[f] > 0 && !pts[f])) return fail(PWPP_ERR_INVALID_ARG, "bad frame pointer/size");
  int rc = bind_device(ctx);
  if (rc) return rc;
  const auto t0 = std::chrono::steady_clock::now();
  ctx->pt_off.assign(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) ctx->pt_off[f + 1] = ctx->pt_off[f] + n[f];
  const long long total = ctx->pt_off[nframes];
  CU_TRY(ctx->d_in.reserve((size_t) std::max<long long>(total, 1)));
  cudaStream_t s = ctx->stream, s_in = ctx->stream_h2d, s_out = ctx->stream_d2h;
  ctx->call_times_valid = false;
  // the staging buffers of the previous call must not be in flight any more (nor a device-input call on a caller's stream)
  if (ctx->last_stream && ctx->last_stream != s) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(s));
  CU_TRY(cudaStreamSynchronize(s_in));
  CU_TRY(cudaStreamSynchronize(s_out));
  rc = prepare_call(ctx, nframes, streams, s);
  if (rc) return rc;
  CU_TRY(ctx->h_out_idx.reserve((size_t) std::max<long long>(total, 1)));
  CU_TRY(ctx->h_counts.reserve((size_t) 3 * nframes));
  const bool packed = (cols == 4 && col_stride == 1 && row_stride == 4);
  bool staged_any = false;
  // Chunks of frames flow through three streams: H2D of chunk k+1 | kernels of chunk k | D2H of chunk k-1.
  // ~64 MB of points per chunk keeps every stage busy without delaying the first kernels.
  int chunk_frames = nframes;
  if (nframes > 1 && total > 0) {
    const long long per_frame = std::max<long long>(1, total / nframes);
    chunk_frames = (int) std::min<long long>(nframes, std::max<long long>(1, (4LL << 20) / per_frame));
  }
  const int nchunks = (nframes + chunk_frames - 1) / chunk_frames;
  // a call that is a single chunk has nothing to pipeline: copies and kernels share one stream (no cross-stream event hops
  // on the critical path of a one-frame call) and four events bracket its three phases (pwpp_call_times_us)
  const bool one_stream = (nchunks == 1);
  if (one_stream) { s_in = s; s_out = s; CU_TRY(cudaEventRecord(ctx->ev_begin, s)); }
  // the launch ranges are the pipeline chunks cut at the run boundaries; per-stage timing needs one range per call
  const bool prof = ctx->profiling && nchunks == 1 && ctx->runs.size() == 2;
  size_t run_cursor = 0;
  for (int k = 0; k < nchunks; ++k) {
    const int f0 = k * chunk_frames, f1 = std::min(nframes, f0 + chunk_frames);
    for (int f = f0; f < f1; ++f) {
      const int64_t cnt = n[f];
      if (cnt == 0) continue;
      bool pinned = false;
      if (packed) {
        cudaPointerAttributes attr;
        if (cudaPointerGetAttributes(&attr, pts[f]) == cudaSuccess) pinned = (attr.type == cudaMemoryTypeHost);
        else cudaGetLastError();
      }
      if (pinned) {  // page-locked caller buffer: DMA straight from it (the private copy of H:152 is the device buffer)
        // frames that follow each other in the caller's buffer travel as one copy
        int f_last = f;
        int64_t run = cnt;
        while (f_last + 1 < f1 && n[f_last + 1] > 0 && pts[f_last + 1] == pts[f_last] + n[f_last] * 4) { ++f_last; run += n[f_last]; }
        CU_TRY(cudaMemcpyAsync(ctx->d_in.p + ctx->pt_off[f], pts[f], (size_t) run * sizeof(float4), cudaMemcpyHostToDevice, s_in));
        f = f_last;
        continue;
      }
      if (row_stride == 1 && col_stride == cnt && cnt > 1) {
        // column-major frame (what the Eigen overload hands over): its cols x n floats are one contiguous block; upload it as
        // it is and repack on the device instead of gathering 4 strided columns per point on the host
        if ((size_t) total * 4 > ctx->d_cm.cap) { CU_TRY(cudaStreamSynchronize(s_in)); CU_TRY(ctx->d_cm.reserve((size_t) total * 4)); }
        float* cm = ctx->d_cm.p + (size_t) ctx->pt_off[f] * 4;
        CU_TRY(cudaMemcpyAsync(cm, pts[f], (size_t) cnt * cols * sizeof(float), cudaMemcpyHostToDevice, s_in));
        k_repack_colmajor<<<(unsigned) ((cnt + 255) / 256), 256, 0, s_in>>>(cm, cnt, cols, ctx->d_in.p + ctx->pt_off[f]);
        ++ctx->launches;
        continue;
      }
      if (!staged_any) { CU_TRY(ctx->h_in.reserve((size_t) std::max<long long>(total, 1))); staged_any = true; }
      float4* dst = ctx->h_in.p + ctx->pt_off[f];
      const float* src = pts[f];
      if (packed) {
        std::memcpy(dst, src, (size_t) cnt * sizeof(float4));
      } else {
        for (int64_t i = 0; i < cnt; ++i) {
          const float* r = src + i * row_stride;
          dst[i] = make_float4(r[0], r[col_stride], r[2 * col_stride], cols == 4 ? r[3 * col_stride] : 0.f);
        }
      }
      CU_TRY(cudaMemcpyAsync(ctx->d_in.p + ctx->pt_off[f], dst, (size_t) cnt * sizeof(float4), cudaMemcpyHostToDevice, s_in));
    }
    CU_TRY(cudaEventRecord(ctx->ev0, s_in));
    if (!one_stream) CU_TRY(cudaStreamWaitEvent(s, ctx->ev0, 0));
    rc = launch_runs(ctx, f0, f1, &run_cursor, ctx->d_in.p, cols == 4 ? 1 : 0, s, prof);
    if (rc) return rc;
    CU_TRY(cudaEventRecord(ctx->ev1, s));
    if (!one_stream) CU_TRY(cudaStreamWaitEvent(s_out, ctx->ev1, 0));
    const long long o0 = ctx->pt_off[f0], o1 = ctx->pt_off[f1];
    if (f0 == 0 && f1 == nframes) {   // the three count rows are one contiguous block when the chunk covers the whole call
      CU_TRY(cudaMemcpyAsync(ctx->h_counts.p, ctx->d_counts.p, (size_t) 3 * nframes * sizeof(int), cudaMemcpyDeviceToHost, s_out));
    } else {
      for (int q = 0; q < 3; ++q)
        CU_TRY(cudaMemcpyAsync(ctx->h_counts.p + (size_t) q * nframes + f0, ctx->d_counts.p + (size_t) q * nframes + f0,
                               (size_t) (f1 - f0) * sizeof(int), cudaMemcpyDeviceToHost, s_out));
    }
    if (o1 > o0) CU_TRY(cudaMemcpyAsync(ctx->h_out_idx.p + o0, ctx->d_out_idx.p + o0, (size_t) (o1 - o0) * sizeof(int), cudaMemcpyDeviceToHost, s_out));
  }
  if (one_stream) CU_TRY(cudaEventRecord(ctx->ev_end, s));
  CU_TRY(cudaStreamSynchronize(s_out));
  CU_TRY(cudaStreamSynchronize(s));
  ctx->call_times_valid = one_stream;
  ctx->counts_fetched = true;
  ctx->idx_fetched = true;
  ctx->last_time_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
  return PWPP_OK;
}

int pwpp_estimate_host(pwpp_ctx* ctx, int nframes, const float* const* pts, const int64_t* n, int cols, int64_t row_stride, int64_t col_stride) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  if (nframes < 1 || nframes > ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "nframes must be in [1, num_streams]");
  return estimate_host_impl(ctx, nframes, ctx->identity.data(), pts, n, cols, row_stride, col_stride);
}

int pwpp_estimate_host_streams(pwpp_ctx* ctx, int nframes, const int32_t* streams, const float* const* pts, const int64_t* n, int cols,
                               int64_t row_stride, int64_t col_stride) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  const int rc = check_streams(ctx, nframes, streams);
  if (rc) return rc;
  return estimate_host_impl(ctx, nframes, streams, pts, n, cols, row_stride, col_stride);
}

// The device path of pwpp_estimate_device and pwpp_estimate_device_streams (stream table checked by the caller).
static int estimate_device_impl(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* d_pts, const int64_t* h_offsets, int has_intensity,
                                void* cuda_stream) {
  if (!h_offsets) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  for (int f = 1; f <= nframes; ++f)
    if (h_offsets[f] < h_offsets[f - 1]) return fail(PWPP_ERR_INVALID_ARG, "offsets must be non-decreasing");
  if (h_offsets[nframes] > h_offsets[0] && !d_pts) return fail(PWPP_ERR_INVALID_ARG, "d_pts is NULL");
  int rc = bind_device(ctx);
  if (rc) return rc;
  const auto t0 = std::chrono::steady_clock::now();
  ctx->pt_off.assign(nframes + 1, 0);
  for (int f = 0; f <= nframes; ++f) ctx->pt_off[f] = h_offsets[f] - h_offsets[0];
  cudaStream_t s = cuda_stream ? (cudaStream_t) cuda_stream : ctx->stream;
  // work buffers are reused stream-ordered: a call on a different stream than the previous one waits for it
  if (ctx->last_stream && ctx->last_stream != s) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  if (!ctx->last_stream && s != ctx->stream) CU_TRY(cudaStreamSynchronize(ctx->stream));   // resets issued before the first call ran on the ctx's own stream
  rc = run_path(ctx, nframes, streams, (const float4*) d_pts + h_offsets[0], has_intensity, s);
  if (rc) return rc;
  ctx->last_time_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
  return PWPP_OK;
}

int pwpp_estimate_device(pwpp_ctx* ctx, int nframes, const void* d_pts, const int64_t* h_offsets, int has_intensity, void* cuda_stream) {
  if (!ctx || !h_offsets) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  if (nframes < 1 || nframes > ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "nframes must be in [1, num_streams]");
  return estimate_device_impl(ctx, nframes, ctx->identity.data(), d_pts, h_offsets, has_intensity, cuda_stream);
}

int pwpp_estimate_device_streams(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* d_pts, const int64_t* h_offsets, int has_intensity,
                                 void* cuda_stream) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  const int rc = check_streams(ctx, nframes, streams);
  if (rc) return rc;
  return estimate_device_impl(ctx, nframes, streams, d_pts, h_offsets, has_intensity, cuda_stream);
}

int pwpp_estimate_device_xyz(pwpp_ctx* ctx, int nframes, const void* d_xyz, const int64_t* h_offsets, void* cuda_stream) {
  if (!ctx || !h_offsets) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  if (nframes < 1 || nframes > ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "nframes must be in [1, num_streams]");
  int rc = bind_device(ctx);
  if (rc) return rc;
  const long long total = h_offsets[nframes] - h_offsets[0];
  if (total < 0 || (total > 0 && !d_xyz)) return fail(PWPP_ERR_INVALID_ARG, "bad offsets / d_xyz is NULL");
  cudaStream_t s = cuda_stream ? (cudaStream_t) cuda_stream : ctx->stream;
  if (ctx->last_stream && ctx->last_stream != s) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  if (!ctx->last_stream && s != ctx->stream) CU_TRY(cudaStreamSynchronize(ctx->stream));
  CU_TRY(ctx->d_in.reserve((size_t) std::max<long long>(total, 1)));
  if (total > 0) {
    k_pad_xyz<<<(unsigned) ((total + 255) / 256), 256, 0, s>>>((const float*) d_xyz + 3 * h_offsets[0], total, ctx->d_in.p);
    ++ctx->launches;
  }
  std::vector<int64_t> offs(h_offsets, h_offsets + nframes + 1);
  for (auto& o : offs) o -= h_offsets[0];
  return pwpp_estimate_device(ctx, nframes, ctx->d_in.p, offs.data(), 0, s);
}

// The checks of both records entry points (include/pwpp.h), before anything is allocated or launched.
static int check_records_call(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* frames, const int64_t* n,
                              const pwpp_point_layout* layouts) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  int rc = check_streams(ctx, nframes, streams);
  if (rc) return rc;
  std::string msg;
  rc = check_record_layouts(nframes, frames, n, layouts, &msg);
  if (rc) return fail(rc, msg);
  for (int f = 0; f < nframes; ++f)
    if (n[f] > 0x7fffffffLL - CHUNK_PTS) return fail(PWPP_ERR_INVALID_ARG, "frame " + std::to_string(f) + ": frame size out of range");
  return PWPP_OK;
}

// Unpacks frames [f0, f1) of the prepared records call into ctx->d_in on stream s: one launch (none when the frames are empty).
static int unpack_records(pwpp_ctx* ctx, int f0, int f1, const std::vector<RecordFrame>& recs, cudaStream_t s) {
  if (ctx->pt_off[f1] == ctx->pt_off[f0]) return PWPP_OK;
  const long long gx = rec_grid_x(ctx->pt_off.data() + f0, recs.data() + f0, f1 - f0);
  k_unpack_records<<<dim3((unsigned) gx, (unsigned) (f1 - f0)), REC_THREADS, 0, s>>>(ctx->d_rec.p + f0, ctx->d_pt_off.p + f0, ctx->d_in.p);
  ++ctx->launches;
  CU_TRY(cudaGetLastError());
  return PWPP_OK;
}

int pwpp_estimate_host_records(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* frames, const int64_t* n,
                               const pwpp_point_layout* layouts) {
  int rc = check_records_call(ctx, nframes, streams, frames, n, layouts);
  if (rc) return rc;
  rc = bind_device(ctx);
  if (rc) return rc;
  const auto t0 = std::chrono::steady_clock::now();
  ctx->pt_off.assign(nframes + 1, 0);
  std::vector<long long> raw_off(nframes + 1, 0);   // every frame's records in the upload buffer, 16-byte aligned
  for (int f = 0; f < nframes; ++f) {
    ctx->pt_off[f + 1] = ctx->pt_off[f] + n[f];
    raw_off[f + 1] = raw_off[f] + ((n[f] * layouts[f].point_step + 15) & ~15LL);
  }
  const long long total = ctx->pt_off[nframes];
  cudaStream_t s = ctx->stream, s_in = ctx->stream_h2d, s_out = ctx->stream_d2h;
  ctx->call_times_valid = false;
  // the buffers of the previous call must not be in flight any more (nor a device-input call on a caller's stream)
  if (ctx->last_stream && ctx->last_stream != s) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(s));
  CU_TRY(cudaStreamSynchronize(s_in));
  CU_TRY(cudaStreamSynchronize(s_out));
  CU_TRY(ctx->d_in.reserve((size_t) std::max<long long>(total, 1)));
  CU_TRY(ctx->d_raw.reserve((size_t) std::max<long long>(raw_off[nframes], 16)));
  std::vector<RecordFrame> recs(nframes);
  int has_intensity = 0;
  for (int f = 0; f < nframes; ++f) {
    recs[f] = record_frame(layouts[f], ctx->d_raw.p + raw_off[f]);
    if (layouts[f].offset[3] >= 0) has_intensity = 1;
  }
  rc = prepare_call(ctx, nframes, streams, s, recs.data());
  if (rc) return rc;
  CU_TRY(ctx->h_out_idx.reserve((size_t) std::max<long long>(total, 1)));
  CU_TRY(ctx->h_counts.reserve((size_t) 3 * nframes));
  bool staged_any = false;
  // the chunk pipeline of pwpp_estimate_host: H2D + unpack of chunk k+1 | kernels of chunk k | D2H of chunk k-1
  int chunk_frames = nframes;
  if (nframes > 1 && total > 0) {
    const long long per_frame = std::max<long long>(1, total / nframes);
    chunk_frames = (int) std::min<long long>(nframes, std::max<long long>(1, (4LL << 20) / per_frame));
  }
  const int nchunks = (nframes + chunk_frames - 1) / chunk_frames;
  const bool one_stream = (nchunks == 1);
  if (one_stream) { s_in = s; s_out = s; CU_TRY(cudaEventRecord(ctx->ev_begin, s)); }
  else CU_TRY(cudaStreamWaitEvent(s_in, ctx->tab_ev[ctx->tab_cur], 0));   // the unpack reads the record table uploaded on s
  const bool prof = ctx->profiling && nchunks == 1 && ctx->runs.size() == 2;
  size_t run_cursor = 0;
  for (int k = 0; k < nchunks; ++k) {
    const int f0 = k * chunk_frames, f1 = std::min(nframes, f0 + chunk_frames);
    for (int f = f0; f < f1; ++f) {
      if (n[f] == 0) continue;
      const size_t bytes = (size_t) n[f] * layouts[f].point_step;
      bool pinned = false;
      cudaPointerAttributes attr;
      if (cudaPointerGetAttributes(&attr, frames[f]) == cudaSuccess) pinned = (attr.type == cudaMemoryTypeHost);
      else cudaGetLastError();
      const void* src = frames[f];
      if (!pinned) {   // pageable: one memcpy into page-locked staging, then DMA
        if (!staged_any) { CU_TRY(ctx->h_raw.reserve((size_t) std::max<long long>(raw_off[nframes], 16))); staged_any = true; }
        std::memcpy(ctx->h_raw.p + raw_off[f], frames[f], bytes);
        src = ctx->h_raw.p + raw_off[f];
      }
      CU_TRY(cudaMemcpyAsync(ctx->d_raw.p + raw_off[f], src, bytes, cudaMemcpyHostToDevice, s_in));
    }
    rc = unpack_records(ctx, f0, f1, recs, s_in);
    if (rc) return rc;
    CU_TRY(cudaEventRecord(ctx->ev0, s_in));
    if (!one_stream) CU_TRY(cudaStreamWaitEvent(s, ctx->ev0, 0));
    rc = launch_runs(ctx, f0, f1, &run_cursor, ctx->d_in.p, has_intensity, s, prof);
    if (rc) return rc;
    CU_TRY(cudaEventRecord(ctx->ev1, s));
    if (!one_stream) CU_TRY(cudaStreamWaitEvent(s_out, ctx->ev1, 0));
    const long long o0 = ctx->pt_off[f0], o1 = ctx->pt_off[f1];
    for (int q = 0; q < 3; ++q)
      CU_TRY(cudaMemcpyAsync(ctx->h_counts.p + (size_t) q * nframes + f0, ctx->d_counts.p + (size_t) q * nframes + f0, (size_t) (f1 - f0) * sizeof(int),
                             cudaMemcpyDeviceToHost, s_out));
    if (o1 > o0) CU_TRY(cudaMemcpyAsync(ctx->h_out_idx.p + o0, ctx->d_out_idx.p + o0, (size_t) (o1 - o0) * sizeof(int), cudaMemcpyDeviceToHost, s_out));
  }
  if (one_stream) CU_TRY(cudaEventRecord(ctx->ev_end, s));
  CU_TRY(cudaStreamSynchronize(s_out));
  CU_TRY(cudaStreamSynchronize(s));
  ctx->call_times_valid = one_stream;
  ctx->counts_fetched = true;
  ctx->idx_fetched = true;
  ctx->last_time_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
  return PWPP_OK;
}

int pwpp_estimate_device_records(pwpp_ctx* ctx, int nframes, const int32_t* streams, const void* const* d_frames, const int64_t* n,
                                 const pwpp_point_layout* layouts, void* cuda_stream) {
  int rc = check_records_call(ctx, nframes, streams, d_frames, n, layouts);
  if (rc) return rc;
  rc = bind_device(ctx);
  if (rc) return rc;
  const auto t0 = std::chrono::steady_clock::now();
  ctx->pt_off.assign(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) ctx->pt_off[f + 1] = ctx->pt_off[f] + n[f];
  const long long total = ctx->pt_off[nframes];
  cudaStream_t s = cuda_stream ? (cudaStream_t) cuda_stream : ctx->stream;
  // stream ordering of pwpp_estimate_device_xyz: the input buffer and work buffers are reused in stream order
  if (ctx->last_stream && ctx->last_stream != s) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  if (!ctx->last_stream && s != ctx->stream) CU_TRY(cudaStreamSynchronize(ctx->stream));
  CU_TRY(ctx->d_in.reserve((size_t) std::max<long long>(total, 1)));
  std::vector<RecordFrame> recs(nframes);
  int has_intensity = 0;
  for (int f = 0; f < nframes; ++f) {
    recs[f] = record_frame(layouts[f], d_frames[f]);
    if (layouts[f].offset[3] >= 0) has_intensity = 1;
  }
  rc = prepare_call(ctx, nframes, streams, s, recs.data());
  if (rc) return rc;
  rc = unpack_records(ctx, 0, nframes, recs, s);
  if (rc) return rc;
  rc = launch_call(ctx, nframes, ctx->d_in.p, has_intensity, s);
  if (rc) return rc;
  ctx->last_time_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
  return PWPP_OK;
}

// Record results of the last call: the first request gathers every frame's records into d_rec_out on the call's stream (one
// launch, none when the call had no points), and no later request of the same call gathers again. The host blocks only where
// a buffer is first reserved or grows, and on the previous request's offset-table upload (include/pwpp.h).
static int gather_records(pwpp_ctx* ctx) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (ctx->last_nframes <= 0) return fail(PWPP_ERR_INVALID_ARG, "no estimate call yet");
  if (ctx->last_recs.empty()) return fail(PWPP_ERR_INVALID_ARG, "the last estimate call did not take records (pwpp_estimate_host_records / pwpp_estimate_device_records)");
  if (ctx->rec_gathered) return PWPP_OK;
  int rc = bind_device(ctx);
  if (rc) return rc;
  const int nf = ctx->last_nframes;
  cudaStream_t s = ctx->last_stream;
  ctx->rec_off.assign(nf + 1, 0);
  rec_out_offsets(ctx->pt_off.data(), ctx->last_recs.data(), nf, ctx->rec_off.data());
  CU_TRY(ctx->d_rec_out.reserve((size_t) std::max<long long>(ctx->rec_off[nf], 16)));
  CU_TRY(ctx->d_rec_off.reserve(nf + 1));
  if (ctx->ev_rec_off) CU_TRY(cudaEventSynchronize(ctx->ev_rec_off));   // the previous gather's upload has read the staging
  else CU_TRY(cudaEventCreateWithFlags(&ctx->ev_rec_off, cudaEventDisableTiming));
  CU_TRY(ctx->h_rec_off.reserve(nf + 1));
  std::memcpy(ctx->h_rec_off.p, ctx->rec_off.data(), (size_t) (nf + 1) * sizeof(long long));
  CU_TRY(cudaMemcpyAsync(ctx->d_rec_off.p, ctx->h_rec_off.p, (size_t) (nf + 1) * sizeof(long long), cudaMemcpyHostToDevice, s));
  CU_TRY(cudaEventRecord(ctx->ev_rec_off, s));
  if (ctx->last_total > 0) {
    const long long gx = rec_grid_x(ctx->pt_off.data(), ctx->last_recs.data(), nf);
    k_gather_records<<<dim3((unsigned) gx, (unsigned) nf), REC_THREADS, 0, s>>>(ctx->d_rec.p, ctx->d_pt_off.p, ctx->d_rec_off.p, ctx->d_counts.p + 2 * nf,
                                                                               ctx->d_out_idx.p, ctx->d_rec_out.p);
    ++ctx->launches;
    CU_TRY(cudaGetLastError());
  }
  ctx->rec_gathered = true;
  return PWPP_OK;
}

// The gathered records in the page-locked host view (one D2H per call), and the counts.
static int fetch_records(pwpp_ctx* ctx) {
  int rc = gather_records(ctx);
  if (rc) return rc;
  rc = fetch_counts(ctx);
  if (rc) return rc;
  if (ctx->rec_fetched) return PWPP_OK;
  const long long bytes = ctx->rec_off[ctx->last_nframes];
  CU_TRY(ctx->h_rec_out.reserve((size_t) std::max<long long>(bytes, 16)));
  if (bytes > 0) CU_TRY(cudaMemcpyAsync(ctx->h_rec_out.p, ctx->d_rec_out.p, (size_t) bytes, cudaMemcpyDeviceToHost, ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  ctx->rec_fetched = true;
  return PWPP_OK;
}

int pwpp_device_record_results(pwpp_ctx* ctx, const void** d_records, const int64_t** h_offsets) {
  const int rc = gather_records(ctx);
  if (rc) return rc;
  if (d_records) *d_records = ctx->d_rec_out.p;
  if (h_offsets) *h_offsets = reinterpret_cast<const int64_t*>(ctx->rec_off.data());
  return PWPP_OK;
}
int pwpp_host_record_results(pwpp_ctx* ctx, const void** h_records, const int64_t** h_offsets) {
  const int rc = fetch_records(ctx);
  if (rc) return rc;
  if (h_records) *h_records = ctx->h_rec_out.p;
  if (h_offsets) *h_offsets = reinterpret_cast<const int64_t*>(ctx->rec_off.data());
  return PWPP_OK;
}
static int copy_records(pwpp_ctx* ctx, int f, void* dst, bool ground) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = fetch_records(ctx);
  if (rc) return rc;
  const long long step = ctx->last_recs[f].step;
  const int ng = ctx->h_counts.p[f];
  const int nn = frame_n(ctx, f) - ng - count_of(ctx, 2, f);
  const long long cnt = ground ? ng : nn;
  if (cnt > 0) std::memcpy(dst, ctx->h_rec_out.p + ctx->rec_off[f] + (ground ? 0 : (long long) ng * step), (size_t) (cnt * step));
  return PWPP_OK;
}
int pwpp_copy_ground_records(pwpp_ctx* ctx, int f, void* dst) { return copy_records(ctx, f, dst, true); }
int pwpp_copy_nonground_records(pwpp_ctx* ctx, int f, void* dst) { return copy_records(ctx, f, dst, false); }

int pwpp_device_synchronize(pwpp_ctx* ctx) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  int rc = bind_device(ctx);
  if (rc) return rc;
  CU_TRY(cudaDeviceSynchronize());
  return PWPP_OK;
}

int pwpp_synchronize(pwpp_ctx* ctx) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  int rc = bind_device(ctx);
  if (rc) return rc;
  CU_TRY(cudaStreamSynchronize(ctx->last_stream ? ctx->last_stream : ctx->stream));
  return PWPP_OK;
}

int64_t pwpp_num_ground(pwpp_ctx* ctx, int f) {
  if (check_frame(ctx, f) || fetch_counts(ctx)) return -1;
  return ctx->h_counts.p[f];
}
int64_t pwpp_num_nonground(pwpp_ctx* ctx, int f) {
  if (check_frame(ctx, f) || fetch_counts(ctx)) return -1;
  return (int64_t) frame_n(ctx, f) - ctx->h_counts.p[f] - count_of(ctx, 2, f);
}
int pwpp_copy_ground_indices(pwpp_ctx* ctx, int f, int32_t* dst) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = fetch_indices(ctx);
  if (rc) return rc;
  const int ng = ctx->h_counts.p[f];
  if (ng > 0) std::memcpy(dst, ctx->h_out_idx.p + ctx->pt_off[f], (size_t) ng * sizeof(int32_t));
  return PWPP_OK;
}
int pwpp_copy_nonground_indices(pwpp_ctx* ctx, int f, int32_t* dst) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = fetch_indices(ctx);
  if (rc) return rc;
  const int ng = ctx->h_counts.p[f];
  const int nn = frame_n(ctx, f) - ng - count_of(ctx, 2, f);
  if (nn > 0) std::memcpy(dst, ctx->h_out_idx.p + ctx->pt_off[f] + ng, (size_t) nn * sizeof(int32_t));
  return PWPP_OK;
}

static int copy_xyz(pwpp_ctx* ctx, int f, float* dst, bool ground) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = fetch_counts(ctx);
  if (rc) return rc;
  const int ng = ctx->h_counts.p[f];
  const int nn = frame_n(ctx, f) - ng - count_of(ctx, 2, f);
  const int cnt = ground ? ng : nn;
  if (cnt <= 0) return PWPP_OK;
  CU_TRY(ctx->d_xyz.reserve((size_t) cnt * 3));
  const int* idx = ctx->d_out_idx.p + ctx->pt_off[f] + (ground ? 0 : ng);
  k_gather_xyz<<<(cnt + 255) / 256, 256, 0, ctx->last_stream>>>(ctx->last_pts + ctx->pt_off[f], idx, cnt, ctx->d_xyz.p);
  CU_TRY(cudaGetLastError());
  CU_TRY(cudaMemcpyAsync(dst, ctx->d_xyz.p, (size_t) cnt * 3 * sizeof(float), cudaMemcpyDeviceToHost, ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  return PWPP_OK;
}
int pwpp_copy_ground_xyz(pwpp_ctx* ctx, int f, float* dst) { return copy_xyz(ctx, f, dst, true); }
int pwpp_copy_nonground_xyz(pwpp_ctx* ctx, int f, float* dst) { return copy_xyz(ctx, f, dst, false); }

int pwpp_num_patches(pwpp_ctx* ctx, int f) {
  if (check_frame(ctx, f) || fetch_counts(ctx)) return -1;
  return count_of(ctx, 1, f);
}
int pwpp_copy_centers(pwpp_ctx* ctx, int f, float* dst) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = fetch_patches(ctx);
  if (rc) return rc;
  const int k = count_of(ctx, 1, f);
  if (k > 0) std::memcpy(dst, ctx->h_centers.p + (size_t) f * ctx->gs.nbs * 3, (size_t) k * 3 * sizeof(float));
  return PWPP_OK;
}
int pwpp_copy_normals(pwpp_ctx* ctx, int f, float* dst) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = fetch_patches(ctx);
  if (rc) return rc;
  const int k = count_of(ctx, 1, f);
  if (k > 0) std::memcpy(dst, ctx->h_normals.p + (size_t) f * ctx->gs.nbs * 3, (size_t) k * 3 * sizeof(float));
  return PWPP_OK;
}

int pwpp_get_state(pwpp_ctx* ctx, int f, pwpp_state* out) {
  if (!ctx || !out || f < 0 || f >= ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "bad argument");
  int rc = bind_device(ctx);
  if (rc) return rc;
  if (ctx->last_stream) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  StreamState s;
  CU_TRY(cudaMemcpy(&s, ctx->d_states.p + f, sizeof(s), cudaMemcpyDeviceToHost));
  out->sensor_height = s.sensor_height;
  for (int i = 0; i < 4; ++i) {
    out->elevation_thr[i] = s.elevation_thr[i]; out->flatness_thr[i] = s.flatness_thr[i];
    out->n_elevation[i] = s.n_elev[i]; out->n_flatness[i] = s.n_flat[i];
  }
  return PWPP_OK;
}
double pwpp_height(pwpp_ctx* ctx, int f) {
  pwpp_state s;
  if (pwpp_get_state(ctx, f, &s)) return NAN;
  return s.sensor_height;
}
double pwpp_time_us(pwpp_ctx* ctx) { return ctx ? ctx->last_time_us : NAN; }

int pwpp_call_times_us(pwpp_ctx* ctx, float out[4]) {
  if (!ctx || !out) return fail(PWPP_ERR_INVALID_ARG, "NULL argument");
  if (!ctx->call_times_valid) return fail(PWPP_ERR_INVALID_ARG, "no single-chunk pwpp_estimate_host call to report on");
  int rc = bind_device(ctx);
  if (rc) return rc;
  float ms[4];
  CU_TRY(cudaEventElapsedTime(&ms[0], ctx->ev_begin, ctx->ev0));
  CU_TRY(cudaEventElapsedTime(&ms[1], ctx->ev0, ctx->ev1));
  CU_TRY(cudaEventElapsedTime(&ms[2], ctx->ev1, ctx->ev_end));
  CU_TRY(cudaEventElapsedTime(&ms[3], ctx->ev_begin, ctx->ev_end));
  for (int i = 0; i < 4; ++i) out[i] = ms[i] * 1000.f;
  return PWPP_OK;
}

int pwpp_copy_history(pwpp_ctx* ctx, int f, int ring, int which, double* dst) {
  if (!ctx || !dst || f < 0 || f >= ctx->num_streams || ring < 0 || ring > 3 || which < 0 || which > 1) return fail(PWPP_ERR_INVALID_ARG, "bad argument");
  pwpp_state s;
  int rc = pwpp_get_state(ctx, f, &s);
  if (rc) return rc;
  const int n = which ? s.n_flatness[ring] : s.n_elevation[ring];
  if (n > 0) CU_TRY(cudaMemcpy(dst, ctx->d_hist.p + (((size_t) f * 2 + which) * 4 + ring) * ctx->hist_stride, (size_t) n * sizeof(double), cudaMemcpyDeviceToHost));
  return PWPP_OK;
}

namespace {
struct StateBlobHeader { uint32_t magic, version; int32_t hcap, state_bytes; };
constexpr uint32_t STATE_BLOB_MAGIC = 0x50575354u;  // "PWST"
}  // namespace
// a stream's blob: header, state, then its eight history rows of its own set's capacity (the layout of a one-set context)
static size_t blob_size_of_cap(int hcap) { return sizeof(StateBlobHeader) + sizeof(StreamState) + (size_t) 2 * 4 * hcap * sizeof(double); }
size_t pwpp_stream_state_blob_size(const pwpp_ctx* ctx, int s) {
  if (!ctx || s < 0 || s >= ctx->num_streams) return 0;
  return blob_size_of_cap(ctx->set_hcap[ctx->stream_set[s]]);
}
size_t pwpp_state_blob_size(const pwpp_ctx* ctx) { return ctx ? blob_size_of_cap(ctx->hist_stride) : 0; }
int pwpp_export_state(pwpp_ctx* ctx, int f, void* blob) {
  if (!ctx || !blob || f < 0 || f >= ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "bad argument");
  int rc = bind_device(ctx);
  if (rc) return rc;
  if (ctx->last_stream) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->stream));
  char* b = static_cast<char*>(blob);
  const int hcap = ctx->set_hcap[ctx->stream_set[f]];
  const StateBlobHeader h{STATE_BLOB_MAGIC, (uint32_t) PWPP_ABI_VERSION, hcap, (int32_t) sizeof(StreamState)};
  std::memcpy(b, &h, sizeof h);
  CU_TRY(cudaMemcpy(b + sizeof h, ctx->d_states.p + f, sizeof(StreamState), cudaMemcpyDeviceToHost));
  CU_TRY(cudaMemcpy2D(b + sizeof h + sizeof(StreamState), (size_t) hcap * sizeof(double), ctx->d_hist.p + (size_t) f * 2 * 4 * ctx->hist_stride,
                      (size_t) ctx->hist_stride * sizeof(double), (size_t) hcap * sizeof(double), 2 * 4, cudaMemcpyDeviceToHost));
  return PWPP_OK;
}
int pwpp_import_state(pwpp_ctx* ctx, int f, const void* blob, size_t bytes) {
  if (!ctx || !blob || f < 0 || f >= ctx->num_streams) return fail(PWPP_ERR_INVALID_ARG, "bad argument");
  if (bytes != pwpp_stream_state_blob_size(ctx, f)) return fail(PWPP_ERR_INVALID_ARG, "state blob has the wrong size for this context (different storage parameters?)");
  const int hcap = ctx->set_hcap[ctx->stream_set[f]];
  const char* b = static_cast<const char*>(blob);
  StateBlobHeader h;
  std::memcpy(&h, b, sizeof h);
  if (h.magic != STATE_BLOB_MAGIC || h.version != (uint32_t) PWPP_ABI_VERSION || h.hcap != hcap || h.state_bytes != (int32_t) sizeof(StreamState))
    return fail(PWPP_ERR_INVALID_ARG, "not a state blob of this library version / parameter set");
  int rc = bind_device(ctx);
  if (rc) return rc;
  // after everything already enqueued (a synchronous copy from pageable memory: the blob may be freed on return)
  if (ctx->last_stream) CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  CU_TRY(cudaStreamSynchronize(ctx->stream));
  CU_TRY(cudaMemcpy(ctx->d_states.p + f, b + sizeof h, sizeof(StreamState), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy2D(ctx->d_hist.p + (size_t) f * 2 * 4 * ctx->hist_stride, (size_t) ctx->hist_stride * sizeof(double), b + sizeof h + sizeof(StreamState),
                      (size_t) hcap * sizeof(double), (size_t) hcap * sizeof(double), 2 * 4, cudaMemcpyHostToDevice));
  return PWPP_OK;
}

int pwpp_device_results(pwpp_ctx* ctx, const int32_t** d_indices, const int32_t** d_num_ground) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (d_indices) *d_indices = ctx->d_out_idx.p;
  if (d_num_ground) *d_num_ground = ctx->d_counts.p;
  return PWPP_OK;
}

int pwpp_set_output_order(pwpp_ctx* ctx, int order) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (order != PWPP_ORDER_BIN && order != PWPP_ORDER_REFERENCE) return fail(PWPP_ERR_INVALID_ARG, "order must be PWPP_ORDER_BIN or PWPP_ORDER_REFERENCE");
  if (order != ctx->order_mode) ++g_alloc_gen;   // captured graphs were recorded with the other launch sequence
  ctx->order_mode = order;
  return PWPP_OK;
}

int pwpp_host_results(pwpp_ctx* ctx, const int32_t** h_indices, const int32_t** h_num_ground, const int64_t** h_offsets) {
  if (!ctx) return fail(PWPP_ERR_INVALID_ARG, "ctx is NULL");
  if (ctx->last_nframes <= 0) return fail(PWPP_ERR_INVALID_ARG, "no estimate call yet");
  int rc = fetch_indices(ctx);
  if (rc) return rc;
  static_assert(sizeof(long long) == sizeof(int64_t), "offset table type");
  if (h_indices) *h_indices = ctx->h_out_idx.p;
  if (h_num_ground) *h_num_ground = ctx->h_counts.p;
  if (h_offsets) *h_offsets = reinterpret_cast<const int64_t*>(ctx->pt_off.data());
  return PWPP_OK;
}

int pwpp_bind_host_to_device(int device) {
  char bus[32] = {0};
  if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) { cudaGetLastError(); return -1; }
  for (char* c = bus; *c; ++c) *c = (char) std::tolower((unsigned char) *c);
  std::string base = std::string("/sys/bus/pci/devices/") + bus;
  int node = -1;
  if (FILE* f = std::fopen((base + "/numa_node").c_str(), "r")) { if (std::fscanf(f, "%d", &node) != 1) node = -1; std::fclose(f); }
  if (node < 0) return -1;
  std::string list;
  if (FILE* f = std::fopen(("/sys/devices/system/node/node" + std::to_string(node) + "/cpulist").c_str(), "r")) {
    char buf[4096] = {0};
    if (std::fgets(buf, sizeof buf, f)) list = buf;
    std::fclose(f);
  }
  if (list.empty()) return -1;
  cpu_set_t set;
  CPU_ZERO(&set);
  int ncpu = 0;
  const char* p = list.c_str();
  while (*p) {   // "0-31,64-95"
    char* end = nullptr;
    long a = std::strtol(p, &end, 10);
    if (end == p) break;
    long b = a;
    if (*end == '-') { p = end + 1; b = std::strtol(p, &end, 10); }
    for (long c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET((int) c, &set); ++ncpu; }
    p = (*end == ',') ? end + 1 : end;
    if (*end != ',' ) break;
  }
  if (ncpu == 0 || sched_setaffinity(0, sizeof set, &set) != 0) return -1;
  return node;
}

int pwpp_copy_bin_results(pwpp_ctx* ctx, int f, pwpp_bin_result* dst) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = bind_device(ctx);
  if (rc) return rc;
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  const int nb = ctx->gs.g[ctx->frame_set[f]].nbins;   // the records of the frame's set
  CU_TRY(cudaMemcpy(dst, ctx->d_fits.p + (size_t) f * ctx->gs.nbs, (size_t) nb * sizeof(BinFit), cudaMemcpyDeviceToHost));
  return PWPP_OK;
}
int pwpp_copy_bin_ids(pwpp_ctx* ctx, int f, uint16_t* dst) {
  int rc = check_frame(ctx, f);
  if (rc) return rc;
  rc = bind_device(ctx);
  if (rc) return rc;
  CU_TRY(cudaStreamSynchronize(ctx->last_stream));
  const int n = frame_n(ctx, f);
  if (n > 0) CU_TRY(cudaMemcpy(dst, ctx->d_bin_ids.p + ctx->pt_off[f], (size_t) n * sizeof(uint16_t), cudaMemcpyDeviceToHost));
  return PWPP_OK;
}

#if defined(PWPP_PHASE_CLOCKS)
// diagnostic builds only: cycles thread 0 of the k_fit_group CTAs spent per phase, [3 classes][16]; reset = 1 clears them
int pwpp_debug_phase_clocks(pwpp_ctx* ctx, unsigned long long* out, int reset) {
  if (!ctx) return PWPP_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  if (out) cudaMemcpyFromSymbol(out, g_phase_clk, sizeof(unsigned long long) * 48);
  if (reset) { static unsigned long long z[48]; cudaMemcpyToSymbol(g_phase_clk, z, sizeof z); }
  return PWPP_OK;
}
int pwpp_debug_events(pwpp_ctx* ctx, unsigned* out, int max_events) {
  if (!ctx) return -1;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  if (out && max_events >= 16384) cudaMemcpyFromSymbol(out, g_ev, (size_t) 16384 * 16);
  static uint4 z[16384];
  cudaMemcpyToSymbol(g_ev, z, sizeof z);
  return 16384;
}
#endif

}  // extern "C"
