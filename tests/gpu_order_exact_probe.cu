// gpu_order_exact_probe.cu — TEST-ONLY: the reference-order sort (k_order_*) and its libstdc++ tie fix-up (k_order_exact_*,
// csrc/pwpp_order_exact.cuh) compiled for sm_90a and launched class by class the way pwpp_capi.cu launches them, so that
// tests/test_order_exact_backends.py runs its cases on the GPU as well as through the SIMT stand-in (simt_order_exact in
// tests/simt/simt_order_exact.cpp). Built by patchwork-plusplus_b200/build.py (build_examples) with the core library's nvcc line.
#include <algorithm>
#include <cstring>
#include <vector>

#include "pwpp.h"
#include "pwpp_kernels.cuh"

using namespace pwpp;

namespace {
template <typename T>
cudaError_t upload(T** d, const T* h, size_t n) {
  cudaError_t e = cudaMalloc(d, (n ? n : 1) * sizeof(T));
  if (e == cudaSuccess && n) e = cudaMemcpy(*d, h, n * sizeof(T), cudaMemcpyHostToDevice);
  return e;
}
template <class F>
cudaError_t smem_limit(F* fn, size_t bytes) {
  return bytes > 48 * 1024 ? cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) bytes) : cudaSuccess;
}
}  // namespace

extern "C" {

// npatch patches back to back, patch p of sizes[p] points with the z values z[...]; point i of the whole array has index i.
// labels[i]: what the fit made of point i (PW_LABEL_GROUND, an R-VPF iteration, PW_LABEL_REJECT), or NULL for all ground.
// out[i]: the patch's index list after both stages, as indices local to the patch; counts[3]: the fix-up's counters.
// Synchronous: PWPP_ERR_INVALID_ARG for a bad size, PWPP_ERR_CUDA for a CUDA error.
int probe_order_exact(int npatch, const float* z, const int64_t* sizes, const unsigned char* labels, int32_t* out, uint64_t* counts) {
  if (npatch < 0) return PWPP_ERR_INVALID_ARG;
  std::vector<long long> off(npatch + 1, 0);
  std::vector<int4> items[NUM_CLASSES];
  for (int p = 0; p < npatch; ++p) {
    if (sizes[p] < 0 || sizes[p] > (1 << 24)) return PWPP_ERR_INVALID_ARG;
    off[p + 1] = off[p] + sizes[p];
    const int n = (int) sizes[p];
    const int c = n <= CLS_S_MAX ? 0 : n <= CLS_M_MAX ? 1 : n <= CLS_L1_MAX ? 2 : n <= CLS_L2_MAX ? 3 : n <= CLS_L3_MAX ? 4 : 5;
    items[c].push_back(make_int4(p, n, (int) (unsigned) (off[p] & 0xffffffffll), (int) (off[p] >> 32)));
  }
  const size_t np = (size_t) off[npatch];
  std::vector<float4> pts(np);
  std::vector<unsigned char> lab(np, PW_LABEL_GROUND);
  for (size_t i = 0; i < np; ++i) {
    const int idx = (int) i;
    float w;
    std::memcpy(&w, &idx, sizeof w);
    pts[i] = make_float4(0.f, 0.f, z[i], w);
    if (labels) lab[i] = labels[i];
  }
  std::vector<int> ctr(2 * NUM_CLASSES + 2 * ORD_NUM_HEADS, 0);
  for (int c = 0; c < NUM_CLASSES; ++c) ctr[c] = (int) items[c].size();
  float4* d_pts = nullptr;
  int4* d_items[NUM_CLASSES] = {};
  int *d_ctr = nullptr, *d_part = nullptr;
  unsigned char* d_lab = nullptr;
  unsigned* d_xws = nullptr;
  unsigned long long* d_cnt = nullptr;
  const unsigned long long zero[OX_NUM_STATS] = {};
  cudaError_t e = upload(&d_pts, pts.data(), np);
  for (int c = 0; c < NUM_CLASSES && e == cudaSuccess; ++c) e = upload(&d_items[c], items[c].data(), items[c].size());
  if (e == cudaSuccess) e = upload(&d_ctr, ctr.data(), ctr.size());
  if (e == cudaSuccess) e = upload(&d_lab, lab.data(), np);
  if (e == cudaSuccess) e = cudaMalloc(&d_part, (np ? np : 1) * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&d_xws, ((size_t) OX_X_WORDS * np + 1) * sizeof(unsigned));
  if (e == cudaSuccess) e = upload(&d_cnt, zero, OX_NUM_STATS);
  const size_t sm_w = ox_warp_smem_bytes();
  if (e == cudaSuccess) e = smem_limit(k_order_cta<512, 5>, ord_cta_smem_bytes(512));
  if (e == cudaSuccess) e = smem_limit(k_order_cta<512, 4>, ord_cta_smem_bytes(512));
  if (e == cudaSuccess) e = smem_limit(k_order_exact_warp, sm_w);
  if (e == cudaSuccess) {
    WorkQueues wq;
    for (int c = 0; c < NUM_CLASSES; ++c) wq.items[c] = d_items[c];
    wq.count = d_ctr;
    wq.head = d_ctr + NUM_CLASSES;
    wq.labels = d_lab;
    int* heads = d_ctr + 2 * NUM_CLASSES;
    int* hx = heads + ORD_NUM_HEADS;
    const int g = 132;
    k_order_cta<512, 5><<<g, 512, ord_cta_smem_bytes(512)>>>(d_pts, wq, heads + 0, d_part);
    k_order_exact_big<5><<<g, OX_WARP_THREADS>>>(d_pts, wq, hx + 0, d_part, d_xws, d_cnt);
    k_order_cta<512, 4><<<g, 512, ord_cta_smem_bytes(512)>>>(d_pts, wq, heads + 1, d_part);
    k_order_exact_big<4><<<g, OX_WARP_THREADS>>>(d_pts, wq, hx + 1, d_part, d_xws, d_cnt);
    k_order_cta<256, 3><<<g, 256, ord_cta_smem_bytes(256)>>>(d_pts, wq, heads + 2, d_part);
    k_order_exact_big<3><<<g, OX_WARP_THREADS>>>(d_pts, wq, hx + 2, d_part, d_xws, d_cnt);
    k_order_cta<128, 2><<<g, 128, ord_cta_smem_bytes(128)>>>(d_pts, wq, heads + 3, d_part);
    k_order_exact_big<2><<<g, OX_WARP_THREADS>>>(d_pts, wq, hx + 3, d_part, d_xws, d_cnt);
    k_order_warp<<<g, ORD_WARP_THREADS>>>(d_pts, wq, heads + 4, d_part);
    k_order_exact_warp<<<g, OX_WARP_THREADS, sm_w>>>(d_pts, wq, hx + 4, d_part, d_cnt);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  std::vector<int> part(np);
  if (e == cudaSuccess && np) e = cudaMemcpy(part.data(), d_part, np * sizeof(int), cudaMemcpyDeviceToHost);
  unsigned long long c[OX_NUM_STATS] = {};
  if (e == cudaSuccess) e = cudaMemcpy(c, d_cnt, sizeof c, cudaMemcpyDeviceToHost);
  cudaFree(d_pts);
  for (auto* p : d_items) cudaFree(p);
  cudaFree(d_ctr);
  cudaFree(d_lab);
  cudaFree(d_part);
  cudaFree(d_xws);
  cudaFree(d_cnt);
  if (e != cudaSuccess) return PWPP_ERR_CUDA;
  for (int p = 0; p < npatch; ++p)
    for (long long i = off[p]; i < off[p + 1]; ++i) out[i] = part[i] - (int) off[p];
  for (int k = 0; k < OX_NUM_STATS; ++k) counts[k] = c[k];
  return PWPP_OK;
}
}  // extern "C"
