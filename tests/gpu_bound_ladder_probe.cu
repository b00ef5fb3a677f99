// gpu_bound_ladder_probe.cu — TEST-ONLY: the width selector of bound calls with a width ladder (csrc/pwpp_ladder.cuh,
// k_ladder_select) compiled for sm_90a and run inside a real CUDA graph, so that tests/test_bound_ladder_backends.py runs the
// cases of tests/test_simt_bound_ladder.py on the GPU as well as through the SIMT stand-in (tests/simt/simt_bound_ladder.cpp).
// The graph is built as pwpp_capi.cu builds a laddered run: a conditional handle created on the capturing graph, the selector
// captured, then a SWITCH node added behind it from the capture's dependencies. Body i of the SWITCH is a memset node that writes
// i, so the probe reads back the value the device API set, not what the kernel meant to set. Host arrays in and out; the return
// value is PWPP_OK or PWPP_ERR_CUDA. Built by patchwork-plusplus_b200/build.py (build_examples) with the core library's nvcc line.
#include <algorithm>

#include "pwpp_ladder.cuh"

extern "C" {

int probe_ladder_select(int nframes, const int32_t* status, const int32_t* widths, int nwidths, int32_t* width, int32_t* index) {
  pwpp::LadderWidths lw{};
  lw.n = nwidths;
  for (int i = 0; i < nwidths; ++i) lw.w[i] = widths[i];
  int *d_status = nullptr, *d_out = nullptr;   // d_out: [0] the width, [1] the body's index
  cudaStream_t s = nullptr;
  cudaGraph_t g = nullptr;
  cudaGraphExec_t x = nullptr;
  const int init[2] = {-1, -1};
  int out[2] = {-1, -1};
  cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
#define STEP(expr) do { if (e == cudaSuccess) e = (expr); } while (0)
  STEP(cudaMalloc(&d_status, (size_t) std::max(nframes, 1) * sizeof(int)));
  STEP(cudaMalloc(&d_out, 2 * sizeof(int)));
  STEP(cudaMemcpy(d_status, status, (size_t) nframes * sizeof(int), cudaMemcpyHostToDevice));
  STEP(cudaMemcpy(d_out, init, sizeof(init), cudaMemcpyHostToDevice));
  STEP(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
  if (e == cudaSuccess) {
    cudaStreamCaptureStatus st;
    cudaGraph_t cg = nullptr;
    cudaGraphConditionalHandle h{};
    STEP(cudaStreamGetCaptureInfo_v3(s, &st, nullptr, &cg));
    STEP(cudaGraphConditionalHandleCreate(&h, cg, (unsigned) nwidths, cudaGraphCondAssignDefault));   // default: no body
    if (e == cudaSuccess) pwpp::k_ladder_select<<<1, pwpp::LS_THREADS, 0, s>>>(nframes, d_status, lw, d_out, h);
    STEP(cudaGetLastError());
    const cudaGraphNode_t* deps = nullptr;
    const cudaGraphEdgeData* edges = nullptr;
    size_t nd = 0;
    STEP(cudaStreamGetCaptureInfo_v3(s, &st, nullptr, &cg, &deps, &edges, &nd));
    cudaGraphNodeParams p = {};
    p.type = cudaGraphNodeTypeConditional;
    p.conditional.handle = h;
    p.conditional.type = cudaGraphCondTypeSwitch;
    p.conditional.size = (unsigned) nwidths;
    cudaGraphNode_t node{};
    STEP(cudaGraphAddNode_v2(&node, cg, deps, edges, nd, &p));
    for (int i = 0; i < nwidths && e == cudaSuccess; ++i) {
      cudaMemsetParams m = {};
      m.dst = d_out + 1;
      m.value = (unsigned) i;
      m.elementSize = sizeof(int);
      m.width = 1;
      m.height = 1;
      cudaGraphNode_t ms;
      STEP(cudaGraphAddMemsetNode(&ms, p.conditional.phGraph_out[i], nullptr, 0, &m));
    }
    STEP(cudaStreamUpdateCaptureDependencies_v2(s, &node, nullptr, 1, cudaStreamSetCaptureDependencies));
    const cudaError_t ee = cudaStreamEndCapture(s, &g);
    STEP(ee);
  }
  STEP(cudaGraphInstantiate(&x, g, 0));
  STEP(cudaGraphLaunch(x, s));
  STEP(cudaStreamSynchronize(s));
  STEP(cudaMemcpy(out, d_out, sizeof(out), cudaMemcpyDeviceToHost));
#undef STEP
  *width = out[0];
  *index = out[1];
  if (x) cudaGraphExecDestroy(x);
  if (g) cudaGraphDestroy(g);
  cudaFree(d_status);
  cudaFree(d_out);
  if (s) cudaStreamDestroy(s);
  return e == cudaSuccess ? PWPP_OK : PWPP_ERR_CUDA;
}

}  // extern "C"
