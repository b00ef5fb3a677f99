// simt_order_exact.cpp — TEST-ONLY: the SIMT twin (simt_twin.cpp, included whole) with the libstdc++ tie fix-up of
// PWPP_ORDER_REFERENCE_EXACT (csrc/pwpp_order_exact.cuh). simt_estimate_exact_multi is the twin's launch sequence with, when the
// option order is 2, the five k_order_exact_* launches behind the five k_order_* launches, as launch_range() in csrc/pwpp_capi.cu
// issues them; the twin's getters read its results. simt_order_exact runs the sort and the fix-up alone over a list of patches
// (the CPU counterpart of tests/gpu_order_exact_probe.cu). Built with plain g++ like the twin (tests/test_order_exact.py).
#include "simt_twin.cpp"

namespace {
unsigned long long g_ox_counts[OX_NUM_STATS] = {};   // counters of every fix-up launch of the process

// the five fix-up launches, in the order of the k_order_* launches; heads: their five ticket counters
void launch_exact(const float4* sorted, WorkQueues wq, int* heads, int* part, unsigned* xws, int grid) {
  unsigned long long* cnt = g_ox_counts;
  simt::launch("k_order_exact_big<X>", grid, OX_WARP_THREADS, 0, [&] { k_order_exact_big<5>(sorted, wq, heads + 0, part, xws, cnt); });
  simt::launch("k_order_exact_big<L3>", grid, OX_WARP_THREADS, 0, [&] { k_order_exact_big<4>(sorted, wq, heads + 1, part, xws, cnt); });
  simt::launch("k_order_exact_big<L2>", grid, OX_WARP_THREADS, 0, [&] { k_order_exact_big<3>(sorted, wq, heads + 2, part, xws, cnt); });
  simt::launch("k_order_exact_big<L1>", grid, OX_WARP_THREADS, 0, [&] { k_order_exact_big<2>(sorted, wq, heads + 3, part, xws, cnt); });
  simt::launch("k_order_exact_warp", grid, OX_WARP_THREADS, ox_warp_smem_bytes(), [&] { k_order_exact_warp(sorted, wq, heads + 4, part, cnt); });
}
}  // namespace

extern "C" {

void simt_order_exact_counts(uint64_t* out) { for (int k = 0; k < OX_NUM_STATS; ++k) out[k] = g_ox_counts[k]; }

// One frame for each of the first nframes streams, as simt_estimate_multi, with the fix-up when the option order is 2.
void simt_estimate_exact_multi(void* h, int nframes, const float* const* pts_in, const int64_t* ns, int cols) {
  SimtTwin* t = (SimtTwin*) h;
  const Geometry g = t->g;
  const AlgoParams ap = t->ap;
  const int nb = g.nbins, nbp = t->nbp, nb_all = nb + PW_NUM_PSEUDO;
  std::vector<long long> pt_off(nframes + 1, 0);
  std::vector<int> chunk_off(nframes + 1, 0);
  int max_chunks = 0;
  for (int f = 0; f < nframes; ++f) {
    pt_off[f + 1] = pt_off[f] + ns[f];
    const int nc = (int) ((ns[f] + CHUNK_PTS - 1) / CHUNK_PTS);
    chunk_off[f + 1] = chunk_off[f] + nc;
    max_chunks = std::max(max_chunks, nc);
  }
  const long long total = pt_off[nframes];
  const int total_chunks = chunk_off[nframes];
  std::vector<float4> pts((size_t) total + 1);
  for (int f = 0; f < nframes; ++f)
    for (int64_t i = 0; i < ns[f]; ++i) {
      const float* p = pts_in[f] + i * cols;
      pts[(size_t) (pt_off[f] + i)] = make_float4(p[0], p[1], p[2], cols >= 4 ? p[3] : 0.f);
    }
  const int has_intensity = cols >= 4;
  std::vector<unsigned short> bin_ids((size_t) total + 1), chist((size_t) total_chunks * nbp + 1);
  std::vector<unsigned int> cbase((size_t) total_chunks * nbp + 1);
  std::vector<int> bin_off((size_t) nframes * (nbp + 1));
  std::vector<float4> sorted((size_t) total + 1);
  std::vector<int> part((size_t) total + 1, -7), out_idx((size_t) total + 1, -7);
  std::vector<BinFit> fits((size_t) nframes * nb);
  std::vector<BinSeg> segs((size_t) nframes * nb_all);
  std::vector<int4> items[NUM_CLASSES];
  for (auto& v : items) v.resize((size_t) nframes * nb + 1);
  std::vector<int> ctr(2 * NUM_CLASSES + 2 * ORD_NUM_HEADS, 0);
  std::vector<unsigned char> labels((size_t) total + 1, 0);
  std::vector<int> counts((size_t) 3 * nframes, 0);
  std::vector<float> centers((size_t) nframes * nb * 3), normals((size_t) nframes * nb * 3);

  FrameTable ft{pt_off.data(), chunk_off.data()};
  StreamState* states = t->states.data();
  const float4* d_pts = pts.data();
  WorkQueues wq;
  for (int c = 0; c < NUM_CLASSES; ++c) wq.items[c] = items[c].data();
  wq.count = ctr.data();
  wq.head = ctr.data() + NUM_CLASSES;
  wq.labels = t->order ? labels.data() : nullptr;
  if (t->front) {   // one cluster per frame (pwpp_front.cuh): the CTAs of a cluster run concurrently, frames one after another
    // front=1: 8 x 256 threads (KITTI-sized frames), front=3: 8 x 512 (what dense frames get)
    const int nt = t->front == 3 ? FC_THREADS_DENSE : FC_THREADS;
    const size_t sm_f = front_cluster_smem_bytes(nbp, nt);
    for (int f = 0; f < nframes; ++f) {
#define FC_ARGS d_pts, ft, states, g, ap, has_intensity, nbp, nb, bin_ids.data(), bin_off.data(), wq, fits.data(), sorted.data()
      if (nt == FC_THREADS_DENSE) {
        if (t->fast) simt::launch_concurrent("k_front_cluster<fast,512>", FC_CS, nt, sm_f, [&] { k_front_cluster<true, CLS_L2_MAX, FC_THREADS_DENSE>(FC_ARGS); }, (unsigned) f);
        else simt::launch_concurrent("k_front_cluster<exact,512>", FC_CS, nt, sm_f, [&] { k_front_cluster<false, CLS_L2_MAX, FC_THREADS_DENSE>(FC_ARGS); }, (unsigned) f);
      } else {
        if (t->fast) simt::launch_concurrent("k_front_cluster<fast>", FC_CS, nt, sm_f, [&] { k_front_cluster<true, CLS_L2_MAX, FC_THREADS>(FC_ARGS); }, (unsigned) f);
        else simt::launch_concurrent("k_front_cluster<exact>", FC_CS, nt, sm_f, [&] { k_front_cluster<false, CLS_L2_MAX, FC_THREADS>(FC_ARGS); }, (unsigned) f);
      }
#undef FC_ARGS
    }
  } else {
    if (max_chunks > 0) {
      dim3 grid(max_chunks, nframes);
      const size_t sm_h = nbp * sizeof(unsigned int);
#define HIST_ARGS d_pts, ft, states, g, ap, has_intensity, nbp, bin_ids.data(), chist.data()
      if (!t->fast) simt::launch("k_bin_hist<false,0>", grid, CHUNK_THREADS, sm_h, [&] { k_bin_hist<false, 0>(HIST_ARGS); });
      else simt::launch("k_bin_hist<true,2>", grid, CHUNK_THREADS, sm_h, [&] { k_bin_hist<true, 2>(HIST_ARGS); });
#undef HIST_ARGS
    }
    simt::launch("k_bin_scan", nframes, 512, (nbp + 1) * sizeof(int),
                 [&] { k_bin_scan<CLS_L2_MAX>(ft, nbp, nb, ap.num_min_pts, chist.data(), cbase.data(), bin_off.data(), wq, fits.data()); });
    if (max_chunks > 0) {
      dim3 grid(max_chunks, nframes);
      const size_t sm_sc = (size_t) (CHUNK_THREADS / 32) * nbp * sizeof(unsigned int);
      simt::launch("k_scatter<false,4>", grid, CHUNK_THREADS, sm_sc, [&] { k_scatter<false, 4>(d_pts, ft, nbp, bin_ids.data(), cbase.data(), sorted.data()); });
    }
  }
#define FIT_ARGS sorted.data(), ft, states, g, ap, nbp, bin_off.data(), wq, part.data(), fits.data()
  const int pg = t->persistent_ctas;
  const size_t sm_m = FITW_WARPS * CLS_M_MAX * sizeof(float4), sm_l2 = 3 * 4096 * sizeof(float), sm_l3 = 3 * 8192 * sizeof(float);
  if (t->patch) {   // PWPP_FIT_PATCH: patches above 512 points on k_fit_patch
    simt::launch("k_fit_patch<16>", pg, 16 * 32, (size_t) 16 * FP_STG * 16, [&] { k_fit_patch<16, 1, 4>(FIT_ARGS); });
    simt::launch("k_fit_patch<8>", pg, 8 * 32, (size_t) 8 * FP_STG * 16, [&] { k_fit_patch<8, 2, 3>(FIT_ARGS); });
    simt::launch("k_fit_patch<4>", pg, 4 * 32, (size_t) 4 * FP_STG * 16, [&] { k_fit_patch<4, 4, 2>(FIT_ARGS); });
  } else {
    simt::launch("k_fit_cta<8192,4,2,8,fuse>", pg, FIT_THREADS, sm_l3, [&] { k_fit_cta<8192, 4, 2, 8, true>(FIT_ARGS); });
    simt::launch("k_fit_cta<4096,3,3,8,fuse,pls>", pg, FIT_THREADS, sm_l2, [&] { k_fit_cta<4096, 3, 3, 8, true, true>(FIT_ARGS); });
    simt::launch("k_fit_warp<false,2,2,pls>", pg, FITW_WARPS * 32, 0, [&] { k_fit_warp<false, 2, 2, 2, 3, false, true>(FIT_ARGS); });
  }
  simt::launch("k_fit_warp<true,1,1,pls>", pg, FITW_WARPS * 32, sm_m, [&] { k_fit_warp<true, 1, 1, 2, 3, false, true>(FIT_ARGS); });
  simt::launch("k_fit_resident<8,8,0>", pg, FIT_THREADS, 0, [&] { k_fit_resident<8, 8, 0, 2>(FIT_ARGS); });
  simt::launch("k_fit_big<16,1,fuse>", pg, 512, 0, [&] { k_fit_big<16, 1, true>(FIT_ARGS); });
#undef FIT_ARGS
  for (int c = 0; c < NUM_CLASSES; ++c)
    if (ctr[NUM_CLASSES + c] < ctr[c]) { std::fprintf(stderr, "simt_twin: class %d queue not drained (%d of %d)\n", c, ctr[NUM_CLASSES + c], ctr[c]); std::abort(); }
  {
    char buf[256];
    std::snprintf(buf, sizeof buf, "S=%d M=%d L1=%d L2=%d L3=%d X=%d", ctr[0], ctr[1], ctr[2], ctr[3], ctr[4], ctr[5]);
    t->last_launches = buf;
  }
  if (t->order) {
    int* heads = ctr.data() + 2 * NUM_CLASSES;
    simt::launch("k_order_cta<X>", pg, 512, ord_cta_smem_bytes(512), [&] { k_order_cta<512, 5>(sorted.data(), wq, heads + 0, part.data()); });
    simt::launch("k_order_cta<L3>", pg, 512, ord_cta_smem_bytes(512), [&] { k_order_cta<512, 4>(sorted.data(), wq, heads + 1, part.data()); });
    simt::launch("k_order_cta<L2>", pg, 256, ord_cta_smem_bytes(256), [&] { k_order_cta<256, 3>(sorted.data(), wq, heads + 2, part.data()); });
    simt::launch("k_order_cta<L1>", pg, 128, ord_cta_smem_bytes(128), [&] { k_order_cta<128, 2>(sorted.data(), wq, heads + 3, part.data()); });
    simt::launch("k_order_warp", pg, ORD_WARP_THREADS, 0, [&] { k_order_warp(sorted.data(), wq, heads + 4, part.data()); });
  }
  if (t->order == PWPP_ORDER_REFERENCE_EXACT) {   // each class's fix-up behind its sort (pwpp_order_exact.cuh)
    int* hx = ctr.data() + 2 * NUM_CLASSES + ORD_NUM_HEADS;
    std::vector<unsigned> xws((size_t) OX_X_WORDS * total + 1);
    launch_exact(sorted.data(), wq, hx, part.data(), xws.data(), pg);
  }
  int* d_ng = counts.data();
  int* d_np = counts.data() + nframes;
  int* d_nd = counts.data() + 2 * nframes;
  {
    const size_t gle_smem = gle_smem_bytes(t->max_sectors);
    simt::launch("k_gle", nframes, 32, gle_smem, [&] {
      k_gle(ft, states, t->hist.data(), t->hcap, g, ap, nbp, t->max_sectors, bin_off.data(), fits.data(), segs.data(), d_ng, d_np, centers.data(), normals.data(), d_nd);
    });
  }
  if (max_chunks > 0) {
    const long long max_pts = (long long) max_chunks * CHUNK_PTS;
    dim3 grid((unsigned) ((max_pts + (long long) EMIT_TILE * EMIT_WARPS - 1) / ((long long) EMIT_TILE * EMIT_WARPS)), nframes);
    simt::launch("k_emit", grid, EMIT_WARPS * 32, 0, [&] { k_emit(ft, g, nbp, bin_off.data(), fits.data(), segs.data(), part.data(), sorted.data(), out_idx.data()); });
  }
  for (int f = 0; f < nframes; ++f) {
    FrameOut& o = t->out[f];
    const long long p0 = pt_off[f];
    const int n = (int) ns[f], ng = d_ng[f], nd = d_nd[f];
    o.ground.assign(out_idx.begin() + p0, out_idx.begin() + p0 + ng);
    o.nonground.assign(out_idx.begin() + p0 + ng, out_idx.begin() + p0 + (n - nd));
    o.bin_ids.assign(bin_ids.begin() + p0, bin_ids.begin() + p0 + n);
    o.fits.assign(fits.begin() + (size_t) f * nb, fits.begin() + (size_t) (f + 1) * nb);
    o.npatch = d_np[f];
    o.centers.assign(centers.begin() + (size_t) f * nb * 3, centers.begin() + (size_t) f * nb * 3 + (size_t) o.npatch * 3);
    o.normals.assign(normals.begin() + (size_t) f * nb * 3, normals.begin() + (size_t) f * nb * 3 + (size_t) o.npatch * 3);
  }
}

void simt_estimate_exact(void* h, const float* pts, int64_t n, int cols) {
  const float* p[1] = {pts};
  const int64_t ns[1] = {n};
  simt_estimate_exact_multi(h, 1, p, ns, cols);
  ((SimtTwin*) h)->sel = 0;
}

// probe_order_exact (tests/gpu_order_exact_probe.cu) through the stand-in: npatch patches back to back, point i of the whole array
// has index i and z value z[i]; labels (or all ground); out: every patch's list after k_order_* and k_order_exact_*, local indices;
// counts: the fix-up's counters of this call.
int simt_order_exact(int npatch, const float* z, const int64_t* sizes, const unsigned char* labels, int32_t* out, uint64_t* counts) {
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
  std::vector<float4> pts(np + 1);
  std::vector<unsigned char> lab(np + 1, PW_LABEL_GROUND);
  for (size_t i = 0; i < np; ++i) {
    pts[i] = make_float4(0.f, 0.f, z[i], __int_as_float((int) i));
    if (labels) lab[i] = labels[i];
  }
  std::vector<int> ctr(2 * NUM_CLASSES + 2 * ORD_NUM_HEADS, 0), part(np + 1, -7);
  std::vector<unsigned> xws((size_t) OX_X_WORDS * np + 1);
  WorkQueues wq;
  for (int c = 0; c < NUM_CLASSES; ++c) { ctr[c] = (int) items[c].size(); items[c].push_back(make_int4(0, 0, 0, 0)); wq.items[c] = items[c].data(); }
  wq.count = ctr.data();
  wq.head = ctr.data() + NUM_CLASSES;
  wq.labels = lab.data();
  int* heads = ctr.data() + 2 * NUM_CLASSES;
  const float4* P = pts.data();
  int* d_part = part.data();
  unsigned long long before[OX_NUM_STATS];
  for (int k = 0; k < OX_NUM_STATS; ++k) before[k] = g_ox_counts[k];
  simt::launch("k_order_cta<X>", 2, 512, ord_cta_smem_bytes(512), [&] { k_order_cta<512, 5>(P, wq, heads + 0, d_part); });
  simt::launch("k_order_cta<L3>", 2, 512, ord_cta_smem_bytes(512), [&] { k_order_cta<512, 4>(P, wq, heads + 1, d_part); });
  simt::launch("k_order_cta<L2>", 2, 256, ord_cta_smem_bytes(256), [&] { k_order_cta<256, 3>(P, wq, heads + 2, d_part); });
  simt::launch("k_order_cta<L1>", 2, 128, ord_cta_smem_bytes(128), [&] { k_order_cta<128, 2>(P, wq, heads + 3, d_part); });
  simt::launch("k_order_warp", 2, ORD_WARP_THREADS, 0, [&] { k_order_warp(P, wq, heads + 4, d_part); });
  launch_exact(P, wq, heads + ORD_NUM_HEADS, d_part, xws.data(), 2);
  for (int p = 0; p < npatch; ++p)
    for (long long i = off[p]; i < off[p + 1]; ++i) out[i] = part[i] - (int) off[p];
  for (int k = 0; k < OX_NUM_STATS; ++k) counts[k] = g_ox_counts[k] - before[k];
  return PWPP_OK;
}
}  // extern "C"
