// simt_ref32.cpp — TEST-ONLY: the SIMT twin (simt_twin.cpp, through simt_order_exact.cpp, included whole) in the reference
// arithmetic (pwpp_set_arithmetic(ctx, PWPP_ARITH_REFERENCE)). simt_estimate_ref32_multi is the launch sequence of launch_range()
// in csrc/pwpp_capi.cu for that mode: the front end, the six k_fit_ref32 launches in place of the fit kernels, the sorts (and the
// libstdc++ tie fix-up when the option order is 2), k_gle<true> and k_emit. The twin's getters read its results.
// simt_jsvd3f exposes the product's fp32 Jacobi SVD (csrc/pwpp_math.cuh) for a direct comparison with the oracle's.
// Built with plain g++ like the twin (tests/test_simt_ref32.py).
#include "simt_order_exact.cpp"

extern "C" {

void simt_jsvd3f(const float* cov, float* sv, float* U) { jacobi_svd3f(cov, sv, U); }

void simt_estimate_ref32_multi(void* h, int nframes, const float* const* pts_in, const int64_t* ns, int cols) {
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
  std::vector<float4> pts((size_t) total + 1);
  for (int f = 0; f < nframes; ++f)
    for (int64_t i = 0; i < ns[f]; ++i) {
      const float* p = pts_in[f] + i * cols;
      pts[(size_t) (pt_off[f] + i)] = make_float4(p[0], p[1], p[2], cols >= 4 ? p[3] : 0.f);
    }
  const int has_intensity = cols >= 4;
  std::vector<unsigned short> bin_ids((size_t) total + 1);
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
  // the global scratch of the patches above a kernel's shared capacity, filled with garbage so that nothing relies on its contents
  std::vector<unsigned long long> s_keys(2 * (size_t) total + 1, 0x5a5a5a5a5a5a5a5aull);
  std::vector<float4> s_pts((size_t) total + 1, make_float4(NAN, NAN, NAN, NAN));
  std::vector<float> s_sel(3 * (size_t) total + 1, NAN);
  std::vector<unsigned char> s_flags(2 * (size_t) total + 1, 0x5a);
  const Ref32Scratch scr{s_keys.data(), s_pts.data(), s_sel.data(), s_flags.data()};

  FrameTable ft{pt_off.data(), chunk_off.data()};
  StreamState* states = t->states.data();
  WorkQueues wq;
  for (int c = 0; c < NUM_CLASSES; ++c) wq.items[c] = items[c].data();
  wq.count = ctr.data();
  wq.head = ctr.data() + NUM_CLASSES;
  wq.labels = t->order ? labels.data() : nullptr;
  {   // one cluster per frame (pwpp_front.cuh), KITTI-sized CTAs
    const size_t sm_f = front_cluster_smem_bytes(nbp, FC_THREADS);
    for (int f = 0; f < nframes; ++f) {
#define FC_ARGS pts.data(), ft, states, g, ap, has_intensity, nbp, nb, bin_ids.data(), bin_off.data(), wq, fits.data(), sorted.data()
      if (t->fast) simt::launch_concurrent("k_front_cluster<fast>", FC_CS, FC_THREADS, sm_f, [&] { k_front_cluster<true, CLS_L2_MAX, FC_THREADS>(FC_ARGS); }, (unsigned) f);
      else simt::launch_concurrent("k_front_cluster<exact>", FC_CS, FC_THREADS, sm_f, [&] { k_front_cluster<false, CLS_L2_MAX, FC_THREADS>(FC_ARGS); }, (unsigned) f);
#undef FC_ARGS
    }
  }
  const int pg = t->persistent_ctas;
#define R32_ARGS sorted.data(), ft, states, g, ap, bin_off.data(), wq, part.data(), fits.data(), scr, t->order == PWPP_ORDER_REFERENCE_EXACT ? 1 : 0
  const size_t sm_s = ref32_smem_bytes(R32_SMALL_CAP), sm_b = ref32_smem_bytes(R32_BIG_CAP);
  simt::launch("k_fit_ref32<L3>", pg, 512, sm_b, [&] { k_fit_ref32<4, 512, R32_BIG_CAP>(R32_ARGS); });
  simt::launch("k_fit_ref32<L2>", pg, 256, sm_b, [&] { k_fit_ref32<3, 256, R32_BIG_CAP>(R32_ARGS); });
  simt::launch("k_fit_ref32<L1>", pg, 256, sm_b, [&] { k_fit_ref32<2, 256, R32_BIG_CAP>(R32_ARGS); });
  simt::launch("k_fit_ref32<M>", pg, 128, sm_s, [&] { k_fit_ref32<1, 128, R32_SMALL_CAP>(R32_ARGS); });
  simt::launch("k_fit_ref32<S>", pg, 128, sm_s, [&] { k_fit_ref32<0, 128, R32_SMALL_CAP>(R32_ARGS); });
  simt::launch("k_fit_ref32<X>", pg, 512, sm_b, [&] { k_fit_ref32<5, 512, R32_BIG_CAP>(R32_ARGS); });
#undef R32_ARGS
  for (int c = 0; c < NUM_CLASSES; ++c)
    if (ctr[NUM_CLASSES + c] < ctr[c]) { std::fprintf(stderr, "simt_ref32: class %d queue not drained (%d of %d)\n", c, ctr[NUM_CLASSES + c], ctr[c]); std::abort(); }
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
  if (t->order == PWPP_ORDER_REFERENCE_EXACT) {
    int* hx = ctr.data() + 2 * NUM_CLASSES + ORD_NUM_HEADS;
    std::vector<unsigned> xws((size_t) OX_X_WORDS * total + 1);
    launch_exact(sorted.data(), wq, hx, part.data(), xws.data(), pg);
  }
  int* d_ng = counts.data();
  int* d_np = counts.data() + nframes;
  int* d_nd = counts.data() + 2 * nframes;
  simt::launch("k_gle<ref32>", nframes, 32, gle_smem_bytes(t->max_sectors), [&] {
    k_gle<true>(ft, states, t->hist.data(), t->hcap, g, ap, nbp, t->max_sectors, bin_off.data(), fits.data(), segs.data(), d_ng, d_np, centers.data(), normals.data(), d_nd);
  });
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

}  // extern "C"
