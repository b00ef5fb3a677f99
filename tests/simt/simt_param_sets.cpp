// simt_param_sets.cpp — TEST-ONLY: the SIMT twin (simt_twin.cpp, included whole) with several parameter sets in one context, the
// CPU counterpart of pwpp_create_sets. Stream s runs with set stream_set[s]; one launch sequence (the kernels of launch_range() in
// csrc/pwpp_capi.cu) mixes frames of every set, with the set tables passed by value and a per-frame set table. Per-frame outputs
// are indexed by call position and sized by the frame's set; state by stream id (simt_select picks either). Built with plain g++
// like the twin. tests/test_simt_param_sets.py compares every frame with the oracle run with its own set.
#include "simt_twin.cpp"

namespace {
struct SetsTwin : SimtTwin {
  int num_sets = 1;
  GeometrySets gs;
  AlgoParamSets aps;
  bool set_fast[MAX_PARAM_SETS] = {};
  std::vector<int> stream_set;
};
}  // namespace

extern "C" {

// hist rows are strided by the largest history_cap of the sets (SimtTwin::hcap, read by simt_history)
void* simt_create_sets(const pwpp_params* sets, int num_sets, const int* stream_set, int num_streams) {
  if (num_sets < 1 || num_sets > MAX_PARAM_SETS) return nullptr;
  SetsTwin* t = new SetsTwin();
  t->num_streams = num_streams;
  t->num_sets = num_sets;
  t->stream_set.assign(stream_set, stream_set + num_streams);
  t->gs.nbs = 0;
  t->hcap = 0;
  for (int k = 0; k < num_sets; ++k) {
    build_geometry(sets[k], t->gs.g[k], t->aps.a[k], t->set_fast[k]);
    t->gs.nbs = std::max(t->gs.nbs, t->gs.g[k].nbins);
    t->hcap = std::max(t->hcap, history_cap(t->gs.g[k], t->aps.a[k]));
    for (int z = 0; z < 4; ++z) t->max_sectors = std::max(t->max_sectors, t->gs.g[k].num_sectors[z]);
  }
  t->g = t->gs.g[0];
  t->ap = t->aps.a[0];
  t->nbp = ((t->gs.nbs + PW_NUM_PSEUDO + 31) / 32) * 32;
  t->states.resize(num_streams);
  for (int s = 0; s < num_streams; ++s) init_state(sets[stream_set[s]], t->states[s]);
  t->hist.assign((size_t) num_streams * 2 * 4 * t->hcap, 0.0);
  t->out.resize(num_streams);
  return static_cast<SimtTwin*>(t);
}

// One launch sequence over frames of pairwise distinct streams (returns -1 otherwise, nothing run). front / patch / order as in
// simt_set_option. The binning kernel is the fp32 filter only when every set the call names allows it (range_fast in
// pwpp_capi.cu); *fast_out reports the choice.
int simt_estimate_sets(void* h, int nframes, const int* streams, const float* const* pts_in, const int64_t* ns, int cols, int* fast_out) {
  SetsTwin* t = static_cast<SetsTwin*>(static_cast<SimtTwin*>(h));
  std::vector<char> used(t->num_streams, 0);
  for (int f = 0; f < nframes; ++f) {
    if (streams[f] < 0 || streams[f] >= t->num_streams || used[streams[f]]) return -1;
    used[streams[f]] = 1;
  }
  if ((int) t->out.size() < nframes) t->out.resize(nframes);
  std::vector<int> pset(nframes);
  bool fast = true;
  for (int f = 0; f < nframes; ++f) { pset[f] = t->stream_set[streams[f]]; fast = fast && t->set_fast[pset[f]]; }
  if (fast_out) *fast_out = fast ? 1 : 0;
  const GeometrySets& gs = t->gs;
  const AlgoParamSets& aps = t->aps;
  const int nb = gs.nbs, nbp = t->nbp, nb_all = nb + PW_NUM_PSEUDO;
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
  std::vector<int> ctr(2 * NUM_CLASSES + ORD_NUM_HEADS, 0);
  std::vector<unsigned char> labels((size_t) total + 1, 0);
  std::vector<int> counts((size_t) 3 * nframes, 0);
  std::vector<float> centers((size_t) nframes * nb * 3), normals((size_t) nframes * nb * 3);

  FrameTable ft{pt_off.data(), chunk_off.data(), streams, pset.data()};
  StreamState* states = t->states.data();
  const float4* d_pts = pts.data();
  WorkQueues wq;
  for (int c = 0; c < NUM_CLASSES; ++c) wq.items[c] = items[c].data();
  wq.count = ctr.data();
  wq.head = ctr.data() + NUM_CLASSES;
  wq.labels = t->order ? labels.data() : nullptr;
  if (t->front) {
    const int nt = t->front == 3 ? FC_THREADS_DENSE : FC_THREADS;
    const size_t sm_f = front_cluster_smem_bytes(nbp, nt);
    for (int f = 0; f < nframes; ++f) {
#define FC_ARGS d_pts, ft, states, gs, aps, has_intensity, nbp, nb, bin_ids.data(), bin_off.data(), wq, fits.data(), sorted.data()
      if (nt == FC_THREADS_DENSE) {
        if (fast) simt::launch_concurrent("k_front_cluster<fast,512>", FC_CS, nt, sm_f, [&] { k_front_cluster<true, CLS_L2_MAX, FC_THREADS_DENSE>(FC_ARGS); }, (unsigned) f);
        else simt::launch_concurrent("k_front_cluster<exact,512>", FC_CS, nt, sm_f, [&] { k_front_cluster<false, CLS_L2_MAX, FC_THREADS_DENSE>(FC_ARGS); }, (unsigned) f);
      } else {
        if (fast) simt::launch_concurrent("k_front_cluster<fast>", FC_CS, nt, sm_f, [&] { k_front_cluster<true, CLS_L2_MAX, FC_THREADS>(FC_ARGS); }, (unsigned) f);
        else simt::launch_concurrent("k_front_cluster<exact>", FC_CS, nt, sm_f, [&] { k_front_cluster<false, CLS_L2_MAX, FC_THREADS>(FC_ARGS); }, (unsigned) f);
      }
#undef FC_ARGS
    }
  } else {
    if (max_chunks > 0) {
      dim3 grid(max_chunks, nframes);
      const size_t sm_h = nbp * sizeof(unsigned int);
#define HIST_ARGS d_pts, ft, states, gs, aps, has_intensity, nbp, bin_ids.data(), chist.data()
      if (!fast) simt::launch("k_bin_hist<false,0>", grid, CHUNK_THREADS, sm_h, [&] { k_bin_hist<false, 0>(HIST_ARGS); });
      else simt::launch("k_bin_hist<true,2>", grid, CHUNK_THREADS, sm_h, [&] { k_bin_hist<true, 2>(HIST_ARGS); });
#undef HIST_ARGS
    }
    simt::launch("k_bin_scan", nframes, 512, (nbp + 1) * sizeof(int),
                 [&] { k_bin_scan<CLS_L2_MAX>(ft, nbp, nb, gs, aps, chist.data(), cbase.data(), bin_off.data(), wq, fits.data()); });
    if (max_chunks > 0) {
      dim3 grid(max_chunks, nframes);
      const size_t sm_sc = (size_t) (CHUNK_THREADS / 32) * nbp * sizeof(unsigned int);
      simt::launch("k_scatter<false,4>", grid, CHUNK_THREADS, sm_sc, [&] { k_scatter<false, 4>(d_pts, ft, nbp, bin_ids.data(), cbase.data(), sorted.data()); });
    }
  }
#define FIT_ARGS sorted.data(), ft, states, gs, aps, nbp, bin_off.data(), wq, part.data(), fits.data()
  const int pg = t->persistent_ctas;
  const size_t sm_m = FITW_WARPS * CLS_M_MAX * sizeof(float4), sm_l2 = 3 * 4096 * sizeof(float), sm_l3 = 3 * 8192 * sizeof(float);
  if (t->patch) {
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
    if (ctr[NUM_CLASSES + c] < ctr[c]) { std::fprintf(stderr, "simt_param_sets: class %d queue not drained (%d of %d)\n", c, ctr[NUM_CLASSES + c], ctr[c]); std::abort(); }
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
  int* d_ng = counts.data();
  int* d_np = counts.data() + nframes;
  int* d_nd = counts.data() + 2 * nframes;
  simt::launch("k_gle", nframes, 32, gle_smem_bytes(t->max_sectors), [&] {
    k_gle(ft, states, t->hist.data(), t->hcap, gs, aps, nbp, t->max_sectors, bin_off.data(), fits.data(), segs.data(), d_ng, d_np, centers.data(), normals.data(), d_nd);
  });
  if (max_chunks > 0) {
    const long long max_pts = (long long) max_chunks * CHUNK_PTS;
    dim3 grid((unsigned) ((max_pts + (long long) EMIT_TILE * EMIT_WARPS - 1) / ((long long) EMIT_TILE * EMIT_WARPS)), nframes);
    simt::launch("k_emit", grid, EMIT_WARPS * 32, 0, [&] { k_emit(ft, gs, nbp, bin_off.data(), fits.data(), segs.data(), part.data(), sorted.data(), out_idx.data()); });
  }
  for (int f = 0; f < nframes; ++f) {
    FrameOut& o = t->out[f];
    const long long p0 = pt_off[f];
    const int n = (int) ns[f], ng = d_ng[f], nd = d_nd[f];
    const int fnb = gs.g[pset[f]].nbins;   // the frame's own set
    o.ground.assign(out_idx.begin() + p0, out_idx.begin() + p0 + ng);
    o.nonground.assign(out_idx.begin() + p0 + ng, out_idx.begin() + p0 + (n - nd));
    o.bin_ids.assign(bin_ids.begin() + p0, bin_ids.begin() + p0 + n);
    o.fits.assign(fits.begin() + (size_t) f * nb, fits.begin() + (size_t) f * nb + fnb);
    o.npatch = d_np[f];
    o.centers.assign(centers.begin() + (size_t) f * nb * 3, centers.begin() + (size_t) f * nb * 3 + (size_t) o.npatch * 3);
    o.normals.assign(normals.begin() + (size_t) f * nb * 3, normals.begin() + (size_t) f * nb * 3 + (size_t) o.npatch * 3);
  }
  return 0;
}

}  // extern "C"
