// simt_bound_rings.cpp — TEST-ONLY: the frame-table kernels of ring-bound calls (csrc/pwpp_records.cuh, k_bound_table_rings and
// k_bound_table_rings_actions), then the record unpack and the part gather over the run's record table they write, executed on
// the CPU by the SIMT stand-in (tests/test_simt_bound_rings.py).
#include "simt_records.cpp"

extern "C" {

int simt_stream_state_bytes() { return (int) sizeof(pwpp::StreamState); }
int simt_record_frame_bytes() { return (int) sizeof(pwpp::RecordFrame); }

// One ring table launch over nframes frames, as pwpp_run_bound_call issues it (host memory here): k_bound_table_rings_actions
// when actions is not NULL (act, scratch, dep, init and states as for simt_bound_table_actions), k_bound_table_rings otherwise.
// Frame f reads ring {bases[f], strides[f], ring_counts[f], num_slots[f]} with layouts[f]; slot receives the run's copy of
// slots, brun (nframes RecordFrames) the run's record table.
void simt_bound_table_rings(int nframes, const int64_t* max_n, const int32_t* b_stream, const int32_t* b_pset, int64_t* pt_off, int32_t* chunk_off,
                            int32_t* stream, int32_t* pset, int32_t* status, const int32_t* actions, int32_t* act, const int32_t* scratch,
                            const int32_t* dep, const void* init, void* states, const int32_t* slots, int32_t* slot, const void* const* bases,
                            const int64_t* const* ring_counts, const int64_t* strides, const int32_t* num_slots, const pwpp_point_layout* layouts,
                            void* brun) {
  std::vector<pwpp::RecordFrame> brec(nframes);
  std::vector<pwpp::BoundRing> ring(nframes);
  for (int f = 0; f < nframes; ++f) {
    brec[f] = pwpp::record_frame(layouts[f], bases[f]);
    ring[f] = pwpp::BoundRing{reinterpret_cast<const long long*>(ring_counts[f]), (long long) strides[f], num_slots[f], 0};
  }
  const pwpp::BoundRings G{slots, slot, ring.data(), brec.data(), static_cast<pwpp::RecordFrame*>(brun)};
  const auto mx = reinterpret_cast<const long long*>(max_n);
  const auto po = reinterpret_cast<long long*>(pt_off);
  if (actions) {
    const pwpp::BoundActions A{actions, act, scratch, dep, static_cast<const pwpp::StreamState*>(init), static_cast<pwpp::StreamState*>(states)};
    simt::launch("k_bound_table_rings_actions", dim3(1), pwpp::BT_THREADS, 0,
                 [&] { pwpp::k_bound_table_rings_actions(nframes, mx, b_stream, b_pset, po, chunk_off, stream, pset, status, A, G); });
  } else {
    simt::launch("k_bound_table_rings", dim3(1), pwpp::BT_THREADS, 0,
                 [&] { pwpp::k_bound_table_rings(nframes, mx, b_stream, b_pset, po, chunk_off, stream, pset, status, G); });
  }
}

// The bound call's unpack over the run's record table brun and point offsets pt_off (the table kernel's), with the grid sized
// from the capacities max_n as pwpp_run_bound_call sizes it. dst receives pt_off[nframes] float4 points.
void simt_unpack_run(int nframes, const void* brun, const int64_t* max_n, const int64_t* pt_off, float* dst) {
  const auto* recs = static_cast<const pwpp::RecordFrame*>(brun);
  std::vector<long long> cap(nframes + 1, 0);
  for (int f = 0; f < nframes; ++f) cap[f + 1] = cap[f] + max_n[f];
  if (cap[nframes] == 0) return;
  const long long gx = pwpp::rec_grid_x(cap.data(), recs, nframes);
  simt::launch("k_unpack_records", dim3((unsigned) gx, (unsigned) nframes), pwpp::REC_THREADS, 0, [&] {
    pwpp::k_unpack_records(recs, reinterpret_cast<const long long*>(pt_off), reinterpret_cast<float4*>(dst));
  });
}

// The bound call's part gather (both parts) over brun and pt_off, grid and regions from the capacities: idx the index lists
// (frame f's at pt_off[f]: ground, then non-ground), counts the count rows [3][nframes]; part_off receives the region offsets.
void simt_gather_parts_run(int nframes, const void* brun, const int64_t* max_n, const int64_t* pt_off, const int32_t* counts, const int32_t* idx,
                           unsigned char* ground, unsigned char* nonground, int64_t* part_off, int32_t* part_cnt) {
  const auto* recs = static_cast<const pwpp::RecordFrame*>(brun);
  std::vector<long long> cap(nframes + 1, 0), poff(nframes + 1);
  for (int f = 0; f < nframes; ++f) cap[f + 1] = cap[f] + max_n[f];
  pwpp::rec_out_offsets(cap.data(), recs, nframes, poff.data());
  for (int f = 0; f <= nframes; ++f) part_off[f] = poff[f];
  const long long gx = pwpp::rec_parts_grid_x(cap.data(), recs, nframes);
  simt::launch("k_gather_record_parts", dim3((unsigned) gx, (unsigned) nframes, 2u), pwpp::REC_THREADS, 0, [&] {
    pwpp::k_gather_record_parts(recs, reinterpret_cast<const long long*>(pt_off), counts, nframes, idx, poff.data(), 0, ground, nonground, part_cnt);
  });
}

}  // extern "C"
