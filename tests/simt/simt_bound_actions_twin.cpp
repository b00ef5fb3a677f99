// simt_bound_actions_twin.cpp — TEST-ONLY: the SIMT twin with a stream table (simt_streams.cpp, included whole) driven the way a
// bound call with per-frame actions runs one run: k_bound_table_actions first, then the launch sequence with the stream table
// and frame sizes the table kernel wrote (tests/test_simt_bound_actions_oracle.py).
#include "simt_streams.cpp"

#include "pwpp_records.cuh"

extern "C" {

// One run of a bound call with actions over nframes frames of pairwise distinct streams: k_bound_table_actions with counts =
// capacities = ns[f] (a frame with a count runs it), scratch[f] the frame's scratch slot (a stream id of the twin past the real
// ones), no frame depending on an earlier run. The table kernel applies the RESETs and redirects the skipped frames; the twin's
// launch sequence then runs every frame with the stream table and sizes it wrote. status receives the table kernel's status.
int simt_bound_actions_run(void* h, int nframes, const int* streams, const int* actions, const int* scratch, const float* const* pts,
                           const int64_t* ns, int cols, int* status) {
  SimtTwin* t = (SimtTwin*) h;
  std::vector<StreamState> init(t->num_streams);
  for (auto& s : init) init_state(t->prm, s);
  std::vector<int> sets(nframes, 0), dep(nframes, 0), act(nframes), stream(nframes), pset(nframes), chunk_off(nframes + 1);
  std::vector<long long> counts(ns, ns + nframes), pt_off(nframes + 1);
  const BoundActions A{actions, act.data(), scratch, dep.data(), init.data(), t->states.data()};
  simt::launch("k_bound_table_actions", dim3(1), BT_THREADS, 0, [&] {
    k_bound_table_actions(nframes, counts.data(), counts.data(), streams, sets.data(), pt_off.data(), chunk_off.data(), stream.data(),
                          pset.data(), status, A);
  });
  std::vector<int64_t> n(nframes);
  for (int f = 0; f < nframes; ++f) n[f] = pt_off[f + 1] - pt_off[f];
  return simt_estimate_streams(h, nframes, stream.data(), pts, n.data(), cols);
}

}  // extern "C"
