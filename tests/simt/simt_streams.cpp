// simt_streams.cpp — TEST-ONLY: the SIMT twin (simt_twin.cpp, included whole) plus one entry point that runs its launch
// sequence with a stream table other than the identity: frame f of the call advances stream streams[f] of the twin's state
// array. tests/test_simt_stream_map.py compares every stream with its own oracle. Built with plain g++ like the twin.
#include "simt_twin.cpp"

extern "C" {

// One launch sequence, as one run of pwpp_estimate_host_streams: the streams must be pairwise distinct ids of the twin
// (returns -1 otherwise, nothing run). Per-frame outputs are indexed by call position, state by stream id (simt_select
// picks either).
int simt_estimate_streams(void* h, int nframes, const int* streams, const float* const* pts, const int64_t* ns, int cols) {
  SimtTwin* t = (SimtTwin*) h;
  std::vector<char> used(t->num_streams, 0);
  for (int f = 0; f < nframes; ++f) {
    if (streams[f] < 0 || streams[f] >= t->num_streams || used[streams[f]]) return -1;
    used[streams[f]] = 1;
  }
  pwpp::g_simt_streams = streams;   // read by the FrameTable of the launch sequence
  simt_estimate_multi(h, nframes, pts, ns, cols);
  pwpp::g_simt_streams = pwpp::simt_identity_streams();
  return 0;
}

}  // extern "C"
