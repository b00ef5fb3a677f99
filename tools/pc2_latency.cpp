// pc2_latency.cpp — one-frame host latency of three ways to hand a KITTI scan laid out as a PointCloud2 message to the engine
// (tools/records_bench.py builds and runs it): usage `pc2_latency SCAN.bin LAYOUT REPS`, LAYOUT one of pcl_xyzi32, velodyne22,
// rec48. Prints one JSON line per (path, buffer) with the median and 10th percentile of the wall-clock time of
// estimateGround, in microseconds:
//   records   patchwork::estimateGround(pw, PointCloud2Message): the records go as they are and are unpacked on the GPU
//   view      patchwork::estimateGround(pw, PointCloud2View): these layouts take its host-side gather into N x 4 floats
//   packed    pw.estimateGround on an N x 4 float array packed in advance (no conversion in the timed call)
// buffer: pageable (std::vector) or page_locked (pwpp_host_alloc).
#include <patchwork/pointcloud2.hpp>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

template <typename F>
static void timed(const char* path, const char* buf, const char* layout, int reps, F&& call) {
  for (int i = 0; i < 20; ++i) call();
  std::vector<double> t(reps);
  for (int i = 0; i < reps; ++i) {
    const auto t0 = std::chrono::steady_clock::now();
    call();
    t[i] = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
  }
  std::sort(t.begin(), t.end());
  std::printf("{\"record\": \"host_latency\", \"layout\": \"%s\", \"path\": \"%s\", \"buffer\": \"%s\", \"median_us\": %.1f, \"p10_us\": %.1f, \"reps\": %d}\n", layout,
              path, buf, t[reps / 2], t[reps / 10], reps);
  std::fflush(stdout);
}

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<float> scan(4 * 200000);
  const size_t n = std::fread(scan.data(), 16, 200000, f);
  std::fclose(f);
  const std::string layout = argv[2];
  const int reps = std::atoi(argv[3]);
  uint32_t step = 0;
  int oi = 0;
  if (layout == "pcl_xyzi32") { step = 32; oi = 16; }
  else if (layout == "velodyne22") { step = 22; oi = 12; }
  else if (layout == "rec48") { step = 48; oi = 16; }
  else return 2;
  patchwork::Params params;
  params.verbose = false;
  patchwork::PatchWorkpp pw(params);
  for (int pinned = 0; pinned < 2; ++pinned) {
    const char* bufname = pinned ? "page_locked" : "pageable";
    std::vector<uint8_t> pageable;
    uint8_t* msg = nullptr;
    float* packed = nullptr;
    std::vector<float> packed_v;
    if (pinned) {
      msg = static_cast<uint8_t*>(pwpp_host_alloc(n * step));
      packed = static_cast<float*>(pwpp_host_alloc(n * 16));
    } else {
      pageable.resize(n * step);
      packed_v.resize(n * 4);
      msg = pageable.data();
      packed = packed_v.data();
    }
    std::memset(msg, 0xAB, n * step);
    for (size_t i = 0; i < n; ++i) {
      std::memcpy(msg + i * step, &scan[4 * i], 12);
      std::memcpy(msg + i * step + oi, &scan[4 * i + 3], 4);
    }
    std::memcpy(packed, scan.data(), n * 16);
    patchwork::PointCloud2Message m;
    m.data = msg; m.num_points = (int64_t) n; m.point_step = step;
    m.fields = {{"x", 0, PWPP_FIELD_FLOAT32, 1}, {"y", 4, PWPP_FIELD_FLOAT32, 1}, {"z", 8, PWPP_FIELD_FLOAT32, 1}, {"intensity", (uint32_t) oi, PWPP_FIELD_FLOAT32, 1}};
    patchwork::PointCloud2View v;
    v.data = msg; v.num_points = (int64_t) n; v.point_step = step; v.off_x = 0; v.off_y = 4; v.off_z = 8; v.off_intensity = oi;
    // alternate the three paths in rounds so that clock or load drift spreads over all of them
    for (int round = 0; round < 3; ++round) {
      timed("records", bufname, layout.c_str(), reps, [&] { patchwork::estimateGround(pw, m); });
      timed("view", bufname, layout.c_str(), reps, [&] { patchwork::estimateGround(pw, v); });
      timed("packed", bufname, layout.c_str(), reps, [&] { pw.estimateGround(packed, (int64_t) n, 4, 4, 1); });
    }
    if (pinned) { pwpp_host_free(msg); pwpp_host_free(packed); }
  }
  return 0;
}
