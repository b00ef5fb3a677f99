// pc2_records_out_latency.cpp — one-frame host latency of the ROS pattern with and without the input's fields in the output
// (tools/records_out_bench.py builds and runs it): usage `pc2_records_out_latency SCAN.bin LAYOUT REPS`, LAYOUT pcl_xyzi32 or
// velodyne22. Prints one JSON line per (output, buffer) with the median and 10th percentile of the wall-clock time, in
// microseconds, of
//   records   estimateGround(pw, message) + makeRecordsPayload for ground and non-ground (whole input records, gathered on the GPU)
//   xyz       estimateGround(pw, message) + makeCloudPayload for ground and non-ground (packed x/y/z, the reference node's output)
// buffer: pageable (std::vector) or page_locked (pwpp_host_alloc).
#include <patchwork/pointcloud2.hpp>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

template <typename F>
static void timed(const char* out, const char* buf, const char* layout, int reps, F&& call) {
  for (int i = 0; i < 20; ++i) call();
  std::vector<double> t(reps);
  for (int i = 0; i < reps; ++i) {
    const auto t0 = std::chrono::steady_clock::now();
    call();
    t[i] = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
  }
  std::sort(t.begin(), t.end());
  std::printf("{\"record\": \"ros_latency\", \"layout\": \"%s\", \"output\": \"%s\", \"buffer\": \"%s\", \"median_us\": %.1f, \"p10_us\": %.1f, \"reps\": %d}\n",
              layout, out, buf, t[reps / 2], t[reps / 10], reps);
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
  else return 2;
  patchwork::Params params;
  params.verbose = false;
  patchwork::PatchWorkpp pw(params);
  size_t sink = 0;
  for (int pinned = 0; pinned < 2; ++pinned) {
    const char* bufname = pinned ? "page_locked" : "pageable";
    std::vector<uint8_t> pageable;
    uint8_t* msg = nullptr;
    if (pinned) {
      msg = static_cast<uint8_t*>(pwpp_host_alloc(n * step));
    } else {
      pageable.resize(n * step);
      msg = pageable.data();
    }
    std::memset(msg, 0xAB, n * step);
    for (size_t i = 0; i < n; ++i) {
      std::memcpy(msg + i * step, &scan[4 * i], 12);
      std::memcpy(msg + i * step + oi, &scan[4 * i + 3], 4);
    }
    patchwork::PointCloud2Message m;
    m.data = msg; m.num_points = (int64_t) n; m.point_step = step;
    m.fields = {{"x", 0, PWPP_FIELD_FLOAT32, 1}, {"y", 4, PWPP_FIELD_FLOAT32, 1}, {"z", 8, PWPP_FIELD_FLOAT32, 1}, {"intensity", (uint32_t) oi, PWPP_FIELD_FLOAT32, 1}};
    // alternate the two outputs in rounds so that clock or load drift spreads over both
    for (int round = 0; round < 3; ++round) {
      timed("records", bufname, layout.c_str(), reps, [&] {
        patchwork::estimateGround(pw, m);
        sink += patchwork::makeRecordsPayload(pw, true, m).data.size() + patchwork::makeRecordsPayload(pw, false, m).data.size();
      });
      timed("xyz", bufname, layout.c_str(), reps, [&] {
        patchwork::estimateGround(pw, m);
        sink += patchwork::makeCloudPayload(pw, true).data.size() + patchwork::makeCloudPayload(pw, false).data.size();
      });
    }
    if (pinned) pwpp_host_free(msg);
  }
  return sink == 0 ? 1 : 0;
}
