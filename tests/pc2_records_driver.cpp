// TEST-ONLY driver for the records path of include/patchwork/pointcloud2.hpp (tests/test_gpu_records.py): reads a scan (float32
// x,y,z,i records), lays it out as PointCloud2 messages of several layouts (described by name / offset / datatype / count, as
// sensor_msgs::msg::PointCloud2 does), runs each through patchwork::estimateGround(pw, message) with default parameters (RNR on)
// and prints "layout ground nonground ground_checksum nonground_ordered_checksum".
#include <patchwork/pointcloud2.hpp>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<float> scan(4 * 200000);
  const size_t n = std::fread(scan.data(), 16, 200000, f);
  std::fclose(f);
  struct Layout { const char* name; uint32_t step; int ox, oy, oz, oi; uint8_t ti; };
  const Layout layouts[] = {
      {"xyz12", 12, 0, 4, 8, -1, 0},
      {"xyzi16", 16, 0, 4, 8, 12, PWPP_FIELD_FLOAT32},
      {"pcl_xyzi32", 32, 0, 4, 8, 16, PWPP_FIELD_FLOAT32},
      {"velodyne22", 22, 0, 4, 8, 12, PWPP_FIELD_FLOAT32},
      {"ouster48_noint", 48, 16, 20, 24, -1, 0},
      {"xyzi13_u8", 13, 0, 4, 8, 12, PWPP_FIELD_UINT8},   // intensity as UINT8: floor(255 * i), clamped to [0, 255]
  };
  patchwork::Params params;
  params.verbose = false;
  for (const Layout& L : layouts) {
    std::vector<uint8_t> msg((size_t) n * L.step, 0xAB);
    for (size_t i = 0; i < n; ++i) {
      uint8_t* p = msg.data() + i * L.step;
      std::memcpy(p + L.ox, &scan[4 * i], 4); std::memcpy(p + L.oy, &scan[4 * i + 1], 4); std::memcpy(p + L.oz, &scan[4 * i + 2], 4);
      if (L.ti == PWPP_FIELD_FLOAT32) std::memcpy(p + L.oi, &scan[4 * i + 3], 4);
      if (L.ti == PWPP_FIELD_UINT8) p[L.oi] = (uint8_t) std::min(255.f, std::max(0.f, std::floor(scan[4 * i + 3] * 255.f)));
    }
    patchwork::PointCloud2Message m;
    m.data = msg.data(); m.num_points = (int64_t) n; m.point_step = L.step;
    m.fields = {{"x", (uint32_t) L.ox, PWPP_FIELD_FLOAT32, 1}, {"y", (uint32_t) L.oy, PWPP_FIELD_FLOAT32, 1}, {"z", (uint32_t) L.oz, PWPP_FIELD_FLOAT32, 1}};
    if (L.oi >= 0) m.fields.push_back({"intensity", (uint32_t) L.oi, L.ti, 1});
    m.fields.push_back({"ring", 0, PWPP_FIELD_UINT16, 1});   // other fields are ignored
    patchwork::PatchWorkpp pw(params);
    patchwork::estimateGround(pw, m);
    long long cg = 0, cn = 0;
    for (int v : pw.getGroundIndicesVec()) cg += (long long) v * (long long) (v % 97 + 1);
    const std::vector<int> ng = pw.getNongroundIndicesVec();
    for (size_t k = 0; k < ng.size(); ++k) cn = (cn * 1000003 + ng[k]) % 1000000007;   // order-dependent
    std::printf("%s %zu %zu %lld %lld\n", L.name, pw.getGroundIndicesVec().size(), ng.size(), cg, cn);
  }
  // a message the function must refuse
  patchwork::PointCloud2Message bad;
  bad.point_step = 16; bad.is_bigendian = true;
  try { patchwork::pointLayout(bad); std::printf("bigendian accepted\n"); } catch (const std::invalid_argument&) { std::printf("bigendian refused\n"); }
  bad.is_bigendian = false;
  bad.fields = {{"x", 0, PWPP_FIELD_FLOAT32, 1}, {"y", 4, PWPP_FIELD_FLOAT32, 1}, {"z", 8, PWPP_FIELD_FLOAT32, 2}};
  try { patchwork::pointLayout(bad); std::printf("count2 accepted\n"); } catch (const std::invalid_argument&) { std::printf("count2 refused\n"); }
  bad.fields.pop_back();
  try { patchwork::pointLayout(bad); std::printf("noz accepted\n"); } catch (const std::invalid_argument&) { std::printf("noz refused\n"); }
  return 0;
}
