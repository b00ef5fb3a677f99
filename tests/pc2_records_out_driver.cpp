// TEST-ONLY driver for makeRecordsPayload (include/patchwork/pointcloud2.hpp) against the real engine (tests/test_gpu_records_out.py):
// reads a scan (float32 x,y,z,i records), lays it out as PointCloud2 messages of three layouts with pseudo-random filler bytes,
// runs estimateGround(pw, message) and makeRecordsPayload for ground and non-ground, and checks every payload against the input
// records at the index lists, byte for byte, and its header fields against the input's. Prints "layout ok ground nonground" or
// "layout MISMATCH <what>", then "float call refused" when the record getters throw after a call that did not take records.
#include <patchwork/pointcloud2.hpp>

#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

static bool same_payload(const patchwork::PointCloud2RecordsPayload& p, const patchwork::PointCloud2Message& m, const std::vector<int>& idx,
                         std::string* what) {
  if (p.point_step != m.point_step || p.height != 1 || p.width != idx.size() || p.row_step != p.width * m.point_step || p.fields.size() != m.fields.size()) {
    *what = "header";
    return false;
  }
  for (size_t k = 0; k < m.fields.size(); ++k)
    if (p.fields[k].name != m.fields[k].name || p.fields[k].offset != m.fields[k].offset || p.fields[k].datatype != m.fields[k].datatype) { *what = "fields"; return false; }
  if (p.data.size() != idx.size() * m.point_step) { *what = "size"; return false; }
  for (size_t k = 0; k < idx.size(); ++k)
    if (std::memcmp(p.data.data() + k * m.point_step, m.data + (size_t) idx[k] * m.point_step, m.point_step) != 0) { *what = "record " + std::to_string(k); return false; }
  return true;
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<float> scan(4 * 200000);
  const size_t n = std::fread(scan.data(), 16, 200000, f);
  std::fclose(f);
  struct Layout { const char* name; uint32_t step; int oi; };
  const Layout layouts[] = {{"velodyne22", 22, 12}, {"pcl_xyzi32", 32, 16}, {"xyz12", 12, -1}};
  patchwork::Params params;
  params.verbose = false;
  patchwork::PatchWorkpp pw(params);
  unsigned state = 12345u;
  for (const Layout& L : layouts) {
    std::vector<uint8_t> msg((size_t) n * L.step);
    for (auto& b : msg) { state = state * 1664525u + 1013904223u; b = (uint8_t) (state >> 24); }
    for (size_t i = 0; i < n; ++i) {
      std::memcpy(msg.data() + i * L.step, &scan[4 * i], 12);
      if (L.oi >= 0) std::memcpy(msg.data() + i * L.step + L.oi, &scan[4 * i + 3], 4);
    }
    patchwork::PointCloud2Message m;
    m.data = msg.data(); m.num_points = (int64_t) n; m.point_step = L.step;
    m.fields = {{"x", 0, PWPP_FIELD_FLOAT32, 1}, {"y", 4, PWPP_FIELD_FLOAT32, 1}, {"z", 8, PWPP_FIELD_FLOAT32, 1}};
    if (L.oi >= 0) m.fields.push_back({"intensity", (uint32_t) L.oi, PWPP_FIELD_FLOAT32, 1});
    if (L.step == 22) { m.fields.push_back({"ring", 16, PWPP_FIELD_UINT16, 1}); m.fields.push_back({"time", 18, PWPP_FIELD_FLOAT32, 1}); }
    patchwork::estimateGround(pw, m);
    const patchwork::PointCloud2RecordsPayload g = patchwork::makeRecordsPayload(pw, true, m);
    const patchwork::PointCloud2RecordsPayload ng = patchwork::makeRecordsPayload(pw, false, m);
    const patchwork::PointCloud2Payload xyz = patchwork::makeCloudPayload(pw, true);   // unchanged beside it
    std::string what;
    const std::vector<int> gi = pw.getGroundIndicesVec(), ni = pw.getNongroundIndicesVec();
    if (!same_payload(g, m, gi, &what)) std::printf("%s MISMATCH ground %s\n", L.name, what.c_str());
    else if (!same_payload(ng, m, ni, &what)) std::printf("%s MISMATCH nonground %s\n", L.name, what.c_str());
    else if (xyz.width != gi.size()) std::printf("%s MISMATCH xyz payload\n", L.name);
    else std::printf("%s ok %zu %zu\n", L.name, gi.size(), ni.size());
  }
  pw.estimateGround(scan.data(), (int64_t) n, 4, 4, 1);
  try { pw.getGroundRecords(); std::printf("float call accepted\n"); } catch (const std::runtime_error&) { std::printf("float call refused\n"); }
  return 0;
}
