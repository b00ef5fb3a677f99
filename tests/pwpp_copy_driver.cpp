// pwpp_copy_driver.cpp — TEST-ONLY: copies of the drop-in patchwork::PatchWorkpp (include/patchwork/patchworkpp.h), as reference
// code makes them (`PatchWorkpp b = a;`, `c = a;`). Usage: pwpp_copy_driver K scan0.bin scan1.bin ... (N x 4 float32 each).
// Instance a runs the first K scans; b is copy-constructed from it, c is a fresh instance that runs a scan of its own and is
// then copy-assigned from a, and a is assigned to itself. Each of a, b, c then runs the remaining scans. A never-run instance
// is copied too, and both run the first scan. Every getter is printed as "<instance> <tag> <digest>" lines: the test
// (tests/test_gpu_state_copy.py) requires equal lines for equal tags. Built by build.py against the real library, and compiled
// without linking in the CPU suite.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

#include "patchwork/patchworkpp.h"

namespace {

std::vector<float> load(const char* path) {
  std::ifstream f(path, std::ios::binary | std::ios::ate);
  std::vector<float> v((size_t) f.tellg() / sizeof(float));
  f.seekg(0);
  f.read(reinterpret_cast<char*>(v.data()), (std::streamsize) (v.size() * sizeof(float)));
  return v;
}

template <typename T>
uint64_t digest(const std::vector<T>& v) {   // FNV-1a over the bytes
  uint64_t h = 1469598103934665603ull;
  const unsigned char* p = reinterpret_cast<const unsigned char*>(v.data());
  for (size_t i = 0; i < v.size() * sizeof(T); ++i) h = (h ^ p[i]) * 1099511628211ull;
  return h ^ v.size();
}

void print(const char* who, const std::string& tag, patchwork::PatchWorkpp& pw) {
  double h = pw.getHeight();
  uint64_t hb;
  std::memcpy(&hb, &h, sizeof hb);
  std::printf("%s %s ground %016llx nonground %016llx gxyz %016llx ngxyz %016llx centers %016llx normals %016llx height %016llx\n", who, tag.c_str(),
              (unsigned long long) digest(pw.getGroundIndicesVec()), (unsigned long long) digest(pw.getNongroundIndicesVec()),
              (unsigned long long) digest(pw.getGroundVec()), (unsigned long long) digest(pw.getNongroundVec()),
              (unsigned long long) digest(pw.getCentersVec()), (unsigned long long) digest(pw.getNormalsVec()), (unsigned long long) hb);
}

void run(patchwork::PatchWorkpp& pw, const std::vector<float>& scan) { pw.estimateGround(scan.data(), (int64_t) (scan.size() / 4), 4, 4, 1); }

}  // namespace

int main(int argc, char** argv) {
  if (argc < 4) {
    std::fprintf(stderr, "usage: %s K scan0.bin scan1.bin ...\n", argv[0]);
    return 2;
  }
  const int k = std::atoi(argv[1]);
  std::vector<std::vector<float>> scans;
  for (int i = 2; i < argc; ++i) scans.push_back(load(argv[i]));
  if (k < 1 || k >= (int) scans.size()) {
    std::fprintf(stderr, "K must leave at least one scan after the first K\n");
    return 2;
  }
  patchwork::Params params;
  patchwork::PatchWorkpp a(params);
  for (int i = 0; i < k; ++i) run(a, scans[i]);
  patchwork::PatchWorkpp b = a;                   // copy construction
  patchwork::PatchWorkpp c(params);
  run(c, scans.back());
  c = a;                                          // copy assignment over an instance with a history of its own
  patchwork::PatchWorkpp& self = a;
  a = self;                                       // self-assignment: nothing happens
  print("a", "copied", a);
  print("b", "copied", b);
  print("c", "copied", c);
  for (int i = k; i < (int) scans.size(); ++i) {
    const std::string tag = "frame" + std::to_string(i);
    run(a, scans[i]);
    run(b, scans[i]);
    run(c, scans[i]);
    print("a", tag, a);
    print("b", tag, b);
    print("c", tag, c);
  }
  patchwork::PatchWorkpp fresh(params);
  patchwork::PatchWorkpp fresh_copy(fresh);       // a copy of a never-run instance: empty getters, same first frame
  std::printf("fresh empty %zu %zu\n", fresh_copy.getGroundIndicesVec().size(), fresh_copy.getCentersVec().size());
  run(fresh, scans[0]);
  run(fresh_copy, scans[0]);
  print("fresh", "first", fresh);
  print("fresh_copy", "first", fresh_copy);
  return 0;
}
