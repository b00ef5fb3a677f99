// pwpp_sequence — runs a directory of KITTI-format scans (raw float32 x,y,z,intensity records, one file per frame)
// through ONE sensor stream of the H100 engine, in file-name order, like the reference's
// cpp/patchworkpp/examples/demo_sequential.cpp:53-79 (construct once, then per frame estimateGround + getters) minus the
// Open3D window. The step before the hot path (SURVEY.md 8f-2): a reader thread loads frame t+1 into the second of two
// page-locked buffers (pwpp_host_alloc) while the GPU works on frame t, so the H2D copy of a frame never waits for the
// disk and needs no staging copy. Frames of one stream are sequentially dependent (adaptive thresholds, S:338-375),
// so the pipeline depth is one frame.
//
//   pwpp_sequence DIR [--device N] [--repeat R] [--quiet]
// Prints per frame: points, ground, non-ground, patches, adaptive sensor height, call time; then frames/s end to end.
//
//   pwpp_sequence DIR [DIR ...] [--frames-per-call K] [--device N] [--repeat R] [--quiet]
// Several sensors (or one sensor in batches): every directory is one stream of one context, and every call of
// pwpp_estimate_host_streams carries the next K scans (default 1) of every directory that still has scans, time-major
// (dir 0 scan t, dir 1 scan t, ..., dir 0 scan t+1, ...). Directories may hold different numbers of scans: a stream
// that ran out is simply not named any more. Each line is prefixed with the stream (directory) index; the height is the
// stream's adaptive sensor height after that frame, "-" where the stream has a later frame in the same call (the state
// between two frames of one call is not kept).
#include <patchwork/patchworkpp.h>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <dirent.h>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

// The several-streams form calls pwpp_estimate_host_streams. The reference to it is weak, so the runner still links, and its
// one-directory form still runs, against a C-ABI library that predates the stream table; the several-streams form then
// says so and exits with 1.
#pragma weak pwpp_estimate_host_streams

namespace {
struct Slot {
  float* data = nullptr;   // page-locked, capacity `cap` floats
  size_t cap = 0;
  int64_t n = 0;           // points loaded
  int frame = -1;          // which file is in it (-1: free)
  std::string name;
};

std::vector<std::string> list_scans(const std::string& dir) {
  std::vector<std::string> v;
  if (DIR* d = opendir(dir.c_str())) {
    while (dirent* e = readdir(d)) {
      const std::string n = e->d_name;
      if (n.size() > 4 && n.substr(n.size() - 4) == ".bin") v.push_back(n);
    }
    closedir(d);
  }
  std::sort(v.begin(), v.end());
  return v;
}

// whole file -> slot (grows the pinned buffer when a scan is larger than anything seen so far)
bool load(const std::string& path, Slot& s) {
  FILE* f = std::fopen(path.c_str(), "rb");
  if (!f) return false;
  std::fseek(f, 0, SEEK_END);
  const long bytes = std::ftell(f);
  std::fseek(f, 0, SEEK_SET);
  const size_t floats = (size_t) bytes / sizeof(float);
  if (floats > s.cap) {
    if (s.data) pwpp_host_free(s.data);
    s.cap = floats + floats / 4;
    s.data = static_cast<float*>(pwpp_host_alloc(s.cap * sizeof(float)));
    if (!s.data) { std::fclose(f); s.cap = 0; return false; }
  }
  const size_t got = std::fread(s.data, sizeof(float), floats, f);
  std::fclose(f);
  s.n = (int64_t) (got / 4);
  return true;
}

// Several directories, one stream each, K scans of every stream per call (see the header comment).
int run_streams(const std::vector<std::string>& dirs, int frames_per_call, int device, int repeat, bool quiet) {
  if (!&pwpp_estimate_host_streams) {
    std::fprintf(stderr, "pwpp_sequence: this libpwpp_b200 has no pwpp_estimate_host_streams (stream table): several directories or "
                         "--frames-per-call need a newer library\n");
    return 1;
  }
  const int ns = (int) dirs.size();
  std::vector<std::vector<std::string>> files(ns);
  size_t longest = 0;
  for (int d = 0; d < ns; ++d) {
    const std::vector<std::string> once = list_scans(dirs[d]);
    if (once.empty()) { std::fprintf(stderr, "no *.bin scans in %s\n", dirs[d].c_str()); return 2; }
    for (int r = 0; r < repeat; ++r) files[d].insert(files[d].end(), once.begin(), once.end());
    longest = std::max(longest, files[d].size());
  }
  pwpp_params params;
  pwpp_params_default(&params);   // reference defaults (patchworkpp.h:79-111)
  pwpp_ctx* ctx = nullptr;
  if (pwpp_create(&params, device, ns, 0, &ctx) != PWPP_OK) { std::fprintf(stderr, "pwpp_sequence: %s\n", pwpp_last_error()); return 1; }
  pwpp_set_output_order(ctx, PWPP_ORDER_REFERENCE);   // the order of the single-directory run (the drop-in class)
  std::vector<Slot> slots;            // one page-locked buffer per frame position of a call
  std::vector<int32_t> streams;
  std::vector<const float*> ptrs;
  std::vector<int64_t> counts;
  std::vector<int> last_of(ns);
  const auto t0 = std::chrono::steady_clock::now();
  long long points = 0;
  int done = 0, calls = 0, rc = 0;
  for (size_t t0_scan = 0; t0_scan < longest && rc == 0; t0_scan += (size_t) frames_per_call) {
    streams.clear(); ptrs.clear(); counts.clear();
    for (size_t t = t0_scan; t < std::min(longest, t0_scan + (size_t) frames_per_call) && rc == 0; ++t)
      for (int d = 0; d < ns; ++d) {
        if (t >= files[d].size()) continue;
        const size_t f = streams.size();
        if (slots.size() <= f) slots.resize(f + 1);
        Slot& s = slots[f];
        s.name = files[d][t];
        if (!load(dirs[d] + "/" + s.name, s)) { std::fprintf(stderr, "failed to read %s\n", s.name.c_str()); rc = 1; break; }
        streams.push_back(d);
        ptrs.push_back(s.data);
        counts.push_back(s.n);
        last_of[d] = (int) f;
      }
    if (rc || streams.empty()) break;
    const int nf = (int) streams.size();
    if (pwpp_estimate_host_streams(ctx, nf, streams.data(), ptrs.data(), counts.data(), 4, 4, 1) != PWPP_OK) {
      std::fprintf(stderr, "pwpp_sequence: %s\n", pwpp_last_error());
      rc = 1;
      break;
    }
    ++calls;
    for (int f = 0; f < nf && !quiet; ++f) {
      const int d = streams[f];
      char height[32] = "-";
      if (last_of[d] == f) std::snprintf(height, sizeof height, "%.4f", pwpp_height(ctx, d));
      std::printf("%-3d %-14s points %7lld  ground %7lld  nonground %7lld  patches %4d  height %s  call %.3f ms\n", d, slots[f].name.c_str(),
                  (long long) counts[f], (long long) pwpp_num_ground(ctx, f), (long long) pwpp_num_nonground(ctx, f), pwpp_num_patches(ctx, f), height,
                  pwpp_time_us(ctx) / 1000.0);
    }
    for (int f = 0; f < nf; ++f) points += counts[f];
    done += nf;
  }
  const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  std::printf("%d frames of %d streams in %d calls, %lld points in %.3f s: %.1f frames/s end to end (disk -> pinned -> GPU -> counts)\n", done, ns, calls,
              points, sec, done / sec);
  for (Slot& s : slots) if (s.data) pwpp_host_free(s.data);
  pwpp_destroy(ctx);
  return rc;
}
}  // namespace

int main(int argc, char** argv) {
  if (argc < 2) { std::fprintf(stderr, "usage: %s DIR [DIR ...] [--frames-per-call K] [--device N] [--repeat R] [--quiet]\n", argv[0]); return 2; }
  std::vector<std::string> dirs{argv[1]};
  int device = 0, repeat = 1, frames_per_call = 0;
  bool quiet = false;
  for (int i = 2; i < argc; ++i) {
    if (!std::strcmp(argv[i], "--device") && i + 1 < argc) device = std::atoi(argv[++i]);
    else if (!std::strcmp(argv[i], "--repeat") && i + 1 < argc) repeat = std::atoi(argv[++i]);
    else if (!std::strcmp(argv[i], "--frames-per-call") && i + 1 < argc) frames_per_call = std::atoi(argv[++i]);
    else if (!std::strcmp(argv[i], "--quiet")) quiet = true;
    else if (std::strncmp(argv[i], "--", 2) != 0) dirs.push_back(argv[i]);
  }
  if (dirs.size() > 1 || frames_per_call > 0) return run_streams(dirs, std::max(1, frames_per_call), device, std::max(1, repeat), quiet);
  const std::string dir = dirs[0];
  const std::vector<std::string> files = list_scans(dir);
  if (files.empty()) { std::fprintf(stderr, "no *.bin scans in %s\n", dir.c_str()); return 2; }
  const int total = (int) files.size() * repeat;

  patchwork::Params params;   // reference defaults (patchworkpp.h:79-111)
  params.verbose = false;
  try {
    patchwork::PatchWorkpp pw(params, device);

    Slot slot[2];
    std::mutex mu;
    std::condition_variable cv;
    bool failed = false;
    // reader: fills slot[t & 1] with frame t as soon as the consumer has released it
    std::thread reader([&] {
      for (int t = 0; t < total; ++t) {
        Slot& s = slot[t & 1];
        { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return s.frame < 0; }); }
        const std::string& name = files[(size_t) t % files.size()];
        const bool ok = load(dir + "/" + name, s);
        { std::lock_guard<std::mutex> lk(mu); s.name = name; s.frame = ok ? t : -2; failed |= !ok; }
        cv.notify_all();
        if (!ok) return;
      }
    });

    const auto t0 = std::chrono::steady_clock::now();
    long long points = 0;
    int done = 0;
    // releases both slots and joins the reader on every way out of the loop (an exception from estimateGround or a getter
    // would otherwise destroy a joinable std::thread -> std::terminate, with the reader possibly blocked on cv)
    struct ReaderGuard {
      std::thread& th; std::mutex& mu; std::condition_variable& cv; Slot* slot;
      ~ReaderGuard() {
        { std::lock_guard<std::mutex> lk(mu); for (int i = 0; i < 2; ++i) if (slot[i].frame != -1) slot[i].frame = -1; }
        cv.notify_all();
        if (th.joinable()) th.join();
      }
    } guard{reader, mu, cv, slot};
    for (int t = 0; t < total; ++t) {
      Slot& s = slot[t & 1];
      { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return s.frame == t || s.frame == -2; }); }
      if (s.frame == -2) { std::fprintf(stderr, "failed to read %s\n", s.name.c_str()); break; }
      pw.estimateGround(s.data, s.n, 4, 4, 1);                     // reference :152 (row-major N x 4, straight from the pinned buffer)
      const std::vector<int> ground = pw.getGroundIndicesVec();    // :159
      const std::vector<int> nonground = pw.getNongroundIndicesVec();
      const std::vector<float> centers = pw.getCentersVec();       // :162
      if (!quiet)
        std::printf("%-14s points %7lld  ground %7zu  nonground %7zu  patches %4zu  height %.4f  time %.3f ms\n", s.name.c_str(), (long long) s.n,
                    ground.size(), nonground.size(), centers.size() / 3, pw.getHeight(), pw.getTimeTaken() / 1000.0);
      points += s.n;
      ++done;
      { std::lock_guard<std::mutex> lk(mu); s.frame = -1; }
      cv.notify_all();
    }
    const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    { std::lock_guard<std::mutex> lk(mu); for (Slot& s : slot) if (s.frame >= 0) s.frame = -1; }
    cv.notify_all();
    reader.join();
    std::printf("%d frames, %lld points in %.3f s: %.1f frames/s end to end (disk -> pinned -> GPU -> index lists)\n", done, points, sec, done / sec);
    for (Slot& s : slot) if (s.data) pwpp_host_free(s.data);
    return failed ? 1 : 0;
  } catch (const std::exception& e) {
    std::fprintf(stderr, "pwpp_sequence: %s\n", e.what());
    return 1;
  }
}
