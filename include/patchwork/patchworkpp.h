// patchwork/patchworkpp.h — drop-in C++ surface of the H100 engine.
//
// Same header path, namespace, type names, member names, defaults and call sequence as the reference's
// cpp/patchworkpp/include/patchwork/patchworkpp.h (struct Params :42-112, class PatchWorkpp :114-163), so a
// caller such as the reference's demos (examples/demo_visualize.cpp:70-93, demo_sequential.cpp:53-79) or
// its ROS2 node (ros/src/GroundSegmentationServer.cpp:50,74-83) compiles against this header unchanged.
// It is header-only glue over the C-ABI in pwpp.h: the per-frame work happens in libpwpp_b200.so on the GPU.
//
// Differences, all at the edges:
//  * Eigen is optional. With <Eigen/Dense> on the include path the Eigen signatures of the reference
//    (estimateGround(Eigen::MatrixXf), Eigen::MatrixX3f / Eigen::VectorXi getters) are provided verbatim;
//    pointer/std::vector overloads are always available (the build container has no Eigen).
//  * Errors that the reference cannot have (no CUDA device, CUDA failure, unsupported parameter values such
//    as num_zones != 4) are thrown as std::runtime_error carrying pwpp_last_error().
//  * Output order inside one polar bin is ascending point index (reference: ascending z with
//    implementation-defined ties); the order of bins follows the reference's emission order.
#ifndef PATCHWORKPP_H
#define PATCHWORKPP_H

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

#include <cstdint>
#include <iostream>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#if defined(__has_include)
#if __has_include(<Eigen/Dense>)
#include <Eigen/Dense>
#define PATCHWORKPP_HAVE_EIGEN 1
#endif
#endif

#include "pwpp.h"

namespace patchwork {

// reference patchworkpp.h:42-112 — identical field names and defaults
struct Params {
  bool verbose = false;
  bool enable_RNR = true;
  bool enable_RVPF = true;
  bool enable_TGR = true;

  int num_iter = 3;               // iterations of the region-wise plane fit
  int num_lpr = 20;               // lowest-point-representative sample size
  int num_min_pts = 10;           // patches with fewer points are non-ground
  int num_zones = 4;              // concentric zone model; must stay 4
  int num_rings_of_interest = 4;  // rings checked for elevation / flatness

  double RNR_ver_angle_thr = -15.0;
  double RNR_intensity_thr = 0.2;

  double sensor_height = 1.723;
  double th_seeds = 0.125;
  double th_dist = 0.125;
  double th_seeds_v = 0.25;
  double th_dist_v = 0.1;
  double max_range = 80.0;
  double min_range = 2.7;
  double uprightness_thr = 0.707;
  double adaptive_seed_selection_margin = -1.2;
  double intensity_thr = 0.0;     // bound in the reference's Python module, never read by the algorithm

  std::vector<int> num_sectors_each_zone{16, 32, 54, 32};
  std::vector<int> num_rings_each_zone{2, 4, 4, 4};

  int max_flatness_storage = 1000;
  int max_elevation_storage = 1000;

  std::vector<double> elevation_thr{0, 0, 0, 0};
  std::vector<double> flatness_thr{0, 0, 0, 0};
};

// order inside a bin of the index lists (PatchWorkpp::setOutputOrder; the values are pwpp.h's PWPP_ORDER_*)
enum class OutputOrder : int { Bin = PWPP_ORDER_BIN, Reference = PWPP_ORDER_REFERENCE, ReferenceExact = PWPP_ORDER_REFERENCE_EXACT };
// arithmetic of the plane fits and of A-GLE (PatchWorkpp::setArithmetic; the values are pwpp.h's PWPP_ARITH_*)
enum class Arithmetic : int { Double = PWPP_ARITH_DOUBLE, Reference = PWPP_ARITH_REFERENCE };

class PatchWorkpp {
 public:
  // reference :120-150. `device` selects the CUDA device (extension; defaults to 0).
  PatchWorkpp(patchwork::Params _params, int device = 0) : params_(_params) {
    pwpp_params p;
    pwpp_params_default(&p);
    p.verbose = params_.verbose; p.enable_RNR = params_.enable_RNR; p.enable_RVPF = params_.enable_RVPF; p.enable_TGR = params_.enable_TGR;
    p.num_iter = params_.num_iter; p.num_lpr = params_.num_lpr; p.num_min_pts = params_.num_min_pts; p.num_zones = params_.num_zones;
    p.num_rings_of_interest = params_.num_rings_of_interest;
    p.RNR_ver_angle_thr = params_.RNR_ver_angle_thr; p.RNR_intensity_thr = params_.RNR_intensity_thr;
    p.sensor_height = params_.sensor_height; p.th_seeds = params_.th_seeds; p.th_dist = params_.th_dist;
    p.th_seeds_v = params_.th_seeds_v; p.th_dist_v = params_.th_dist_v; p.max_range = params_.max_range; p.min_range = params_.min_range;
    p.uprightness_thr = params_.uprightness_thr; p.adaptive_seed_selection_margin = params_.adaptive_seed_selection_margin;
    p.intensity_thr = params_.intensity_thr;
    p.max_flatness_storage = params_.max_flatness_storage; p.max_elevation_storage = params_.max_elevation_storage;
    for (int k = 0; k < 4; ++k) {
      // .at(): std::out_of_range for short vectors, like the reference constructor (:127-134)
      p.num_sectors_each_zone[k] = params_.num_sectors_each_zone.at(k);
      p.num_rings_each_zone[k] = params_.num_rings_each_zone.at(k);
      p.elevation_thr[k] = k < (int) params_.elevation_thr.size() ? params_.elevation_thr[k] : 0.0;
      p.flatness_thr[k] = k < (int) params_.flatness_thr.size() ? params_.flatness_thr[k] : 0.0;
    }
    if (pwpp_create(&p, device, 1, 0, &ctx_) != PWPP_OK) throw std::runtime_error(std::string("PatchWorkpp: ") + pwpp_last_error());
    pwpp_set_output_order(ctx_, PWPP_ORDER_REFERENCE);   // the drop-in class emits the reference's order (stable per-bin z sort)
    std::cout << "PatchWorkpp::PatchWorkpp() - INITIALIZATION COMPLETE" << std::endl;  // reference :149
  }
  ~PatchWorkpp() { if (ctx_) pwpp_destroy(ctx_); }
  // Copies, like the reference's implicit ones (its members are values): the copy gets the parameters, the adaptive state
  // (sensor height, thresholds, both histories, the plane carried for a no-plane patch) and the last frame's results, on a
  // ctx of its own on the same device (pwpp_clone), and prints no banner. Both then continue identically. The last call's
  // records are not carried: getGroundRecords() / getNongroundRecords() on the copy throw until it takes records itself.
  PatchWorkpp(const PatchWorkpp& o) : params_(o.params_), n_(o.n_), ran_(o.ran_), step_(o.step_) {
    if (o.ctx_) check(pwpp_clone(o.ctx_, -1, &ctx_));
  }
  // builds the copy first, so a failure leaves *this as it was
  PatchWorkpp& operator=(const PatchWorkpp& o) {
    if (this != &o) {
      PatchWorkpp copy(o);
      std::swap(params_, copy.params_);
      std::swap(ctx_, copy.ctx_);
      std::swap(n_, copy.n_);
      std::swap(ran_, copy.ran_);
      std::swap(step_, copy.step_);
    }
    return *this;
  }
  PatchWorkpp(PatchWorkpp&& o) noexcept : params_(o.params_), ctx_(o.ctx_), n_(o.n_), ran_(o.ran_), step_(o.step_) { o.ctx_ = nullptr; }

  // reference :152 for raw buffers: element (i,c) of the N x cols cloud is data[i*row_stride + c*col_stride].
  void estimateGround(const float* data, int64_t n, int cols, int64_t row_stride, int64_t col_stride) {
    if (cols < 3) throw std::runtime_error("PatchWorkpp::estimateGround: need at least x,y,z columns");
    if (cols < 4 && params_.enable_RNR) std::cout << "RNR requires intensity information !" << std::endl;  // reference src :380
    const float* ptrs[1] = {data};
    const int64_t ns[1] = {n};
    check(pwpp_estimate_host(ctx_, 1, ptrs, ns, cols >= 4 ? 4 : 3, row_stride, col_stride));
    n_ = n;
    ran_ = true;
    step_ = 0;
  }

  // Device-resident cloud (zero-copy path, SURVEY 8f-1): packed N x 4 {x,y,z,intensity} or N x 3 rows in device memory.
  // stream == nullptr: the device is synchronized before and after (any producer / consumer stream is safe); otherwise the
  // work is enqueued on `stream` and the device results below are valid in stream order.
  void estimateGroundDevice(const float* d_data, int64_t n, int cols, void* stream = nullptr) {
    if (cols != 3 && cols != 4) throw std::runtime_error("PatchWorkpp::estimateGroundDevice: packed N x 3 or N x 4 float32 rows expected");
    if (cols < 4 && params_.enable_RNR) std::cout << "RNR requires intensity information !" << std::endl;  // reference src :380
    const int64_t offs[2] = {0, n};
    if (!stream) check(pwpp_device_synchronize(ctx_));
    check(cols == 4 ? pwpp_estimate_device(ctx_, 1, d_data, offs, 1, stream) : pwpp_estimate_device_xyz(ctx_, 1, d_data, offs, stream));
    if (!stream) check(pwpp_device_synchronize(ctx_));
    n_ = n;
    ran_ = true;
    step_ = 0;
  }
  // Sensor records of any PointCloud2 layout (pwpp_estimate_host_records / pwpp_estimate_device_records): n records of
  // layout.point_step bytes at `data`, unpacked on the GPU. on_device: `data` is device memory, with the stream rules of
  // estimateGroundDevice. RNR runs when the layout has an intensity field of any datatype.
  void estimateGroundRecords(const void* data, int64_t n, const pwpp_point_layout& layout, bool on_device = false, void* stream = nullptr) {
    if (layout.offset[3] < 0 && params_.enable_RNR) std::cout << "RNR requires intensity information !" << std::endl;  // reference src :380
    const void* frames[1] = {data};
    const int64_t ns[1] = {n};
    const int32_t streams[1] = {0};
    if (on_device) {
      if (!stream) check(pwpp_device_synchronize(ctx_));
      check(pwpp_estimate_device_records(ctx_, 1, streams, frames, ns, &layout, stream));
      if (!stream) check(pwpp_device_synchronize(ctx_));
    } else {
      check(pwpp_estimate_host_records(ctx_, 1, streams, frames, ns, &layout));
    }
    n_ = n;
    ran_ = true;
    step_ = (size_t) layout.point_step;
  }
  // device views of the last call's index lists (int32, valid until the next estimateGround*): {pointer, count}
  std::pair<const int32_t*, int64_t> groundIndicesDevice() {
    const int32_t* idx = nullptr;
    check(pwpp_device_results(ctx_, &idx, nullptr));
    return {idx, count(pwpp_num_ground(ctx_, 0))};
  }
  std::pair<const int32_t*, int64_t> nongroundIndicesDevice() {
    const int32_t* idx = nullptr;
    check(pwpp_device_results(ctx_, &idx, nullptr));
    const int64_t ng = count(pwpp_num_ground(ctx_, 0));
    return {idx + ng, count(pwpp_num_nonground(ctx_, 0))};
  }

  double getHeight() { return pwpp_height(ctx_, 0); }        // reference :154 (adaptive sensor height)
  double getTimeTaken() { return pwpp_time_us(ctx_); }       // reference :155 (microseconds)

  // std::vector flavours of the getters (:157-163)
  std::vector<int> getGroundIndicesVec() { std::vector<int> v((size_t) count(pwpp_num_ground(ctx_, 0))); if (!v.empty()) check(pwpp_copy_ground_indices(ctx_, 0, v.data())); return v; }
  std::vector<int> getNongroundIndicesVec() { std::vector<int> v((size_t) count(pwpp_num_nonground(ctx_, 0))); if (!v.empty()) check(pwpp_copy_nonground_indices(ctx_, 0, v.data())); return v; }
  // row-major n x 3
  std::vector<float> getGroundVec() { std::vector<float> v(3 * (size_t) count(pwpp_num_ground(ctx_, 0))); if (!v.empty()) check(pwpp_copy_ground_xyz(ctx_, 0, v.data())); return v; }
  std::vector<float> getNongroundVec() { std::vector<float> v(3 * (size_t) count(pwpp_num_nonground(ctx_, 0))); if (!v.empty()) check(pwpp_copy_nonground_xyz(ctx_, 0, v.data())); return v; }
  std::vector<float> getCentersVec() { std::vector<float> v(3 * (size_t) count(pwpp_num_patches(ctx_, 0))); if (!v.empty()) check(pwpp_copy_centers(ctx_, 0, v.data())); return v; }
  std::vector<float> getNormalsVec() { std::vector<float> v(3 * (size_t) count(pwpp_num_patches(ctx_, 0))); if (!v.empty()) check(pwpp_copy_normals(ctx_, 0, v.data())); return v; }
  // Ground / non-ground points of the last estimateGroundRecords() as whole records of its layout, byte for byte (every field
  // the sensor sent): count * point_step bytes (pwpp_copy_ground_records / pwpp_copy_nonground_records). Throws after a call
  // that did not take records.
  std::vector<uint8_t> getGroundRecords() { return records(true); }
  std::vector<uint8_t> getNongroundRecords() { return records(false); }

#ifdef PATCHWORKPP_HAVE_EIGEN
  // the reference's exact signatures (:152, :157-163)
  void estimateGround(Eigen::MatrixXf cloud_in) {
    estimateGround(cloud_in.data(), (int64_t) cloud_in.rows(), (int) cloud_in.cols(), 1, (int64_t) cloud_in.rows());  // column-major
  }
  Eigen::MatrixX3f getGround() { return toEigenCloud(getGroundVec()); }
  Eigen::MatrixX3f getNonground() { return toEigenCloud(getNongroundVec()); }
  Eigen::VectorXi getGroundIndices() { return toIndices(getGroundIndicesVec()); }
  Eigen::VectorXi getNongroundIndices() { return toIndices(getNongroundIndicesVec()); }
  Eigen::MatrixX3f getCenters() { return toEigenCloud(getCentersVec()); }
  Eigen::MatrixX3f getNormals() { return toEigenCloud(getNormalsVec()); }
#endif

  // true (default): index lists in the reference's order inside every bin (ascending z, R-VPF removals first in the
  // non-ground part); false: ascending point index inside a bin (no sorting pass)
  void setReferenceOrder(bool on) { check(pwpp_set_output_order(ctx_, on ? PWPP_ORDER_REFERENCE : PWPP_ORDER_BIN)); }
  // Bin: ascending point index inside a bin; Reference (default): the reference's order, equal z in ascending point index;
  // ReferenceExact: the reference's order with equal z where libstdc++'s std::sort leaves them, so the lists equal the
  // unmodified reference's whenever the label sets do (pwpp.h, PWPP_ORDER_REFERENCE_EXACT)
  void setOutputOrder(OutputOrder order) { check(pwpp_set_output_order(ctx_, static_cast<int>(order))); }
  // Double (default): order-free double sums; Reference: the reference's fp32 arithmetic, so that every getter returns the CPU
  // library's values bit for bit (pwpp.h, PWPP_ARITH_REFERENCE)
  void setArithmetic(Arithmetic arith) { check(pwpp_set_arithmetic(ctx_, static_cast<int>(arith))); }

  pwpp_ctx* handle() { return ctx_; }

 private:
  patchwork::Params params_;
  pwpp_ctx* ctx_ = nullptr;
  int64_t n_ = 0;
  bool ran_ = false;
  size_t step_ = 0;   // point_step of the last estimateGroundRecords() (0 after any other call)

  static void check(int rc) { if (rc != PWPP_OK) throw std::runtime_error(std::string("PatchWorkpp: ") + pwpp_last_error()); }
  std::vector<uint8_t> records(bool ground) {
    check(pwpp_host_record_results(ctx_, nullptr, nullptr));   // (fails, with its message, when the last call did not take records)
    std::vector<uint8_t> v((size_t) count(ground ? pwpp_num_ground(ctx_, 0) : pwpp_num_nonground(ctx_, 0)) * step_);
    if (!v.empty()) check(ground ? pwpp_copy_ground_records(ctx_, 0, v.data()) : pwpp_copy_nonground_records(ctx_, 0, v.data()));
    return v;
  }
  // before the first estimateGround() the reference's getters return empty matrices (its members are empty): a count
  // of -1 with nothing processed yet is 0 here, any other failure throws
  int64_t count(int64_t c) const { if (c < 0) { if (!ran_) return 0; throw std::runtime_error(std::string("PatchWorkpp: ") + pwpp_last_error()); } return c; }
#ifdef PATCHWORKPP_HAVE_EIGEN
  static Eigen::MatrixX3f toEigenCloud(const std::vector<float>& v) {
    Eigen::MatrixX3f m(v.size() / 3, 3);
    for (size_t i = 0; i < v.size() / 3; ++i) for (int c = 0; c < 3; ++c) m(i, c) = v[3 * i + c];
    return m;
  }
  static Eigen::VectorXi toIndices(const std::vector<int>& v) {
    Eigen::VectorXi m(v.size());
    for (size_t i = 0; i < v.size(); ++i) m(i) = v[i];
    return m;
  }
#endif
};

}  // namespace patchwork

#endif
