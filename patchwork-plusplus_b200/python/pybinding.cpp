// pypatchworkpp — Python module with the surface of the reference binding
// (reference python/patchworkpp/pybinding.cpp:9-55): class `Parameters` (same fields) and class
// `patchworkpp` (same nine methods). numpy in, numpy out: estimateGround takes any float-convertible
// 2-D array (n,3|4) in C or Fortran order without an extra copy; getters return float32 (n,3)
// Fortran-ordered arrays / int32 (n,) arrays like pybind11/eigen.h produces for the reference.
// The GIL is released while the GPU works.
//
// Device arrays (SURVEY 8f-1): estimateGround also takes any object that exposes `__cuda_array_interface__` (torch, cupy,
// numba) or `__dlpack__` (torch, jax, cupy) with a C-contiguous float32 (n, 3|4) CUDA tensor — no host copy at all — and
// getGroundIndicesDevice() / getNongroundIndicesDevice() return int32 device views (objects with
// `__cuda_array_interface__`; torch.as_tensor(v, device="cuda") / cupy.asarray(v) wrap them without copying; valid until the
// next estimateGround call).
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "patchwork/patchworkpp.h"

namespace py = pybind11;

namespace {
py::array_t<float> x3(const std::vector<float>& v) {
  const py::ssize_t n = (py::ssize_t) (v.size() / 3);
  py::array_t<float, py::array::f_style> a({n, (py::ssize_t) 3});
  auto r = a.mutable_unchecked<2>();
  for (py::ssize_t i = 0; i < n; ++i) for (int c = 0; c < 3; ++c) r(i, c) = v[3 * i + c];
  return a;
}
py::array_t<int> ivec(const std::vector<int>& v) {
  py::array_t<int> a((py::ssize_t) v.size());
  if (!v.empty()) std::memcpy(a.mutable_data(), v.data(), v.size() * sizeof(int));
  return a;
}

// ---- device arrays -----------------------------------------------------------------------------------------------
struct DeviceView {   // what the *Device getters return
  std::uintptr_t ptr = 0;
  py::ssize_t n = 0;
  py::object owner;   // keeps the engine alive
  py::dict cai() const {
    py::dict d;
    d["shape"] = py::make_tuple(n);
    d["typestr"] = "<i4";
    d["data"] = py::make_tuple(ptr, false);   // (torch refuses read-only device arrays; the lists are overwritten by the next call anyway)
    d["version"] = 3;
    d["strides"] = py::none();
    return d;
  }
};

// minimal DLPack (v0.x) structures: https://dmlc.github.io/dlpack/latest/c_api.html
struct DLDev { int32_t device_type; int32_t device_id; };
struct DLDType { uint8_t code; uint8_t bits; uint16_t lanes; };
struct DLTensorMin { void* data; DLDev device; int32_t ndim; DLDType dtype; int64_t* shape; int64_t* strides; uint64_t byte_offset; };
struct DLManagedTensorMin { DLTensorMin dl_tensor; void* manager_ctx; void (*deleter)(DLManagedTensorMin*); };

struct DeviceCloud { const float* ptr = nullptr; int64_t n = 0; int cols = 0; py::object keep; };

bool device_cloud_from(py::object obj, DeviceCloud& out) {
  if (py::hasattr(obj, "__cuda_array_interface__")) {
    py::dict d = obj.attr("__cuda_array_interface__");
    const std::string ts = py::str(d["typestr"]);
    py::tuple shape = d["shape"];
    if (ts != "<f4" || shape.size() != 2) throw std::runtime_error("estimateGround: device array must be float32 with shape (n, 3|4)");
    out.n = shape[0].cast<int64_t>(); out.cols = shape[1].cast<int>();
    if (d.contains("strides") && !d["strides"].is_none()) {
      py::tuple st = d["strides"];
      if (st[1].cast<int64_t>() != 4 || st[0].cast<int64_t>() != 4 * out.cols) throw std::runtime_error("estimateGround: device array must be C-contiguous");
    }
    py::tuple data = d["data"];
    out.ptr = reinterpret_cast<const float*>(data[0].cast<std::uintptr_t>());
    out.keep = obj;
    return true;
  }
  if (py::hasattr(obj, "__dlpack__") && py::hasattr(obj, "__dlpack_device__")) {
    py::tuple dev = obj.attr("__dlpack_device__")();
    if (dev[0].cast<int>() != 2 /* kDLCUDA */) return false;   // a host tensor: take the numpy path
    py::capsule cap = obj.attr("__dlpack__")();
    auto* mt = static_cast<DLManagedTensorMin*>(PyCapsule_GetPointer(cap.ptr(), "dltensor"));
    if (!mt) throw std::runtime_error("estimateGround: bad DLPack capsule");
    const DLTensorMin& t = mt->dl_tensor;
    if (t.ndim != 2 || t.dtype.code != 2 /* float */ || t.dtype.bits != 32 || t.dtype.lanes != 1) throw std::runtime_error("estimateGround: DLPack tensor must be float32 with shape (n, 3|4)");
    out.n = t.shape[0]; out.cols = (int) t.shape[1];
    if (t.strides && (t.strides[1] != 1 || t.strides[0] != out.cols)) throw std::runtime_error("estimateGround: DLPack tensor must be C-contiguous");
    out.ptr = reinterpret_cast<const float*>(static_cast<char*>(t.data) + t.byte_offset);
    out.keep = cap;   // the capsule (not renamed to "used_dltensor") releases the tensor when it is collected; obj outlives the call
    return true;
  }
  return false;
}
}  // namespace

PYBIND11_MODULE(pypatchworkpp, m) {
  m.doc() = "Python Patchwork++ (H100 engine)";
  m.attr("__version__") = "0.0.1";

  py::class_<patchwork::Params>(m, "Parameters")
      .def(py::init<>())
      .def_readwrite("sensor_height", &patchwork::Params::sensor_height)
      .def_readwrite("verbose", &patchwork::Params::verbose)
      .def_readwrite("enable_RNR", &patchwork::Params::enable_RNR)
      .def_readwrite("enable_RVPF", &patchwork::Params::enable_RVPF)
      .def_readwrite("enable_TGR", &patchwork::Params::enable_TGR)
      .def_readwrite("num_iter", &patchwork::Params::num_iter)
      .def_readwrite("num_lpr", &patchwork::Params::num_lpr)
      .def_readwrite("num_min_pts", &patchwork::Params::num_min_pts)
      .def_readwrite("num_zones", &patchwork::Params::num_zones)
      .def_readwrite("num_rings_of_interest", &patchwork::Params::num_rings_of_interest)
      .def_readwrite("RNR_ver_angle_thr", &patchwork::Params::RNR_ver_angle_thr)
      .def_readwrite("RNR_intensity_thr", &patchwork::Params::RNR_intensity_thr)
      .def_readwrite("th_seeds", &patchwork::Params::th_seeds)
      .def_readwrite("th_dist", &patchwork::Params::th_dist)
      .def_readwrite("th_seeds_v", &patchwork::Params::th_seeds_v)
      .def_readwrite("th_dist_v", &patchwork::Params::th_dist_v)
      .def_readwrite("max_range", &patchwork::Params::max_range)
      .def_readwrite("min_range", &patchwork::Params::min_range)
      .def_readwrite("uprightness_thr", &patchwork::Params::uprightness_thr)
      .def_readwrite("adaptive_seed_selection_margin", &patchwork::Params::adaptive_seed_selection_margin)
      .def_readwrite("intensity_thr", &patchwork::Params::intensity_thr)
      .def_readwrite("num_sectors_each_zone", &patchwork::Params::num_sectors_each_zone)
      .def_readwrite("num_rings_each_zone", &patchwork::Params::num_rings_each_zone)
      .def_readwrite("max_flatness_storage", &patchwork::Params::max_flatness_storage)
      .def_readwrite("max_elevation_storage", &patchwork::Params::max_elevation_storage)
      .def_readwrite("elevation_thr", &patchwork::Params::elevation_thr)
      .def_readwrite("flatness_thr", &patchwork::Params::flatness_thr);

  py::class_<patchwork::PatchWorkpp>(m, "patchworkpp")
      .def(py::init<patchwork::Params>())
      .def(py::init<patchwork::Params, int>(), py::arg("params"), py::arg("device"))
      .def("getHeight", &patchwork::PatchWorkpp::getHeight)
      .def("getTimeTaken", &patchwork::PatchWorkpp::getTimeTaken)
      .def("getGround", [](patchwork::PatchWorkpp& s) { return x3(s.getGroundVec()); })
      .def("getNonground", [](patchwork::PatchWorkpp& s) { return x3(s.getNongroundVec()); })
      .def("getCenters", [](patchwork::PatchWorkpp& s) { return x3(s.getCentersVec()); })
      .def("getGroundIndices", [](patchwork::PatchWorkpp& s) { return ivec(s.getGroundIndicesVec()); })
      .def("getNongroundIndices", [](patchwork::PatchWorkpp& s) { return ivec(s.getNongroundIndicesVec()); })
      .def("getNormals", [](patchwork::PatchWorkpp& s) { return x3(s.getNormalsVec()); })
      .def("setReferenceOrder", &patchwork::PatchWorkpp::setReferenceOrder, py::arg("on"),
           "True (default): index lists in the reference's order inside every bin; False: ascending point index inside a bin")
      .def("setOutputOrder", [](patchwork::PatchWorkpp& s, const std::string& order) {
        if (order == "bin") s.setOutputOrder(patchwork::OutputOrder::Bin);
        else if (order == "reference") s.setOutputOrder(patchwork::OutputOrder::Reference);
        else if (order == "reference_exact") s.setOutputOrder(patchwork::OutputOrder::ReferenceExact);
        else throw py::value_error("order must be \"bin\", \"reference\" or \"reference_exact\"");
      }, py::arg("order"),
           "\"bin\": ascending point index inside a bin; \"reference\" (default): the reference's order, equal z in ascending point "
           "index; \"reference_exact\": equal z where the reference's std::sort (libstdc++) leaves them")
      .def("setArithmetic", [](patchwork::PatchWorkpp& s, const std::string& arith) {
        if (arith == "double") s.setArithmetic(patchwork::Arithmetic::Double);
        else if (arith == "reference") s.setArithmetic(patchwork::Arithmetic::Reference);
        else throw py::value_error("arith must be \"double\" or \"reference\"");
      }, py::arg("arith"),
           "\"double\" (default): order-free double sums; \"reference\": the reference's fp32 arithmetic, every result bit for bit "
           "the CPU library's")
      .def("getGroundIndicesDevice", [](py::object self) {
        auto& s = self.cast<patchwork::PatchWorkpp&>();
        const auto v = s.groundIndicesDevice();
        return DeviceView{reinterpret_cast<std::uintptr_t>(v.first), (py::ssize_t) v.second, self};
      }, "int32 device view of the ground index list of the last call (zero-copy; valid until the next estimateGround)")
      .def("getNongroundIndicesDevice", [](py::object self) {
        auto& s = self.cast<patchwork::PatchWorkpp&>();
        const auto v = s.nongroundIndicesDevice();
        return DeviceView{reinterpret_cast<std::uintptr_t>(v.first), (py::ssize_t) v.second, self};
      })
      .def("estimateGround", [](patchwork::PatchWorkpp& s, py::object obj, std::uintptr_t stream) {
        DeviceCloud dc;
        if (device_cloud_from(obj, dc)) {   // device-resident cloud: no host copy
          if (dc.cols != 3 && dc.cols != 4) throw std::runtime_error("estimateGround: device array must have 3 or 4 columns");
          py::gil_scoped_release nogil;
          s.estimateGroundDevice(dc.ptr, dc.n, dc.cols, reinterpret_cast<void*>(stream));
          return;
        }
        py::array_t<float, py::array::forcecast> cloud = py::array_t<float, py::array::forcecast>::ensure(obj);
        if (!cloud) throw std::runtime_error("estimateGround: expected a float-convertible 2-D array (n, 3|4)");
        if (cloud.ndim() != 2) throw std::runtime_error("estimateGround: expected a 2-D array (n, 3|4)");
        const float* data = cloud.data();
        const int64_t n = cloud.shape(0);
        const int cols = (int) cloud.shape(1);
        const int64_t rs = cloud.strides(0) / (py::ssize_t) sizeof(float), cs = cloud.strides(1) / (py::ssize_t) sizeof(float);
        py::gil_scoped_release nogil;
        s.estimateGround(data, n, cols, rs, cs);
      }, py::arg("cloud"), py::arg("stream") = (std::uintptr_t) 0,
         "cloud: numpy-convertible (n, 3|4) array, or a CUDA tensor (__cuda_array_interface__ / __dlpack__); stream: CUDA stream "
         "handle the device cloud is ready on (0: the device is synchronized before and after the call)");

  py::class_<DeviceView>(m, "DeviceView")
      .def_property_readonly("__cuda_array_interface__", &DeviceView::cai)
      .def("__len__", [](const DeviceView& v) { return v.n; })
      .def_readonly("ptr", &DeviceView::ptr);
}
