// patchwork/pointcloud2.hpp — the ROS 2 node's message handling (reference ros/src/GroundSegmentationServer.cpp:74-95,
// ros/src/Utils.hpp:158-195) without ROS: a PointCloud2-shaped VIEW (raw data pointer, point_step, float32 field
// offsets) in, packed x/y/z payloads out. A node written against rclcpp fills the view from
// sensor_msgs::msg::PointCloud2 {data.data(), width * height, point_step, fields[i].offset} and copies the payloads
// into its outgoing messages; nothing here depends on ROS headers, so it builds (and is tested) where ROS is absent.
//
// What the reference does per message (Utils.hpp:158-172): walk three PointCloud2ConstIterator<float> over x, y, z into
// an N x 3 Eigen matrix (one float at a time), with RNR disabled because intensity is not carried (":47 ToDo. Support
// intensity"). Here the message buffer is handed to the engine as a STRIDED N x 3 (or N x 4 with intensity) view:
// element (i, c) = data[i * point_step + offset_c], no intermediate matrix, when the offsets are 4-byte aligned and
// equally spaced (x,y,z at 0,4,8 as every common driver publishes); any other layout is gathered once into a buffer.
#ifndef PATCHWORKPP_POINTCLOUD2_HPP
#define PATCHWORKPP_POINTCLOUD2_HPP

#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "patchwork/patchworkpp.h"

namespace patchwork {

struct PointCloud2View {
  const uint8_t* data = nullptr;   // sensor_msgs::msg::PointCloud2::data.data()
  int64_t num_points = 0;          // width * height
  uint32_t point_step = 0;         // bytes between consecutive points
  int32_t off_x = 0, off_y = 4, off_z = 8;   // byte offsets of the FLOAT32 fields inside a point
  int32_t off_intensity = -1;      // < 0: no intensity field (the reference node's case: RNR is skipped)
};

// estimateGround on a PointCloud2-shaped buffer (reference GroundSegmentationServer.cpp:74-78). Returns true when the
// buffer was passed through without a host-side gather.
inline bool estimateGround(PatchWorkpp& pw, const PointCloud2View& v) {
  if (v.num_points < 0 || (v.num_points > 0 && !v.data) || v.point_step < 12) throw std::invalid_argument("PointCloud2View: bad buffer");
  const bool has_i = v.off_intensity >= 0;
  const int cols = has_i ? 4 : 3;
  const int32_t offs[4] = {v.off_x, v.off_y, v.off_z, v.off_intensity};
  for (int c = 0; c < cols; ++c)
    if (offs[c] < 0 || offs[c] + 4 > (int32_t) v.point_step) throw std::invalid_argument("PointCloud2View: field offset outside the point");
  const int32_t d = v.off_y - v.off_x;
  bool strided = v.point_step % 4 == 0 && v.off_x % 4 == 0 && d != 0 && d % 4 == 0 && v.off_z - v.off_y == d && (!has_i || v.off_intensity - v.off_z == d) &&
                 reinterpret_cast<uintptr_t>(v.data) % 4 == 0;
  if (strided) {
    // element (i, c) at float index i * (point_step / 4) + c * (d / 4), counted from the x field of point 0
    pw.estimateGround(reinterpret_cast<const float*>(v.data + v.off_x), v.num_points, cols, (int64_t) (v.point_step / 4), (int64_t) (d / 4));
    return true;
  }
  std::vector<float> packed((size_t) v.num_points * cols);
  for (int64_t i = 0; i < v.num_points; ++i)
    for (int c = 0; c < cols; ++c) std::memcpy(&packed[(size_t) i * cols + c], v.data + (size_t) i * v.point_step + offs[c], 4);
  pw.estimateGround(packed.data(), v.num_points, cols, cols, 1);
  return false;
}

// The description of a sensor_msgs::msg::PointCloud2 as the message carries it: every field's name, offset, datatype
// (sensor_msgs/PointField codes = PWPP_FIELD_*) and count, plus is_bigendian. A ROS 2 node fills it from the message:
//   for (auto& f : msg->fields) m.fields.push_back({f.name, f.offset, f.datatype, f.count});
struct PointField {
  std::string name;
  uint32_t offset = 0;
  uint8_t datatype = 0;
  uint32_t count = 1;
};
struct PointCloud2Message {
  const uint8_t* data = nullptr;   // msg->data.data()
  int64_t num_points = 0;          // width * height
  uint32_t point_step = 0;
  bool is_bigendian = false;
  std::vector<PointField> fields;
};

// The record layout of a message: fields `x`, `y`, `z` and, when present, `intensity`, found by name (the fields the reference
// node's iterators read, ros/src/Utils.hpp:158-172). Throws std::invalid_argument for a big-endian message, a used field with
// count != 1 and missing x / y / z; the datatypes and offsets themselves are checked by the engine.
inline pwpp_point_layout pointLayout(const PointCloud2Message& m) {
  if (m.is_bigendian) throw std::invalid_argument("PointCloud2Message: big-endian records are not supported");
  static const char* names[4] = {"x", "y", "z", "intensity"};
  pwpp_point_layout L;
  L.point_step = (int32_t) m.point_step;
  for (int c = 0; c < 4; ++c) {
    L.offset[c] = -1;
    L.datatype[c] = 0;
    for (const PointField& f : m.fields) {
      if (f.name != names[c]) continue;
      if (f.count != 1) throw std::invalid_argument(std::string("PointCloud2Message: field ") + names[c] + " has count != 1");
      L.offset[c] = (int32_t) f.offset;
      L.datatype[c] = f.datatype;
      break;
    }
    if (c < 3 && L.offset[c] < 0) throw std::invalid_argument(std::string("PointCloud2Message: no field ") + names[c]);
  }
  return L;
}

// estimateGround on a message of any layout (reference GroundSegmentationServer.cpp:74-78): the records go to the GPU as they
// are and are unpacked there, intensity of any datatype included (RNR then runs, unlike the reference node, :46-47).
inline void estimateGround(PatchWorkpp& pw, const PointCloud2Message& m) {
  if (m.num_points < 0 || (m.num_points > 0 && !m.data)) throw std::invalid_argument("PointCloud2Message: bad buffer");
  pw.estimateGroundRecords(m.data, m.num_points, pointLayout(m));
}

// Payload of an outgoing x/y/z PointCloud2 (reference Utils.hpp:174-195 EigenMatToPointCloud2 -> FillPointCloud2XYZ):
// point_step 12, fields x,y,z FLOAT32 at 0,4,8, is_dense. `which` = true: ground, false: non-ground.
struct PointCloud2Payload {
  std::vector<uint8_t> data;
  uint32_t width = 0, height = 1, point_step = 12, row_step = 0;
};
inline PointCloud2Payload makeCloudPayload(PatchWorkpp& pw, bool ground) {
  const std::vector<float> xyz = ground ? pw.getGroundVec() : pw.getNongroundVec();   // reference :82-83
  PointCloud2Payload p;
  p.width = (uint32_t) (xyz.size() / 3);
  p.row_step = p.width * p.point_step;
  p.data.resize(xyz.size() * sizeof(float));
  if (!xyz.empty()) std::memcpy(p.data.data(), xyz.data(), p.data.size());
  return p;
}

// Payload of an outgoing PointCloud2 in the INPUT's own layout: the ground (ground = true) or non-ground points of the last
// estimateGround(pw, in) as whole records, byte for byte (intensity, ring, per-point time, padding: every field the sensor
// sent, which the reference node's x/y/z messages drop), gathered on the GPU. The message takes in.point_step and in.fields,
// height 1, width = the count. `in` describes the message of that call (its data is not read again).
struct PointCloud2RecordsPayload {
  std::vector<uint8_t> data;
  uint32_t width = 0, height = 1, point_step = 0, row_step = 0;
  bool is_bigendian = false;
  std::vector<PointField> fields;
};
inline PointCloud2RecordsPayload makeRecordsPayload(PatchWorkpp& pw, bool ground, const PointCloud2Message& in) {
  PointCloud2RecordsPayload p;
  p.data = ground ? pw.getGroundRecords() : pw.getNongroundRecords();
  p.point_step = in.point_step;
  p.fields = in.fields;
  p.is_bigendian = in.is_bigendian;
  p.width = in.point_step ? (uint32_t) (p.data.size() / in.point_step) : 0;
  p.row_step = p.width * p.point_step;
  return p;
}

}  // namespace patchwork
#endif
