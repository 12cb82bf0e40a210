// sensor_msgs/PointCloud2.h STAND-IN (test infrastructure): the fields of the ROS 1 message that extract_raw_points
// reads, with ros::Time::toSec as roscpp defines it (double(sec) + 1e-9 * double(nsec)).
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <unordered_map>  // through ros/ros.h in a ROS build
#include <vector>
namespace ros {
struct Time {
  uint32_t sec = 0, nsec = 0;
  double toSec() const { return static_cast<double>(sec) + 1e-9 * static_cast<double>(nsec); }
};
}  // namespace ros
namespace sensor_msgs {
struct PointField {
  enum { INT8 = 1, UINT8 = 2, INT16 = 3, UINT16 = 4, INT32 = 5, UINT32 = 6, FLOAT32 = 7, FLOAT64 = 8 };
  std::string name;
  uint32_t offset = 0;
  uint8_t datatype = 0;
  uint32_t count = 1;
};
struct Header {
  uint32_t seq = 0;
  ros::Time stamp;
  std::string frame_id;
};
struct PointCloud2 {
  using Ptr = std::shared_ptr<PointCloud2>;
  using ConstPtr = std::shared_ptr<const PointCloud2>;
  Header header;
  uint32_t height = 0, width = 0;
  std::vector<PointField> fields;
  uint8_t is_bigendian = 0;
  uint32_t point_step = 0, row_step = 0;
  std::vector<uint8_t> data;
  uint8_t is_dense = 0;
};
}  // namespace sensor_msgs
