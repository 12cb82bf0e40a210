// glk/pointcloud_buffer.hpp STAND-IN for the bag pin (test infrastructure): the viewer calls compile and do nothing.
#pragma once
namespace glk {
struct PointCloudBuffer {
  template <class... A>
  PointCloudBuffer(const A&...) {}
};
}  // namespace glk
