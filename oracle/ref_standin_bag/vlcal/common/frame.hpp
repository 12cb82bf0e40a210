// vlcal/common/frame.hpp STAND-IN for the bag pin (test infrastructure; shadows the reference's header, which pulls in
// boost::poly_collection traits): the point container fields static_point_cloud_integrator.cpp reads.
#pragma once
#include <memory>
#include <Eigen/Core>
namespace vlcal {
struct Frame {
  using Ptr = std::shared_ptr<Frame>;
  using ConstPtr = std::shared_ptr<const Frame>;
  virtual ~Frame() {}
  int size() const { return static_cast<int>(num_points); }
  size_t num_points = 0;
  Eigen::Vector4d* points = nullptr;
  double* times = nullptr;
  double* intensities = nullptr;
};
}  // namespace vlcal
