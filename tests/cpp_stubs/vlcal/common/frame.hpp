// Stand-in with the members of vlcal::Frame the BFGS binding (include/vlcal_b200/nid_cost_cuda.hpp) reads
// (test scaffolding only).
#pragma once
#include <cstddef>
#include <memory>
#include <Eigen/Core>
namespace vlcal {
struct Frame {
  using ConstPtr = std::shared_ptr<const Frame>;
  Eigen::Vector4d* points = nullptr;
  double* intensities = nullptr;
  size_t num_points = 0;
  size_t size() const { return num_points; }
};
}  // namespace vlcal
