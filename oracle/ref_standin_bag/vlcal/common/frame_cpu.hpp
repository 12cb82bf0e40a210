// vlcal/common/frame_cpu.hpp STAND-IN for the bag pin (test infrastructure): an owning Frame.  Points of dimension D
// become (p.cast<double>(), 1) in the first D coefficients of a Vector4d, as FrameCPU's constructor stores them.
#pragma once
#include <vector>
#include <vlcal/common/frame.hpp>
namespace vlcal {
struct FrameCPU : public Frame {
  using Ptr = std::shared_ptr<FrameCPU>;
  using ConstPtr = std::shared_ptr<const FrameCPU>;
  template <class T, int D, class Alloc>
  explicit FrameCPU(const std::vector<Eigen::Matrix<T, D, 1>, Alloc>& pts) : points_storage(pts.size()) {
    for (size_t i = 0; i < pts.size(); i++) {
      Eigen::Vector4d v(0.0, 0.0, 0.0, 1.0);
      for (int k = 0; k < D; k++) v[k] = static_cast<double>(pts[i][k]);
      points_storage[i] = v;
    }
    num_points = pts.size();
    points = points_storage.data();
  }
  template <class T>
  void add_intensities(const std::vector<T>& v) {
    intensities_storage.assign(v.begin(), v.end());
    intensities = intensities_storage.data();
  }
  std::vector<Eigen::Vector4d> points_storage;
  std::vector<double> intensities_storage;
};
}  // namespace vlcal
