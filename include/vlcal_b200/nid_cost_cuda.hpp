// nid_cost_cuda.hpp -- reference-side binding for the NID_BFGS branch: keeps Ceres and the Sophus manifold, replaces
// the per-bag cost functor and its autodiff by the sm_90a value + gradient kernel of libvlcal_nid.so.
//
// In VisualCameraCalibration::estimate_pose_bfgs (src/vlcal/calib/visual_camera_calibration.cpp:187-238) the reference
// builds, per bag,   std::shared_ptr<NIDCost>(new NIDCost(proj, normalized_image, culled_points, bins))        (:203)
// sums them in       MultiNIDCost                                                                         (:141-173)
// and differentiates ceres::AutoDiffFirstOrderFunction<MultiNIDCost, Sophus::SE3d::num_parameters>            (:211)
// A maintainer replaces those three by
//   auto sum_nid = new vlcal::MultiNIDCostFunction(T_camera_lidar);
//   sum_nid->add(std::make_shared<vlcal::NIDCostCuda>(camera_model, intrinsics, distortion, dataset[i]->image, culled_points, params.nid_bins));
//   ceres::GradientProblem problem(sum_nid, new Sophus::Manifold<Sophus::SE3>());
// Everything else (options, callbacks, ceres::Solve) stays.  Evaluate() returns exactly what the autodiff function
// returns: the summed NID and its 7 ambient partials d/d(qx qy qz qw tx ty tz); the validity region around the start pose
// (:152-156) and "any bag failed => false" (:172) are kept.
//
// Compile-checked inside the reference tree's headers (with stand-ins for Ceres / Sophus / Eigen, which this repository's
// image lacks) by tests/test_cpp_shim.py.
#pragma once

#include <cmath>
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include <ceres/first_order_function.h>
#include <opencv2/core.hpp>
#include <sophus/se3.hpp>
#include <vlcal/common/frame.hpp>

#include "vlcal_nid.h"

namespace vlcal {

// one bag: replaces vlcal::NIDCost (include/vlcal/costs/nid_cost.hpp:22-107), value AND Jet evaluation
class NIDCostCuda {
public:
  // image: the mono8 image itself (CV_8UC1, visual_lidar_data.hpp:16) -- the library forms the 1/255-normalised bin
  // lookup of nid_cost.hpp:78-79 itself, so no convertTo(CV_64FC1) copy is needed.
  NIDCostCuda(
    const std::string& camera_model,
    const std::vector<double>& intrinsics,
    const std::vector<double>& distortion_coeffs,
    const cv::Mat& image,
    const Frame::ConstPtr& points,
    int bins = 16,
    int device = -1)
  : ctx(nullptr) {
    const int model = vlcal_camera_model_id(camera_model.c_str());
    if (model < 0) {
      throw std::runtime_error(std::string("NIDCostCuda: ") + vlcal_nid_last_error());
    }
    const int rc = vlcal_nid_create(
      &ctx,
      device,
      VLCAL_NID_MODE_BSPLINE,
      model,
      intrinsics.data(),
      static_cast<int>(intrinsics.size()),
      distortion_coeffs.data(),
      static_cast<int>(distortion_coeffs.size()),
      image.data,
      image.cols,
      image.rows,
      static_cast<int>(image.step),
      reinterpret_cast<const double*>(points->points),
      points->intensities,
      static_cast<int64_t>(points->size()),
      bins,
      /*max_fov_rad=*/0.0);  // mode B has no FoV test (nid_cost.hpp:46-58)
    if (rc != VLCAL_OK) {
      throw std::runtime_error(std::string("NIDCostCuda: ") + vlcal_nid_last_error());
    }
  }
  ~NIDCostCuda() { vlcal_nid_destroy(ctx); }
  NIDCostCuda(const NIDCostCuda&) = delete;
  NIDCostCuda& operator=(const NIDCostCuda&) = delete;

  // NIDCost::operator()<double> (gradient7 == nullptr) / operator()<ceres::Jet<double, 7>>: residual[0], its partials,
  // and the functor's bool (false = non-finite NID, nid_cost.hpp:98-102)
  bool evaluate(const double* T_camera_lidar_params, double* residual, double* gradient7) const {
    int32_t ok = 0;
    int rc;
    if (gradient7) {
      rc = vlcal_nid_evaluate_bspline_grad(ctx, T_camera_lidar_params, 1, residual, gradient7, &ok);
    } else {
      rc = vlcal_nid_evaluate_bspline(ctx, T_camera_lidar_params, 1, residual, &ok, nullptr);
    }
    if (rc != VLCAL_OK) {
      throw std::runtime_error(std::string("NIDCostCuda::evaluate: ") + vlcal_nid_last_error());
    }
    return ok != 0;
  }

private:
  vlcal_nid_ctx* ctx;
};

// all bags: replaces MultiNIDCost + ceres::AutoDiffFirstOrderFunction<MultiNIDCost, 7> (visual_camera_calibration.cpp:141-173,211)
class MultiNIDCostFunction : public ceres::FirstOrderFunction {
public:
  explicit MultiNIDCostFunction(const Sophus::SE3d& init_T_camera_lidar) : init_T_camera_lidar(init_T_camera_lidar) {}

  void add(const std::shared_ptr<NIDCostCuda>& cost) { costs.emplace_back(cost); }

  bool Evaluate(const double* const parameters, double* cost, double* gradient) const override {
    const Eigen::Map<const Sophus::SE3d> T_camera_lidar(parameters);
    const Sophus::SE3d delta = init_T_camera_lidar.inverse() * T_camera_lidar;
    if (delta.translation().norm() > 0.2 || Eigen::AngleAxisd(delta.rotationMatrix()).angle() > 2.0 * M_PI / 180.0) {
      return false;  // :154-156
    }
    bool all_ok = true;
    double total = 0.0;
    double g[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (const auto& c : costs) {  // bag order, like residuals[0] += residuals[i] (:167-169)
      double r = 0.0, gi[7];
      all_ok = c->evaluate(parameters, &r, gradient ? gi : nullptr) && all_ok;
      total += r;
      if (gradient) {
        for (int k = 0; k < 7; k++) g[k] += gi[k];
      }
    }
    *cost = total;
    if (gradient) {
      for (int k = 0; k < 7; k++) gradient[k] = g[k];
    }
    return all_ok;  // :172
  }

  int NumParameters() const override { return Sophus::SE3d::num_parameters; }

private:
  Sophus::SE3d init_T_camera_lidar;
  std::vector<std::shared_ptr<NIDCostCuda>> costs;
};

}  // namespace vlcal
