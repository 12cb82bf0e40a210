// Compiles include/vlcal_b200/nid_cost_cuda.hpp (the NID_BFGS binding) against the stand-in third-party headers of
// oracle/ref_standin (Ceres, Sophus, Eigen, cv::Mat) and the Frame stand-in of tests/cpp_stubs, and drives
// MultiNIDCostFunction the way visual_camera_calibration.cpp:208-228 would: through ceres::FirstOrderFunction.
// Output: "EVAL ok=<0|1> n=<parameters> cost=<value> g0=<d cost / d qx>", or "EXCEPTION <message>" with exit code 3.
#include <cstdio>
#include <memory>
#include <vector>

#include <vlcal_b200/nid_cost_cuda.hpp>

int main() {
  const int W = 64, H = 48, N = 500;
  std::vector<unsigned char> pixels(W * H);
  for (int i = 0; i < W * H; i++) pixels[i] = static_cast<unsigned char>((i * 37) % 251);
  std::vector<Eigen::Vector4d> pts;
  std::vector<double> intens;
  for (int i = 0; i < N; i++) {  // a patch in front of the camera (z = 2 m), spread over most of the image
    pts.emplace_back(-0.8 + 1.6 * (i % 25) / 24.0, -0.6 + 1.2 * (i / 25) / 19.0, 2.0, 1.0);
    intens.push_back((i % 16) / 16.0);
  }
  auto frame = std::make_shared<vlcal::Frame>();
  frame->num_points = N, frame->points = pts.data(), frame->intensities = intens.data();
  const cv::Mat image(H, W, CV_8UC1, pixels.data(), static_cast<size_t>(W));
  try {
    const Sophus::SE3d init;
    auto* fn = new vlcal::MultiNIDCostFunction(init);
    fn->add(std::make_shared<vlcal::NIDCostCuda>("plumb_bob", std::vector<double>{60.0, 60.0, 32.0, 24.0}, std::vector<double>{}, image, frame, 16));
    std::unique_ptr<ceres::FirstOrderFunction> f(fn);
    double x[7] = {0, 0, 0, 1, 0, 0, 0}, cost = 0.0, grad[7];
    const bool ok = f->Evaluate(x, &cost, grad);
    std::printf("EVAL ok=%d n=%d cost=%.17g g0=%.17g\n", ok ? 1 : 0, f->NumParameters(), cost, grad[0]);
  } catch (const std::exception& e) {
    std::printf("EXCEPTION %s\n", e.what());
    return 3;
  }
  return 0;
}
