// The reference's OpenMP bag loop (visual_camera_calibration.cpp:107-110) driven through
// include/vlcal_b200/cost_calculator_nid_cuda.hpp: one CostCalculatorNIDCuda per bag, calculate(T) from the workers of
// `#pragma omp parallel for`.  Construction and destruction run in parallel loops too, so uploads overlap and pooled
// device blocks pass from one thread to another between rounds.
//
// argv[1] = binary file written by the test:
//   [int32 B, P, R]
//   B x [int32 W, H, N][u8 image W*H][f64 points N*4][f64 intensities N]
//   P x [f64 T 16] (column-major)
// Round r builds slot i from bag (i + r) % B, so bag sizes move between threads from round to round.
// Output: "VAL r slot bag pose value" per call, then "INFLIGHT calc <k>" and "INFLIGHT create <k>", the largest number of
// calculate() calls / constructors whose omp_get_wtime windows overlapped, then "OK".
// Exit codes: 0 ok, 2 unreadable input, 3 an exception (the library's message follows "EXCEPTION").
#include <omp.h>

#include <algorithm>
#include <cstdio>
#include <memory>
#include <string>
#include <utility>
#include <vector>
#include <vlcal_b200/cost_calculator_nid_cuda.hpp>

namespace camera {
GenericCameraBase::ConstPtr create_camera(const std::string&, const std::vector<double>&, const std::vector<double>&) {
  return nullptr;  // the CUDA cost takes the camera by name and parameters here
}
}  // namespace camera

struct BagData {
  int W = 0, H = 0, N = 0;
  std::vector<unsigned char> image;
  std::vector<Eigen::Vector4d> points;
  std::vector<double> intensities;
  std::shared_ptr<vlcal::VisualLiDARData> data;
};

// the largest number of [start, end) windows that contain one instant
static int max_in_flight(const std::vector<std::pair<double, double>>& windows) {
  std::vector<std::pair<double, int>> ev;
  for (const auto& w : windows) ev.emplace_back(w.first, 1), ev.emplace_back(w.second, -1);
  std::sort(ev.begin(), ev.end());  // at equal times the end (-1) sorts first: touching windows do not overlap
  int cur = 0, best = 0;
  for (const auto& e : ev) best = std::max(best, cur += e.second);
  return best;
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  int hdr[3];
  if (std::fread(hdr, sizeof(int), 3, f) != 3) return 2;
  const int B = hdr[0], P = hdr[1], R = hdr[2];
  std::vector<BagData> bags(B);
  for (auto& b : bags) {
    int d[3];
    if (std::fread(d, sizeof(int), 3, f) != 3) return 2;
    b.W = d[0], b.H = d[1], b.N = d[2];
    b.image.resize(static_cast<size_t>(b.W) * b.H);
    b.points.resize(b.N);
    b.intensities.resize(b.N);
    if (std::fread(b.image.data(), 1, b.image.size(), f) != b.image.size()) return 2;
    if (std::fread(b.points.data(), sizeof(Eigen::Vector4d), b.N, f) != static_cast<size_t>(b.N)) return 2;
    if (std::fread(b.intensities.data(), sizeof(double), b.N, f) != static_cast<size_t>(b.N)) return 2;
    b.data = std::make_shared<vlcal::VisualLiDARData>();
    b.data->image.data = b.image.data(), b.data->image.cols = b.W, b.data->image.rows = b.H, b.data->image.step = b.W;
    b.data->points = std::make_shared<vlcal::FrameCPU>();
    b.data->points->points = b.points.data(), b.data->points->intensities = b.intensities.data(), b.data->points->num_points = b.N;
  }
  std::vector<Eigen::Isometry3d> Ts(P);
  for (auto& T : Ts)
    if (std::fread(T.matrix().data(), sizeof(double), 16, f) != 16) return 2;
  std::fclose(f);

  const std::vector<double> intr{400.0, 410.0, 320.0, 240.0}, dist{-0.04, 0.08, 1e-4, -3e-4, -0.04};
  std::vector<std::pair<double, double>> calc_windows, create_windows;
  std::vector<std::string> errors(B);
  for (int r = 0; r < R; r++) {
    std::vector<std::shared_ptr<vlcal::CostCalculator>> costs(B);
    std::vector<std::pair<double, double>> cw(B);
#pragma omp parallel for schedule(static)
    for (int i = 0; i < B; i++) {
      cw[i].first = omp_get_wtime();
      try {
        costs[i] = std::make_shared<vlcal::CostCalculatorNIDCuda>("plumb_bob", intr, dist, bags[(i + r) % B].data, 16);
      } catch (const std::exception& e) {
        errors[i] = e.what();
      }
      cw[i].second = omp_get_wtime();
    }
    create_windows.insert(create_windows.end(), cw.begin(), cw.end());
    for (const auto& e : errors) {
      if (!e.empty()) {
        std::printf("EXCEPTION %s\n", e.c_str());
        return 3;
      }
    }
    for (int p = 0; p < P; p++) {
      const Eigen::Isometry3d T_camera_lidar = Ts[p];
      std::vector<double> results(B);
      std::vector<std::pair<double, double>> w(B);
#pragma omp parallel for schedule(static)
      for (int i = 0; i < B; i++) {
        w[i].first = omp_get_wtime();
        try {
          results[i] = costs[i]->calculate(T_camera_lidar);
        } catch (const std::exception& e) {
          errors[i] = e.what();
        }
        w[i].second = omp_get_wtime();
      }
      calc_windows.insert(calc_windows.end(), w.begin(), w.end());
      for (const auto& e : errors) {
        if (!e.empty()) {
          std::printf("EXCEPTION %s\n", e.c_str());
          return 3;
        }
      }
      for (int i = 0; i < B; i++) std::printf("VAL %d %d %d %d %.17g\n", r, i, (i + r) % B, p, results[i]);
    }
#pragma omp parallel for schedule(static)
    for (int i = 0; i < B; i++) costs[i].reset();
  }
  std::printf("INFLIGHT calc %d\nINFLIGHT create %d\nOK\n", max_in_flight(calc_windows), max_in_flight(create_windows));
  return 0;
}
