// bag_ref_shim.cpp -- C entry points into the reference's OWN per-scan code of `preprocess` (test infrastructure):
// extract_raw_points (include/vlcal/common/ros_cloud_converter.hpp, ROS 1 branch), TimeKeeper::process
// (src/vlcal/common/time_keeper.cpp) and StaticPointCloudIntegrator::insert_points / get_points
// (src/vlcal/preprocess/static_point_cloud_integrator.cpp), compiled where they lie against the stand-ins of
// ref_standin_bag/ (bag_ref.mk).  tests/golden/make_reference_bag_outputs.py records what they return.
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include <vlcal/common/ros_cloud_converter.hpp>
#include <vlcal/common/time_keeper.hpp>
#include <vlcal/common/frame_cpu.hpp>
#include <vlcal/preprocess/static_point_cloud_integrator.hpp>

extern "C" {

// One PointCloud2 through extract_raw_points -> 0 when it returns nullptr, else 1 with n x 4 doubles (x, y, z, 1),
// the intensities (*n_int of them) and the times (*n_times).
int bagref_extract(const uint8_t* data, int64_t data_len, uint32_t width, uint32_t height, uint32_t point_step, int n_fields, const char** names,
                   const uint32_t* offsets, const uint8_t* datatypes, const char* intensity_channel, uint32_t sec, uint32_t nsec, double* points_out,
                   double* intensities_out, int64_t* n_int, double* times_out, int64_t* n_times, double* stamp_out) {
  sensor_msgs::PointCloud2 msg;
  msg.header.stamp.sec = sec, msg.header.stamp.nsec = nsec;
  msg.width = width, msg.height = height, msg.point_step = point_step;
  for (int i = 0; i < n_fields; i++) {
    sensor_msgs::PointField f;
    f.name = names[i], f.offset = offsets[i], f.datatype = datatypes[i];
    msg.fields.push_back(f);
  }
  msg.data.assign(data, data + data_len);
  const auto raw = vlcal::extract_raw_points(msg, intensity_channel);
  if (!raw) return 0;
  for (size_t i = 0; i < raw->points.size(); i++)
    for (int k = 0; k < 4; k++) points_out[4 * i + k] = raw->points[i][k];
  std::memcpy(intensities_out, raw->intensities.data(), sizeof(double) * raw->intensities.size());
  std::memcpy(times_out, raw->times.data(), sizeof(double) * raw->times.size());
  *n_int = raw->intensities.size();
  *n_times = raw->times.size();
  *stamp_out = raw->stamp;
  return 1;
}

// A sequence of frames through one TimeKeeper: frame f has stamp stamps[f], n_points[f] points and times
// times[times_first[f] .. times_first[f + 1]) (empty: no per-point times) -> accept_out[f] = process().
void bagref_time_keeper(int n_frames, const double* stamps, const int64_t* n_points, const int64_t* times_first, const double* times, int* accept_out) {
  vlcal::TimeKeeper keeper;
  for (int f = 0; f < n_frames; f++) {
    auto raw = std::make_shared<vlcal::RawPoints>();
    raw->stamp = stamps[f];
    raw->points.resize(n_points[f]);
    raw->times.assign(times + times_first[f], times + times_first[f + 1]);
    accept_out[f] = keeper.process(raw) ? 1 : 0;
  }
}

// Frames of (x, y, z, 1) points and intensities through insert_points in order, then get_points -> the voxel count,
// with (x, y, z, intensity) of each in the hash table's iteration order.
int64_t bagref_integrate(int n_frames, const int64_t* frame_first, const double* xyzw, const double* intensities, double voxel_resolution,
                         double min_distance, double* out) {
  vlcal::StaticPointCloudIntegratorParams params;
  params.voxel_resolution = voxel_resolution;
  params.min_distance = min_distance;
  vlcal::StaticPointCloudIntegrator integrator(params);
  for (int f = 0; f < n_frames; f++) {
    const int64_t b = frame_first[f], e = frame_first[f + 1];
    std::vector<Eigen::Vector4d, Eigen::aligned_allocator<Eigen::Vector4d>> pts(e - b);
    for (int64_t i = b; i < e; i++) pts[i - b] = Eigen::Vector4d(xyzw[4 * i], xyzw[4 * i + 1], xyzw[4 * i + 2], xyzw[4 * i + 3]);
    auto frame = std::make_shared<vlcal::FrameCPU>(pts);
    frame->add_intensities(std::vector<double>(intensities + b, intensities + e));
    integrator.insert_points(frame);
  }
  const auto points = integrator.get_points();
  for (int i = 0; i < points->size(); i++) {
    for (int k = 0; k < 3; k++) out[4 * i + k] = points->points[i][k];
    out[4 * i + 3] = points->intensities[i];
  }
  return points->size();
}
}
