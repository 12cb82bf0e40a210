// Prints, in hexadecimal floating point, the quaternion the Eigen stand-in (oracle/ref_standin) forms for
// preprocess_map's virtual pinhole camera, AngleAxisd(pi/2, Y) * AngleAxisd(-pi/2, Z) (preprocess_map.cpp:189), and the
// stand-in's rotation of the three unit vectors by it and by AngleAxisd(-pi/2, X) (:195).
#include <Eigen/Core>
#include <Eigen/Geometry>
#include <cmath>
#include <cstdio>

int main() {
  const Eigen::Quaterniond q = Eigen::AngleAxisd(M_PI_2, Eigen::Vector3d(0.0, 1.0, 0.0)) * Eigen::AngleAxisd(-M_PI_2, Eigen::Vector3d(0.0, 0.0, 1.0));
  std::printf("%a %a %a %a\n", q.w(), q.x(), q.y(), q.z());
  const Eigen::AngleAxisd rx(-M_PI_2, Eigen::Vector3d(1.0, 0.0, 0.0));
  for (int k = 0; k < 3; k++) {
    Eigen::Vector3d e(0.0, 0.0, 0.0);
    e[k] = 1.0;
    const Eigen::Vector3d a = q * e, b = rx * e;
    std::printf("%a %a %a %a %a %a\n", a[0], a[1], a[2], b[0], b[1], b[2]);
  }
  return 0;
}
