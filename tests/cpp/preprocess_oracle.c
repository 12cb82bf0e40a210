/* preprocess_oracle.c -- plain sequential restatements of preprocess_map's point stages, the CPU checker of
 * csrc/preprocess.cu (built by tests/preprocess_oracle.py with -ffp-contract=off).
 *
 *   orc_approximate_voxel_grid  pcl::ApproximateVoxelGrid<PointXYZI>::applyFilter (PCL 1.10-1.12, approximate_voxel_grid.hpp),
 *                               the 512-entry history table walked in input order, exactly as the reference runs it
 *   orc_voxel_grid_fov          pcl::VoxelGrid<PointXYZ>::applyFilter at 0.2 m with its INT32_MAX fallback, voxel sums in
 *                               point-index order, then estimate_fov.cpp:63-66's `norm() < 1.0` removal
 *   orc_rank_equalize           preprocess_map.cpp:158-167 with a stable tie rule (ties by point index)
 *   orc_min_bearing_cosine      estimate_fov.cpp:72-89 with the Eigen stand-in's term order
 *   orc_virtual_lidar_rotation  preprocess_map.cpp:189/:195 with Eigen's quaternion product and toRotationMatrix
 * The PCL parts are restated from PCL's sources, not pinned against a PCL binary. */
#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* static_cast<int>(float) on x86-64 (cvttss2si): INT_MIN out of range.  Written out so the checker has no UB. */
static int f2i_x86(float f) { return (f >= -2147483648.0f && f < 2147483648.0f) ? (int)f : INT_MIN; }

typedef struct {
  int ix, iy, iz;
  int count;
  float centroid[4];
} he;

static void flush(he* h, float* out, int64_t op) {
  const float c = (float)h->count;
  for (int k = 0; k < 4; k++) out[4 * op + k] = h->centroid[k] / c; /* centroid /= float(count) */
}

int64_t orc_approximate_voxel_grid(const float* xyzi, int64_t n, double leaf_size, float* out) {
  const float leaf = (float)leaf_size;
  const float inv = 1.0f / leaf;
  he history[512];
  for (int i = 0; i < 512; i++) {
    history[i].count = 0;
    for (int k = 0; k < 4; k++) history[i].centroid[k] = 0.0f;
  }
  int64_t op = 0;
  for (int64_t cp = 0; cp < n; cp++) {
    const float* p = xyzi + 4 * cp;
    const int ix = f2i_x86(floorf(p[0] * inv));
    const int iy = f2i_x86(floorf(p[1] * inv));
    const int iz = f2i_x86(floorf(p[2] * inv));
    const unsigned int hash = ((unsigned int)ix * 7171u + (unsigned int)iy * 3079u + (unsigned int)iz * 4231u) & 511u;
    he* h = &history[hash];
    if (h->count && (ix != h->ix || iy != h->iy || iz != h->iz)) {
      flush(h, out, op++);
      h->count = 0;
      for (int k = 0; k < 4; k++) h->centroid[k] = 0.0f;
    }
    h->ix = ix;
    h->iy = iy;
    h->iz = iz;
    h->count++;
    for (int k = 0; k < 4; k++) h->centroid[k] += p[k];
  }
  for (int i = 0; i < 512; i++)
    if (history[i].count) flush(&history[i], out, op++);
  return op;
}

typedef struct {
  unsigned int key;
  int64_t index;
} keyed;

static int cmp_keyed(const void* a, const void* b) {
  const keyed* x = (const keyed*)a;
  const keyed* y = (const keyed*)b;
  if (x->key != y->key) return x->key < y->key ? -1 : 1;
  return (x->index > y->index) - (x->index < y->index);
}

static int keep_by_norm(float x, float y, float z) { return !(sqrtf((x * x + y * y) + z * z) < 1.0f); }

int64_t orc_voxel_grid_fov(const float* xyz, int64_t n, float* out, int* unfiltered) {
  const float inv = 1.0f / 0.2f;
  float min_p[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, max_p[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int64_t i = 0; i < n; i++) {
    for (int c = 0; c < 3; c++) {
      const float v = xyz[3 * i + c];
      if (v < min_p[c]) min_p[c] = v;
      if (v > max_p[c]) max_p[c] = v;
    }
  }
  int overflow = 0;
  int64_t d[3] = {0, 0, 0};
  for (int c = 0; c < 3; c++) {
    const float ext = (max_p[c] - min_p[c]) * inv;
    if (!(ext < 9.2e18f)) overflow = 1;
    else d[c] = (int64_t)ext + 1;
  }
  if (!overflow) overflow = (int64_t)((uint64_t)d[0] * (uint64_t)d[1] * (uint64_t)d[2]) > (int64_t)INT32_MAX;
  *unfiltered = overflow;
  int64_t m = 0;
  if (overflow) { /* output = *input_ */
    for (int64_t i = 0; i < n; i++) {
      if (keep_by_norm(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2])) {
        for (int c = 0; c < 3; c++) out[3 * m + c] = xyz[3 * i + c];
        m++;
      }
    }
    return m;
  }
  int min_b[3], div_b[3];
  for (int c = 0; c < 3; c++) {
    min_b[c] = f2i_x86(floorf(min_p[c] * inv));
    const int max_b = f2i_x86(floorf(max_p[c] * inv));
    div_b[c] = (int)((unsigned int)max_b - (unsigned int)min_b[c] + 1u);
  }
  const unsigned int mul1 = (unsigned int)div_b[0], mul2 = (unsigned int)div_b[0] * (unsigned int)div_b[1];
  keyed* v = (keyed*)malloc(sizeof(keyed) * (n ? n : 1));
  for (int64_t i = 0; i < n; i++) {
    unsigned int ijk[3];
    for (int c = 0; c < 3; c++) ijk[c] = (unsigned int)f2i_x86(floorf(xyz[3 * i + c] * inv) - (float)min_b[c]);
    v[i].key = ijk[0] + ijk[1] * mul1 + ijk[2] * mul2;
    v[i].index = i;
  }
  qsort(v, (size_t)n, sizeof(keyed), cmp_keyed);
  for (int64_t s = 0; s < n;) {
    int64_t e = s + 1;
    while (e < n && v[e].key == v[s].key) e++;
    float sum[3] = {0.0f, 0.0f, 0.0f};
    for (int64_t k = s; k < e; k++)
      for (int c = 0; c < 3; c++) sum[c] += xyz[3 * v[k].index + c];
    const float cnt = (float)(e - s);
    const float cx = sum[0] / cnt, cy = sum[1] / cnt, cz = sum[2] / cnt;
    if (keep_by_norm(cx, cy, cz)) {
      out[3 * m] = cx;
      out[3 * m + 1] = cy;
      out[3 * m + 2] = cz;
      m++;
    }
    s = e;
  }
  free(v);
  return m;
}

typedef struct {
  double value;
  int64_t index;
} ranked;

static int cmp_ranked(const void* a, const void* b) {
  const ranked* x = (const ranked*)a;
  const ranked* y = (const ranked*)b;
  if (x->value < y->value) return -1;
  if (y->value < x->value) return 1;
  return (x->index > y->index) - (x->index < y->index);
}

void orc_rank_equalize(const float* intensities, int64_t n, double* out) {
  ranked* r = (ranked*)malloc(sizeof(ranked) * (n ? n : 1));
  for (int64_t i = 0; i < n; i++) {
    r[i].value = (double)intensities[i];
    r[i].index = i;
  }
  qsort(r, (size_t)n, sizeof(ranked), cmp_ranked);
  const int bins = 256;
  for (int64_t i = 0; i < n; i++) out[r[i].index] = floor(bins * (double)i / (double)n) / bins;
  free(r);
}

double orc_min_bearing_cosine(const float* xyz, int64_t n) {
  double* dirs = (double*)malloc(sizeof(double) * 3 * (n ? n : 1));
  for (int64_t i = 0; i < n; i++) {
    const double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    const double n2 = (x * x + y * y) + z * z;
    if (n2 > 0.0) {
      const double nn = sqrt(n2);
      dirs[3 * i] = x / nn, dirs[3 * i + 1] = y / nn, dirs[3 * i + 2] = z / nn;
    } else {
      dirs[3 * i] = x, dirs[3 * i + 1] = y, dirs[3 * i + 2] = z;
    }
  }
  double min_cosine = M_PI;
  for (int64_t i = 0; i < n; i++) {
    for (int64_t j = i + 1; j < n; j++) {
      const double* a = dirs + 3 * i;
      const double* b = dirs + 3 * j;
      const double cosine = (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2];
      min_cosine = cosine < min_cosine ? cosine : min_cosine; /* std::min(cosine, min_cosine) */
    }
  }
  free(dirs);
  return min_cosine;
}

/* R row-major.  wide = 0: (AngleAxisd(pi/2, Y) * AngleAxisd(-pi/2, Z)).toRotationMatrix(); 1: AngleAxisd(-pi/2, X). */
void orc_virtual_lidar_rotation(int wide, double* R) {
  if (!wide) {
    const double ha1 = 0.5 * M_PI_2, s1 = sin(ha1), ha2 = 0.5 * -M_PI_2, s2 = sin(ha2);
    const double aw = cos(ha1), ax = s1 * 0.0, ay = s1 * 1.0, az = s1 * 0.0;
    const double bw = cos(ha2), bx = s2 * 0.0, by = s2 * 0.0, bz = s2 * 1.0;
    const double w = aw * bw - ax * bx - ay * by - az * bz;
    const double x = aw * bx + ax * bw + ay * bz - az * by;
    const double y = aw * by + ay * bw + az * bx - ax * bz;
    const double z = aw * bz + az * bw + ax * by - ay * bx;
    const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w;
    const double txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1.0 - (tyy + tzz), R[1] = txy - twz, R[2] = txz + twy;
    R[3] = txy + twz, R[4] = 1.0 - (txx + tzz), R[5] = tyz - twx;
    R[6] = txz - twy, R[7] = tyz + twx, R[8] = 1.0 - (txx + tyy);
  } else {
    const double angle = -M_PI_2, axis[3] = {1.0, 0.0, 0.0};
    const double c = cos(angle), s = sin(angle);
    double sin_axis[3], cos1_axis[3];
    for (int i = 0; i < 3; i++) sin_axis[i] = s * axis[i], cos1_axis[i] = (1.0 - c) * axis[i];
    double tmp = cos1_axis[0] * axis[1];
    R[1] = tmp - sin_axis[2], R[3] = tmp + sin_axis[2];
    tmp = cos1_axis[0] * axis[2];
    R[2] = tmp + sin_axis[1], R[6] = tmp - sin_axis[1];
    tmp = cos1_axis[1] * axis[2];
    R[5] = tmp - sin_axis[0], R[7] = tmp + sin_axis[0];
    for (int i = 0; i < 3; i++) R[4 * i] = cos1_axis[i] * axis[i] + c;
  }
}
