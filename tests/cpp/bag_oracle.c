/* bag_oracle.c -- a plain sequential restatement of preprocess's per-scan loop, the CPU checker of csrc/bag_integrate.cu
 * (built by tests/bag_oracle.py with -ffp-contract=off).
 *
 *   orc_bag_integrate  for every point of every scan in order: extract_raw_points (ros_cloud_converter.hpp:107-170; z
 *                      read with x's datatype, intensities from uint8/16/32 and float32/64), the finiteness filter
 *                      (preprocess.cpp:457), StaticPointCloudIntegrator::insert_points (norm < min_distance dropped,
 *                      voxelgrid[floor(p / voxel_resolution)] = point) and get_points (float casts).  The map keeps its
 *                      voxels in first-write order: an open-addressing table gives each voxel the slot of its first
 *                      write, and every later write to it overwrites that slot. */
#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
  int64_t byte_offset;
  int64_t n_points;
  int32_t point_step;
  int32_t x_offset, y_offset, z_offset;
  int32_t xyz_type;
  int32_t intensity_offset;
  int32_t intensity_type;
  int32_t reserved;
} scan_desc;

/* static_cast<int>(double) on x86-64 (cvttsd2si): INT_MIN out of range.  Written out so the checker has no UB. */
static int d2i_x86(double d) { return (d >= -2147483648.0 && d < 2147483648.0) ? (int)d : INT_MIN; }

static double rd_coord(const unsigned char* p, int type) {
  if (type == 7) {
    float f;
    memcpy(&f, p, 4);
    return (double)f;
  }
  double d;
  memcpy(&d, p, 8);
  return d;
}

static double rd_intensity(const unsigned char* p, int type) {
  switch (type) {
    case 2: return (double)p[0];
    case 4: { uint16_t v; memcpy(&v, p, 2); return (double)v; }
    case 6: { uint32_t v; memcpy(&v, p, 4); return (double)v; }
    case 7: { float v; memcpy(&v, p, 4); return (double)v; }
    default: { double v; memcpy(&v, p, 8); return v; }
  }
}

/* Extracted fields of one scan, before any filter: (x, y, z, intensity) as doubles, n x 4. */
void orc_extract_scan(const unsigned char* data, const scan_desc* s, double* out) {
  for (int64_t i = 0; i < s->n_points; i++) {
    const unsigned char* p = data + s->byte_offset + (int64_t)s->point_step * i;
    out[4 * i] = rd_coord(p + s->x_offset, s->xyz_type);
    out[4 * i + 1] = rd_coord(p + s->y_offset, s->xyz_type);
    out[4 * i + 2] = rd_coord(p + s->z_offset, s->xyz_type);
    out[4 * i + 3] = rd_intensity(p + s->intensity_offset, s->intensity_type);
  }
}

static uint64_t mix(int ix, int iy, int iz) {
  uint64_t h = (uint64_t)(uint32_t)ix * 0x9E3779B97F4A7C15ull;
  h ^= (uint64_t)(uint32_t)iy * 0xC2B2AE3D27D4EB4Full + (h >> 29);
  h ^= (uint64_t)(uint32_t)iz * 0x165667B19E3779F9ull + (h >> 31);
  return h ^ (h >> 32);
}

/* -> number of voxels; out: room for 4 floats per input point.  *out_of_range counts the kept points with an axis index
 * outside int range.  Returns -1 if the table cannot be allocated. */
int64_t orc_bag_integrate(const unsigned char* data, const scan_desc* scans, int64_t n_scans, double res, double min_distance, float* out,
                          int64_t* out_of_range) {
  int64_t total = 0;
  for (int64_t s = 0; s < n_scans; s++) total += scans[s].n_points;
  uint64_t cap = 16;
  while (cap < 2 * (uint64_t)total) cap <<= 1;
  int64_t* table = malloc(sizeof(int64_t) * cap); /* slot + 1, 0 = empty */
  int* keys = malloc(sizeof(int) * 3 * (total ? total : 1));
  if (!table || !keys) {
    free(table);
    free(keys);
    return -1;
  }
  memset(table, 0, sizeof(int64_t) * cap);
  int64_t n_vox = 0, oor = 0;
  for (int64_t s = 0; s < n_scans; s++) {
    const scan_desc* d = &scans[s];
    for (int64_t i = 0; i < d->n_points; i++) {
      const unsigned char* p = data + d->byte_offset + (int64_t)d->point_step * i;
      const double x = rd_coord(p + d->x_offset, d->xyz_type), y = rd_coord(p + d->y_offset, d->xyz_type), z = rd_coord(p + d->z_offset, d->xyz_type);
      const double w = rd_intensity(p + d->intensity_offset, d->intensity_type);
      if (!(isfinite(x) && isfinite(y) && isfinite(z))) continue;
      if (sqrt((x * x + y * y) + z * z) < min_distance) continue;
      const double fx = floor(x / res), fy = floor(y / res), fz = floor(z / res);
      const int ix = d2i_x86(fx), iy = d2i_x86(fy), iz = d2i_x86(fz);
      if ((ix == INT_MIN && fx != -2147483648.0) || (iy == INT_MIN && fy != -2147483648.0) || (iz == INT_MIN && fz != -2147483648.0)) oor++;
      uint64_t h = mix(ix, iy, iz) & (cap - 1);
      int64_t slot;
      for (;;) {
        if (!table[h]) {
          slot = n_vox++;
          table[h] = slot + 1;
          keys[3 * slot] = ix, keys[3 * slot + 1] = iy, keys[3 * slot + 2] = iz;
          break;
        }
        slot = table[h] - 1;
        if (keys[3 * slot] == ix && keys[3 * slot + 1] == iy && keys[3 * slot + 2] == iz) break;
        h = (h + 1) & (cap - 1);
      }
      out[4 * slot] = (float)x;
      out[4 * slot + 1] = (float)y;
      out[4 * slot + 2] = (float)z;
      out[4 * slot + 3] = (float)w;
    }
  }
  free(table);
  free(keys);
  if (out_of_range) *out_of_range = oor;
  return n_vox;
}
