// turbo_blend.cuh -- the viewer's colouring, shared by the headless viewer (viewer.cu) and the agreement map
// (agreement.cu): turbo(x) blended over the camera's gray value as PointsColorUpdater::update blends
// (points_color_updater.cpp:54-57), in float32 with one rounding per operation (see viewer.cu).
#pragma once

#include <cstdint>

#include "turbo_colormap.hpp"

namespace vlcal {

// one copy per translation unit (the library is compiled without relocatable device code)
static __constant__ unsigned char c_turbo_rgb[768] = {VLCAL_TURBO_RGB_BYTES};

__device__ __forceinline__ int turbo_index(float intensity) {
  const double v = static_cast<double>(intensity) * 255.0;
  if (!(v > 0.0)) return 0;  // negative, zero and NaN
  return v >= 255.0 ? 255 : __double2int_rz(v);
}

// gray * w + turbo * (1 - w) per channel, alpha from 1 and 1 (points_color_updater.cpp:55-57)
__device__ __forceinline__ float4 blend_colors(uint8_t pix, float intensity, float w, float one_minus_w) {
  const float gray = __fmul_rn(__fdiv_rn(static_cast<float>(pix), 255.0f), w);
  const unsigned char* t = c_turbo_rgb + 3 * turbo_index(intensity);
  float4 c;
  c.x = __fadd_rn(gray, __fmul_rn(__fdiv_rn(static_cast<float>(t[0]), 255.0f), one_minus_w));
  c.y = __fadd_rn(gray, __fmul_rn(__fdiv_rn(static_cast<float>(t[1]), 255.0f), one_minus_w));
  c.z = __fadd_rn(gray, __fmul_rn(__fdiv_rn(static_cast<float>(t[2]), 255.0f), one_minus_w));
  c.w = __fadd_rn(w, one_minus_w);
  return c;
}

__device__ __forceinline__ uint8_t to_byte(float c) {
  return static_cast<uint8_t>(min(max(__float2int_rn(__fmul_rn(c, 255.0f)), 0), 255));
}

}  // namespace vlcal
