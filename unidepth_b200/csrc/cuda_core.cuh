// Device helpers shared by the CUDA-core kernels of elementwise.cu and v1_kernels.cu: warp reductions, ATen's resampling
// index and weight rules, the back-projection of UniDepthV1 / UniDepthV2old and the camera-head decode.  One copy of
// each rule, so that a fix reaches every model.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace udb {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// reflect padding (torch "reflect", edge not repeated) of index i into [0, n)
__device__ __forceinline__ int reflect_idx(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i); }

// The two taps and weights of ATen's bilinear resampling at source coordinate src >= 0: i0 = floor(src) (clamped to the
// input), i1 = i0 + 1 unless i0 is the last row, l1 = src - i0, l0 = 1 - l1.
__device__ __forceinline__ void bilinear_taps(float src, int in_size, int& i0, int& i1, float& l0, float& l1) {
  i0 = (int)src;
  if (i0 > in_size - 1) i0 = in_size - 1;
  i1 = i0 + ((i0 < in_size - 1) ? 1 : 0);
  l1 = src - (float)i0;
  l0 = 1.f - l1;
}
__device__ __forceinline__ void bilinear_src(float scale, int dst, int in_size, int& i0, int& i1, float& l0, float& l1) {
  // ATen area_pixel_compute_source_index (align_corners=False): fp32 index arithmetic
  float src = scale * ((float)dst + 0.5f) - 0.5f;
  if (src < 0.f) src = 0.f;
  bilinear_taps(src, in_size, i0, i1, l0, l1);
}

// ------------------------------------------------------------------------------------------------------------------
// Antialiased bilinear weights of ONE axis, exactly ATen's _compute_indices_min_size_weights_aa (UpSampleKernel.cpp;
// F.interpolate(mode="bilinear", align_corners=False, antialias=True)): triangle filter of half-width
// max(scale, 1) around scale*(i+0.5), window clipped to the input, weights renormalised.
// Taps j = 0 .. xsize-1 read input xmin + j.  tri(j, s) = tri((j + xmin - center + 0.5) * invscale) * s; the normalised
// weight w(j) is tri(j, norm) with norm = 1 / sum, sum the total of tri(j, 1.f) over the window.
// ------------------------------------------------------------------------------------------------------------------
struct AAxis {
  int xmin, xsize;
  float center, invscale, sum, norm;
  __device__ __forceinline__ float tri(int j, float s) const {
    const float x = fabsf(((float)(j + xmin) - center + 0.5f) * invscale);
    return x < 1.f ? (1.f - x) * s : 0.f;
  }
  __device__ __forceinline__ float w(int j) const { return tri(j, norm); }
};
__device__ __forceinline__ AAxis aa_axis(int i, int in_size, float scale) {
  AAxis a;
  const float support = scale >= 1.f ? scale : 1.f;
  a.center = scale * ((float)i + 0.5f);
  a.invscale = scale >= 1.f ? 1.f / scale : 1.f;
  a.xmin = max((int)(a.center - support + 0.5f), 0);
  a.xsize = min((int)(a.center + support + 0.5f), in_size) - a.xmin;
  a.sum = 0.f;
  for (int j = 0; j < a.xsize; ++j) a.sum += a.tri(j, 1.f);
  a.norm = a.sum != 0.f ? 1.f / a.sum : 1.f;
  return a;
}

// One output pixel of an antialiased bilinear resize of the row-major map m (row length ld) from the axes' weights.
__device__ __forceinline__ float aa_sample(const float* __restrict__ m, const AAxis& ay, const AAxis& ax, int ld) {
  float v = 0.f;
  for (int jy = 0; jy < ay.xsize; ++jy) {
    float r = 0.f;
    for (int jx = 0; jx < ax.xsize; ++jx) r += ax.w(jx) * m[(long long)(ay.xmin + jy) * ld + ax.xmin + jx];
    v += ay.w(jy) * r;
  }
  return v;
}

// Points of UniDepthV1 / UniDepthV2old: z * (tan(theta), 1 / tan(phi) / cos(theta), 1) with (theta, phi) of the unit
// ray through pixel (X, Y) of k4 = (fx, fy, cx, cy) (spherical_zbuffer_to_euclidean, geometric.py:57-73), written to
// pts[0], pts[plane] and pts[2 * plane].
__device__ __forceinline__ void backproject(const float* k4, int X, int Y, float z, float* pts, long long plane) {
  const float dx = ((float)X + 0.5f - k4[2]) / k4[0], dy = ((float)Y + 0.5f - k4[3]) / k4[1];
  const float inv = 1.0f / fmaxf(sqrtf(dx * dx + dy * dy + 1.0f), 1e-12f);
  const float rx = dx * inv, ry = dy * inv, rz = inv;
  const float theta = atan2f(rx, rz), phi = acosf(ry);
  pts[0] = z * tanf(theta);
  pts[plane] = z / tanf(phi) / cosf(theta);
  pts[2 * plane] = z;
}

// Camera-head decode of x = (log fx', log fy', logit cx', logit cy'): (fx, fy, cx, cy) = (s exp, s exp, sigmoid * net_w,
// sigmoid * net_h), with the focal scale s of the model.
__device__ __forceinline__ float4 decode_camera(const float* x, float s, int net_h, int net_w) {
  return make_float4(s * expf(x[0]), s * expf(x[1]), (1.f / (1.f + expf(-x[2]))) * (float)net_w,
                     (1.f / (1.f + expf(-x[3]))) * (float)net_h);
}

// the row-major 3x3 pinhole K [[fx, 0, cx], [0, fy, cy], [0, 0, 1]]
__device__ __forceinline__ void store_k3(float* k, float fx, float fy, float cx, float cy) {
  k[0] = fx; k[1] = 0.f; k[2] = cx; k[3] = 0.f; k[4] = fy; k[5] = cy; k[6] = 0.f; k[7] = 0.f; k[8] = 1.f;
}

}  // namespace udb
