// GT-camera rays (udb_camera_rays, include/udb.h): the unit rays of a camera model at the pixel centres of the network
// input, for infer(rgb, camera=<Camera object>) (reference unidepthv2.py:267-303,361-362; utils/camera.py).  The camera
// arrives in input-image pixels; the kernel applies the class's own crop(-paddings) and resize(factor) rules and then
// its unproject + get_rays arithmetic, op for op as unidepth_b200/camera.py evaluates it in fp32 torch.  Every
// multiply / add is rounded on its own (__f*_rn: no FMA contraction) so the closed forms round like torch's eager ops.
#include "common.h"

namespace udb {

__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float dvd(float a, float b) { return __fdiv_rn(a, b); }

// Camera.crop(left = -pad_l, top = -pad_t, ...) then Camera.resize(factor), on one packed row (camera.py:188-198,
// Spherical :364-380).  For Pinhole the row is K row-major and the same edits apply to K (skew included).
template <int MODEL>
__device__ __forceinline__ void crop_resize(float (&q)[16], float pl, float pr, float pt, float pb, float factor) {
  if constexpr (MODEL == UDB_CAM_PINHOLE) {
    q[2] = add(q[2], pl);
    q[5] = add(q[5], pt);
#pragma unroll
    for (int i = 0; i < 6; ++i) q[i] = mul(q[i], factor);
  } else if constexpr (MODEL == UDB_CAM_SPHERICAL) {
    q[2] = add(q[2], pl);
    q[3] = add(q[3], pt);
    const float W = q[4], H = q[5];
    const float keep_w = dvd(add(add(W, pl), pr), W), keep_h = dvd(add(add(H, pt), pb), H);
    q[4] = add(W, pl + pr);          // pl + pr: exact small integers
    q[5] = add(H, pt + pb);
    q[6] = mul(q[6], keep_w);
    q[7] = mul(q[7], keep_h);
#pragma unroll
    for (int i = 0; i < 6; ++i) q[i] = mul(q[i], factor);   // the image size scales, the angular extent does not
  } else {
    q[2] = add(q[2], pl);
    q[3] = add(q[3], pt);
#pragma unroll
    for (int i = 0; i < 4; ++i) q[i] = mul(q[i], factor);
  }
}

// _tan_prism + its Jacobian (camera.py:85-108) inside _undo_tan_prism's Newton loop (:111-119)
__device__ __forceinline__ void undo_tan_prism(float& x, float& y, float p0, float p1, bool prism, float s0, float s1,
                                               float s2, float s3, int iters) {
  const float tx = x, ty = y;
  for (int it = 0; it < iters; ++it) {
    const float r2 = add(mul(x, x), mul(y, y));
    const float xy2 = mul(mul(2.f, x), y);
    float dx = add(add(x, mul(add(mul(mul(2.f, x), x), r2), p0)), mul(xy2, p1));
    float dy = add(add(y, mul(add(mul(mul(2.f, y), y), r2), p1)), mul(xy2, p0));
    float j00 = add(add(1.f, mul(mul(6.f, x), p0)), mul(mul(2.f, y), p1));
    const float off = mul(2.f, add(mul(x, p1), mul(y, p0)));
    float j01 = off, j10 = off;
    float j11 = add(add(1.f, mul(mul(6.f, y), p1)), mul(mul(2.f, x), p0));
    if (prism) {
      dx = add(dx, add(mul(s0, r2), mul(mul(s1, r2), r2)));
      dy = add(dy, add(mul(s2, r2), mul(mul(s3, r2), r2)));
      const float t1 = mul(2.f, add(s0, mul(mul(2.f, s1), r2)));
      const float t2 = mul(2.f, add(s2, mul(mul(2.f, s3), r2)));
      j00 = add(j00, mul(x, t1));
      j01 = add(j01, mul(y, t1));
      j10 = add(j10, mul(x, t2));
      j11 = add(j11, mul(y, t2));
    }
    const float ex = sub(tx, dx), ey = sub(ty, dy);
    const float det = sub(mul(j00, j11), mul(j01, j10));
    x = add(x, dvd(sub(mul(j11, ex), mul(j01, ey)), det));
    y = add(y, dvd(sub(mul(j00, ey), mul(j10, ex)), det));
  }
}

// _undo_radial (camera.py:122-137): t (1 + sum_i c_i t^(2i+2)) = rd, 25 Newton steps clamped to +-0.25 and t >= 0
template <int N>
__device__ __forceinline__ float undo_radial(float rd, const float* c) {
  float t = rd;
  for (int it = 0; it < 25; ++it) {
    const float t2 = mul(t, t);
    float pw = t2, s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      if (i) pw = mul(pw, t2);
      const float pc = mul(pw, c[i]);
      s1 = add(s1, pc);
      s2 = add(s2, mul(pc, 2.f * i + 3.f));
    }
    const float f = sub(mul(t, add(1.f, s1)), rd);
    float df = add(1.f, s2);
    if (fabsf(df) < 1e-6f) df = 1e-6f;
    const float step = fminf(fmaxf(dvd(f, df), -0.25f), 0.25f);
    t = fmaxf(sub(t, step), 0.f);
  }
  return t;
}

// grid (x: pixel chunks, y: image); one camera row per image, prepared once per thread, then a grid-stride loop over the
// pixels of that image.  rays [B, net_h*net_w, 3].
template <int MODEL>
__global__ void __launch_bounds__(256) camera_rays_kernel(const float* __restrict__ params, int net_h, int net_w, float pl,
                                                          float pr, float pt, float pb, float factor, float* __restrict__ rays) {
  const int b = blockIdx.y;
  const float* row = params + static_cast<size_t>(b) * UDB_CAM_STRIDE;
  float q[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) q[i] = row[i];
  const bool use_radial = row[16] != 0.f, use_tangential = row[17] != 0.f, use_prism = row[18] != 0.f;
  crop_resize<MODEL>(q, pl, pr, pt, pb, factor);
  float inv[9];
  if (MODEL == UDB_CAM_PINHOLE) {   // torch.inverse(K) of Pinhole.unproject (camera.py:313-319), by the adjugate
    const float c0 = q[4] * q[8] - q[5] * q[7], c1 = q[5] * q[6] - q[3] * q[8], c2 = q[3] * q[7] - q[4] * q[6];
    const float rdet = 1.f / (q[0] * c0 + q[1] * c1 + q[2] * c2);
    inv[0] = c0 * rdet; inv[1] = (q[2] * q[7] - q[1] * q[8]) * rdet; inv[2] = (q[1] * q[5] - q[2] * q[4]) * rdet;
    inv[3] = c1 * rdet; inv[4] = (q[0] * q[8] - q[2] * q[6]) * rdet; inv[5] = (q[2] * q[3] - q[0] * q[5]) * rdet;
    inv[6] = c2 * rdet; inv[7] = (q[1] * q[6] - q[0] * q[7]) * rdet; inv[8] = (q[0] * q[4] - q[1] * q[3]) * rdet;
  }
  const int hw = net_h * net_w;
  float* out = rays + static_cast<size_t>(b) * hw * 3;
  for (int px = blockIdx.x * blockDim.x + threadIdx.x; px < hw; px += gridDim.x * blockDim.x) {
    const float u = static_cast<float>(px % net_w) + 0.5f, v = static_cast<float>(px / net_w) + 0.5f;   // pixel_grid
    float rx, ry, rz;
    if (MODEL == UDB_CAM_PINHOLE) {
      const float x = inv[0] * u + inv[1] * v + inv[2];
      const float y = inv[3] * u + inv[4] * v + inv[5];
      const float z = inv[6] * u + inv[7] * v + inv[8];
      const float zc = fmaxf(z, 1e-4f);
      rx = dvd(x, zc); ry = dvd(y, zc); rz = dvd(z, zc);
    } else if (MODEL == UDB_CAM_EUCM) {   // EUCM.unproject (camera.py:344-355)
      const float alpha = q[4], beta = q[5];
      const float mx = dvd(sub(u, q[2]), q[0]), my = dvd(sub(v, q[3]), q[1]);
      const float r2 = add(mul(mx, mx), mul(my, my));
      const float root = sqrtf(fmaxf(sub(1.f, mul(mul(sub(mul(2.f, alpha), 1.f), beta), r2)), 1e-5f));
      const float mz = dvd(sub(1.f, mul(mul(mul(beta, alpha), alpha), r2)), add(mul(alpha, root), sub(1.f, alpha)));
      const float inv_n = dvd(1.f, sqrtf(add(add(r2, mul(mz, mz)), 1e-5f)));
      rx = mul(inv_n, mx); ry = mul(inv_n, my); rz = fmaxf(mul(inv_n, mz), 1e-3f);
    } else if (MODEL == UDB_CAM_SPHERICAL) {   // Spherical.unproject (camera.py:395-400)
      const float w1 = sub(q[4], 1.f), h1 = sub(q[5], 1.f);
      const float lon = mul(dvd(sub(u, dvd(w1, 2.f)), w1), mul(2.f, q[6]));
      const float lat = mul(dvd(sub(v, dvd(h1, 2.f)), h1), mul(2.f, q[7]));
      const float cl = cosf(lat);
      rx = mul(cl, sinf(lon)); ry = sinf(lat); rz = mul(cl, cosf(lon));
      const float n = fmaxf(sqrtf(add(add(mul(rx, rx), mul(ry, ry)), mul(rz, rz))), 1e-5f);
      rx = dvd(rx, n); ry = dvd(ry, n); rz = dvd(rz, n);
    } else if (MODEL == UDB_CAM_OPENCV || MODEL == UDB_CAM_FISHEYE624) {   // _Distorted._start_unproject + unproject
      float x = dvd(sub(u, q[2]), q[0]), y = dvd(sub(v, q[3]), q[1]);
      if (use_tangential || use_prism) undo_tan_prism(x, y, q[10], q[11], use_prism, q[12], q[13], q[14], q[15], 10);
      const float rd = sqrtf(add(mul(x, x), mul(y, y)));
      float scale = 1.f;
      if (MODEL == UDB_CAM_OPENCV) {       // r_d = r (1 + k1 r^2 + k2 r^4 + k3 r^6)
        const float r = use_radial ? undo_radial<3>(rd, q + 4) : rd;
        if (!(rd < 1e-6f)) scale = dvd(r, fmaxf(rd, 1e-12f));
      } else {                             // r_d = theta (1 + k1 theta^2 + ... + k6 theta^12), r = tan(theta)
        const float th = use_radial ? undo_radial<6>(rd, q + 4) : rd;
        if (!(rd < 1e-6f)) scale = dvd(tanf(th), fmaxf(rd, 1e-12f));
      }
      rx = mul(x, scale); ry = mul(y, scale); rz = 1.f;
    } else {                                 // MEI.unproject (camera.py:543-558)
      float x = dvd(sub(u, q[2]), q[0]), y = dvd(sub(v, q[3]), q[1]);
      if (use_tangential) undo_tan_prism(x, y, q[6], q[7], false, 0.f, 0.f, 0.f, 0.f, 20);
      const float rd = sqrtf(add(mul(x, x), mul(y, y)));
      const float r = use_radial ? undo_radial<2>(rd, q + 4) : rd;
      const float scale = rd < 1e-6f ? 1.f : dvd(r, fmaxf(rd, 1e-12f));
      rx = mul(x, scale); ry = mul(y, scale);
      const float xi = q[8];
      const float rho2 = add(mul(rx, rx), mul(ry, ry));
      if (xi == 1.f) {
        rz = dvd(sub(1.f, rho2), 2.f);
      } else {
        const float den = add(xi, sqrtf(add(1.f, mul(sub(1.f, mul(xi, xi)), rho2))));
        rz = sub(1.f, dvd(mul(xi, add(rho2, 1.f)), den));
      }
    }
    // get_rays: rays / |rays|.clamp(min=1e-4)  (camera.py:171-175)
    const float n = fmaxf(sqrtf(add(add(mul(rx, rx), mul(ry, ry)), mul(rz, rz))), 1e-4f);
    float* o = out + static_cast<size_t>(px) * 3;
    o[0] = dvd(rx, n);
    o[1] = dvd(ry, n);
    o[2] = dvd(rz, n);
  }
}

}  // namespace udb

using namespace udb;

extern "C" int udb_camera_rays(int32_t model, const float* params, int32_t B, int32_t net_h, int32_t net_w, int32_t pad_l,
                               int32_t pad_r, int32_t pad_t, int32_t pad_b, float factor, float* rays, void* stream) {
  if (model < UDB_CAM_PINHOLE || model > UDB_CAM_MEI) {
    set_error("udb_camera_rays: `model` %d is not a UDB_CAM_* camera model (1..6)", model);
    return 1;
  }
  if (B < 1 || B > 65535) { set_error("udb_camera_rays: B=%d must be in [1, 65535]", B); return 1; }
  if (net_h < 1 || net_w < 1) { set_error("udb_camera_rays: net_h=%d, net_w=%d must be >= 1", net_h, net_w); return 1; }
  if (static_cast<long long>(net_h) * net_w > (1ll << 30)) { set_error("udb_camera_rays: net_h * net_w exceeds 2^30"); return 1; }
  if (!params) { set_error("udb_camera_rays: `params` is null"); return 1; }
  if (reinterpret_cast<uintptr_t>(params) & 15) { set_error("udb_camera_rays: `params` must be 16-byte aligned"); return 1; }
  if (!rays) { set_error("udb_camera_rays: `rays` is null"); return 1; }
  if (reinterpret_cast<uintptr_t>(rays) & 3) { set_error("udb_camera_rays: `rays` must be 4-byte aligned"); return 1; }
  const long long hw = static_cast<long long>(net_h) * net_w;
  // a few pixels per thread so the per-image camera preparation is amortised, and still >= 8 blocks per SM overall
  long long gx = (hw + 255) / 256;
  const long long cap = (8ll * num_sms() + B - 1) / B;
  if (gx > cap) gx = cap;
  const dim3 grid(static_cast<unsigned>(gx), static_cast<unsigned>(B));
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  const float fl = static_cast<float>(pad_l), fr = static_cast<float>(pad_r), ft = static_cast<float>(pad_t),
              fb = static_cast<float>(pad_b);
  note_work(0.0, 12.0 * B * hw + 4.0 * B * UDB_CAM_STRIDE);
  switch (model) {
    case UDB_CAM_PINHOLE: camera_rays_kernel<UDB_CAM_PINHOLE><<<grid, 256, 0, st>>>(params, net_h, net_w, fl, fr, ft, fb, factor, rays); break;
    case UDB_CAM_EUCM: camera_rays_kernel<UDB_CAM_EUCM><<<grid, 256, 0, st>>>(params, net_h, net_w, fl, fr, ft, fb, factor, rays); break;
    case UDB_CAM_SPHERICAL: camera_rays_kernel<UDB_CAM_SPHERICAL><<<grid, 256, 0, st>>>(params, net_h, net_w, fl, fr, ft, fb, factor, rays); break;
    case UDB_CAM_OPENCV: camera_rays_kernel<UDB_CAM_OPENCV><<<grid, 256, 0, st>>>(params, net_h, net_w, fl, fr, ft, fb, factor, rays); break;
    case UDB_CAM_FISHEYE624: camera_rays_kernel<UDB_CAM_FISHEYE624><<<grid, 256, 0, st>>>(params, net_h, net_w, fl, fr, ft, fb, factor, rays); break;
    default: camera_rays_kernel<UDB_CAM_MEI><<<grid, 256, 0, st>>>(params, net_h, net_w, fl, fr, ft, fb, factor, rays); break;
  }
  return check_launch("camera_rays_kernel");
}
