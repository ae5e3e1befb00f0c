// HBM-bound / latency-bound kernels of the UniDepthV2.infer() path: LayerNorm, preprocessing +
// patch extraction, position-embedding resize, the fp32 camera head, ray embedding, bilinear
// resamplers and the output assembly.  Reference call sites are cited in include/udb.h.
#include "common.h"
#include "ptx.cuh"

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

// ------------------------------------------------------------------------------------ LayerNorm
// One warp per R rows (R = 1 by default; the R = 2 variant -- both rows' loads in flight before the first
// reduction -- measured slower, see udb_layernorm); dim % 128 == 0, dim <= 1024; lane owns float4
// #(lane + 32*i).
template <bool IN_F32, bool OUT_F32, int R>
__global__ void __launch_bounds__(256) layernorm_kernel(const udb_layernorm_t p) {
  const int row0 = (blockIdx.x * 8 + (threadIdx.x >> 5)) * R;
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();
  pdl_wait();
  if (row0 >= p.rows) return;
  const int nvec = p.dim >> 7;  // float4 per lane
  float4 x[R][8];
  float s[R];
  bool live[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int row = row0 + r;
    live[r] = row < p.rows;
    long long irow = live[r] ? row : row0;
    if (p.rows_per_group > 0)
      irow = (long long)(irow / p.rows_per_group) * p.group_stride + (irow % p.rows_per_group) + p.row_offset;
    s[r] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i < nvec) {
        const int e = (lane + 32 * i) * 4;
        if (IN_F32) {
          x[r][i] = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.in) + irow * p.ld_in + e);
        } else {
          const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(p.in) + irow * p.ld_in + e);
          const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
          const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
          x[r][i] = make_float4(a.x, a.y, b.x, b.y);
        }
      }
    }
  }
  float mean[R], rstd[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (i < nvec) s[r] += (x[r][i].x + x[r][i].y) + (x[r][i].z + x[r][i].w);
    mean[r] = warp_sum(s[r]) / (float)p.dim;
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i < nvec) {
        const float a = x[r][i].x - mean[r], b = x[r][i].y - mean[r], c = x[r][i].z - mean[r], d = x[r][i].w - mean[r];
        v += (a * a + b * b) + (c * c + d * d);
      }
    }
    rstd[r] = rsqrtf(warp_sum(v) / (float)p.dim + p.eps);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (i < nvec) {
      const int e = (lane + 32 * i) * 4;
      const float4 w = __ldg(reinterpret_cast<const float4*>(p.weight + e));
      const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + e));
#pragma unroll
      for (int r = 0; r < R; ++r) {
        if (!live[r]) continue;
        const float y0 = (x[r][i].x - mean[r]) * rstd[r] * w.x + b.x;
        const float y1 = (x[r][i].y - mean[r]) * rstd[r] * w.y + b.y;
        const float y2 = (x[r][i].z - mean[r]) * rstd[r] * w.z + b.z;
        const float y3 = (x[r][i].w - mean[r]) * rstd[r] * w.w + b.w;
        if (OUT_F32) {
          *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + (long long)(row0 + r) * p.ld_out + e) =
              make_float4(y0, y1, y2, y3);
        } else {
          __half* op = reinterpret_cast<__half*>(p.out) + (long long)(row0 + r) * p.ld_out + e;
          const uint2 hi = make_uint2(pack_half2(y0, y1), pack_half2(y2, y3));
          *reinterpret_cast<uint2*>(op) = hi;
          if (p.out_split > 0) {      // split-f16 precise mode: lo = f16(y - f32(hi)) at column + out_split
            const float2 h01 = __half22float2(*reinterpret_cast<const __half2*>(&hi.x));
            const float2 h23 = __half22float2(*reinterpret_cast<const __half2*>(&hi.y));
            *reinterpret_cast<uint2*>(op + p.out_split) = make_uint2(pack_half2(y0 - h01.x, y1 - h01.y), pack_half2(y2 - h23.x, y3 - h23.y));
          }
        }
      }
    }
  }
}

// f16 -> f16 rows of 8*LPR elements (64 / 128 / 256): LPR lanes per row, 16 bytes per lane, so a warp
// moves 512 contiguous bytes per instruction (the one-warp-per-row kernel above would move 128-256 B).
template <int LPR>
__global__ void __launch_bounds__(256) layernorm_f16_small_kernel(const udb_layernorm_t p) {
  constexpr int RPW = 32 / LPR;                       // rows per warp
  const int lane = threadIdx.x & 31;
  const long long row = ((long long)blockIdx.x * 8 + (threadIdx.x >> 5)) * RPW + lane / LPR;
  const int sub = lane % LPR;
  const bool valid = row < p.rows;
  float x[8];
  if (valid) {
    const uint4 u = *reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(p.in) + row * p.ld_in + sub * 8);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 f = __half22float2(h[q]);
      x[2 * q] = f.x;
      x[2 * q + 1] = f.y;
    }
  } else {
#pragma unroll
    for (int q = 0; q < 8; ++q) x[q] = 0.f;
  }
  // zero-padded channel rows: statistics over the first n_valid columns only (multiple of 8)
  const int n_valid = p.dim_valid > 0 ? p.dim_valid : p.dim;
  const bool in_range = sub * 8 < n_valid;
  float s = in_range ? ((x[0] + x[1]) + (x[2] + x[3])) + ((x[4] + x[5]) + (x[6] + x[7])) : 0.f;
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)n_valid;
  float v = 0.f;
#pragma unroll
  for (int q = 0; q < 8; ++q) v += (x[q] - mean) * (x[q] - mean);
  v = in_range ? v : 0.f;
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const float rstd = rsqrtf(v / (float)n_valid + p.eps);
  if (valid) {
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(p.weight + sub * 8)), w1 = __ldg(reinterpret_cast<const float4*>(p.weight + sub * 8 + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bias + sub * 8)), b1 = __ldg(reinterpret_cast<const float4*>(p.bias + sub * 8 + 4));
    const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
    const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    float y[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) y[q] = (x[q] - mean) * rstd * w[q] + b[q];
    *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.out) + row * p.ld_out + sub * 8) =
        make_uint4(pack_half2(y[0], y[1]), pack_half2(y[2], y[3]), pack_half2(y[4], y[5]), pack_half2(y[6], y[7]));
  }
}

// ------------------------------------------------------------------------------------ preprocess
__device__ __forceinline__ void bilinear_src(float scale, int dst, int in_size, int& i0, int& i1, float& l0, float& l1) {
  // ATen area_pixel_compute_source_index (align_corners=False): fp32 index arithmetic
  float src = scale * ((float)dst + 0.5f) - 0.5f;
  if (src < 0.f) src = 0.f;
  i0 = (int)src;
  if (i0 > in_size - 1) i0 = in_size - 1;
  i1 = i0 + ((i0 < in_size - 1) ? 1 : 0);
  l1 = src - (float)i0;
  l0 = 1.f - l1;
}

// One thread per 8 consecutive patch-matrix columns (one 16-byte store).  `split`: the row holds [hi | lo] halves of
// ldp/2 columns each, lo = f16(val - f32(hi)) (split-f16 precise mode, see udb_gemm_t.a_split_k).
__global__ void __launch_bounds__(256) preprocess_patchify_kernel(const udb_preprocess_t p, int gh, int gw, float sh, float sw) {
  const int vec_per_row = p.ldp >> 3;
  const long long total = (long long)p.B * gh * gw * vec_per_row;
  const float mean[3] = {0.485f, 0.456f, 0.406f};
  const float stdv[3] = {0.229f, 0.224f, 0.225f};
  const int padded_h = p.H + p.pad_t + p.pad_b, padded_w = p.W + p.pad_l + p.pad_r;
  const int half_w = p.split ? (p.ldp >> 1) : p.ldp;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int col_store = (int)(idx % vec_per_row) * 8;
    const long long rowi = idx / vec_per_row;
    const bool lo_half = col_store >= half_w;
    const int col0 = lo_half ? col_store - half_w : col_store;
    const int gx = (int)(rowi % gw), gy = (int)((rowi / gw) % gh), b = (int)(rowi / ((long long)gw * gh));
    float val[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = col0 + j;
      float v = 0.f;
      if (col < 588) {
        const int c = col / 196, py = (col % 196) / 14, px = col % 14;
        const int Y = gy * 14 + py, X = gx * 14 + px;
        int y0, y1, x0, x1;
        float ly0, ly1, lx0, lx1;
        bilinear_src(sh, Y, padded_h, y0, y1, ly0, ly1);
        bilinear_src(sw, X, padded_w, x0, x1, lx0, lx1);
        auto fetch = [&](int yy, int xx) -> float {
          const int oy = yy - p.pad_t, ox = xx - p.pad_l;
          if (oy < 0 || oy >= p.H || ox < 0 || ox >= p.W) return 0.f;
          const long long o = (((long long)b * 3 + c) * p.H + oy) * p.W + ox;
          float t = p.rgb_is_u8 ? (float)__ldg(reinterpret_cast<const uint8_t*>(p.rgb) + o)
                                : __ldg(reinterpret_cast<const float*>(p.rgb) + o);
          if (p.normalize) t = (t / 255.0f - mean[c]) / stdv[c];
          return t;
        };
        v = ly0 * (lx0 * fetch(y0, x0) + lx1 * fetch(y0, x1)) + ly1 * (lx0 * fetch(y1, x0) + lx1 * fetch(y1, x1));
      }
      if (lo_half) v -= __half2float(__float2half_rn(v));
      val[j] = v;
    }
    uint4 o4 = make_uint4(pack_half2(val[0], val[1]), pack_half2(val[2], val[3]), pack_half2(val[4], val[5]), pack_half2(val[6], val[7]));
    *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.patches) + rowi * p.ldp + col_store) = o4;
  }
}

// ------------------------------------------------------------------------------------ pos-embed bicubic
__device__ __forceinline__ float cubic1(float x, float A) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic2(float x, float A) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }

__global__ void __launch_bounds__(256) posembed_bicubic_kernel(const float* __restrict__ grid, int m, int dim,
                                                               float* __restrict__ out, int gh, int gw) {
  const float A = -0.75f;
  const float sy = (float)m / (float)gh, sx = (float)m / (float)gw;
  const long long total = (long long)gh * gw * dim;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(idx % dim);
    const int j = (int)((idx / dim) % gw);
    const int i = (int)(idx / ((long long)dim * gw));
    const float ry = sy * ((float)i + 0.5f) - 0.5f, rx = sx * ((float)j + 0.5f) - 0.5f;
    const float fy = floorf(ry), fx = floorf(rx);
    const int iy = (int)fy, ix = (int)fx;
    const float ty = ry - fy, tx = rx - fx;
    const float wy[4] = {cubic2(ty + 1.f, A), cubic1(ty, A), cubic1(1.f - ty, A), cubic2(2.f - ty, A)};
    const float wx[4] = {cubic2(tx + 1.f, A), cubic1(tx, A), cubic1(1.f - tx, A), cubic2(2.f - tx, A)};
    float acc = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int yy = min(max(iy - 1 + a, 0), m - 1);
      float r = 0.f;
#pragma unroll
      for (int bq = 0; bq < 4; ++bq) {
        const int xx = min(max(ix - 1 + bq, 0), m - 1);
        r += wx[bq] * grid[((long long)yy * m + xx) * dim + d];
      }
      acc += wy[a] * r;
    }
    out[idx] = acc;
  }
}

__global__ void set_cls_rows_kernel(float* x, const float* cls, const float* pos0, int B, int T, int D) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * D) return;
  const int b = idx / D, d = idx % D;
  x[(long long)b * T * D + d] = cls[d] + pos0[d];
}

// cls rows for the fused-LayerNorm encoder: besides x (f32) also the f16 copy and the per-part {mean, centred sum of
// squares} the consumer GEMM merges (udb_gemm_t.ln_stats_in).  One block per image, warp w handles parts w, w+8, ...
__global__ void __launch_bounds__(256) set_cls_rows_ln_kernel(float* x, __half* x16, float* stats, const float* cls, const float* pos0, int T, int D,
                                                             int parts, int part_cols) {
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = (long long)b * T;
  for (int pt = warp; pt < parts; pt += 8) {
    float s = 0.f;
    for (int c = lane; c < part_cols; c += 32) {
      const int d = pt * part_cols + c;
      const float v = cls[d] + pos0[d];
      x[row * D + d] = v;
      x16[row * D + d] = __float2half_rn(v);
      s += v;
    }
    const float mean = warp_sum(s) / (float)part_cols;
    float m2 = 0.f;
    for (int c = lane; c < part_cols; c += 32) {
      const int d = pt * part_cols + c;
      const float dl = cls[d] + pos0[d] - mean;
      m2 += dl * dl;
    }
    m2 = warp_sum(m2);
    if (lane == 0) reinterpret_cast<float2*>(stats)[row * parts + pt] = make_float2(mean, m2);
  }
}

// ------------------------------------------------------------------------------------ camera head (fp32)
// one warp per output feature and 8 rows (the 32-row camera head is latency bound: favour many
// small warps over reuse); lanes stride over K with 128-bit loads when K % 128 == 0
__global__ void __launch_bounds__(128) small_linear_kernel(const udb_small_linear_t p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * 4 + warp;
  const int m0 = blockIdx.y * 8;
  if (n >= p.N) return;
  const long long ldx = p.ldx > 0 ? p.ldx : p.K, ldy = p.ldy > 0 ? p.ldy : p.N, ldr = p.ldr > 0 ? p.ldr : p.N;
  float acc[8];
#pragma unroll
  for (int m = 0; m < 8; ++m) acc[m] = 0.f;
  const float* wr = p.w + (long long)n * p.K;
  if ((p.K & 127) == 0 && (ldx & 3) == 0) {
    for (int k = lane * 4; k < p.K; k += 128) {
      const float4 wv = __ldg(reinterpret_cast<const float4*>(wr + k));
#pragma unroll
      for (int m = 0; m < 8; ++m) {
        if (m0 + m < p.M) {
          const float4 xv = *reinterpret_cast<const float4*>(p.x + (long long)(m0 + m) * ldx + k);
          acc[m] = fmaf(wv.x, xv.x, fmaf(wv.y, xv.y, fmaf(wv.z, xv.z, fmaf(wv.w, xv.w, acc[m]))));
        }
      }
    }
  } else {
    for (int k = lane; k < p.K; k += 32) {
      const float wv = wr[k];
#pragma unroll
      for (int m = 0; m < 8; ++m)
        if (m0 + m < p.M) acc[m] = fmaf(wv, p.x[(long long)(m0 + m) * ldx + k], acc[m]);
    }
  }
#pragma unroll
  for (int m = 0; m < 8; ++m) acc[m] = warp_sum(acc[m]);
  if (lane < 8 && m0 + lane < p.M) {
    float v = 0.f;
#pragma unroll
    for (int m = 0; m < 8; ++m) v = (lane == m) ? acc[m] : v;
    v += p.bias ? p.bias[n] : 0.f;
    if (p.act == UDB_ACT_GELU) v = gelu_erf(v);
    if (p.gamma) v *= p.gamma[n];
    if (p.resid) v += p.resid[(long long)(m0 + lane) * ldr + n];
    p.y[(long long)(m0 + lane) * ldy + n] = v;
  }
}

// one warp per (b, head, query token); 4 tokens
__global__ void camera_attn4_kernel(const float* q, const float* kv, const float* pos, float* out, int B, int C, int heads) {
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= B * heads * 4) return;
  const int t = gw % 4, h = (gw / 4) % heads, b = gw / (4 * heads);
  const int d = C / heads;
  const float scale = rsqrtf((float)d);
  float s[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float a = 0.f;
    for (int e = lane; e < d; e += 32) {
      const float qv = q[((long long)b * 4 + t) * C + h * d + e] + pos[t * C + h * d + e];
      a += qv * kv[((long long)b * 4 + j) * 2 * C + h * d + e];
    }
    s[j] = warp_sum(a) * scale;
  }
  const float mx = fmaxf(fmaxf(s[0], s[1]), fmaxf(s[2], s[3]));
  float den = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) { s[j] = expf(s[j] - mx); den += s[j]; }
  for (int e = lane; e < d; e += 32) {
    float a = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) a += s[j] * kv[((long long)b * 4 + j) * 2 * C + C + h * d + e];
    out[((long long)b * 4 + t) * C + h * d + e] = a / den;
  }
}

__global__ void camera_intrinsics_kernel(const float* x, int B, int net_h, int net_w, float factor, int pad_l,
                                         int pad_t, float* intr4, float* k_net, float* k_out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float diag = sqrtf((float)(net_h * net_h + net_w * net_w));
  const float fx = expf(x[b * 4 + 0]) * (0.7f * diag);
  const float fy = expf(x[b * 4 + 1]) * (0.7f * diag);
  const float cx = (1.f / (1.f + expf(-x[b * 4 + 2]))) * (float)net_w;
  const float cy = (1.f / (1.f + expf(-x[b * 4 + 3]))) * (float)net_h;
  intr4[b * 4 + 0] = fx; intr4[b * 4 + 1] = fy; intr4[b * 4 + 2] = cx; intr4[b * 4 + 3] = cy;
  float* k = k_net + b * 9;
  k[0] = fx; k[1] = 0.f; k[2] = cx; k[3] = 0.f; k[4] = fy; k[5] = cy; k[6] = 0.f; k[7] = 0.f; k[8] = 1.f;
  float* o = k_out + b * 9;
  o[0] = fx / factor; o[1] = 0.f; o[2] = cx / factor - (float)pad_l;
  o[3] = 0.f; o[4] = fy / factor; o[5] = cy / factor - (float)pad_t;
  o[6] = 0.f; o[7] = 0.f; o[8] = 1.f;
}

// ------------------------------------------------------------------------------------ rays
__device__ __forceinline__ float3 unit_ray(const float4 k /*fx,fy,cx,cy*/, int y, int x) {
  // K^-1 [u, v, 1]^T with u = x + 0.5, v = y + 0.5 (coords_grid), then L2-normalise (clamp 1e-5)
  const float rx = (1.0f / k.x) * ((float)x + 0.5f) + (-k.z / k.x);
  const float ry = (1.0f / k.y) * ((float)y + 0.5f) + (-k.w / k.y);
  const float n = fmaxf(sqrtf(rx * rx + ry * ry + 1.0f), 1e-5f);
  return make_float3(rx / n, ry / n, 1.0f / n);
}

// antialiased-bilinear tap range along one axis (ATen _upsample_bilinear2d_aa weights)
__device__ __forceinline__ void aa_range(float scale, int o, int in_size, int& lo, int& cnt, float& center) {
  const float support = (scale >= 1.f) ? scale : 1.f;
  center = scale * ((float)o + 0.5f);
  lo = max((int)(center - support + 0.5f), 0);
  cnt = min((int)(center + support + 0.5f), in_size) - lo;
}
__device__ __forceinline__ float aa_w(float scale, int k, float center) {
  const float inv = (scale >= 1.f) ? 1.f / scale : 1.f;
  return fmaxf(0.f, 1.f - fabsf(((float)k - center + 0.5f) * inv));
}

// one warp per output token
__global__ void __launch_bounds__(256) ray_embed_kernel(const udb_ray_embed_t p) {
  const int tok = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int n = p.gh * p.gw;
  if (tok >= p.B * n) return;
  const int b = tok / n, i = (tok % n) / p.gw, j = tok % p.gw;
  const float sy = (float)p.net_h / (float)p.gh, sx = (float)p.net_w / (float)p.gw;
  int ylo, ycnt, xlo, xcnt;
  float yc, xc;
  aa_range(sy, i, p.net_h, ylo, ycnt, yc);
  aa_range(sx, j, p.net_w, xlo, xcnt, xc);
  float4 k = make_float4(1.f, 1.f, 0.f, 0.f);
  if (!p.rays_in) k = *reinterpret_cast<const float4*>(p.intr4 + b * 4);
  float ax = 0.f, ay = 0.f, az = 0.f, wsum_y = 0.f, wsum_x = 0.f;
  for (int a = 0; a < ycnt; ++a) wsum_y += aa_w(sy, ylo + a, yc);
  for (int a = 0; a < xcnt; ++a) wsum_x += aa_w(sx, xlo + a, xc);
  const int taps = ycnt * xcnt;
  for (int t = lane; t < taps; t += 32) {
    const int yy = ylo + t / xcnt, xx = xlo + t % xcnt;
    const float w = (aa_w(sy, yy, yc) / wsum_y) * (aa_w(sx, xx, xc) / wsum_x);
    float3 r;
    if (p.rays_in) {
      const float* rp = p.rays_in + ((long long)b * p.net_h * p.net_w + (long long)yy * p.net_w + xx) * 3;
      r = make_float3(rp[0], rp[1], rp[2]);
    } else {
      r = unit_ray(k, yy, xx);
    }
    ax = fmaf(w, r.x, ax); ay = fmaf(w, r.y, ay); az = fmaf(w, r.z, az);
  }
  ax = warp_sum(ax); ay = warp_sum(ay); az = warp_sum(az);
  const float nrm = fmaxf(sqrtf(ax * ax + ay * ay + az * az), 1e-4f);
  ax /= nrm; ay /= nrm; az /= nrm;
  const float polar = acosf(az);
  const float xcl = fmaxf(fabsf(ax), 1e-3f) * ((ax >= 0.f) ? 1.f : -1.f);
  const float azim = atan2f(ay, xcl);
  const float pi = 3.14159265358979323846f;
  for (int f = lane; f < 2 * p.bands; f += 32) {
    const float ang = (f < p.bands) ? polar : azim;
    const float sc = __ldg(p.scales + (f % p.bands));
    const float v = sinf(ang * sc * pi);
    if (p.out_f32) reinterpret_cast<float*>(p.out)[(long long)tok * 2 * p.bands + f] = v;
    else reinterpret_cast<__half*>(p.out)[(long long)tok * 2 * p.bands + f] = __float2half_rn(v);
  }
}

// ------------------------------------------------------------------------------------ resamplers (NHWC f16, 8 ch / thread)
__device__ __forceinline__ void lerp8(const uint4& a, const uint4& b, float wa, float wb, float (&acc)[8], float scale) {
  const __half2* ha = reinterpret_cast<const __half2*>(&a);
  const __half2* hb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float2 fa = __half22float2(ha[q]), fb = __half22float2(hb[q]);
    acc[2 * q] += scale * (wa * fa.x + wb * fb.x);
    acc[2 * q + 1] += scale * (wa * fa.y + wb * fb.y);
  }
}
__device__ __forceinline__ uint4 pack8(const float (&v)[8]) {
  return make_uint4(pack_half2(v[0], v[1]), pack_half2(v[2], v[3]), pack_half2(v[4], v[5]), pack_half2(v[6], v[7]));
}

// grid: (ceil(out_w * C/8 / 256), out_h, B) -- 32-bit index math, no 64-bit div/mod per element
__global__ void __launch_bounds__(256) upsample2x_kernel(const __half* __restrict__ in, __half* __restrict__ out, int H, int W, int C) {
  const int cv = C >> 3;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= 2 * W * cv) return;
  const int X = t / cv, c8 = t - X * cv;
  const int Y = blockIdx.y, b = blockIdx.z;
  int y0, y1, x0, x1;
  float ly0, ly1, lx0, lx1;
  bilinear_src(0.5f, Y, H, y0, y1, ly0, ly1);
  bilinear_src(0.5f, X, W, x0, x1, lx0, lx1);
  const uint4* base = reinterpret_cast<const uint4*>(in) + (size_t)b * H * W * cv + c8;
  const uint4 v00 = base[(size_t)(y0 * W + x0) * cv], v01 = base[(size_t)(y0 * W + x1) * cv];
  const uint4 v10 = base[(size_t)(y1 * W + x0) * cv], v11 = base[(size_t)(y1 * W + x1) * cv];
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  lerp8(v00, v01, lx0, lx1, acc, ly0);
  lerp8(v10, v11, lx0, lx1, acc, ly1);
  reinterpret_cast<uint4*>(out)[((size_t)(b * 2 * H + Y) * 2 * W + X) * cv + c8] = pack8(acc);
}

__device__ __forceinline__ int reflect_idx(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i); }

__global__ void __launch_bounds__(256) resize_ac_pad_kernel(const __half* __restrict__ in, __half* __restrict__ out, int H, int W,
                                                            int C, int oh, int ow, int pad, float sh, float sw) {
  const int cv = C >> 3;
  const int ph = oh + 2 * pad, pw = ow + 2 * pad;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= pw * cv) return;
  const int PX = t / cv, c8 = t - PX * cv;
  const int PY = blockIdx.y, b = blockIdx.z;
  const int Y = reflect_idx(PY - pad, oh), X = reflect_idx(PX - pad, ow);
  const float fy = sh * (float)Y, fx = sw * (float)X;
  const int y0 = min((int)fy, H - 1), x0 = min((int)fx, W - 1);
  const int y1 = y0 + ((y0 < H - 1) ? 1 : 0), x1 = x0 + ((x0 < W - 1) ? 1 : 0);
  const float ly1 = fy - (float)y0, lx1 = fx - (float)x0;
  const float ly0 = 1.f - ly1, lx0 = 1.f - lx1;
  const uint4* base = reinterpret_cast<const uint4*>(in) + (size_t)b * H * W * cv + c8;
  const uint4 v00 = base[(size_t)(y0 * W + x0) * cv], v01 = base[(size_t)(y0 * W + x1) * cv];
  const uint4 v10 = base[(size_t)(y1 * W + x0) * cv], v11 = base[(size_t)(y1 * W + x1) * cv];
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  lerp8(v00, v01, lx0, lx1, acc, ly0);
  lerp8(v10, v11, lx0, lx1, acc, ly1);
  reinterpret_cast<uint4*>(out)[((size_t)(b * ph + PY) * pw + PX) * cv + c8] = pack8(acc);
}

__global__ void __launch_bounds__(256) reflect_pad1_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int H, int W, int cv) {
  const int pw = W + 2;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= pw * cv) return;
  const int PX = t / cv, c8 = t - PX * cv;
  const int PY = blockIdx.y, b = blockIdx.z;
  const int Y = reflect_idx(PY - 1, H), X = reflect_idx(PX - 1, W);
  out[((size_t)(b * (H + 2) + PY) * pw + PX) * cv + c8] = in[((size_t)(b * H + Y) * W + X) * cv + c8];
}

// border of a padded [B,H+2,W+2,C] buffer from its (already written) interior; grid: (blocks, B)
__global__ void __launch_bounds__(256) reflect_border_fill_kernel(uint4* __restrict__ buf, int H, int W, int cv) {
  const int ph = H + 2, pw = W + 2;
  const int n_border = 2 * pw + 2 * H;               // top row, bottom row, left / right columns
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= n_border * cv) return;
  const int i = t / cv, c8 = t - i * cv;
  int PY, PX;
  if (i < pw) { PY = 0; PX = i; }
  else if (i < 2 * pw) { PY = ph - 1; PX = i - pw; }
  else if (i < 2 * pw + H) { PY = i - 2 * pw + 1; PX = 0; }
  else { PY = i - 2 * pw - H + 1; PX = pw - 1; }
  const int Y = reflect_idx(PY - 1, H) + 1, X = reflect_idx(PX - 1, W) + 1;
  uint4* img = buf + (size_t)blockIdx.y * ph * pw * cv;
  img[((size_t)PY * pw + PX) * cv + c8] = img[((size_t)Y * pw + X) * cv + c8];
}

// ------------------------------------------------------------------------------------ output assembly
// radius = |points|, depth = points.z, rays / max(|rays|, 1e-5) of one resampled output pixel
__device__ __forceinline__ void store_outputs(const udb_postprocess_t& p, int b, int y, int x, float conf, float px, float py,
                                              float pz, float rx, float ry, float rz) {
  const long long plane = (long long)p.H * p.W;
  const long long pix = (long long)y * p.W + x;
  p.out_confidence[b * plane + pix] = conf;
  p.out_radius[b * plane + pix] = sqrtf(px * px + py * py + pz * pz);
  p.out_depth[b * plane + pix] = pz;
  p.out_points[(b * 3 + 0) * plane + pix] = px;
  p.out_points[(b * 3 + 1) * plane + pix] = py;
  p.out_points[(b * 3 + 2) * plane + pix] = pz;
  const float rn = fmaxf(sqrtf(rx * rx + ry * ry + rz * rz), 1e-5f);
  p.out_rays[(b * 3 + 0) * plane + pix] = rx / rn;
  p.out_rays[(b * 3 + 1) * plane + pix] = ry / rn;
  p.out_rays[(b * 3 + 2) * plane + pix] = rz / rn;
}

__global__ void __launch_bounds__(256) postprocess_kernel(const udb_postprocess_t p) {
  const long long total = (long long)p.B * p.H * p.W;
  const float sh = (float)p.net_h / (float)p.padded_h, sw = (float)p.net_w / (float)p.padded_w;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % p.W), y = (int)((idx / p.W) % p.H), b = (int)(idx / ((long long)p.W * p.H));
    int y0, y1, x0, x1;
    float ly0, ly1, lx0, lx1;
    bilinear_src(sh, y + p.pad_t, p.net_h, y0, y1, ly0, ly1);
    bilinear_src(sw, x + p.pad_l, p.net_w, x0, x1, lx0, lx1);
    float4 k = make_float4(1.f, 1.f, 0.f, 0.f);
    if (!p.rays_in) k = *reinterpret_cast<const float4*>(p.intr4 + b * 4);
    const int ys[2] = {y0, y1}, xs[2] = {x0, x1};
    const float wy[2] = {ly0, ly1}, wx[2] = {lx0, lx1};
    float conf = 0.f, px = 0.f, py = 0.f, pz = 0.f, rx = 0.f, ry = 0.f, rz = 0.f;
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      float c_r = 0.f, px_r = 0.f, py_r = 0.f, pz_r = 0.f, rx_r = 0.f, ry_r = 0.f, rz_r = 0.f;
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const long long o = ((long long)b * p.net_h + ys[a]) * p.net_w + xs[c];
        float3 r;
        if (p.rays_in) { const float* rp = p.rays_in + o * 3; r = make_float3(rp[0], rp[1], rp[2]); }
        else r = unit_ray(k, ys[a], xs[c]);
        const float rad = p.radius[o];
        c_r += wx[c] * p.confidence[o];
        px_r += wx[c] * (r.x * rad); py_r += wx[c] * (r.y * rad); pz_r += wx[c] * (r.z * rad);
        rx_r += wx[c] * r.x; ry_r += wx[c] * r.y; rz_r += wx[c] * r.z;
      }
      conf += wy[a] * c_r; px += wy[a] * px_r; py += wy[a] * py_r; pz += wy[a] * pz_r;
      rx += wy[a] * rx_r; ry += wy[a] * ry_r; rz += wy[a] * rz_r;
    }
    store_outputs(p, b, y, x, conf, px, py, pz, rx, ry, rz);
  }
}

// ATen upsample_bicubic2d (align_corners=False): source index scale*(dst+0.5)-0.5 NOT clamped at 0, x0 = floor,
// taps x0-1 .. x0+2 clamped to [0, in-1], Keys coefficients (A = -0.75) in get_cubic_upsample_coefficients' order.
__device__ __forceinline__ void bicubic_src(float scale, int dst, int in_size, int (&idx)[4], float (&w)[4]) {
  const float src = scale * ((float)dst + 0.5f) - 0.5f;
  const float f = floorf(src);
  const float t = src - f;
  const int i0 = (int)f;
#pragma unroll
  for (int k = 0; k < 4; ++k) idx[k] = min(max(i0 - 1 + k, 0), in_size - 1);
  const float A = -0.75f;
  const float t2 = 1.f - t;
  w[0] = cubic2(t + 1.f, A); w[1] = cubic1(t, A); w[2] = cubic1(t2, A); w[3] = cubic2(t2 + 1.f, A);
}

// Same fusion as postprocess_kernel (points = rays*radius per tap; confidence, points and rays resampled with the same
// weights; radius / depth / ray normalisation afterwards), bicubic weights: per output pixel, four horizontal 1-D
// interpolations of the seven channels (one per tap row), then one vertical, in the order of ATen's CUDA kernel.
// No clamping of the result: near depth edges the overshoot can make depth and confidence <= 0, as in the reference.
__global__ void __launch_bounds__(256) postprocess_bicubic_kernel(const udb_postprocess_t p) {
  const long long total = (long long)p.B * p.H * p.W;
  const float sh = (float)p.net_h / (float)p.padded_h, sw = (float)p.net_w / (float)p.padded_w;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % p.W), y = (int)((idx / p.W) % p.H), b = (int)(idx / ((long long)p.W * p.H));
    int ys[4], xs[4];
    float wy[4], wx[4];
    bicubic_src(sh, y + p.pad_t, p.net_h, ys, wy);
    bicubic_src(sw, x + p.pad_l, p.net_w, xs, wx);
    float4 k = make_float4(1.f, 1.f, 0.f, 0.f);
    if (!p.rays_in) k = *reinterpret_cast<const float4*>(p.intr4 + b * 4);
    float conf = 0.f, px = 0.f, py = 0.f, pz = 0.f, rx = 0.f, ry = 0.f, rz = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      float c_r = 0.f, px_r = 0.f, py_r = 0.f, pz_r = 0.f, rx_r = 0.f, ry_r = 0.f, rz_r = 0.f;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const long long o = ((long long)b * p.net_h + ys[a]) * p.net_w + xs[c];
        float3 r;
        if (p.rays_in) { const float* rp = p.rays_in + o * 3; r = make_float3(rp[0], rp[1], rp[2]); }
        else r = unit_ray(k, ys[a], xs[c]);
        const float rad = p.radius[o];
        c_r += p.confidence[o] * wx[c];
        px_r += (r.x * rad) * wx[c]; py_r += (r.y * rad) * wx[c]; pz_r += (r.z * rad) * wx[c];
        rx_r += r.x * wx[c]; ry_r += r.y * wx[c]; rz_r += r.z * wx[c];
      }
      conf += c_r * wy[a]; px += px_r * wy[a]; py += py_r * wy[a]; pz += pz_r * wy[a];
      rx += rx_r * wy[a]; ry += ry_r * wy[a]; rz += rz_r * wy[a];
    }
    store_outputs(p, b, y, x, conf, px, py, pz, rx, ry, rz);
  }
}

static inline int grid_for(long long total, int block = 256) {
  long long g = (total + block - 1) / block;
  const long long cap = (long long)num_sms() * 16;
  return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace udb

using namespace udb;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int udb_layernorm(const udb_layernorm_t* p, void* stream) {
  note_work(0.0, (double)p->rows * p->dim * ((p->in_f32 ? 4 : 2) + (p->out_f32 ? 4 : 2) + (p->out_split ? 2 : 0)));
  if (p->dim_valid < 0 || p->dim_valid > p->dim || p->dim_valid % 8) {
    set_error("udb_layernorm: dim_valid %d must be a multiple of 8 in [0, dim]", p->dim_valid);
    return 1;
  }
  if (!p->in_f32 && !p->out_f32 && p->rows_per_group <= 0 && (p->dim == 64 || p->dim == 128 || p->dim == 256)) {
    const int lpr = p->dim / 8, rpb = 8 * (32 / lpr);
    const int g = (p->rows + rpb - 1) / rpb;
    if (g == 0) return 0;
    if (lpr == 8) layernorm_f16_small_kernel<8><<<g, 256, 0, ST(stream)>>>(*p);
    else if (lpr == 16) layernorm_f16_small_kernel<16><<<g, 256, 0, ST(stream)>>>(*p);
    else layernorm_f16_small_kernel<32><<<g, 256, 0, ST(stream)>>>(*p);
    return check_launch("layernorm_f16_small_kernel");
  }
  if (p->dim_valid > 0 && p->dim_valid != p->dim) {
    set_error("udb_layernorm: dim_valid is only supported for f16->f16 rows of 64/128/256 columns");
    return 1;
  }
  if (p->dim % 128 != 0 || p->dim > 1024) { set_error("udb_layernorm: dim %d unsupported (multiple of 128, <= 1024)", p->dim); return 1; }
  // UDB_LN_ROWS=2: two rows per warp.  Measured on 12888x1024 f32->f16: 26.6 us vs 22.5 us with one row per warp
  // (a plain f32->f16 cast copy of the same bytes takes 18.5 us with the same event overhead), so one row is the default.
  static const int rows_per_warp_env = [] { const char* e = getenv("UDB_LN_ROWS"); return e ? atoi(e) : 1; }();
  const int R = (p->rows >= 2048 && rows_per_warp_env == 2) ? 2 : 1;
  const int grid = (p->rows + 8 * R - 1) / (8 * R);
  if (grid == 0) return 0;
  cudaError_t e;
  const dim3 g(grid), blk(256);
  if (R == 2) {
    if (p->in_f32 && p->out_f32) e = launch_ex(layernorm_kernel<true, true, 2>, g, blk, 0, ST(stream), 1, *p);
    else if (p->in_f32) e = launch_ex(layernorm_kernel<true, false, 2>, g, blk, 0, ST(stream), 1, *p);
    else if (p->out_f32) e = launch_ex(layernorm_kernel<false, true, 2>, g, blk, 0, ST(stream), 1, *p);
    else e = launch_ex(layernorm_kernel<false, false, 2>, g, blk, 0, ST(stream), 1, *p);
  } else {
    if (p->in_f32 && p->out_f32) e = launch_ex(layernorm_kernel<true, true, 1>, g, blk, 0, ST(stream), 1, *p);
    else if (p->in_f32) e = launch_ex(layernorm_kernel<true, false, 1>, g, blk, 0, ST(stream), 1, *p);
    else if (p->out_f32) e = launch_ex(layernorm_kernel<false, true, 1>, g, blk, 0, ST(stream), 1, *p);
    else e = launch_ex(layernorm_kernel<false, false, 1>, g, blk, 0, ST(stream), 1, *p);
  }
  if (e != cudaSuccess) { set_error("layernorm_kernel launch: %s", cudaGetErrorString(e)); return 1; }
  return check_launch("layernorm_kernel");
}

extern "C" int udb_preprocess_patchify(const udb_preprocess_t* p, void* stream) {
  if (p->net_h % 14 || p->net_w % 14 || p->ldp < (p->split ? 1184 : 592) || p->ldp % 16) {
    set_error("udb_preprocess_patchify: bad shape (net %dx%d, ldp %d)", p->net_h, p->net_w, p->ldp);
    return 1;
  }
  const int gh = p->net_h / 14, gw = p->net_w / 14;
  const int padded_h = p->H + p->pad_t + p->pad_b, padded_w = p->W + p->pad_l + p->pad_r;
  const float sh = (float)padded_h / (float)p->net_h, sw = (float)padded_w / (float)p->net_w;
  const long long total = (long long)p->B * gh * gw * (p->ldp / 8);
  note_work(0.0, (double)p->B * 3 * p->H * p->W * (p->rgb_is_u8 ? 1 : 4) + (double)p->B * gh * gw * p->ldp * 2);
  preprocess_patchify_kernel<<<grid_for(total), 256, 0, ST(stream)>>>(*p, gh, gw, sh, sw);
  return check_launch("preprocess_patchify_kernel");
}

extern "C" int udb_posembed_bicubic(const float* grid, int32_t m, int32_t dim, float* out, int32_t gh, int32_t gw, void* stream) {
  posembed_bicubic_kernel<<<grid_for((long long)gh * gw * dim), 256, 0, ST(stream)>>>(grid, m, dim, out, gh, gw);
  return check_launch("posembed_bicubic_kernel");
}

extern "C" int udb_set_cls_rows(float* x, const float* cls_token, const float* pos0, int32_t B, int32_t T, int32_t D, void* stream) {
  set_cls_rows_kernel<<<(B * D + 255) / 256, 256, 0, ST(stream)>>>(x, cls_token, pos0, B, T, D);
  return check_launch("set_cls_rows_kernel");
}

extern "C" int udb_set_cls_rows_ln(float* x, void* x16, float* stats, const float* cls_token, const float* pos0, int32_t B, int32_t T, int32_t D,
                                   int32_t parts, int32_t part_cols, void* stream) {
  if (parts * part_cols != D) { set_error("udb_set_cls_rows_ln: parts * part_cols != D"); return 1; }
  set_cls_rows_ln_kernel<<<B, 256, 0, ST(stream)>>>(x, reinterpret_cast<__half*>(x16), stats, cls_token, pos0, T, D, parts, part_cols);
  return check_launch("set_cls_rows_ln_kernel");
}

extern "C" int udb_small_linear_f32(const udb_small_linear_t* p, void* stream) {
  dim3 grid((p->N + 3) / 4, (p->M + 7) / 8);
  small_linear_kernel<<<grid, 128, 0, ST(stream)>>>(*p);
  return check_launch("small_linear_kernel");
}

extern "C" int udb_camera_attn4_f32(const float* q, const float* kv, const float* pos, float* out, int32_t B, int32_t C, int32_t heads, void* stream) {
  const int warps = B * heads * 4;
  camera_attn4_kernel<<<(warps * 32 + 127) / 128, 128, 0, ST(stream)>>>(q, kv, pos, out, B, C, heads);
  return check_launch("camera_attn4_kernel");
}

extern "C" int udb_camera_intrinsics(const float* x, int32_t B, int32_t net_h, int32_t net_w, float factor, int32_t pad_l,
                                     int32_t pad_t, float* intr4, float* k_net, float* k_out, void* stream) {
  camera_intrinsics_kernel<<<(B + 63) / 64, 64, 0, ST(stream)>>>(x, B, net_h, net_w, factor, pad_l, pad_t, intr4, k_net, k_out);
  return check_launch("camera_intrinsics_kernel");
}

// infer(camera=K): the reference wraps K in Pinhole/BatchCamera, shifts the principal point by the
// paddings (`crop`, utils/camera.py:115-120) and scales by the resize factor (`resize`, :78-81) before
// generating rays; (fx, fy, cx, cy) in network-input pixels, float32 like the reference.
__global__ void camera_adjust_k_kernel(const float* __restrict__ K, int B, float factor, float pad_l, float pad_t,
                                       float* __restrict__ intr4) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float* k = K + b * 9;
  intr4[b * 4 + 0] = k[0] * factor;
  intr4[b * 4 + 1] = k[4] * factor;
  intr4[b * 4 + 2] = (k[2] + pad_l) * factor;
  intr4[b * 4 + 3] = (k[5] + pad_t) * factor;
}

extern "C" int udb_camera_adjust_k(const float* K, int32_t B, float factor, int32_t pad_l, int32_t pad_t, float* intr4,
                                   void* stream) {
  camera_adjust_k_kernel<<<(B + 63) / 64, 64, 0, ST(stream)>>>(K, B, factor, static_cast<float>(pad_l),
                                                              static_cast<float>(pad_t), intr4);
  return check_launch("camera_adjust_k_kernel");
}

extern "C" int udb_ray_embed(const udb_ray_embed_t* p, void* stream) {
  const int toks = p->B * p->gh * p->gw;
  note_work(0.0, (double)toks * 2 * p->bands * (p->out_f32 ? 4 : 2));
  ray_embed_kernel<<<(toks + 7) / 8, 256, 0, ST(stream)>>>(*p);
  return check_launch("ray_embed_kernel");
}

extern "C" int udb_upsample2x_nhwc_f16(const void* in, void* out, int32_t B, int32_t H, int32_t W, int32_t C, void* stream) {
  if (C % 8) { set_error("udb_upsample2x_nhwc_f16: C %% 8 != 0"); return 1; }
  dim3 grid((2 * W * (C / 8) + 255) / 256, 2 * H, B);
  note_work(0.0, 2.0 * B * H * W * C * 5);
  upsample2x_kernel<<<grid, 256, 0, ST(stream)>>>(reinterpret_cast<const __half*>(in), reinterpret_cast<__half*>(out), H, W, C);
  return check_launch("upsample2x_kernel");
}

extern "C" int udb_resize_ac_pad_nhwc_f16(const void* in, void* out, int32_t B, int32_t H, int32_t W, int32_t C, int32_t oh,
                                          int32_t ow, int32_t pad, void* stream) {
  if (C % 8) { set_error("udb_resize_ac_pad_nhwc_f16: C %% 8 != 0"); return 1; }
  const float sh = (oh > 1) ? (float)(H - 1) / (float)(oh - 1) : 0.f;
  const float sw = (ow > 1) ? (float)(W - 1) / (float)(ow - 1) : 0.f;
  dim3 grid(((ow + 2 * pad) * (C / 8) + 255) / 256, oh + 2 * pad, B);
  note_work(0.0, 2.0 * B * C * ((double)H * W + (double)(oh + 2 * pad) * (ow + 2 * pad)));
  resize_ac_pad_kernel<<<grid, 256, 0, ST(stream)>>>(reinterpret_cast<const __half*>(in), reinterpret_cast<__half*>(out), H, W, C, oh, ow, pad, sh, sw);
  return check_launch("resize_ac_pad_kernel");
}

extern "C" int udb_reflect_pad1_nhwc_f16(const void* in, void* out, int32_t B, int32_t H, int32_t W, int32_t C, void* stream) {
  if (C % 8) { set_error("udb_reflect_pad1_nhwc_f16: C %% 8 != 0"); return 1; }
  dim3 grid(((W + 2) * (C / 8) + 255) / 256, H + 2, B);
  reflect_pad1_kernel<<<grid, 256, 0, ST(stream)>>>(reinterpret_cast<const uint4*>(in), reinterpret_cast<uint4*>(out), H, W, C / 8);
  return check_launch("reflect_pad1_kernel");
}

extern "C" int udb_reflect_border_fill_nhwc_f16(void* buf, int32_t B, int32_t H, int32_t W, int32_t C, void* stream) {
  if (C % 8) { set_error("udb_reflect_border_fill_nhwc_f16: C %% 8 != 0"); return 1; }
  dim3 grid(((2 * (W + 2) + 2 * H) * (C / 8) + 255) / 256, B);
  reflect_border_fill_kernel<<<grid, 256, 0, ST(stream)>>>(reinterpret_cast<uint4*>(buf), H, W, C / 8);
  return check_launch("reflect_border_fill_kernel");
}

extern "C" int udb_postprocess(const udb_postprocess_t* p, void* stream) {
  if (p->mode != UDB_INTERP_BILINEAR && p->mode != UDB_INTERP_BICUBIC) {
    set_error("udb_postprocess: `mode` %d is neither UDB_INTERP_BILINEAR (0) nor UDB_INTERP_BICUBIC (1)", p->mode);
    return 1;
  }
  note_work(0.0, 4.0 * p->B * (2.0 * p->net_h * p->net_w + 9.0 * p->H * p->W));
  const int grid = grid_for((long long)p->B * p->H * p->W);
  if (p->mode == UDB_INTERP_BICUBIC) {
    postprocess_bicubic_kernel<<<grid, 256, 0, ST(stream)>>>(*p);
    return check_launch("postprocess_bicubic_kernel");
  }
  postprocess_kernel<<<grid, 256, 0, ST(stream)>>>(*p);
  return check_launch("postprocess_kernel");
}
