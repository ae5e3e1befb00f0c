// HBM-bound / latency-bound kernels of the UniDepthV2.infer() path: LayerNorm, preprocessing +
// patch extraction, position-embedding resize, the fp32 camera head, ray embedding, bilinear
// resamplers and the output assembly.  Reference call sites are cited in include/udb.h.
#include "common.h"
#include "cuda_core.cuh"
#include "ptx.cuh"

namespace udb {

// ------------------------------------------------------------------------------------ LayerNorm
// One warp per R rows (R = 1 by default; the R = 2 variant -- both rows' loads in flight before the first
// reduction -- measured slower, see udb_layernorm); dim % 128 == 0, dim <= 1024; lane owns float4
// #(lane + 32*i).
// E4M3 (R = 1, f32 in): the normalised row stays in registers, is scaled by its amax and written as e4m3 bytes plus the
// row scale to out_scale (udb_layernorm_e4m3).
template <bool IN_F32, bool OUT_F32, int R, bool E4M3 = false>
__global__ void __launch_bounds__(256) layernorm_kernel(const udb_layernorm_t p, float* out_scale) {
  static_assert(!E4M3 || (IN_F32 && !OUT_F32 && R == 1), "e4m3 output: f32 rows, one per warp");
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
  if constexpr (E4M3) {
    float am = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i < nvec) {
        const int e = (lane + 32 * i) * 4;
        const float4 w = __ldg(reinterpret_cast<const float4*>(p.weight + e));
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + e));
        const float y0 = (x[0][i].x - mean[0]) * rstd[0] * w.x + b.x;   // the same expression as the f16 / f32 outputs
        const float y1 = (x[0][i].y - mean[0]) * rstd[0] * w.y + b.y;
        const float y2 = (x[0][i].z - mean[0]) * rstd[0] * w.z + b.z;
        const float y3 = (x[0][i].w - mean[0]) * rstd[0] * w.w + b.w;
        x[0][i] = make_float4(y0, y1, y2, y3);
        am = fmaxf(am, fmaxf(fmaxf(fabsf(y0), fabsf(y1)), fmaxf(fabsf(y2), fabsf(y3))));
      }
    }
    const E4m3Row q(warp_max(am));
    if (lane == 0) out_scale[row0] = q.scale;
    uint8_t* op = reinterpret_cast<uint8_t*>(p.out) + (long long)row0 * p.ld_out;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i < nvec) {
        const int e = (lane + 32 * i) * 4;
        *reinterpret_cast<uint32_t*>(op + e) = q.q4(x[0][i].x, x[0][i].y, x[0][i].z, x[0][i].w);
      }
    }
  } else {
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
// small warps over reuse); lanes stride over K with 128-bit loads when K % 128 == 0 and every row of x and w starts on
// a 16-byte boundary (a row-strided view may begin 4 bytes into an allocation); otherwise one float per lane
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
  if ((p.K & 127) == 0 && (ldx & 3) == 0 && ((reinterpret_cast<uintptr_t>(p.x) | reinterpret_cast<uintptr_t>(p.w)) & 15) == 0) {
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
  const float4 k = decode_camera(x + b * 4, 0.7f * diag, net_h, net_w);
  intr4[b * 4 + 0] = k.x; intr4[b * 4 + 1] = k.y; intr4[b * 4 + 2] = k.z; intr4[b * 4 + 3] = k.w;
  store_k3(k_net + b * 9, k.x, k.y, k.z, k.w);
  store_k3(k_out + b * 9, k.x / factor, k.y / factor, k.z / factor - (float)pad_l, k.w / factor - (float)pad_t);
}

// ------------------------------------------------------------------------------------ rays
__device__ __forceinline__ float3 unit_ray(const float4 k /*fx,fy,cx,cy*/, int y, int x) {
  // K^-1 [u, v, 1]^T with u = x + 0.5, v = y + 0.5 (coords_grid), then L2-normalise (clamp 1e-5)
  const float rx = (1.0f / k.x) * ((float)x + 0.5f) + (-k.z / k.x);
  const float ry = (1.0f / k.y) * ((float)y + 0.5f) + (-k.w / k.y);
  const float n = fmaxf(sqrtf(rx * rx + ry * ry + 1.0f), 1e-5f);
  return make_float3(rx / n, ry / n, 1.0f / n);
}

// one warp per output token
// ld_cat: 0 for UniDepthV2's angle features, else UniDepthV2old's Fourier features of the ray with the ray appended,
// rows of ld_cat values
__global__ void __launch_bounds__(256) ray_embed_kernel(const udb_ray_embed_t p, const int ld_cat) {
  const int tok = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int n = p.gh * p.gw;
  if (tok >= p.B * n) return;
  const int b = tok / n, i = (tok % n) / p.gw, j = tok % p.gw;
  const float sy = (float)p.net_h / (float)p.gh, sx = (float)p.net_w / (float)p.gw;
  const AAxis wy = aa_axis(i, p.net_h, sy), wx = aa_axis(j, p.net_w, sx);
  float4 k = make_float4(1.f, 1.f, 0.f, 0.f);
  if (!p.rays_in) k = *reinterpret_cast<const float4*>(p.intr4 + b * 4);
  float ax = 0.f, ay = 0.f, az = 0.f;
  const int taps = wy.xsize * wx.xsize;
  for (int t = lane; t < taps; t += 32) {
    const int ty = t / wx.xsize, tx = t % wx.xsize, yy = wy.xmin + ty, xx = wx.xmin + tx;
    // raw weight / window sum, not times `norm` (1 / sum), which rounds differently
    const float w = (wy.tri(ty, 1.f) / wy.sum) * (wx.tri(tx, 1.f) / wx.sum);
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
  if (ld_cat) {
    // UniDepthV2old (decoder_old.py:111-121 / 237-247, positional_embedding.py:218-256 with use_log, cat_orig): sin of each
    // axis of the unit ray times the `bands` frequencies and pi (axis-major), then the ray itself, zero up to `ld_cat`.
    // out_f32 == 2: split-f16 rows [hi | lo] of ld_cat / 2 features each, hi = f16(v), lo = f16(v - f32(hi))
    const float r3[3] = {ax, ay, az};
    const float pi = 3.14159265358979323846f;
    const bool split = p.out_f32 == 2;
    const int nf = split ? ld_cat / 2 : ld_cat;
    for (int f = lane; f < nf; f += 32) {
      float v = 0.f;
      if (f < 3 * p.bands) v = sinf(r3[f / p.bands] * __ldg(p.scales + (f % p.bands)) * pi);
      else if (f < 3 * p.bands + 3) v = r3[f - 3 * p.bands];
      const long long o = (long long)tok * ld_cat + f;
      if (split) {
        const __half hi = __float2half_rn(v);
        reinterpret_cast<__half*>(p.out)[o] = hi;
        reinterpret_cast<__half*>(p.out)[o + nf] = __float2half_rn(v - __half2float(hi));
      } else if (p.out_f32) {
        reinterpret_cast<float*>(p.out)[o] = v;
      } else {
        reinterpret_cast<__half*>(p.out)[o] = __float2half_rn(v);
      }
    }
    return;
  }
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

// Output assembly of the evaluation forward (udb_match_gt), its own kernel so that postprocess_kernel keeps its code.
// Matched maps: one thread per output pixel, the four taps of ATen's CUDA upsample_bilinear2d on the crop, combined in its
// order (h0 * (w0 * v00 + w1 * v01) + h1 * (w0 * v10 + w1 * v11)); a tap of the points is rays * radius rounded once, as
// network_forward's points are.  Threads below B * net_h * net_w also write one network pixel's rays, threads below B
// one matched K.  An image whose pads are negative or leave no row or column gets NaN maps and K (no read out of range).
__device__ __forceinline__ void match_tap(const udb_match_gt_t& p, const float4 k, long long o, int y, int x, float& c,
                                          float& px, float& py, float& pz) {
  float3 r;
  if (p.rays_in) { const float* rp = p.rays_in + o * 3; r = make_float3(rp[0], rp[1], rp[2]); }
  else r = unit_ray(k, y, x);
  const float rad = p.radius[o];
  c = p.confidence[o];
  px = __fmul_rn(r.x, rad); py = __fmul_rn(r.y, rad); pz = __fmul_rn(r.z, rad);
}

__global__ void __launch_bounds__(256) match_gt_kernel(const udb_match_gt_t p, long long total) {
  const long long n_out = (long long)p.B * p.H * p.W, n_net = (long long)p.B * p.net_h * p.net_w;
  const float nan = __int_as_float(0x7fc00000);
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    if (idx < n_out) {
      const int x = (int)(idx % p.W), y = (int)((idx / p.W) % p.H), b = (int)(idx / ((long long)p.W * p.H));
      const int* pd = p.pads + b * 4;
      const int l = pd[0], r = pd[1], t = pd[2], bo = pd[3];
      const int ch = p.net_h - t - bo, cw = p.net_w - l - r;
      const long long plane = (long long)p.H * p.W, pix = (long long)y * p.W + x;
      float conf = nan, px = nan, py = nan, pz = nan;
      if (min(min(l, r), min(t, bo)) >= 0 && ch >= 1 && cw >= 1) {
        int y0, y1, x0, x1;
        float ly0, ly1, lx0, lx1;
        bilinear_src((float)ch / (float)p.H, y, ch, y0, y1, ly0, ly1);
        bilinear_src((float)cw / (float)p.W, x, cw, x0, x1, lx0, lx1);
        y0 += t; y1 += t; x0 += l; x1 += l;
        float4 k = make_float4(1.f, 1.f, 0.f, 0.f);
        if (!p.rays_in) k = *reinterpret_cast<const float4*>(p.intr4 + b * 4);
        const long long rb = (long long)b * p.net_h;
        float c[4], X[4], Y[4], Z[4];
        match_tap(p, k, (rb + y0) * p.net_w + x0, y0, x0, c[0], X[0], Y[0], Z[0]);
        match_tap(p, k, (rb + y0) * p.net_w + x1, y0, x1, c[1], X[1], Y[1], Z[1]);
        match_tap(p, k, (rb + y1) * p.net_w + x0, y1, x0, c[2], X[2], Y[2], Z[2]);
        match_tap(p, k, (rb + y1) * p.net_w + x1, y1, x1, c[3], X[3], Y[3], Z[3]);
        auto lerp = [&](const float* v) { return ly0 * (lx0 * v[0] + lx1 * v[1]) + ly1 * (lx0 * v[2] + lx1 * v[3]); };
        conf = lerp(c); px = lerp(X); py = lerp(Y); pz = lerp(Z);
      }
      p.out_confidence[b * plane + pix] = conf;
      p.out_depth[b * plane + pix] = pz;
      p.out_points[(b * 3 + 0) * plane + pix] = px;
      p.out_points[(b * 3 + 1) * plane + pix] = py;
      p.out_points[(b * 3 + 2) * plane + pix] = pz;
    }
    if (idx < n_net) {
      // the rays network_forward returns (one normalisation), normalised once more as forward_test does
      const int x = (int)(idx % p.net_w), y = (int)((idx / p.net_w) % p.net_h), b = (int)(idx / ((long long)p.net_w * p.net_h));
      float3 r;
      if (p.rays_in) { const float* rp = p.rays_in + idx * 3; r = make_float3(rp[0], rp[1], rp[2]); }
      else r = unit_ray(*reinterpret_cast<const float4*>(p.intr4 + b * 4), y, x);
      const float n1 = fmaxf(sqrtf(r.x * r.x + r.y * r.y + r.z * r.z), 1e-5f);
      const float ax = r.x / n1, ay = r.y / n1, az = r.z / n1;
      const float n2 = fmaxf(sqrtf(ax * ax + ay * ay + az * az), 1e-5f);
      const long long plane = (long long)p.net_h * p.net_w, pix = (long long)y * p.net_w + x;
      p.out_rays[(b * 3 + 0) * plane + pix] = ax / n2;
      p.out_rays[(b * 3 + 1) * plane + pix] = ay / n2;
      p.out_rays[(b * 3 + 2) * plane + pix] = az / n2;
    }
    if (idx < p.B) {
      // match_intrinsics (misc.py:645-690) in f32 and in its op order; the target has no padding (padding2 = None)
      const int b = (int)idx;
      const int* pd = p.pads + b * 4;
      const int l = pd[0], t = pd[2];
      const int ch = p.net_h - t - pd[3], cw = p.net_w - l - pd[1];
      float* K = p.intrinsics + b * 9;
      if (min(min(l, pd[1]), min(t, pd[3])) >= 0 && ch >= 1 && cw >= 1) {
        const float sx = (float)((double)p.W / (double)cw), sy = (float)((double)p.H / (double)ch);
        K[0] = __fmul_rn(K[0], sx);
        K[4] = __fmul_rn(K[4], sy);
        K[2] = __fadd_rn(__fmul_rn(__fsub_rn(K[2], (float)l), sx), 0.f);
        K[5] = __fadd_rn(__fmul_rn(__fsub_rn(K[5], (float)t), sy), 0.f);
      } else {
        for (int i = 0; i < 9; ++i) K[i] = nan;
      }
    }
  }
}

// f16 rows -> e4m3 rows + row scales (udb_quantize_rows_e4m3): one warp per row, lane holds 16-byte chunks
// lane + 32 i (i < NCH: up to NCH * 256 columns) in registers between the amax reduction and the conversion.  NCH = 16
// serves up to 4096 columns (the DINOv2 MLP), NCH = 24 up to 6144 (ConvNeXt-L stage 3's 4 x 1536); the amax is a max,
// so both give the same bytes where both apply.
template <int NCH>
__global__ void __launch_bounds__(256) quantize_rows_e4m3_kernel(const __half* __restrict__ in, long long ld_in,
                                                                 uint8_t* __restrict__ out, long long ld_out,
                                                                 float* __restrict__ scale, int rows, int cols) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int nch = cols >> 3;
  const uint4* ip = reinterpret_cast<const uint4*>(in + (long long)row * ld_in);
  uint4 v[NCH];
  __half2 am2 = __float2half2_rn(0.f);
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nch) {
      v[i] = ip[c];
      const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
#pragma unroll
      for (int k = 0; k < 4; ++k) am2 = __hmax2(am2, __habs2(h[k]));
    }
  }
  const E4m3Row q(warp_max(fmaxf(__low2float(am2), __high2float(am2))));
  if (lane == 0) scale[row] = q.scale;
  uint2* op = reinterpret_cast<uint2*>(out + (long long)row * ld_out);
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int c = lane + 32 * i;
    if (c < nch) {
      const __half2* h = reinterpret_cast<const __half2*>(&v[i]);
      const float2 a = __half22float2(h[0]), b = __half22float2(h[1]), d = __half22float2(h[2]), f = __half22float2(h[3]);
      op[c] = make_uint2(q.q4(a.x, a.y, b.x, b.y), q.q4(d.x, d.y, f.x, f.y));
    }
  }
}

}  // namespace udb

using namespace udb;

extern "C" int udb_layernorm_e4m3(const udb_layernorm_t* p, float* out_scale, void* stream) {
  if (!p || !p->in_f32 || p->out_split || (p->dim_valid && p->dim_valid != p->dim) || !out_scale || (reinterpret_cast<uintptr_t>(out_scale) & 3)) {
    set_error("udb_layernorm_e4m3: needs f32 input, no out_split / dim_valid and a 4-byte aligned out_scale");
    return 1;
  }
  if (p->dim % 128 != 0 || p->dim > 1024) { set_error("udb_layernorm_e4m3: dim %d unsupported (multiple of 128, <= 1024)", p->dim); return 1; }
  if (p->ld_out < p->dim || p->ld_out % 4 || (reinterpret_cast<uintptr_t>(p->out) & 3)) {
    set_error("udb_layernorm_e4m3: `out` needs 4-byte alignment and ld_out >= dim, a multiple of 4 (ld_out %lld)", (long long)p->ld_out);
    return 1;
  }
  note_work(0.0, (double)p->rows * p->dim * (4 + 1) + 4.0 * p->rows);
  const int grid = (p->rows + 7) / 8;
  if (grid == 0) return 0;
  const cudaError_t e = launch_ex(layernorm_kernel<true, false, 1, true>, dim3(grid), dim3(256), 0, ST(stream), 1, *p, out_scale);
  if (e != cudaSuccess) { set_error("layernorm_kernel launch: %s", cudaGetErrorString(e)); return 1; }
  return check_launch("layernorm_e4m3_kernel");
}

extern "C" int udb_layernorm(const udb_layernorm_t* p, void* stream) {
  if (p->out_split < 0 || (p->out_split > 0 && (!p->in_f32 || p->out_f32))) {
    set_error("udb_layernorm: `out_split` %d needs f32 input and f16 output (in_f32 %d, out_f32 %d)", p->out_split, p->in_f32,
              p->out_f32);
    return 1;
  }
  if (p->ld_out < (int64_t)p->dim + p->out_split) {
    set_error("udb_layernorm: `ld_out` %lld < dim %d + out_split %d", (long long)p->ld_out, p->dim, p->out_split);
    return 1;
  }
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
    if (p->in_f32 && p->out_f32) e = launch_ex(layernorm_kernel<true, true, 2>, g, blk, 0, ST(stream), 1, *p, static_cast<float*>(nullptr));
    else if (p->in_f32) e = launch_ex(layernorm_kernel<true, false, 2>, g, blk, 0, ST(stream), 1, *p, static_cast<float*>(nullptr));
    else if (p->out_f32) e = launch_ex(layernorm_kernel<false, true, 2>, g, blk, 0, ST(stream), 1, *p, static_cast<float*>(nullptr));
    else e = launch_ex(layernorm_kernel<false, false, 2>, g, blk, 0, ST(stream), 1, *p, static_cast<float*>(nullptr));
  } else {
    if (p->in_f32 && p->out_f32) e = launch_ex(layernorm_kernel<true, true, 1>, g, blk, 0, ST(stream), 1, *p, static_cast<float*>(nullptr));
    else if (p->in_f32) e = launch_ex(layernorm_kernel<true, false, 1>, g, blk, 0, ST(stream), 1, *p, static_cast<float*>(nullptr));
    else if (p->out_f32) e = launch_ex(layernorm_kernel<false, true, 1>, g, blk, 0, ST(stream), 1, *p, static_cast<float*>(nullptr));
    else e = launch_ex(layernorm_kernel<false, false, 1>, g, blk, 0, ST(stream), 1, *p, static_cast<float*>(nullptr));
  }
  if (e != cudaSuccess) { set_error("layernorm_kernel launch: %s", cudaGetErrorString(e)); return 1; }
  return check_launch("layernorm_kernel");
}

extern "C" int udb_quantize_rows_e4m3(const void* in, int64_t ld_in, void* out, int64_t ld_out, float* scale, int32_t rows,
                                      int32_t cols, void* stream) {
  if (!in || !out || !scale || rows < 0 || cols < 8 || cols > 6144 || cols % 8) {
    set_error("udb_quantize_rows_e4m3: bad arguments (rows %d, cols %d: need a multiple of 8 in [8, 6144])", rows, cols);
    return 1;
  }
  if (ld_in < cols || ld_in % 8 || ld_out < cols || ld_out % 8 || (reinterpret_cast<uintptr_t>(in) & 15) ||
      (reinterpret_cast<uintptr_t>(out) & 15) || (reinterpret_cast<uintptr_t>(scale) & 3)) {
    set_error("udb_quantize_rows_e4m3: ld_in %lld / ld_out %lld must be >= cols and multiples of 8, in / out 16-byte aligned",
              (long long)ld_in, (long long)ld_out);
    return 1;
  }
  note_work(0.0, (double)rows * cols * (2 + 1) + 4.0 * rows);
  if (rows == 0) return 0;
  const auto kernel = cols <= 4096 ? quantize_rows_e4m3_kernel<16> : quantize_rows_e4m3_kernel<24>;
  kernel<<<(rows + 7) / 8, 256, 0, ST(stream)>>>(static_cast<const __half*>(in), ld_in, static_cast<uint8_t*>(out), ld_out, scale,
                                                 rows, cols);
  return check_launch("quantize_rows_e4m3_kernel");
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
  preprocess_patchify_kernel<<<grid_1d(total, 16), 256, 0, ST(stream)>>>(*p, gh, gw, sh, sw);
  return check_launch("preprocess_patchify_kernel");
}

extern "C" int udb_posembed_bicubic(const float* grid, int32_t m, int32_t dim, float* out, int32_t gh, int32_t gw, void* stream) {
  posembed_bicubic_kernel<<<grid_1d((long long)gh * gw * dim, 16), 256, 0, ST(stream)>>>(grid, m, dim, out, gh, gw);
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
  if (B < 1 || heads < 1 || C < heads || C % heads) {
    set_error("udb_camera_attn4_f32: B=%d, C=%d, heads=%d: needs B >= 1, heads >= 1 and C a multiple of heads", B, C, heads);
    return 1;
  }
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
  ray_embed_kernel<<<(toks + 7) / 8, 256, 0, ST(stream)>>>(*p, 0);
  return check_launch("ray_embed_kernel");
}

extern "C" int udb_ray_embed_cat_orig(const udb_ray_embed_t* p, int32_t ld_out, void* stream) {
  if (!p || !p->intr4 || !p->scales || !p->out) { set_error("udb_ray_embed_cat_orig: null argument (intr4, scales and out are required)"); return 1; }
  if (p->bands < 1 || ld_out < 3 * p->bands + 3) {
    set_error("udb_ray_embed_cat_orig: needs bands >= 1 and ld_out >= 3*bands + 3 (bands=%d ld_out=%d)", p->bands, ld_out);
    return 1;
  }
  if (p->out_f32 == 2 && (ld_out % 2 || ld_out / 2 < 3 * p->bands + 3)) {
    set_error("udb_ray_embed_cat_orig: split output needs an even ld_out >= 2*(3*bands + 3) to hold both halves (bands=%d ld_out=%d)",
              p->bands, ld_out);
    return 1;
  }
  if (p->B < 1 || p->gh < 1 || p->gw < 1 || p->net_h < 1 || p->net_w < 1) {
    set_error("udb_ray_embed_cat_orig: B=%d gh=%d gw=%d net_h=%d net_w=%d must all be >= 1", p->B, p->gh, p->gw, p->net_h, p->net_w);
    return 1;
  }
  const int toks = p->B * p->gh * p->gw;
  note_work(0.0, (double)toks * ld_out * (p->out_f32 == 1 ? 4 : 2));
  ray_embed_kernel<<<(toks + 7) / 8, 256, 0, ST(stream)>>>(*p, ld_out);
  return check_launch("ray_embed_cat_orig_kernel");
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
  const int grid = grid_1d((long long)p->B * p->H * p->W, 16);
  if (p->mode == UDB_INTERP_BICUBIC) {
    postprocess_bicubic_kernel<<<grid, 256, 0, ST(stream)>>>(*p);
    return check_launch("postprocess_bicubic_kernel");
  }
  postprocess_kernel<<<grid, 256, 0, ST(stream)>>>(*p);
  return check_launch("postprocess_kernel");
}

extern "C" int udb_match_gt(const udb_match_gt_t* p, void* stream) {
  if (check_dims("udb_match_gt", {{p->B, "B"}, {p->H, "H"}, {p->W, "W"}, {p->net_h, "net_h"}, {p->net_w, "net_w"}})) return 1;
  if (check_ptrs("udb_match_gt", {{p->radius, "radius"}, {p->confidence, "confidence"}, {p->pads, "pads"}, {p->intrinsics, "intrinsics"},
                                  {p->out_confidence, "out_confidence"}, {p->out_depth, "out_depth"}, {p->out_points, "out_points"},
                                  {p->out_rays, "out_rays"}}))
    return 1;
  if (!p->rays_in && !p->intr4) { set_error("udb_match_gt: `intr4` must be non-null when `rays_in` is null"); return 1; }
  if (!p->rays_in && (reinterpret_cast<uintptr_t>(p->intr4) & 15)) { set_error("udb_match_gt: `intr4` must be 16-byte aligned"); return 1; }
  const long long n_out = (long long)p->B * p->H * p->W, n_net = (long long)p->B * p->net_h * p->net_w;
  const long long total = n_out > n_net ? n_out : n_net;
  note_work(0.0, 4.0 * (2.0 * n_net + 5.0 * n_out + 3.0 * n_net));
  match_gt_kernel<<<grid_1d(total, 16), 256, 0, ST(stream)>>>(*p, total);
  return check_launch("match_gt_kernel");
}
