// Kernels that only the UniDepthV1 / ConvNeXt path needs (BASELINE config 4; include/udb.h "UniDepthV1 operators"):
// depthwise 7x7, channel LayerNorm for ConvNeXt widths (with space-to-depth output for the k2 s2 downsample and an
// additive table for "tokens + positional embedding"), antialiased bilinear resampling, the fused ray -> SH-81 ->
// LayerNorm embedding, the small dense-attention pieces (row softmax, 4-query cross attention, Nystrom landmarks /
// pseudo-inverse matmuls), single-output 3x3 convolutions and the V1 pre / post-processing.  All HBM- or
// latency-bound CUDA-core work; the GEMM-shaped parts of V1 run on the wgmma kernels of gemm.cu / attention.cu.
#include <cooperative_groups.h>
#include <math.h>

#include "common.h"
#include "cuda_core.cuh"
#include "ptx.cuh"

namespace udb {

// ------------------------------------------------------------------------------------------------------------------
// V1 pre-processing (unidepthv1.py:49-63,298-317): u8 / f32 NCHW -> /255 -> ImageNet normalise -> antialiased bilinear
// to (rh, rw) -> zero pad to the fixed network shape -> P x P stride-P patch rows f16:
//   P = 4:  [B*gh*gw, 64]  (48 used: column c*16 + py*4 + px, the ConvNeXt stem conv's im2col, convnext.py:371-383)
//   P = 14: [B*gh*gw, 640] (588 used: column c*196 + py*14 + px, the DINOv2 patch embedding's im2col, patch_embed.py)
// SPLIT: rows of 2 x COLS halves, hi = f16(v) (the rows above) and lo = f16(v - f32(hi)) COLS columns to the right.
// ------------------------------------------------------------------------------------------------------------------
template <int P, bool SPLIT>
__global__ void __launch_bounds__(256) v1_preprocess_kernel(const udb_v1_preprocess_t p, int gh, int gw, float sh, float sw) {
  constexpr int COLS = P == 4 ? 64 : 640, USED = 3 * P * P, NV8 = COLS / 8;
  const long long total = (long long)p.B * gh * gw * NV8;   // NV8 x (8 columns) per patch row
  const float mean[3] = {0.485f, 0.456f, 0.406f};
  const float stdv[3] = {0.229f, 0.224f, 0.225f};
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int v8 = (int)(idx % NV8);
    const long long row = idx / NV8;
    const int gx = (int)(row % gw), gy = (int)((row / gw) % gh), b = (int)(row / ((long long)gw * gh));
    float val[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = v8 * 8 + j;
      float acc = 0.f;
      if (col < USED) {
        const int c = col / (P * P), py = (col % (P * P)) / P, px = col % P;
        const int Y = gy * P + py - p.pad_t, X = gx * P + px - p.pad_l;     // position in the resized image
        if (Y >= 0 && Y < p.rh && X >= 0 && X < p.rw) {
          const AAxis ay = aa_axis(Y, p.H, sh), ax = aa_axis(X, p.W, sw);
          for (int jy = 0; jy < ay.xsize; ++jy) {
            float r = 0.f;
            const long long base = (((long long)b * 3 + c) * p.H + (ay.xmin + jy)) * p.W + ax.xmin;
            for (int jx = 0; jx < ax.xsize; ++jx) {
              float t = p.rgb_is_u8 ? (float)__ldg(reinterpret_cast<const uint8_t*>(p.rgb) + base + jx)
                                    : __ldg(reinterpret_cast<const float*>(p.rgb) + base + jx);
              if (p.scale255) t = t / 255.0f;
              if (p.normalize) t = (t - mean[c]) / stdv[c];
              r += ax.w(jx) * t;
            }
            acc += ay.w(jy) * r;
          }
        }
      }
      val[j] = acc;
    }
    if (SPLIT) {
      float lo[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) lo[j] = val[j] - __half2float(__float2half_rn(val[j]));
      __half* dst = reinterpret_cast<__half*>(p.patches) + row * 2 * COLS + v8 * 8;
      *reinterpret_cast<uint4*>(dst) =
          make_uint4(pack_half2(val[0], val[1]), pack_half2(val[2], val[3]), pack_half2(val[4], val[5]), pack_half2(val[6], val[7]));
      *reinterpret_cast<uint4*>(dst + COLS) =
          make_uint4(pack_half2(lo[0], lo[1]), pack_half2(lo[2], lo[3]), pack_half2(lo[4], lo[5]), pack_half2(lo[6], lo[7]));
      continue;
    }
    *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.patches) + row * COLS + v8 * 8) =
        make_uint4(pack_half2(val[0], val[1]), pack_half2(val[2], val[3]), pack_half2(val[4], val[5]), pack_half2(val[6], val[7]));
  }
}

// ------------------------------------------------------------------------------------------------------------------
// LayerNorm over the channels for any width that is a multiple of 64 up to 1536 (ConvNeXt: 192 / 384 / 768 / 1536;
// timm LayerNorm2d == channels-last LayerNorm, convnext.py:252-263; eps 1e-6 in the encoder, 1e-5 in the decoder).
// One warp per row, lane owns element pairs.  Extras: an additive f32 table (in = x[row] + add[row % add_mod]) for
// "tokens + positional embedding" (decoder.py:92-94), and a space-to-depth output mapping that writes pixel (y, x) of
// an [B,H,W,C] map into row (b, y/2, x/2), columns ((y&1)*2 + (x&1))*C + c of the k2 s2 downsample's im2col matrix
// (odd trailing row / column dropped, as the strided conv does).  OUT: 0 f16, 1 f32, 2 split f16 (hi = f16(y) where the
// f16 output goes, lo = f16(y - f32(hi)) ld_out / 2 columns further right).
// ------------------------------------------------------------------------------------------------------------------
template <bool IN_F32, int OUT, int R, int NV>
__global__ void __launch_bounds__(256) layernorm_any_kernel(const udb_layernorm_any_t p) {
  // one warp normalises R consecutive rows; all loads of the R rows are issued before the first reduction (narrow rows
  // alone -- 192 channels = 384 B -- do not keep enough bytes in flight); NV = max float2 per lane per row
  const long long row0 = ((long long)blockIdx.x * 8 + (threadIdx.x >> 5)) * R;
  const int lane = threadIdx.x & 31;
  if (row0 >= p.rows) return;
  const int nv = p.dim >> 6;   // float2 per lane
  float2 x[R][NV];
  float s[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const long long row = row0 + r < p.rows ? row0 + r : p.rows - 1;
    s[r] = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      if (i < nv) {
        const int e = (lane + 32 * i) * 2;
        if (IN_F32) {
          x[r][i] = *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(p.in) + row * p.ld_in + e);
        } else {
          x[r][i] = __half22float2(*reinterpret_cast<const __half2*>(reinterpret_cast<const __half*>(p.in) + row * p.ld_in + e));
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const long long row = row0 + r < p.rows ? row0 + r : p.rows - 1;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      if (i < nv) {
        if (p.add) {
          const float2 a = *reinterpret_cast<const float2*>(p.add + (row % p.add_mod) * p.dim + (lane + 32 * i) * 2);
          x[r][i].x += a.x;
          x[r][i].y += a.y;
        }
        s[r] += x[r][i].x + x[r][i].y;
      }
    }
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const long long row = row0 + r;
    const float mean = warp_sum(s[r]) / (float)p.dim;
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (i < nv) v += (x[r][i].x - mean) * (x[r][i].x - mean) + (x[r][i].y - mean) * (x[r][i].y - mean);
    const float rstd = rsqrtf(warp_sum(v) / (float)p.dim + p.eps);
    if (row >= p.rows) continue;
    long long obase = row * p.ld_out;
    if (p.s2d_w > 0) {
      const int xw = (int)(row % p.s2d_w), yh = (int)((row / p.s2d_w) % p.s2d_h), b = (int)(row / ((long long)p.s2d_w * p.s2d_h));
      const int oh = p.s2d_h >> 1, ow = p.s2d_w >> 1;
      if ((yh >> 1) >= oh || (xw >> 1) >= ow) continue;
      obase = (((long long)b * oh + (yh >> 1)) * ow + (xw >> 1)) * p.ld_out + ((yh & 1) * 2 + (xw & 1)) * p.dim;
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      if (i < nv) {
        const int e = (lane + 32 * i) * 2;
        const float2 w = __ldg(reinterpret_cast<const float2*>(p.weight + e));
        const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + e));
        const float y0 = (x[r][i].x - mean) * rstd * w.x + bb.x, y1 = (x[r][i].y - mean) * rstd * w.y + bb.y;
        if (OUT == 1) {
          *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + obase + e) = make_float2(y0, y1);
        } else {
          *reinterpret_cast<uint32_t*>(reinterpret_cast<__half*>(p.out) + obase + e) = pack_half2(y0, y1);
          if (OUT == 2)
            *reinterpret_cast<uint32_t*>(reinterpret_cast<__half*>(p.out) + obase + (p.ld_out >> 1) + e) =
                pack_half2(y0 - __half2float(__float2half_rn(y0)), y1 - __half2float(__float2half_rn(y1)));
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Depthwise 7x7 convolution, zero padding 3, NHWC f16 -> NHWC f16 (+bias), f32 accumulation
// (convnext.py:208-211 `conv_dw`, layers/convnext.py:16-24 `dwconv`).  A block owns an 8x16-pixel tile of 64 channels:
// the 14x22 halo is staged once in shared memory (2.4x read amplification instead of 49x), each thread slides along 8
// consecutive x for one 4-channel group, so per dy it loads 14 inputs + 7 weights for 56 FMA4.
// ------------------------------------------------------------------------------------------------------------------
constexpr int DW_CB = 64;
constexpr int DW_PS = DW_CB + 4;   // pixel stride in halves (136 B): keeps the 8-byte row reads of a warp on distinct banks

// TW = tile width (16 or 8), tile height = 128 / TW: wide tiles have the smaller halo, narrow ones waste fewer pixels on the
// small late-stage maps (28x38, 14x19); the launcher picks the shape with the least padded area.
template <int TW>
__global__ void __launch_bounds__(256) dwconv7_kernel(const __half* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                     __half* __restrict__ y, int H, int W, int C, int tiles_x) {
  constexpr int TH = 128 / TW, HH = TH + 6, HW = TW + 6;
  __shared__ __align__(16) __half tile[HH * HW * DW_PS];
  const int tx0 = (blockIdx.x % tiles_x) * TW, ty0 = (blockIdx.x / tiles_x) * TH;
  const int c0 = blockIdx.y * DW_CB, b = blockIdx.z;
  const __half* xb = x + (long long)b * H * W * C;
  for (int i = threadIdx.x; i < HH * HW * (DW_CB / 8); i += 256) {
    const int ch = i & 7, pix = i >> 3;
    const int hy = pix / HW, hx = pix - hy * HW;
    const int gy = ty0 + hy - 3, gx = tx0 + hx - 3;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = __ldg(reinterpret_cast<const uint4*>(xb + ((long long)gy * W + gx) * C + c0 + ch * 8));
    uint2* d = reinterpret_cast<uint2*>(tile + pix * DW_PS + ch * 8);      // 8-byte aligned (136 B pixel stride)
    d[0] = make_uint2(v.x, v.y);
    d[1] = make_uint2(v.z, v.w);
  }
  __syncthreads();
  const int cg = threadIdx.x & 15, pg = threadIdx.x >> 4;
  const int r = TW == 16 ? (pg >> 1) : pg, xh = TW == 16 ? (pg & 1) * 8 : 0;     // each thread: 8 consecutive x of one row
  uint64_t acc[8][2];          // f32 pairs: (c0,c1), (c2,c3)
  {
    const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + c0 + cg * 4));
#pragma unroll
    for (int i = 0; i < 8; ++i) { acc[i][0] = pack2(bv.x, bv.y); acc[i][1] = pack2(bv.z, bv.w); }
  }
#pragma unroll 1
  for (int dy = 0; dy < 7; ++dy) {
    uint64_t in[14][2];
#pragma unroll
    for (int i = 0; i < 14; ++i) {
      const uint2 u = *reinterpret_cast<const uint2*>(tile + ((r + dy) * HW + xh + i) * DW_PS + cg * 4);
      const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
      const float2 c = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
      in[i][0] = pack2(a.x, a.y);
      in[i][1] = pack2(c.x, c.y);
    }
#pragma unroll
    for (int dx = 0; dx < 7; ++dx) {
      const float4 wv = __ldg(reinterpret_cast<const float4*>(w + (long long)(dy * 7 + dx) * C + c0 + cg * 4));
      const uint64_t w0 = pack2(wv.x, wv.y), w1 = pack2(wv.z, wv.w);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        acc[i][0] = fma2(in[i + dx][0], w0, acc[i][0]);
        acc[i][1] = fma2(in[i + dx][1], w1, acc[i][1]);
      }
    }
  }
  const int gy = ty0 + r;
  if (gy < H) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int gx = tx0 + xh + i;
      if (gx < W) {
        float a0, a1, a2, a3;
        unpack2(acc[i][0], a0, a1);
        unpack2(acc[i][1], a2, a3);
        *reinterpret_cast<uint2*>(y + (((long long)b * H + gy) * W + gx) * C + c0 + cg * 4) = make_uint2(pack_half2(a0, a1), pack_half2(a2, a3));
      }
    }
  }
}

// The same convolution on f32 NHWC maps (split-precision mode: it reads the f32 residual stream).  A block owns a 16x8
// tile of 32 channels (the 22x14 halo in f32 is 39 KB of shared memory); each thread slides along 4 consecutive x of one
// row for one 4-channel group.  Bias first, then dy outer / dx inner fmaf: the taps, padding and summation order of
// dwconv7_kernel, so an input that is exactly f16 gives that kernel's f32 sums.
constexpr int DWF_CB = 32, DWF_TW = 16, DWF_TH = 8;

__global__ void __launch_bounds__(256) dwconv7_f32_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                         float* __restrict__ y, int H, int W, int C, int tiles_x) {
  constexpr int HH = DWF_TH + 6, HW = DWF_TW + 6;
  __shared__ __align__(16) float tile[HH * HW * DWF_CB];
  const int tx0 = (blockIdx.x % tiles_x) * DWF_TW, ty0 = (blockIdx.x / tiles_x) * DWF_TH;
  const int c0 = blockIdx.y * DWF_CB, b = blockIdx.z;
  const float* xb = x + (long long)b * H * W * C;
  for (int i = threadIdx.x; i < HH * HW * (DWF_CB / 4); i += 256) {
    const int ch = i & 7, pix = i >> 3;
    const int hy = pix / HW, hx = pix - hy * HW;
    const int gy = ty0 + hy - 3, gx = tx0 + hx - 3;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = __ldg(reinterpret_cast<const float4*>(xb + ((long long)gy * W + gx) * C + c0 + ch * 4));
    *reinterpret_cast<float4*>(tile + pix * DWF_CB + ch * 4) = v;
  }
  __syncthreads();
  const int cg = threadIdx.x & 7, xs = ((threadIdx.x >> 3) & 3) * 4, r = threadIdx.x >> 5;
  float acc[4][4];
  {
    const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + c0 + cg * 4));
#pragma unroll
    for (int i = 0; i < 4; ++i) { acc[i][0] = bv.x; acc[i][1] = bv.y; acc[i][2] = bv.z; acc[i][3] = bv.w; }
  }
#pragma unroll 1
  for (int dy = 0; dy < 7; ++dy) {
    float4 in[10];
#pragma unroll
    for (int i = 0; i < 10; ++i) in[i] = *reinterpret_cast<const float4*>(tile + ((r + dy) * HW + xs + i) * DWF_CB + cg * 4);
#pragma unroll
    for (int dx = 0; dx < 7; ++dx) {
      const float4 wv = __ldg(reinterpret_cast<const float4*>(w + (long long)(dy * 7 + dx) * C + c0 + cg * 4));
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        acc[i][0] = fmaf(in[i + dx].x, wv.x, acc[i][0]);
        acc[i][1] = fmaf(in[i + dx].y, wv.y, acc[i][1]);
        acc[i][2] = fmaf(in[i + dx].z, wv.z, acc[i][2]);
        acc[i][3] = fmaf(in[i + dx].w, wv.w, acc[i][3]);
      }
    }
  }
  const int gy = ty0 + r;
  if (gy < H) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int gx = tx0 + xs + i;
      if (gx < W)
        *reinterpret_cast<float4*>(y + (((long long)b * H + gy) * W + gx) * C + c0 + cg * 4) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// ConvNeXt block head in e4m3 mode (udb_dwconv7_ln_e4m3): depthwise 7x7 -> f16 -> LayerNorm (eps 1e-6) -> e4m3 rows +
// row scales, the A operand of the fc1 GEMM.  LayerNorm needs a pixel's whole channel row, so a CLUSTER of K blocks owns
// a 128-pixel tile (TW x 128/TW, as dwconv7_kernel) across all channels: block k of the cluster takes the 64-channel
// chunks k, k + K, ... (at most 3; K = ceil(C / 192), up to 8 for C = 1536), which bounds its shared memory whatever C
// is.  Each chunk is convolved exactly as dwconv7_kernel does it (halo in shared memory, 8 consecutive x x 4 channels
// per thread, the same f32 FMA order) and its f16 outputs stay in the block's shared memory.  The per-pixel sum, sum of
// squared deviations and amax are each reduced over the cluster through distributed shared memory, in rank order, so
// the result does not depend on scheduling; then every block writes its channels of each row quantised.
// ------------------------------------------------------------------------------------------------------------------
constexpr int DWL_PX = 128;
constexpr int DWL_HALO_BYTES = 14 * 22 * DW_PS * 2;                 // one 64-channel chunk of the halo (either tile shape)
constexpr int DWL_CPB = 3;                                          // 64-channel chunks per block at most
constexpr int DWL_MAXC = 1536;
constexpr int DWL_YS_LD = DWL_CPB * DW_CB + 8;                      // f16 conv outputs [128 px][this block's channels]
constexpr int DWL_SMEM = DWL_HALO_BYTES + DWL_PX * DWL_YS_LD * 2 + 3 * DWL_PX * 4;

template <int TW>
__global__ void __launch_bounds__(256) dwconv7_ln_e4m3_kernel(const __half* __restrict__ x, const float* __restrict__ w,
                                                             const float* __restrict__ bias, const float* __restrict__ ln_w,
                                                             const float* __restrict__ ln_b, uint8_t* __restrict__ out,
                                                             float* __restrict__ out_scale, int H, int W, int C, int tiles_x) {
  constexpr int TH = DWL_PX / TW, HH = TH + 6, HW = TW + 6;
  extern __shared__ __align__(16) unsigned char dwl_smem[];
  __half* tile = reinterpret_cast<__half*>(dwl_smem);
  __half* ys = reinterpret_cast<__half*>(dwl_smem + DWL_HALO_BYTES);
  float (*part)[DWL_PX] = reinterpret_cast<float (*)[DWL_PX]>(dwl_smem + DWL_HALO_BYTES + DWL_PX * DWL_YS_LD * 2);   // sum / squares / amax
  namespace cgr = cooperative_groups;
  cgr::cluster_group cluster = cgr::this_cluster();
  const int K = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int t = blockIdx.x / K;
  const int tx0 = (t % tiles_x) * TW, ty0 = (t / tiles_x) * TH, b = blockIdx.y;
  const __half* xb = x + (long long)b * H * W * C;
  const int cg = threadIdx.x & 15, pg = threadIdx.x >> 4;
  const int r = TW == 16 ? (pg >> 1) : pg, xh = TW == 16 ? (pg & 1) * 8 : 0;   // each thread: 8 consecutive x, 4 channels
  pdl_wait();                                      // x16 is written by the previous block's fc2 GEMM
  int nloc = 0;
  for (int c0 = rank * DW_CB; c0 < C; c0 += K * DW_CB, ++nloc) {
    if (nloc) __syncthreads();                     // the previous chunk's halo is no longer read
    for (int i = threadIdx.x; i < HH * HW * (DW_CB / 8); i += 256) {
      const int ch = i & 7, pix = i >> 3;
      const int hy = pix / HW, hx = pix - hy * HW;
      const int gy = ty0 + hy - 3, gx = tx0 + hx - 3;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = __ldg(reinterpret_cast<const uint4*>(xb + ((long long)gy * W + gx) * C + c0 + ch * 8));
      uint2* d = reinterpret_cast<uint2*>(tile + pix * DW_PS + ch * 8);
      d[0] = make_uint2(v.x, v.y);
      d[1] = make_uint2(v.z, v.w);
    }
    __syncthreads();
    uint64_t acc[8][2];
    {
      const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + c0 + cg * 4));
#pragma unroll
      for (int i = 0; i < 8; ++i) { acc[i][0] = pack2(bv.x, bv.y); acc[i][1] = pack2(bv.z, bv.w); }
    }
#pragma unroll 1
    for (int dy = 0; dy < 7; ++dy) {
      uint64_t in[14][2];
#pragma unroll
      for (int i = 0; i < 14; ++i) {
        const uint2 u = *reinterpret_cast<const uint2*>(tile + ((r + dy) * HW + xh + i) * DW_PS + cg * 4);
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
        const float2 c = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
        in[i][0] = pack2(a.x, a.y);
        in[i][1] = pack2(c.x, c.y);
      }
#pragma unroll
      for (int dx = 0; dx < 7; ++dx) {
        const float4 wv = __ldg(reinterpret_cast<const float4*>(w + (long long)(dy * 7 + dx) * C + c0 + cg * 4));
        const uint64_t w0 = pack2(wv.x, wv.y), w1 = pack2(wv.z, wv.w);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          acc[i][0] = fma2(in[i + dx][0], w0, acc[i][0]);
          acc[i][1] = fma2(in[i + dx][1], w1, acc[i][1]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float a0, a1, a2, a3;
      unpack2(acc[i][0], a0, a1);
      unpack2(acc[i][1], a2, a3);
      *reinterpret_cast<uint2*>(ys + (r * TW + xh + i) * DWL_YS_LD + nloc * DW_CB + cg * 4) =
          make_uint2(pack_half2(a0, a1), pack_half2(a2, a3));
    }
  }
  __syncthreads();
  // LayerNorm + quantisation: warp per pixel; lane l holds 8 channels of local chunk l / 8 (global chunk rank + K * (l / 8))
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool mine = lane < nloc * 8;
  const int col = (rank + K * (lane >> 3)) * DW_CB + (lane & 7) * 8;
  const auto load = [&](int p, float (&f)[8]) {
    const uint4 u = mine ? *reinterpret_cast<const uint4*>(ys + p * DWL_YS_LD + lane * 8) : make_uint4(0u, 0u, 0u, 0u);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int k = 0; k < 4; ++k) { const float2 v = __half22float2(h[k]); f[2 * k] = v.x; f[2 * k + 1] = v.y; }
  };
  // a pixel's value over the cluster's blocks: lane k < K reads block k's partial (one distributed-shared-memory load per
  // lane, not K dependent ones per lane), then every lane combines them in rank order, so the result does not depend on
  // scheduling
  const auto gather = [&](int which, int p) { return lane < K ? cluster.map_shared_rank(&part[which][0], lane)[p] : 0.f; };
  const auto total = [&](int which, int p) {
    const float g = gather(which, p);
    float v = 0.f;
    for (int k = 0; k < K; ++k) v += __shfl_sync(0xffffffffu, g, k);
    return v;
  };
  const auto total_max = [&](int p) {
    const float g = gather(2, p);
    float v = 0.f;
    for (int k = 0; k < K; ++k) v = fmaxf(v, __shfl_sync(0xffffffffu, g, k));
    return v;
  };
  for (int p = warp; p < DWL_PX; p += 8) {
    float f[8];
    load(p, f);
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += f[k];
    s = warp_sum(mine ? s : 0.f);
    if (lane == 0) part[0][p] = s;
  }
  cluster.sync();
  float mean[DWL_PX / 8];
  #pragma unroll
  for (int i = 0; i < DWL_PX / 8; ++i) {
    const int p = warp + 8 * i;
    float f[8];
    load(p, f);
    mean[i] = total(0, p) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) q += (f[k] - mean[i]) * (f[k] - mean[i]);
    q = warp_sum(mine ? q : 0.f);
    if (lane == 0) part[1][p] = q;
  }
  cluster.sync();
  float wk[8], bk[8];
  if (mine) {
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(ln_w + col)), w1 = __ldg(reinterpret_cast<const float4*>(ln_w + col + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(ln_b + col)), b1 = __ldg(reinterpret_cast<const float4*>(ln_b + col + 4));
    wk[0] = w0.x; wk[1] = w0.y; wk[2] = w0.z; wk[3] = w0.w; wk[4] = w1.x; wk[5] = w1.y; wk[6] = w1.z; wk[7] = w1.w;
    bk[0] = b0.x; bk[1] = b0.y; bk[2] = b0.z; bk[3] = b0.w; bk[4] = b1.x; bk[5] = b1.y; bk[6] = b1.z; bk[7] = b1.w;
  }
  float rstd[DWL_PX / 8];
  #pragma unroll
  for (int i = 0; i < DWL_PX / 8; ++i) {
    const int p = warp + 8 * i;
    float f[8];
    load(p, f);
    rstd[i] = rsqrtf(total(1, p) / (float)C + 1e-6f);
    float am = 0.f;
    if (mine) {
#pragma unroll
      for (int k = 0; k < 8; ++k) am = fmaxf(am, fabsf((f[k] - mean[i]) * rstd[i] * wk[k] + bk[k]));
    }
    am = warp_max(am);
    if (lane == 0) part[2][p] = am;
  }
  cluster.sync();
  #pragma unroll
  for (int i = 0; i < DWL_PX / 8; ++i) {
    const int p = warp + 8 * i;
    const int gy = ty0 + p / TW, gx = tx0 + p % TW;
    if (gy >= H || gx >= W) continue;              // outside the map: computed for the statistics' shape only
    const E4m3Row e(total_max(p));
    const long long row = ((long long)b * H + gy) * W + gx;
    if (rank == 0 && lane == 0) out_scale[row] = e.scale;
    if (mine) {
      float f[8];
      load(p, f);
      float y[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) y[k] = (f[k] - mean[i]) * rstd[i] * wk[k] + bk[k];    // the expression of the amax pass
      *reinterpret_cast<uint2*>(out + row * C + col) = make_uint2(e.q4(y[0], y[1], y[2], y[3]), e.q4(y[4], y[5], y[6], y[7]));
    }
  }
  cluster.sync();                                  // no block leaves while another still reads its partials
}

// running element-wise maximum over a stage's block outputs (decoder.py:371-374 `max_stack`): dst = first ? src : max(dst, src)
__global__ void __launch_bounds__(256) max_accum_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, long long n8, int first) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    uint4 s = src[i];
    if (!first) {
      const uint4 d = dst[i];
      __half2* sh = reinterpret_cast<__half2*>(&s);
      const __half2* dh = reinterpret_cast<const __half2*>(&d);
#pragma unroll
      for (int j = 0; j < 4; ++j) sh[j] = __hmax2(sh[j], dh[j]);
    }
    dst[i] = s;
  }
}

// the same running maximum over f32 values (split-precision mode keeps the encoder levels in f32)
__global__ void __launch_bounds__(256) max_accum_f32_kernel(const float4* __restrict__ src, float4* __restrict__ dst, long long n4, int first) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 s = src[i];
    if (!first) {
      const float4 d = dst[i];
      s = make_float4(fmaxf(s.x, d.x), fmaxf(s.y, d.y), fmaxf(s.z, d.z), fmaxf(s.w, d.w));
    }
    dst[i] = s;
  }
}

// DINOv2 block output -> decoder level (unidepthv1.py:322-326, decoder.py:371-379): one thread per 8 channels of a patch
// token, acc = first ? f16(x_tok + x_cls) : max(acc, f16(x_tok + x_cls)); the trailing B*D/8 work items copy the raw cls
// rows to cls_out.  HBM-bound: 32 B of x read and 16 (first) or 32 B of acc moved per item; the cls row stays in L1/L2.
// F32: the level is kept in f32 (split-precision mode), acc holds 2 x uint4 = 8 floats per item, no rounding.
template <bool F32>
__global__ void __launch_bounds__(256) vit_tap_kernel(const float* __restrict__ x, uint4* __restrict__ acc, float* __restrict__ cls_out,
                                                     int B, int N, int D, int first) {
  const int d8 = D / 8;
  const long long n_acc = (long long)B * N * d8;
  const long long total = n_acc + (cls_out ? (long long)B * d8 : 0);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    if (i >= n_acc) {
      const long long j = i - n_acc;
      const int b = (int)(j / d8), c = (int)(j % d8) * 8;
      const float4* src = reinterpret_cast<const float4*>(x + (long long)b * (N + 1) * D + c);
      float4* dst = reinterpret_cast<float4*>(cls_out + (long long)b * D + c);
      dst[0] = src[0];
      dst[1] = src[1];
      continue;
    }
    const int c = (int)(i % d8) * 8;
    const long long r = i / d8;                     // b*N + t
    const int b = (int)(r / N);
    const long long t = r - (long long)b * N;
    const float4* tok = reinterpret_cast<const float4*>(x + ((long long)b * (N + 1) + 1 + t) * D + c);
    const float4* cls = reinterpret_cast<const float4*>(x + (long long)b * (N + 1) * D + c);
    const float4 a0 = tok[0], a1 = tok[1], c0 = __ldg(cls), c1 = __ldg(cls + 1);
    if (F32) {
      float4 s0 = make_float4(a0.x + c0.x, a0.y + c0.y, a0.z + c0.z, a0.w + c0.w);
      float4 s1 = make_float4(a1.x + c1.x, a1.y + c1.y, a1.z + c1.z, a1.w + c1.w);
      float4* af = reinterpret_cast<float4*>(acc) + 2 * i;
      if (!first) {
        const float4 d0 = af[0], d1 = af[1];
        s0 = make_float4(fmaxf(s0.x, d0.x), fmaxf(s0.y, d0.y), fmaxf(s0.z, d0.z), fmaxf(s0.w, d0.w));
        s1 = make_float4(fmaxf(s1.x, d1.x), fmaxf(s1.y, d1.y), fmaxf(s1.z, d1.z), fmaxf(s1.w, d1.w));
      }
      af[0] = s0;
      af[1] = s1;
      continue;
    }
    uint4 v = make_uint4(pack_half2(a0.x + c0.x, a0.y + c0.y), pack_half2(a0.z + c0.z, a0.w + c0.w),
                         pack_half2(a1.x + c1.x, a1.y + c1.y), pack_half2(a1.z + c1.z, a1.w + c1.w));
    if (!first) {
      const uint4 d = acc[i];
      __half2* vh = reinterpret_cast<__half2*>(&v);
      const __half2* dh = reinterpret_cast<const __half2*>(&d);
#pragma unroll
      for (int j = 0; j < 4; ++j) vh[j] = __hmax2(vh[j], dh[j]);
    }
    acc[i] = v;
  }
}

// spatial mean of an NHWC f32 map -> [B, C] f32 (ConvNeXt "cls tokens", convnext.py:471)
__global__ void __launch_bounds__(256) spatial_mean_kernel(const float* __restrict__ x, float* __restrict__ out, int HW, int C) {
  const int b = blockIdx.y;
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int part = threadIdx.x >> 5;   // 8 row groups
  __shared__ float red[8][33];
  float s = 0.f;
  if (c < C)
    for (int i = part; i < HW; i += 8) s += x[((long long)b * HW + i) * C + c];
  red[part][threadIdx.x & 31] = s;
  __syncthreads();
  if (part == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x & 31];
    out[(long long)b * C + c] = t / (float)HW;
  }
}

// antialiased bilinear resize of an NHWC f16 or f32 map (flat_interpolate, geometric.py:228-252): one thread per 8
// channels; the same weights and summation order for both element types
__device__ __forceinline__ void load8(const __half* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int q = 0; q < 4; ++q) { const float2 t = __half22float2(h[q]); f[2 * q] = t.x; f[2 * q + 1] = t.y; }
}
__device__ __forceinline__ void load8(const float* p, float (&f)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void store8(__half* p, const float (&f)[8]) {
  *reinterpret_cast<uint4*>(p) = make_uint4(pack_half2(f[0], f[1]), pack_half2(f[2], f[3]), pack_half2(f[4], f[5]), pack_half2(f[6], f[7]));
}
__device__ __forceinline__ void store8(float* p, const float (&f)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
}

template <class T>
__global__ void __launch_bounds__(256) aa_resize_nhwc_kernel(const T* __restrict__ in, T* __restrict__ out, int B, int H, int W, int C,
                                                            int oh, int ow, float sh, float sw) {
  const int cv = C >> 3;
  const long long total = (long long)B * oh * ow * cv;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(idx % cv);
    const long long pix = idx / cv;
    const int ox = (int)(pix % ow), oy = (int)((pix / ow) % oh), b = (int)(pix / ((long long)ow * oh));
    const AAxis ay = aa_axis(oy, H, sh), ax = aa_axis(ox, W, sw);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int jy = 0; jy < ay.xsize; ++jy) {
      float r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = 0.f;
      for (int jx = 0; jx < ax.xsize; ++jx) {
        float f[8];
        load8(in + (((long long)b * H + ay.xmin + jy) * W + ax.xmin + jx) * C + c8 * 8, f);
        const float wx = ax.w(jx);
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] += wx * f[j];
      }
      const float wy = ay.w(jy);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += wy * r[j];
    }
    store8(out + pix * C + c8 * 8, acc);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Ray embedding of one decoder level (decoder.py:203-220): unit rays of the pinhole K at network resolution
// (generate_rays, geometric.py:13-45) are never materialised -- each token antialias-averages the analytic rays of its
// window (flat_interpolate), re-normalises, evaluates the 81 real spherical harmonics up to degree 8 by recurrence
// (rsh_cart_8, sht.py:833; same index l*(l+1)+m) and applies the MLP's input LayerNorm (81 wide, eps 1e-5).  Output
// f16 [B*gh*gw, 128], columns >= 81 zero (the projection GEMM's K is zero-extended).  One warp per token.
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rays_sh81_kernel(const udb_v1_rays_t p) {
  const long long tok = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (tok >= (long long)p.B * p.gh * p.gw) return;
  const int gx = (int)(tok % p.gw), gy = (int)((tok / p.gw) % p.gh), b = (int)(tok / ((long long)p.gw * p.gh));
  const float fx = p.intr4[b * 4], fy = p.intr4[b * 4 + 1], cx = p.intr4[b * 4 + 2], cy = p.intr4[b * 4 + 3];
  const float sh = (float)p.net_h / (float)p.gh, sw = (float)p.net_w / (float)p.gw;
  const AAxis ay = aa_axis(gy, p.net_h, sh), ax = aa_axis(gx, p.net_w, sw);
  float rx = 0.f, ry = 0.f, rz = 0.f;
  const int taps = ay.xsize * ax.xsize;
  for (int t = lane; t < taps; t += 32) {
    const int jy = t / ax.xsize, jx = t % ax.xsize;
    const float dx = ((float)(ax.xmin + jx) + 0.5f - cx) / fx, dy = ((float)(ay.xmin + jy) + 0.5f - cy) / fy;
    const float inv = 1.0f / fmaxf(sqrtf(dx * dx + dy * dy + 1.0f), 1e-12f);
    const float wgt = ay.w(jy) * ax.w(jx);
    rx += wgt * dx * inv;
    ry += wgt * dy * inv;
    rz += wgt * inv;
  }
  rx = warp_sum(rx); ry = warp_sum(ry); rz = warp_sum(rz);
  {
    const float inv = 1.0f / fmaxf(sqrtf(rx * rx + ry * ry + rz * rz), 1e-12f);
    rx *= inv; ry *= inv; rz *= inv;
  }
  // every lane evaluates the recurrence (cheap, keeps the warp converged) and keeps the entries it stores
  float mine[3] = {0.f, 0.f, 0.f};
  float sum = 0.f, sq = 0.f;
  float A = 1.f, Bm = 0.f, pmm = 1.f;
  for (int m = 0; m <= 8; ++m) {
    if (m > 0) {
      const float a2 = rx * A - ry * Bm, b2 = rx * Bm + ry * A;
      A = a2; Bm = b2;
      pmm *= -(float)(2 * m - 1);
    }
    float pprev = 0.f, pcur = pmm;
    for (int l = m; l <= 8; ++l) {
      if (l == m + 1) { pprev = pcur; pcur = (float)(2 * m + 1) * rz * pcur; }
      else if (l > m + 1) { const float t = ((float)(2 * l - 1) * rz * pcur - (float)(l + m - 1) * pprev) / (float)(l - m); pprev = pcur; pcur = t; }
      const float k = p.sh_k[l * 9 + m];
      if (m == 0) {
        const float v = k * pcur;
        const int id = l * (l + 1);
        sum += v; sq += v * v;
        if ((id & 31) == lane) mine[id >> 5] = v;
      } else {
        const float va = k * A * pcur, vb = k * Bm * pcur;
        const int ia = l * (l + 1) + m, ib = l * (l + 1) - m;
        sum += va + vb; sq += va * va + vb * vb;
        if ((ia & 31) == lane) mine[ia >> 5] = va;
        if ((ib & 31) == lane) mine[ib >> 5] = vb;
      }
    }
  }
  const float mean = sum / 81.f;
  // two-pass variance from the stored entries (each lane holds up to 3 of the 81)
  float v = 0.f;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const int id = lane + 32 * j;
    if (id < 81) v += (mine[j] - mean) * (mine[j] - mean);
  }
  (void)sq;
  const float rstd = rsqrtf(warp_sum(v) / 81.f + 1e-5f);
  __half* o = reinterpret_cast<__half*>(p.out) + tok * 128;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int id = lane + 32 * j;
    float y = 0.f;
    if (id < 81) y = (mine[j < 3 ? j : 0] - mean) * rstd * p.ln_w[id] + p.ln_b[id];
    o[id] = __float2half_rn(y);
  }
}

// V1 camera head tail (decoder.py:96-106,326-331; unidepthv1.py:88-91): x4 = (log fx', log fy', logit cx', logit cy') ->
// K at network resolution (intr4 = fx, fy, cx, cy) and the intrinsics returned to the caller (un-padded, / ratio).
// With GT intrinsics: K_net = K*ratio (+pads) (unidepthv1.py:56-62); skip_camera returns the GT K instead of the prediction.
__global__ void v1_camera_intrinsics_kernel(const float* x4, const float* gt_k, int B, int net_h, int net_w, float ratio, int pad_l, int pad_t,
                                            int skip_camera, float* intr4_rays, float* k_out, float* k4_points) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float fx = 0.f, fy = 0.f, cx = 0.f, cy = 0.f;
  if (x4) {
    const float4 k = decode_camera(x4 + b * 4, (float)max(net_h, net_w) / 2.0f, net_h, net_w);
    fx = k.x; fy = k.y; cx = k.z; cy = k.w;
  }
  float rfx = fx, rfy = fy, rcx = cx, rcy = cy;     // K the rays are generated from
  if (gt_k) {
    rfx = gt_k[b * 9] * ratio;
    rfy = gt_k[b * 9 + 4] * ratio;
    rcx = gt_k[b * 9 + 2] * ratio + (float)pad_l;
    rcy = gt_k[b * 9 + 5] * ratio + (float)pad_t;
    if (skip_camera || !x4) { fx = rfx; fy = rfy; cx = rcx; cy = rcy; }
  }
  intr4_rays[b * 4] = rfx; intr4_rays[b * 4 + 1] = rfy; intr4_rays[b * 4 + 2] = rcx; intr4_rays[b * 4 + 3] = rcy;
  float* k = k_out + b * 9;
  store_k3(k, fx / ratio, fy / ratio, (cx - (float)pad_l) / ratio, (cy - (float)pad_t) / ratio);
  // K the final back-projection uses on the ORIGINAL pixel grid (unidepthv1.py:354-356): the pre-processed GT K when one
  // was given (the reference does not undo its resize there), else the returned prediction
  float* kp = k4_points + b * 4;
  if (gt_k) { kp[0] = rfx; kp[1] = rfy; kp[2] = rcx; kp[3] = rcy; }
  else { kp[0] = k[0]; kp[1] = k[4]; kp[2] = k[2]; kp[3] = k[5]; }
}

// 4-query cross attention of the camera head (decoder.py:95, AttentionBlock num_heads=1): q f32 [B*nq, D] (+ q_pos), kv f16
// [B*nk, 2D] (k | v), out f32 [B*nq, D].  Keys are split over CA_SPLITS blocks per image (flash-decoding style): each block
// reads its slice of K and V ONCE for all queries and writes a partial (max, sum, weighted V); a second kernel merges.
// KV = float: the same kernel on f32 keys and values (split-precision mode), same summation order.
constexpr int CA_SPLITS = 16, CA_MAXQ = 4;

__device__ __forceinline__ float2 load2(const __half* p) { return __half22float2(*reinterpret_cast<const __half2*>(p)); }
__device__ __forceinline__ float2 load2(const float* p) { return *reinterpret_cast<const float2*>(p); }
__device__ __forceinline__ void ldg8(const __half* p, float (&f)[8]) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int t = 0; t < 4; ++t) { const float2 v = __half22float2(h[t]); f[2 * t] = v.x; f[2 * t + 1] = v.y; }
}
__device__ __forceinline__ void ldg8(const float* p, float (&f)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p + 4));
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

template <class KV>
__global__ void __launch_bounds__(256) cross_attn_partial_kernel(const float* __restrict__ q, const float* __restrict__ q_pos,
                                                                const KV* __restrict__ kv, float* __restrict__ part, int nq, int nk, int D,
                                                                float scale) {
  extern __shared__ float sm[];
  const int chunk = (nk + CA_SPLITS - 1) / CA_SPLITS;
  float* qs = sm;                       // [nq][D]
  float* sc = qs + nq * D;              // [nq][chunk]
  float* red = sc + nq * chunk;         // [nq][8] partial max / sum
  const int b = blockIdx.y, sp = blockIdx.x;
  const int j0 = sp * chunk, j1 = min(nk, j0 + chunk), n = max(j1 - j0, 0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < nq * D; i += 256)
    qs[i] = (q[(long long)b * nq * D + i] + (q_pos ? q_pos[i] : 0.f)) * scale;
  __syncthreads();
  const KV* kb = kv + (long long)b * nk * 2 * D;
  for (int j = warp; j < n; j += 8) {
    float a[CA_MAXQ] = {0.f, 0.f, 0.f, 0.f};
    const KV* kr = kb + (long long)(j0 + j) * 2 * D;
    for (int d = lane * 8; d < D; d += 256) {
      float kf[8];
      ldg8(kr + d, kf);
#pragma unroll
      for (int qi = 0; qi < CA_MAXQ; ++qi)
        if (qi < nq) {
#pragma unroll
          for (int t = 0; t < 8; ++t) a[qi] = fmaf(qs[qi * D + d + t], kf[t], a[qi]);
        }
    }
#pragma unroll
    for (int qi = 0; qi < CA_MAXQ; ++qi)
      if (qi < nq) {
        const float v = warp_sum(a[qi]);
        if (lane == 0) sc[qi * chunk + j] = v;
      }
  }
  __syncthreads();
  // per query: max, exp, sum over this block's keys (warp qi handles query qi)
  if (warp < nq) {
    float m = -INFINITY;
    for (int j = lane; j < n; j += 32) m = fmaxf(m, sc[warp * chunk + j]);
    m = warp_max(m);
    float l = 0.f;
    for (int j = lane; j < n; j += 32) {
      const float e = expf(sc[warp * chunk + j] - m);
      sc[warp * chunk + j] = e;
      l += e;
    }
    l = warp_sum(l);
    if (lane == 0) { red[warp * 2] = m; red[warp * 2 + 1] = l; }
  }
  __syncthreads();
  float* pb = part + ((long long)(b * CA_SPLITS + sp) * nq) * (D + 2);
  for (int d = threadIdx.x * 2; d < D; d += 512) {
    float acc[CA_MAXQ][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};
    for (int j = 0; j < n; ++j) {
      const float2 vf = load2(kb + (long long)(j0 + j) * 2 * D + D + d);
#pragma unroll
      for (int qi = 0; qi < CA_MAXQ; ++qi)
        if (qi < nq) {
          const float pw = sc[qi * chunk + j];
          acc[qi][0] = fmaf(pw, vf.x, acc[qi][0]);
          acc[qi][1] = fmaf(pw, vf.y, acc[qi][1]);
        }
    }
    for (int qi = 0; qi < nq; ++qi) {
      pb[qi * (D + 2) + 2 + d] = acc[qi][0];
      pb[qi * (D + 2) + 2 + d + 1] = acc[qi][1];
    }
  }
  if (threadIdx.x < nq) {
    pb[threadIdx.x * (D + 2)] = n > 0 ? red[threadIdx.x * 2] : -INFINITY;
    pb[threadIdx.x * (D + 2) + 1] = n > 0 ? red[threadIdx.x * 2 + 1] : 0.f;
  }
}

__global__ void __launch_bounds__(256) cross_attn_merge_kernel(const float* __restrict__ part, float* __restrict__ out, int nq, int D) {
  const int b = blockIdx.y, qi = blockIdx.x;
  float m = -INFINITY;
  for (int s = 0; s < CA_SPLITS; ++s) m = fmaxf(m, part[((long long)(b * CA_SPLITS + s) * nq + qi) * (D + 2)]);
  float wgt[CA_SPLITS], tot = 0.f;
#pragma unroll
  for (int s = 0; s < CA_SPLITS; ++s) {
    const float* pp = part + ((long long)(b * CA_SPLITS + s) * nq + qi) * (D + 2);
    wgt[s] = expf(pp[0] - m);
    tot += wgt[s] * pp[1];
  }
  const float inv = 1.0f / tot;
  for (int d = threadIdx.x; d < D; d += 256) {
    float a = 0.f;
#pragma unroll
    for (int s = 0; s < CA_SPLITS; ++s) a = fmaf(wgt[s], part[((long long)(b * CA_SPLITS + s) * nq + qi) * (D + 2) + 2 + d], a);
    out[((long long)b * nq + qi) * D + d] = a * inv;
  }
}

// softmax over the first n_valid columns of f32 rows [rows, ld_in] -> f16 probabilities [rows, ld_out] (columns
// n_valid .. ld_out-1 zero): the P operand of the dense single-head attentions (aggregate_16 / prompt_camera).
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ s, __half* __restrict__ p, long long rows, int n_valid,
                                                          int ld_in, int ld_out, float scale) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* sr = s + row * ld_in;
  float m = -INFINITY;
  for (int j = lane; j < n_valid; j += 32) m = fmaxf(m, sr[j]);
  m = warp_max(m);
  float tot = 0.f;
  for (int j = lane; j < n_valid; j += 32) tot += expf((sr[j] - m) * scale);
  tot = warp_sum(tot);
  const float inv = 1.0f / tot;
  __half* pr = p + row * ld_out;
  for (int j = lane; j < ld_out; j += 32) pr[j] = __float2half_rn(j < n_valid ? expf((sr[j] - m) * scale) * inv : 0.f);
}

// out[i] = a[i] + b[i] (f32, + optional f16 copy): `latents + rays_embedding` before each ConvUpsample (decoder.py:246-252)
__global__ void __launch_bounds__(256) add_f32_kernel(const float4* __restrict__ a, const float4* __restrict__ b, float4* __restrict__ o,
                                                     uint2* __restrict__ o16, long long n4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 x = a[i], y = b[i];
    const float4 r = make_float4(x.x + y.x, x.y + y.y, x.z + y.z, x.w + y.w);
    if (o) o[i] = r;
    if (o16) o16[i] = make_uint2(pack_half2(r.x, r.y), pack_half2(r.z, r.w));
  }
}

// f32 rows -> f16 rows with independent row strides (cls tokens appended to the camera head's context, decoder.py:94)
__global__ void copy_rows_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst, int groups, int rows_per_group, int D,
                                     long long dst_group_stride, long long dst_row0) {
  const long long total = (long long)groups * rows_per_group * D;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(i % D);
    const long long r = i / D;
    const long long g = r / rows_per_group, rr = r % rows_per_group;
    dst[(g * dst_group_stride + dst_row0 + rr) * D + d] = __float2half_rn(src[i]);
  }
}

// 3x3 convolution with ONE output channel, zero padding, fused exp(clamp(., -10, 10)) (decoder.py:253,268,283,292-294
// `out8/out4/out2`): NHWC f16 in, f32 plane out.  One warp per output pixel, lanes over channel pairs.
template <int LPP>      // lanes per pixel = C / 8 (8, 16 or 32): each lane owns 8 channels (one 16-byte load per tap)
__global__ void __launch_bounds__(256) conv3x3_c1_kernel(const __half* __restrict__ x, const float* __restrict__ w, float bias, float* __restrict__ out,
                                                        int B, int H, int W, int C) {
  constexpr int PPW = 32 / LPP;                      // pixels per warp
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPP;
  const long long pix = ((long long)blockIdx.x * 8 + (threadIdx.x >> 5)) * PPW + lane / LPP;
  const bool live = pix < (long long)B * H * W;
  const long long pc = live ? pix : 0;
  const int px = (int)(pc % W), py = (int)((pc / W) % H), b = (int)(pc / ((long long)W * H));
  float a = 0.f;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int yy = py + t / 3 - 1, xx = px + t % 3 - 1;
    if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(x + (((long long)b * H + yy) * W + xx) * C + sub * 8));
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(w + t * C + sub * 8)), w1 = __ldg(reinterpret_cast<const float4*>(w + t * C + sub * 8 + 4));
    const __half2* h = reinterpret_cast<const __half2*>(&u);
    const float2 f0 = __half22float2(h[0]), f1 = __half22float2(h[1]), f2 = __half22float2(h[2]), f3 = __half22float2(h[3]);
    a = fmaf(f0.x, w0.x, fmaf(f0.y, w0.y, fmaf(f1.x, w0.z, fmaf(f1.y, w0.w, a))));
    a = fmaf(f2.x, w1.x, fmaf(f2.y, w1.y, fmaf(f3.x, w1.z, fmaf(f3.y, w1.w, a))));
  }
#pragma unroll
  for (int o = LPP / 2; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (live && sub == 0) out[pix] = expf(fminf(fmaxf(a + bias, -10.0f), 10.0f));
}

// ------------------------------------------------------------------------------------------------------------------
// Nystrom attention pieces (layers/nystrom_attention.py:22-84 -> xformers NystromAttention(num_landmarks=128); the
// restated algorithm is in oracle/unidepth_v1_oracle.py, PARITY UNPINNED).  Landmarks = segment means of q and k.
// q lives in qbuf [B*n, ldq] (cols h*64..), k in kvbuf [B*n, ldkv]; out f16 [B*128, 2*heads*64] = (q landmarks | k landmarks).
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(64) nystrom_landmarks_kernel(const __half* __restrict__ q, int ldq, const __half* __restrict__ kv, int ldkv,
                                                              __half* __restrict__ out, int n, int heads, int m) {
  const int lm = blockIdx.x, h = blockIdx.y, b = blockIdx.z, d = threadIdx.x;
  const int seg = n / m, n_round = m - n % m;      // first n_round segments have `seg` rows, the rest seg + 1
  int start, len;
  if (n % m == 0 || lm < n_round) { start = lm * seg; len = seg; }
  else { start = n_round * seg + (lm - n_round) * (seg + 1); len = seg + 1; }
  float sq = 0.f, sk = 0.f;
  for (int r = 0; r < len; ++r) {
    const long long row = (long long)b * n + start + r;
    sq += __half2float(q[row * ldq + h * 64 + d]);
    sk += __half2float(kv[row * ldkv + h * 64 + d]);
  }
  __half* o = out + ((long long)b * m + lm) * (2 * heads * 64);
  o[h * 64 + d] = __float2half_rn(sq / (float)len);
  o[heads * 64 + h * 64 + d] = __float2half_rn(sk / (float)len);
}

// kernel_2 = softmax(q_landmarks . k_landmarks^T / sqrt(64)) per (b, head): f32 [B*heads, 128, 128].  One warp per row.
__global__ void __launch_bounds__(128) nystrom_k2_kernel(const __half* __restrict__ lmk, float* __restrict__ k2, int heads, int m) {
  const int bh = blockIdx.y, b = bh / heads, h = bh % heads;
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= m) return;
  const int ld = 2 * heads * 64;
  const __half* qr = lmk + ((long long)b * m + row) * ld + h * 64;
  float qv[2];
  qv[0] = __half2float(qr[lane * 2]);
  qv[1] = __half2float(qr[lane * 2 + 1]);
  float s[4];      // m == 128: 4 columns per lane
  float mx = -INFINITY;
  for (int j = 0; j < 4; ++j) {
    const int col = lane + 32 * j;
    const __half* kr = lmk + ((long long)b * m + col) * ld + heads * 64 + h * 64;
    float a = 0.f;
    for (int d = 0; d < 64; d += 2) {
      const float2 kf = __half22float2(*reinterpret_cast<const __half2*>(kr + d));
      const float q0 = __shfl_sync(0xffffffffu, qv[0], d >> 1), q1 = __shfl_sync(0xffffffffu, qv[1], d >> 1);
      a = fmaf(q0, kf.x, fmaf(q1, kf.y, a));
    }
    s[j] = a * 0.125f;
    mx = fmaxf(mx, s[j]);
  }
  mx = warp_max(mx);
  float tot = 0.f;
  for (int j = 0; j < 4; ++j) { s[j] = expf(s[j] - mx); tot += s[j]; }
  tot = warp_sum(tot);
  for (int j = 0; j < 4; ++j) k2[((long long)bh * m + row) * m + lane + 32 * j] = s[j] / tot;
}

// Z0 = K^T / max_j(sum_i K[i][j]) (exact 1/||K||_1 initialisation of the Newton-Schulz iteration), per matrix
__global__ void __launch_bounds__(128) nystrom_pinv_init_kernel(const float* __restrict__ k2, float* __restrict__ z, int m) {
  const float* K = k2 + (long long)blockIdx.x * m * m;
  float* Z = z + (long long)blockIdx.x * m * m;
  __shared__ float red[4];
  const int j = threadIdx.x;      // m == 128 threads: column sums
  float cs = 0.f;
  for (int i = 0; i < m; ++i) cs += K[i * m + j];
  float mx = warp_max(cs);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  const float inv = 1.0f / mx;
  for (int i = 0; i < m; ++i) Z[j * m + i] = K[i * m + j] * inv;     // Z[j][i] = K[i][j] / ||K||_1
}

// T = c*I - X over a batch of m x m matrices
__global__ void __launch_bounds__(256) eye_minus_kernel(const float* __restrict__ x, float* __restrict__ t, float c, int m, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(i % ((long long)m * m));
    t[i] = ((e / m) == (e % m) ? c : 0.f) - x[i];
  }
}

// batched small matmul, f32:  C = diag * I + alpha * (A @ B), A [M,K], B [K,N] (f32, or f16 with row stride ldb),
// C [M,N] f32 or f16 with row stride ldc.
struct BmmArgs {
  const float* A; long long sA; int lda;
  const void* Bp; long long sB1, sB2; int ldb; int b_f16; int inner;   // batch index bh -> (bh / inner, bh % inner) for B and C strides
  void* C; long long sC1, sC2; int ldc; int c_f16;
  int M, N, K;
  float alpha, diag;
};
__global__ void __launch_bounds__(256) bmm_f32_kernel(const BmmArgs p) {
  // 64 x 64 output tile per block, 4 x 4 per thread, K in steps of 16 through shared memory
  __shared__ float As[16][64 + 4], Bs[16][64 + 4];
  const int bh = blockIdx.z, o = bh / p.inner, i2 = bh % p.inner;
  const float* A = p.A + (long long)bh * p.sA;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;      // outputs rows ty*4.., cols tx*4..
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < p.K; k0 += 16) {
    // A tile 64 x 16 (stored transposed [k][m]); B tile 16 x 64
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int idx = threadIdx.x + 256 * t;             // 1024 elements each
      const int am = idx >> 4, ak = idx & 15;
      const int mm = m0 + am, kk = k0 + ak;
      As[ak][am] = (mm < p.M && kk < p.K) ? A[(long long)mm * p.lda + kk] : 0.f;
      const int bk = idx >> 6, bn = idx & 63;
      const int kr = k0 + bk, nn = n0 + bn;
      float bv = 0.f;
      if (kr < p.K && nn < p.N) {
        const long long off = o * p.sB1 + i2 * p.sB2 + (long long)kr * p.ldb + nn;
        bv = p.b_f16 ? __half2float(reinterpret_cast<const __half*>(p.Bp)[off]) : reinterpret_cast<const float*>(p.Bp)[off];
      }
      Bs[bk][bn] = bv;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float a[4] = {av.x, av.y, av.z, av.w}, bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int mm = m0 + ty * 4 + i, nn = n0 + tx * 4 + j;
      if (mm < p.M && nn < p.N) {
        const float v = p.alpha * acc[i][j] + (mm == nn ? p.diag : 0.f);
        const long long off = o * p.sC1 + i2 * p.sC2 + (long long)mm * p.ldc + nn;
        if (p.c_f16) reinterpret_cast<__half*>(p.C)[off] = __float2half_rn(v);
        else reinterpret_cast<float*>(p.C)[off] = v;
      }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// V1 post-processing (unidepthv1.py:66-94,352-366).  Stage 1: the three exp'ed maps are antialias-resized to the
// network shape and averaged.  Stage 2: crop the paddings, antialias-resize to the original size -> depth (z), and
// back-project with (theta, phi) of the unit ray through each original pixel: x = z tan(theta) = z rx/rz,
// y = z / tan(phi) / cos(theta) (spherical_zbuffer_to_euclidean, geometric.py:57-73).
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) v1_mean_maps_kernel(const float* __restrict__ o8, const float* __restrict__ o4, const float* __restrict__ o2,
                                                          float* __restrict__ mean, int B, int gh, int gw, int net_h, int net_w) {
  const long long total = (long long)B * net_h * net_w;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(idx % net_w), Y = (int)((idx / net_w) % net_h), b = (int)(idx / ((long long)net_w * net_h));
    float tot = 0.f;
#pragma unroll
    for (int lvl = 0; lvl < 3; ++lvl) {
      const int h = gh << (lvl + 1), w = gw << (lvl + 1);
      const float* src = (lvl == 0 ? o8 : (lvl == 1 ? o4 : o2)) + (long long)b * h * w;
      tot += aa_sample(src, aa_axis(Y, h, (float)h / (float)net_h), aa_axis(X, w, (float)w / (float)net_w), w);
    }
    mean[idx] = tot / 3.0f;
  }
}

__global__ void __launch_bounds__(256) v1_postprocess_kernel(const udb_v1_postprocess_t p) {
  const long long total = (long long)p.B * p.H * p.W;
  const int ch = p.net_h - p.pad_t - p.pad_b, cw = p.net_w - p.pad_l - p.pad_r;     // cropped size
  const float sh = (float)ch / (float)p.H, sw = (float)cw / (float)p.W;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(idx % p.W), Y = (int)((idx / p.W) % p.H), b = (int)(idx / ((long long)p.W * p.H));
    const float* src = p.mean + (long long)b * p.net_h * p.net_w + (long long)p.pad_t * p.net_w + p.pad_l;   // the crop
    const float z = aa_sample(src, aa_axis(Y, ch, sh), aa_axis(X, cw, sw), p.net_w);
    const long long hw = (long long)p.H * p.W, pix = (long long)Y * p.W + X;
    p.out_depth[b * hw + pix] = z;
    backproject(p.k4 + b * 4, X, Y, z, p.out_points + b * 3 * hw + pix, hw);   // k4: the K the points are generated with
  }
}

// udb_v1_preprocess (f16 patch rows) and udb_v1_preprocess_split ([hi | lo] rows), errors under the name `fn`
template <bool SPLIT>
static int v1_preprocess(const char* fn, const udb_v1_preprocess_t* p, void* stream) {
  const float sh = (float)p->H / (float)p->rh, sw = (float)p->W / (float)p->rw;
  if (p->patch == 14) {
    if (p->net_h % 14 || p->net_w % 14) { set_error("%s: network shape %dx%d is not a multiple of 14", fn, p->net_h, p->net_w); return 1; }
    const int gh = p->net_h / 14, gw = p->net_w / 14;
    v1_preprocess_kernel<14, SPLIT><<<grid_1d((long long)p->B * gh * gw * 80, 32), 256, 0, ST(stream)>>>(*p, gh, gw, sh, sw);
    return check_launch(SPLIT ? "v1_preprocess_split_kernel<14>" : "v1_preprocess_kernel<14>");
  }
  if (p->patch != 0 && p->patch != 4) { set_error("%s: patch %d unsupported (0 / 4 or 14)", fn, p->patch); return 1; }
  if (p->net_h < 4 || p->net_w < 4) { set_error("%s: bad network shape", fn); return 1; }
  const int gh = (p->net_h - 4) / 4 + 1, gw = (p->net_w - 4) / 4 + 1;
  v1_preprocess_kernel<4, SPLIT><<<grid_1d((long long)p->B * gh * gw * 8, 32), 256, 0, ST(stream)>>>(*p, gh, gw, sh, sw);
  return check_launch(SPLIT ? "v1_preprocess_split_kernel" : "v1_preprocess_kernel");
}

}  // namespace udb

using namespace udb;

extern "C" {

int udb_v1_preprocess(const udb_v1_preprocess_t* p, void* stream) { return v1_preprocess<false>("udb_v1_preprocess", p, stream); }

int udb_v1_preprocess_split(const udb_v1_preprocess_t* p, void* stream) {
  return v1_preprocess<true>("udb_v1_preprocess_split", p, stream);
}

int udb_layernorm_any(const udb_layernorm_any_t* p, void* stream) {
  if (p->dim % 64 || p->dim > 1536 || p->dim <= 0) { set_error("udb_layernorm_any: dim %d unsupported (multiple of 64, <= 1536)", p->dim); return 1; }
  const bool split = p->out_f32 == UDB_LN_OUT_SPLIT;
  if (split && (p->ld_out % 2 || p->ld_out / 2 < (p->s2d_w > 0 ? 4LL : 1LL) * p->dim)) {
    set_error("udb_layernorm_any: split output needs an even ld_out with room for both halves (ld_out=%lld, dim=%d%s)",
              (long long)p->ld_out, p->dim, p->s2d_w > 0 ? ", space-to-depth" : "");
    return 1;
  }
  if (p->rows <= 0) return 0;
  note_work(0.0, (double)p->rows * p->dim * ((p->in_f32 ? 4 : 2) + (p->out_f32 ? 4 : 2)));
  // rows per warp by width: 4 up to 256 channels, 2 up to 768, 1 beyond (registers: R * dim / 32 floats)
#define UDB_LN_ANY(R_, NV_)                                                                                        \
  do {                                                                                                             \
    const int grid = (int)((p->rows + 8 * (R_) - 1) / (8 * (R_)));                                                 \
    if (split && p->in_f32) layernorm_any_kernel<true, 2, R_, NV_><<<grid, 256, 0, ST(stream)>>>(*p);             \
    else if (split) layernorm_any_kernel<false, 2, R_, NV_><<<grid, 256, 0, ST(stream)>>>(*p);                    \
    else if (p->in_f32 && p->out_f32) layernorm_any_kernel<true, 1, R_, NV_><<<grid, 256, 0, ST(stream)>>>(*p);   \
    else if (p->in_f32) layernorm_any_kernel<true, 0, R_, NV_><<<grid, 256, 0, ST(stream)>>>(*p);                 \
    else if (p->out_f32) layernorm_any_kernel<false, 1, R_, NV_><<<grid, 256, 0, ST(stream)>>>(*p);               \
    else layernorm_any_kernel<false, 0, R_, NV_><<<grid, 256, 0, ST(stream)>>>(*p);                               \
  } while (0)
  if (p->dim <= 256) UDB_LN_ANY(4, 4);
  else if (p->dim <= 768) UDB_LN_ANY(2, 12);
  else UDB_LN_ANY(1, 24);
#undef UDB_LN_ANY
  return check_launch("layernorm_any_kernel");
}

int udb_dwconv7_nhwc_f16(const void* x, const float* w, const float* bias, void* y, int32_t B, int32_t H, int32_t W, int32_t C, void* stream) {
  if (C % DW_CB) { set_error("udb_dwconv7_nhwc_f16: C=%d must be a multiple of 64", C); return 1; }
  // 16x8 or 8x16 (W x H) pixel tiles: whichever pads the map less
  const long long area16 = (long long)((W + 15) / 16) * ((H + 7) / 8), area8 = (long long)((W + 7) / 8) * ((H + 15) / 16);
  note_work(2.0 * 49 * B * H * W * C, 4.0 * B * H * W * C);
  const __half* xh = reinterpret_cast<const __half*>(x);
  __half* yh = reinterpret_cast<__half*>(y);
  if (area16 <= area8) {
    const int tx = (W + 15) / 16, ty = (H + 7) / 8;
    dwconv7_kernel<16><<<dim3(tx * ty, C / DW_CB, B), 256, 0, ST(stream)>>>(xh, w, bias, yh, H, W, C, tx);
  } else {
    const int tx = (W + 7) / 8, ty = (H + 15) / 16;
    dwconv7_kernel<8><<<dim3(tx * ty, C / DW_CB, B), 256, 0, ST(stream)>>>(xh, w, bias, yh, H, W, C, tx);
  }
  return check_launch("dwconv7_kernel");
}

int udb_dwconv7_ln_e4m3(const void* x, const float* w, const float* bias, const float* ln_w, const float* ln_b, void* out,
                        float* out_scale, int32_t B, int32_t H, int32_t W, int32_t C, void* stream) {
  if (C <= 0 || C % DW_CB || C > DWL_MAXC) { set_error("udb_dwconv7_ln_e4m3: C=%d must be a multiple of 64 up to 1536", C); return 1; }
  if (check_dims("udb_dwconv7_ln_e4m3", {{B, "B"}, {H, "H"}, {W, "W"}})) return 1;
  if (check_ptrs("udb_dwconv7_ln_e4m3", {{x, "x"}, {w, "w"}, {bias, "bias"}, {ln_w, "ln_w"}, {ln_b, "ln_b"}, {out, "out"}, {out_scale, "out_scale"}},
                 16, "device pointer"))
    return 1;
  const int chunks = C / DW_CB, K = (chunks + DWL_CPB - 1) / DWL_CPB;     // cluster size: 1..8
  static std::atomic<uint64_t> attr_mask{0};
  if (first_on_device(attr_mask)) {
    for (auto kern : {dwconv7_ln_e4m3_kernel<16>, dwconv7_ln_e4m3_kernel<8>}) {
      const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, DWL_SMEM);
      if (e != cudaSuccess) { set_error("udb_dwconv7_ln_e4m3: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return 1; }
    }
  }
  const double px = (double)B * H * W;
  note_work(2.0 * 49 * px * C + 8.0 * px * C, px * C * (2 + 1) + 4.0 * px);
  // 16x8 or 8x16 (W x H) pixel tiles: whichever pads the map less (as udb_dwconv7_nhwc_f16)
  const long long area16 = (long long)((W + 15) / 16) * ((H + 7) / 8), area8 = (long long)((W + 7) / 8) * ((H + 15) / 16);
  const int tw = area16 <= area8 ? 16 : 8, tx = (W + tw - 1) / tw, ty = (H + DWL_PX / tw - 1) / (DWL_PX / tw);
  const cudaError_t e = launch_ex(tw == 16 ? dwconv7_ln_e4m3_kernel<16> : dwconv7_ln_e4m3_kernel<8>, dim3(tx * ty * K, B), dim3(256),
                                  DWL_SMEM, ST(stream), K, reinterpret_cast<const __half*>(x), w, bias, ln_w, ln_b,
                                  reinterpret_cast<uint8_t*>(out), out_scale, H, W, C, tx);
  if (e != cudaSuccess) { set_error("dwconv7_ln_e4m3_kernel launch: %s", cudaGetErrorString(e)); return 1; }
  return check_launch("dwconv7_ln_e4m3_kernel");
}

int udb_dwconv7_nhwc_f32(const float* x, const float* w, const float* bias, float* y, int32_t B, int32_t H, int32_t W, int32_t C, void* stream) {
  if (C <= 0 || C % DWF_CB || B < 1 || H < 1 || W < 1) {
    set_error("udb_dwconv7_nhwc_f32: B=%d H=%d W=%d C=%d unsupported (C a multiple of 32, the rest >= 1)", B, H, W, C);
    return 1;
  }
  note_work(2.0 * 49 * B * H * W * C, 8.0 * B * H * W * C);
  const int tx = (W + DWF_TW - 1) / DWF_TW, ty = (H + DWF_TH - 1) / DWF_TH;
  dwconv7_f32_kernel<<<dim3(tx * ty, C / DWF_CB, B), 256, 0, ST(stream)>>>(x, w, bias, y, H, W, C, tx);
  return check_launch("dwconv7_f32_kernel");
}

int udb_max_accum_f32(const float* src, float* dst, int64_t n, int32_t first, void* stream) {
  if (n % 4) { set_error("udb_max_accum_f32: n must be a multiple of 4"); return 1; }
  note_work(0.0, (first ? 8.0 : 12.0) * n);
  max_accum_f32_kernel<<<grid_1d(n / 4, 32), 256, 0, ST(stream)>>>(reinterpret_cast<const float4*>(src), reinterpret_cast<float4*>(dst), n / 4, first);
  return check_launch("max_accum_f32_kernel");
}

int udb_max_accum_f16(const void* src, void* dst, int64_t n, int32_t first, void* stream) {
  if (n % 8) { set_error("udb_max_accum_f16: n must be a multiple of 8"); return 1; }
  note_work(0.0, (first ? 4.0 : 6.0) * n);
  max_accum_kernel<<<grid_1d(n / 8, 32), 256, 0, ST(stream)>>>(reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), n / 8, first);
  return check_launch("max_accum_kernel");
}

int udb_vit_tap(const float* x, void* acc, float* cls_out, int32_t B, int32_t N, int32_t D, int32_t first, void* stream) {
  if (D % 8 || D <= 0 || N <= 0 || B <= 0) { set_error("udb_vit_tap: bad shape B=%d N=%d D=%d (D %% 8 == 0)", B, N, D); return 1; }
  const long long items = (long long)B * N * (D / 8) + (cls_out ? (long long)B * (D / 8) : 0);
  note_work((double)B * N * D, (double)B * N * D * (4.0 + (first ? 2.0 : 4.0)) + (cls_out ? 8.0 * B * D : 0.0));
  vit_tap_kernel<false><<<grid_1d(items, 32), 256, 0, ST(stream)>>>(x, reinterpret_cast<uint4*>(acc), cls_out, B, N, D, first);
  return check_launch("vit_tap_kernel");
}

int udb_vit_tap_f32(const float* x, float* acc, float* cls_out, int32_t B, int32_t N, int32_t D, int32_t first, void* stream) {
  if (D % 8 || D <= 0 || N <= 0 || B <= 0) { set_error("udb_vit_tap_f32: bad shape B=%d N=%d D=%d (D %% 8 == 0)", B, N, D); return 1; }
  const long long items = (long long)B * N * (D / 8) + (cls_out ? (long long)B * (D / 8) : 0);
  note_work((double)B * N * D, (double)B * N * D * (4.0 + (first ? 4.0 : 8.0)) + (cls_out ? 8.0 * B * D : 0.0));
  vit_tap_kernel<true><<<grid_1d(items, 32), 256, 0, ST(stream)>>>(x, reinterpret_cast<uint4*>(acc), cls_out, B, N, D, first);
  return check_launch("vit_tap_f32_kernel");
}

int udb_spatial_mean_f32(const float* x, float* out, int32_t B, int32_t HW, int32_t C, void* stream) {
  if (B < 1 || HW < 1 || C < 1) { set_error("udb_spatial_mean_f32: B=%d HW=%d C=%d must all be >= 1", B, HW, C); return 1; }
  dim3 grid((C + 31) / 32, B);
  spatial_mean_kernel<<<grid, 256, 0, ST(stream)>>>(x, out, HW, C);
  return check_launch("spatial_mean_kernel");
}

int udb_aa_resize_nhwc_f16(const void* in, void* out, int32_t B, int32_t H, int32_t W, int32_t C, int32_t oh, int32_t ow, void* stream) {
  if (C % 8) { set_error("udb_aa_resize_nhwc_f16: C must be a multiple of 8"); return 1; }
  note_work(0.0, 2.0 * B * C * ((double)H * W + (double)oh * ow));
  aa_resize_nhwc_kernel<__half><<<grid_1d((long long)B * oh * ow * (C / 8), 32), 256, 0, ST(stream)>>>(
      reinterpret_cast<const __half*>(in), reinterpret_cast<__half*>(out), B, H, W, C, oh, ow, (float)H / (float)oh, (float)W / (float)ow);
  return check_launch("aa_resize_nhwc_kernel");
}

int udb_aa_resize_nhwc_f32(const float* in, float* out, int32_t B, int32_t H, int32_t W, int32_t C, int32_t oh, int32_t ow, void* stream) {
  if (C % 8) { set_error("udb_aa_resize_nhwc_f32: C must be a multiple of 8"); return 1; }
  note_work(0.0, 4.0 * B * C * ((double)H * W + (double)oh * ow));
  aa_resize_nhwc_kernel<float><<<grid_1d((long long)B * oh * ow * (C / 8), 32), 256, 0, ST(stream)>>>(
      in, out, B, H, W, C, oh, ow, (float)H / (float)oh, (float)W / (float)ow);
  return check_launch("aa_resize_nhwc_f32_kernel");
}

int udb_v1_rays_sh81(const udb_v1_rays_t* p, void* stream) {
  const long long toks = (long long)p->B * p->gh * p->gw;
  rays_sh81_kernel<<<(int)((toks + 7) / 8), 256, 0, ST(stream)>>>(*p);
  return check_launch("rays_sh81_kernel");
}

int udb_v1_camera_intrinsics(const float* x4, const float* gt_k, int32_t B, int32_t net_h, int32_t net_w, float ratio, int32_t pad_l,
                             int32_t pad_t, int32_t skip_camera, float* intr4_rays, float* k_out, float* k4_points, void* stream) {
  v1_camera_intrinsics_kernel<<<(B + 63) / 64, 64, 0, ST(stream)>>>(x4, gt_k, B, net_h, net_w, ratio, pad_l, pad_t, skip_camera, intr4_rays, k_out,
                                                                     k4_points);
  return check_launch("v1_camera_intrinsics_kernel");
}

}  // extern "C"

namespace udb {
int cross_attn_small_check(const char* fn, int nq, int nk, int D) {
  if (nq < 1 || nq > CA_MAXQ || D % 256) { set_error("%s: nq=%d D=%d unsupported (nq <= 4, D %% 256 == 0)", fn, nq, D); return 1; }
  // the partial kernel stages the nq queries and the scores of one split's keys in shared memory (at most 200 KB)
  const int chunk = (nk + CA_SPLITS - 1) / CA_SPLITS;
  if ((size_t)(nq * D + nq * chunk + 16) * 4 > 200 * 1024) { set_error("%s: nk=%d too large for nq=%d D=%d", fn, nk, nq, D); return 1; }
  return 0;
}

// udb_cross_attn_small / udb_cross_attn_small_f32: f16 or f32 (k | v) rows
template <class KV>
static int cross_attn_small(const char* fn, const float* q, const float* q_pos, const KV* kv, float* out, float* scratch, int B, int nq, int nk,
                            int D, float scale, void* stream) {
  if (!scratch) { set_error("%s: nq=%d D=%d unsupported (nq <= 4, D %% 256 == 0)", fn, nq, D); return 1; }
  if (cross_attn_small_check(fn, nq, nk, D)) return 1;
  const int chunk = (nk + CA_SPLITS - 1) / CA_SPLITS;
  const size_t smem = (size_t)(nq * D + nq * chunk + 16) * 4;
  static std::atomic<size_t> set_for[64];
  int dev = 0;
  cudaGetDevice(&dev);
  if (smem > 48 * 1024 && smem > set_for[dev & 63].load()) {
    if (cudaFuncSetAttribute(cross_attn_partial_kernel<KV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
      set_error("%s: cudaFuncSetAttribute failed", fn); return 1;
    }
    set_for[dev & 63].store(smem);
  }
  note_work(4.0 * B * nq * (double)nk * D, 2.0 * sizeof(KV) * B * nk * D);
  cross_attn_partial_kernel<KV><<<dim3(CA_SPLITS, B), 256, smem, ST(stream)>>>(q, q_pos, kv, scratch, nq, nk, D, scale);
  if (check_launch(sizeof(KV) == 2 ? "cross_attn_partial_kernel" : "cross_attn_partial_f32_kernel")) return 1;
  cross_attn_merge_kernel<<<dim3(nq, B), 256, 0, ST(stream)>>>(scratch, out, nq, D);
  return check_launch("cross_attn_merge_kernel");
}
}  // namespace udb

extern "C" {

int udb_cross_attn_small(const float* q, const float* q_pos, const void* kv, float* out, float* scratch, int32_t B, int32_t nq, int32_t nk,
                         int32_t D, float scale, void* stream) {
  return cross_attn_small("udb_cross_attn_small", q, q_pos, reinterpret_cast<const __half*>(kv), out, scratch, B, nq, nk, D, scale, stream);
}

int udb_cross_attn_small_f32(const float* q, const float* q_pos, const float* kv, float* out, float* scratch, int32_t B, int32_t nq,
                             int32_t nk, int32_t D, float scale, void* stream) {
  return cross_attn_small("udb_cross_attn_small_f32", q, q_pos, kv, out, scratch, B, nq, nk, D, scale, stream);
}

int udb_softmax_rows(const float* s, void* p, int64_t rows, int32_t n_valid, int32_t ld_in, int32_t ld_out, float scale, void* stream) {
  if (rows < 0 || n_valid < 1 || n_valid > ld_in || n_valid > ld_out) {
    set_error("udb_softmax_rows: rows=%lld n_valid=%d ld_in=%d ld_out=%d: needs rows >= 0 and 1 <= n_valid <= ld_in, ld_out",
              (long long)rows, n_valid, ld_in, ld_out);
    return 1;
  }
  if (rows == 0) return 0;
  softmax_rows_kernel<<<(int)((rows + 7) / 8), 256, 0, ST(stream)>>>(s, reinterpret_cast<__half*>(p), rows, n_valid, ld_in, ld_out, scale);
  return check_launch("softmax_rows_kernel");
}

int udb_add_f32(const float* a, const float* b, float* out, void* out_f16, int64_t n, void* stream) {
  if (n % 4) { set_error("udb_add_f32: n must be a multiple of 4"); return 1; }
  note_work(0.0, (8.0 + (out ? 4.0 : 0.0) + (out_f16 ? 2.0 : 0.0)) * n);
  add_f32_kernel<<<grid_1d(n / 4, 32), 256, 0, ST(stream)>>>(reinterpret_cast<const float4*>(a), reinterpret_cast<const float4*>(b),
                                                         reinterpret_cast<float4*>(out), reinterpret_cast<uint2*>(out_f16), n / 4);
  return check_launch("add_f32_kernel");
}

int udb_copy_rows_f32_to_f16(const float* src, void* dst, int32_t groups, int32_t rows_per_group, int32_t D, int64_t dst_group_stride,
                             int64_t dst_row0, void* stream) {
  if (groups < 1 || rows_per_group < 1 || D < 1) {
    set_error("udb_copy_rows_f32_to_f16: groups=%d rows_per_group=%d D=%d must all be >= 1", groups, rows_per_group, D);
    return 1;
  }
  copy_rows_f16_kernel<<<grid_1d((long long)groups * rows_per_group * D, 32), 256, 0, ST(stream)>>>(src, reinterpret_cast<__half*>(dst), groups,
                                                                                                rows_per_group, D, dst_group_stride, dst_row0);
  return check_launch("copy_rows_f16_kernel");
}

int udb_conv3x3_c1_exp(const void* x, const float* w, float bias, float* out, int32_t B, int32_t H, int32_t W, int32_t C, void* stream) {
  if (C != 64 && C != 128 && C != 256) { set_error("udb_conv3x3_c1_exp: C=%d unsupported (64, 128 or 256)", C); return 1; }
  const long long px = (long long)B * H * W;
  const int lpp = C / 8, ppb = 8 * (32 / lpp);
  const int grid = (int)((px + ppb - 1) / ppb);
  note_work(2.0 * px * 9 * C, 2.0 * px * C + 4.0 * px);
  const __half* xh = reinterpret_cast<const __half*>(x);
  if (lpp == 8) conv3x3_c1_kernel<8><<<grid, 256, 0, ST(stream)>>>(xh, w, bias, out, B, H, W, C);
  else if (lpp == 16) conv3x3_c1_kernel<16><<<grid, 256, 0, ST(stream)>>>(xh, w, bias, out, B, H, W, C);
  else conv3x3_c1_kernel<32><<<grid, 256, 0, ST(stream)>>>(xh, w, bias, out, B, H, W, C);
  return check_launch("conv3x3_c1_kernel");
}

int udb_nystrom_landmarks(const void* q, int32_t ldq, const void* kv, int32_t ldkv, void* out, int32_t B, int32_t n, int32_t heads, void* stream) {
  if (n < 128) { set_error("udb_nystrom_landmarks: sequence %d shorter than the 128 landmarks", n); return 1; }
  nystrom_landmarks_kernel<<<dim3(128, heads, B), 64, 0, ST(stream)>>>(reinterpret_cast<const __half*>(q), ldq, reinterpret_cast<const __half*>(kv),
                                                                       ldkv, reinterpret_cast<__half*>(out), n, heads, 128);
  return check_launch("nystrom_landmarks_kernel");
}

int udb_nystrom_k2_pinv(const void* landmarks, float* k2, float* z, float* tmp, int32_t B, int32_t heads, int32_t iters, void* stream) {
  // kernel_2 = softmax(ql kl^T / 8); Z = pinv(kernel_2) by `iters` Newton-Schulz steps (Razavi et al.):
  //   KV = K Z;  T1 = 7I - KV;  T2 = 15I - KV T1;  T3 = 13I - KV T2;  Z <- 0.25 Z T3        (tmp: 3 matrices per (b, head))
  const int m = 128, nb = B * heads;
  const long long mm = (long long)m * m;
  nystrom_k2_kernel<<<dim3(m / 4, nb), 128, 0, ST(stream)>>>(reinterpret_cast<const __half*>(landmarks), k2, heads, m);
  if (check_launch("nystrom_k2_kernel")) return 1;
  nystrom_pinv_init_kernel<<<nb, 128, 0, ST(stream)>>>(k2, z, m);
  if (check_launch("nystrom_pinv_init_kernel")) return 1;
  float* KV = tmp;
  float* Ta = tmp + nb * mm;
  float* Tb = tmp + 2 * nb * mm;
  auto mmul = [&](const float* A, const float* Bm, float* C, float alpha, float diag) {
    BmmArgs a{};
    a.A = A; a.sA = mm; a.lda = m;
    a.Bp = Bm; a.sB1 = mm; a.sB2 = 0; a.ldb = m; a.b_f16 = 0; a.inner = 1;
    a.C = C; a.sC1 = mm; a.sC2 = 0; a.ldc = m; a.c_f16 = 0;
    a.M = m; a.N = m; a.K = m; a.alpha = alpha; a.diag = diag;
    bmm_f32_kernel<<<dim3(m / 64, m / 64, nb), 256, 0, ST(stream)>>>(a);
    return check_launch("bmm_f32_kernel");
  };
  float* Z = z;
  float* spare = Tb;
  for (int it = 0; it < iters; ++it) {
    float* T2 = spare;
    if (mmul(k2, Z, KV, 1.f, 0.f)) return 1;                       // KV = K Z
    eye_minus_kernel<<<grid_1d(nb * mm, 32), 256, 0, ST(stream)>>>(KV, Ta, 7.f, m, nb * mm);     // T1 = 7I - KV
    if (check_launch("eye_minus_kernel")) return 1;
    if (mmul(KV, Ta, T2, -1.f, 15.f)) return 1;                    // T2 = 15I - KV T1
    if (mmul(KV, T2, Ta, -1.f, 13.f)) return 1;                    // T3 = 13I - KV T2   (over T1)
    if (mmul(Z, Ta, T2, 0.25f, 0.f)) return 1;                     // Z' = 0.25 Z T3     (over T2)
    spare = Z;
    Z = T2;
  }
  if (Z != z && cudaMemcpyAsync(z, Z, sizeof(float) * nb * mm, cudaMemcpyDeviceToDevice, ST(stream)) != cudaSuccess) {
    set_error("udb_nystrom_k2_pinv: copy failed"); return 1;
  }
  return 0;
}

// out[(b, lm), h*64 + d] (f16, row stride ldo) = sum_j Z[b,h][lm][j] * k3[(b, j), h*64 + d]: the (pinv . kernel_3) product that
// becomes the V operand of the final softmax(q kl^T) attention.
int udb_nystrom_zk3(const float* z, const void* k3, int32_t ldk3, void* out, int32_t ldo, int32_t B, int32_t heads, void* stream) {
  const int m = 128;
  BmmArgs a{};
  a.A = z; a.sA = (long long)m * m; a.lda = m;
  a.Bp = k3; a.sB1 = (long long)m * ldk3; a.sB2 = 64; a.ldb = ldk3; a.b_f16 = 1; a.inner = heads;
  a.C = out; a.sC1 = (long long)m * ldo; a.sC2 = 64; a.ldc = ldo; a.c_f16 = 1;
  a.M = m; a.N = 64; a.K = m; a.alpha = 1.f; a.diag = 0.f;
  bmm_f32_kernel<<<dim3(1, m / 64, B * heads), 256, 0, ST(stream)>>>(a);
  return check_launch("bmm_f32_kernel");
}

int udb_v1_mean_maps(const float* o8, const float* o4, const float* o2, float* mean, int32_t B, int32_t gh, int32_t gw, int32_t net_h,
                     int32_t net_w, void* stream) {
  if (check_dims("udb_v1_mean_maps", {{B, "B"}, {gh, "gh"}, {gw, "gw"}, {net_h, "net_h"}, {net_w, "net_w"}})) return 1;
  v1_mean_maps_kernel<<<grid_1d((long long)B * net_h * net_w, 32), 256, 0, ST(stream)>>>(o8, o4, o2, mean, B, gh, gw, net_h, net_w);
  return check_launch("v1_mean_maps_kernel");
}

int udb_v1_postprocess(const udb_v1_postprocess_t* p, void* stream) {
  if (check_dims("udb_v1_postprocess", {{p->B, "B"}, {p->H, "H"}, {p->W, "W"}, {p->net_h - p->pad_t - p->pad_b, "net_h - pad_t - pad_b"},
                                        {p->net_w - p->pad_l - p->pad_r, "net_w - pad_l - pad_r"}}))
    return 1;
  const int pads[] = {p->pad_l, p->pad_r, p->pad_t, p->pad_b};
  for (int i = 0; i < 4; ++i)
    if (pads[i] < 0) { set_error("udb_v1_postprocess: paddings (pad_l, pad_r, pad_t, pad_b) must be >= 0"); return 1; }
  v1_postprocess_kernel<<<grid_1d((long long)p->B * p->H * p->W, 32), 256, 0, ST(stream)>>>(*p);
  return check_launch("v1_postprocess_kernel");
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------------
// UniDepthV2old (unidepthv2/decoder_old.py, unidepthv2_old.py).  CUDA-core kernels for the four steps no existing kernel
// computes.
// ------------------------------------------------------------------------------------------------------------------
namespace udb {

// ConvUpsampleShuffleResidual's up branch before its 3x3 conv (layers/upsample.py:110-121): PixelShuffle(2) of the NHWC
// f16 map [B,h,w,C] (out channel c of pixel (Y, X) is input channel 4c + 2(Y%2) + X%2 of pixel (Y/2, X/2)), then the
// depthwise 7x7 (zero padding) on the C/4 shuffled channels, then ReLU.  Written to an f16 map [B,2h,2w,ldo] whose channels
// C/4..ldo-1 are zero, so that the following 3x3 conv runs on the wgmma path, which needs 64-channel multiples.  No
// existing kernel reads a pixel-shuffled operand: udb_dwconv7_nhwc_f16 needs C % 64 == 0 and a plain NHWC map.
// One thread per output (pixel, channel); taps tap-major [49, C/4] f32 as the ConvNeXt depthwise weights.
__global__ void __launch_bounds__(256) pshuffle_dw7_relu_kernel(const __half* __restrict__ x, const float* __restrict__ w,
                                                                const float* __restrict__ bias, __half* __restrict__ out, int B,
                                                                int h, int wd, int C, int ldo) {
  const int Cq = C / 4, H2 = 2 * h, W2 = 2 * wd;
  const long long total = (long long)B * H2 * W2 * ldo;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % ldo);
    const long long px = i / ldo;
    if (c >= Cq) { out[i] = __float2half_rn(0.f); continue; }
    const int X = (int)(px % W2), Y = (int)((px / W2) % H2), b = (int)(px / ((long long)W2 * H2));
    float acc = bias[c];
    for (int dy = 0; dy < 7; ++dy) {
      const int yy = Y + dy - 3;
      if (yy < 0 || yy >= H2) continue;
      for (int dx = 0; dx < 7; ++dx) {
        const int xx = X + dx - 3;
        if (xx < 0 || xx >= W2) continue;
        const int ch = 4 * c + 2 * (yy & 1) + (xx & 1);
        const float v = __half2float(x[(((long long)b * h + (yy >> 1)) * wd + (xx >> 1)) * C + ch]);
        acc = fmaf(w[(dy * 7 + dx) * Cq + c], v, acc);
      }
    }
    out[i] = __float2half_rn(fmaxf(acc, 0.f));
  }
}

// The depth and confidence convolutions of DepthHead.decode_depth (decoder_old.py:282-304): each level's 32-channel MLP
// output ([depth 16 | confidence 16], f32 NHWC at (2gh, 2gw) << i) is bilinearly resized (align_corners=False, no
// antialias) to the network shape and concatenated finest level first (channel block 2 - i), and a 7x7 reflect-padded
// conv maps the 48 channels to one.  The resized maps are never stored: each of the 49 taps samples the levels where it
// lands.  Writes the log-depth and the sigmoid of the confidence logit.  One thread per network pixel; weights in shared
// memory ([2][48][49]: depth then confidence).

__global__ void __launch_bounds__(256) v2old_heads_kernel(const udb_v2old_heads_t p) {
  __shared__ float ws[2 * 48 * 49];
  for (int i = threadIdx.x; i < 2 * 48 * 49; i += blockDim.x) ws[i] = p.w[i];
  __syncthreads();
  const long long total = (long long)p.B * p.net_h * p.net_w;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(idx % p.net_w), Y = (int)((idx / p.net_w) % p.net_h), b = (int)(idx / ((long long)p.net_w * p.net_h));
    float ad = p.bias_depth, ac = p.bias_conf;
    for (int lvl = 0; lvl < 3; ++lvl) {
      const int lh = (2 * p.gh) << lvl, lw = (2 * p.gw) << lvl;
      const float sy = (float)lh / (float)p.net_h, sx = (float)lw / (float)p.net_w;
      const float* src = p.levels[lvl] + (long long)b * lh * lw * 32;
      const float* wd = ws + (2 - lvl) * 16 * 49;
      const float* wc = ws + 48 * 49 + (2 - lvl) * 16 * 49;
      for (int dy = 0; dy < 7; ++dy) {
        const int yy = reflect_idx(Y + dy - 3, p.net_h);
        int y0, y1;
        float ly0, ly;
        bilinear_taps(fmaxf(sy * ((float)yy + 0.5f) - 0.5f, 0.f), lh, y0, y1, ly0, ly);
        for (int dx = 0; dx < 7; ++dx) {
          const int xx = reflect_idx(X + dx - 3, p.net_w);
          int x0, x1;
          float lx0, lx;
          bilinear_taps(fmaxf(sx * ((float)xx + 0.5f) - 0.5f, 0.f), lw, x0, x1, lx0, lx);
          const float4* r00 = reinterpret_cast<const float4*>(src + ((long long)y0 * lw + x0) * 32);
          const float4* r01 = reinterpret_cast<const float4*>(src + ((long long)y0 * lw + x1) * 32);
          const float4* r10 = reinterpret_cast<const float4*>(src + ((long long)y1 * lw + x0) * 32);
          const float4* r11 = reinterpret_cast<const float4*>(src + ((long long)y1 * lw + x1) * 32);
          const float w00 = ly0 * lx0, w01 = ly0 * lx, w10 = ly * lx0, w11 = ly * lx;
          const int tap = dy * 7 + dx;
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const float4 a = __ldg(r00 + q), bb = __ldg(r01 + q), cc = __ldg(r10 + q), d = __ldg(r11 + q);
            const float v[4] = {w00 * a.x + w01 * bb.x + w10 * cc.x + w11 * d.x, w00 * a.y + w01 * bb.y + w10 * cc.y + w11 * d.y,
                                w00 * a.z + w01 * bb.z + w10 * cc.z + w11 * d.z, w00 * a.w + w01 * bb.w + w10 * cc.w + w11 * d.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int ch = q * 4 + e;
              if (ch < 16) ad = fmaf(wd[ch * 49 + tap], v[e], ad);
              else ac = fmaf(wc[(ch - 16) * 49 + tap], v[e], ac);
            }
          }
        }
      }
    }
    p.logdepth[idx] = ad;
    p.confidence[idx] = 1.f / (1.f + expf(-ac));
  }
}

// The decoder's tail (decoder_old.py:505-514) in place on the log-depth map of one image per block: LayerNorm over the whole
// H x W map (no affine, eps 1e-5; mean then variance, two passes, double accumulation), exp, (x + shift) * scale with
// (log scale, shift) from the global head, softplus with beta 10 (threshold 20, as torch).  A per-map reduction fused
// with its pointwise tail: no existing LayerNorm kernel normalises over a whole map.
__global__ void __launch_bounds__(1024) v2old_depth_tail_kernel(float* __restrict__ d, const float* __restrict__ scale_shift, long long hw) {
  __shared__ double red[32];
  __shared__ double bc;
  float* m = d + blockIdx.x * hw;
  auto block_sum = [&](double v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
      double t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0;
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if (threadIdx.x == 0) bc = t;
    }
    __syncthreads();
    const double r = bc;
    __syncthreads();
    return r;
  };
  double s = 0.0;
  for (long long i = threadIdx.x; i < hw; i += blockDim.x) s += m[i];
  const float mean = (float)(block_sum(s) / (double)hw);
  double v = 0.0;
  for (long long i = threadIdx.x; i < hw; i += blockDim.x) { const double t = (double)m[i] - mean; v += t * t; }
  const float rstd = rsqrtf((float)(block_sum(v) / (double)hw) + 1e-5f);
  const float sc = expf(scale_shift[blockIdx.x * 2]), sh = scale_shift[blockIdx.x * 2 + 1];
  for (long long i = threadIdx.x; i < hw; i += blockDim.x) {
    const float z = (expf((m[i] - mean) * rstd) + sh) * sc;
    m[i] = 10.f * z > 20.f ? z : log1pf(expf(10.f * z)) / 10.f;
  }
}

// Output assembly at the input size (unidepthv2_old.py:107-116,267-274): depth resized from the network shape with
// bilinear (align_corners=False, no antialias) or nearest-exact, confidence with antialiased bilinear (aa_axis), and the
// points z * (tan(theta), 1 / tan(phi) / cos(theta), 1) of the unit ray of each input pixel through k4 (fx, fy, cx, cy).
// DEPTH_AA (depth_aa) resizes the depth with antialiased bilinear too, as the reference's `forward` does
// (unidepthv2_old.py:166-179); at equal sizes the weights are (1, 0) and the depth is copied bit for bit.  A template
// argument, so that the code of the two `infer` modes is exactly what it was without it.
// V1's post-processing crops paddings and resizes depth with antialias only; V2's assembles radius-based points from
// padded maps; neither resizes with these two modes.
template <bool DEPTH_AA>
__global__ void __launch_bounds__(256) v2old_postprocess_kernel(const udb_v2old_postprocess_t p) {
  const long long total = (long long)p.B * p.H * p.W;
  const float sh = (float)p.net_h / (float)p.H, sw = (float)p.net_w / (float)p.W;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int X = (int)(idx % p.W), Y = (int)((idx / p.W) % p.H), b = (int)(idx / ((long long)p.W * p.H));
    const long long nhw = (long long)p.net_h * p.net_w;
    const float* dm = p.depth + b * nhw;
    float z;
    if (DEPTH_AA) {
      z = aa_sample(dm, aa_axis(Y, p.net_h, sh), aa_axis(X, p.net_w, sw), p.net_w);
    } else if (p.mode == UDB_V2OLD_NEAREST_EXACT) {
      const int yi = min((int)floorf(((float)Y + 0.5f) * sh), p.net_h - 1), xi = min((int)floorf(((float)X + 0.5f) * sw), p.net_w - 1);
      z = dm[(long long)yi * p.net_w + xi];
    } else {
      int y0, y1, x0, x1;
      float ly0, ly1, lx0, lx1;
      bilinear_taps(fmaxf(sh * ((float)Y + 0.5f) - 0.5f, 0.f), p.net_h, y0, y1, ly0, ly1);
      bilinear_taps(fmaxf(sw * ((float)X + 0.5f) - 0.5f, 0.f), p.net_w, x0, x1, lx0, lx1);
      z = ly0 * (lx0 * dm[(long long)y0 * p.net_w + x0] + lx1 * dm[(long long)y0 * p.net_w + x1]) +
          ly1 * (lx0 * dm[(long long)y1 * p.net_w + x0] + lx1 * dm[(long long)y1 * p.net_w + x1]);
    }
    const float conf = aa_sample(p.confidence + b * nhw, aa_axis(Y, p.net_h, sh), aa_axis(X, p.net_w, sw), p.net_w);
    const long long hw = (long long)p.H * p.W, pix = (long long)Y * p.W + X;
    p.out_depth[b * hw + pix] = z;
    p.out_confidence[b * hw + pix] = conf;
    backproject(p.k4 + b * 4, X, Y, z, p.out_points + b * 3 * hw + pix, hw);
  }
}

// The camera of UniDepthV2old (decoder_old.py:55-64,396-399; unidepthv2_old.py:95-104,112-115,268): the predicted K at the
// network shape (focal max(h, w)/2 exp(x), principal point sigmoid(x) times the side) and at the input size (divided
// by `ratio`: out_k, always the prediction), the K of the rays (the caller's K times `ratio`, else the prediction) and
// the K of the points (the caller's K, else the prediction at the input size).
__global__ void v2old_camera_kernel(const float* __restrict__ x4, const float* __restrict__ gt_k, int B, int net_h, int net_w,
                                    float ratio, float* intr4_rays, float* k_out, float* k4_points) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float4 k = decode_camera(x4 + b * 4, (float)(net_h > net_w ? net_h : net_w) / 2.f, net_h, net_w);
  const float fx = k.x, fy = k.y, cx = k.z, cy = k.w;
  const float kf[4] = {fx / ratio, fy / ratio, cx / ratio, cy / ratio};
  store_k3(k_out + b * 9, kf[0], kf[1], kf[2], kf[3]);
  if (gt_k) {
    const float* g = gt_k + b * 9;
    const float gk[4] = {g[0], g[4], g[2], g[5]};
    for (int i = 0; i < 4; ++i) { intr4_rays[b * 4 + i] = gk[i] * ratio; k4_points[b * 4 + i] = gk[i]; }
  } else {
    const float pk[4] = {fx, fy, cx, cy};
    for (int i = 0; i < 4; ++i) { intr4_rays[b * 4 + i] = pk[i]; k4_points[b * 4 + i] = kf[i]; }
  }
}

}  // namespace udb

extern "C" {

int udb_pshuffle_dw7_relu(const void* x, const float* w, const float* bias, void* out, int32_t B, int32_t h, int32_t wd, int32_t C,
                          int32_t ldo, void* stream) {
  if (check_dims("udb_pshuffle_dw7_relu", {{B, "B"}, {h, "h"}, {wd, "w"}, {C, "C"}})) return 1;
  if (C % 4) { set_error("udb_pshuffle_dw7_relu: C=%d must be a multiple of 4 (PixelShuffle(2))", C); return 1; }
  if (ldo < C / 4) { set_error("udb_pshuffle_dw7_relu: ldo=%d must be >= C/4=%d", ldo, C / 4); return 1; }
  if (check_ptrs("udb_pshuffle_dw7_relu", {{x, "x"}, {w, "w"}, {bias, "bias"}, {out, "out"}})) return 1;
  const long long total = 4LL * B * h * wd * ldo;
  note_work(2.0 * 49 * 4.0 * B * h * wd * (C / 4), 2.0 * B * h * wd * C + 2.0 * total);
  pshuffle_dw7_relu_kernel<<<grid_1d(total, 32), 256, 0, ST(stream)>>>(reinterpret_cast<const __half*>(x), w, bias,
                                                                    reinterpret_cast<__half*>(out), B, h, wd, C, ldo);
  return check_launch("pshuffle_dw7_relu_kernel");
}

int udb_v2old_heads(const udb_v2old_heads_t* p, void* stream) {
  if (!p) { set_error("udb_v2old_heads: null argument"); return 1; }
  if (check_dims("udb_v2old_heads", {{p->B, "B"}, {p->gh, "gh"}, {p->gw, "gw"}, {p->net_h, "net_h"}, {p->net_w, "net_w"}})) return 1;
  if (p->net_h < 4 || p->net_w < 4) { set_error("udb_v2old_heads: net_h=%d net_w=%d: the 7x7 reflect padding needs >= 4", p->net_h, p->net_w); return 1; }
  if (check_ptrs("udb_v2old_heads", {{p->levels[0], "levels[0]"}, {p->levels[1], "levels[1]"}, {p->levels[2], "levels[2]"}, {p->w, "w"},
                                     {p->logdepth, "logdepth"}, {p->confidence, "confidence"}}, 16))
    return 1;
  const long long px = (long long)p->B * p->net_h * p->net_w;
  note_work(px * 49.0 * 3 * (8.0 * 32 + 2.0 * 32), px * 8.0);
  v2old_heads_kernel<<<grid_1d(px, 32), 256, 0, ST(stream)>>>(*p);
  return check_launch("v2old_heads_kernel");
}

int udb_v2old_depth_tail(float* depth, const float* scale_shift, int32_t B, int64_t hw, void* stream) {
  if (B < 1 || hw < 1) { set_error("udb_v2old_depth_tail: B=%d hw=%lld must be >= 1", B, (long long)hw); return 1; }
  if (!depth || !scale_shift) { set_error("udb_v2old_depth_tail: `%s` must be non-null", depth ? "scale_shift" : "depth"); return 1; }
  note_work(12.0 * B * hw, 16.0 * B * hw);
  v2old_depth_tail_kernel<<<B, 1024, 0, ST(stream)>>>(depth, scale_shift, hw);
  return check_launch("v2old_depth_tail_kernel");
}

int udb_v2old_postprocess(const udb_v2old_postprocess_t* p, void* stream) {
  if (!p) { set_error("udb_v2old_postprocess: null argument"); return 1; }
  if (check_dims("udb_v2old_postprocess", {{p->B, "B"}, {p->H, "H"}, {p->W, "W"}, {p->net_h, "net_h"}, {p->net_w, "net_w"}})) return 1;
  if (p->depth_aa != 0 && p->depth_aa != 1) { set_error("udb_v2old_postprocess: `depth_aa` %d is neither 0 nor 1", p->depth_aa); return 1; }
  if (!p->depth_aa && p->mode != UDB_V2OLD_BILINEAR && p->mode != UDB_V2OLD_NEAREST_EXACT) {
    set_error("udb_v2old_postprocess: `mode` %d is neither UDB_V2OLD_BILINEAR (0) nor UDB_V2OLD_NEAREST_EXACT (1)", p->mode);
    return 1;
  }
  if (check_ptrs("udb_v2old_postprocess", {{p->depth, "depth"}, {p->confidence, "confidence"}, {p->k4, "k4"}, {p->out_depth, "out_depth"},
                                           {p->out_confidence, "out_confidence"}, {p->out_points, "out_points"}}))
    return 1;
  if (p->depth_aa) v2old_postprocess_kernel<true><<<grid_1d((long long)p->B * p->H * p->W, 32), 256, 0, ST(stream)>>>(*p);
  else v2old_postprocess_kernel<false><<<grid_1d((long long)p->B * p->H * p->W, 32), 256, 0, ST(stream)>>>(*p);
  return check_launch("v2old_postprocess_kernel");
}

int udb_v2old_camera(const float* x4, const float* gt_k, int32_t B, int32_t net_h, int32_t net_w, float ratio, float* intr4_rays,
                     float* k_out, float* k4_points, void* stream) {
  if (B < 1 || net_h < 1 || net_w < 1 || !(ratio > 0.f)) {
    set_error("udb_v2old_camera: B=%d net_h=%d net_w=%d ratio=%g: all must be > 0", B, net_h, net_w, ratio);
    return 1;
  }
  if (!x4 || !intr4_rays || !k_out || !k4_points) { set_error("udb_v2old_camera: null output or camera-head pointer"); return 1; }
  v2old_camera_kernel<<<(B + 63) / 64, 64, 0, ST(stream)>>>(x4, gt_k, B, net_h, net_w, ratio, intr4_rays, k_out, k4_points);
  return check_launch("v2old_camera_kernel");
}

}  // extern "C"
