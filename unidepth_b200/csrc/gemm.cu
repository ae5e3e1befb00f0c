// Persistent warp-specialised wgmma GEMM for sm_90a:   D = epilogue(A . W^T)
//
//   warps 0..7 : two consumer warpgroups; warpgroup g multiplies rows [64g, 64g+64) of the 128 x BN tile
//                (wgmma m64nBNk16, both operands from 128B-swizzled shared memory, f32 accumulator in registers)
//                and then runs the epilogue (bias/act/gamma/residual/LayerNorm statistics -> global)
//   warps 8..11: producer warpgroup; warp 8 issues the TMA loads (A tile 128x64 f16, W tile BNx64 f16, 128B swizzle,
//                mbarrier ring).  It hands its registers to the consumers (setmaxnreg 40 / 232): the BN = 256
//                accumulator alone is 128 registers per consumer thread.
//
// The A operand is either a row-major matrix (2-D tensor map) or a 3x3 convolution window over an
// NHWC image (4-D tensor map, one (dy,dx,64-channel) slab per k-block; zero padding comes from TMA
// out-of-bounds fill), so linear layers, 1x1 / 3x3 convolutions and k=s transposed convolutions all
// run through this one kernel.  See include/udb.h (udb_gemm) for the reference call sites.
//
// Two epilogues.  The general one (epilogue_tile) transposes each 32-column chunk through per-warp shared-memory tiles
// and stores rows with st.global; it serves every store mode.  The TMA epilogue (epilogue_tile_tma; plain ROWS stores
// with an identity row map, see tma_epilogue_ok) stages each warpgroup's 64 x 32 chunk in a swizzled box, stores it with
// an asynchronous TMA store and goes on to the next chunk / tile's MMAs while the store drains; warp 9 of the producer
// warpgroup prefetches the f32 residual into the same boxes.  Both run the same per-element arithmetic, so their
// outputs are bit-identical.
#include <stdlib.h>
#include <string.h>

#include "common.h"
#include "ptx.cuh"

namespace udb {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kEpiWarps = 8;
constexpr int kTP = 36;   // pitch (floats) of the per-warp 32-row transpose tile: 16 B aligned rows, conflict-free 128-bit access
constexpr int kThreads = (kEpiWarps + 4) * 32;

struct GemmArgs {
  int M, N, K, num_kb;
  int tiles_m, tiles_n;
  int a_mode;
  int conv_B, conv_H, conv_W, conv_cpb /*64-ch blocks per tap*/, conv_off, conv_TH, conv_TW, conv_tx, conv_ty;
  const float* bias;
  const float* gamma;
  const void* resid;
  int resid_f32;
  void* out;
  int out_f32;
  __half* out2;
  int out2_leaky;
  int act;
  int store_mode;
  long long ldc, ldr;
  int rpg, gstride, roff;
  int resid_mod, resid_roff;
  int ct_k, ct_cout, ct_h, ct_w, ct_pad;
  int conv_coff;
  const float* head_w;
  float head_b, head_add;
  int a_wrap;      // split-f16 operands: k-blocks at or beyond this element offset re-read A from (k - a_wrap); 0 = off
  int out_split;   // f16 `out`: lo half stored out_split elements to the right; 0 = off
  // Fused LayerNorm (udb_gemm_t.ln_*): a PRODUCER writes, per output row and per (column tile, column half), the mean and
  // the centred sum of squares of the values it stores; a CONSUMER whose A operand is the un-normalised f16 copy of those
  // rows merges the partials and applies  v = rstd * (acc - mean * c1[n]) + bias[n]  (weights pre-multiplied by the
  // LayerNorm scale, c1 = their row sums, bias = W ln_bias + bias).
  float* stats_out;
  const float* ln_stats;
  const float* ln_c1;
  int ln_parts, ln_part_cols;
  float ln_eps;
};

// TMA epilogue staging box: one warpgroup's 64 rows x 32 columns, f32 (128 B rows, 128B swizzle) or f16 (64 B rows,
// 64B swizzle, first half of the box).  Two buffers; buffer b holds both warpgroups' boxes back to back, so one 128-row
// TMA load fills it with a residual chunk of the whole tile.
constexpr int kEpiBox = 64 * 32 * 4;

template <int BN, bool TMAE = false>
struct GemmCfg {
  // as many operand stages as fit next to the epilogue staging in 227 KB
  static constexpr int kStages = TMAE ? (BN >= 192 ? 4 : (BN >= 128 ? 6 : 8))
                                      : (BN >= 256 ? 3 : (BN >= 192 ? 4 : (BN >= 128 ? 5 : 7)));
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  // epilogue staging: per epilogue warp a 32x32 f32 transpose tile and 2 x 32 row offsets, so that global loads/stores
  // are row-contiguous (coalesced) per instruction -- or, for the TMA epilogue, 2 buffers x 2 warpgroups x kEpiBox
  static constexpr int kStagingBytes = TMAE ? 2 * 2 * kEpiBox : kEpiWarps * (32 * kTP * 4 + 2 * 32 * 4);
  static constexpr int kSmemBytes = kStages * kStageBytes + kStagingBytes + 256 /*barriers*/;
  static_assert(kSmemBytes <= 232448, "shared memory per block");
  static_assert(2 * kStages + 4 <= 32, "barriers");
};

// The activation step of the epilogue arithmetic (bias -> activation -> gamma -> + residual), shared by both epilogues.
template <int N>
__device__ __forceinline__ void apply_act(const int act, float (&v)[N]) {
  if (act == UDB_ACT_GELU) {
#pragma unroll
    for (int j = 0; j < N; j += 2) gelu_erf_pair(v[j], v[j + 1]);
  } else if (act == UDB_ACT_LEAKY) {
#pragma unroll
    for (int j = 0; j < N; ++j) v[j] = leaky(v[j]);
  }
}

// One accumulator tile (128 rows x BN columns; warpgroup g holds rows [64g, 64g+64) in registers) -> global memory.
// `mt` indexes this CTA's 128-row block (matrix rows mt*128.. or spatial conv tile mt), `nt` the BN-wide column block.
// Epilogue warp w of warpgroup g owns tile rows 64g + 32 (w & 1) + [0, 32) and column half w >> 1; for every 32-column
// chunk the warpgroup first moves its accumulator fragments into the owners' transpose tiles (thread == row afterwards).
struct EpiWarp {
  float* T;              // [32][kTP] transpose tile of this warp; the warpgroup's four tiles are contiguous
  float* Twg;            // first transpose tile of this warpgroup
  uint32_t* roff_out;    // [32] element offsets of this warp's rows in out / out2
  uint32_t* roff_res;    // [32] element offsets in resid
  int wg, wq, grp, lane, r_in_tile;
};

// LNF: compile the fused-LayerNorm producer / consumer code in (udb_gemm_t.ln_*); the default instantiation does not carry it.
template <int BN, bool LNF>
__device__ __forceinline__ void epilogue_tile(const GemmArgs& p, const EpiWarp& w, const float (&acc)[BN / 2], const int mt,
                                              const int nt) {
  constexpr int kGroups = BN >= 64 ? 2 : 1;
  constexpr int kColsPerGrp = BN / kGroups;
  const int grp = w.grp, lane = w.lane, r_in_tile = w.r_in_tile;
  const bool active = grp < kGroups;
  float* T = w.T;
  uint32_t* roff_out = w.roff_out;
  uint32_t* roff_res = w.roff_res;
  bool valid = false;
  long long out_off = 0, res_off = 0;
  uint32_t vmask = 0;
  float ln_mean = 0.f, ln_rstd = 1.f;
  float st_pivot = 0.f, st_s1 = 0.f, st_s2 = 0.f;
  bool st_first = true;
  if (active) {

    // ---- per-row addressing
    const int m = mt * BM + r_in_tile;
    if (p.store_mode == UDB_STORE_CONVTILE || p.store_mode == UDB_STORE_HEAD) {
      const int per_img = p.conv_tx * p.conv_ty;
      const int b = mt / per_img;
      const int r = mt % per_img;
      const int y = (r / p.conv_tx) * p.conv_TH + r_in_tile / p.conv_TW;
      const int x = (r % p.conv_tx) * p.conv_TW + r_in_tile % p.conv_TW;
      valid = (b < p.conv_B) && (y < p.conv_H) && (x < p.conv_W);
      out_off = (((long long)b * p.conv_H + y) * p.conv_W + x) * p.ldc;
      res_off = (((long long)b * p.conv_H + y) * p.conv_W + x) * p.ldr;
    } else if (p.store_mode == UDB_STORE_CONVT) {
      valid = m < p.M;
      const int hw = p.ct_h * p.ct_w;
      const int b = m / hw;
      const int r = m % hw;
      const int y = r / p.ct_w, x = r % p.ct_w;
      const long long W2 = (long long)p.ct_w * p.ct_k + 2 * p.ct_pad;
      const long long H2 = (long long)p.ct_h * p.ct_k + 2 * p.ct_pad;
      out_off = ((b * H2 + (long long)y * p.ct_k + p.ct_pad) * W2 + (long long)x * p.ct_k + p.ct_pad) * p.ct_cout;
      res_off = out_off;
    } else {
      valid = m < p.M;
      long long orow = m;
      if (p.rpg > 0) orow = (long long)(m / p.rpg) * p.gstride + (m % p.rpg) + p.roff;
      out_off = orow * p.ldc;
      res_off = (p.resid_mod > 0) ? ((long long)(m % p.resid_mod) + p.resid_roff) * p.ldr
                                  : orow * p.ldr;
    }
    vmask = __ballot_sync(0xffffffffu, valid);
    roff_out[lane] = static_cast<uint32_t>(out_off);
    roff_res[lane] = static_cast<uint32_t>(res_off);
    __syncwarp();
    // fused LayerNorm, consumer side: merge this row's partial statistics (equal counts: plain mean of the means,
    // M2 = sum M2_p + n_p * sum (mean_p - mean)^2)
    if (LNF && p.ln_stats) {
      const float2* sp = reinterpret_cast<const float2*>(p.ln_stats) + (long long)(valid ? m : 0) * p.ln_parts;
      float ms = 0.f, m2 = 0.f;
      for (int q = 0; q < p.ln_parts; ++q) ms += sp[q].x;
      ln_mean = ms / (float)p.ln_parts;
      for (int q = 0; q < p.ln_parts; ++q) {
        const float2 t = sp[q];
        m2 += t.y + (float)p.ln_part_cols * (t.x - ln_mean) * (t.x - ln_mean);
      }
      ln_rstd = rsqrtf(m2 / (float)(p.ln_parts * p.ln_part_cols) + p.ln_eps);
    }
  }
  // fragment row of this thread inside the warpgroup's 64 rows (and +8), as a row of its owner's transpose tile
  const int frow = 16 * (w.wq & 1) + (lane >> 2), fcol = 2 * (lane & 3);
#pragma unroll
  for (int c = 0; c < kColsPerGrp; c += 32) {
    bar_sync(1 + w.wg, 128);                   // every transpose tile of the warpgroup is free again
#pragma unroll
    for (int gi = 0; gi < kGroups; ++gi) {
      float* Tt = w.Twg + ((w.wq >> 1) | (gi << 1)) * 32 * kTP;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int f = ((gi * kColsPerGrp + c) / 8 + j) * 4;
        *reinterpret_cast<float2*>(Tt + frow * kTP + 8 * j + fcol) = make_float2(acc[f], acc[f + 1]);
        *reinterpret_cast<float2*>(Tt + (frow + 8) * kTP + 8 * j + fcol) = make_float2(acc[f + 2], acc[f + 3]);
      }
    }
    bar_sync(1 + w.wg, 128);
    if (!active) continue;
    const int col = grp * kColsPerGrp + c;   // column inside the tile
    const int n0 = nt * BN + col;            // global column
    float v[32];
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      const float4 t = *reinterpret_cast<const float4*>(T + lane * kTP + j);
      v[j] = t.x; v[j + 1] = t.y; v[j + 2] = t.z; v[j + 3] = t.w;
    }
    __syncwarp();
    if (n0 >= p.N) continue;   // warp-uniform
    if (LNF && p.ln_stats) {
      const float4* cp = reinterpret_cast<const float4*>(p.ln_c1 + n0);
      const float mr = ln_mean * ln_rstd;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 c4 = __ldg(cp + j);
        v[4 * j] = fmaf(v[4 * j], ln_rstd, -mr * c4.x);
        v[4 * j + 1] = fmaf(v[4 * j + 1], ln_rstd, -mr * c4.y);
        v[4 * j + 2] = fmaf(v[4 * j + 2], ln_rstd, -mr * c4.z);
        v[4 * j + 3] = fmaf(v[4 * j + 3], ln_rstd, -mr * c4.w);
      }
    }
    if (p.bias) {
      const float4* bp = reinterpret_cast<const float4*>(p.bias + n0);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 b4 = __ldg(bp + j);
        v[4 * j] += b4.x; v[4 * j + 1] += b4.y; v[4 * j + 2] += b4.z; v[4 * j + 3] += b4.w;
      }
    }
    apply_act(p.act, v);
    if (p.store_mode == UDB_STORE_HEAD) {
      float head = p.head_b;
#pragma unroll
      for (int j = 0; j < 32; ++j) head = fmaf(v[j], __ldg(p.head_w + j), head);
      head = fminf(fmaxf(head, -8.0f), 8.0f) + p.head_add;
      if (valid) reinterpret_cast<float*>(p.out)[out_off] = expf(head);
      continue;
    }
    if (p.gamma) {
      const float4* gp = reinterpret_cast<const float4*>(p.gamma + n0);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 g4 = __ldg(gp + j);
        v[4 * j] *= g4.x; v[4 * j + 1] *= g4.y; v[4 * j + 2] *= g4.z; v[4 * j + 3] *= g4.w;
      }
    }
    long long coff = n0;
    if (p.store_mode == UDB_STORE_CONVT) {
      const int tap = n0 / p.ct_cout;
      const int co = n0 % p.ct_cout;
      const long long W2 = (long long)p.ct_w * p.ct_k + 2 * p.ct_pad;
      coff = ((long long)(tap / p.ct_k) * W2 + (tap % p.ct_k)) * p.ct_cout + co;
    }
    // ---- residual / stores through the per-warp transpose tile T[32][TP]: in registers a thread
    //      owns a row; in global memory 8 lanes x 16 B (f32) or 8 B (f16) cover one 32-column row
    //      segment and one instruction covers 4 rows, so every access is contiguous.  All smem
    //      traffic is 128-bit and conflict-free with the 36-float pitch.
    const uint32_t c32 = static_cast<uint32_t>(coff);
    const int l4 = (lane & 7) * 4, rq = lane >> 3;
    float* Trow = T + lane * kTP;
    auto stage_rows = [&](const float (&x)[32]) {      // thread == row  ->  T
#pragma unroll
      for (int j = 0; j < 32; j += 4)
        *reinterpret_cast<float4*>(Trow + j) = make_float4(x[j], x[j + 1], x[j + 2], x[j + 3]);
    };
    auto for_rows = [&](auto&& body) {                 // body(rr, valid) for this lane's 8 rows
      if (vmask == 0xffffffffu) {
#pragma unroll
        for (int i = 0; i < 8; ++i) body(4 * i + rq, true);
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) body(4 * i + rq, ((vmask >> (4 * i + rq)) & 1u) != 0);
      }
    };
    if (p.resid) {
      // all 8 row-segment loads of a lane are issued before the first use (latency-bound)
      if (p.resid_f32) {
        const float* rp = reinterpret_cast<const float*>(p.resid) + c32 + l4;
        float4 tmp[8];
        int k = 0;
        for_rows([&](int rr, bool ok) {
          tmp[k++] = ok ? *reinterpret_cast<const float4*>(rp + roff_res[rr]) : make_float4(0.f, 0.f, 0.f, 0.f);
        });
#pragma unroll
        for (int i = 0; i < 8; ++i) *reinterpret_cast<float4*>(T + (4 * i + rq) * kTP + l4) = tmp[i];
      } else {
        const __half* rp = reinterpret_cast<const __half*>(p.resid) + c32 + l4;
        uint2 tmp[8];
        int k = 0;
        for_rows([&](int rr, bool ok) {
          tmp[k++] = ok ? *reinterpret_cast<const uint2*>(rp + roff_res[rr]) : make_uint2(0u, 0u);
        });
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&tmp[i].x));
          const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&tmp[i].y));
          *reinterpret_cast<float4*>(T + (4 * i + rq) * kTP + l4) = make_float4(a.x, a.y, b.x, b.y);
        }
      }
      __syncwarp();
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const float4 t = *reinterpret_cast<const float4*>(Trow + j);
        v[j] += t.x; v[j + 1] += t.y; v[j + 2] += t.z; v[j + 3] += t.w;
      }
      __syncwarp();
    }
    if (LNF && p.stats_out) {
      if (st_first) { st_pivot = v[0]; st_first = false; }
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float dlt = v[j] - st_pivot;
        st_s1 += dlt;
        st_s2 = fmaf(dlt, dlt, st_s2);
      }
    }
    if (p.out) {
      stage_rows(v);
      __syncwarp();
      if (p.out_f32) {
        float* op = reinterpret_cast<float*>(p.out) + c32 + l4;
        for_rows([&](int rr, bool ok) {
          if (ok) *reinterpret_cast<float4*>(op + roff_out[rr]) = *reinterpret_cast<const float4*>(T + rr * kTP + l4);
        });
      } else {
        __half* op = reinterpret_cast<__half*>(p.out) + c32 + l4;
        if (p.out_split == 0) {
          for_rows([&](int rr, bool ok) {
            const float4 t = *reinterpret_cast<const float4*>(T + rr * kTP + l4);
            if (ok) *reinterpret_cast<uint2*>(op + roff_out[rr]) = make_uint2(pack_half2(t.x, t.y), pack_half2(t.z, t.w));
          });
        } else {   // split-f16 output: hi and lo = f16(v - f32(hi))
          for_rows([&](int rr, bool ok) {
            const float4 t = *reinterpret_cast<const float4*>(T + rr * kTP + l4);
            const uint2 hi = make_uint2(pack_half2(t.x, t.y), pack_half2(t.z, t.w));
            const float2 h01 = __half22float2(*reinterpret_cast<const __half2*>(&hi.x));
            const float2 h23 = __half22float2(*reinterpret_cast<const __half2*>(&hi.y));
            if (ok) {
              *reinterpret_cast<uint2*>(op + roff_out[rr]) = hi;
              *reinterpret_cast<uint2*>(op + roff_out[rr] + p.out_split) =
                  make_uint2(pack_half2(t.x - h01.x, t.y - h01.y), pack_half2(t.z - h23.x, t.w - h23.y));
            }
          });
        }
      }
      __syncwarp();
    }
    if (p.out2) {
      if (p.out2_leaky) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = leaky(v[j]);
        stage_rows(v);
      } else if (!p.out) {
        stage_rows(v);
      }   // else: T still holds v from the `out` pass
      __syncwarp();
      __half* op = p.out2 + c32 + l4;
      for_rows([&](int rr, bool ok) {
        const float4 t = *reinterpret_cast<const float4*>(T + rr * kTP + l4);
        if (ok) *reinterpret_cast<uint2*>(op + roff_out[rr]) = make_uint2(pack_half2(t.x, t.y), pack_half2(t.z, t.w));
      });
      __syncwarp();
    }
  }
  if (LNF && p.stats_out && active && valid && !st_first) {
    const float n = (float)kColsPerGrp;
    const float mean_p = st_pivot + st_s1 / n;
    const float m2_p = fmaxf(st_s2 - st_s1 * st_s1 / n, 0.f);
    const long long orow = out_off / p.ldc;
    reinterpret_cast<float2*>(p.stats_out)[orow * (p.tiles_n * kGroups) + nt * kGroups + grp] = make_float2(mean_p, m2_p);
  }
}

// Shared-memory state of the TMA epilogue.  `chunk` counts this warpgroup's 32-column chunks over all its tiles; chunk i
// uses buffer i & 1.  With a residual, the residual producer (warp 9) fills a buffer (full[b], expect_tx) once both
// warpgroups have released it (empty[b], one arrival per warpgroup after its TMA store has read the box).
struct EpiTma {
  uint8_t* buf;        // [2 buffers][2 warpgroups][kEpiBox]
  uint64_t* full;      // [2]
  uint64_t* empty;     // [2]
  uint32_t chunk;
};

// TMA epilogue of one tile (ROWS store, identity row map; udb_gemm_f16 checks the conditions in tma_epilogue_ok).
// Thread (warp wq, lane) of warpgroup g holds rows 16 wq + lane / 4 (+ 8) and columns 8 j + 2 (lane % 4) (+ 1) of every
// 32-column chunk; it applies the epilogue arithmetic there and writes the result into the swizzled box, one elected
// thread per warpgroup stores the box with TMA.  Rows past M are clipped by the tensor map.
template <int BN>
__device__ __forceinline__ void epilogue_tile_tma(const GemmArgs& p, const CUtensorMap* tmC, EpiTma& e,
                                                  const float (&acc)[BN / 2], const int mt, const int nt, const int wg,
                                                  const int wq, const int lane) {
  const bool leader = wq == 0 && lane == 0;   // issues, commits and waits for this warpgroup's stores
  const int q = lane & 3, rr = lane >> 2;     // rr == row & 7 for both fragment rows
  const bool has_res = p.resid != nullptr;
  const int row0 = mt * BM + 64 * wg;
#pragma unroll
  for (int c = 0; c < BN / 32; ++c, ++e.chunk) {
    const int b = e.chunk & 1;
    uint8_t* box = e.buf + (2 * b + wg) * kEpiBox;
    if (has_res) {
      mbar_wait(&e.full[b], (e.chunk >> 1) & 1);   // residual chunk landed (and the box's previous store has read it)
    } else {
      if (leader) bulk_wait_read<1>();             // the store issued from this box two chunks ago has read it
      bar_sync(1 + wg, 128);
    }
    const int n0 = nt * BN + 32 * c;
    float v[16];   // v[4 j + 2 h + x]: row 16 wq + rr + 8 h, column n0 + 8 j + 2 q + x
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = acc[16 * c + j];
    if (p.bias) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 b2 = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + 8 * j + 2 * q));
        v[4 * j] += b2.x; v[4 * j + 1] += b2.y; v[4 * j + 2] += b2.x; v[4 * j + 3] += b2.y;
      }
    }
    apply_act(p.act, v);
    if (p.gamma) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 g2 = __ldg(reinterpret_cast<const float2*>(p.gamma + n0 + 8 * j + 2 * q));
        v[4 * j] *= g2.x; v[4 * j + 1] *= g2.y; v[4 * j + 2] *= g2.x; v[4 * j + 3] *= g2.y;
      }
    }
    if (p.out_f32) {
      // 128B swizzle: 16-byte unit u of row r sits at unit u ^ (r & 7); conflict-free 8-byte accesses
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = 16 * wq + rr + 8 * h;
          float2* s = reinterpret_cast<float2*>(box + r * 128 + (((2 * j + (q >> 1)) ^ rr) << 4) + 8 * (q & 1));
          float x0 = v[4 * j + 2 * h], x1 = v[4 * j + 2 * h + 1];
          if (has_res) {
            const float2 t = *s;
            x0 += t.x; x1 += t.y;
          }
          *s = make_float2(x0, x1);
        }
      }
    } else {
      // 64B swizzle: 16-byte unit u of row r sits at unit u ^ ((r >> 1) & 3)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = 16 * wq + rr + 8 * h;
          *reinterpret_cast<uint32_t*>(box + r * 64 + ((j ^ ((r >> 1) & 3)) << 4) + 4 * q) =
              pack_half2(v[4 * j + 2 * h], v[4 * j + 2 * h + 1]);
        }
      }
    }
    fence_proxy_async_smem();   // the box's generic-proxy writes -> visible to the TMA store
    bar_sync(1 + wg, 128);
    if (leader) {
      if (row0 < p.M) tma_store_2d(tmC, box, n0, row0);
      bulk_commit();
      if (has_res) {
        bulk_wait_read<0>();
        mbar_arrive(&e.empty[b]);
      }
    }
  }
}

// TMAE: TMA epilogue (tmC: `out`, box 32 x 64; tmR: f32 `resid`, box 32 x 128; both unused otherwise)
template <int BN, bool LNF, bool TMAE>
__global__ void __launch_bounds__(kThreads, 1)
gemm_f16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR, const GemmArgs p) {
  static_assert(!(TMAE && LNF), "the TMA epilogue carries no fused-LayerNorm code");
  using Cfg = GemmCfg<BN, TMAE>;
  constexpr int kStages = Cfg::kStages;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sA = smem;
  uint8_t* sB = smem + kStages * Cfg::kABytes;
  uint8_t* staging = smem + kStages * Cfg::kStageBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(staging + Cfg::kStagingBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;
  uint64_t* epi_full = bars + 2 * kStages;    // TMA epilogue: [2] residual chunk landed in buffer b
  uint64_t* epi_empty = epi_full + 2;         //               [2] both warpgroups' stores have read buffer b

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();

  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023) __trap();   // 128B-swizzle atoms need a 1024 B aligned base
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kEpiWarps);   // every consumer warp releases the stage after its own wgmma wait
    }
    if constexpr (TMAE) {
      prefetch_tmap(&tmC);
      if (p.resid) prefetch_tmap(&tmR);
      for (int i = 0; i < 2; ++i) {
        mbar_init(&epi_full[i], 1);
        mbar_init(&epi_empty[i], 2);
      }
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();   // everything above overlapped the previous kernel's tail

  const int num_tiles = p.tiles_m * p.tiles_n;

  if (warp >= kEpiWarps) {
    setmaxnreg_dec<40>();
    if constexpr (TMAE) {
      if (warp == kEpiWarps + 1 && p.resid) {
        // ---------------------------------------------------------------- residual producer (TMA epilogue)
        // Loads every 32-column residual chunk of this CTA's tiles, in the order the consumers store them, as soon as
        // the buffer is free; the first two chunks of a tile so arrive during its main loop.
        const bool elected = elect_one();
        uint32_t chunk = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
          const int mt = tile / p.tiles_n;
          const int nt = tile % p.tiles_n;
          for (int c = 0; c < BN / 32; ++c, ++chunk) {
            const int b = chunk & 1;
            mbar_wait(&epi_empty[b], ((chunk >> 1) & 1) ^ 1);
            if (elected) {
              mbar_arrive_expect_tx(&epi_full[b], 2 * kEpiBox);
              tma_load_2d(staging + 2 * b * kEpiBox, &tmR, &epi_full[b], nt * BN + 32 * c, mt * BM);
            }
            __syncwarp();
          }
        }
      }
    }
    if (warp != kEpiWarps) return;
    // ------------------------------------------------------------------ TMA producer
    // (whole warp in the control flow, one elected lane issues: keeps addresses/descriptors in uniform
    //  registers -- under a lane-0 branch ptxas wraps each TMA in an ELECT+R2UR waterfall loop)
    const bool elected = elect_one();
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int mt = tile / p.tiles_n;
      const int nt = tile % p.tiles_n;
      int cb = 0, cy = 0, cx = 0;
      if (p.a_mode == UDB_A_CONV3X3) {
        const int per_img = p.conv_tx * p.conv_ty;
        cb = mt / per_img;
        const int r = mt % per_img;
        cy = (r / p.conv_tx) * p.conv_TH + p.conv_off;
        cx = (r % p.conv_tx) * p.conv_TW + p.conv_off;
      }
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (elected) {
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if (p.a_mode == UDB_A_CONV3X3) {
            const int tap = kb / p.conv_cpb;
            const int c0 = p.conv_coff + (kb % p.conv_cpb) * BK;
            tma_load_4d(sA + stage * Cfg::kABytes, &tmA, &full_bar[stage], c0, cx + tap % 3, cy + tap / 3, cb);
          } else {
            int ka = kb * BK;
            if (p.a_wrap && ka >= p.a_wrap) ka -= p.a_wrap;
            tma_load_2d(sA + stage * Cfg::kABytes, &tmA, &full_bar[stage], ka, mt * BM);
          }
          tma_load_2d(sB + stage * Cfg::kBBytes, &tmB, &full_bar[stage], kb * BK, nt * BN);
        }
        __syncwarp();
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ MMA + epilogue (two warpgroups)
    setmaxnreg_inc<232>();
    const int wg = warp >> 2, wq = warp & 3;
    float* Twg = reinterpret_cast<float*>(staging) + wg * 4 * 32 * kTP;
    uint32_t* roff = reinterpret_cast<uint32_t*>(staging + kEpiWarps * 32 * kTP * 4) + warp * 64;
    const EpiWarp ctx{Twg + wq * 32 * kTP, Twg, roff, roff + 32, wg, wq, wq >> 1, lane, 64 * wg + 32 * (wq & 1) + lane};
    EpiTma etma{staging, epi_full, epi_empty, 0};
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int mt = tile / p.tiles_n;
      const int nt = tile % p.tiles_n;
      int prev = -1;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t da = gmma_desc_sw128(smem_u32(sA + stage * Cfg::kABytes + wg * 64 * 128), 16, 1024);
        const uint64_t db = gmma_desc_sw128(smem_u32(sB + stage * Cfg::kBBytes), 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) WgmmaSS<BN>::run(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();   // the previous k-block's MMAs are done: release its stage
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      if constexpr (TMAE) epilogue_tile_tma<BN>(p, &tmC, etma, acc, mt, nt, wg, wq, lane);
      else epilogue_tile<BN, LNF>(p, ctx, acc, mt, nt);
    }
    if constexpr (TMAE) {
      if (wq == 0 && lane == 0) bulk_wait<0>();   // the last stores have written global memory before the CTA retires
    }
  }
}

template <int BN, bool LNF, bool TMAE>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const CUtensorMap& tmR,
                       const GemmArgs& a, cudaStream_t st) {
  using Cfg = GemmCfg<BN, TMAE>;
  static std::atomic<uint64_t> attr_mask{0};
  if (first_on_device(attr_mask)) {
    cudaError_t e = cudaFuncSetAttribute(gemm_f16_kernel<BN, LNF, TMAE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      set_error("gemm: cudaFuncSetAttribute(%d B smem): %s", Cfg::kSmemBytes, cudaGetErrorString(e));
      return 1;
    }
  }
  const int tiles = a.tiles_m * a.tiles_n;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  cudaError_t e = launch_ex(gemm_f16_kernel<BN, LNF, TMAE>, dim3(grid), dim3(kThreads), Cfg::kSmemBytes, st, 1, tmA, tmB, tmC,
                            tmR, a);
  if (e != cudaSuccess) {
    set_error("gemm_f16_kernel launch: %s", cudaGetErrorString(e));
    return 1;
  }
  return check_launch("gemm_f16_kernel");
}

static bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

// Layouts the epilogue's vector accesses and 32-bit row offsets can handle (include/udb.h, udb_gemm_t).  Host-only: runs
// before any CUDA call, so a rejected call launches nothing.
static int check_gemm_layout(const udb_gemm_t* g) {
  const int sm = g->store_mode;
  if (g->M < 1 || g->N < 1 || g->K < 1) { set_error("udb_gemm_f16: M=%d N=%d K=%d must be >= 1", g->M, g->N, g->K); return 1; }
  if (sm < UDB_STORE_ROWS || sm > UDB_STORE_HEAD) { set_error("udb_gemm_f16: unknown store_mode %d", sm); return 1; }
  const long long ldr = g->ldr > 0 ? g->ldr : g->ldc;
  // every vector load / store of the epilogue: f32 rows move as float4, f16 rows as 4 halves (uint2)
  if (sm == UDB_STORE_HEAD) {
    if (!g->out || !g->out_f32 || !aligned(g->out, 4)) { set_error("udb_gemm_f16: HEAD store needs a 4-byte aligned f32 `out`"); return 1; }
    if (!g->head_w || !aligned(g->head_w, 16)) { set_error("udb_gemm_f16: `head_w` must be non-null and 16-byte aligned"); return 1; }
  } else {
    if (g->out && !aligned(g->out, g->out_f32 ? 16 : 8)) {
      set_error("udb_gemm_f16: `out` %p must be %d-byte aligned", g->out, g->out_f32 ? 16 : 8); return 1;
    }
    if (g->out2 && !aligned(g->out2, 8)) { set_error("udb_gemm_f16: `out2` %p must be 8-byte aligned", g->out2); return 1; }
    if (g->resid && !aligned(g->resid, g->resid_f32 ? 16 : 8)) {
      set_error("udb_gemm_f16: `resid` %p must be %d-byte aligned", g->resid, g->resid_f32 ? 16 : 8); return 1;
    }
    if (sm != UDB_STORE_CONVT) {   // CONVT addresses its pixels through ct_cout, not ldc / ldr
      if ((g->out || g->out2) && (g->ldc < 1 || g->ldc % 4)) { set_error("udb_gemm_f16: `ldc`=%lld must be a positive multiple of 4", (long long)g->ldc); return 1; }
      if (g->resid && (ldr < 1 || ldr % 4)) { set_error("udb_gemm_f16: `ldr`=%lld must be a positive multiple of 4", ldr); return 1; }
      if ((g->out || g->out2) && g->ldc < (long long)g->N + g->out_split) {
        set_error("udb_gemm_f16: `ldc`=%lld < N + out_split = %lld: rows would overlap", (long long)g->ldc, (long long)g->N + g->out_split);
        return 1;
      }
      if (g->resid && ldr < g->N) { set_error("udb_gemm_f16: `ldr`=%lld < N=%d: residual rows would overlap", ldr, g->N); return 1; }
    }
  }
  if (g->out_split < 0 || g->out_split % 4) { set_error("udb_gemm_f16: `out_split`=%d must be a non-negative multiple of 4", g->out_split); return 1; }
  if (!aligned(g->bias, 16)) { set_error("udb_gemm_f16: `bias` %p must be 16-byte aligned", (const void*)g->bias); return 1; }
  if (!aligned(g->gamma, 16)) { set_error("udb_gemm_f16: `gamma` %p must be 16-byte aligned", (const void*)g->gamma); return 1; }
  if (!aligned(g->ln_c1, 16)) { set_error("udb_gemm_f16: `ln_c1` %p must be 16-byte aligned", (const void*)g->ln_c1); return 1; }
  if (!aligned(g->ln_stats_out, 8) || !aligned(g->ln_stats_in, 8)) { set_error("udb_gemm_f16: `ln_stats_*` must be 8-byte aligned"); return 1; }

  // the epilogue keeps each row's element offset in 32 bits (EpiWarp::roff_out / roff_res)
  long long out_row = 0, res_row = 0;   // element offset of the last row written / read
  if (sm == UDB_STORE_ROWS) {
    const int m = g->M - 1;
    long long orow = m;
    if (g->rows_per_group > 0) {
      if (g->group_stride < 0 || g->row_offset < 0) {
        set_error("udb_gemm_f16: `group_stride`=%d and `row_offset`=%d must be >= 0", g->group_stride, g->row_offset); return 1;
      }
      const long long rpg = g->rows_per_group, grp = m / rpg;
      orow = grp * g->group_stride + m % rpg + g->row_offset;
      if (grp > 0 && (grp - 1) * g->group_stride + rpg - 1 + g->row_offset > orow) orow = (grp - 1) * g->group_stride + rpg - 1 + g->row_offset;
    }
    long long rrow = orow;
    if (g->resid_mod > 0) {
      if (g->resid_row_offset < 0) { set_error("udb_gemm_f16: `resid_row_offset`=%d must be >= 0", g->resid_row_offset); return 1; }
      rrow = (long long)(g->resid_mod < g->M ? g->resid_mod : g->M) - 1 + g->resid_row_offset;
    }
    out_row = orow * g->ldc;
    res_row = rrow * ldr;
  } else if (sm == UDB_STORE_CONVT) {
    if (g->ct_k < 1 || g->ct_h < 1 || g->ct_w < 1 || g->ct_pad < 0 || g->ct_cout < 1) {
      set_error("udb_gemm_f16: CONVT geometry `ct_k`=%d `ct_h`=%d `ct_w`=%d `ct_pad`=%d `ct_cout`=%d", g->ct_k, g->ct_h, g->ct_w, g->ct_pad,
                g->ct_cout);
      return 1;
    }
    if (g->N != g->ct_k * g->ct_k * g->ct_cout) { set_error("udb_gemm_f16: CONVT needs N == ct_k^2 * ct_cout (N=%d)", g->N); return 1; }
    const long long m = g->M - 1, hw = (long long)g->ct_h * g->ct_w, b = m / hw, r = m % hw, y = r / g->ct_w, x = r % g->ct_w;
    const long long W2 = (long long)g->ct_w * g->ct_k + 2 * g->ct_pad, H2 = (long long)g->ct_h * g->ct_k + 2 * g->ct_pad;
    out_row = res_row = ((b * H2 + y * g->ct_k + g->ct_pad) * W2 + x * g->ct_k + g->ct_pad) * g->ct_cout;
  } else {
    if (g->conv_B < 1 || g->conv_H < 1 || g->conv_W < 1) {
      set_error("udb_gemm_f16: conv_B=%d conv_H=%d conv_W=%d must be >= 1", g->conv_B, g->conv_H, g->conv_W); return 1;
    }
    const long long last_px = (long long)g->conv_B * g->conv_H * g->conv_W - 1;
    out_row = last_px * g->ldc;
    res_row = last_px * ldr;
  }
  const long long lim = 1ll << 32;
  if ((g->out || g->out2) && out_row >= lim) { set_error("udb_gemm_f16: `out` row offset %lld exceeds 2^32 elements", out_row); return 1; }
  if (g->resid && res_row >= lim) { set_error("udb_gemm_f16: `resid` row offset %lld exceeds 2^32 elements", res_row); return 1; }

  if (g->a_mode == UDB_A_CONV3X3) {
    const int pad = g->conv_off == 0 ? 2 : (g->conv_off == -1 ? 0 : -1);
    if (pad < 0) { set_error("udb_gemm_f16: `conv_off`=%d must be 0 (prepadded) or -1 (zero padding)", g->conv_off); return 1; }
    if (g->conv_inH != g->conv_H + pad || g->conv_inW != g->conv_W + pad) {
      set_error("udb_gemm_f16: `conv_inH`x`conv_inW` = %dx%d must be %dx%d for conv_off %d", g->conv_inH, g->conv_inW, g->conv_H + pad,
                g->conv_W + pad, g->conv_off);
      return 1;
    }
  }
  return 0;
}

// Calls the TMA epilogue serves: a plain ROWS store (identity row map, no second output, split output or fused LayerNorm
// statistics) whose `out` -- and f32 `resid`, if any, with an f32 `out` -- TMA can address: 16-byte aligned bases and row
// pitches.  The rest run the general epilogue; this only chooses the path and never fails a call.
// UDB_GEMM_TMA_EPILOGUE=0 (read on every call) sends every call to the general epilogue, for A/B comparisons.
static bool tma_epilogue_ok(const udb_gemm_t* g) {
  const char* env = getenv("UDB_GEMM_TMA_EPILOGUE");
  if (env && atoi(env) == 0) return false;
  if (g->store_mode != UDB_STORE_ROWS || g->a_mode != UDB_A_MATRIX || g->rows_per_group > 0 || g->resid_mod > 0) return false;
  if (g->out_split || g->out2 || g->ln_stats_out || g->ln_stats_in || !g->out) return false;
  if (!aligned(g->out, 16) || (g->ldc * (g->out_f32 ? 4 : 2)) % 16) return false;
  const long long ldr = g->ldr > 0 ? g->ldr : g->ldc;
  return !g->resid || (g->resid_f32 && g->out_f32 && aligned(g->resid, 16) && (ldr * 4) % 16 == 0);
}

static thread_local int g_last_tma_epilogue = 0;

}  // namespace udb

extern "C" int udb_gemm_tma_epilogue_used(void) { return udb::g_last_tma_epilogue; }

extern "C" int udb_gemm_f16(const udb_gemm_t* g, void* stream) {
  using namespace udb;
  if (!g || !g->a || !g->w) { set_error("udb_gemm_f16: null operand"); return 1; }
  if (g->N % 32 != 0) { set_error("udb_gemm_f16: N=%d must be a multiple of 32", g->N); return 1; }
  if (check_gemm_layout(g)) return 1;
  GemmArgs a{};
  a.M = g->M; a.N = g->N; a.K = g->K;
  a.num_kb = (g->K + BK - 1) / BK;
  a.a_mode = g->a_mode;
  a.bias = g->bias; a.gamma = g->gamma; a.resid = g->resid; a.resid_f32 = g->resid_f32;
  a.out = g->out; a.out_f32 = g->out_f32; a.out2 = reinterpret_cast<__half*>(g->out2); a.out2_leaky = g->out2_leaky;
  a.act = g->act; a.store_mode = g->store_mode;
  a.ldc = g->ldc; a.ldr = g->ldr > 0 ? g->ldr : g->ldc;
  a.rpg = g->rows_per_group; a.gstride = g->group_stride; a.roff = g->row_offset;
  a.resid_mod = g->resid_mod; a.resid_roff = g->resid_row_offset;
  a.ct_k = g->ct_k; a.ct_cout = g->ct_cout; a.ct_h = g->ct_h; a.ct_w = g->ct_w; a.ct_pad = g->ct_pad;
  a.conv_coff = g->conv_coff;
  a.head_w = g->head_w; a.head_b = g->head_b; a.head_add = g->head_add;
  a.a_wrap = 0;
  a.out_split = g->out_split;
  if (g->a_split_k > 0) {
    if (g->a_mode != UDB_A_MATRIX || g->a_split_k % BK || g->K != 3 * g->a_split_k || g->lda < 2 * g->a_split_k) {
      set_error("udb_gemm_f16: split operands need a_mode MATRIX, K1 %% 64 == 0, K == 3*K1, lda >= 2*K1 (K1=%d K=%d lda=%d)",
                g->a_split_k, g->K, g->lda);
      return 1;
    }
    a.a_wrap = 2 * g->a_split_k;
  }
  a.stats_out = g->ln_stats_out; a.ln_stats = g->ln_stats_in; a.ln_c1 = g->ln_c1; a.ln_eps = g->ln_eps;
  a.ln_parts = g->ln_parts; a.ln_part_cols = g->ln_part_cols;
  if ((g->ln_stats_out || g->ln_stats_in) && g->store_mode != UDB_STORE_ROWS) {
    set_error("udb_gemm_f16: fused LayerNorm statistics need the ROWS store"); return 1;
  }
  if (g->ln_stats_in && (!g->ln_c1 || g->ln_parts <= 0 || g->ln_part_cols <= 0 || g->rows_per_group > 0)) {
    set_error("udb_gemm_f16: ln_stats_in needs ln_c1, ln_parts, ln_part_cols and an identity row map"); return 1;
  }
  if (g->out_split && (g->out_f32 || !g->out || g->store_mode != UDB_STORE_ROWS)) {
    set_error("udb_gemm_f16: out_split needs an f16 `out` with the ROWS store"); return 1;
  }

  // tile width: widest that divides the work sensibly
  int bn;
  if (g->store_mode == UDB_STORE_HEAD) {
    if (g->N != 32) { set_error("udb_gemm_f16: HEAD store needs N == 32"); return 1; }
    bn = 32;
  } else if (g->N % 256 == 0) bn = 256;
  else if (g->N % 192 == 0) bn = 192;      // ConvNeXt widths 192 / 384: 3 (or 6) times fewer passes over A than 64 / 128
  else if (g->N % 128 == 0) bn = 128;
  else if (g->N % 64 == 0) bn = 64;
  else bn = 32;
  if (g->store_mode == UDB_STORE_CONVT && (g->ct_cout % 32) != 0) {
    set_error("udb_gemm_f16: CONVT needs Cout %% 32 == 0"); return 1;
  }
  a.tiles_n = (g->N + bn - 1) / bn;
  if (g->ln_stats_out) {
    const int groups = bn >= 64 ? 2 : 1;
    if (g->N % bn || g->ln_parts != a.tiles_n * groups || g->ln_part_cols != bn / groups) {
      set_error("udb_gemm_f16: ln_stats_out with N=%d runs as %d parts of %d columns (caller said %d x %d)", g->N, a.tiles_n * groups,
                bn / groups, g->ln_parts, g->ln_part_cols);
      return 1;
    }
  }

  CUtensorMap tmA, tmB;
  if (g->a_mode == UDB_A_CONV3X3) {
    if (g->conv_C % BK != 0 || g->K != 9 * g->conv_C) {
      set_error("udb_gemm_f16: conv3x3 needs C %% 64 == 0 and K == 9*C (C=%d K=%d)", g->conv_C, g->K);
      return 1;
    }
    if (g->store_mode != UDB_STORE_CONVTILE && g->store_mode != UDB_STORE_HEAD) {
      set_error("udb_gemm_f16: conv3x3 operand needs a CONVTILE or HEAD store"); return 1;
    }
    const int TH = g->conv_TH > 0 ? g->conv_TH : 8, TW = g->conv_TW > 0 ? g->conv_TW : 16;
    if (TH * TW != BM) { set_error("udb_gemm_f16: conv tile %dx%d != 128 pixels", TH, TW); return 1; }
    a.conv_B = g->conv_B; a.conv_H = g->conv_H; a.conv_W = g->conv_W; a.conv_cpb = g->conv_C / BK; a.conv_off = g->conv_off;
    a.conv_TH = TH; a.conv_TW = TW;
    a.conv_tx = (g->conv_W + TW - 1) / TW; a.conv_ty = (g->conv_H + TH - 1) / TH;
    a.tiles_m = g->conv_B * a.conv_tx * a.conv_ty;
    a.M = a.tiles_m * BM;
    const uint64_t cs = g->conv_cstride > 0 ? g->conv_cstride : g->conv_C;
    if ((uint64_t)g->conv_coff + g->conv_C > cs || (g->conv_coff % 8)) {
      set_error("udb_gemm_f16: bad conv channel slice (off %d, C %d, stride %d)", g->conv_coff, g->conv_C, (int)cs);
      return 1;
    }
    const uint64_t dims[4] = {cs, (uint64_t)g->conv_inW, (uint64_t)g->conv_inH, (uint64_t)g->conv_B};
    const uint64_t str[3] = {cs * 2, (uint64_t)g->conv_inW * cs * 2, (uint64_t)g->conv_inH * g->conv_inW * cs * 2};
    const uint32_t box[4] = {(uint32_t)BK, (uint32_t)TW, (uint32_t)TH, 1};
    if (make_tmap_f16(&tmA, g->a, 4, dims, str, box, true)) return 1;
  } else {
    a.tiles_m = (g->M + BM - 1) / BM;
    if (g->store_mode == UDB_STORE_CONVTILE || g->store_mode == UDB_STORE_HEAD) {
      set_error("udb_gemm_f16: tile store modes need a_mode == CONV3X3"); return 1;
    }
    const uint64_t dims[2] = {(uint64_t)(g->a_split_k > 0 ? 2 * g->a_split_k : g->K), (uint64_t)g->M};
    const uint64_t str[1] = {(uint64_t)g->lda * 2};
    const uint32_t box[2] = {(uint32_t)BK, (uint32_t)BM};
    if (make_tmap_f16(&tmA, g->a, 2, dims, str, box, true)) return 1;
  }
  {
    const uint64_t dims[2] = {(uint64_t)g->K, (uint64_t)g->N};
    const uint64_t str[1] = {(uint64_t)g->ldw * 2};
    const uint32_t box[2] = {(uint32_t)BK, (uint32_t)bn};
    if (make_tmap_f16(&tmB, g->w, 2, dims, str, box, true)) return 1;
  }
  const bool tmae = tma_epilogue_ok(g);
  CUtensorMap tmC, tmR;
  memset(&tmC, 0, sizeof(tmC));
  memset(&tmR, 0, sizeof(tmR));
  if (tmae) {
    const uint64_t dims[2] = {(uint64_t)g->N, (uint64_t)g->M};
    const uint64_t str_c[1] = {(uint64_t)g->ldc * (g->out_f32 ? 4 : 2)};
    const uint32_t box_c[2] = {32, 64};
    if (make_tmap(&tmC, g->out, 2, dims, str_c, box_c, g->out_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                  g->out_f32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B))
      return 1;
    if (g->resid) {
      const uint64_t str_r[1] = {(uint64_t)a.ldr * 4};
      const uint32_t box_r[2] = {32, BM};
      if (make_tmap(&tmR, g->resid, 2, dims, str_r, box_r, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
    }
  }
  g_last_tma_epilogue = tmae ? 1 : 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  note_work(2.0 * a.M * (double)g->N * g->K,
            2.0 * ((double)a.M * (g->a_mode == UDB_A_CONV3X3 ? g->conv_C : (g->a_split_k ? 2 * g->a_split_k : g->K)) + (double)g->N * g->K) +
                (double)a.M * g->N * ((g->out ? (g->out_f32 ? 4 : 2) : 0) + (g->out2 ? 2 : 0) + (g->resid ? (g->resid_f32 ? 4 : 2) : 0)));
  const bool lnf = g->ln_stats_out || g->ln_stats_in;
  if (lnf) {
    switch (bn) {
      case 256: return launch_gemm<256, true, false>(tmA, tmB, tmC, tmR, a, st);
      case 192: return launch_gemm<192, true, false>(tmA, tmB, tmC, tmR, a, st);
      case 128: return launch_gemm<128, true, false>(tmA, tmB, tmC, tmR, a, st);
      case 64: return launch_gemm<64, true, false>(tmA, tmB, tmC, tmR, a, st);
      default: return launch_gemm<32, true, false>(tmA, tmB, tmC, tmR, a, st);
    }
  }
  if (tmae) {
    switch (bn) {
      case 256: return launch_gemm<256, false, true>(tmA, tmB, tmC, tmR, a, st);
      case 192: return launch_gemm<192, false, true>(tmA, tmB, tmC, tmR, a, st);
      case 128: return launch_gemm<128, false, true>(tmA, tmB, tmC, tmR, a, st);
      case 64: return launch_gemm<64, false, true>(tmA, tmB, tmC, tmR, a, st);
      default: return launch_gemm<32, false, true>(tmA, tmB, tmC, tmR, a, st);
    }
  }
  switch (bn) {
    case 256: return launch_gemm<256, false, false>(tmA, tmB, tmC, tmR, a, st);
    case 192: return launch_gemm<192, false, false>(tmA, tmB, tmC, tmR, a, st);
    case 128: return launch_gemm<128, false, false>(tmA, tmB, tmC, tmR, a, st);
    case 64: return launch_gemm<64, false, false>(tmA, tmB, tmC, tmR, a, st);
    default: return launch_gemm<32, false, false>(tmA, tmB, tmC, tmR, a, st);
  }
}
