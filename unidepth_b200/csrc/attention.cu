// Fused attention forward for sm_90a:  O = softmax(Q K^T * scale) V   (no mask, no dropout), head dim 64.
// One kernel, attn_fwd_kernel (design notes in front of it); a split-f16 fp32 variant for the parity mode at the end.
// Replaces F.scaled_dot_product_attention (reference: metadinov2/attention.py:58, layers/attention.py:136).
#include "common.h"
#include "ptx.cuh"

namespace udb {

constexpr int AT_BQ = 128;       // queries per CTA (two warpgroups of 64)
constexpr int AT_BK = 128;       // keys per tile
constexpr int AT_STAGES = 3;     // K / V rings
constexpr int AT_THREADS = 288;  // two consumer warpgroups + the TMA warp

struct AttnArgs {
  __half* out;
  int seq_q, seq_k, n_kv_tiles;
  int ldo, o_col0;
  int q_col0, k_col0, v_col0;
  float scale_log2;
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// ---------------------------------------------------------------------------------------------
// One CTA = one (batch, head, 128-query tile).  Warps 0..7 are two consumer warpgroups, warpgroup g owns queries
// [64g, 64g+64); warp 8 is the TMA producer (Q once, K / V tiles of 128 keys through AT_STAGES-deep rings).  Per key tile
// a warpgroup computes S = Q K^T with one m64n128 wgmma chain (both operands in shared memory), runs the online softmax
// on the accumulator registers (a row lives in the four lanes of a quad: max / sum by two shuffles), converts P to f16
// in place -- the m64n128 accumulator fragment of keys [16k, 16k+16) is exactly the register A fragment of the k-th
// m64k16 step -- and accumulates O += P V with register-A wgmmas (V read MN-major from shared memory).  P never touches
// shared memory; the two warpgroups run independently and overlap each other's softmax with their MMAs.
// ---------------------------------------------------------------------------------------------
template <int HD>
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnArgs p) {
  static_assert(HD == 64, "head_dim 64 only");
  constexpr int kQBytes = AT_BQ * HD * 2;      // 16 KB
  constexpr int kKBytes = AT_BK * HD * 2;      // 16 KB
  constexpr int NS = AT_STAGES;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kQBytes;                  // NS stages
  uint8_t* sV = sK + NS * kKBytes;             // NS stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + NS * kKBytes);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;             // [NS]
  uint64_t* v_full = k_full + NS;          // [NS]
  uint64_t* k_empty = v_full + NS;         // [NS]  every consumer warp's QK^T of the tile has completed
  uint64_t* v_empty = k_empty + NS;        // [NS]  every consumer warp's PV of the tile has completed

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * AT_BQ;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int n_tiles = p.n_kv_tiles;
  pdl_launch_dependents();

  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023) __trap();
    prefetch_tmap(&tmQ);
    prefetch_tmap(&tmK);
    prefetch_tmap(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < NS; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&k_empty[i], 8);
      mbar_init(&v_empty[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == 8) {
    const bool leader = elect_one();
    if (leader) {
      mbar_arrive_expect_tx(q_full, kQBytes);
      tma_load_3d(sQ, &tmQ, q_full, p.q_col0 + head * HD, q0, b);
    }
    __syncwarp();
    int st = 0;
    uint32_t ph = 1;
    for (int j = 0; j < n_tiles; ++j) {
      mbar_wait(&k_empty[st], ph);
      if (leader) {
        mbar_arrive_expect_tx(&k_full[st], kKBytes);
        tma_load_3d(sK + st * kKBytes, &tmK, &k_full[st], p.k_col0 + head * HD, j * AT_BK, b);
      }
      __syncwarp();
      mbar_wait(&v_empty[st], ph);
      if (leader) {
        mbar_arrive_expect_tx(&v_full[st], kKBytes);
        tma_load_3d(sV + st * kKBytes, &tmV, &v_full[st], p.v_col0 + head * HD, j * AT_BK, b);
      }
      __syncwarp();
      if (++st == NS) { st = 0; ph ^= 1; }
    }
    return;
  }

  // ------------------------------------------------------------------ consumer warpgroups
  const int wg = warp >> 2, wq = warp & 3;
  const int cq = 2 * (lane & 3);                       // first of this thread's two columns in every 8-column group
  const float sc = p.scale_log2;
  const uint64_t dq = gmma_desc_sw128(smem_u32(sQ + wg * 64 * 128), 16, 1024);
  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // rows lane/4 and lane/4 + 8 of the warp's 16
  mbar_wait(q_full, 0);
  int st = 0;
  uint32_t ph = 0;
  for (int j = 0; j < n_tiles; ++j) {
    float s[AT_BK / 2];
    mbar_wait(&k_full[st], ph);
    {
      const uint64_t dk = gmma_desc_sw128(smem_u32(sK + st * kKBytes), 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < HD / 16; ++k) wgmma_ss_n128(s, dq + 2 * k, dk + 2 * k, k != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(s);
    }
    if (lane == 0) mbar_arrive(&k_empty[st]);
    const int kv_left = p.seq_k - j * AT_BK;           // valid keys in this tile (>= 1)
    if (kv_left < AT_BK) {
#pragma unroll
      for (int i = 0; i < AT_BK / 2; ++i)
        if (8 * (i >> 2) + cq + (i & 1) >= kv_left) s[i] = -INFINITY;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < AT_BK / 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx * sc);
      const float alpha = ex2(m_run[h] - m_new);        // 0 on the first tile
      m_run[h] = m_new;
      float ls = 0.f;
#pragma unroll
      for (int jj = 0; jj < AT_BK / 8; ++jj) {
        const float e0 = ex2(fmaf(s[4 * jj + 2 * h], sc, -m_new));
        const float e1 = ex2(fmaf(s[4 * jj + 2 * h + 1], sc, -m_new));
        s[4 * jj + 2 * h] = e0;
        s[4 * jj + 2 * h + 1] = e1;
        ls += e0 + e1;
      }
      l_run[h] = fmaf(l_run[h], alpha, ls);
#pragma unroll
      for (int jj = 0; jj < HD / 8; ++jj) {
        o[4 * jj + 2 * h] *= alpha;
        o[4 * jj + 2 * h + 1] *= alpha;
      }
    }
    uint32_t pa[AT_BK / 16][4];
#pragma unroll
    for (int kk = 0; kk < AT_BK / 16; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) pa[kk][r] = pack_half2(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
    mbar_wait(&v_full[st], ph);
    {
      // V tile [128 keys][64] is the MN-major B operand; keys [16kk, 16kk+16) start 2 KB apart
      const uint64_t dv = gmma_desc_sw128(smem_u32(sV + st * kKBytes), 1024, 1024);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < AT_BK / 16; ++kk) wgmma_rs_n64_tb(o, pa[kk], dv + (uint64_t)(kk * 2048 >> 4), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
    }
    if (lane == 0) mbar_arrive(&v_empty[st]);
    if (++st == NS) { st = 0; ph ^= 1; }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.0f / l;
    const int q = q0 + 64 * wg + 16 * wq + (lane >> 2) + 8 * h;
    if (q < p.seq_q) {
      __half* op = p.out + ((long long)b * p.seq_q + q) * p.ldo + p.o_col0 + head * HD + cq;
#pragma unroll
      for (int jj = 0; jj < HD / 8; ++jj)
        *reinterpret_cast<uint32_t*>(op + 8 * jj) = pack_half2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Split-f16 ("precise") attention: operands arrive as hi + lo f16 pairs, everything is computed in
// fp32 on the CUDA cores (exact expf, f32 products and sums) and the result leaves as a hi/lo pair.
// A parity / debugging mode (udb_attn_t.split): it exists to show that the default path's residual
// against the fp32 reference is operand rounding, not logic.  64 queries x 64 keys per step, 256 threads,
// thread (ty, tx) owns rows ty+16i and columns / head dims tx+16j.
// ---------------------------------------------------------------------------------------------
constexpr int SP_T = 64;          // tile edge
constexpr int SP_P = 65;          // smem pitch (floats): conflict-free row-strided reads
constexpr int SP_SMEM = (4 * SP_T * SP_P + 3 * SP_T) * 4;

__global__ void __launch_bounds__(256) attn_split_f32_kernel(const udb_attn_t a) {
  extern __shared__ float sp_smem[];
  float* Qs = sp_smem;
  float* Ks = Qs + SP_T * SP_P;
  float* Vs = Ks + SP_T * SP_P;
  float* Ps = Vs + SP_T * SP_P;
  float* m_s = Ps + SP_T * SP_P;
  float* l_s = m_s + SP_T;
  float* al_s = l_s + SP_T;
  const int t = threadIdx.x, ty = t >> 4, tx = t & 15;
  const int q0 = blockIdx.x * SP_T, h = blockIdx.y, b = blockIdx.z;
  const __half* qp = reinterpret_cast<const __half*>(a.q);
  const __half* kp = reinterpret_cast<const __half*>(a.k);
  const __half* vp = reinterpret_cast<const __half*>(a.v);
  auto ld = [](const __half* base, long long off, int lo_off) {
    return __half2float(base[off]) + (lo_off ? __half2float(base[off + lo_off]) : 0.f);
  };
  for (int i = t; i < SP_T * SP_T; i += 256) {
    const int r = i >> 6, d = i & 63;
    const int sq = q0 + r;
    Qs[r * SP_P + d] = sq < a.seq_q ? ld(qp, ((long long)b * a.seq_q + sq) * a.ldq + a.q_col0 + h * 64 + d, a.lo_off_q) * a.scale : 0.f;
  }
  if (t < SP_T) { m_s[t] = -INFINITY; l_s[t] = 0.f; }
  float O[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) O[i][j] = 0.f;
  const int n_kt = (a.seq_k + SP_T - 1) / SP_T;
  for (int kt = 0; kt < n_kt; ++kt) {
    __syncthreads();     // previous tile's Ks / Vs / Ps fully consumed (and Qs / m / l initialised)
    for (int i = t; i < SP_T * SP_T; i += 256) {
      const int r = i >> 6, d = i & 63;
      const int sk = kt * SP_T + r;
      const bool ok = sk < a.seq_k;
      const long long row = (long long)b * a.seq_k + sk;
      Ks[r * SP_P + d] = ok ? ld(kp, row * a.ldk + a.k_col0 + h * 64 + d, a.lo_off_k) : 0.f;
      Vs[r * SP_P + d] = ok ? ld(vp, row * a.ldv + a.v_col0 + h * 64 + d, a.lo_off_v) : 0.f;
    }
    __syncthreads();
    float S[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) S[i][j] = 0.f;
    for (int d = 0; d < 64; ++d) {
      float qv[4], kv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) qv[i] = Qs[(ty + 16 * i) * SP_P + d];
#pragma unroll
      for (int j = 0; j < 4; ++j) kv[j] = Ks[(tx + 16 * j) * SP_P + d];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) S[i][j] = fmaf(qv[i], kv[j], S[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = tx + 16 * j;
        Ps[(ty + 16 * i) * SP_P + c] = (kt * SP_T + c < a.seq_k) ? S[i][j] : -INFINITY;
      }
    __syncthreads();
    {   // online softmax: 4 threads per row, 16 columns each
      const int r = t >> 2, part = t & 3;
      float* pr = Ps + r * SP_P + part * 16;
      float mx = -INFINITY;
#pragma unroll
      for (int c = 0; c < 16; ++c) mx = fmaxf(mx, pr[c]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_old = m_s[r];
      const float m_new = fmaxf(m_old, mx);
      float sum = 0.f;
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        const float pv = expf(pr[c] - m_new);
        pr[c] = pv;
        sum += pv;
      }
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      __syncwarp();
      if (part == 0) {
        const float al = expf(m_old - m_new);
        al_s[r] = al;
        m_s[r] = m_new;
        l_s[r] = l_s[r] * al + sum;
      }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float al = al_s[ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) O[i][j] *= al;
    }
    for (int c = 0; c < SP_T; ++c) {
      float pv[4], vv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) pv[i] = Ps[(ty + 16 * i) * SP_P + c];
#pragma unroll
      for (int j = 0; j < 4; ++j) vv[j] = Vs[c * SP_P + tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) O[i][j] = fmaf(pv[i], vv[j], O[i][j]);
    }
  }
  __half* op = reinterpret_cast<__half*>(a.out);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = ty + 16 * i;
    const int sq = q0 + r;
    if (sq >= a.seq_q) continue;
    const float inv = 1.0f / l_s[r];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float v = O[i][j] * inv;
      const long long off = ((long long)b * a.seq_q + sq) * a.ldo + a.o_col0 + h * 64 + tx + 16 * j;
      const __half hi = __float2half_rn(v);
      op[off] = hi;
      if (a.lo_off_o) op[off + a.lo_off_o] = __float2half_rn(v - __half2float(hi));
    }
  }
}

}  // namespace udb

extern "C" int udb_attention_f16(const udb_attn_t* a, void* stream) {
  using namespace udb;
  if (a->head_dim != 64) { set_error("udb_attention_f16: head_dim %d unsupported (64 only)", a->head_dim); return 1; }
  if ((a->ldq | a->ldk | a->ldv | a->ldo) % 8) { set_error("udb_attention_f16: leading dims must be multiples of 8"); return 1; }
  // Layout checks, all before the first CUDA call.  seq_k == 0 would leave every row sum at 0 (NaN outputs); the
  // epilogue stores f16 pairs as 32-bit words at out + row*ldo + o_col0 + head*64 + even column.
  if (a->B < 1 || a->heads < 1 || a->seq_q < 1 || a->seq_k < 1) {
    set_error("udb_attention_f16: B=%d heads=%d seq_q=%d seq_k=%d must be >= 1", a->B, a->heads, a->seq_q, a->seq_k); return 1;
  }
  if (!a->q || !a->k || !a->v || !a->out) { set_error("udb_attention_f16: null q / k / v / out"); return 1; }
  if (reinterpret_cast<uintptr_t>(a->out) & 3) { set_error("udb_attention_f16: `out` %p must be 4-byte aligned", a->out); return 1; }
  const int lo_q = a->split ? a->lo_off_q : 0, lo_k = a->split ? a->lo_off_k : 0, lo_v = a->split ? a->lo_off_v : 0;
  const int lo_o = a->split ? a->lo_off_o : 0;
  if (a->o_col0 < 0 || (a->o_col0 & 1)) { set_error("udb_attention_f16: `o_col0`=%d must be even and >= 0", a->o_col0); return 1; }
  if (lo_o < 0 || (lo_o & 1)) { set_error("udb_attention_f16: `lo_off_o`=%d must be even and >= 0", lo_o); return 1; }
  if (lo_q < 0 || lo_k < 0 || lo_v < 0) { set_error("udb_attention_f16: `lo_off_q/k/v` must be >= 0"); return 1; }
  const long long span = (long long)a->heads * 64;
  if (a->ldo < a->o_col0 + span + lo_o) {
    set_error("udb_attention_f16: `ldo`=%d < o_col0 + heads*64 + lo_off_o = %lld", a->ldo, a->o_col0 + span + lo_o); return 1;
  }
  if (a->q_col0 < 0 || a->ldq < a->q_col0 + span + lo_q) {
    set_error("udb_attention_f16: `ldq`=%d < q_col0 + heads*64 = %lld (q_col0 >= 0)", a->ldq, a->q_col0 + span + lo_q); return 1;
  }
  if (a->k_col0 < 0 || a->ldk < a->k_col0 + span + lo_k) {
    set_error("udb_attention_f16: `ldk`=%d < k_col0 + heads*64 = %lld (k_col0 >= 0)", a->ldk, a->k_col0 + span + lo_k); return 1;
  }
  if (a->v_col0 < 0 || a->ldv < a->v_col0 + span + lo_v) {
    set_error("udb_attention_f16: `ldv`=%d < v_col0 + heads*64 = %lld (v_col0 >= 0)", a->ldv, a->v_col0 + span + lo_v); return 1;
  }
  if (a->split) {
    static std::atomic<uint64_t> sp_mask{0};
    if (first_on_device(sp_mask)) {
      cudaError_t e = cudaFuncSetAttribute(attn_split_f32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SP_SMEM);
      if (e != cudaSuccess) { set_error("attention(split): cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return 1; }
    }
    dim3 grid((a->seq_q + SP_T - 1) / SP_T, a->heads, a->B);
    attn_split_f32_kernel<<<grid, 256, SP_SMEM, reinterpret_cast<cudaStream_t>(stream)>>>(*a);
    return check_launch("attn_split_f32_kernel");
  }
  constexpr int HD = 64;
  CUtensorMap tq, tk, tv;
  const uint32_t box_q[3] = {HD, AT_BQ, 1};
  const uint32_t box_kv[3] = {HD, AT_BK, 1};
  {
    const uint64_t dims[3] = {(uint64_t)a->ldq, (uint64_t)a->seq_q, (uint64_t)a->B};
    const uint64_t str[2] = {(uint64_t)a->ldq * 2, (uint64_t)a->seq_q * a->ldq * 2};
    if (make_tmap_f16(&tq, a->q, 3, dims, str, box_q, true)) return 1;
  }
  {
    const uint64_t dims[3] = {(uint64_t)a->ldk, (uint64_t)a->seq_k, (uint64_t)a->B};
    const uint64_t str[2] = {(uint64_t)a->ldk * 2, (uint64_t)a->seq_k * a->ldk * 2};
    if (make_tmap_f16(&tk, a->k, 3, dims, str, box_kv, true)) return 1;
  }
  {
    const uint64_t dims[3] = {(uint64_t)a->ldv, (uint64_t)a->seq_k, (uint64_t)a->B};
    const uint64_t str[2] = {(uint64_t)a->ldv * 2, (uint64_t)a->seq_k * a->ldv * 2};
    if (make_tmap_f16(&tv, a->v, 3, dims, str, box_kv, true)) return 1;
  }
  AttnArgs p{};
  p.out = reinterpret_cast<__half*>(a->out);
  p.seq_q = a->seq_q; p.seq_k = a->seq_k;
  p.n_kv_tiles = (a->seq_k + AT_BK - 1) / AT_BK;
  p.ldo = a->ldo; p.o_col0 = a->o_col0;
  p.q_col0 = a->q_col0; p.k_col0 = a->k_col0; p.v_col0 = a->v_col0;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  dim3 grid((a->seq_q + AT_BQ - 1) / AT_BQ, a->heads, a->B);
  note_work(4.0 * a->B * a->heads * (double)a->seq_q * a->seq_k * HD, 2.0 * a->B * a->heads * HD * (2.0 * a->seq_q + 2.0 * a->seq_k));
  constexpr int smem_bytes = 16384 + 2 * AT_STAGES * (AT_BK * 128) + 256;
  static std::atomic<uint64_t> attr_mask{0};
  if (first_on_device(attr_mask)) {
    cudaError_t ea = cudaFuncSetAttribute(attn_fwd_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
    if (ea != cudaSuccess) { set_error("attention: cudaFuncSetAttribute: %s", cudaGetErrorString(ea)); return 1; }
  }
  cudaError_t e = launch_ex(attn_fwd_kernel<HD>, grid, dim3(AT_THREADS), smem_bytes, reinterpret_cast<cudaStream_t>(stream), 1,
                            tq, tk, tv, p);
  if (e != cudaSuccess) { set_error("attn_fwd_kernel launch: %s", cudaGetErrorString(e)); return 1; }
  return check_launch("attn_fwd_kernel");
}
