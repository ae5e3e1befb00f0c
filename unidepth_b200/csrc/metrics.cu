// Evaluation metrics (include/udb.h udb_nearest_neighbor, udb_depth_metrics, udb_point_metrics): the reference's
// eval_depth / eval_3d (unidepth/utils/evaluation_depth.py:37-170) and the K = 1, L2 nearest-neighbour search of its
// ChamferDistance (chamfer_distance.py:59-158 -> ops/knn knn_cpu.cpp:13-69), on the GPU.
//
// Exactness.  Every distance, ratio and rescaled value is formed with __f*_rn ops in the reference's fp32 op order, so
// nvcc cannot contract to FMA.  The squared distance is ((dx*dx) + dy*dy) + dz*dz with dx = x - y, each op rounded on its
// own, exactly as the CPU KNN forms it.  FMA would take about 30 % fewer instructions in the NN loop, but then `dist`
// would no longer be bit-identical to the reference and F1's threshold counts (dist < t) could change; exact counts win.
// Counts are integers; every floating-point sum is an f64 per-CTA partial reduced in a fixed order (no floating-point
// atomics), so two runs give bit-identical results.
#include <math.h>

#include "common.h"

namespace udb {

namespace {

__device__ __forceinline__ float sq_dist(float ax, float ay, float az, float bx, float by, float bz) {
  const float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by), dz = __fsub_rn(az, bz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// (dist, index) as one 64-bit key: dist >= 0, so its bit pattern orders like the value, and the low word breaks ties
// towards the lower index -- the CPU implementation's strict `<` over ascending indices.
__device__ __forceinline__ unsigned long long nn_key(float d, int i) {
  return (static_cast<unsigned long long>(__float_as_uint(d)) << 32) | static_cast<unsigned>(i);
}

__device__ __forceinline__ void shfl_min(float& d, int& i, int mask) {
  const float od = __shfl_xor_sync(0xffffffffu, d, mask);
  const int oi = __shfl_xor_sync(0xffffffffu, i, mask);
  if (od < d || (od == d && oi < i)) { d = od; i = oi; }
}

__device__ __forceinline__ int64_t clamp_len(const int64_t* lengths, int n, int P) {
  if (!lengths) return P;
  const int64_t l = lengths[n];
  return l < 0 ? 0 : (l > P ? P : l);
}

// ------------------------------------------------------------------------------------------------- nearest neighbour
// CTA: 128 queries (x) x a range of 128-point reference (y) tiles of one cloud.  256 threads; warp w, lane l owns rows
// (l & 15) * 8 .. +7 and columns (2w + (l >> 4)) * 8 .. +7 of each 128 x 128 tile, so the 16 lanes that share a column
// group sit in one warp and the column (y -> x) minima reduce with four shuffles.  Row minima stay in registers across
// the tiles; each CTA's partial row / column minima merge into the packed 64-bit keys with atomicMin.  References
// stream through a double-buffered shared tile: the next tile is loaded into registers before the current one is
// computed and stored after it, so one barrier per tile suffices.  Points past a cloud's length read as +inf: their
// distances are inf or NaN and never win a strict `<`.
constexpr int NN_Q = 128, NN_R = 128, NN_THREADS = 256;

template <bool BOTH>
__global__ void __launch_bounds__(NN_THREADS, 2)
nn_kernel(const float* __restrict__ x, const float* __restrict__ y, const int64_t* __restrict__ len1,
          const int64_t* __restrict__ len2, int P1, int P2, int tiles_per_split,
          unsigned long long* __restrict__ key_x, unsigned long long* __restrict__ key_y) {
  const int n = blockIdx.z;
  const int L1 = static_cast<int>(clamp_len(len1, n, P1)), L2 = static_cast<int>(clamp_len(len2, n, P2));
  const int q0 = blockIdx.x * NN_Q;
  const int t0 = blockIdx.y * tiles_per_split;
  const int t1 = min(t0 + tiles_per_split, (L2 + NN_R - 1) / NN_R);
  if (q0 >= L1 || t0 >= t1) return;

  __shared__ __align__(16) float ys[2][NN_R * 3];
  const int tid = threadIdx.x, lane = tid & 31, rg = lane & 15, cg = (tid >> 5) * 2 + (lane >> 4);
  const float inf = __int_as_float(0x7f800000);

  float qx[8], qy[8], qz[8];
  const float* xn = x + static_cast<size_t>(n) * P1 * 3;
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int row = q0 + rg * 8 + r;
    const bool ok = row < L1;
    qx[r] = ok ? xn[static_cast<size_t>(row) * 3 + 0] : inf;
    qy[r] = ok ? xn[static_cast<size_t>(row) * 3 + 1] : inf;
    qz[r] = ok ? xn[static_cast<size_t>(row) * 3 + 2] : inf;
  }
  float bd[8];
  int bi[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) { bd[r] = inf; bi[r] = t0 * NN_R; }

  const float* yn = y + static_cast<size_t>(n) * P2 * 3;
  const int lim = 3 * L2;   // floats of the valid points
  auto fetch = [&](int t, int e) {
    const int f = t * (NN_R * 3) + e;
    return f < lim ? yn[f] : inf;
  };
  ys[0][tid] = fetch(t0, tid);
  if (tid < NN_R * 3 - NN_THREADS) ys[0][NN_THREADS + tid] = fetch(t0, NN_THREADS + tid);
  __syncthreads();

  for (int t = t0; t < t1; ++t) {
    const int buf = (t - t0) & 1;
    float n0 = 0.f, n1 = 0.f;
    if (t + 1 < t1) {
      n0 = fetch(t + 1, tid);
      if (tid < NN_R * 3 - NN_THREADS) n1 = fetch(t + 1, NN_THREADS + tid);
    }
    float c[24];
    const float4* s4 = reinterpret_cast<const float4*>(&ys[buf][cg * 24]);
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const float4 v = s4[k];
      c[4 * k] = v.x; c[4 * k + 1] = v.y; c[4 * k + 2] = v.z; c[4 * k + 3] = v.w;
    }
    const int jb = t * NN_R + cg * 8;
    float cd[8];
    int ci[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { cd[k] = inf; ci[k] = 0; }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float d = sq_dist(qx[r], qy[r], qz[r], c[3 * k], c[3 * k + 1], c[3 * k + 2]);
        if (d < bd[r]) { bd[r] = d; bi[r] = jb + k; }
        if (BOTH && d < cd[k]) { cd[k] = d; ci[k] = r; }
      }
    }
    if (BOTH) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        float d = cd[k];
        int i = q0 + rg * 8 + ci[k];
        shfl_min(d, i, 1); shfl_min(d, i, 2); shfl_min(d, i, 4); shfl_min(d, i, 8);
        const int col = jb + k;
        if (rg == 0 && col < L2) atomicMin(key_y + static_cast<size_t>(n) * P2 + col, nn_key(d, i));
      }
    }
    if (t + 1 < t1) {
      ys[buf ^ 1][tid] = n0;
      if (tid < NN_R * 3 - NN_THREADS) ys[buf ^ 1][NN_THREADS + tid] = n1;
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    float d = bd[r];
    int i = bi[r];
    shfl_min(d, i, 16);
    const int row = q0 + rg * 8 + r;
    if (lane < 16 && row < L1) atomicMin(key_x + static_cast<size_t>(n) * P1 + row, nn_key(d, i));
  }
}

// Unpack the keys in place: idx = low word, dist = high word; rows past their cloud's length, or whose other cloud is
// empty, get dist = 0 and idx = 0 (the reference's zero-initialised outputs).
__global__ void __launch_bounds__(256) nn_finish_kernel(int N, int P1, int P2, const int64_t* __restrict__ len1,
                                                        const int64_t* __restrict__ len2, float* __restrict__ dist_x,
                                                        int64_t* __restrict__ idx_x, float* __restrict__ dist_y,
                                                        int64_t* __restrict__ idx_y) {
  const long long nx = static_cast<long long>(N) * P1, total = nx + (dist_y ? static_cast<long long>(N) * P2 : 0);
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const bool is_x = e < nx;
    const long long k = is_x ? e : e - nx;
    const int P = is_x ? P1 : P2;
    const int n = static_cast<int>(k / P), row = static_cast<int>(k % P);
    const int64_t Lown = is_x ? clamp_len(len1, n, P1) : clamp_len(len2, n, P2);
    const int64_t Loth = is_x ? clamp_len(len2, n, P2) : clamp_len(len1, n, P1);
    float* dist = is_x ? dist_x : dist_y;
    int64_t* idx = is_x ? idx_x : idx_y;
    if (row < Lown && Loth > 0) {
      const unsigned long long v = static_cast<unsigned long long>(idx[k]);
      dist[k] = __uint_as_float(static_cast<unsigned>(v >> 32));
      idx[k] = static_cast<int64_t>(v & 0xffffffffull);
    } else {
      dist[k] = 0.f;
      idx[k] = 0;
    }
  }
}

// --------------------------------------------------------------------------------------------------- metric reductions
constexpr int MET_THREADS = 256;

// Sum K doubles over the CTA in a fixed order (shuffle tree, then warps 0..7); thread 0 gets the totals.
template <int K>
__device__ __forceinline__ void block_sum(double (&v)[K], double* red /* [8][K] shared */) {
#pragma unroll
  for (int k = 0; k < K; ++k)
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], m);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int k = 0; k < K; ++k) red[w * K + k] = v[k];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double s = red[k];
      for (int ww = 1; ww < MET_THREADS / 32; ++ww) s += red[ww * K + k];
      v[k] = s;
    }
}

// number of ascending thresholds t[0..T) with t <= v, i.e. the first i with v < t[i]; NaN -> T (below none)
__device__ __forceinline__ int first_above(const float* t, int T, float v) {
  int lo = 0, hi = T;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (t[mid] > v) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// torch.maximum: NaN propagates
__device__ __forceinline__ float tmax(float a, float b) { return a != a ? a : (b != b ? b : fmaxf(a, b)); }

__device__ __forceinline__ float ratio_of(float g, float p) { return tmax(__fdiv_rn(g, p), __fdiv_rn(p, g)); }

// Pass 1: the plain and si metrics, the ssi normal-equation sums and the d_auc histogram.
// Pass 2: the ssi metrics, with the per-image (scale, shift) the reduction solved after pass 1.
template <int PASS>
__global__ void __launch_bounds__(MET_THREADS) depth_metrics_kernel(udb_depth_metrics_t p, int nblk) {
  constexpr int K = PASS == 1 ? 19 : 3;
  __shared__ float thr[UDB_DM_AUC_BINS];
  __shared__ unsigned hist[UDB_DM_AUC_BINS];
  __shared__ double red[(MET_THREADS / 32) * K];
  const int b = blockIdx.y, tid = threadIdx.x;
  if (PASS == 1 && tid < UDB_DM_AUC_BINS) { thr[tid] = p.auc_thresholds[tid]; hist[tid] = 0u; }
  __syncthreads();
  const float* gt = p.gt + static_cast<size_t>(b) * p.HW;
  const float* pr = p.pred + static_cast<size_t>(b) * p.HW;
  const uint8_t* mk = p.mask + static_cast<size_t>(b) * p.HW;
  float mg = 0.f, mp = 1.f, sc = 0.f, sh = 0.f;
  if (PASS == 1) { mg = p.medians[2 * b]; mp = p.medians[2 * b + 1]; }
  else { sc = p.ssi[2 * b]; sh = p.ssi[2 * b + 1]; }
  double v[K];
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = 0.0;
  unsigned cnt[PASS == 1 ? 7 : 2] = {};
  for (long long i = static_cast<long long>(blockIdx.x) * MET_THREADS + tid; i < p.HW;
       i += static_cast<long long>(nblk) * MET_THREADS) {
    const float g = gt[i], q = pr[i];
    if (!mk[i] || (p.use_max_depth && !(g <= p.max_depth))) continue;
    if (PASS == 1) {
      const float ratio = ratio_of(g, q);
      cnt[0] += 1u;
      cnt[1] += ratio < p.thr_d1;
      cnt[2] += ratio < p.thr_d2;
      cnt[3] += ratio < p.thr_d3;
      cnt[4] += ratio < p.thr_tau;
      const float e = __fsub_rn(g, q), e2 = __fmul_rn(e, e);
      const float lgg = logf(g), lgp = logf(q);
      const float el = __fsub_rn(lgg, lgp);
      const float lg = __fsub_rn(lgp, lgg);
      v[0] += e2;                                           // rmse
      v[1] += __fmul_rn(el, el);                            // rmselog
      v[2] += __fdiv_rn(fabsf(e), g);                       // arel
      v[3] += __fdiv_rn(e2, g);                             // sqrel
      v[4] += fabsf(__fsub_rn(log10f(q), log10f(g)));       // log10
      v[5] += lg;                                           // silog: sum and sum of squares
      v[6] += static_cast<double>(lg) * lg;
      const float qs = __fdiv_rn(__fmul_rn(q, mg), mp);     // si: pred * median(gt) / median(pred)
      const float rs = ratio_of(g, qs);
      cnt[5] += rs < p.thr_d1;
      cnt[6] += rs < p.thr_tau;
      v[7] += __fdiv_rn(fabsf(__fsub_rn(g, qs)), g);
      v[8] += static_cast<double>(q) * q;                   // ssi normal equations
      v[9] += q;
      v[10] += static_cast<double>(q) * g;
      v[11] += g;
      const int k = first_above(thr, UDB_DM_AUC_BINS, ratio);
      if (k < UDB_DM_AUC_BINS) atomicAdd(&hist[k], 1u);
    } else {
      const float qs = __fadd_rn(__fmul_rn(q, sc), sh);    // ssi: pred * scale + shift
      const float rs = ratio_of(g, qs);
      cnt[0] += rs < p.thr_d1;
      cnt[1] += rs < p.thr_tau;
      v[0] += __fdiv_rn(fabsf(__fsub_rn(g, qs)), g);
    }
  }
  if (PASS == 1) {
#pragma unroll
    for (int k = 0; k < 7; ++k) v[12 + k] = cnt[k];
  } else {
    v[1] = cnt[0];
    v[2] = cnt[1];
  }
  block_sum<K>(v, red);
  double* part = p.partials + (static_cast<size_t>(b) * nblk + blockIdx.x) * UDB_DM_NACC;
  if (tid == 0) {
    if (PASS == 1) {
      part[UDB_DM_N] = v[12];
      part[UDB_DM_D1] = v[13]; part[UDB_DM_D2] = v[14]; part[UDB_DM_D3] = v[15]; part[UDB_DM_TAU] = v[16];
      part[UDB_DM_SQ] = v[0]; part[UDB_DM_SQLOG] = v[1]; part[UDB_DM_AREL] = v[2]; part[UDB_DM_SQREL] = v[3];
      part[UDB_DM_LOG10] = v[4]; part[UDB_DM_LG] = v[5]; part[UDB_DM_LG2] = v[6];
      part[UDB_DM_D1_SI] = v[17]; part[UDB_DM_TAU_SI] = v[18]; part[UDB_DM_AREL_SI] = v[7];
      part[UDB_DM_PP] = v[8]; part[UDB_DM_P] = v[9]; part[UDB_DM_PG] = v[10]; part[UDB_DM_G] = v[11];
    } else {
      part[UDB_DM_AREL_SSI] = v[0]; part[UDB_DM_D1_SSI] = v[1]; part[UDB_DM_TAU_SSI] = v[2];
    }
  }
  if (PASS == 1 && tid < UDB_DM_AUC_BINS) part[UDB_DM_AUC + tid] = hist[tid];   // hist complete: block_sum synced
}

// out[b, k0..k1) = sum over the nblk partials in block order.  With ssi: then solve the reference's ssi normal
// equations (evaluation_depth.py:47-56) in f64 -- [[pp, p], [p, n]] + f32(1e-9) I -- and store (scale, shift) as f32.
__global__ void __launch_bounds__(128) metric_reduce_kernel(const double* __restrict__ partials, int nblk, int nacc,
                                                            int k0, int k1, double* __restrict__ out,
                                                            float* __restrict__ ssi) {
  const int b = blockIdx.x;
  for (int k = k0 + threadIdx.x; k < k1; k += blockDim.x) {
    double s = 0.0;
    for (int j = 0; j < nblk; ++j) s += partials[(static_cast<size_t>(b) * nblk + j) * nacc + k];
    out[static_cast<size_t>(b) * nacc + k] = s;
  }
  if (!ssi) return;
  __syncthreads();
  if (threadIdx.x == 0) {
    const double* o = out + static_cast<size_t>(b) * nacc;
    const double eps = static_cast<double>(1e-9f);
    const double a00 = o[UDB_DM_PP] + eps, a01 = o[UDB_DM_P], a11 = o[UDB_DM_N] + eps;
    const double r0 = o[UDB_DM_PG], r1 = o[UDB_DM_G];
    const double det = a00 * a11 - a01 * a01;
    ssi[2 * b] = static_cast<float>((a11 * r0 - a01 * r1) / det);
    ssi[2 * b + 1] = static_cast<float>((a00 * r1 - a01 * r0) / det);
  }
}

// Point metrics of eval_3d (evaluation_depth.py:112-122): per valid point the norm |gt - pred|, the chamfer term
// (sqrt(dist_x) + sqrt(dist_y)) / 2, and the F1 threshold histograms of dist_x (precision) and dist_y (recall).
__global__ void __launch_bounds__(MET_THREADS) point_metrics_kernel(udb_point_metrics_t p, int nblk) {
  extern __shared__ unsigned char smem_raw[];
  const int T = p.n_thresholds, nacc = 2 + 2 * T;
  float* thr = reinterpret_cast<float*>(smem_raw);
  unsigned* hx = reinterpret_cast<unsigned*>(thr + T);
  unsigned* hy = hx + T;
  __shared__ double red[(MET_THREADS / 32) * 2];
  const int n = blockIdx.y, tid = threadIdx.x;
  for (int k = tid; k < T; k += MET_THREADS) { thr[k] = p.thresholds[k]; hx[k] = 0u; hy[k] = 0u; }
  __syncthreads();
  const int L = static_cast<int>(clamp_len(p.lengths, n, p.P));
  const float* g = p.gt + static_cast<size_t>(n) * p.P * 3;
  const float* q = p.pred + static_cast<size_t>(n) * p.P * 3;
  const float* dx = p.dist_x + static_cast<size_t>(n) * p.P;
  const float* dy = p.dist_y + static_cast<size_t>(n) * p.P;
  double v[2] = {0.0, 0.0};
  for (int i = blockIdx.x * MET_THREADS + tid; i < L; i += nblk * MET_THREADS) {
    const float* a = g + static_cast<size_t>(i) * 3;
    const float* c = q + static_cast<size_t>(i) * 3;
    v[0] += sqrtf(sq_dist(a[0], a[1], a[2], c[0], c[1], c[2]));
    const float ex = dx[i], ey = dy[i];
    v[1] += __fdiv_rn(__fadd_rn(sqrtf(ex), sqrtf(ey)), 2.f);
    const int kx = first_above(thr, T, ex), ky = first_above(thr, T, ey);
    if (kx < T) atomicAdd(&hx[kx], 1u);
    if (ky < T) atomicAdd(&hy[ky], 1u);
  }
  block_sum<2>(v, red);
  double* part = p.partials + (static_cast<size_t>(n) * nblk + blockIdx.x) * nacc;
  if (tid == 0) { part[0] = v[0]; part[1] = v[1]; }
  for (int k = tid; k < T; k += MET_THREADS) { part[2 + k] = hx[k]; part[2 + T + k] = hy[k]; }
}

int metric_blocks(long long items) {
  const long long b = (items + 8 * MET_THREADS - 1) / (8 * MET_THREADS);
  return static_cast<int>(b < 1 ? 1 : (b > UDB_METRIC_MAX_BLOCKS ? UDB_METRIC_MAX_BLOCKS : b));
}

bool misaligned(const void* ptr, uintptr_t a) { return reinterpret_cast<uintptr_t>(ptr) & (a - 1); }

}  // namespace

}  // namespace udb

using namespace udb;

#define REQUIRE(cond, ...)         \
  do {                             \
    if (!(cond)) {                 \
      set_error(__VA_ARGS__);      \
      return 1;                    \
    }                              \
  } while (0)

extern "C" int udb_nearest_neighbor(const udb_nn_t* p, void* stream) {
  REQUIRE(p, "udb_nearest_neighbor: `p` is null");
  REQUIRE(p->N >= 1 && p->N <= 65535, "udb_nearest_neighbor: N=%d must be in [1, 65535]", p->N);
  REQUIRE(p->P1 >= 1 && p->P2 >= 1, "udb_nearest_neighbor: P1=%d, P2=%d must be >= 1", p->P1, p->P2);
  REQUIRE(p->x && !misaligned(p->x, 4), "udb_nearest_neighbor: `x` must be non-null and 4-byte aligned");
  REQUIRE(p->y && !misaligned(p->y, 4), "udb_nearest_neighbor: `y` must be non-null and 4-byte aligned");
  REQUIRE(!misaligned(p->lengths1, 8), "udb_nearest_neighbor: `lengths1` must be 8-byte aligned");
  REQUIRE(!misaligned(p->lengths2, 8), "udb_nearest_neighbor: `lengths2` must be 8-byte aligned");
  REQUIRE(p->dist_x && !misaligned(p->dist_x, 4), "udb_nearest_neighbor: `dist_x` must be non-null and 4-byte aligned");
  REQUIRE(p->idx_x && !misaligned(p->idx_x, 8), "udb_nearest_neighbor: `idx_x` must be non-null and 8-byte aligned");
  REQUIRE(!p->dist_y == !p->idx_y, "udb_nearest_neighbor: `dist_y` and `idx_y` must both be set or both be null");
  REQUIRE(!misaligned(p->dist_y, 4), "udb_nearest_neighbor: `dist_y` must be 4-byte aligned");
  REQUIRE(!misaligned(p->idx_y, 8), "udb_nearest_neighbor: `idx_y` must be 8-byte aligned");
  const bool both = p->dist_y != nullptr;
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  const int qb = (p->P1 + NN_Q - 1) / NN_Q, rt = (p->P2 + NN_R - 1) / NN_R;
  // split the reference tiles until the grid holds about four CTAs per SM (two are resident at a time)
  long long want = (4ll * num_sms() + static_cast<long long>(qb) * p->N - 1) / (static_cast<long long>(qb) * p->N);
  if (want < 1) want = 1;
  if (want > rt) want = rt;
  const int tps = static_cast<int>((rt + want - 1) / want);
  const int splits = (rt + tps - 1) / tps;
  auto* kx = reinterpret_cast<unsigned long long*>(p->idx_x);
  auto* ky = reinterpret_cast<unsigned long long*>(p->idx_y);
  if (cudaMemsetAsync(kx, 0xff, sizeof(int64_t) * p->N * static_cast<size_t>(p->P1), st) != cudaSuccess ||
      (both && cudaMemsetAsync(ky, 0xff, sizeof(int64_t) * p->N * static_cast<size_t>(p->P2), st) != cudaSuccess)) {
    set_error("udb_nearest_neighbor: cudaMemsetAsync failed: %s", cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  const dim3 grid(qb, splits, p->N);
  note_work(8.0 * p->N * static_cast<double>(p->P1) * p->P2, 12.0 * p->N * (static_cast<double>(p->P1) + p->P2));
  if (both) nn_kernel<true><<<grid, NN_THREADS, 0, st>>>(p->x, p->y, p->lengths1, p->lengths2, p->P1, p->P2, tps, kx, ky);
  else nn_kernel<false><<<grid, NN_THREADS, 0, st>>>(p->x, p->y, p->lengths1, p->lengths2, p->P1, p->P2, tps, kx, nullptr);
  if (int rc = check_launch("nn_kernel")) return rc;
  const long long total = static_cast<long long>(p->N) * (p->P1 + (both ? p->P2 : 0));
  long long fb = (total + 255) / 256;
  if (fb > 8ll * num_sms()) fb = 8ll * num_sms();
  note_work(0.0, 20.0 * total);
  nn_finish_kernel<<<static_cast<unsigned>(fb), 256, 0, st>>>(p->N, p->P1, p->P2, p->lengths1, p->lengths2, p->dist_x,
                                                               p->idx_x, p->dist_y, p->idx_y);
  return check_launch("nn_finish_kernel");
}

extern "C" int udb_depth_metrics(const udb_depth_metrics_t* p, void* stream) {
  REQUIRE(p, "udb_depth_metrics: `p` is null");
  REQUIRE(p->B >= 1 && p->B <= 65535, "udb_depth_metrics: B=%d must be in [1, 65535]", p->B);
  REQUIRE(p->HW >= 1, "udb_depth_metrics: HW=%lld must be >= 1", static_cast<long long>(p->HW));
  REQUIRE(p->gt && !misaligned(p->gt, 4), "udb_depth_metrics: `gt` must be non-null and 4-byte aligned");
  REQUIRE(p->pred && !misaligned(p->pred, 4), "udb_depth_metrics: `pred` must be non-null and 4-byte aligned");
  REQUIRE(p->mask, "udb_depth_metrics: `mask` is null");
  REQUIRE(p->auc_thresholds && !misaligned(p->auc_thresholds, 4),
          "udb_depth_metrics: `auc_thresholds` must be non-null and 4-byte aligned");
  REQUIRE(p->medians && !misaligned(p->medians, 4), "udb_depth_metrics: `medians` must be non-null and 4-byte aligned");
  REQUIRE(p->partials && !misaligned(p->partials, 8), "udb_depth_metrics: `partials` must be non-null and 8-byte aligned");
  REQUIRE(p->out && !misaligned(p->out, 8), "udb_depth_metrics: `out` must be non-null and 8-byte aligned");
  REQUIRE(p->ssi && !misaligned(p->ssi, 4), "udb_depth_metrics: `ssi` must be non-null and 4-byte aligned");
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  const int nblk = metric_blocks(p->HW);
  const dim3 grid(nblk, p->B);
  note_work(0.0, 9.0 * p->B * static_cast<double>(p->HW));
  depth_metrics_kernel<1><<<grid, MET_THREADS, 0, st>>>(*p, nblk);
  if (int rc = check_launch("depth_metrics_kernel<1>")) return rc;
  note_work(0.0, 8.0 * p->B * nblk * UDB_DM_NACC);
  metric_reduce_kernel<<<p->B, 128, 0, st>>>(p->partials, nblk, UDB_DM_NACC, 0, UDB_DM_AREL_SSI, p->out, p->ssi);
  if (int rc = check_launch("metric_reduce_kernel")) return rc;
  note_work(0.0, 9.0 * p->B * static_cast<double>(p->HW));
  depth_metrics_kernel<2><<<grid, MET_THREADS, 0, st>>>(*p, nblk);
  if (int rc = check_launch("depth_metrics_kernel<2>")) return rc;
  note_work(0.0, 8.0 * p->B * nblk * 3);
  metric_reduce_kernel<<<p->B, 128, 0, st>>>(p->partials, nblk, UDB_DM_NACC, UDB_DM_AREL_SSI, UDB_DM_NACC, p->out,
                                              nullptr);
  return check_launch("metric_reduce_kernel");
}

extern "C" int udb_point_metrics(const udb_point_metrics_t* p, void* stream) {
  REQUIRE(p, "udb_point_metrics: `p` is null");
  REQUIRE(p->N >= 1 && p->N <= 65535, "udb_point_metrics: N=%d must be in [1, 65535]", p->N);
  REQUIRE(p->P >= 1, "udb_point_metrics: P=%d must be >= 1", p->P);
  REQUIRE(p->n_thresholds >= 1 && p->n_thresholds <= UDB_PM_MAX_THRESHOLDS,
          "udb_point_metrics: n_thresholds=%d must be in [1, %d]", p->n_thresholds, UDB_PM_MAX_THRESHOLDS);
  REQUIRE(p->gt && !misaligned(p->gt, 4), "udb_point_metrics: `gt` must be non-null and 4-byte aligned");
  REQUIRE(p->pred && !misaligned(p->pred, 4), "udb_point_metrics: `pred` must be non-null and 4-byte aligned");
  REQUIRE(!misaligned(p->lengths, 8), "udb_point_metrics: `lengths` must be 8-byte aligned");
  REQUIRE(p->dist_x && !misaligned(p->dist_x, 4), "udb_point_metrics: `dist_x` must be non-null and 4-byte aligned");
  REQUIRE(p->dist_y && !misaligned(p->dist_y, 4), "udb_point_metrics: `dist_y` must be non-null and 4-byte aligned");
  REQUIRE(p->thresholds && !misaligned(p->thresholds, 4),
          "udb_point_metrics: `thresholds` must be non-null and 4-byte aligned");
  REQUIRE(p->partials && !misaligned(p->partials, 8), "udb_point_metrics: `partials` must be non-null and 8-byte aligned");
  REQUIRE(p->out && !misaligned(p->out, 8), "udb_point_metrics: `out` must be non-null and 8-byte aligned");
  const auto st = reinterpret_cast<cudaStream_t>(stream);
  const int nblk = metric_blocks(p->P), nacc = 2 + 2 * p->n_thresholds;
  note_work(0.0, 32.0 * p->N * static_cast<double>(p->P));
  point_metrics_kernel<<<dim3(nblk, p->N), MET_THREADS, 12 * p->n_thresholds, st>>>(*p, nblk);
  if (int rc = check_launch("point_metrics_kernel")) return rc;
  note_work(0.0, 8.0 * p->N * nblk * nacc);
  metric_reduce_kernel<<<p->N, 128, 0, st>>>(p->partials, nblk, nacc, 0, nacc, p->out, nullptr);
  return check_launch("metric_reduce_kernel");
}
