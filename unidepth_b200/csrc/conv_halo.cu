// 3x3 convolution with few output channels (Cout = 32 / 64) over a pre-padded NHWC f16 image, as an
// implicit GEMM whose A operand is loaded ONCE per tile: the (16+2) x 16-pixel halo of a 16 x 8-pixel
// output tile is brought into shared memory by one TMA box per 64-channel slab and all nine filter
// taps read it through shifted wgmma descriptors (start address + (dy*16 + dx) pixel rows, 8-pixel row
// groups 2 KB apart).  The generic implicit-GEMM path (gemm.cu, UDB_A_CONV3X3) re-fetches the tile
// for every tap and is L2-bandwidth bound when Cout is small (each 16 KB A tile feeds only 32-64
// output columns); here the per-tile L2 traffic drops from 9 x 16 KB to 36 KB per slab and the
// weights (<= 147 KB) stay resident in shared memory for the whole persistent kernel.
//
// Covers the decoder heads (reference unidepth/models/unidepthv2/decoder.py:200-229, 288-313):
//   to_*_lr  (128 -> 64, reflect)                       -> f16 NHWC out
//   to_*_hr  (64 -> 32, reflect) + LeakyReLU + 1x1 + clip + exp  -> f32 plane
#include "common.h"
#include "ptx.cuh"

namespace udb {

constexpr int HC_TH = 16, HC_TW = 8;          // output tile (128 pixels = two wgmma M = 64 blocks)
constexpr int HC_HW = 16, HC_HH = HC_TH + 2;  // halo box: 16 x 18 pixels (10 of the 16 columns are used)
constexpr int HC_SLAB_BYTES = HC_HW * HC_HH * 128;   // 36864
constexpr int HC_THREADS = 384;

struct HaloArgs {
  int B, H, W;            // output size (input is [B, H+2, W+2, cstride])
  int slabs;              // C / 64
  int coff;               // first input channel
  int tiles_x, tiles_y, num_tiles;
  int a_stages;           // slab buffers in the ring
  const float* bias;      // [COUT]
  int act;                // UDB_ACT_*
  // f16 NHWC output (ldc elements per pixel) or fused head (f32 plane)
  __half* out;
  long long ldc;
  const float* head_w;
  float head_b, head_add;
  float* head_out;
};

// warps 0..7: two consumer warpgroups (warpgroup g: output tile rows [8g, 8g+8) = operand rows [64g, 64g+64), wgmma
// m64nCOUTk16, epilogue straight from the accumulator registers); warps 8..11: producer warpgroup, warp 8 issues the TMA
// loads (weights once, then the halo slabs through the ring).
constexpr int HC_CONSUMER_WARPS = 8;

template <int COUT>
__global__ void __launch_bounds__(HC_THREADS, 1)
conv3x3_halo_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const HaloArgs p) {
  constexpr int kWTile = COUT * 128;                 // one (tap, slab) weight tile
  extern __shared__ __align__(1024) uint8_t smem[];
  const int w_bytes = 9 * p.slabs * kWTile;
  uint8_t* sW = smem;
  uint8_t* sA = smem + ((w_bytes + 1023) & ~1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sA + p.a_stages * HC_SLAB_BYTES);
  uint64_t* w_full = bars;
  uint64_t* a_full = bars + 1;                       // [a_stages] (<= 4)
  uint64_t* a_empty = bars + 5;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023) __trap();
    prefetch_tmap(&tmX);
    prefetch_tmap(&tmW);
    mbar_init(w_full, 1);
    for (int i = 0; i < p.a_stages; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], HC_CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  const int per_img = p.tiles_x * p.tiles_y;
  if (warp >= HC_CONSUMER_WARPS) {
    setmaxnreg_dec<40>();
    if (warp != HC_CONSUMER_WARPS) return;
    // whole warp in the control flow, one elected lane issues (operands stay in uniform registers;
    // a lane-0 branch makes ptxas wrap every TMA in an ELECT + R2UR waterfall loop)
    const bool elected = elect_one();
    // weights: resident for the whole kernel
    if (elected) {
      mbar_arrive_expect_tx(w_full, w_bytes);
      for (int kb = 0; kb < 9 * p.slabs; ++kb) tma_load_2d(sW + kb * kWTile, &tmW, w_full, kb * 64, 0);
    }
    __syncwarp();
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int b = tile / per_img, r = tile % per_img;
      const int y0 = (r / p.tiles_x) * HC_TH, x0 = (r % p.tiles_x) * HC_TW;
      for (int s = 0; s < p.slabs; ++s) {
        mbar_wait(&a_empty[stage], phase ^ 1);
        if (elected) {
          mbar_arrive_expect_tx(&a_full[stage], HC_SLAB_BYTES);
          tma_load_4d(sA + stage * HC_SLAB_BYTES, &tmX, &a_full[stage], p.coff + s * 64, x0, y0, b);
        }
        __syncwarp();
        if (++stage == p.a_stages) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int wg = warp >> 2, wq = warp & 3;
    // this thread's two accumulator rows: tile rows r0 and r0 + 8 (one output row apart, same column)
    const int r0 = 64 * wg + 16 * wq + (lane >> 2);
    const int ty = r0 / HC_TW, tx = r0 % HC_TW;
    const int cq = 2 * (lane & 3);
    float acc[COUT / 2];
#pragma unroll
    for (int i = 0; i < COUT / 2; ++i) acc[i] = 0.f;
    mbar_wait(w_full, 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      int prev = -1;
      for (int s = 0; s < p.slabs; ++s) {
        mbar_wait(&a_full[stage], phase);
        const uint32_t a_base = smem_u32(sA + stage * HC_SLAB_BYTES) + wg * 8 * HC_HW * 128;
        wgmma_fence();
#pragma unroll 1
        for (int tap = 0; tap < 9; ++tap) {
          const int dy = tap / 3, dx = tap % 3;
          // rows of the operand = pixels (y+dy, x+dx): 8-pixel groups, one per tile row, 16 pixel rows apart
          const uint32_t a_addr = a_base + (dy * HC_HW + dx) * 128;
          // descriptor base offset 0 although the start lies dx rows into the 8-row swizzle pattern: the 128B swizzle
          // follows the absolute shared-memory address bits, as TMA wrote them (tests/test_gemm_gpu.py::test_conv3x3_halo
          // passes on the H100 with this form)
          const uint64_t da = gmma_desc_sw128(a_addr, 16, HC_HW * 128);
          const uint64_t dw = gmma_desc_sw128(smem_u32(sW + (tap * p.slabs + s) * kWTile), 16, 1024);
#pragma unroll
          for (int k = 0; k < 4; ++k) WgmmaSS<COUT>::run(acc, da + 2 * k, dw + 2 * k, (s | tap | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&a_empty[prev]);
        prev = stage;
        if (++stage == p.a_stages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(&a_empty[prev]);
      const int b = tile / per_img, r = tile % per_img;
      const int x = (r % p.tiles_x) * HC_TW + tx;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int y = (r / p.tiles_x) * HC_TH + ty + h;
        const bool valid = y < p.H && x < p.W;
        float head_acc = 0.f;
        __half* op = p.out + (((long long)b * p.H + y) * p.W + x) * p.ldc + cq;
#pragma unroll
        for (int j = 0; j < COUT / 8; ++j) {
          const int c = 8 * j + cq;
          float v0 = acc[4 * j + 2 * h] + __ldg(p.bias + c), v1 = acc[4 * j + 2 * h + 1] + __ldg(p.bias + c + 1);
          if (p.act == UDB_ACT_LEAKY) { v0 = leaky(v0); v1 = leaky(v1); }
          if (p.head_out) head_acc = fmaf(v1, __ldg(p.head_w + c + 1), fmaf(v0, __ldg(p.head_w + c), head_acc));
          else if (valid) *reinterpret_cast<uint32_t*>(op + 8 * j) = pack_half2(v0, v1);
        }
        if (p.head_out) {   // the four lanes of a row hold its 32 channels between them
          head_acc += __shfl_xor_sync(0xffffffffu, head_acc, 1);
          head_acc += __shfl_xor_sync(0xffffffffu, head_acc, 2);
          if (valid && (lane & 3) == 0)
            p.head_out[((long long)b * p.H + y) * p.W + x] = expf(fminf(fmaxf(head_acc + p.head_b, -8.0f), 8.0f) + p.head_add);
        }
      }
    }
  }
}

template <int COUT>
static int launch_halo(const CUtensorMap& tx, const CUtensorMap& tw, const HaloArgs& a, size_t smem, cudaStream_t st) {
  static std::atomic<size_t> set_for[64];
  int dev = 0;
  cudaGetDevice(&dev);
  if (smem > set_for[dev & 63].load()) {
    cudaError_t e = cudaFuncSetAttribute(conv3x3_halo_kernel<COUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("conv3x3_halo: cudaFuncSetAttribute(%zu): %s", smem, cudaGetErrorString(e)); return 1; }
    set_for[dev & 63].store(smem);
  }
  const int grid = a.num_tiles < num_sms() ? a.num_tiles : num_sms();
  note_work(2.0 * a.B * (double)a.H * a.W * COUT * 9 * 64 * a.slabs, 0.0);
  cudaError_t e = launch_ex(conv3x3_halo_kernel<COUT>, dim3(grid), dim3(HC_THREADS), smem, st, 1, tx, tw, a);
  if (e != cudaSuccess) { set_error("conv3x3_halo_kernel launch: %s", cudaGetErrorString(e)); return 1; }
  return check_launch("conv3x3_halo_kernel");
}

}  // namespace udb

extern "C" int udb_conv3x3_halo_f16(const udb_conv_halo_t* c, void* stream) {
  using namespace udb;
  if (c->C % 64 || (c->cout != 32 && c->cout != 64)) { set_error("udb_conv3x3_halo_f16: needs C %% 64 == 0 and Cout in {32, 64}"); return 1; }
  const int cs = c->cstride > 0 ? c->cstride : c->C;
  // Layout checks, all before the first CUDA call: channels past cstride would read as TMA zero fill, and the f16 output
  // is stored as 32-bit channel pairs at out + pixel*ldc + even channel.
  if (c->B < 1 || c->H < 1 || c->W < 1) { set_error("udb_conv3x3_halo_f16: B=%d H=%d W=%d must be >= 1", c->B, c->H, c->W); return 1; }
  if (!c->x || !c->w || !c->bias) { set_error("udb_conv3x3_halo_f16: null x / w / bias"); return 1; }
  if (c->coff < 0 || (long long)c->coff + c->C > cs) {
    set_error("udb_conv3x3_halo_f16: `coff`=%d + C=%d exceeds `cstride`=%d", c->coff, c->C, cs); return 1;
  }
  if (c->head_out) {
    if (!c->head_w) { set_error("udb_conv3x3_halo_f16: `head_w` is null while head_out is set"); return 1; }
    if (reinterpret_cast<uintptr_t>(c->head_out) & 3) { set_error("udb_conv3x3_halo_f16: `head_out` must be 4-byte aligned"); return 1; }
  } else {
    const long long ldc = c->ldc > 0 ? c->ldc : c->cout;
    if (!c->out) { set_error("udb_conv3x3_halo_f16: `out` is null (and no head_out)"); return 1; }
    if (reinterpret_cast<uintptr_t>(c->out) & 3) { set_error("udb_conv3x3_halo_f16: `out` %p must be 4-byte aligned", c->out); return 1; }
    if ((ldc & 1) || ldc < c->cout) { set_error("udb_conv3x3_halo_f16: `ldc`=%lld must be even and >= cout=%d", ldc, c->cout); return 1; }
  }
  HaloArgs a{};
  a.B = c->B; a.H = c->H; a.W = c->W;
  a.slabs = c->C / 64; a.coff = c->coff;
  a.tiles_x = (c->W + HC_TW - 1) / HC_TW; a.tiles_y = (c->H + HC_TH - 1) / HC_TH;
  a.num_tiles = c->B * a.tiles_x * a.tiles_y;
  a.bias = c->bias; a.act = c->act;
  a.out = reinterpret_cast<__half*>(c->out); a.ldc = c->ldc > 0 ? c->ldc : c->cout;
  a.head_w = c->head_w; a.head_b = c->head_b; a.head_add = c->head_add; a.head_out = c->head_out;
  if (a.head_out && c->cout != 32) { set_error("udb_conv3x3_halo_f16: fused head needs Cout == 32"); return 1; }
  const size_t w_bytes = (size_t)9 * a.slabs * c->cout * 128;
  const size_t w_al = (w_bytes + 1023) & ~size_t(1023);
  int stages = (int)((232448 - 256 - w_al) / HC_SLAB_BYTES);
  if (stages > 4) stages = 4;
  if (stages < 2) { set_error("udb_conv3x3_halo_f16: weights too large for shared memory"); return 1; }
  a.a_stages = stages;
  const size_t smem = w_al + (size_t)stages * HC_SLAB_BYTES + 256;
  CUtensorMap tx, tw;
  {
    const uint64_t dims[4] = {(uint64_t)cs, (uint64_t)c->W + 2, (uint64_t)c->H + 2, (uint64_t)c->B};
    const uint64_t str[3] = {(uint64_t)cs * 2, (uint64_t)(c->W + 2) * cs * 2, (uint64_t)(c->H + 2) * (c->W + 2) * cs * 2};
    const uint32_t box[4] = {64, (uint32_t)HC_HW, (uint32_t)HC_HH, 1};
    if (make_tmap_f16(&tx, c->x, 4, dims, str, box, true)) return 1;
  }
  {
    const uint64_t dims[2] = {(uint64_t)9 * c->C, (uint64_t)c->cout};
    const uint64_t str[1] = {(uint64_t)9 * c->C * 2};
    const uint32_t box[2] = {64, (uint32_t)c->cout};
    if (make_tmap_f16(&tw, c->w, 2, dims, str, box, true)) return 1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return c->cout == 32 ? launch_halo<32>(tx, tw, a, smem, st) : launch_halo<64>(tx, tw, a, smem, st);
}
