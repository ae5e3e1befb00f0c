/* udb.h -- C ABI of libudb.so: the sm_90a kernels behind unidepth_b200's UniDepthV2.infer().
 *
 * The reference (lpiccinelli-eth/UniDepth) has no FFI on its inference path: every op below
 * replaces a PyTorch library call made by the reference's Python (file:line cited per entry,
 * relative to the reference repo root).  The Python host (unidepth_b200/) binds these with ctypes;
 * INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; the caller (PyTorch's
 *     caching allocator) owns all memory, the library never allocates, frees, copies to the host
 *     or synchronises the device;
 *   - every launch goes to the `stream` argument (a cudaStream_t passed as void*), so calls are
 *     CUDA-graph capturable;
 *   - return value 0 = OK; non-zero = error, message via udb_last_error() (thread-local);
 *   - "f16" tensors are IEEE half, "f32" are float; activations that feed tensor-core GEMMs are
 *     f16, residual streams / LayerNorm statistics / softmax / epilogue math are f32.
 */
#ifndef UDB_H_
#define UDB_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UDB_VERSION 1

int udb_version(void);

/* Per-launch profile: between begin and end every kernel this library enqueues on `stream` is followed by a CUDA event;
 * end synchronises and returns, per launch in order, the kernel's name, the time since the previous event (its duration
 * when the stream stays busy) and the algorithmic flops / bytes its launcher declared.  Returns the number of launches
 * (which may exceed cap; only the first cap entries are written), -1 on error.  Not for use under stream capture. */
typedef struct udb_profile_entry_t {
  char name[48];
  float ms;
  double flops;
  double bytes;
} udb_profile_entry_t;
int udb_profile_begin(void* stream);
int udb_profile_end(udb_profile_entry_t* out, int32_t cap);
const char* udb_last_error(void);
/* Number of kernels launched by this library on the calling process since load (bench evidence). */
int64_t udb_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * Tensor-core GEMM  D = epilogue(A . W^T)  (wgmma f16, fp32 accumulation in registers, TMA
 * operand loads, persistent warp-specialised kernel).
 * Replaces nn.Linear / nn.Conv2d(k=s=14) / nn.Conv2d(1x1, 3x3) / nn.ConvTranspose2d(k=s) calls:
 *   unidepth/models/backbones/metadinov2/{patch_embed.py:82, attention.py:55-61, mlp.py:36-40},
 *   unidepth/layers/{attention.py:119-138, mlp.py:29-34, upsample.py:171-180,218-222},
 *   unidepth/models/unidepthv2/decoder.py:43,264,279,288-303.
 * ------------------------------------------------------------------------------------------- */
enum { UDB_A_MATRIX = 0, UDB_A_CONV3X3 = 1 };
enum { UDB_ACT_NONE = 0, UDB_ACT_GELU = 1, UDB_ACT_LEAKY = 2 };
enum { UDB_STORE_ROWS = 0, UDB_STORE_CONVT = 1, UDB_STORE_CONVTILE = 2, UDB_STORE_HEAD = 3 };

typedef struct udb_gemm_t {
  /* operands: A f16 [M,K] row-major (lda elements) or NHWC f16 image for UDB_A_CONV3X3;
   * W f16 [N,K] row-major (ldw elements).  K-extent is zero-extended to a multiple of 64. */
  const void* a;
  const void* w;
  int32_t M, N, K;  /* all >= 1; N % 32 == 0 */
  int32_t lda, ldw;
  int32_t a_mode;
  /* UDB_A_CONV3X3: input [B, H(+2), W(+2), C] f16 NHWC; K = 9*C ordered (dy,dx,c); the output
   * pixel (y,x) reads input (y+dy+off, x+dx+off), off = -1 for zero padding (out-of-range taps
   * read 0 through TMA out-of-bounds fill) or 0 when the input was padded by the caller
   * (reflect padding, in_H = H+2, in_W = W+2).  Checked: conv_off is 0 or -1, and conv_inH / conv_inW are H+2 / W+2
   * when it is 0, H / W when it is -1. */
  int32_t conv_B, conv_H, conv_W, conv_C, conv_inH, conv_inW, conv_off, conv_TH, conv_TW;
  /* the input may be a channel slice [conv_coff, conv_coff + conv_C) of a wider NHWC buffer with
   * conv_cstride channels per pixel (0 = conv_C) */
  int32_t conv_cstride, conv_coff;
  /* epilogue: v = acc + bias[n]; v = act(v); v *= gamma[n]; v += resid[...]; out = v;
   * out2 = f16(v) or f16(leaky(v)) (optional second f16 copy, e.g. the next conv's input)
   * Alignment (the epilogue moves 4 columns per vector access): bias / gamma / ln_c1 / head_w 16-byte aligned; f32
   * out / resid 16-byte, f16 out / out2 / resid 8-byte aligned (HEAD: f32 out, 4-byte); ldc and ldr multiples of 4 (ROWS
   * and CONVTILE stores).  The epilogue keeps each row's element offset in 32 bits: the last row written through out /
   * out2 / resid must start below 2^32 elements. */
  const float* bias;
  const float* gamma;
  const void* resid;
  int32_t resid_f32; /* 1: f32, 0: f16 */
  void* out;
  int32_t out_f32;
  void* out2;
  int32_t out2_leaky; /* 1: out2 = f16(leaky(v)); 0: out2 = f16(v) */
  int32_t act;
  int32_t store_mode;
  int64_t ldc; /* elements between consecutive output rows / pixels; ROWS / CONVTILE: >= N + out_split */
  /* UDB_STORE_ROWS: out_row = (m / rows_per_group)*group_stride + m % rows_per_group + row_offset
   * (rows_per_group <= 0: identity).  resid row = resid_mod > 0 ? m % resid_mod + resid_row_offset
   * : out_row, with leading dimension ldr.  group_stride, row_offset and resid_row_offset >= 0. */
  int32_t rows_per_group, group_stride, row_offset;
  int32_t resid_mod, resid_row_offset;
  int64_t ldr; /* 0 = ldc; with a residual (ROWS / CONVTILE): >= N */
  /* UDB_STORE_CONVT: row m = (b, y, x) of a [B,h,w] grid; column n = (dy*k+dx)*Cout + co;
   * writes NHWC pixel (b, y*k+dy+pad, x*k+dx+pad, co) of a [B, h*k+2*pad, w*k+2*pad, Cout] map
   * (pad > 0: the interior of a buffer whose border udb_reflect_border_fill_nhwc_f16 fills). */
  int32_t ct_k, ct_cout, ct_h, ct_w, ct_pad;
  /* UDB_STORE_HEAD (N == 32): out_pixel = exp(clamp(sum_n head_w[n]*leaky(acc+bias)[n] + head_b,
   * -8, 8) + head_add) written as f32 to out[b*H*W + y*W + x]. */
  const float* head_w;
  float head_b, head_add;
  /* Split-f16 ("precise") operands, UDB_A_MATRIX only.  a_split_k = K1 > 0: every A row holds [hi(K1) | lo(K1)] with
   * x = hi + lo to ~22 bits (lo = f16(x - f32(hi))), lda >= 2*K1; W is packed [N, 3*K1] = [W_hi | W_hi | W_lo];
   * K must be 3*K1.  The k-blocks of the third segment re-read A's hi half, so the same MMAs accumulate
   * hi.W_hi + lo.W_hi + hi.W_lo in f32 -- the f16 product error (2^-11 per operand) drops to ~2^-21.
   * out_split > 0 (f16 `out`): also store lo = f16(v - f32(hi)) at column n + out_split, i.e. the output is itself a
   * split operand for the next GEMM. */
  int32_t a_split_k;
  int32_t out_split;
  /* Fused LayerNorm (the north_star's "fused LayerNorm + QKV projection"; reference metadinov2/block.py:84-109: the
   * LayerNorm that follows a residual update never runs as its own pass).
   * PRODUCER (ln_stats_out != NULL, ROWS store): besides its normal outputs the GEMM writes, for every output row and
   * every (column tile, column half) part, float2 {mean, centred sum of squares} of the values it stored:
   * ln_stats_out[(row * ln_parts + part)], ln_parts = (N / tile width) * 2, ln_part_cols = tile width / 2 (the call
   * fails if the caller's ln_parts / ln_part_cols do not match the tiling).  Use out2 for the f16 copy of the rows.
   * CONSUMER (ln_stats_in != NULL): A is that un-normalised f16 copy, W holds W * diag(ln_weight); the epilogue merges the
   * row's parts into mean / rstd (eps = ln_eps) and computes rstd * (acc - mean * ln_c1[n]) + bias[n], with
   * ln_c1[n] = sum_k W'[n,k] and bias = W ln_bias + linear bias -- algebraically LayerNorm followed by the Linear. */
  float* ln_stats_out;
  const float* ln_stats_in;
  const float* ln_c1;
  int32_t ln_parts, ln_part_cols;
  float ln_eps;
} udb_gemm_t;

int udb_gemm_f16(const udb_gemm_t* g, void* stream);
/* The same GEMM on FP8 E4M3 operands (UniDepthV2 precision "fp8"): A [M,K] and W [N,K] of `g` are e4m3 bytes, both
 * K-major (lda / ldw in bytes: >= K and multiples of 16), with f32 per-row scales a_scale[M] and per-column scales
 * w_scale[N] (both 16-byte aligned): the epilogue starts from v = acc * a_scale[m] * w_scale[n], then adds bias, applies
 * act / gamma / resid and stores as above.  The MMA partial sums are promoted into an f32 accumulator after every 128
 * values of K.  a_mode MATRIX and the ROWS store only; no split operands, out_split or ln_stats_*. */
int udb_gemm_e4m3(const udb_gemm_t* g, const float* a_scale, const float* w_scale, void* stream);
/* Epilogue of the last udb_gemm_f16 call on the calling thread that got past its checks: 1 = the TMA-store epilogue
 * (plain ROWS store with an identity row map, no out2 / out_split / ln_stats_*, 16-byte aligned out and row pitch, and
 * a residual only as f32 with an f32 out), 0 = the general one.  Both give bit-identical outputs; setting the
 * environment variable UDB_GEMM_TMA_EPILOGUE=0 routes every call to the general one. */
int udb_gemm_tma_epilogue_used(void);

/* ---------------------------------------------------------------------------------------------
 * 3x3 convolution with few output channels over a PRE-PADDED NHWC f16 image [B, H+2, W+2, cstride]
 * (channel slice [coff, coff+C)), weights f16 [Cout, 9*C] ordered (dy,dx,c), Cout in {32, 64}.
 * The input halo of each 16x8-pixel tile is loaded once and shared by the nine taps (shifted wgmma
 * descriptors); weights stay resident in shared memory.  out: f16 NHWC [B,H,W,ldc] -- or, with
 * head_out != NULL (Cout == 32), the fused head exp(clamp(sum_n head_w[n]*act(conv)[n] + head_b,
 * -8, 8) + head_add) as an f32 plane [B,H,W].  Replaces the reflect-padded nn.Conv2d calls of
 * unidepth/models/unidepthv2/decoder.py:200-229 (to_depth_lr/hr, to_confidence_lr/hr).
 * ------------------------------------------------------------------------------------------- */
typedef struct udb_conv_halo_t {
  const void* x;
  const void* w;
  const float* bias;   /* [cout], required */
  int32_t B, H, W, C, cstride, coff, cout, act;   /* B, H, W >= 1; coff + C <= cstride (0 = C) */
  void* out;           /* 4-byte aligned */
  int64_t ldc;         /* 0 = cout; even and >= cout */
  const float* head_w; /* required when head_out is set */
  float head_b, head_add;
  float* head_out;
} udb_conv_halo_t;
int udb_conv3x3_halo_f16(const udb_conv_halo_t* c, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fused softmax(Q K^T / sqrt(d)) V  (flash-style, wgmma QK^T and PV, S/O accumulators in registers).
 * Replaces F.scaled_dot_product_attention: metadinov2/attention.py:58, layers/attention.py:136.
 * q/k/v are f16 matrices with row stride ld* (elements); head h occupies columns
 * [col0 + h*head_dim, +head_dim).  Row of (batch b, position s) = b*seq + s.  out f16 [B*Sq, ldo].
 * ------------------------------------------------------------------------------------------- */
typedef struct udb_attn_t {
  const void* q;
  const void* k;
  const void* v;
  void* out; /* 4-byte aligned (f16 pairs are stored as 32-bit words) */
  int32_t B, heads, seq_q, seq_k, head_dim; /* B, heads, seq_q, seq_k >= 1; head_dim 64 */
  /* multiples of 8; each >= its col0 + heads*64 (+ its lo_off_* in split mode) */
  int32_t ldq, ldk, ldv, ldo;
  int32_t q_col0, k_col0, v_col0, o_col0; /* >= 0; o_col0 (and lo_off_o) even */
  float scale; /* 1/sqrt(head_dim) */
  /* Split-f16 ("precise") mode: when split != 0 the lo halves of q / k / v / out live lo_off_* elements to the right of
   * the hi halves (value = hi + lo) and the attention runs in an fp32 CUDA-core kernel (exact exp, f32 products):
   * a debugging / parity mode, ~50x slower than the wgmma kernel. */
  int32_t split;
  int32_t lo_off_q, lo_off_k, lo_off_v, lo_off_o;
} udb_attn_t;

int udb_attention_f16(const udb_attn_t* a, void* stream);

/* ---------------------------------------------------------------------------------------------
 * LayerNorm over the last dim (F.layer_norm): metadinov2/block.py:86,89 (eps 1e-6),
 * dinov2.py:336-345 (final norm, eps 1e-5), layers/attention.py:116-117, layers/mlp.py:30,
 * unidepthv2/decoder.py:190-199.  Input row r is read from in + in_row(r)*ld_in with
 * in_row(r) = (r / rows_per_group)*group_stride + r % rows_per_group + row_offset (identity if
 * rows_per_group <= 0) -- used to drop / pick the cls token of each image.
 * ------------------------------------------------------------------------------------------- */
typedef struct udb_layernorm_t {
  const void* in;
  int32_t in_f32;
  void* out;
  int32_t out_f32;
  const float* weight;
  const float* bias;
  int32_t rows, dim;
  int64_t ld_in, ld_out; /* ld_out >= dim + out_split */
  int32_t rows_per_group, group_stride, row_offset;
  float eps;
  int32_t dim_valid; /* 0 = dim.  f16->f16 rows of 64/128/256 only: statistics over the first dim_valid
                        columns (zero-padded channel rows, e.g. ViT-B's 96-channel map stored as 128) */
  int32_t out_split; /* > 0: also store lo = f16(y - f32(hi)) at column + out_split.  Only with in_f32 = 1 and
                        out_f32 = 0: any other combination (or a negative value) is rejected */
} udb_layernorm_t;

int udb_layernorm(const udb_layernorm_t* p, void* stream);
/* LayerNorm of f32 rows (in_f32 = 1, dim a multiple of 128 and <= 1024, no out_split / dim_valid; out_f32 is ignored) to
 * FP8 E4M3 bytes -- the A operand and a_scale of udb_gemm_e4m3: with the row scale s = amax|y| / 448 (1 for an all-zero
 * row) stored to out_scale[row], out[row, c] = e4m3(y * (448 / amax)), rounded to nearest even.  ld_out in bytes, a
 * multiple of 4; out 4-byte aligned. */
int udb_layernorm_e4m3(const udb_layernorm_t* p, float* out_scale, void* stream);

/* Row quantiser f16 -> FP8 E4M3 for the A operand of udb_gemm_e4m3: out[r, c] = e4m3(in[r, c] * 448 / amax_r) with
 * amax_r = max_c |in[r, c]|, round to nearest even, and the scale s[r] = amax_r / 448 (1 for an all-zero row) stored to
 * scale[r].  cols % 8 == 0 and
 * cols <= 6144; ld_in (elements) and ld_out (bytes) >= cols and multiples of 8; in / out 16-byte aligned. */
int udb_quantize_rows_e4m3(const void* in, int64_t ld_in, void* out, int64_t ld_out, float* scale, int32_t rows, int32_t cols,
                           void* stream);

/* ---------------------------------------------------------------------------------------------
 * Pre-processing + patch extraction (unidepthv2.py:288-297 + patch_embed.py:82's im2col):
 * uint8 (or f32 0..255) NCHW -> /255 -> (x-mean)/std -> zero pad -> bilinear (align_corners=False)
 * to (net_h, net_w) -> f16 patch matrix [B*gh*gw, ldp] with column c*196 + py*14 + px
 * (columns >= 588 zero).
 * ------------------------------------------------------------------------------------------- */
typedef struct udb_preprocess_t {
  const void* rgb;
  int32_t rgb_is_u8; /* 1: uint8, 0: float32 */
  int32_t normalize;
  int32_t B, H, W;
  int32_t pad_l, pad_r, pad_t, pad_b;
  int32_t net_h, net_w;
  void* patches;
  int32_t ldp;
  int32_t split; /* 1: rows hold [hi | lo] halves of ldp/2 columns each (split-f16 precise mode) */
} udb_preprocess_t;

int udb_preprocess_patchify(const udb_preprocess_t* p, void* stream);

/* Bicubic (A=-0.75, align_corners=False, no antialias) resize of the [1,M,M,D] position grid to
 * [gh,gw,D] (dinov2.py:267-304, interpolate_offset == 0).  f32 -> f32. */
int udb_posembed_bicubic(const float* grid, int32_t m, int32_t dim, float* out, int32_t gh,
                         int32_t gw, void* stream);

/* x[b, 0, :] = cls_token + pos_embed[0]   (dinov2.py:314-315); x f32 [B, T, D]. */
int udb_set_cls_rows(float* x, const float* cls_token, const float* pos0, int32_t B, int32_t T,
                     int32_t D, void* stream);
/* Same, for the fused-LayerNorm encoder (udb_gemm_t.ln_*): also writes the f16 copy of the cls rows and their per-part
 * {mean, centred sum of squares} (parts * part_cols == D, the producer GEMMs' tiling). */
int udb_set_cls_rows_ln(float* x, void* x16, float* stats, const float* cls_token, const float* pos0, int32_t B, int32_t T,
                        int32_t D, int32_t parts, int32_t part_cols, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Small fp32 dense layer for the 4-token camera head (unidepthv2/decoder.py:101-111), kept in
 * fp32 on CUDA cores to protect the 1e-4 intrinsics bar:
 *   y[m, n] = resid[m,n] + gamma[n] * act(sum_k x[m,k] * w[n,k] + bias[n])      M <= 64
 * ------------------------------------------------------------------------------------------- */
typedef struct udb_small_linear_t {
  const float* x;
  const float* w;
  const float* bias;
  const float* gamma;
  const float* resid;
  float* y;
  int32_t M, N, K;
  int32_t act;
  int32_t ldx, ldy, ldr; /* row strides (elements) of x, y, resid; 0 = dense (K, N, N).  16-byte loads along K when
                            K % 128 == 0, ldx % 4 == 0 and x, w are 16-byte aligned; one float per lane otherwise */
} udb_small_linear_t;
int udb_small_linear_f32(const udb_small_linear_t* p, void* stream);

/* Self-attention over the 4 camera tokens, fp32 (layers/attention.py:110-138 with pos_embed added
 * to q only).  q [B,4,C], kv [B,4,2C] (k then v), pos [4,C] -> out [B,4,C].  B >= 1, heads >= 1, C % heads == 0. */
int udb_camera_attn4_f32(const float* q, const float* kv, const float* pos, float* out, int32_t B,
                         int32_t C, int32_t heads, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Camera tail + rays (unidepthv2/decoder.py:85-99, 361-403; utils/coordinate.py:4-20):
 *   x[B,4] -> (fx,fy,cx,cy) = (exp,exp,sigmoid,sigmoid) * (0.7*diag, 0.7*diag, W, H)
 *   K_net[B,3,3]; K_out[B,3,3] = post-processed (unidepthv2.py:92-108); intr4[B,4].
 * ------------------------------------------------------------------------------------------- */
int udb_camera_intrinsics(const float* x, int32_t B, int32_t net_h, int32_t net_w, float factor,
                          int32_t pad_l, int32_t pad_t, float* intr4, float* k_net, float* k_out,
                          void* stream);

/* Ray embedding (unidepthv2/decoder.py:234-253; utils/geometric.py:227-252;
 * utils/positional_embedding.py:218-256): unit rays from intr4 (or from rays_in [B,net_h*net_w,3]
 * when not NULL) -> antialiased bilinear down-sample by `net/grid` -> renormalise -> polar,
 * azimuth -> sin(angle * pi * scales[j]); out f32/f16 [B*gh*gw, 2*bands]. */
/* infer(camera=K) (unidepthv2.py:267-303; Camera.crop / resize utils/camera.py:78-81,115-120):
 * K [B,3,3] pinhole in input-image pixels -> (fx,fy,cx,cy) in network-input pixels. */
int udb_camera_adjust_k(const float* K, int32_t B, float factor, int32_t pad_l, int32_t pad_t,
                        float* intr4, void* stream);

/* GT-camera rays for infer(camera=<Camera object>) (unidepthv2.py:267-303,361-362; utils/camera.py): the unit rays
 * [B, net_h*net_w, 3] f32 of each image's camera at the network-input pixel centres (u + 0.5, v + 0.5), i.e.
 * BatchCamera.from_camera(cam).crop(-pads).resize(factor).get_rays((B, net_h, net_w)) in the layout rays_in takes.
 * The camera is given in INPUT-image pixels, as the caller passes it to infer; the kernel applies the class's crop /
 * resize rules (Spherical also updates its W, H and half-FOVs) and its unproject arithmetic:
 *   UDB_CAM_PINHOLE     K (skew kept), inverted in the kernel; xyz / clip(z, 1e-4)
 *   UDB_CAM_EUCM        closed form                            UDB_CAM_SPHERICAL   closed form (equirectangular)
 *   UDB_CAM_OPENCV      16-parameter layout: undo tangential + thin prism (10 Newton steps), then radial k1..k3 (25)
 *   UDB_CAM_FISHEYE624  16-parameter layout: same, radial k1..k6 on theta, r = tan(theta)
 *   UDB_CAM_MEI         undo tangential (20 steps), radial k1, k2 (25), then the xi lift (xi == 1 handled)
 * params: [B, UDB_CAM_STRIDE] f32, 16-byte aligned, one row per image:
 *   [0..8]   Pinhole: K row-major;  other models: the class's params (fx fy cx cy ...), zero-padded to 16 ([0..15])
 *   [16..18] use_radial, use_tangential, use_thin_prism (1 or 0) as the class decided them on its parameters (a part
 *            whose coefficients sum to <= 1e-6 in absolute value is skipped); [19] unused
 * Rays are normalised as get_rays does (norm clamped at 1e-4).  Checked before launch, udb_last_error() naming the
 * argument: model known, B, net_h, net_w >= 1, params / rays non-null and aligned (16 / 4 bytes). */
enum {
  UDB_CAM_NONE = 0, UDB_CAM_PINHOLE = 1, UDB_CAM_EUCM = 2, UDB_CAM_SPHERICAL = 3, UDB_CAM_OPENCV = 4,
  UDB_CAM_FISHEYE624 = 5, UDB_CAM_MEI = 6
};
#define UDB_CAM_STRIDE 20
int udb_camera_rays(int32_t model, const float* params, int32_t B, int32_t net_h, int32_t net_w, int32_t pad_l,
                    int32_t pad_r, int32_t pad_t, int32_t pad_b, float factor, float* rays, void* stream);

/* Ground-truth point map (utils/camera.py reconstruct; the evaluation's camera.reconstruct(depth)): points [B, 3, H, W]
 * f32, planar, of each image's camera at the pixel centres of its depth map depth [B, 1, H, W] f32.  params are the
 * packed rows of udb_camera_rays, in the depth map's own pixels; no crop or resize is applied.  Each class's rule:
 *   UDB_CAM_PINHOLE     unproject(uv) * clip(depth, 0)
 *   UDB_CAM_SPHERICAL   unproject(uv) * depth                  (depth is the range)
 *   other models        xyz / clamp(xyz_z, 1e-4) * clamp(depth, 1e-4), xyz the class's unproject before get_rays
 * Clamps propagate NaN as torch's do, so a pixel outside the model's domain (MEI with xi > 1 far off axis) is NaN in all
 * three planes, as the class gives it.  Checked before launch as udb_camera_rays: model known, B in [1, 65535],
 * H, W >= 1, H * W <= 2^30, params / depth / points non-null and aligned (16 / 4 / 4 bytes). */
int udb_camera_reconstruct(int32_t model, const float* params, int32_t B, int32_t H, int32_t W, const float* depth,
                           float* points, void* stream);

typedef struct udb_ray_embed_t {
  const float* intr4;
  const float* rays_in;
  const float* scales; /* [bands] */
  int32_t B, net_h, net_w, gh, gw, bands;
  void* out;
  int32_t out_f32;
} udb_ray_embed_t;
int udb_ray_embed(const udb_ray_embed_t* p, void* stream);
/* The same resampled unit rays as UniDepthV2old's ray features (decoder_old.py:111-121, positional_embedding.py:218-256
 * with use_log and cat_orig): sin(pi * scales[k] * axis) for the three axes of the ray (axis-major, 3*bands features),
 * then the ray itself, zero-filled up to the row stride ld_out >= 3*bands + 3.
 * out_f32 = 2: split-f16 rows in the udb_gemm_t.a_split_k layout [hi | lo] of ld_out / 2 features each, hi = f16(y)
 * (what out_f32 = 0 stores) and lo = f16(y - f32(hi)), both halves zero past the 3*bands + 3 features; ld_out must be
 * even and ld_out / 2 >= 3*bands + 3. */
int udb_ray_embed_cat_orig(const udb_ray_embed_t* p, int32_t ld_out, void* stream);

/* x2 bilinear up-sample, align_corners=False (layers/upsample.py:215), NHWC f16 -> f16.
 * Optionally fused: out = up(x) is followed by nothing; see udb_gemm for the convT add. */
int udb_upsample2x_nhwc_f16(const void* in, void* out, int32_t B, int32_t H, int32_t W, int32_t C,
                            void* stream);

/* Bilinear align_corners=True resize NHWC f16 [B,H,W,C] -> [B,oh,ow,C] written into a buffer
 * reflect-padded by `pad` pixels on each side ([B,oh+2*pad,ow+2*pad,C]); pad = 0 gives the plain
 * resize (unidepthv2/decoder.py:299-301 + the reflect pad of the following conv :207-219). */
int udb_resize_ac_pad_nhwc_f16(const void* in, void* out, int32_t B, int32_t H, int32_t W,
                               int32_t C, int32_t oh, int32_t ow, int32_t pad, void* stream);

/* Reflect-pad by 1 pixel: NHWC f16 [B,H,W,C] -> [B,H+2,W+2,C] (nn.Conv2d padding_mode="reflect",
 * unidepthv2/decoder.py:200-213). */
int udb_reflect_pad1_nhwc_f16(const void* in, void* out, int32_t B, int32_t H, int32_t W, int32_t C,
                              void* stream);

/* Fill the 1-pixel border of a padded NHWC f16 buffer [B,H+2,W+2,C] by reflection of its interior
 * (the interior having been written by a GEMM with ct_pad = 1). */
int udb_reflect_border_fill_nhwc_f16(void* buf, int32_t B, int32_t H, int32_t W, int32_t C, void* stream);

/* =============================================================================================
 * UniDepthV1 operators (ConvNeXt encoder + V1 decoder; BASELINE config 4).  Reference call sites:
 * unidepth/models/backbones/convnext.py:130-298,459-471, unidepth/models/unidepthv1/decoder.py:38-300,
 * unidepth/models/unidepthv1/unidepthv1.py:30-94,288-373, unidepth/layers/{convnext,upsample,nystrom_attention}.py,
 * unidepth/utils/geometric.py:13-73,228-252, unidepth/utils/sht.py:833.  GEMM-shaped V1 work (every Linear, the stem /
 * downsample convolutions as im2col GEMMs, 1x1 and 3x3 convolutions, the 8x64-head attention blocks) reuses
 * udb_gemm_f16 / udb_attention_f16 above.
 * ============================================================================================= */

/* V1 pre-processing + stem im2col (unidepthv1.py:49-63,298-317; convnext.py:371-383): uint8 / f32 NCHW -> (/255) ->
 * ImageNet normalise -> antialiased bilinear to (rh, rw) -> zero pad (pad_l, pad_t) into (net_h, net_w) -> f16 rows
 * [B*gh*gw, 64] of the 4x4 stride-4 patches (column c*16 + py*4 + px, 48 used; gh = (net_h-4)/4+1).
 * patch == 14 (DINOv2 encoder): rows [B*(net_h/14)*(net_w/14), 640] of the 14x14 patches instead, column
 * c*196 + py*14 + px (588 used, the rest zero: the layout udb_preprocess_patchify writes for the V2 patch embedding). */
typedef struct udb_v1_preprocess_t {
  const void* rgb;
  int32_t rgb_is_u8, scale255, normalize;
  int32_t B, H, W;
  int32_t rh, rw, pad_l, pad_t;
  int32_t net_h, net_w;
  int32_t patch;          /* 0 or 4: the ConvNeXt stem layout above; 14: DINOv2 patch rows */
  void* patches;
} udb_v1_preprocess_t;
int udb_v1_preprocess(const udb_v1_preprocess_t* p, void* stream);
/* The same rows as split-f16 operands (UniDepthV1 precision "split"; udb_gemm_t.a_split_k): each row holds
 * [hi | lo], 2 x 64 (stem) or 2 x 640 (patch == 14) columns, hi = f16(v) -- bit for bit what udb_v1_preprocess
 * writes -- and lo = f16(v - f32(hi)). */
int udb_v1_preprocess_split(const udb_v1_preprocess_t* p, void* stream);

/* DINOv2 block output -> UniDepthV1 decoder level (unidepthv1.py:322-326 adds each block's cls token to its patch tokens;
 * decoder.py:371-379 takes the max over a slice of blocks).  x f32 [B, 1+N, D] (cls row first):
 *   acc[b*N + t, :] = first ? f16(x[b,1+t,:] + x[b,0,:]) : max(acc[b*N + t, :], f16(x[b,1+t,:] + x[b,0,:]))
 * f16 round-to-nearest is monotone, so the running max kept in f16 equals f16 of the f32 max.  cls_out (may be NULL)
 * [B, D] f32 = x[b,0,:], the raw cls row the camera head reads.  D % 8 == 0. */
int udb_vit_tap(const float* x, void* acc, float* cls_out, int32_t B, int32_t N, int32_t D, int32_t first, void* stream);
/* The same with the running max kept in f32 (acc f32 [B*N, D]; no rounding): UniDepthV1 precision "split". */
int udb_vit_tap_f32(const float* x, float* acc, float* cls_out, int32_t B, int32_t N, int32_t D, int32_t first, void* stream);

/* LayerNorm over the last dim for widths that are multiples of 64 up to 1536 (ConvNeXt channel LayerNorm / LayerNorm2d,
 * convnext.py:214,252-263; decoder LayerNorms).  in row r at in + r*ld_in (+ add[(r % add_mod)*dim ..] when add != NULL:
 * "tokens + positional embedding", decoder.py:92-94,224).  s2d_w > 0: rows are the pixels of [B, s2d_h, s2d_w] maps and
 * pixel (y,x) is written to row (b, y/2, x/2), columns ((y&1)*2+(x&1))*dim.. of the k2 s2 downsample's im2col matrix
 * [B*(s2d_h/2)*(s2d_w/2), ld_out] (a trailing odd row / column is dropped, as the strided convolution drops it).
 * out_f32: 0 f16, 1 (any other non-zero value but 2) f32, UDB_LN_OUT_SPLIT (2) a split-f16 operand: hi = f16(y) where
 * the f16 output goes and lo = f16(y - f32(hi)) ld_out/2 columns further right (ld_out even; ld_out/2 >= dim, or
 * >= 4*dim with space-to-depth, so that a row holds [hi | lo] of a udb_gemm_t.a_split_k operand). */
#define UDB_LN_OUT_SPLIT 2
typedef struct udb_layernorm_any_t {
  const void* in;
  int32_t in_f32;
  void* out;
  int32_t out_f32;
  const float* weight;
  const float* bias;
  int64_t rows;
  int32_t dim;
  int64_t ld_in, ld_out;
  float eps;
  const float* add;
  int64_t add_mod;
  int32_t s2d_h, s2d_w;
} udb_layernorm_any_t;
int udb_layernorm_any(const udb_layernorm_any_t* p, void* stream);

/* Depthwise 7x7, zero padding 3 (convnext.py:208-211 conv_dw; layers/convnext.py:16-24 dwconv): x f16 NHWC [B,H,W,C],
 * w f32 [49, C] (tap-major), bias f32 [C] -> y f16 NHWC.  C % 64 == 0. */
int udb_dwconv7_nhwc_f16(const void* x, const float* w, const float* bias, void* y, int32_t B, int32_t H, int32_t W,
                         int32_t C, void* stream);
/* The same convolution on f32 NHWC maps x -> y (same taps, zero padding, bias and f32 summation order: an input that is
 * exactly f16 gives the f32 sums udb_dwconv7_nhwc_f16 rounds).  C % 32 == 0; B, H, W >= 1. */
int udb_dwconv7_nhwc_f32(const float* x, const float* w, const float* bias, float* y, int32_t B, int32_t H, int32_t W,
                         int32_t C, void* stream);
/* ConvNeXt block head of UniDepthV1 precision "fp8" (convnext.py:208-212: conv_dw -> norm), fused: the depthwise 7x7 of
 * udb_dwconv7_nhwc_f16 (same x / w / bias, f32 accumulation, result rounded to f16 as that call stores it), then
 * LayerNorm over the channels (eps 1e-6, f32 statistics; ln_w / ln_b f32 [C]) written straight as FP8 E4M3 bytes out
 * [B*H*W, C] with the row scale s = amax|y| / 448 (1 for an all-zero row) in out_scale[B*H*W] and
 * out = e4m3(y * (448 / amax)), rounded to nearest even -- the A operand and a_scale of udb_gemm_e4m3, with the
 * arithmetic of udb_layernorm_e4m3.  C % 64 == 0 and C <= 1536; B, H, W >= 1; every pointer 16-byte aligned. */
int udb_dwconv7_ln_e4m3(const void* x, const float* w, const float* bias, const float* ln_w, const float* ln_b, void* out,
                        float* out_scale, int32_t B, int32_t H, int32_t W, int32_t C, void* stream);

/* dst = first ? src : max(dst, src) element-wise over n f16 values (decoder.py:371-374 max_stack over a stage's blocks). */
int udb_max_accum_f16(const void* src, void* dst, int64_t n, int32_t first, void* stream);
/* The same over n f32 values, n % 4 == 0. */
int udb_max_accum_f32(const float* src, float* dst, int64_t n, int32_t first, void* stream);

/* Mean over the HW pixels of an f32 NHWC map -> [B, C] (ConvNeXt "cls tokens", convnext.py:471).  B, HW, C >= 1. */
int udb_spatial_mean_f32(const float* x, float* out, int32_t B, int32_t HW, int32_t C, void* stream);

/* F.interpolate(bilinear, align_corners=False, antialias=True) of an f16 NHWC map (flat_interpolate, geometric.py:228-252). */
int udb_aa_resize_nhwc_f16(const void* in, void* out, int32_t B, int32_t H, int32_t W, int32_t C, int32_t oh, int32_t ow,
                           void* stream);
/* The same resize of an f32 NHWC map, with the same weights and summation order.  C % 8 == 0. */
int udb_aa_resize_nhwc_f32(const float* in, float* out, int32_t B, int32_t H, int32_t W, int32_t C, int32_t oh, int32_t ow,
                           void* stream);

/* Ray embedding of one decoder level (decoder.py:203-220): analytic unit rays of K (intr4 = fx,fy,cx,cy per image, network
 * resolution) antialias-averaged per token, re-normalised, 81 real spherical harmonics (sht.py:833, index l*(l+1)+m),
 * then the projection MLP's input LayerNorm (ln_w / ln_b [81], eps 1e-5).  out f16 [B*gh*gw, 128], columns >= 81 zero.
 * sh_k[l*9+m] = K_l^m (times sqrt(2) for m > 0). */
typedef struct udb_v1_rays_t {
  const float* intr4;
  int32_t B, net_h, net_w, gh, gw;
  const float* ln_w;
  const float* ln_b;
  void* out;
  float sh_k[81];
} udb_v1_rays_t;
int udb_v1_rays_sh81(const udb_v1_rays_t* p, void* stream);

/* Camera head tail (decoder.py:96-106,326-331; unidepthv1.py:56-62,88-91,354-356).  x4 [B,4] (may be NULL with
 * skip_camera) -> intr4_rays [B,4]: K the decoder's rays use (prediction, or the pre-processed GT K); k_out [B,3,3]: the
 * intrinsics returned to the caller; k4_points [B,4]: K of the final back-projection. */
int udb_v1_camera_intrinsics(const float* x4, const float* gt_k, int32_t B, int32_t net_h, int32_t net_w, float ratio,
                             int32_t pad_l, int32_t pad_t, int32_t skip_camera, float* intr4_rays, float* k_out,
                             float* k4_points, void* stream);

/* Single-head cross attention with a handful of queries (camera head `aggregate`, decoder.py:95): q f32 [B*nq, D]
 * (+ q_pos [nq, D] when not NULL: the learned latents_pos, layers/attention.py:129-131; then scaled by `scale`),
 * kv f16 [B*nk, 2D] = (k | v), out f32 [B*nq, D].  nq <= 4, D % 256 == 0; scratch: B*16*nq*(D+2) floats (the keys are split
 * over 16 blocks per image, partial results are merged by a second kernel). */
int udb_cross_attn_small(const float* q, const float* q_pos, const void* kv, float* out, float* scratch, int32_t B, int32_t nq,
                         int32_t nk, int32_t D, float scale, void* stream);
/* The same with kv f32 [B*nk, 2D] (UniDepthV1 precision "split"); same summation order. */
int udb_cross_attn_small_f32(const float* q, const float* q_pos, const float* kv, float* out, float* scratch, int32_t B,
                             int32_t nq, int32_t nk, int32_t D, float scale, void* stream);

/* p[r, j] = softmax_j(scale * s[r, j]) over j < n_valid, f32 [rows, ld_in] -> f16 [rows, ld_out], columns >= n_valid zero
 * (the P operand of the dense single-head attentions aggregate_16 / prompt_camera, decoder.py:231-236).  rows >= 0,
 * 1 <= n_valid <= ld_in and n_valid <= ld_out; columns >= n_valid of s are never read. */
int udb_softmax_rows(const float* s, void* p, int64_t rows, int32_t n_valid, int32_t ld_in, int32_t ld_out, float scale,
                     void* stream);

/* out = a + b (f32; out and/or an f16 copy), n % 4 == 0 (decoder.py:246-252 `latents + rays_embedding`). */
int udb_add_f32(const float* a, const float* b, float* out, void* out_f16, int64_t n, void* stream);

/* f32 [groups*rows_per_group, D] -> f16 rows (g*dst_group_stride + dst_row0 + r) of dst (decoder.py:94 torch.cat).
 * groups, rows_per_group, D >= 1. */
int udb_copy_rows_f32_to_f16(const float* src, void* dst, int32_t groups, int32_t rows_per_group, int32_t D,
                             int64_t dst_group_stride, int64_t dst_row0, void* stream);

/* exp(clamp(conv3x3(x; w [9, C], bias), -10, 10)) with one output channel, zero padding: x f16 NHWC -> f32 [B,H,W]
 * (decoder.py:253,268,283,292-294 out8 / out4 / out2). */
int udb_conv3x3_c1_exp(const void* x, const float* w, float bias, float* out, int32_t B, int32_t H, int32_t W, int32_t C,
                       void* stream);

/* Nystrom attention pieces (layers/nystrom_attention.py:22-84 -> xformers NystromAttention(num_landmarks=128); restated
 * algorithm and its "parity unpinned" status: oracle/unidepth_v1_oracle.py).  64-wide heads.
 * landmarks: segment means of q (qbuf [B*n, ldq]) and k (kvbuf [B*n, ldkv]) -> f16 [B*128, 2*heads*64] = (ql | kl).
 * k2_pinv:   kernel_2 = softmax(ql kl^T / 8) -> k2 [B*heads,128,128] f32; z = its Newton-Schulz pseudo-inverse
 *            (`iters` steps, tmp = 3 * B*heads*128*128 floats).
 * zk3:       out[(b, lm), h*64+d] = sum_j z[b,h][lm][j] * k3[(b, j), h*64+d]   (f16 in / out). */
int udb_nystrom_landmarks(const void* q, int32_t ldq, const void* kv, int32_t ldkv, void* out, int32_t B, int32_t n,
                          int32_t heads, void* stream);
int udb_nystrom_k2_pinv(const void* landmarks, float* k2, float* z, float* tmp, int32_t B, int32_t heads, int32_t iters,
                        void* stream);
int udb_nystrom_zk3(const float* z, const void* k3, int32_t ldk3, void* out, int32_t ldo, int32_t B, int32_t heads, void* stream);

/* V1 post-processing (unidepthv1.py:66-94,352-366).  mean_maps: the three exp'ed maps (gh*2, gh*4, gh*8 grids) antialias-
 * resized to the network shape and averaged (B, gh, gw, net_h, net_w >= 1).  postprocess: crop the paddings, antialias-resize
 * to (H, W) -> depth; points = spherical_zbuffer_to_euclidean(theta, phi, z) with the angles of the unit ray of k4
 * (fx,fy,cx,cy) through each pixel.  B, H, W >= 1, paddings >= 0 and the cropped size net - pads >= 1 on both axes. */
int udb_v1_mean_maps(const float* o8, const float* o4, const float* o2, float* mean, int32_t B, int32_t gh, int32_t gw,
                     int32_t net_h, int32_t net_w, void* stream);
typedef struct udb_v1_postprocess_t {
  const float* mean;
  const float* k4;
  int32_t B, net_h, net_w, pad_l, pad_r, pad_t, pad_b, H, W;
  float* out_depth;
  float* out_points;
} udb_v1_postprocess_t;
int udb_v1_postprocess(const udb_v1_postprocess_t* p, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Output assembly (unidepthv2.py:80-89, 311-339, 375-377; unidepthv2/decoder.py:456-462):
 * radius/confidence f32 [B,net_h,net_w] (already exp'ed), rays from intr4 (or rays_in) ->
 * points = rays*radius -> resize (F.interpolate(mode, align_corners=False), no antialias) to
 * (padded_h, padded_w) -> crop pads -> confidence[B,1,H,W], radius[B,1,H,W]=|points|,
 * depth[B,1,H,W]=points.z, points[B,3,H,W], rays[B,3,H,W] renormalised.  All f32.
 * mode: the reference's `interpolation_mode` (unidepthv2.py:80-89), UDB_INTERP_BILINEAR (0) or
 * UDB_INTERP_BICUBIC (1, ATen upsample_bicubic2d: A = -0.75, border taps clamped; the result is not
 * clamped, so depth and confidence can overshoot to <= 0 at edges).  Any other value fails before launch.
 * ------------------------------------------------------------------------------------------- */
enum { UDB_INTERP_BILINEAR = 0, UDB_INTERP_BICUBIC = 1 };
typedef struct udb_postprocess_t {
  const float* radius;
  const float* confidence;
  const float* intr4;
  const float* rays_in; /* optional [B, net_h*net_w, 3] */
  int32_t B, net_h, net_w, padded_h, padded_w, pad_l, pad_t, H, W;
  int32_t mode;         /* UDB_INTERP_*; fills the alignment slot before the output pointers (the size is unchanged) */
  float* out_confidence;
  float* out_radius;
  float* out_depth;
  float* out_points;
  float* out_rays;
} udb_postprocess_t;
int udb_postprocess(const udb_postprocess_t* p, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Output assembly of the evaluation forward (unidepthv2.py:134-160 `forward_test`, with
 * utils/misc.py:596-642 `match_gt` and :645-690 `match_intrinsics`), one launch:
 *   per image b with pads[b] = (l, r, t, b) of the network input, crop the network maps to
 *   [t, net_h-b) x [l, net_w-r) and resize the crop to H x W with bilinear (align_corners=False, no
 *   antialias; ATen upsample_bilinear2d's fp32 index arithmetic, scale = crop / out, source clamped
 *   at 0), taking the taps of points = rays*radius -> out_points [B,3,H,W], out_depth [B,1,H,W] =
 *   points.z, out_confidence [B,1,H,W];
 *   out_rays [B,3,net_h,net_w]: the network's rays, normalised twice (max(|r|, 1e-5)), at the
 *   network size (the reference returns them unmatched);
 *   intrinsics [B,3,3] IN PLACE: the K of the network input in, match_intrinsics' K out (f32, fx*sx,
 *   fy*sy, (cx-l)*sx, (cy-t)*sy with sx = f32(W / (net_w-l-r)) rounded from the double ratio).
 * rays come from rays_in when given, else from intr4 (fx, fy, cx, cy).  pads is DEVICE memory, so a
 * negative pad or a crop that leaves no row or column cannot be refused before the launch: that
 * image's maps and K come out NaN, nothing is read out of range.  The caller checks the pads (the
 * Python boundary class does, before anything runs).
 * ------------------------------------------------------------------------------------------- */
typedef struct udb_match_gt_t {
  const float* radius;       /* [B, net_h, net_w] */
  const float* confidence;   /* [B, net_h, net_w] */
  const float* intr4;        /* [B,4], read when rays_in is NULL */
  const float* rays_in;      /* optional [B, net_h*net_w, 3] */
  const int32_t* pads;       /* device [B,4] l r t b, each >= 0 */
  int32_t B, net_h, net_w, H, W;
  float* intrinsics;         /* [B,3,3] in place */
  float* out_confidence;
  float* out_depth;
  float* out_points;
  float* out_rays;
} udb_match_gt_t;
int udb_match_gt(const udb_match_gt_t* p, void* stream);

/* ======================================================================================
 * Whole-path engine: one handle = one UniDepthV2 model on one device.
 *
 * Replaces the body of `UniDepthV2.infer` (unidepth/models/unidepthv2/unidepthv2.py:239-339:
 * pre-process -> `encode_decode` :341-377 -> `_postprocess` :80-108) as ONE call that only enqueues
 * kernels on the caller's stream: no allocation, no host<->device copy, no synchronisation, so the
 * call is CUDA-graph capturable.  The caller (the Python boundary class, or any C program) owns all
 * memory: packed weights, the workspace and the seven output tensors.
 *
 * Life cycle:   udb_create -> udb_set_weight / udb_set_scalar (once per packed tensor)
 *               -> udb_workspace_bytes(B,H,W,level)  [per new input shape; also prepares the
 *                  shape-dependent tables: resized position embedding, ray-embedding frequencies]
 *               -> udb_infer_v2 (any number of times) -> udb_destroy.
 * A handle is not thread-safe (neither is a reference model instance: `infer` mutates module state,
 * decoder.py:436,447-448).  All functions return 0 on success, non-zero + udb_last_error() otherwise.
 * ====================================================================================== */
typedef struct udb_engine udb_engine;

enum { UDB_DT_F16 = 0, UDB_DT_F32 = 1, UDB_DT_E4M3 = 2 };

typedef struct udb_config_t {
  /* DINOv2 encoder (unidepth/models/backbones/dinov2.py:388-427, encoder.py:139-193) */
  int32_t embed_dim, depth, enc_heads;
  int32_t taps[4];      /* 1-based indices of the four block outputs consumed (unidepthv2.py:365-372) */
  int32_t pos_grid;     /* side of the stored position-embedding grid (37) */
  /* decoder (unidepth/models/unidepthv2/decoder.py:470-524) */
  int32_t hidden, dec_heads, expansion, out_dim;
  int32_t n_stages;     /* len(depths) */
  int32_t dec_depths[4];
  /* data.augmentations.shape_constraints of the model config (unidepthv2.py:247-262) */
  double ratio_min, ratio_max;
  double pixels_min, pixels_max;
} udb_config_t;

int udb_create(const udb_config_t* cfg, udb_engine** out);
void udb_destroy(udb_engine* e);

/* Register one PACKED tensor (device pointer, borrowed for the life of the handle) under the engine's
 * own name; the packing (f16 operand layouts, folded LayerNorm->Linear heads, zero-padded narrow
 * heads) is described in DESIGN.md and done once per checkpoint by the boundary class from the
 * reference's state_dict (SURVEY.md 8b).  dtype: UDB_DT_*. */
int udb_set_weight(udb_engine* e, const char* name, const void* dev_ptr, const int64_t* shape, int32_t ndim,
                   int32_t dtype);
/* Host scalars of the packed model (the two 1x1 head biases and their additive constants), and the encoder mode:
 * "precision" 0 = f16 operands, 1 = split-f16 (hi/lo) operands, 2 = FP8 E4M3 operands for the four linear layers of every
 * encoder block (blocks.{i}.{qkv,proj,fc1,fc2}_w8 [N, K] UDB_DT_E4M3 with f32 per-output-channel scales *_w8s [N]; the
 * activations are quantised per row on the fly); "fuse_ln" 1 = fused LayerNorm (precision 0 only).  The schedule
 * (udb_workspace_bytes, udb_schedule_bytes, udb_infer_v2) refuses any other "precision", and precision 1 with a patch_w
 * that is not split-packed ([D, 3*640]), naming the mode. */
int udb_set_scalar(udb_engine* e, const char* name, double value);

/* Geometry of one call, same arithmetic as get_paddings / get_resize_factor (unidepthv2.py:36-77). */
typedef struct udb_geometry_t {
  int32_t pad_l, pad_r, pad_t, pad_b;
  int32_t padded_h, padded_w;
  int32_t net_h, net_w;   /* network input, multiples of 14 */
  int32_t gh, gw;         /* patch grid */
  double factor;
} udb_geometry_t;
/* resolution_level: 0..9, -1 = attribute unset (default pixel bounds), or UDB_LEVEL_NETWORK_ONLY: the input
 * already is the network input (normalised float tensor, H and W multiples of 14): identity geometry, the
 * outputs are the network's own (the reference's `encode_decode` as used by `forward_test`,
 * unidepthv2.py:134-160, and by the ONNX wrappers, export.py:27-45). */
#define UDB_LEVEL_NETWORK_ONLY (-2)
int udb_geometry(const udb_engine* e, int32_t H, int32_t W, int32_t resolution_level, udb_geometry_t* out);

/* Bytes of scratch udb_infer_v2 needs for this shape; also prepares the per-shape tables (may
 * allocate and launch on the default stream: call it outside graph capture). 0 = error. */
size_t udb_workspace_bytes(udb_engine* e, int32_t B, int32_t H, int32_t W, int32_t resolution_level);
/* The same number from a dry run of the schedule alone: walks every stage with the registered operands, checks their
 * names and shapes, sizes the bump allocator -- and touches no device (no table is prepared, nothing is recorded), so it
 * also works on a machine without a GPU.  udb_infer_v2 still requires udb_workspace_bytes.  0 = error. */
size_t udb_schedule_bytes(udb_engine* e, int32_t B, int32_t H, int32_t W, int32_t resolution_level);

typedef struct udb_infer_args_t {
  const void* rgb;            /* [B,3,H,W] uint8 or float32 (0..255 when normalize) */
  int32_t rgb_is_u8, normalize;
  int32_t B, H, W;
  int32_t resolution_level;   /* 0..9 or -1 */
  int32_t interpolation;      /* UDB_INTERP_* of the output resize (the reference's `interpolation_mode`); 0, what a
                                 zero-initialised struct holds, is bilinear, the reference's default */
  const float* camera_k;      /* optional [B,3,3] pinhole K in input-image pixels (infer(camera=K),
                                 unidepthv2.py:267-303): rays come from it, intrinsics stay predicted */
  const float* camera_rays;   /* optional [B, net_h*net_w, 3] unit rays at network-input resolution produced by the
                                 caller's camera model (infer(camera=<Camera object>): camera.crop / resize /
                                 get_rays, unidepthv2.py:299-303,361-362; decoder.py:400); overrides camera_k */
  int32_t camera_model;       /* UDB_CAM_* of camera_params; 0 (UDB_CAM_NONE) = no camera model.  With a model the engine
                                 generates the rays itself (udb_camera_rays into its workspace) from the camera in
                                 input-image pixels; setting it together with camera_k or camera_rays is an error */
  const float* camera_params; /* [B, UDB_CAM_STRIDE] packed camera rows (see udb_camera_rays), with camera_model */
  const float* ray_scales;   /* optional [hidden/2] frequency table (positional_embedding.py:231-233);
                                 NULL = the engine's own table */
  void* workspace;
  size_t workspace_bytes;
  /* outputs, float32, caller-allocated (keys of the dict returned by infer, unidepthv2.py:331-339) */
  float* confidence;          /* [B,1,H,W] */
  float* intrinsics;          /* [B,3,3]   */
  float* radius;              /* [B,1,H,W] */
  float* depth;               /* [B,1,H,W] */
  float* points;              /* [B,3,H,W] */
  float* rays;                /* [B,3,H,W] */
  float* depth_features;      /* [B,gh,gw,hidden] channel-last (the reference returns the same values
                                 as [B,hidden,gh,gw]; the boundary class returns a permuted view) */
} udb_infer_args_t;

int udb_infer_v2(udb_engine* e, const udb_infer_args_t* a, void* stream);

/* Evaluation forward (`forward_test`, unidepthv2.py:134-160): `args` as for udb_infer_v2 with resolution_level
 * UDB_LEVEL_NETWORK_ONLY, and the output assembly of udb_match_gt selected by match_h, match_w >= 1 and match_pads:
 * confidence, depth and points are the network maps cropped by match_pads and resized to [B,*,match_h,match_w]
 * (`match_gt`), intrinsics is `match_intrinsics`' K, rays stay [B,3,H,W] at the network size, and radius is not written
 * (may be NULL).  All three zero: exactly udb_infer_v2(args).  The engine refuses, before any launch, match fields at
 * another resolution_level, and a size without pads or pads without a size.  match_pads lives on the device, so the
 * engine cannot see a crop that leaves no row or column (that image's outputs come out NaN): the caller checks
 * H - t - b >= 1, W - l - r >= 1 and every pad >= 0.  The matching takes no workspace: udb_workspace_bytes of the
 * network-only shape applies.  A struct of its own, so that udb_infer_args_t keeps its layout for existing callers. */
typedef struct udb_infer_match_args_t {
  udb_infer_args_t args;
  int32_t match_h, match_w;
  const int32_t* match_pads;  /* device [B,4] int32: l r t b of each network input */
} udb_infer_match_args_t;
int udb_infer_v2_match(udb_engine* e, const udb_infer_match_args_t* a, void* stream);

/* ---------------------------------------------------------------------------------------------
 * UniDepthV1 engine: the whole `UniDepthV1.infer` path (ConvNeXt or DINOv2 encoder) as one call (SURVEY.md section 8b
 * `udb_infer_v1`; reference unidepth/models/unidepthv1/unidepthv1.py:288-373).  Same contract as the V2 engine: the
 * caller owns packed weights (names listed by unidepth_b200/unidepthv1.py UniDepthV1._pack_tensors, with the packers
 * the V1-family decoders share in unidepth_b200/_pack.py), workspace and outputs; nothing is allocated, copied or
 * synchronised inside udb_infer_v1.
 * ------------------------------------------------------------------------------------------- */
typedef struct udb_engine_v1 udb_engine_v1;

#define UDB_V1_ENCODER_CONVNEXT 0
#define UDB_V1_ENCODER_DINOV2 1

typedef struct udb_v1_config_t {
  int32_t depths[4];      /* ConvNeXt blocks per stage (convnext_large: 3,3,27,3); DINOv2: blocks per max-pooled slice
                             (ViT-L: 5,7,6,6 = output_idx 5,12,18,24) */
  int32_t dims[4];        /* stage widths (192,384,768,1536); DINOv2: the embedding width four times */
  int32_t hidden, heads, expansion;
  int32_t dec_depths[3];  /* attention blocks at 1/16, Nystrom blocks at 1/8 and 1/4 (config pixel_decoder.depths) */
  int32_t encoder;        /* UDB_V1_ENCODER_*; 0 (ConvNeXt) for zero-initialised configs */
  int32_t net_h, net_w;   /* fixed network input (config data.image_shape: 462 x 616) */
} udb_v1_config_t;

int udb_v1_create(const udb_v1_config_t* cfg, udb_engine_v1** out);
void udb_v1_destroy(udb_engine_v1* e);
int udb_v1_set_weight(udb_engine_v1* e, const char* name, const void* dev_ptr, const int64_t* shape, int32_t ndim,
                      int32_t dtype);
/* Host scalars of the packed V1 model (the three output-head biases) and the encoder mode "precision": 0 (or absent) = f16
 * operands, 1 = split-f16 operands (parity mode, as UniDepthV2's): every GEMM operand of the encoder and of the camera
 * head's context path is a [hi | lo] pair and its weight is packed [N, 3K] = [hi | hi | lo] (udb_gemm_t.a_split_k) --
 * stem_w, ds{i}.w, s{i}.b{j}.w1 / w2 or the DINOv2 blocks and patch_w, adapt.{l}.w_cam (the adapters' copy feeding the
 * camera head), cam.inf.w1 / w2 and cam.agg.kv_w -- the residual stream, the encoder levels and the camera context stay
 * f32 and the DINOv2 attention runs in the fp32 kernel; the depth head reads the f16 (hi) half and runs as in the f16
 * mode.  2 = FP8 E4M3 operands for the two MLP linear layers of the ConvNeXt encoder blocks of the stages the schedule
 * runs in e4m3 (engine_v1.cu kFp8Stage; none at present, as none is faster that way) (s{i}.b{j}.w1_8 [4C, C],
 * w2_8 [C, 4C] UDB_DT_E4M3 with f32 per-output-channel scales w1_8s / w2_8s; udb_dwconv7_ln_e4m3 and
 * udb_quantize_rows_e4m3 quantise the activations per row) or for the four linear layers of every DINOv2 block (the
 * blocks.{i}.*_w8 operands of the V2 engine's fp8 mode); there the stem, downsample layers, attention and the decoder
 * stay f16. */
int udb_v1_set_scalar(udb_engine_v1* e, const char* name, double value);
/* Shape arithmetic of one V1 call, the engine's own copy of `_shapes` / `_paddings` (unidepthv1.py:30-46): the image is resized
 * by `ratio` to (resized_h, resized_w) -- the larger side-ratio that still fits the fixed network input -- and zero-padded
 * (pad_* >= 0 here; Python floor division kept for the general case) to net_h x net_w. */
typedef struct udb_v1_geometry_t {
  int32_t resized_h, resized_w;
  int32_t pad_l, pad_r, pad_t, pad_b;
  double ratio;
} udb_v1_geometry_t;
int udb_v1_geometry(int32_t H, int32_t W, int32_t net_h, int32_t net_w, udb_v1_geometry_t* out);
/* bytes of workspace udb_infer_v1 needs for this shape (0 + udb_last_error on failure); must be called once per
 * (B, H, W) after the weights are registered and outside stream capture */
size_t udb_v1_workspace_bytes(udb_engine_v1* e, int32_t B, int32_t H, int32_t W);

typedef struct udb_infer_v1_args_t {
  const void* rgb;        /* [B,3,H,W] uint8 or float32 */
  int32_t rgb_is_u8;
  int32_t scale255;       /* divide by 255 first (uint8, or float data with max > 5: unidepthv1.py:301-302) */
  int32_t normalize;      /* ImageNet mean / std (data in [0,1] after the optional /255: unidepthv1.py:303-308) */
  int32_t B, H, W;
  const float* intrinsics; /* optional GT pinhole K [B,3,3] (original image frame) */
  int32_t skip_camera;     /* with intrinsics: do not run the camera head, return the GT K (unidepthv1.py:336) */
  void* workspace;
  size_t workspace_bytes;
  float* out_intrinsics;  /* [B,3,3] */
  float* out_points;      /* [B,3,H,W] */
  float* out_depth;       /* [B,1,H,W] */
} udb_infer_v1_args_t;

int udb_infer_v1(udb_engine_v1* e, const udb_infer_v1_args_t* a, void* stream);

/* ---------------------------------------------------------------------------------------------
 * UniDepthV2old engine: the whole `UniDepthV2old.infer` path (DINOv2 ViT-L/14 or ViT-S/14) as one call (reference
 * unidepth/models/unidepthv2/unidepthv2_old.py:198-282, decoder_old.py).  One engine per network shape (net_h, net_w),
 * which `udb_v2old_geometry` derives from the input size and the resolution level; otherwise the contract of the V1 engine:
 * the caller owns the packed weights (names listed by unidepth_b200/unidepthv2old.py UniDepthV2old._pack_tensors, with
 * the packers the V1-family decoders share in unidepth_b200/_pack.py), workspace and outputs, and nothing is allocated,
 * copied or synchronised inside udb_infer_v2old.
 * ------------------------------------------------------------------------------------------- */
typedef struct udb_engine_v2old udb_engine_v2old;

typedef struct udb_v2old_config_t {
  int32_t embed_dim, enc_depth, enc_heads;  /* DINOv2: 1024 / 24 / 16 (ViT-L) or 384 / 12 / 6 (ViT-S) */
  int32_t output_idx[4];  /* encoder blocks (1-based) whose normed patch tokens feed the decoder (21..24 or 9..12) */
  int32_t hidden, heads, expansion;   /* 512 / 8 / 4 */
  int32_t nystrom_depth;  /* Nystrom blocks at the first decoder level (config pixel_decoder.depths[0]: 6) */
  int32_t net_h, net_w;   /* the network shape, multiples of 14 */
} udb_v2old_config_t;

int udb_v2old_create(const udb_v2old_config_t* cfg, udb_engine_v2old** out);
void udb_v2old_destroy(udb_engine_v2old* e);
int udb_v2old_set_weight(udb_engine_v2old* e, const char* name, const void* dev_ptr, const int64_t* shape, int32_t ndim,
                         int32_t dtype);
int udb_v2old_set_scalar(udb_engine_v2old* e, const char* name, double value);
/* Shape arithmetic of `infer` (unidepthv2_old.py:45-92): the pixel count of `resolution_level` (clipped to [0, 10]; pass
 * 10 for the reference's None) between pixels_lo and pixels_hi patches, and the network shape with the input's aspect
 * ratio at that many patches (both sides multiples of 14), with ratio = net_h / H.  The reference's warnings (level out
 * of range, aspect ratio out of bounds) are the caller's. */
typedef struct udb_v2old_geometry_t {
  int32_t pixels;          /* patches of the resolution level */
  int32_t net_h, net_w;
  double ratio;
} udb_v2old_geometry_t;
int udb_v2old_geometry(int32_t H, int32_t W, int32_t resolution_level, int32_t pixels_lo, int32_t pixels_hi,
                       udb_v2old_geometry_t* out);
/* bytes of workspace udb_infer_v2old needs for (B, H, W) (0 + udb_last_error on failure), from a dry run of the
 * schedule that launches nothing: udb_v2old_schedule_bytes only sizes (and names the first missing or mis-shaped
 * operand), udb_v2old_workspace_bytes also records the shape as prepared; call it once per (B, H, W) before
 * udb_infer_v2old, outside stream capture. */
size_t udb_v2old_schedule_bytes(udb_engine_v2old* e, int32_t B, int32_t H, int32_t W);
size_t udb_v2old_workspace_bytes(udb_engine_v2old* e, int32_t B, int32_t H, int32_t W);

#define UDB_V2OLD_BILINEAR 0
#define UDB_V2OLD_NEAREST_EXACT 1

typedef struct udb_infer_v2old_args_t {
  const void* rgb;         /* [B,3,H,W] uint8 or float32 */
  int32_t rgb_is_u8;
  int32_t scale255;        /* divide by 255 first (uint8, or float data with max > 5) */
  int32_t normalize;       /* ImageNet mean / std (data in [0,1] after the optional /255) */
  int32_t B, H, W;
  const float* intrinsics; /* optional GT pinhole K [B,3,3] (input image frame): rays and points use it */
  int32_t interpolation;   /* depth resize to H x W: UDB_V2OLD_BILINEAR or UDB_V2OLD_NEAREST_EXACT */
  void* workspace;
  size_t workspace_bytes;
  float* out_intrinsics;   /* [B,3,3] predicted K at the input size */
  float* out_points;       /* [B,3,H,W] */
  float* out_depth;        /* [B,1,H,W] */
  float* out_confidence;   /* [B,1,H,W] */
  /* Network-only mode (the reference's `forward(inputs, image_metas)`, unidepthv2_old.py:134-196), selected by
   * network_only = 1; all zero gives `infer` as above.  `rgb` is the network input itself: f32 (rgb_is_u8, scale255
   * and normalize 0), already normalised, with (H, W) the engine's network shape, else a named error before any launch.
   * The ratio is 1: a given K drives the rays as it is, and must then come with (out_h, out_w) == (H, W).  `interpolation`
   * is not read.  Outputs: out_intrinsics the predicted K (also when K is given); out_depth and out_confidence
   * [B,1,out_h,out_w], antialiased bilinear from the network shape; out_points [B,3,out_h,out_w] through the predicted K
   * on the out_h x out_w grid. */
  int32_t network_only;
  int32_t out_h, out_w;    /* network-only: size of the depth, confidence and points outputs */
  float* out_depth_features; /* network-only, optional: [B, (H/14)*(W/14), hidden] f32 latents of the depth head after
                                aggregate_16 and prompt_camera, before the Nystrom blocks */
} udb_infer_v2old_args_t;

int udb_infer_v2old(udb_engine_v2old* e, const udb_infer_v2old_args_t* a, void* stream);

/* Kernels of the UniDepthV2old decoder no other model runs (unidepth_b200/csrc/v1_kernels.cu). */
/* PixelShuffle(2) of NHWC f16 [B,h,w,C] -> depthwise 7x7 (zero pad; w tap-major [49, C/4] f32, bias [C/4]) -> ReLU ->
 * NHWC f16 [B,2h,2w,ldo], channels C/4..ldo-1 zero (layers/upsample.py:110-121 before the 3x3 conv) */
int udb_pshuffle_dw7_relu(const void* x, const float* w, const float* bias, void* out, int32_t B, int32_t h, int32_t wd, int32_t C,
                          int32_t ldo, void* stream);
typedef struct udb_v2old_heads_t {
  const float* levels[3];  /* level i: f32 NHWC [B, 2gh<<i, 2gw<<i, 32] = [depth MLP 16 | confidence MLP 16] */
  const float* w;          /* [2][48][49]: to_depth then to_confidence, input channel block 2-i for level i */
  float bias_depth, bias_conf;
  int32_t B, gh, gw, net_h, net_w;
  float* logdepth;         /* [B, net_h, net_w] */
  float* confidence;       /* [B, net_h, net_w], after the sigmoid */
} udb_v2old_heads_t;
int udb_v2old_heads(const udb_v2old_heads_t* p, void* stream);
/* in place on [B, hw] log-depth: LayerNorm over each map, exp, (x + shift) * exp(log_scale), softplus(beta 10);
 * scale_shift [B, 2] = (log_scale, shift) */
int udb_v2old_depth_tail(float* depth, const float* scale_shift, int32_t B, int64_t hw, void* stream);
typedef struct udb_v2old_postprocess_t {
  const float* depth;      /* [B, net_h, net_w] */
  const float* confidence; /* [B, net_h, net_w] */
  const float* k4;         /* [B, 4] fx, fy, cx, cy of the points' K at the input size */
  int32_t B, net_h, net_w, H, W, mode;   /* mode: UDB_V2OLD_BILINEAR or UDB_V2OLD_NEAREST_EXACT */
  float* out_depth;        /* [B,1,H,W] */
  float* out_confidence;   /* [B,1,H,W] antialiased bilinear */
  float* out_points;       /* [B,3,H,W] */
  int32_t depth_aa;        /* 1: depth with antialiased bilinear, as the confidence (`mode` is then not read) */
} udb_v2old_postprocess_t;
int udb_v2old_postprocess(const udb_v2old_postprocess_t* p, void* stream);
/* x4 [B,4] camera-head output -> intr4_rays [B,4] (gt_k * ratio, else the prediction at the network shape), k_out [B,3,3]
 * (the prediction at the input size), k4_points [B,4] (gt_k, else the prediction at the input size) */
int udb_v2old_camera(const float* x4, const float* gt_k, int32_t B, int32_t net_h, int32_t net_w, float ratio, float* intr4_rays,
                     float* k_out, float* k4_points, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Peer-memory plumbing of the multi-GPU output gather (one process per GPU on one node; SURVEY.md section 8e).
 * alloc: device buffer (zero-filled) + its 64-byte CUDA IPC handle, to be exchanged out of band (torch.distributed);
 * open: map a peer's buffer; barrier: device-side barrier over flags in peer memory (flag arrays of `world` uint32,
 * peer_flags_dev = device array of the ranks' flag-array pointers as mapped HERE; epochs only grow; a missing peer sets
 * *timeout_flag_dev instead of hanging); copy: copy-engine device-to-device copy (no SM involved).
 * ------------------------------------------------------------------------------------------- */
int udb_p2p_alloc(size_t bytes, void** dev_ptr, void* handle64);
int udb_p2p_open(const void* handle64, void** peer_ptr);
int udb_p2p_close(void* peer_ptr);
int udb_p2p_free(void* dev_ptr);
int udb_p2p_barrier(void* const* peer_flags_dev, void* my_flags, int32_t rank, int32_t world, uint32_t epoch,
                    int32_t* timeout_flag_dev, void* stream);
int udb_p2p_copy(void* dst, const void* src, size_t bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Evaluation metrics (reference unidepth/utils/evaluation_depth.py, chamfer_distance.py:59-158, ops/knn with K = 1,
 * norm = 2).  Distances, ratios and rescaled values use the reference's fp32 op order with no FMA contraction; counts
 * are integers and every floating-point sum is an f64 per-CTA partial reduced in a fixed order, so results are
 * deterministic.  Inputs must be finite.  Checked before launch, udb_last_error() naming the argument.  No host sync.
 * ------------------------------------------------------------------------------------------- */

/* Nearest neighbour: for every valid point of x, the squared L2 distance ((dx*dx) + dy*dy) + dz*dz (dx = x - y, each op
 * rounded, as knn_cpu.cpp forms it) to its nearest valid y point and that point's index, ties to the lowest index.
 * x [N, P1, 3], y [N, P2, 3] f32 contiguous; lengths1 / lengths2: [N] int64 on the device or NULL (= P1 / P2), clamped
 * to [0, P] in the kernel.  Rows past lengths1, or of a cloud with lengths2 == 0, get dist = 0 and idx = 0.  With
 * dist_y / idx_y set, the y -> x direction comes from the same pass (both or neither).  idx_x / idx_y double as the
 * packed (dist, idx) accumulators while the kernel runs. */
typedef struct udb_nn_t {
  const float* x;
  const float* y;
  const int64_t* lengths1;
  const int64_t* lengths2;
  int32_t N, P1, P2, pad0;
  float* dist_x;   /* [N, P1] */
  int64_t* idx_x;  /* [N, P1] */
  float* dist_y;   /* [N, P2] or NULL */
  int64_t* idx_y;  /* [N, P2] or NULL */
} udb_nn_t;
int udb_nearest_neighbor(const udb_nn_t* p, void* stream);

/* Most CTAs per image (per cloud) of the metric reductions; partials hold [B, UDB_METRIC_MAX_BLOCKS, nacc] doubles. */
#define UDB_METRIC_MAX_BLOCKS 64

/* Depth metrics of eval_depth over the pixels with mask != 0 and (use_max_depth ? gt <= max_depth : true).
 * gt, pred [B, HW] f32 (pred already resized to gt), mask [B, HW] uint8.  thr_*: the fp32 delta / tau thresholds;
 * auc_thresholds: the UDB_DM_AUC_BINS d_auc thresholds, ascending; medians [B, 2]: median(gt), median(pred) of the
 * valid pixels (si).  out [B, UDB_DM_NACC] f64 (layout below; counts are exact integers), ssi [B, 2] f32: the ssi
 * (scale, shift) solved in f64 from the normal-equation sums with the reference's 1e-9 I stabiliser.  Two passes. */
#define UDB_DM_AUC_BINS 100
enum {
  UDB_DM_N = 0, UDB_DM_D1, UDB_DM_D2, UDB_DM_D3, UDB_DM_TAU,                /* counts of ratio < threshold */
  UDB_DM_SQ, UDB_DM_SQLOG, UDB_DM_AREL, UDB_DM_SQREL, UDB_DM_LOG10,          /* sums of the per-pixel terms */
  UDB_DM_LG, UDB_DM_LG2,                                                     /* sum of log p - log g and of its square */
  UDB_DM_D1_SI, UDB_DM_TAU_SI, UDB_DM_AREL_SI,                               /* si-rescaled counts / sum */
  UDB_DM_PP, UDB_DM_P, UDB_DM_PG, UDB_DM_G,                                  /* ssi normal equations */
  UDB_DM_AUC,                                        /* UDB_DM_AUC_BINS bins: pixels whose first threshold > ratio is k */
  UDB_DM_AREL_SSI = UDB_DM_AUC + UDB_DM_AUC_BINS, UDB_DM_D1_SSI, UDB_DM_TAU_SSI,   /* ssi-rescaled sum / counts */
  UDB_DM_NACC
};
typedef struct udb_depth_metrics_t {
  const float* gt;
  const float* pred;
  const uint8_t* mask;
  int32_t B, pad0;
  int64_t HW;
  float max_depth;
  int32_t use_max_depth;
  float thr_d1, thr_d2, thr_d3, thr_tau;
  const float* auc_thresholds;
  const float* medians;
  double* partials;  /* workspace: [B, UDB_METRIC_MAX_BLOCKS, UDB_DM_NACC] */
  double* out;
  float* ssi;
} udb_depth_metrics_t;
int udb_depth_metrics(const udb_depth_metrics_t* p, void* stream);

/* Point metrics of eval_3d on compacted clouds gt, pred [N, P, 3] f32 with lengths [N] int64 (device, or NULL = P)
 * and the NN distances dist_x (gt -> pred), dist_y (pred -> gt) [N, P].  thresholds: n_thresholds f32, ascending.
 * out [N, 2 + 2 * n_thresholds] f64: [0] sum of |gt - pred|_2, [1] sum of (sqrt(dist_x) + sqrt(dist_y)) / 2, then the
 * histograms of dist_x and of dist_y, bin k counting the points whose first threshold above the distance is k (the
 * count below threshold i is the sum of bins 0..i). */
#define UDB_PM_MAX_THRESHOLDS 1024
typedef struct udb_point_metrics_t {
  const float* gt;
  const float* pred;
  const int64_t* lengths;
  const float* dist_x;
  const float* dist_y;
  const float* thresholds;
  int32_t N, P, n_thresholds, pad0;
  double* partials;  /* workspace: [N, UDB_METRIC_MAX_BLOCKS, 2 + 2 * n_thresholds] */
  double* out;
} udb_point_metrics_t;
int udb_point_metrics(const udb_point_metrics_t* p, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* UDB_H_ */
