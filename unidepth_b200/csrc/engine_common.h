// Shared by the three whole-path engines (engine.cu: UniDepthV2, engine_v1.cu: UniDepthV1, engine_v2old.cu: UniDepthV2old):
// registered weights and prepared shapes, the bump allocator over the caller's workspace, NVTX stage ranges, the launch
// gate, thin wrappers that fill the operator argument structs, the "precision" scalar, and the schedule stages more than
// one engine runs (the DINOv2 patch embedding and block loop, V1's and V2old's decoder blocks, adapters and camera context).
#pragma once
#include <cuda_fp16.h>
#include <math.h>
#include <string.h>

#include <string>
#include <unordered_map>
#include <vector>

#include <nvtx3/nvToolsExt.h>   // header-only NVTX v3: stage ranges for nsys / ncu --nvtx (no-ops when no tool is attached)

#include "common.h"

namespace udb {

// NVTX range per stage of the schedule (host-side: it brackets the enqueue of that stage's kernels)
struct Stage {
  bool open = false;
  void next(const char* name) {
    if (open) nvtxRangePop();
    nvtxRangePushA(name);
    open = true;
  }
  ~Stage() { if (open) nvtxRangePop(); }
};

struct Weight {
  const void* p = nullptr;
  int dtype = 0;
  int ndim = 0;
  int64_t shape[4] = {0, 0, 0, 0};
};

// Registered operands / scalars (what the schedule helpers, Ctx, read) and the prepared shapes of an engine.  `fn` is the
// calling entry point's name, the prefix of every error message.
struct EngineBase {
  std::unordered_map<std::string, Weight> w;
  std::unordered_map<std::string, double> scalars;
  std::unordered_map<std::string, size_t> ws_need;   // prepared shape (as the messages print it) -> workspace bytes

  static int set_weight(EngineBase* e, const char* fn, const char* name, const void* dev_ptr, const int64_t* shape,
                        int32_t ndim, int32_t dtype) {
    if (!e || !name || !dev_ptr || ndim < 0 || ndim > 4) { set_error("%s: bad argument", fn); return 1; }
    if (reinterpret_cast<uintptr_t>(dev_ptr) & 15) { set_error("%s(%s): pointer must be 16-byte aligned", fn, name); return 1; }
    Weight x;
    x.p = dev_ptr; x.dtype = dtype; x.ndim = ndim;
    for (int i = 0; i < ndim; ++i) x.shape[i] = shape[i];
    e->w[name] = x;
    return 0;
  }
  static int set_scalar(EngineBase* e, const char* fn, const char* name, double value) {
    if (!e || !name) { set_error("%s: bad argument", fn); return 1; }
    e->scalars[name] = value;
    return 0;
  }
  // the sizing entry point records the workspace a shape needs; only a recorded shape may be launched, and the size and
  // alignment of the caller's workspace are checked before anything is enqueued
  size_t prepared(const std::string& shape, size_t bytes) { return ws_need[shape] = bytes; }
  int check_workspace(const char* fn, const char* sizing_fn, const std::string& shape, const void* ws, size_t bytes) const {
    auto need = ws_need.find(shape);
    if (need == ws_need.end()) { set_error("%s: shape %s not prepared; call %s first", fn, shape.c_str(), sizing_fn); return 1; }
    if (bytes < need->second) {
      set_error("%s: workspace too small (%zu bytes given, %zu needed)", fn, bytes, need->second);
      return 1;
    }
    if (reinterpret_cast<uintptr_t>(ws) & 255) { set_error("%s: workspace must be 256-byte aligned", fn); return 1; }
    return 0;
  }
};

// Python's v // 2 (the reference's padding arithmetic)
static inline int floordiv2(int v) { return v >= 0 ? v / 2 : -((-v + 1) / 2); }

// result of a CUDA runtime call the engine makes itself (not through an operator) as the engine's return code; the error
// text is `what` + `name` + the CUDA error
static inline int cuda_rc(cudaError_t err, const char* what, const std::string& name = "") {
  if (err == cudaSuccess) return 0;
  set_error("%s%s: %s", what, name.c_str(), cudaGetErrorString(err));
  return 1;
}

// ------------------------------------------------------------------------------------------ arena
struct Arena {
  uintptr_t base;
  size_t cap, off = 0, peak = 0;
  bool dry;
  bool overflow = false;
  Arena(void* p, size_t c) : base(reinterpret_cast<uintptr_t>(p)), cap(c), dry(p == nullptr) {}
  void* alloc(size_t bytes) {
    off = (off + 255) & ~size_t(255);
    const size_t at = off;
    off += bytes;
    if (off > peak) peak = off;
    if (!dry && off > cap) overflow = true;
    return reinterpret_cast<void*>(base + at);
  }
  size_t mark() const { return off; }
  void release(size_t m) { off = m; }
  __half* h(size_t n) { return static_cast<__half*>(alloc(n * 2)); }
  float* f(size_t n) { return static_cast<float*>(alloc(n * 4)); }
};

// ------------------------------------------------------------------------------------------ run context
struct Ctx {
  EngineBase* e;
  Arena* ar;
  void* st;
  bool dry;
  int rc = 0;

  const Weight* W(const std::string& name) {
    auto it = e->w.find(name);
    if (it == e->w.end()) {
      if (!rc) set_error("engine: packed tensor '%s' was not registered (udb_set_weight)", name.c_str());
      rc = 1;
      static const Weight none;
      return &none;
    }
    return &it->second;
  }
  const __half* H(const std::string& n) { return static_cast<const __half*>(W(n)->p); }
  const float* F(const std::string& n) { return static_cast<const float*>(W(n)->p); }
  double S(const std::string& n) {
    auto it = e->scalars.find(n);
    if (it == e->scalars.end()) {
      if (!rc) set_error("engine: scalar '%s' was not registered (udb_set_scalar)", n.c_str());
      rc = 1;
      return 0.0;
    }
    return it->second;
  }
  // The one launch gate: every operator or CUDA call of a schedule is enqueued through here.  A dry run (which only sizes
  // the workspace) and a run that has already failed enqueue nothing; otherwise a non-zero result of the call (an error
  // whose text it has set) is kept.  Operands are looked up before the gate, so that a dry run names a missing one.
  template <class Call>
  void launch(Call&& call) {
    if (dry || rc) return;
    if (const int r = call()) rc = r;
  }
  // registered 2-D operand must have exactly this shape (a mis-packed weight would otherwise be read with the
  // wrong leading dimension and silently produce garbage)
  void expect2(const std::string& name, int64_t rows, int64_t cols) {
    const Weight* w = W(name);
    if (rc) return;
    if (w->ndim != 2 || w->shape[0] != rows || w->shape[1] != cols) {
      set_error("engine: packed tensor '%s' has shape [%lld, %lld] (ndim %d), expected [%lld, %lld]", name.c_str(),
                (long long)w->shape[0], (long long)w->shape[1], w->ndim, (long long)rows, (long long)cols);
      rc = 1;
    }
  }

  // registered 1-D operand (a per-channel scale or bias vector) must have exactly n entries
  void expect1(const std::string& name, int64_t n) {
    const Weight* w = W(name);
    if (rc) return;
    if (w->ndim != 1 || w->shape[0] != n) {
      set_error("engine: packed tensor '%s' has shape [%lld] (ndim %d), expected [%lld]", name.c_str(), (long long)w->shape[0],
                w->ndim, (long long)n);
      rc = 1;
    }
  }

  // registered operand must hold e4m3 bytes (f16 bytes would be read as e4m3 pairs)
  void expect_e4m3(const std::string& name) {
    const Weight* w = W(name);
    if (!rc && w->dtype != UDB_DT_E4M3) {
      set_error("engine: packed tensor '%s' has dtype %d, expected e4m3 (%d)", name.c_str(), w->dtype, UDB_DT_E4M3);
      rc = 1;
    }
  }

  // out[row(m), :] = resid + gamma * act(a @ w^T + bias)     (ops.gemm)
  struct G {
    const void* a; const void* w; int M, N, K; int lda = 0, ldw = 0;
    const float* bias = nullptr; const float* gamma = nullptr; const void* resid = nullptr; int resid_f32 = 0;
    long long ldr = 0; void* out = nullptr; int out_f32 = 0; long long ldc = 0; void* out2 = nullptr; int out2_leaky = 1;
    int act = UDB_ACT_NONE; int rows_per_group = 0, group_stride = 0, row_offset = 0, resid_mod = 0, resid_row_offset = 0;
    int a_split_k = 0, out_split = 0;    // split-f16 precise mode (udb_gemm_t)
    float* ln_stats_out = nullptr; const float* ln_stats_in = nullptr; const float* ln_c1 = nullptr;   // fused LayerNorm (udb_gemm_t.ln_*)
    int ln_parts = 0, ln_part_cols = 0; float ln_eps = 0.f;
    const float* a_scale = nullptr; const float* w_scale = nullptr;   // set: e4m3 operands (udb_gemm_e4m3)
  };
  void gemm(const G& q) {
    udb_gemm_t g;
    memset(&g, 0, sizeof(g));
    g.a = q.a; g.w = q.w; g.M = q.M; g.N = q.N; g.K = q.K;
    g.lda = q.lda ? q.lda : q.K; g.ldw = q.ldw ? q.ldw : q.K;
    g.a_mode = UDB_A_MATRIX;
    g.bias = q.bias; g.gamma = q.gamma;
    g.resid = q.resid; g.resid_f32 = q.resid_f32; g.ldr = q.resid ? (q.ldr ? q.ldr : q.N) : 0;
    g.out = q.out; g.out_f32 = q.out_f32; g.ldc = q.ldc ? q.ldc : q.N;
    g.out2 = q.out2; g.out2_leaky = q.out2_leaky;
    g.act = q.act; g.store_mode = UDB_STORE_ROWS;
    g.rows_per_group = q.rows_per_group; g.group_stride = q.group_stride; g.row_offset = q.row_offset;
    g.resid_mod = q.resid_mod; g.resid_row_offset = q.resid_row_offset;
    g.a_split_k = q.a_split_k; g.out_split = q.out_split;
    g.ln_stats_out = q.ln_stats_out; g.ln_stats_in = q.ln_stats_in; g.ln_c1 = q.ln_c1;
    g.ln_parts = q.ln_parts; g.ln_part_cols = q.ln_part_cols; g.ln_eps = q.ln_eps;
    launch([&] { return q.a_scale ? udb_gemm_e4m3(&g, q.a_scale, q.w_scale, st) : udb_gemm_f16(&g, st); });
  }
  // ConvTranspose2d with kernel == stride == k as a GEMM with a pixel-shuffle store (ops.conv_transpose_ks)
  void conv_transpose(const void* x, int M, int K, const void* w, int k, int cout, int h, int ww, const float* bias,
                      const void* resid, int resid_f32, void* out, int out_f32, void* out2, int out2_leaky, int pad) {
    udb_gemm_t g;
    memset(&g, 0, sizeof(g));
    g.a = x; g.w = w; g.M = M; g.N = k * k * cout; g.K = K; g.lda = K; g.ldw = K;
    g.a_mode = UDB_A_MATRIX;
    g.bias = bias; g.resid = resid; g.resid_f32 = resid_f32;
    g.out = out; g.out_f32 = out_f32; g.ldc = cout; g.out2 = out2; g.out2_leaky = out2_leaky;
    g.store_mode = UDB_STORE_CONVT;
    g.ct_k = k; g.ct_cout = cout; g.ct_h = h; g.ct_w = ww; g.ct_pad = pad;
    launch([&] { return udb_gemm_f16(&g, st); });
  }
  // 3x3 zero-padded convolution over NHWC f16 (ops.conv3x3, tile 8x16)
  void conv3x3(const void* x, int B, int H, int Wd, int C, const void* w, int N, const float* bias, int act,
               const float* gamma, const void* resid, int resid_f32, void* out, int out_f32, void* out2, int out2_leaky) {
    udb_gemm_t g;
    memset(&g, 0, sizeof(g));
    g.a = x; g.w = w; g.M = B * H * Wd; g.N = N; g.K = 9 * C; g.lda = C; g.ldw = 9 * C;
    g.a_mode = UDB_A_CONV3X3;
    g.conv_B = B; g.conv_H = H; g.conv_W = Wd; g.conv_C = C; g.conv_inH = H; g.conv_inW = Wd; g.conv_off = -1;
    g.conv_TH = 8; g.conv_TW = 16; g.conv_cstride = C; g.conv_coff = 0;
    g.bias = bias; g.gamma = gamma; g.act = act; g.store_mode = UDB_STORE_CONVTILE;
    g.out = out; g.out_f32 = out_f32; g.ldc = N;
    g.resid = resid; g.resid_f32 = resid_f32; g.ldr = resid ? N : 0;
    g.out2 = out2; g.out2_leaky = out2_leaky;
    launch([&] { return udb_gemm_f16(&g, st); });
  }
  void conv_halo(const void* x, int B, int H, int Wd, int C, int cstride, int coff, const void* w, int cout,
                 const float* bias, int act, void* out, const float* head_w, float head_b, float head_add, float* head_out) {
    udb_conv_halo_t c;
    memset(&c, 0, sizeof(c));
    c.x = x; c.w = w; c.bias = bias; c.B = B; c.H = H; c.W = Wd; c.C = C; c.cstride = cstride; c.coff = coff;
    c.cout = cout; c.act = act; c.out = out; c.ldc = cout;
    c.head_w = head_w; c.head_b = head_b; c.head_add = head_add; c.head_out = head_out;
    launch([&] { return udb_conv3x3_halo_f16(&c, st); });
  }
  void attention(const void* q, const void* k, const void* v, void* out, int B, int heads, int sq, int sk, int ldq,
                 int ldk, int ldv, int ldo, int q0, int k0, int v0, float scale, int lo_in = 0, int lo_out = 0) {
    udb_attn_t a;
    memset(&a, 0, sizeof(a));
    a.q = q; a.k = k; a.v = v; a.out = out; a.B = B; a.heads = heads; a.seq_q = sq; a.seq_k = sk; a.head_dim = 64;
    a.ldq = ldq; a.ldk = ldk; a.ldv = ldv; a.ldo = ldo; a.q_col0 = q0; a.k_col0 = k0; a.v_col0 = v0; a.o_col0 = 0;
    a.scale = scale;
    if (lo_in) { a.split = 1; a.lo_off_q = a.lo_off_k = a.lo_off_v = lo_in; a.lo_off_o = lo_out; }
    launch([&] { return udb_attention_f16(&a, st); });
  }
  void layernorm(const void* in, int in_f32, void* out, int out_f32, const float* w, const float* b, int rows, int dim,
                 float eps, int rows_per_group = 0, int group_stride = 0, int row_offset = 0, int dim_valid = 0,
                 int out_split = 0) {
    udb_layernorm_t p;
    memset(&p, 0, sizeof(p));
    p.in = in; p.in_f32 = in_f32; p.out = out; p.out_f32 = out_f32; p.weight = w; p.bias = b;
    p.rows = rows; p.dim = dim; p.ld_in = dim; p.ld_out = out_split ? 2 * dim : dim;
    p.rows_per_group = rows_per_group; p.group_stride = group_stride; p.row_offset = row_offset; p.eps = eps;
    p.dim_valid = dim_valid;
    p.out_split = out_split;
    launch([&] { return udb_layernorm(&p, st); });
  }
  // LayerNorm of f32 rows straight to e4m3 bytes + row scales (the A operand of an e4m3 GEMM)
  void layernorm_e4m3(const float* in, void* out, float* scale, const float* w, const float* b, int rows, int dim, float eps) {
    udb_layernorm_t p;
    memset(&p, 0, sizeof(p));
    p.in = in; p.in_f32 = 1; p.out = out; p.weight = w; p.bias = b;
    p.rows = rows; p.dim = dim; p.ld_in = dim; p.ld_out = dim; p.eps = eps;
    launch([&] { return udb_layernorm_e4m3(&p, scale, st); });
  }
  // f16 rows -> dense e4m3 rows + row scales
  void quantize_e4m3(const __half* in, long long ld_in, void* out, float* scale, int rows, int cols) {
    launch([&] { return udb_quantize_rows_e4m3(in, ld_in, out, cols, scale, rows, cols, st); });
  }
  // LayerNorm for any width that is a multiple of 64, with the optional added term and space-to-depth store (UniDepthV1)
  void ln_any(const void* in, int in_f32, void* out, int out_f32, const float* w, const float* b, long long rows, int dim,
              float eps, long long ld_out = 0, const float* add = nullptr, long long add_mod = 0, int s2d_h = 0,
              int s2d_w = 0) {
    udb_layernorm_any_t p;
    memset(&p, 0, sizeof(p));
    p.in = in; p.in_f32 = in_f32; p.out = out; p.out_f32 = out_f32; p.weight = w; p.bias = b;
    p.rows = rows; p.dim = dim; p.ld_in = dim; p.ld_out = ld_out ? ld_out : dim; p.eps = eps;
    p.add = add; p.add_mod = add_mod; p.s2d_h = s2d_h; p.s2d_w = s2d_w;
    launch([&] { return udb_layernorm_any(&p, st); });
  }
  void small_linear(const float* x, int M, int K, const float* w, int N, const float* bias, int act, const float* gamma,
                    const float* resid, float* y, int ldx = 0, int ldy = 0, int ldr = 0) {
    udb_small_linear_t p;
    memset(&p, 0, sizeof(p));
    p.x = x; p.w = w; p.bias = bias; p.gamma = gamma; p.resid = resid; p.y = y; p.M = M; p.N = N; p.K = K; p.act = act;
    p.ldx = ldx ? ldx : K; p.ldy = ldy ? ldy : N; p.ldr = resid ? (ldr ? ldr : N) : 0;
    launch([&] { return udb_small_linear_f32(&p, st); });
  }
};

// The "precision" scalar: 0 (absent) f16 operands; 1 split-f16 operands (parity mode: [hi | lo] operand pairs times
// [hi | hi | lo] weights, see each engine for the GEMMs it covers); 2 e4m3 operands for the encoder blocks.  Any other
// value is refused, and so is precision 1 when `weight`, the encoder's first GEMM weight, does not have the split
// packing's `split_cols` columns: an f16 packing is named for what it is, not only by its first mis-shaped operand.  `fn`,
// the calling entry point, prefixes the message; PREC_BAD means the error is set.
enum Precision { PREC_BAD = -1, PREC_F16 = 0, PREC_SPLIT = 1, PREC_E4M3 = 2 };
static inline Precision encoder_precision(Ctx& c, const char* fn, const char* weight, int64_t split_cols) {
  const auto it = c.e->scalars.find("precision");
  const double p = it == c.e->scalars.end() ? 0.0 : it->second;
  if (p != 0.0 && p != 1.0 && p != 2.0) { set_error("%s: precision %g unsupported (0 f16, 1 split f16, 2 e4m3)", fn, p); return PREC_BAD; }
  if (p == 1.0) {
    const Weight* w = c.W(weight);
    if (c.rc) return PREC_BAD;
    if (w->ndim != 2 || w->shape[1] != split_cols) {
      set_error("%s: precision 1 (split f16) needs the split packing: '%s' has %lld columns, expected %lld", fn, weight,
                static_cast<long long>(w->shape[1]), static_cast<long long>(split_cols));
      return PREC_BAD;
    }
  }
  return static_cast<Precision>(static_cast<int>(p));
}

// LN -> Linear -> GELU -> Linear (+ gamma, + residual), fp32, camera head (layers/mlp.py:9-35)
static inline float* cam_mlp(Ctx& c, const std::string& pre, const float* x, int rows, int hid, int mid, int out_dim,
                      const float* resid, const float* gamma) {
  float* y = c.ar->f(static_cast<size_t>(rows) * hid);
  c.layernorm(x, 1, y, 1, c.F(pre + ".nw"), c.F(pre + ".nb"), rows, hid, 1e-5f);
  float* z = c.ar->f(static_cast<size_t>(rows) * mid);
  c.small_linear(y, rows, hid, c.F(pre + ".w1"), mid, c.F(pre + ".b1"), UDB_ACT_GELU, nullptr, nullptr, z);
  float* o = c.ar->f(static_cast<size_t>(rows) * out_dim);
  c.small_linear(z, rows, mid, c.F(pre + ".w2"), out_dim, c.F(pre + ".b2"), UDB_ACT_NONE, gamma, resid, o);
  return o;
}

static inline std::string idx(const char* fmt, int i) {
  char b[64];
  snprintf(b, sizeof(b), fmt, i);
  return b;
}
static inline std::string idx2(const char* fmt, int i, int j) {
  char b[64];
  snprintf(b, sizeof(b), fmt, i, j);
  return b;
}
// a batch shape B x H x W as the prepared-shape table stores it and the error messages print it
static inline std::string shape_name(int B, int H, int W) {
  char b[64];
  snprintf(b, sizeof(b), "%dx%dx%d", B, H, W);
  return b;
}

// ------------------------------------------------------------------------------------------ decoder blocks
// Shared by the UniDepthV1 and UniDepthV2old decoders (layers/{attention,nystrom_attention,mlp,convnext}.py).
// LayerNorm to f16 for any decoder / encoder width: the V2 kernels where they apply (128-multiples up to 1024 from f32,
// 64/128/256 from f16), the generic one otherwise
static inline void ln16(Ctx& c, const void* in, int in_f32, void* out, const std::string& wn, const std::string& bn, long long rows,
                 int dim, float eps) {
  const bool v2_ok = in_f32 ? (dim % 128 == 0 && dim <= 1024) : (dim == 64 || dim == 128 || dim == 256 || (dim % 128 == 0 && dim <= 1024));
  if (v2_ok) c.layernorm(in, in_f32, out, 0, c.F(wn), c.F(bn), static_cast<int>(rows), dim, eps);
  else c.ln_any(in, in_f32, out, 0, c.F(wn), c.F(bn), rows, dim, eps);
}

// MLP tail on the f32 residual stream x [rows, C]:  x += gamma * (W2 gelu(W1 LN(x) + b1) + b2)        (layers/mlp.py:9-35)
static inline void mlp_resid(Ctx& c, const std::string& p, float* x, long long rows, int C, int mid, const float* gamma,
                      __half* x16 = nullptr) {
  Arena& ar = *c.ar;
  const size_t m = ar.mark();
  __half* hN = ar.h(rows * C);
  __half* md = ar.h(rows * mid);
  ln16(c, x, 1, hN, p + "nw", p + "nb", rows, C, 1e-5f);
  { Ctx::G q{hN, c.H(p + "w1"), static_cast<int>(rows), mid, C}; q.bias = c.F(p + "b1"); q.act = UDB_ACT_GELU; q.out = md; c.gemm(q); }
  { Ctx::G q{md, c.H(p + "w2"), static_cast<int>(rows), C, mid}; q.bias = c.F(p + "b2"); q.gamma = gamma; q.resid = x; q.resid_f32 = 1;
    q.out = x; q.out_f32 = 1; q.out2 = x16; q.out2_leaky = 0; c.gemm(q); }
  ar.release(m);
}

// ConvNeXt-style block on an NHWC map: x f32 (+ its f16 copy x16) [B,H,W,C] updated in place
// (convnext.py:208-223 with eps 1e-6; layers/convnext.py:34-44 with eps 1e-5)
static inline void cvnxt_block(Ctx& c, const std::string& p, float* x, __half* x16, int B, int Hh, int Ww, int C, float eps) {
  Arena& ar = *c.ar;
  const size_t m = ar.mark();
  const long long rows = static_cast<long long>(B) * Hh * Ww;
  __half* y = ar.h(rows * C);
  __half* hN = ar.h(rows * C);
  __half* md = ar.h(rows * 4 * C);
  const float* dw_w = c.F(p + "dw_w");
  const float* dw_b = c.F(p + "dw_b");
  c.launch([&] { return udb_dwconv7_nhwc_f16(x16, dw_w, dw_b, y, B, Hh, Ww, C, c.st); });
  ln16(c, y, 0, hN, p + "ln_w", p + "ln_b", rows, C, eps);
  { Ctx::G q{hN, c.H(p + "w1"), static_cast<int>(rows), 4 * C, C}; q.bias = c.F(p + "b1"); q.act = UDB_ACT_GELU; q.out = md; c.gemm(q); }
  { Ctx::G q{md, c.H(p + "w2"), static_cast<int>(rows), C, 4 * C}; q.bias = c.F(p + "b2"); q.gamma = c.F(p + "gamma"); q.resid = x;
    q.resid_f32 = 1; q.out = x; q.out_f32 = 1; q.out2 = x16; q.out2_leaky = 0; c.gemm(q); }
  ar.release(m);
}

static inline long long rup(long long v, long long m) { return (v + m - 1) / m * m; }

// Single-head (head dim = D) attention block with a separate context (decoder.py:225-236 aggregate_16 / prompt_camera),
// computed densely: S = q k^T (GEMM) -> row softmax -> P v (GEMM with v^T as the K-major operand).
static inline void dense_attn_block(Ctx& c, const std::string& p, float* x, int B, int nq, int D, const void* ctx, int ctx_f32, int nk,
                             const float* pos_ctx) {
  Arena& ar = *c.ar;
  const size_t m = ar.mark();
  const long long Rq = static_cast<long long>(B) * nq, Rk = static_cast<long long>(B) * nk;
  const int kp = static_cast<int>(rup(nk, 64));
  __half* xn = ar.h(Rq * D);
  __half* cn = ar.h((Rk + 64) * D);
  ln16(c, x, 1, xn, p + "nxw", p + "nxb", Rq, D, 1e-5f);
  ln16(c, ctx, ctx_f32, cn, p + "ncw", p + "ncb", Rk, D, 1e-5f);
  c.launch([&] {
    return cuda_rc(cudaMemsetAsync(cn + Rk * D, 0, sizeof(__half) * 64 * D, static_cast<cudaStream_t>(c.st)),
                   "engine: zeroing the padding rows of the normalised context of ", p);
  });
  __half* q = ar.h(Rq * D);
  { Ctx::G g{xn, c.H(p + "q_w"), static_cast<int>(Rq), D, D}; g.bias = c.F(p + "q_b"); g.out = q; c.gemm(g); }
  __half* k = ar.h(static_cast<long long>(B) * kp * D);
  c.launch([&] {
    return cuda_rc(cudaMemsetAsync(k, 0, sizeof(__half) * B * kp * D, static_cast<cudaStream_t>(c.st)),
                   "engine: zeroing the padded keys of ", p);
  });
  { Ctx::G g{cn, c.H(p + "k_w"), static_cast<int>(Rk), D, D}; g.bias = c.F(p + "k_b"); g.out = k;
    g.rows_per_group = nk; g.group_stride = kp; g.row_offset = 0;
    if (pos_ctx) { g.resid = pos_ctx; g.resid_f32 = 1; g.ldr = D; g.resid_mod = nk; g.resid_row_offset = 0; }
    c.gemm(g); }
  __half* vt = ar.h(static_cast<long long>(B) * D * kp);
  float* S = ar.f(static_cast<long long>(nq) * kp);
  __half* P = ar.h(static_cast<long long>(nq) * kp);
  __half* o = ar.h(Rq * D);
  const float scale = 1.0f / sqrtf(static_cast<float>(D));
  for (int b = 0; b < B; ++b) {
    // v^T [D, kp] = W_v . ctx_b^T  (the value bias is added after P v: softmax rows sum to 1)
    { Ctx::G g{c.H(p + "v_w"), cn + static_cast<long long>(b) * nk * D, D, kp, D}; g.out = vt + static_cast<long long>(b) * D * kp; c.gemm(g); }
    { Ctx::G g{q + static_cast<long long>(b) * nq * D, k + static_cast<long long>(b) * kp * D, nq, kp, D}; g.out = S; g.out_f32 = 1; c.gemm(g); }
    c.launch([&] { return udb_softmax_rows(S, P, nq, nk, kp, kp, scale, c.st); });
    { Ctx::G g{P, vt + static_cast<long long>(b) * D * kp, nq, D, kp}; g.bias = c.F(p + "v_b"); g.out = o + static_cast<long long>(b) * nq * D; c.gemm(g); }
  }
  { Ctx::G g{o, c.H(p + "out_w"), static_cast<int>(Rq), D, D}; g.bias = c.F(p + "out_b"); g.gamma = c.F(p + "ls1"); g.resid = x; g.resid_f32 = 1;
    g.out = x; g.out_f32 = 1; c.gemm(g); }
  ar.release(m);
  mlp_resid(c, p + "m", x, Rq, D, 4 * D, c.F(p + "ls2"));
}

// Multi-head self-attention block with 64-wide heads and a positional term added to q (decoder.py:239-241,256-258,271-273):
// exact attention (AttentionBlock) or the Nystrom approximation with 128 landmarks (NystromBlock).
static inline void mh_attn_block(Ctx& c, const std::string& p, float* x, int B, int n, int C, int heads, const float* pos, bool nystrom) {
  Arena& ar = *c.ar;
  const size_t m = ar.mark();
  const long long R = static_cast<long long>(B) * n;
  __half* xn = ar.h(R * C);
  __half* cn = ar.h(R * C);
  ln16(c, x, 1, xn, p + "nxw", p + "nxb", R, C, 1e-5f);
  ln16(c, x, 1, cn, p + "ncw", p + "ncb", R, C, 1e-5f);
  __half* q = ar.h(R * C);
  { Ctx::G g{xn, c.H(p + "q_w"), static_cast<int>(R), C, C}; g.bias = c.F(p + "q_b"); g.resid = pos; g.resid_f32 = 1; g.out = q; c.gemm(g); }
  __half* kv = ar.h(R * 2 * C);
  { Ctx::G g{cn, c.H(p + "kv_w"), static_cast<int>(R), 2 * C, C}; g.bias = c.F(p + "kv_b"); g.out = kv; c.gemm(g); }
  __half* o = ar.h(R * C);
  if (!nystrom) {
    c.attention(q, kv, kv, o, B, heads, n, n, C, 2 * C, 2 * C, C, 0, 0, C, 0.125f);
  } else {
    const long long L = static_cast<long long>(B) * 128, mm = static_cast<long long>(B) * heads * 128 * 128;
    __half* lm = ar.h(L * 2 * C);          // (q landmarks | k landmarks)
    float* k2 = ar.f(mm);
    float* z = ar.f(mm);
    float* tmp = ar.f(3 * mm);
    __half* k3 = ar.h(L * C);
    __half* w2 = ar.h(L * C);
    c.launch([&] { return udb_nystrom_landmarks(q, C, kv, 2 * C, lm, B, n, heads, c.st); });
    c.launch([&] { return udb_nystrom_k2_pinv(lm, k2, z, tmp, B, heads, 6, c.st); });
    c.attention(lm, kv, kv, k3, B, heads, 128, n, 2 * C, 2 * C, 2 * C, C, 0, 0, C, 0.125f);        // softmax(ql k^T) v
    c.launch([&] { return udb_nystrom_zk3(z, k3, C, w2, C, B, heads, c.st); });           // pinv . kernel_3
    c.attention(q, lm, w2, o, B, heads, n, 128, C, 2 * C, C, C, 0, C, 0, 0.125f);                  // softmax(q kl^T) (pinv kernel_3)
  }
  { Ctx::G g{o, c.H(p + "out_w"), static_cast<int>(R), C, C}; g.bias = c.F(p + "out_b"); g.gamma = c.F(p + "ls1"); g.resid = x; g.resid_f32 = 1;
    g.out = x; g.out_f32 = 1; c.gemm(g); }
  ar.release(m);
  mlp_resid(c, p + "m", x, R, C, 4 * C, c.F(p + "ls2"));
}

// The four input adapters (decoder.py:395-408, decoder_old.py:448-461).  Level l, [B, sh[l], sw[l], dims[l]] f16 (f32 in
// split mode), is resized (antialiased) to the common grid hc x wc when its own grid differs, then LayerNorm -> Linear ->
// GELU writes it twice: rows [l*nq, (l+1)*nq) of each image in tokens [B, 4*nq, hid] and columns [l*hid, (l+1)*hid) of
// featcat [B*nq, 4*hid].  Split mode (`sp`): the LayerNorm writes a [hi | lo] operand whose hi half those two GEMMs read,
// and the heads' copy of the tokens multiplies the whole operand with "adapt.<l>.w_cam" [hid, 3*C], into head_f32 (f32
// rows) and head_split ([hi | lo] rows), each where non-null.
static inline void adapters(Ctx& c, void* const* levels, const int* dims, const int* sh, const int* sw, int B, int hc, int wc,
                            int hid, bool sp, __half* tokens, __half* featcat, float* head_f32, __half* head_split) {
  Arena& ar = *c.ar;
  const int nq = hc * wc, sx = sp ? 2 : 1;
  const long long Rq = static_cast<long long>(B) * nq;
  for (int l = 0; l < 4; ++l) {
    const size_t m = ar.mark();
    const int C = dims[l];
    const void* src = levels[l];
    if (sh[l] != hc || sw[l] != wc) {
      void* r = ar.alloc(Rq * C * (sp ? 4 : 2));
      c.launch([&] {
        return sp ? udb_aa_resize_nhwc_f32(static_cast<const float*>(levels[l]), static_cast<float*>(r), B, sh[l], sw[l], C, hc, wc, c.st)
                  : udb_aa_resize_nhwc_f16(levels[l], r, B, sh[l], sw[l], C, hc, wc, c.st);
      });
      src = r;
    }
    const std::string ad = idx("adapt.%d.", l);
    __half* an = ar.h(Rq * C * sx);
    if (sp) c.ln_any(src, 1, an, UDB_LN_OUT_SPLIT, c.F(ad + "ln_w"), c.F(ad + "ln_b"), Rq, C, 1e-5f, 2 * C);
    else ln16(c, src, 0, an, ad + "ln_w", ad + "ln_b", Rq, C, 1e-5f);
    { Ctx::G q{an, c.H(ad + "w"), static_cast<int>(Rq), hid, C}; q.lda = C * sx; q.bias = c.F(ad + "b"); q.act = UDB_ACT_GELU; q.out = tokens;
      q.rows_per_group = nq; q.group_stride = 4 * nq; q.row_offset = l * nq; c.gemm(q); }
    { Ctx::G q{an, c.H(ad + "w"), static_cast<int>(Rq), hid, C}; q.lda = C * sx; q.bias = c.F(ad + "b"); q.act = UDB_ACT_GELU;
      q.out = featcat + l * hid; q.ldc = 4 * hid; c.gemm(q); }
    void* const head[2] = {head_f32, head_split};
    if (head[0] || head[1]) c.expect2(ad + "w_cam", hid, 3 * C);
    for (int k = 0; k < 2; ++k) {
      if (!head[k]) continue;
      Ctx::G q{an, c.H(ad + "w_cam"), static_cast<int>(Rq), hid, 3 * C}; q.lda = 2 * C; q.a_split_k = C; q.bias = c.F(ad + "b");
      q.act = UDB_ACT_GELU; q.rows_per_group = nq; q.group_stride = 4 * nq; q.row_offset = l * nq; q.out = head[k];
      if (k == 0) q.out_f32 = 1;
      else { q.ldc = 2 * hid; q.out_split = hid; }
      c.gemm(q);
    }
    ar.release(m);
  }
}

// The n cls tokens cls[i], f32 [B, dims[i]] -> LN + Linear + GELU per token (ListAdapter, decoder.py:395-408,
// decoder_old.py:13-29) -> f32 [B, n, hid]
static inline float* token_adapter(Ctx& c, const std::string& p, float* const* cls, const int* dims, int n, int B, int hid) {
  float* toks = c.ar->f(static_cast<size_t>(B) * n * hid);
  for (int i = 0; i < n; ++i) {
    const std::string tk = p + idx("%d.", i);
    const int D = dims[i];
    float* t = c.ar->f(static_cast<size_t>(B) * D);
    c.ln_any(cls[i], 1, t, 1, c.F(tk + "ln_w"), c.F(tk + "ln_b"), B, D, 1e-5f);
    c.small_linear(t, B, D, c.F(tk + "w"), hid, c.F(tk + "b"), UDB_ACT_GELU, nullptr, nullptr, toks + i * hid, D, n * hid, 0);
  }
  return toks;
}

// The n head tokens x f32 [B*n, hid] into rows [row0, row0 + n) of each image's nk context rows: f16, or f32 in split mode
static inline void copy_cls_rows(Ctx& c, const float* x, void* ctx, int B, int n, int hid, long long nk, long long row0, bool sp) {
  c.launch([&] {
    if (!sp) return udb_copy_rows_f32_to_f16(x, ctx, B, n, hid, nk, row0, c.st);
    const size_t row = sizeof(float) * hid;
    return cuda_rc(cudaMemcpy2DAsync(static_cast<float*>(ctx) + row0 * hid, nk * row, x, n * row, n * row, B,
                                     cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(c.st)),
                   "engine: copying the head tokens into the f32 context");
  });
}

// The camera head's context (decoder.py:311-343, decoder_old.py:378-406), 4*nq + n rows per image: in_features (LN ->
// Linear -> GELU -> Linear) of tokens + tokens_pos [4*nq, hid] into the first 4*nq, then the n head tokens x f32 [B*n, hid]
// after them.  f16 from the f16 tokens; split mode (`sp`): from the f32 head tokens through [hi | lo] operands and
// [N, 3K] weights into f32 rows.  The context is allocated before the scratch of in_features, which is released.
static inline void* camera_context(Ctx& c, const void* tokens, const float* tokens_pos, const float* x, int B, int nq, int n,
                                   int hid, bool sp) {
  Arena& ar = *c.ar;
  const long long Rt = 4LL * B * nq, nk = 4LL * nq + n;
  const int sx = sp ? 2 : 1, kx = sp ? 3 : 1;
  void* ctx = ar.alloc(B * nk * hid * (sp ? 4 : 2));
  const size_t m = ar.mark();
  __half* a1 = ar.h(Rt * hid * sx);
  __half* m1 = ar.h(Rt * 2 * hid * sx);
  if (sp) {
    c.expect2("cam.inf.w1", 2 * hid, 3 * hid);
    c.expect2("cam.inf.w2", hid, 6 * hid);
  }
  c.ln_any(tokens, sp ? 1 : 0, a1, sp ? UDB_LN_OUT_SPLIT : 0, c.F("cam.inf.nw"), c.F("cam.inf.nb"), Rt, hid, 1e-5f, sp ? 2 * hid : 0,
           tokens_pos, 4LL * nq);
  { Ctx::G q{a1, c.H("cam.inf.w1"), static_cast<int>(Rt), 2 * hid, hid * kx}; q.lda = hid * sx; q.a_split_k = sp ? hid : 0;
    q.bias = c.F("cam.inf.b1"); q.act = UDB_ACT_GELU; q.out = m1; q.ldc = 2 * hid * sx; q.out_split = sp ? 2 * hid : 0; c.gemm(q); }
  { Ctx::G q{m1, c.H("cam.inf.w2"), static_cast<int>(Rt), hid, 2 * hid * kx}; q.lda = 2 * hid * sx; q.a_split_k = sp ? 2 * hid : 0;
    q.bias = c.F("cam.inf.b2"); q.out = ctx; q.out_f32 = sp ? 1 : 0; q.rows_per_group = 4 * nq; q.group_stride = static_cast<int>(nk);
    q.row_offset = 0; c.gemm(q); }
  ar.release(m);
  copy_cls_rows(c, x, ctx, B, n, hid, nk, 4LL * nq, sp);
  return ctx;
}

// AttentionBlock with one head over a long context and at most four queries (decoder.py:225-236, decoder_old.py:72-77,
// 142-143): the heads' aggregate blocks, on the split-key cross attention.  x f32 [B*nq, hid] -> new f32 rows.  f16
// context; split mode (`sp`): the context is f32, its LayerNorm writes a split operand for the kv GEMM ([2*hid, 3*hid]
// weight), and the attention reads f32 (k | v) rows.
static inline float* small_cross_block(Ctx& c, const std::string& p, const float* x, int B, int nq, const void* ctx, long long nk,
                                       const float* q_pos, int hid, int expansion, bool sp) {
  Arena& ar = *c.ar;
  const int R = B * nq;
  const long long Rc = static_cast<long long>(B) * nk;
  float* xn = ar.f(static_cast<size_t>(R) * hid);
  float* q = ar.f(static_cast<size_t>(R) * hid);
  float* at = ar.f(static_cast<size_t>(R) * hid);
  float* scratch = ar.f(static_cast<size_t>(B) * 16 * 4 * (hid + 2));
  c.layernorm(x, 1, xn, 1, c.F(p + "nxw"), c.F(p + "nxb"), R, hid, 1e-5f);
  c.small_linear(xn, R, hid, c.F(p + "q_w"), hid, c.F(p + "q_b"), UDB_ACT_NONE, nullptr, nullptr, q);
  const size_t m = ar.mark();          // the normalised context and its (k | v) rows: dead once the attention has run
  void* kv;
  if (sp) {
    __half* cn = ar.h(Rc * 2 * hid);
    c.ln_any(ctx, 1, cn, UDB_LN_OUT_SPLIT, c.F(p + "ncw"), c.F(p + "ncb"), Rc, hid, 1e-5f, 2 * hid);
    kv = ar.f(Rc * 2 * hid);
    c.expect2(p + "kv_w", 2 * hid, 3 * hid);
    Ctx::G g{cn, c.H(p + "kv_w"), static_cast<int>(Rc), 2 * hid, 3 * hid}; g.lda = 2 * hid; g.a_split_k = hid;
    g.bias = c.F(p + "kv_b"); g.out = kv; g.out_f32 = 1; c.gemm(g);
  } else {
    __half* cn = ar.h(Rc * hid);
    ln16(c, ctx, 0, cn, p + "ncw", p + "ncb", Rc, hid, 1e-5f);
    kv = ar.h(Rc * 2 * hid);
    Ctx::G g{cn, c.H(p + "kv_w"), static_cast<int>(Rc), 2 * hid, hid}; g.bias = c.F(p + "kv_b"); g.out = kv; c.gemm(g);
  }
  c.launch([&] {
    const float scale = 1.0f / sqrtf(static_cast<float>(hid));
    return sp ? udb_cross_attn_small_f32(q, q_pos, static_cast<const float*>(kv), at, scratch, B, nq, static_cast<int>(nk), hid, scale, c.st)
              : udb_cross_attn_small(q, q_pos, kv, at, scratch, B, nq, static_cast<int>(nk), hid, scale, c.st);
  });
  ar.release(m);
  float* t2 = xn;
  c.small_linear(at, R, hid, c.F(p + "out_w"), hid, c.F(p + "out_b"), UDB_ACT_NONE, c.F(p + "ls1"), x, t2);
  return cam_mlp(c, p + "mlp", t2, R, hid, expansion * hid, hid, t2, c.F(p + "ls2"));
}

// ------------------------------------------------------------------------------------------ DINOv2 blocks
// Shape and packing mode of the DINOv2 block loop (UniDepthV2 uses every mode; UniDepthV1 ViT-L the f16 and e4m3 ones).
struct VitBlocks {
  int B, T, D, heads, depth;
  bool split = false;          // split-f16 precise mode: operands are [hi | lo] pairs, weights [N, 3K] = [hi | hi | lo]
  bool fuse = false;           // fused LayerNorm: norm1 / norm2 folded into qkv / fc1 (udb_gemm_t.ln_*)
  bool fp8 = false;            // e4m3 mode: qkv / proj / fc1 / fc2 on e4m3 operands with per-row / per-channel scales
  __half* x16 = nullptr;       // fused mode: f16 copy of x and its per-part LayerNorm statistics, kept up to date by the
  float* stats = nullptr;      // GEMMs that write x (the patch embedding included)
  int ln_parts = 0, ln_pc = 0;
};

// DINOv2 patch embedding (dinov2.py:306-347) in the block loop's mode `v`: the patch GEMM of the B*N pre-processed patch
// rows (N = T - 1; [hi | lo] rows and a [D, 3*640] weight in split mode) into rows 1..N of each image's T rows of the f32
// residual stream x, with the position table pos [T, D] (cls row first) as row-mapped residual, then the cls rows
// (cls + pos[0]).  In the fused mode both also write the f16 copy of x and its LayerNorm statistics.
static inline void vit_embed(Ctx& c, const __half* patches, const float* pos, float* x, const VitBlocks& v) {
  const int B = v.B, T = v.T, D = v.D, N = T - 1, K = v.split ? 3 * 640 : 640;
  c.expect2("patch_w", D, K);
  Ctx::G q{patches, c.H("patch_w"), B * N, D, K};
  q.lda = v.split ? 2 * 640 : 640; q.a_split_k = v.split ? 640 : 0;
  q.bias = c.F("patch_b"); q.resid = pos; q.resid_f32 = 1; q.ldr = D; q.out = x; q.out_f32 = 1;
  q.rows_per_group = N; q.group_stride = T; q.row_offset = 1; q.resid_mod = N; q.resid_row_offset = 1;
  if (v.fuse) { q.out2 = v.x16; q.out2_leaky = 0; q.ln_stats_out = v.stats; q.ln_parts = v.ln_parts; q.ln_part_cols = v.ln_pc; }
  c.gemm(q);
  const float* cls = c.F("cls");
  c.launch([&] {
    return v.fuse ? udb_set_cls_rows_ln(x, v.x16, v.stats, cls, pos, B, T, D, v.ln_parts, v.ln_pc, c.st)
                  : udb_set_cls_rows(x, cls, pos, B, T, D, c.st);
  });
}

// One block in e4m3 mode: each of the four linear layers reads an e4m3 copy of its input (LayerNorm or row quantiser,
// one scale per row) and e4m3 weights with one scale per output channel; attention and the epilogues are those of the
// f16 mode.  `q8` / `qs` hold the current GEMM's A operand and row scales; the stream orders their reuse.
static inline void vit_block_e4m3(Ctx& c, const std::string& b, float* x, const VitBlocks& v, __half* qkv, __half* att,
                                  __half* mid, void* q8, float* qs) {
  const int D = v.D, BT = v.B * v.T;
  c.expect2(b + "qkv_w8", 3 * D, D);
  c.expect2(b + "proj_w8", D, D);
  c.expect2(b + "fc1_w8", 4 * D, D);
  c.expect2(b + "fc2_w8", D, 4 * D);
  for (const char* n : {"qkv_w8", "proj_w8", "fc1_w8", "fc2_w8"}) c.expect_e4m3(b + n);
  c.expect1(b + "qkv_w8s", 3 * D);
  c.expect1(b + "proj_w8s", D);
  c.expect1(b + "fc1_w8s", 4 * D);
  c.expect1(b + "fc2_w8s", D);
  c.layernorm_e4m3(x, q8, qs, c.F(b + "n1w"), c.F(b + "n1b"), BT, D, 1e-6f);
  { Ctx::G q{q8, c.W(b + "qkv_w8")->p, BT, 3 * D, D}; q.a_scale = qs; q.w_scale = c.F(b + "qkv_w8s");
    q.bias = c.F(b + "qkv_b"); q.out = qkv; c.gemm(q); }
  c.attention(qkv, qkv, qkv, att, v.B, v.heads, v.T, v.T, 3 * D, 3 * D, 3 * D, D, 0, D, 2 * D, 0.125f);
  c.quantize_e4m3(att, D, q8, qs, BT, D);
  { Ctx::G q{q8, c.W(b + "proj_w8")->p, BT, D, D}; q.a_scale = qs; q.w_scale = c.F(b + "proj_w8s");
    q.bias = c.F(b + "proj_b"); q.gamma = c.F(b + "ls1"); q.resid = x; q.resid_f32 = 1; q.out = x; q.out_f32 = 1; c.gemm(q); }
  c.layernorm_e4m3(x, q8, qs, c.F(b + "n2w"), c.F(b + "n2b"), BT, D, 1e-6f);
  { Ctx::G q{q8, c.W(b + "fc1_w8")->p, BT, 4 * D, D}; q.a_scale = qs; q.w_scale = c.F(b + "fc1_w8s");
    q.bias = c.F(b + "fc1_b"); q.act = UDB_ACT_GELU; q.out = mid; c.gemm(q); }
  c.quantize_e4m3(mid, 4 * D, q8, qs, BT, 4 * D);
  { Ctx::G q{q8, c.W(b + "fc2_w8")->p, BT, D, 4 * D}; q.a_scale = qs; q.w_scale = c.F(b + "fc2_w8s");
    q.bias = c.F(b + "fc2_b"); q.gamma = c.F(b + "ls2"); q.resid = x; q.resid_f32 = 1; q.out = x; q.out_f32 = 1; c.gemm(q); }
}

// `depth` pre-norm transformer blocks (metadinov2/block.py:84-109, LayerNorm eps 1e-6) on the f32 residual stream
// x [B*T, D], weights "<prefix><i>.<operand>" as _pack.pack_vit_encoder packs them.  after_block(i) runs once block
// i has updated x (the engines read their encoder outputs there).  The scratch it allocates is released on return.
template <class Hook>
static inline void vit_blocks(Ctx& c, const std::string& prefix, float* x, const VitBlocks& v, Hook&& after_block) {
  Arena& ar = *c.ar;
  const int D = v.D;
  const size_t BT = static_cast<size_t>(v.B) * v.T;
  const bool sp = v.split, fuse = v.fuse;
  const int sx = sp ? 2 : 1;
  __half* x16 = v.x16;
  float* stats = v.stats;
  const int ln_parts = v.ln_parts, ln_pc = v.ln_pc;
  const size_t m = ar.mark();
  __half* h = (fuse || v.fp8) ? nullptr : ar.h(BT * D * sx);
  __half* qkv = ar.h(BT * 3 * D * sx);
  __half* att = ar.h(BT * D * sx);
  __half* mid = ar.h(BT * 4 * D * sx);
  void* q8 = v.fp8 ? ar.alloc(BT * 4 * D) : nullptr;   // e4m3 mode: A operand (up to 4D bytes per row) and row scales
  float* qs = v.fp8 ? ar.f(BT) : nullptr;
  const int kx = sp ? 3 : 1;          // logical K multiplier of a split operand
  for (int i = 0; i < v.depth; ++i) {
    const std::string b = prefix + idx("%d.", i);
    if (v.fp8) {
      vit_block_e4m3(c, b, x, v, qkv, att, mid, q8, qs);
      after_block(i);
      continue;
    }
    // a weight packed for another mode (or transposed) must be refused, not read with the wrong leading dimension
    c.expect2(b + (fuse ? "qkv_wf" : "qkv_w"), 3 * D, D * kx);
    c.expect2(b + (fuse ? "fc1_wf" : "fc1_w"), 4 * D, D * kx);
    c.expect2(b + "proj_w", D, D * kx);
    c.expect2(b + "fc2_w", D, 4 * D * kx);
    if (fuse) {
      Ctx::G q{x16, c.H(b + "qkv_wf"), static_cast<int>(BT), 3 * D, D};
      q.bias = c.F(b + "qkv_c2"); q.ln_stats_in = stats; q.ln_c1 = c.F(b + "qkv_c1"); q.ln_parts = ln_parts; q.ln_part_cols = ln_pc;
      q.ln_eps = 1e-6f; q.out = qkv; c.gemm(q);
    } else {
      c.layernorm(x, 1, h, 0, c.F(b + "n1w"), c.F(b + "n1b"), static_cast<int>(BT), D, 1e-6f, 0, 0, 0, 0, sp ? D : 0);
      Ctx::G q{h, c.H(b + "qkv_w"), static_cast<int>(BT), 3 * D, D * kx}; q.lda = D * sx; q.a_split_k = sp ? D : 0;
      q.bias = c.F(b + "qkv_b"); q.out = qkv; q.ldc = 3 * D * sx; q.out_split = sp ? 3 * D : 0; c.gemm(q);
    }
    c.attention(qkv, qkv, qkv, att, v.B, v.heads, v.T, v.T, 3 * D * sx, 3 * D * sx, 3 * D * sx, D * sx, 0, D, 2 * D, 0.125f,
                sp ? 3 * D : 0, sp ? D : 0);
    { Ctx::G q{att, c.H(b + "proj_w"), static_cast<int>(BT), D, D * kx}; q.lda = D * sx; q.a_split_k = sp ? D : 0;
      q.bias = c.F(b + "proj_b"); q.gamma = c.F(b + "ls1");
      q.resid = x; q.resid_f32 = 1; q.out = x; q.out_f32 = 1;
      if (fuse) { q.out2 = x16; q.out2_leaky = 0; q.ln_stats_out = stats; q.ln_parts = ln_parts; q.ln_part_cols = ln_pc; }
      c.gemm(q); }
    if (fuse) {
      Ctx::G q{x16, c.H(b + "fc1_wf"), static_cast<int>(BT), 4 * D, D};
      q.bias = c.F(b + "fc1_c2"); q.ln_stats_in = stats; q.ln_c1 = c.F(b + "fc1_c1"); q.ln_parts = ln_parts; q.ln_part_cols = ln_pc;
      q.ln_eps = 1e-6f; q.act = UDB_ACT_GELU; q.out = mid; c.gemm(q);
    } else {
      c.layernorm(x, 1, h, 0, c.F(b + "n2w"), c.F(b + "n2b"), static_cast<int>(BT), D, 1e-6f, 0, 0, 0, 0, sp ? D : 0);
      Ctx::G q{h, c.H(b + "fc1_w"), static_cast<int>(BT), 4 * D, D * kx}; q.lda = D * sx; q.a_split_k = sp ? D : 0;
      q.bias = c.F(b + "fc1_b"); q.act = UDB_ACT_GELU;
      q.out = mid; q.ldc = 4 * D * sx; q.out_split = sp ? 4 * D : 0; c.gemm(q);
    }
    { Ctx::G q{mid, c.H(b + "fc2_w"), static_cast<int>(BT), D, 4 * D * kx}; q.lda = 4 * D * sx; q.a_split_k = sp ? 4 * D : 0;
      q.bias = c.F(b + "fc2_b"); q.gamma = c.F(b + "ls2");
      q.resid = x; q.resid_f32 = 1; q.out = x; q.out_f32 = 1;
      if (fuse) { q.out2 = x16; q.out2_leaky = 0; q.ln_stats_out = stats; q.ln_parts = ln_parts; q.ln_part_cols = ln_pc; }
      c.gemm(q); }
    after_block(i);
  }
  ar.release(m);
}

}  // namespace udb
