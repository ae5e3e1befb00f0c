// Whole-path engine for UniDepthV1.infer with the ConvNeXt encoder (BASELINE config 4) or the DINOv2 ViT-L/14 encoder
// (config_v1_vitl14; the block loop is the one UniDepthV2 runs, engine_common.h `vit_blocks`), behind udb_v1_create /
// udb_v1_set_weight / udb_v1_workspace_bytes / udb_infer_v1 (include/udb.h).  Host-side schedule only: it enqueues the
// kernels of this library on the caller's stream over a bump-allocated workspace (no allocation, copy or sync inside
// udb_infer_v1, so the call is graph-capturable).  Reference call stack it replaces:
//   UniDepthV1.infer                 unidepth/models/unidepthv1/unidepthv1.py:288-373 (_shapes/_paddings/_preprocess/_postprocess :30-94)
//     pixel_encoder = ConvNeXt       unidepth/models/backbones/convnext.py:459-471 (stem :371-383, stage :289-298, block :208-223)
//     pixel_decoder = Decoder        unidepth/models/unidepthv1/decoder.py:364-463 (run_camera :311-343, CameraHead :85-106,
//                                    DepthHead :195-300), layers/{attention,nystrom_attention,mlp,upsample,convnext}.py
#include "engine_common.h"

struct udb_engine_v1 : udb::EngineBase {
  udb_v1_config_t cfg;
};

namespace udb {

struct V1Geom {
  int rh, rw;                       // resized image inside the network frame
  double ratio;
  int pad_l, pad_r, pad_t, pad_b;
};

// unidepthv1.py:30-46 (Python float == C double; ceil(x - 0.5))
static V1Geom v1_geometry(int H, int W, int net_h, int net_w) {
  V1Geom g;
  const double in_ratio = static_cast<double>(W) / H, out_ratio = static_cast<double>(net_w) / net_h;
  g.ratio = out_ratio > in_ratio ? static_cast<double>(net_h) / H : static_cast<double>(net_w) / W;
  g.rh = static_cast<int>(ceil(H * g.ratio - 0.5));
  g.rw = static_cast<int>(ceil(W * g.ratio - 0.5));
  const int dh = net_h - g.rh, dw = net_w - g.rw;
  g.pad_t = floordiv2(dh); g.pad_b = dh - g.pad_t;
  g.pad_l = floordiv2(dw); g.pad_r = dw - g.pad_l;
  return g;
}

// Encoder stages whose ConvNeXt blocks run in e4m3 mode (precision 2); the others keep the f16 block.  A fixed rule of the
// schedule: a stage runs e4m3 only where its profiled block time is below the f16 block's.  On an H100 none is (DESIGN.md
// section 8): in stages 0 and 1 the e4m3 MLP GEMMs save less than the GELU row quantiser costs, and in stages 2 and 3 the
// GEMMs' saving is outweighed by that quantiser plus udb_dwconv7_ln_e4m3, which takes longer than the f16 depthwise
// conv and LayerNorm together.  So ConvNeXt-L runs its f16 blocks in both modes.  unidepthv1.py FP8_STAGES packs the
// same set.
static constexpr bool kFp8Stage[4] = {false, false, false, false};

// The same block in e4m3 mode: udb_dwconv7_ln_e4m3 writes fc1's e4m3 operand and row scales, the GELU output is quantised
// per row for fc2, and both GEMMs read e4m3 weights with one scale per output channel; the epilogues are those of the
// f16 block.  Its scratch -- the two e4m3 operands (rows x C, then rows x 4C bytes, sharing one rows x 4C region), the
// row scales (rows x 4 bytes) and the f16 GELU output -- is rows x 4 bytes more than the f16 block's y, hN and GELU output.
static void cvnxt_block_e4m3(Ctx& c, const std::string& p, float* x, __half* x16, int B, int Hh, int Ww, int C) {
  Arena& ar = *c.ar;
  const size_t m = ar.mark();
  const long long rows = static_cast<long long>(B) * Hh * Ww;
  void* a8 = ar.alloc(rows * 4 * C);
  float* as = ar.f(rows);
  __half* md = ar.h(rows * 4 * C);
  c.expect2(p + "w1_8", 4 * C, C);
  c.expect2(p + "w2_8", C, 4 * C);
  c.expect_e4m3(p + "w1_8");
  c.expect_e4m3(p + "w2_8");
  const float* dw_w = c.F(p + "dw_w");
  const float* dw_b = c.F(p + "dw_b");
  const float* ln_w = c.F(p + "ln_w");
  const float* ln_b = c.F(p + "ln_b");
  c.launch([&] { return udb_dwconv7_ln_e4m3(x16, dw_w, dw_b, ln_w, ln_b, a8, as, B, Hh, Ww, C, c.st); });
  { Ctx::G q{a8, c.W(p + "w1_8")->p, static_cast<int>(rows), 4 * C, C}; q.a_scale = as; q.w_scale = c.F(p + "w1_8s");
    q.bias = c.F(p + "b1"); q.act = UDB_ACT_GELU; q.out = md; c.gemm(q); }
  c.quantize_e4m3(md, 4 * C, a8, as, static_cast<int>(rows), 4 * C);
  { Ctx::G q{a8, c.W(p + "w2_8")->p, static_cast<int>(rows), C, 4 * C}; q.a_scale = as; q.w_scale = c.F(p + "w2_8s");
    q.bias = c.F(p + "b2"); q.gamma = c.F(p + "gamma"); q.resid = x; q.resid_f32 = 1; q.out = x; q.out_f32 = 1; q.out2 = x16;
    q.out2_leaky = 0; c.gemm(q); }
  ar.release(m);
}

// The same block in split-precision mode (precision 1): the depthwise 7x7 reads the f32 residual stream and writes f32,
// LayerNorm writes the [hi | lo] operand of fc1, fc1 writes its GELU output as a split operand for fc2, and both GEMMs
// read [N, 3K] = [hi | hi | lo] weights (udb_gemm_t.a_split_k).  There is no f16 copy of x in this mode.
static void cvnxt_block_split(Ctx& c, const std::string& p, float* x, int B, int Hh, int Ww, int C) {
  Arena& ar = *c.ar;
  const size_t m = ar.mark();
  const long long rows = static_cast<long long>(B) * Hh * Ww;
  float* y = ar.f(rows * C);
  __half* hN = ar.h(rows * 2 * C);
  __half* md = ar.h(rows * 8 * C);
  c.expect2(p + "w1", 4 * C, 3 * C);
  c.expect2(p + "w2", C, 12 * C);
  const float* dw_w = c.F(p + "dw_w");
  const float* dw_b = c.F(p + "dw_b");
  c.launch([&] { return udb_dwconv7_nhwc_f32(x, dw_w, dw_b, y, B, Hh, Ww, C, c.st); });
  c.ln_any(y, 1, hN, UDB_LN_OUT_SPLIT, c.F(p + "ln_w"), c.F(p + "ln_b"), rows, C, 1e-6f, 2 * C);
  { Ctx::G q{hN, c.H(p + "w1"), static_cast<int>(rows), 4 * C, 3 * C}; q.lda = 2 * C; q.a_split_k = C; q.bias = c.F(p + "b1");
    q.act = UDB_ACT_GELU; q.out = md; q.ldc = 8 * C; q.out_split = 4 * C; c.gemm(q); }
  { Ctx::G q{md, c.H(p + "w2"), static_cast<int>(rows), C, 12 * C}; q.lda = 8 * C; q.a_split_k = 4 * C; q.bias = c.F(p + "b2");
    q.gamma = c.F(p + "gamma"); q.resid = x; q.resid_f32 = 1; q.out = x; q.out_f32 = 1; c.gemm(q); }
  ar.release(m);
}

// pre-processing of the input batch into the encoder's patch rows (unidepthv1.py _preprocess): 4x4 im2col rows of the
// ConvNeXt stem (`patch` 0) or 14x14 DINOv2 patch rows (`patch` 14); `split`: as [hi | lo] operands
static void preprocess(Ctx& c, const udb_v1_config_t& cf, const udb_infer_v1_args_t& a, const V1Geom& g, __half* patches,
                       int patch, bool split = false) {
  udb_v1_preprocess_t p;
  memset(&p, 0, sizeof(p));
  p.rgb = a.rgb; p.rgb_is_u8 = a.rgb_is_u8; p.scale255 = a.scale255; p.normalize = a.normalize; p.B = a.B; p.H = a.H; p.W = a.W;
  p.rh = g.rh; p.rw = g.rw; p.pad_l = g.pad_l; p.pad_t = g.pad_t; p.net_h = cf.net_h; p.net_w = cf.net_w; p.patches = patches;
  p.patch = patch;
  c.launch([&] { return split ? udb_v1_preprocess_split(&p, c.st) : udb_v1_preprocess(&p, c.st); });
}

// ConvNeXt encoder in split-precision mode (convnext.py:371-383,289-298 as in run_v1's f16 encoder): split stem rows ->
// stem GEMM to f32 -> LayerNorm f32 -> stages of cvnxt_block_split; each downsample is a space-to-depth LayerNorm with
// split output and the k2 s2 GEMM on it.  The running max of each stage's block outputs is kept in f32 (levels[i]).
static void convnext_encoder_split(Ctx& c, const udb_v1_config_t& cf, const udb_infer_v1_args_t& a, const V1Geom& g, const int* sh,
                                   const int* sw, void* const* levels, float* const* clsbuf, int total_blocks) {
  Arena& ar = *c.ar;
  const size_t m = ar.mark();
  const int B = a.B, C0 = cf.dims[0];
  const long long n0 = static_cast<long long>(B) * sh[0] * sw[0];
  __half* patches = ar.h(n0 * 128);
  preprocess(c, cf, a, g, patches, 0, true);
  float* y0 = ar.f(n0 * C0);
  c.expect2("stem_w", C0, 192);
  { Ctx::G q{patches, c.H("stem_w"), static_cast<int>(n0), C0, 192}; q.lda = 128; q.a_split_k = 64; q.bias = c.F("stem_b");
    q.out = y0; q.out_f32 = 1; c.gemm(q); }
  float* x = ar.f(n0 * C0);
  c.ln_any(y0, 1, x, 1, c.F("stem_ln_w"), c.F("stem_ln_b"), n0, C0, 1e-6f);
  int blk = 0;
  for (int i = 0; i < 4; ++i) {
    const int C = cf.dims[i];
    const long long n = static_cast<long long>(B) * sh[i] * sw[i];
    if (i > 0) {
      const int Cp = cf.dims[i - 1];
      __half* A = ar.h(n * 8 * Cp);
      const std::string d = idx("ds%d.", i);
      c.ln_any(x, 1, A, UDB_LN_OUT_SPLIT, c.F(d + "ln_w"), c.F(d + "ln_b"), static_cast<long long>(B) * sh[i - 1] * sw[i - 1], Cp, 1e-6f,
               8 * Cp, nullptr, 0, sh[i - 1], sw[i - 1]);
      float* xn = ar.f(n * C);
      c.expect2(d + "w", C, 12 * Cp);
      { Ctx::G q{A, c.H(d + "w"), static_cast<int>(n), C, 12 * Cp}; q.lda = 8 * Cp; q.a_split_k = 4 * Cp; q.bias = c.F(d + "b");
        q.out = xn; q.out_f32 = 1; c.gemm(q); }
      x = xn;
    }
    for (int j = 0; j < cf.depths[i]; ++j, ++blk) {
      cvnxt_block_split(c, idx2("s%d.b%d.", i, j), x, B, sh[i], sw[i], C);
      c.launch([&] { return udb_max_accum_f32(x, static_cast<float*>(levels[i]), n * C, j == 0, c.st); });
      const int from_end = total_blocks - 1 - blk;
      if (from_end < 4) c.launch([&] { return udb_spatial_mean_f32(x, clsbuf[from_end], B, sh[i] * sw[i], C, c.st); });
    }
  }
  ar.release(m);
}

// ConvUpsample (layers/upsample.py:13-45): (lat + emb) -> 2 CvnxtBlocks -> conv1x1 C->C/2 -> x2 bilinear (align_corners=True)
// -> conv3x3 (zero pad).  Returns the next level's f32 tokens and their f16 copy (allocated before the scratch mark).
static void conv_upsample(Ctx& c, const std::string& p, const float* lat, const float* emb, int B, int h, int w, int C, float* next,
                          __half* next16) {
  Arena& ar = *c.ar;
  const size_t m = ar.mark();
  const long long R = static_cast<long long>(B) * h * w;
  float* xs = ar.f(R * C);
  __half* xs16 = ar.h(R * C);
  c.launch([&] { return udb_add_f32(lat, emb, xs, xs16, R * C, c.st); });
  for (int j = 0; j < 2; ++j) cvnxt_block(c, p + (j ? "c1." : "c0."), xs, xs16, B, h, w, C, 1e-5f);
  const int C2 = C / 2;
  __half* u = ar.h(R * C2);
  { Ctx::G g{xs16, c.H(p + "up_w"), static_cast<int>(R), C2, C}; g.bias = c.F(p + "up_b"); g.out = u; c.gemm(g); }
  __half* up = ar.h(R * 4 * C2);
  c.launch([&] { return udb_resize_ac_pad_nhwc_f16(u, up, B, h, w, C2, 2 * h, 2 * w, 0, c.st); });
  c.expect2(p + "conv_w", C2, 9 * C2);
  c.conv3x3(up, B, 2 * h, 2 * w, C2, c.H(p + "conv_w"), C2, c.F(p + "conv_b"), UDB_ACT_NONE, nullptr, nullptr, 0, next, 1, next16, 0);
  ar.release(m);
}

// DINOv2 encoder of UniDepthV1 (unidepthv1.py:316-326; dinov2.py:306-347 with use_norm=False): 14x14 patch rows of the
// pre-processed image -> patch GEMM with the pack-time position table ("pos" [1 + gh*gw, D], cls row first: offset-0.1
// bicubic resize of the 37x37 grid) as row-mapped residual -> cls rows -> the shared block loop.  After every block the
// tap kernel folds (patch tokens + cls token) into the running max of its slice (levels[s], decoder.py:371-379; slice s
// holds cf.depths[s] blocks) and copies the raw cls rows of the last four blocks into clsbuf[k] (block last - k).
// Split-precision mode (`split`): split patch rows and patch weight [D, 3*640], the shared block loop's split mode and
// f32 levels (udb_vit_tap_f32).
static void dino_encoder(Ctx& c, const udb_v1_config_t& cf, const udb_infer_v1_args_t& a, const V1Geom& g, int gh, int gw,
                         void* const* levels, float* const* clsbuf, bool fp8, bool split) {
  Arena& ar = *c.ar;
  const int B = a.B, D = cf.dims[0], N = gh * gw, T = N + 1;
  const size_t BN = static_cast<size_t>(B) * N, BT = static_cast<size_t>(B) * T;
  int depth = 0;
  for (int i = 0; i < 4; ++i) depth += cf.depths[i];
  const size_t m = ar.mark();
  const int sx = split ? 2 : 1;
  __half* patches = ar.h(BN * 640 * sx);
  preprocess(c, cf, a, g, patches, 14, split);
  float* x = ar.f(BT * D);           // fp32 residual stream [B, 1 + N, D]
  VitBlocks v{B, T, D, D / 64, depth};
  v.fp8 = fp8;
  v.split = split;
  c.expect2("pos", T, D);
  vit_embed(c, patches, c.F("pos"), x, v);
  int slice = 0, start = 0;
  vit_blocks(c, "blocks.", x, v, [&](int i) {
    if (i == start + cf.depths[slice]) { start = i; ++slice; }
    const int from_end = depth - 1 - i;
    float* cls_out = from_end < 4 ? clsbuf[from_end] : nullptr;
    c.launch([&] {
      return split ? udb_vit_tap_f32(x, static_cast<float*>(levels[slice]), cls_out, B, N, D, i == start, c.st)
                   : udb_vit_tap(x, levels[slice], cls_out, B, N, D, i == start, c.st);
    });
  });
  ar.release(m);
}

static int run_v1(udb_engine_v1* e, const udb_infer_v1_args_t& a, Arena& ar, void* st) {
  const udb_v1_config_t& cf = e->cfg;
  Ctx c{e, &ar, st, ar.dry};
  const int B = a.B, net_h = cf.net_h, net_w = cf.net_w, hid = cf.hidden;
  const V1Geom g = v1_geometry(a.H, a.W, net_h, net_w);
  const bool dino = cf.encoder == UDB_V1_ENCODER_DINOV2;
  int sh[4], sw[4];
  if (dino) {                       // one 14-pixel patch grid for every level (decoder.py:381-396: flat_interpolate is the identity)
    for (int i = 0; i < 4; ++i) { sh[i] = net_h / 14; sw[i] = net_w / 14; }
  } else {
    sh[0] = (net_h - 4) / 4 + 1; sw[0] = (net_w - 4) / 4 + 1;
    for (int i = 1; i < 4; ++i) { sh[i] = sh[i - 1] / 2; sw[i] = sw[i - 1] / 2; }
  }
  // Bounds the network grid puts on the kernels, checked here so that the dry run names them before anything is launched:
  // the 1/8 and 1/4 decoder levels run Nystrom attention with 128 landmarks, which needs more tokens than landmarks (the
  // reference's xformers module pools segments of seq // 128 rows, and switches to exact attention at exactly 128), and
  // the camera head's single-head cross attention over the 4*hc*wc + 4 context tokens has a shared-memory bound.
  {
    const int n8 = 4 * sh[2] * sw[2];
    if (n8 <= 128) {
      set_error("udb_v1: network shape %dx%d gives %d tokens at the 1/8 decoder level (%dx%d); Nystrom attention needs more "
                "than its 128 landmarks", net_h, net_w, n8, 2 * sh[2], 2 * sw[2]);
      return 1;
    }
    if (cross_attn_small_check("udb_v1: camera head cross attention", 4, 4 * sh[2] * sw[2] + 4, hid)) return 1;
  }
  Stage stage;
  // "precision": 0 (absent) = f16 operands, 2 = e4m3 operands for the encoder blocks' MLP (ConvNeXt) or all four linear
  // layers (DINOv2); the stem, downsample layers and the decoder are the same in both.  1 = split-f16 operands (parity
  // mode): every GEMM of the encoder and of the camera head's context path (adapters, in_features, the aggregate block's
  // kv) multiplies [hi | lo] operands with [hi | hi | lo] weights, and the encoder levels and camera context are f32;
  // the depth head reads the hi half of the adapters' LayerNorm and runs as in the f16 mode.
  const Precision prec = encoder_precision(c, "udb_infer_v1", dino ? "patch_w" : "stem_w", dino ? 3 * 640 : 3 * 64);
  if (prec == PREC_BAD) return 1;
  const bool f8 = prec == PREC_E4M3, sp = prec == PREC_SPLIT;

  // ---- pre-processing + stem (convnext.py:371-383: conv k4 s4 as an im2col GEMM, then LayerNorm2d)
  stage.next("udb_v1:preprocess+stem");
  void* levels[4];                  // f16, or f32 in split mode
  float* clsbuf[4];
  for (int i = 0; i < 4; ++i) levels[i] = ar.alloc(static_cast<size_t>(B) * sh[i] * sw[i] * cf.dims[i] * (sp ? 4 : 2));
  int total_blocks = 0;
  for (int i = 0; i < 4; ++i) total_blocks += cf.depths[i];
  // decoder.py:377-379: the cls tokens of the LAST FOUR BLOCKS, newest first
  int cls_dim[4];
  {
    int k = 0;
    for (int i = 3; i >= 0 && k < 4; --i)
      for (int j = cf.depths[i] - 1; j >= 0 && k < 4; --j) cls_dim[k++] = cf.dims[i];
    if (k != 4) { set_error("udb_infer_v1: the encoder needs at least four blocks"); return 1; }
  }
  for (int k = 0; k < 4; ++k) clsbuf[k] = ar.f(static_cast<size_t>(B) * cls_dim[k]);     // clsbuf[k]: block (last - k)
  if (dino) {
    stage.next("udb_v1:dinov2_encoder");
    dino_encoder(c, cf, a, g, sh[0], sw[0], levels, clsbuf, f8, sp);
  } else if (sp) {
    stage.next("udb_v1:convnext_stages");
    convnext_encoder_split(c, cf, a, g, sh, sw, levels, clsbuf, total_blocks);
  } else {
    const size_t enc_mark = ar.mark();
    const long long n0 = static_cast<long long>(B) * sh[0] * sw[0];
    __half* patches = ar.h(n0 * 64);
    preprocess(c, cf, a, g, patches, 0);
    const int C0 = cf.dims[0];
    __half* y0 = ar.h(n0 * C0);
    { Ctx::G q{patches, c.H("stem_w"), static_cast<int>(n0), C0, 64}; q.bias = c.F("stem_b"); q.out = y0; c.gemm(q); }
    float* x = ar.f(n0 * C0);
    __half* x16 = ar.h(n0 * C0);
    c.ln_any(y0, 0, x, 1, c.F("stem_ln_w"), c.F("stem_ln_b"), n0, C0, 1e-6f);
    c.ln_any(y0, 0, x16, 0, c.F("stem_ln_w"), c.F("stem_ln_b"), n0, C0, 1e-6f);

    // ---- ConvNeXt stages (convnext.py:289-298); running max of each stage's block outputs (decoder.py:371-374)
    stage.next("udb_v1:convnext_stages");
    int blk = 0;
    for (int i = 0; i < 4; ++i) {
      const int C = cf.dims[i];
      const long long n = static_cast<long long>(B) * sh[i] * sw[i];
      if (i > 0) {
        const int Cp = cf.dims[i - 1];
        __half* A = ar.h(n * 4 * Cp);
        const std::string d = idx("ds%d.", i);
        c.ln_any(x, 1, A, 0, c.F(d + "ln_w"), c.F(d + "ln_b"), static_cast<long long>(B) * sh[i - 1] * sw[i - 1], Cp, 1e-6f, 4 * Cp, nullptr, 0,
                 sh[i - 1], sw[i - 1]);
        float* xn = ar.f(n * C);
        __half* xn16 = ar.h(n * C);
        c.expect2(d + "w", C, 4 * Cp);
        { Ctx::G q{A, c.H(d + "w"), static_cast<int>(n), C, 4 * Cp}; q.bias = c.F(d + "b"); q.out = xn; q.out_f32 = 1; q.out2 = xn16; q.out2_leaky = 0;
          c.gemm(q); }
        x = xn;
        x16 = xn16;
      }
      for (int j = 0; j < cf.depths[i]; ++j, ++blk) {
        if (f8 && kFp8Stage[i]) cvnxt_block_e4m3(c, idx2("s%d.b%d.", i, j), x, x16, B, sh[i], sw[i], C);
        else cvnxt_block(c, idx2("s%d.b%d.", i, j), x, x16, B, sh[i], sw[i], C, 1e-6f);
        c.launch([&] { return udb_max_accum_f16(x16, levels[i], n * C, j == 0, st); });
        const int from_end = total_blocks - 1 - blk;
        if (from_end < 4) c.launch([&] { return udb_spatial_mean_f32(x, clsbuf[from_end], B, sh[i] * sw[i], C, st); });
      }
    }
    ar.release(enc_mark);
  }

  // ---- decoder: common grid = second-smallest level (decoder.py:381-392), adapters (:395-408)
  stage.next("udb_v1:adapters");
  const int hc = sh[2], wc = sw[2], nq = hc * wc;
  const long long Rq = static_cast<long long>(B) * nq;
  __half* featcat = ar.h(Rq * 4 * hid);                          // [B*nq, 4*hid]   (features_channels, decoder.py:224)
  __half* tokens = ar.h((Rq * 4 + 64) * hid);                    // [B, 4*nq, hid]  (features_tokens,   decoder.py:220)
  // split mode: the camera head's copy of the tokens, f32 from split operands (the depth head keeps the f16 tokens)
  float* cam_tokens = sp ? ar.f(Rq * 4 * hid) : nullptr;
  adapters(c, levels, cf.dims, sh, sw, B, hc, wc, hid, sp, tokens, featcat, cam_tokens, nullptr);
  const float* tokens_pos = c.F("tokens_pos");                     // [4*nq, hid]: sine position + level embedding (decoder.py:410-433)
  {
    const Weight* tp = c.W("tokens_pos");
    if (!c.rc && (tp->shape[0] != 4LL * nq || tp->shape[1] != hid)) { set_error("engine_v1: tokens_pos must be [%d, %d]", 4 * nq, hid); return 1; }
  }

  // ---- camera head (decoder.py:311-343, 85-106), fp32 on the CUDA cores except the two context GEMMs
  stage.next("udb_v1:camera_head");
  float* intr4 = ar.f(static_cast<size_t>(B) * 4);
  float* k4_points = ar.f(static_cast<size_t>(B) * 4);
  const size_t cam_mark = ar.mark();          // the camera head's scratch: dead once the intrinsics kernel has read x4
  const float* x4 = nullptr;
  if (!(a.skip_camera && a.intrinsics)) {
    const int R4 = B * 4;
    float* toks = token_adapter(c, "tok.", clsbuf, cls_dim, 4, B, hid);
    // cls_project: LN -> Linear(hid -> hid/2) -> GELU -> Linear(hid/2 -> hid)
    float* cl = cam_mlp(c, "cam.cls", toks, R4, hid, hid / 2, hid, nullptr, nullptr);
    const void* ctx = camera_context(c, sp ? static_cast<const void*>(cam_tokens) : tokens, tokens_pos, cl, B, nq, 4, hid, sp);
    // aggregate: the 4 tokens attend to the context (single head of width hid, position term on q)
    float* t = small_cross_block(c, "cam.agg.", cl, B, 4, ctx, 4LL * nq + 4, c.F("cam.pos"), hid, cf.expansion, sp);
    for (int i = 0; i < 2; ++i) {
      const std::string ly = idx("cam.l%d.", i);
      float* xn = ar.f(static_cast<size_t>(R4) * hid);
      float* cn = ar.f(static_cast<size_t>(R4) * hid);
      c.layernorm(t, 1, xn, 1, c.F(ly + "nxw"), c.F(ly + "nxb"), R4, hid, 1e-5f);
      c.layernorm(t, 1, cn, 1, c.F(ly + "ncw"), c.F(ly + "ncb"), R4, hid, 1e-5f);
      float* q = ar.f(static_cast<size_t>(R4) * hid);
      float* kv = ar.f(static_cast<size_t>(R4) * 2 * hid);
      c.small_linear(xn, R4, hid, c.F(ly + "q_w"), hid, c.F(ly + "q_b"), UDB_ACT_NONE, nullptr, nullptr, q);
      c.small_linear(cn, R4, hid, c.F(ly + "kv_w"), 2 * hid, c.F(ly + "kv_b"), UDB_ACT_NONE, nullptr, nullptr, kv);
      float* a4 = ar.f(static_cast<size_t>(R4) * hid);
      const float* cam_pos = c.F("cam.pos");
      c.launch([&] { return udb_camera_attn4_f32(q, kv, cam_pos, a4, B, hid, cf.heads, st); });
      float* t2 = ar.f(static_cast<size_t>(R4) * hid);
      c.small_linear(a4, R4, hid, c.F(ly + "out_w"), hid, c.F(ly + "out_b"), UDB_ACT_NONE, c.F(ly + "ls1"), t, t2);
      t = cam_mlp(c, ly + "mlp", t2, R4, hid, cf.expansion * hid, hid, t2, c.F(ly + "ls2"));
    }
    x4 = cam_mlp(c, "cam.out", t, R4, hid, 2 * hid, 1, nullptr, nullptr);       // [B*4, 1] == [B, 4]
  }
  c.launch([&] {
    return udb_v1_camera_intrinsics(x4, a.intrinsics, B, net_h, net_w, static_cast<float>(g.ratio), g.pad_l, g.pad_t, a.skip_camera,
                                    intr4, a.out_intrinsics, k4_points, st);
  });
  ar.release(cam_mark);

  // ---- ray embeddings at the three decoder levels (decoder.py:203-220)
  stage.next("udb_v1:ray_embeddings");
  float* emb[3];
  {
    float shk[81];
    for (int l = 0; l <= 8; ++l)
      for (int mo = 0; mo <= 8; ++mo) {
        double k = 0.0;
        if (mo <= l) {
          double ratio_f = 1.0;                       // (l-m)! / (l+m)!
          for (int t = l - mo + 1; t <= l + mo; ++t) ratio_f /= t;
          k = sqrt((2 * l + 1) / (4.0 * M_PI) * ratio_f) * (mo > 0 ? sqrt(2.0) : 1.0);
        }
        shk[l * 9 + mo] = static_cast<float>(k);
      }
    const char* names[3] = {"rays.16.", "rays.8.", "rays.4."};
    for (int s = 0; s < 3; ++s) {
      const int gh = hc << s, gw = wc << s, Cs = hid >> s;
      const long long R = static_cast<long long>(B) * gh * gw;
      emb[s] = ar.f(R * Cs);
      const size_t m = ar.mark();
      __half* r = ar.h(R * 128);
      __half* m1 = ar.h(R * 384);
      {
        udb_v1_rays_t p;
        memset(&p, 0, sizeof(p));
        p.intr4 = intr4; p.B = B; p.net_h = net_h; p.net_w = net_w; p.gh = gh; p.gw = gw;
        p.ln_w = c.F(std::string(names[s]) + "ln_w"); p.ln_b = c.F(std::string(names[s]) + "ln_b"); p.out = r;
        memcpy(p.sh_k, shk, sizeof(shk));
        c.launch([&] { return udb_v1_rays_sh81(&p, st); });
      }
      const std::string n = names[s];
      c.expect2(n + "w1", 384, 128);
      { Ctx::G q{r, c.H(n + "w1"), static_cast<int>(R), 384, 128}; q.bias = c.F(n + "b1"); q.act = UDB_ACT_GELU; q.out = m1; c.gemm(q); }
      { Ctx::G q{m1, c.H(n + "w2"), static_cast<int>(R), Cs, 384}; q.bias = c.F(n + "b2"); q.out = emb[s]; q.out_f32 = 1; c.gemm(q); }
      ar.release(m);
    }
  }

  // ---- depth head (decoder.py:222-300)
  stage.next("udb_v1:depth_head_16");
  float* lat16 = ar.f(Rq * hid);
  {
    const size_t m = ar.mark();
    __half* f16l = ar.h(Rq * hid);
    { Ctx::G q{featcat, c.H("fcc_w"), static_cast<int>(Rq), hid, 4 * hid}; q.bias = c.F("fcc_b"); q.out = f16l; c.gemm(q); }
    __half* hN = ar.h(Rq * hid);
    __half* md = ar.h(Rq * 2 * hid);
    ln16(c, f16l, 0, hN, "lat.nw", "lat.nb", Rq, hid, 1e-5f);
    { Ctx::G q{hN, c.H("lat.w1"), static_cast<int>(Rq), 2 * hid, hid}; q.bias = c.F("lat.b1"); q.act = UDB_ACT_GELU; q.out = md; c.gemm(q); }
    { Ctx::G q{md, c.H("lat.w2"), static_cast<int>(Rq), hid, 2 * hid}; q.bias = c.F("lat.b2"); q.out = lat16; q.out_f32 = 1; c.gemm(q); }
    ar.release(m);
  }
  dense_attn_block(c, "agg16.", lat16, B, nq, hid, tokens, 0, 4 * nq, tokens_pos);
  dense_attn_block(c, "prompt.", lat16, B, nq, hid, emb[0], 1, nq, nullptr);
  for (int i = 0; i < cf.dec_depths[0]; ++i) mh_attn_block(c, idx("l16.%d.", i), lat16, B, nq, hid, cf.heads, emb[0], false);

  float* outs[3];
  float* lat = lat16;
  const char* ups[3] = {"up8.", "up4.", "up2."};
  const char* lys[3] = {"", "l8.%d.", "l4.%d."};
  const char* ons[3] = {"out8", "out4", "out2"};
  int ch = hc, cw = wc, C = hid;
  for (int s = 0; s < 3; ++s) {
    stage.next(s == 0 ? "udb_v1:up8" : (s == 1 ? "udb_v1:layers_8+up4" : "udb_v1:layers_4+up2"));
    if (s > 0)
      for (int i = 0; i < cf.dec_depths[s]; ++i) mh_attn_block(c, idx(lys[s], i), lat, B, ch * cw, C, cf.heads >> s, emb[s], true);
    const long long Rn = static_cast<long long>(B) * 4 * ch * cw;
    float* nxt = ar.f(Rn * (C / 2));
    __half* nxt16 = ar.h(Rn * (C / 2));
    outs[s] = ar.f(Rn);
    conv_upsample(c, ups[s], lat, emb[s], B, ch, cw, C, nxt, nxt16);
    const float* head_w = c.F(std::string(ons[s]) + ".w");
    const float head_b = static_cast<float>(c.S(std::string(ons[s]) + ".b"));
    c.launch([&] { return udb_conv3x3_c1_exp(nxt16, head_w, head_b, outs[s], B, 2 * ch, 2 * cw, C / 2, st); });
    lat = nxt;
    ch *= 2; cw *= 2; C /= 2;
  }

  // ---- post-processing (unidepthv1.py:66-94,352-366)
  stage.next("udb_v1:postprocess");
  float* mean = ar.f(static_cast<size_t>(B) * net_h * net_w);
  c.launch([&] { return udb_v1_mean_maps(outs[0], outs[1], outs[2], mean, B, hc, wc, net_h, net_w, st); });
  {
    udb_v1_postprocess_t p;
    memset(&p, 0, sizeof(p));
    p.mean = mean; p.k4 = k4_points; p.B = B; p.net_h = net_h; p.net_w = net_w;
    p.pad_l = g.pad_l; p.pad_r = g.pad_r; p.pad_t = g.pad_t; p.pad_b = g.pad_b; p.H = a.H; p.W = a.W;
    p.out_depth = a.out_depth; p.out_points = a.out_points;
    c.launch([&] { return udb_v1_postprocess(&p, st); });
  }
  if (!c.rc && ar.overflow) { set_error("engine_v1: workspace too small (%zu bytes needed)", ar.peak); return 1; }
  return c.rc;
}

}  // namespace udb

using namespace udb;

extern "C" {

int udb_v1_create(const udb_v1_config_t* cfg, udb_engine_v1** out) {
  if (!cfg || !out) { set_error("udb_v1_create: null argument"); return 1; }
  if (cfg->encoder != UDB_V1_ENCODER_CONVNEXT && cfg->encoder != UDB_V1_ENCODER_DINOV2) {
    set_error("udb_v1_create: encoder %d unknown (0 ConvNeXt, 1 DINOv2)", cfg->encoder);
    return 1;
  }
  if (cfg->encoder == UDB_V1_ENCODER_DINOV2) {
    if (cfg->net_h % 14 || cfg->net_w % 14) {
      set_error("udb_v1_create: DINOv2 network shape %dx%d must be a multiple of the 14-pixel patch", cfg->net_h, cfg->net_w);
      return 1;
    }
    for (int i = 1; i < 4; ++i)
      if (cfg->dims[i] != cfg->dims[0]) { set_error("udb_v1_create: DINOv2 slices must all have the embedding width"); return 1; }
  }
  for (int i = 0; i < 4; ++i)
    if (cfg->dims[i] <= 0 || cfg->dims[i] % 64 || cfg->dims[i] > 1536 || cfg->depths[i] <= 0) {
      set_error("udb_v1_create: stage %d (depth %d, width %d): widths must be multiples of 64 up to 1536", i, cfg->depths[i], cfg->dims[i]);
      return 1;
    }
  if (cfg->hidden != 512 || cfg->heads != 8) {
    set_error("udb_v1_create: decoder hidden %d / heads %d not supported (512 / 8: 64-wide heads at every level)", cfg->hidden, cfg->heads);
    return 1;
  }
  if (cfg->net_h < 64 || cfg->net_w < 64) { set_error("udb_v1_create: network shape %dx%d too small", cfg->net_h, cfg->net_w); return 1; }
  udb_engine_v1* e = new udb_engine_v1();
  e->cfg = *cfg;
  *out = e;
  return 0;
}

void udb_v1_destroy(udb_engine_v1* e) { delete e; }

int udb_v1_geometry(int32_t H, int32_t W, int32_t net_h, int32_t net_w, udb_v1_geometry_t* out) {
  if (!out || H <= 0 || W <= 0 || net_h <= 0 || net_w <= 0) { set_error("udb_v1_geometry: bad argument"); return 1; }
  const V1Geom g = v1_geometry(H, W, net_h, net_w);      // the function run_v1 uses
  out->resized_h = g.rh; out->resized_w = g.rw;
  out->pad_l = g.pad_l; out->pad_r = g.pad_r; out->pad_t = g.pad_t; out->pad_b = g.pad_b;
  out->ratio = g.ratio;
  return 0;
}

int udb_v1_set_weight(udb_engine_v1* e, const char* name, const void* dev_ptr, const int64_t* shape, int32_t ndim, int32_t dtype) {
  return EngineBase::set_weight(e, "udb_v1_set_weight", name, dev_ptr, shape, ndim, dtype);
}

int udb_v1_set_scalar(udb_engine_v1* e, const char* name, double value) {
  return EngineBase::set_scalar(e, "udb_v1_set_scalar", name, value);
}

size_t udb_v1_workspace_bytes(udb_engine_v1* e, int32_t B, int32_t H, int32_t W) {
  if (!e || B <= 0 || H <= 0 || W <= 0) { set_error("udb_v1_workspace_bytes: bad argument"); return 0; }
  udb_infer_v1_args_t a;
  memset(&a, 0, sizeof(a));
  a.B = B; a.H = H; a.W = W;
  Arena ar(nullptr, 0);
  if (run_v1(e, a, ar, nullptr)) return 0;
  return e->prepared(shape_name(B, H, W), ar.peak + 256);
}

int udb_infer_v1(udb_engine_v1* e, const udb_infer_v1_args_t* a, void* stream) {
  if (!e || !a || !a->rgb || !a->workspace) { set_error("udb_infer_v1: null argument"); return 1; }
  if (!a->out_intrinsics || !a->out_points || !a->out_depth) { set_error("udb_infer_v1: all three output pointers are required"); return 1; }
  if (a->skip_camera && !a->intrinsics) { set_error("udb_infer_v1: skip_camera needs intrinsics"); return 1; }
  if (e->check_workspace("udb_infer_v1", "udb_v1_workspace_bytes", shape_name(a->B, a->H, a->W), a->workspace, a->workspace_bytes))
    return 1;
  Arena ar(a->workspace, a->workspace_bytes);
  return run_v1(e, *a, ar, stream);
}

}  // extern "C"
