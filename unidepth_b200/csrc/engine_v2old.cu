// Whole-path engine for UniDepthV2old.infer and the evaluation .forward (DINOv2 ViT-L/14 or ViT-S/14) behind
// udb_v2old_create / udb_v2old_set_weight / udb_v2old_workspace_bytes / udb_infer_v2old (include/udb.h).  Host-side
// schedule only, on the skeleton of the other two engines (engine_common.h): the shared DINOv2 patch embedding and block
// loop, V1's decoder stages (adapters, cls-token adapters, camera context, dense and Nystrom attention, ConvNeXt blocks,
// the heads' cross attention) and the V2old kernels of v1_kernels.cu.  Reference call stack:
//   UniDepthV2old.infer              unidepth/models/unidepthv2/unidepthv2_old.py:198-282 (_shapes/_preprocess/_postprocess :33-116)
//     pixel_encoder = DINOv2         backbones/dinov2.py:324-347 (use_norm: every block output through the final norm)
//     pixel_decoder = Decoder        unidepthv2/decoder_old.py:428-522 (CameraHead :32-86, GlobalHead :89-146,
//                                    DepthHead :149-343), layers/{attention,nystrom_attention,mlp,upsample,convnext}.py
#include "engine_common.h"

struct udb_engine_v2old : udb::EngineBase {
  udb_v2old_config_t cfg;
};

namespace udb {

constexpr int RAY_K = 128;          // 99 ray features (96 Fourier + the ray) zero-extended to the GEMM's K step
constexpr int RAY_BANDS = 32;       // camera_dim 96 / 3 axes

// unidepthv2_old.py:45-92 (Python float == C double; ceil(x - 0.5))
static udb_v2old_geometry_t v2old_geometry(int H, int W, int level, int lo, int hi) {
  udb_v2old_geometry_t g;
  const int lv = level < 0 ? 0 : (level > 10 ? 10 : level);
  g.pixels = lo + static_cast<int>(ceil(static_cast<double>(hi - lo) * lv / 10));
  const double ratio = static_cast<double>(W) / H;
  const double n = fmax(fmin((static_cast<double>(H) / 14) * (static_cast<double>(W) / 14), g.pixels), g.pixels);
  const int gh = static_cast<int>(ceil(sqrt(n / ratio) - 0.5));
  const int gw = static_cast<int>(ceil(gh * ratio - 0.5));
  g.net_h = gh * 14;
  g.net_w = gw * 14;
  g.ratio = static_cast<double>(gh) / H * 14;
  return g;
}

static int run_v2old(udb_engine_v2old* e, const udb_infer_v2old_args_t& a, Arena& ar, void* st) {
  const udb_v2old_config_t& cf = e->cfg;
  Ctx c{e, &ar, st, ar.dry};
  const int B = a.B, net_h = cf.net_h, net_w = cf.net_w, hid = cf.hidden, D = cf.embed_dim;
  const int gh = net_h / 14, gw = net_w / 14, N = gh * gw, T = N + 1, nq = N;
  const size_t BN = static_cast<size_t>(B) * N, BT = static_cast<size_t>(B) * T;
  const long long Rq = static_cast<long long>(B) * nq;
  // network-only mode (`forward`, unidepthv2_old.py:134-196): the input is the network input and the ratio 1
  const bool net_only = a.network_only != 0;
  const double ratio = net_only ? 1.0 : static_cast<double>(gh) / a.H * 14;     // unidepthv2_old.py:88
  // Nystrom attention with 128 landmarks at the first decoder level needs more tokens than landmarks, and the heads'
  // cross attention has a shared-memory bound: both named by the dry run before anything is launched
  if (nq <= 128) {
    set_error("udb_v2old: network shape %dx%d gives %d tokens; Nystrom attention needs more than its 128 landmarks", net_h, net_w, nq);
    return 1;
  }
  if (cross_attn_small_check("udb_v2old: camera head cross attention", 4, 4 * nq + 4, hid)) return 1;
  // "precision": 0 (absent) = f16 operands; 2 = e4m3 operands for the encoder blocks' four linear layers (the taps, heads
  // and decoder as in f16); 1 = split-f16 operands (parity mode): every GEMM on the path from the image to the intrinsics
  // and to the global (scale, shift) -- patch embedding, encoder blocks, the adapters' copy for the two heads, the camera
  // head's in_features and kv, the global head's project_rays, in_features and kv -- multiplies [hi | lo] operands with
  // [hi | hi | lo] weights; the taps and the two heads' contexts are f32.  The depth head reads the hi half of the
  // adapters' LayerNorm and of the first level's ray features and runs as in the f16 mode.
  const Precision prec = encoder_precision(c, "udb_infer_v2old", "patch_w", 3 * 640);
  if (prec == PREC_BAD) return 1;
  const bool sp = prec == PREC_SPLIT;
  const int sx = sp ? 2 : 1;          // columns of a split operand per logical column
  const int kx = sp ? 3 : 1;          // columns of a split weight per logical column
  const int widths[4] = {D, D, D, D}; // of every tap and cls token
  Stage stage;

  // ---- pre-processing + patch embedding (unidepthv2_old.py:211-230: /255, ImageNet normalisation, antialiased resize)
  stage.next("udb_v2old:encoder");
  // the four tapped final-norm outputs: f16, or f32 in split mode (the adapters' LayerNorm writes their split operands)
  void* feats[4];
  for (int l = 0; l < 4; ++l) feats[l] = ar.alloc(BN * D * (sp ? 4 : 2));
  // normed cls rows of the last three blocks (cls[-3..-1]) and of the third output block (the stacked tokens[-2])
  float* cls[4];
  for (int k = 0; k < 4; ++k) cls[k] = ar.f(static_cast<size_t>(B) * D);
  {
    const size_t m = ar.mark();
    __half* patches = ar.h(BN * 640 * sx);
    {
      udb_v1_preprocess_t p;
      memset(&p, 0, sizeof(p));
      p.rgb = a.rgb; p.rgb_is_u8 = a.rgb_is_u8; p.scale255 = a.scale255; p.normalize = a.normalize; p.B = B; p.H = a.H; p.W = a.W;
      p.rh = net_h; p.rw = net_w; p.net_h = net_h; p.net_w = net_w; p.patches = patches; p.patch = 14;
      c.launch([&] { return sp ? udb_v1_preprocess_split(&p, st) : udb_v1_preprocess(&p, st); });
    }
    float* x = ar.f(BT * D);
    VitBlocks v{B, T, D, cf.enc_heads, cf.enc_depth};
    v.fp8 = prec == PREC_E4M3;
    v.split = sp;
    c.expect2("pos", T, D);
    vit_embed(c, patches, c.F("pos"), x, v);
    int tap = 0;
    vit_blocks(c, "blocks.", x, v, [&](int i) {
      if (tap < 4 && i + 1 == cf.output_idx[tap]) {
        c.layernorm(x, 1, feats[tap], sp ? 1 : 0, c.F("norm_w"), c.F("norm_b"), static_cast<int>(BN), D, 1e-5f, N, T, 1);
        ++tap;
      }
      const int from_end = cf.enc_depth - 1 - i;
      if (from_end < 3) c.layernorm(x, 1, cls[2 - from_end], 1, c.F("norm_w"), c.F("norm_b"), B, D, 1e-5f, 1, T, 0);
      if (i + 1 == cf.output_idx[2]) c.layernorm(x, 1, cls[3], 1, c.F("norm_w"), c.F("norm_b"), B, D, 1e-5f, 1, T, 0);
    });
    ar.release(m);
  }

  // ---- adapters (decoder_old.py:448-461): tokens [B, 4*nq, hid] for the context and featcat [B*nq, 4*hid] for the latents
  stage.next("udb_v2old:adapters");
  __half* featcat = ar.h(Rq * 4 * hid);
  __half* tokens = ar.h((Rq * 4 + 64) * hid);
  // split mode: the two heads' copy of the tokens from split operands, f32 for the camera head's LayerNorm and as a split
  // operand for the global head's in_features GEMM (the depth head keeps the f16 tokens)
  float* head_tokens = sp ? ar.f(Rq * 4 * hid) : nullptr;
  __half* head_tokens2 = sp ? ar.h(Rq * 4 * 2 * hid) : nullptr;
  const int grid_h[4] = {gh, gh, gh, gh}, grid_w[4] = {gw, gw, gw, gw};
  adapters(c, feats, widths, grid_h, grid_w, B, gh, gw, hid, sp, tokens, featcat, head_tokens, head_tokens2);
  const float* tokens_pos = c.F("tokens_pos");         // [4*nq, hid]: sine position + level embedding (decoder_old.py:463-479)
  c.expect2("tokens_pos", 4LL * nq, hid);

  // ---- camera head (decoder_old.py:378-406, 66-83)
  stage.next("udb_v2old:camera_head");
  float* intr4 = ar.f(static_cast<size_t>(B) * 4);
  float* k4_points = ar.f(static_cast<size_t>(B) * 4);
  {
    const size_t m = ar.mark();
    const int R4 = B * 4;
    float* toks = token_adapter(c, "ctok.", cls, widths, 4, B, hid);
    float* cl = cam_mlp(c, "cam.cls", toks, R4, hid, 4 * hid, hid, nullptr, nullptr);
    const void* ctx = camera_context(c, sp ? static_cast<const void*>(head_tokens) : tokens, tokens_pos, cl, B, nq, 4, hid, sp);
    const float* cam_pos = c.F("cam.pos");
    float* t = small_cross_block(c, "cam.agg1.", cl, B, 4, ctx, 4LL * nq + 4, cam_pos, hid, cf.expansion, sp);
    t = small_cross_block(c, "cam.agg2.", t, B, 4, ctx, 4LL * nq + 4, cam_pos, hid, cf.expansion, sp);
    float* x4 = cam_mlp(c, "cam.out", t, R4, hid, 2 * hid, 1, nullptr, nullptr);     // [B*4, 1] == [B, 4]
    if (net_only && a.intrinsics) {
      // `forward` with K: the rays follow the given K, the points the prediction (unidepthv2_old.py:154-159).  At ratio 1
      // the kernel writes the same values to its rays and points outputs, so each call passes one buffer for both: the
      // prediction into k4_points, then the given K into intr4.  out_intrinsics is the prediction in both calls.
      c.launch([&] { return udb_v2old_camera(x4, nullptr, B, net_h, net_w, 1.f, k4_points, a.out_intrinsics, k4_points, st); });
      c.launch([&] { return udb_v2old_camera(x4, a.intrinsics, B, net_h, net_w, 1.f, intr4, a.out_intrinsics, intr4, st); });
    } else {
      c.launch([&] {
        return udb_v2old_camera(x4, a.intrinsics, B, net_h, net_w, static_cast<float>(ratio), intr4, a.out_intrinsics, k4_points, st);
      });
    }
    ar.release(m);
  }

  // ---- ray features at the three decoder grids (GlobalHead / DepthHead.embed_rays, decoder_old.py:111-121,237-255)
  stage.next("udb_v2old:ray_features");
  // split mode: the first level, which the global head reads, as [hi | lo] rows; the depth head reads its hi half
  __half* rayf[3];
  int ray_ld[3];
  for (int s = 0; s < 3; ++s) {
    const int lh = gh << s, lw = gw << s;
    const bool split_rays = sp && s == 0;
    ray_ld[s] = split_rays ? 2 * RAY_K : RAY_K;
    rayf[s] = ar.h(static_cast<size_t>(B) * lh * lw * ray_ld[s]);
    udb_ray_embed_t p;
    memset(&p, 0, sizeof(p));
    p.intr4 = intr4; p.scales = c.F(idx("ray_scales.%d", s)); p.B = B; p.net_h = net_h; p.net_w = net_w; p.gh = lh; p.gw = lw;
    p.bands = RAY_BANDS; p.out = rayf[s]; p.out_f32 = split_rays ? 2 : 0;
    const int ld = ray_ld[s];
    c.launch([&] { return udb_ray_embed_cat_orig(&p, ld, st); });
  }

  // ---- global head (decoder_old.py:408-426, 135-146): (scale, shift) of the depth
  stage.next("udb_v2old:global_head");
  float* scale_shift = ar.f(static_cast<size_t>(B) * 2);
  {
    const size_t m = ar.mark();
    const int R2 = B * 2;
    float* gtok[2] = {cls[1], cls[2]};
    float* toks = token_adapter(c, "gtok.", gtok, widths, 2, B, hid);
    float* gcl = cam_mlp(c, "glob.cls", toks, R2, hid, 4 * hid, hid, nullptr, nullptr);
    // in_features(features + project_rays(rays)) = W_in features + (W_in project_rays(rays) + b_in), the second term per
    // token of the grid and shared by the four levels
    // split mode: the same three GEMMs on split operands ([N, 3K] weights), project_rays writing a split operand for
    // in_features, and an f32 context
    __half* pr = ar.h(Rq * hid * sx);
    c.expect2("glob.rays_w", hid, RAY_K * kx);
    c.expect2("glob.in_w", hid, hid * kx);
    { Ctx::G q{rayf[0], c.H("glob.rays_w"), static_cast<int>(Rq), hid, RAY_K * kx}; q.lda = ray_ld[0]; q.a_split_k = sp ? RAY_K : 0;
      q.bias = c.F("glob.rays_b"); q.out = pr; q.ldc = hid * sx; q.out_split = sp ? hid : 0; c.gemm(q); }
    float* rr = ar.f(Rq * hid);
    { Ctx::G q{pr, c.H("glob.in_w"), static_cast<int>(Rq), hid, hid * kx}; q.lda = hid * sx; q.a_split_k = sp ? hid : 0;
      q.bias = c.F("glob.in_b"); q.out = rr; q.out_f32 = 1; c.gemm(q); }
    const long long nk = 4LL * nq + 2;
    void* gctx = ar.alloc(B * nk * hid * (sp ? 4 : 2));
    for (int b = 0; b < B; ++b) {
      const __half* tb = sp ? head_tokens2 + static_cast<long long>(b) * 4 * nq * 2 * hid : tokens + static_cast<long long>(b) * 4 * nq * hid;
      Ctx::G q{tb, c.H("glob.in_w"), 4 * nq, hid, hid * kx}; q.lda = hid * sx; q.a_split_k = sp ? hid : 0;
      q.resid = rr + static_cast<long long>(b) * nq * hid; q.resid_f32 = 1; q.ldr = hid; q.resid_mod = nq; q.resid_row_offset = 0;
      q.out = static_cast<char*>(gctx) + static_cast<long long>(b) * nk * hid * (sp ? 4 : 2); q.out_f32 = sp ? 1 : 0; c.gemm(q);
    }
    copy_cls_rows(c, gcl, gctx, B, 2, hid, nk, 4LL * nq, sp);
    float* t = small_cross_block(c, "glob.agg1.", gcl, B, 2, gctx, nk, nullptr, hid, cf.expansion, sp);
    t = small_cross_block(c, "glob.agg2.", t, B, 2, gctx, nk, nullptr, hid, cf.expansion, sp);
    float* x2 = cam_mlp(c, "glob.out", t, R2, hid, 2 * hid, 1, nullptr, nullptr);    // [B*2, 1] == [B, 2]: log scale, shift
    c.launch([&] {
      return cuda_rc(cudaMemcpyAsync(scale_shift, x2, sizeof(float) * 2 * B, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(st)),
                     "engine_v2old: copying the global head's scale and shift");
    });
    ar.release(m);
  }

  // ---- depth head (decoder_old.py:317-343)
  stage.next("udb_v2old:depth_head");
  float* emb[3];
  for (int s = 0; s < 3; ++s) {
    const long long R = static_cast<long long>(B) * (gh << s) * (gw << s);
    const std::string n = idx("rays.%d.", s);
    emb[s] = ar.f(R * (hid >> s));
    c.expect2(n + "w", hid >> s, RAY_K);
    Ctx::G q{rayf[s], c.H(n + "w"), static_cast<int>(R), hid >> s, RAY_K}; q.lda = ray_ld[s];
    q.bias = c.F(n + "b"); q.out = emb[s]; q.out_f32 = 1; c.gemm(q);
  }
  float* lat = ar.f(Rq * hid);
  {
    const size_t m = ar.mark();
    __half* f16l = ar.h(Rq * hid);
    { Ctx::G q{featcat, c.H("fcc_w"), static_cast<int>(Rq), hid, 4 * hid}; q.bias = c.F("fcc_b"); q.out = f16l; c.gemm(q); }
    __half* hN = ar.h(Rq * hid);
    __half* md = ar.h(Rq * 2 * hid);
    ln16(c, f16l, 0, hN, "lat.nw", "lat.nb", Rq, hid, 1e-5f);
    { Ctx::G q{hN, c.H("lat.w1"), static_cast<int>(Rq), 2 * hid, hid}; q.bias = c.F("lat.b1"); q.act = UDB_ACT_GELU; q.out = md; c.gemm(q); }
    { Ctx::G q{md, c.H("lat.w2"), static_cast<int>(Rq), hid, 2 * hid}; q.bias = c.F("lat.b2"); q.resid = f16l; q.resid_f32 = 0;
      q.out = lat; q.out_f32 = 1; c.gemm(q); }
    ar.release(m);
  }
  dense_attn_block(c, "agg16.", lat, B, nq, hid, tokens, 0, 4 * nq, tokens_pos);
  dense_attn_block(c, "prompt.", lat, B, nq, hid, emb[0], 1, nq, nullptr);
  if (a.out_depth_features)          // `forward`'s "depth_features" (decoder_old.py:339-343)
    c.launch([&] {
      return cuda_rc(cudaMemcpyAsync(a.out_depth_features, lat, sizeof(float) * Rq * hid, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(st)),
                     "engine_v2old: copying the depth features");
    });
  for (int i = 0; i < cf.nystrom_depth; ++i) mh_attn_block(c, idx("nys.%d.", i), lat, B, nq, hid, cf.heads, emb[0], true);

  // ConvUpsampleShuffleResidual per level (layers/upsample.py:82-130), then the level's [depth | confidence] MLPs
  float* heads_in[3];
  int ch = gh, cw = gw, C = hid;
  for (int s = 0; s < 3; ++s) {
    const std::string u = idx("up.%d.", s);
    const long long R = static_cast<long long>(B) * ch * cw, Rn = 4 * R;
    const int C2 = C / 2, Cq = C / 4, Cqp = static_cast<int>(rup(Cq, 64));
    float* nxt = ar.f(Rn * C2);
    heads_in[s] = ar.f(Rn * 32);
    const size_t m = ar.mark();
    float* xs = ar.f(R * C);
    __half* xs16 = ar.h(R * C);
    c.launch([&] { return udb_add_f32(lat, emb[s], xs, xs16, R * C, st); });
    for (int j = 0; j < 2; ++j) cvnxt_block(c, u + (j ? "c1." : "c0."), xs, xs16, B, ch, cw, C, 1e-5f);
    __half* r1 = ar.h(R * C2);
    { Ctx::G q{xs16, c.H(u + "res_w"), static_cast<int>(R), C2, C}; q.bias = c.F(u + "res_b"); q.out = r1; c.gemm(q); }
    __half* res = ar.h(Rn * C2);
    c.launch([&] { return udb_resize_ac_pad_nhwc_f16(r1, res, B, ch, cw, C2, 2 * ch, 2 * cw, 0, st); });
    __half* sh = ar.h(Rn * Cqp);
    const float* dw_w = c.F(u + "dw_w");
    const float* dw_b = c.F(u + "dw_b");
    c.launch([&] { return udb_pshuffle_dw7_relu(xs16, dw_w, dw_b, sh, B, ch, cw, C, Cqp, st); });
    c.expect2(u + "conv_w", C2, 9 * Cqp);
    __half* nxt16 = ar.h(Rn * C2);
    c.conv3x3(sh, B, 2 * ch, 2 * cw, Cqp, c.H(u + "conv_w"), C2, c.F(u + "conv_b"), UDB_ACT_NONE, nullptr, res, 0, nxt, 1, nxt16, 0);
    // depth_mlp / confidence_mlp (LN -> Linear -> GELU -> Linear(-> 16)) side by side: [hd | hc] then one block-diagonal GEMM
    const std::string hm = idx("hmlp.%d.", s);
    __half* hn = ar.h(Rn * C2);
    __half* hm1 = ar.h(Rn * C);
    for (int k = 0; k < 2; ++k) {
      const std::string p = hm + (k ? "c." : "d.");
      ln16(c, nxt, 1, hn, p + "nw", p + "nb", Rn, C2, 1e-5f);
      Ctx::G q{hn, c.H(p + "w1"), static_cast<int>(Rn), C2, C2}; q.bias = c.F(p + "b1"); q.act = UDB_ACT_GELU; q.out = hm1 + k * C2; q.ldc = C; c.gemm(q);
    }
    c.expect2(hm + "w2", 32, C);
    { Ctx::G q{hm1, c.H(hm + "w2"), static_cast<int>(Rn), 32, C}; q.bias = c.F(hm + "b2"); q.out = heads_in[s]; q.out_f32 = 1; c.gemm(q); }
    ar.release(m);
    lat = nxt;
    ch *= 2; cw *= 2; C = C2;
  }

  // ---- depth / confidence convolutions at the network shape, the depth tail, output assembly (unidepthv2_old.py:107-116,262-274)
  stage.next("udb_v2old:heads+postprocess");
  const long long nhw = static_cast<long long>(net_h) * net_w;
  float* dmap = ar.f(B * nhw);
  float* cmap = ar.f(B * nhw);
  {
    udb_v2old_heads_t p;
    memset(&p, 0, sizeof(p));
    for (int s = 0; s < 3; ++s) p.levels[s] = heads_in[s];
    p.w = c.F("head_w"); p.bias_depth = static_cast<float>(c.S("head_b_depth")); p.bias_conf = static_cast<float>(c.S("head_b_conf"));
    p.B = B; p.gh = gh; p.gw = gw; p.net_h = net_h; p.net_w = net_w; p.logdepth = dmap; p.confidence = cmap;
    c.launch([&] { return udb_v2old_heads(&p, st); });
  }
  c.launch([&] { return udb_v2old_depth_tail(dmap, scale_shift, B, nhw, st); });
  {
    udb_v2old_postprocess_t p;
    memset(&p, 0, sizeof(p));
    p.depth = dmap; p.confidence = cmap; p.k4 = k4_points; p.B = B; p.net_h = net_h; p.net_w = net_w;
    p.H = net_only ? a.out_h : a.H; p.W = net_only ? a.out_w : a.W;
    p.mode = a.interpolation; p.out_depth = a.out_depth; p.out_confidence = a.out_confidence; p.out_points = a.out_points;
    p.depth_aa = net_only ? 1 : 0;
    c.launch([&] { return udb_v2old_postprocess(&p, st); });
  }
  if (!c.rc && ar.overflow) { set_error("engine_v2old: workspace too small (%zu bytes needed)", ar.peak); return 1; }
  return c.rc;
}

static size_t dry_run(udb_engine_v2old* e, int B, int H, int W) {
  if (!e || B <= 0 || H <= 0 || W <= 0) { set_error("udb_v2old_workspace_bytes: bad argument"); return 0; }
  udb_infer_v2old_args_t a;
  memset(&a, 0, sizeof(a));
  a.B = B; a.H = H; a.W = W;
  Arena ar(nullptr, 0);
  if (run_v2old(e, a, ar, nullptr)) return 0;
  return ar.peak + 256;
}

}  // namespace udb

using namespace udb;

extern "C" {

int udb_v2old_create(const udb_v2old_config_t* cfg, udb_engine_v2old** out) {
  if (!cfg || !out) { set_error("udb_v2old_create: null argument"); return 1; }
  if (cfg->embed_dim <= 0 || cfg->embed_dim % 128 || cfg->embed_dim > 1024 || cfg->enc_heads <= 0 || cfg->embed_dim / cfg->enc_heads != 64) {
    set_error("udb_v2old_create: encoder width %d / heads %d: 64-wide heads and a width that is a multiple of 128 up to 1024",
              cfg->embed_dim, cfg->enc_heads);
    return 1;
  }
  for (int i = 0; i < 4; ++i)
    if (cfg->output_idx[i] < 1 || cfg->output_idx[i] > cfg->enc_depth || (i && cfg->output_idx[i] <= cfg->output_idx[i - 1])) {
      set_error("udb_v2old_create: output_idx must be four increasing block indices in [1, %d]", cfg->enc_depth);
      return 1;
    }
  if (cfg->enc_depth < 3) { set_error("udb_v2old_create: the camera head reads the cls tokens of the last three blocks (depth %d)", cfg->enc_depth); return 1; }
  if (cfg->hidden != 512 || cfg->heads != 8 || cfg->expansion != 4) {
    set_error("udb_v2old_create: decoder hidden %d / heads %d / expansion %d not supported (512 / 8 / 4)", cfg->hidden, cfg->heads, cfg->expansion);
    return 1;
  }
  if (cfg->nystrom_depth < 0) { set_error("udb_v2old_create: nystrom_depth %d must be >= 0", cfg->nystrom_depth); return 1; }
  if (cfg->net_h < 56 || cfg->net_w < 56 || cfg->net_h % 14 || cfg->net_w % 14) {
    set_error("udb_v2old_create: network shape %dx%d must be multiples of 14, at least 56", cfg->net_h, cfg->net_w);
    return 1;
  }
  udb_engine_v2old* e = new udb_engine_v2old();
  e->cfg = *cfg;
  *out = e;
  return 0;
}

void udb_v2old_destroy(udb_engine_v2old* e) { delete e; }

int udb_v2old_geometry(int32_t H, int32_t W, int32_t resolution_level, int32_t pixels_lo, int32_t pixels_hi, udb_v2old_geometry_t* out) {
  if (!out || H <= 0 || W <= 0 || pixels_lo <= 0 || pixels_hi < pixels_lo) { set_error("udb_v2old_geometry: bad argument"); return 1; }
  *out = v2old_geometry(H, W, resolution_level, pixels_lo, pixels_hi);       // the function the Python boundary keys engines by
  return 0;
}

int udb_v2old_set_weight(udb_engine_v2old* e, const char* name, const void* dev_ptr, const int64_t* shape, int32_t ndim, int32_t dtype) {
  return EngineBase::set_weight(e, "udb_v2old_set_weight", name, dev_ptr, shape, ndim, dtype);
}

int udb_v2old_set_scalar(udb_engine_v2old* e, const char* name, double value) {
  return EngineBase::set_scalar(e, "udb_v2old_set_scalar", name, value);
}

size_t udb_v2old_schedule_bytes(udb_engine_v2old* e, int32_t B, int32_t H, int32_t W) { return dry_run(e, B, H, W); }

size_t udb_v2old_workspace_bytes(udb_engine_v2old* e, int32_t B, int32_t H, int32_t W) {
  const size_t n = dry_run(e, B, H, W);
  return n ? e->prepared(shape_name(B, H, W), n) : 0;
}

int udb_infer_v2old(udb_engine_v2old* e, const udb_infer_v2old_args_t* a, void* stream) {
  if (!e || !a || !a->rgb || !a->workspace) { set_error("udb_infer_v2old: null argument"); return 1; }
  if (!a->out_intrinsics || !a->out_points || !a->out_depth || !a->out_confidence) {
    set_error("udb_infer_v2old: all four output pointers are required");
    return 1;
  }
  if (!a->network_only && a->interpolation != UDB_V2OLD_BILINEAR && a->interpolation != UDB_V2OLD_NEAREST_EXACT) {
    set_error("udb_infer_v2old: `interpolation` %d is neither UDB_V2OLD_BILINEAR (0) nor UDB_V2OLD_NEAREST_EXACT (1)", a->interpolation);
    return 1;
  }
  if (a->network_only != 0 && a->network_only != 1) { set_error("udb_infer_v2old: `network_only` %d is neither 0 nor 1", a->network_only); return 1; }
  if (!a->network_only && (a->out_h || a->out_w || a->out_depth_features)) {
    set_error("udb_infer_v2old: out_h, out_w and out_depth_features are read in network-only mode only (network_only = 1)");
    return 1;
  }
  if (a->network_only) {
    const udb_v2old_config_t& cf = e->cfg;
    if (a->rgb_is_u8 || a->scale255 || a->normalize) {
      set_error("udb_infer_v2old: network-only input must be f32 and already normalised (rgb_is_u8 %d, scale255 %d, normalize %d must be 0)",
                a->rgb_is_u8, a->scale255, a->normalize);
      return 1;
    }
    if (a->H != cf.net_h || a->W != cf.net_w) {
      set_error("udb_infer_v2old: network-only input is %dx%d but the engine's network shape is %dx%d", a->H, a->W, cf.net_h, cf.net_w);
      return 1;
    }
    if (a->out_h < 1 || a->out_w < 1) { set_error("udb_infer_v2old: network-only output size %dx%d must be positive", a->out_h, a->out_w); return 1; }
    if (a->intrinsics && (a->out_h != a->H || a->out_w != a->W)) {
      set_error("udb_infer_v2old: a given K needs the output size %dx%d to equal the network input's %dx%d (the reference reshapes "
                "its rays to the image grid)", a->out_h, a->out_w, a->H, a->W);
      return 1;
    }
  }
  if (e->check_workspace("udb_infer_v2old", "udb_v2old_workspace_bytes", shape_name(a->B, a->H, a->W), a->workspace, a->workspace_bytes))
    return 1;
  Arena ar(a->workspace, a->workspace_bytes);
  return run_v2old(e, *a, ar, stream);
}

}  // extern "C"
