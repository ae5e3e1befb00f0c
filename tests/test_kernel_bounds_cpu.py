"""The per-element bounds of tests/kernel_ref.py, which tests/test_kernel_conformance_gpu.py holds the kernels to, on the
CPU: a float32 model of each kernel's arithmetic (f16 operands, f32 accumulation, f16 rounding where the kernel rounds)
stays inside them, and each of these plausible kernel bugs falls outside them:

  a dropped K-tail block, two adjacent output columns swapped, an off-by-one row map, an unmasked zero-filled key in the
  last tile, a key leaked from the next image, a padded head scaled by 1/sqrt(64) instead of 1/sqrt(true dim), and a
  halo tap read one pixel off;

  and for the CUDA-core kernels: a dropped row of a partly filled warp, LayerNorm statistics over dim instead of
  dim_valid, a swapped space-to-depth quadrant, softmax over ld_in instead of n_valid, an empty cross-attention split
  merged with weight 1, an antialias window one tap short, reflect instead of zero padding in the single-output conv, a
  dropped K tail of the f32 dense layer, dropped tail pixels of the spatial mean, an align-corners source index in the 2x
  upsample, a reflect index one off, a head scaled by the full width, equal Nystrom segments, part statistics centred on
  the whole row, a back-projection through the pixel corner, and a Newton-Schulz run one iteration short.

The kernels that only copy, add once or take a maximum have no bound: tests/test_cuda_core_conformance_gpu.py compares
them bit for bit, which is their guard."""
import math

import torch
import torch.nn.functional as F

import kernel_ref as R


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _gemm_model(a, w, bias):
    """what the GEMM kernel computes: exact f16 products summed in f32, f32 bias, f16 output"""
    return (a.float() @ w.float().T + bias).half()


def _attn_model(q, k, v, scale):
    """the attention kernel's arithmetic: f32 logits and softmax, P rounded to f16 for PV, l from the f32 P, f16 output"""
    s = q.float() @ k.float().transpose(-1, -2) * scale
    p = torch.exp(s - s.amax(-1, keepdim=True))
    return ((p.half().float() @ v.float()) / p.sum(-1, keepdim=True)).half()


def _rejects(got, ref, bound):
    r = R.ratio(got, ref, bound)
    print(f"max err/bound of the planted bug: {r:.3g}")
    return r > 1.0


def test_gemm_bound_rejects_dropped_k_tail_and_swapped_columns():
    g = _gen(0)
    M, N, K = 40, 64, 72                                   # K = 72: one full k-block and an 8-wide tail
    a = torch.randn(M, K, generator=g).half()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).half()
    bias = torch.randn(N, generator=g)
    ref, bnd = R.gemm_ref(a, w, bias=bias)
    bnd = R.f16_out(ref, bnd)
    good = _gemm_model(a, w, bias)
    R.within(good, ref, bnd, "f32 model of the GEMM")
    assert _rejects(_gemm_model(a[:, :64], w[:, :64], bias), ref, bnd)         # the tail k-block never accumulated
    swapped = good.clone()
    swapped[:, [36, 37]] = swapped[:, [37, 36]]                                   # two adjacent columns of one store
    assert _rejects(swapped, ref, bnd)


def test_gemm_bound_rejects_off_by_one_row_map():
    g = _gen(1)
    Bn, Np, N, K = 3, 50, 32, 64
    T = Np + 1
    a = torch.randn(Bn * Np, K, generator=g).half()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).half()
    pos = torch.randn(T, N, generator=g)
    ref, bnd = R.gemm_ref(a, w, resid=pos[1:].repeat(Bn, 1))
    lin = a.float() @ w.float().T

    def store(row_offset):                                 # rows b*T + row_offset + n of the token map
        x = torch.zeros(Bn * T + 1, N)
        for b in range(Bn):
            x[b * T + row_offset:b * T + row_offset + Np] = lin[b * Np:(b + 1) * Np] + pos[1:]
        return torch.cat([x[b * T + 1:b * T + 1 + Np] for b in range(Bn)])

    R.within(store(1), ref, bnd, "row map")
    assert _rejects(store(2), ref, bnd)


def test_attention_bound_rejects_unmasked_zero_key():
    """seq_k = 130: the last tile holds 2 valid keys; a third, zero-filled one that escapes the mask gets weight
    exp(0 - m) on a zero V row"""
    g = _gen(2)
    q, k, v = R.attn_inputs(1, 2, 64, 130, g)
    ref, bnd = R.attention_ref(q, k, v, 0.125)
    R.within(_attn_model(q, k, v, 0.125), ref, bnd, "f32 model of the attention kernel")
    z = torch.zeros(1, 2, 1, 64, dtype=torch.float16)
    assert _rejects(_attn_model(q, torch.cat([k, z], 2), torch.cat([v, z], 2), 0.125), ref, bnd)


def test_attention_bound_rejects_key_from_next_image():
    g = _gen(3)
    q, k, v = R.isolation_inputs(2, 64, 130, g)
    ref, bnd = R.attention_ref(q[:1], k[:1], v[:1], 0.125)
    R.within(_attn_model(q[:1], k[:1], v[:1], 0.125), ref, bnd, "isolation, image 0")
    leaked_k, leaked_v = torch.cat([k[:1], k[1:, :, :1]], 2), torch.cat([v[:1], v[1:, :, :1]], 2)
    assert _rejects(_attn_model(q[:1], leaked_k, leaked_v, 0.125), ref, bnd)


def test_attention_bound_rejects_padded_head_with_scale_of_64():
    g = _gen(4)
    q, k, v = R.attn_inputs(1, 2, 64, 200, g)
    for t in (q, k, v):
        t[..., 32:] = 0                                    # true head dim 32, zero-padded to 64
    ref, bnd = R.attention_ref(q, k, v, 32 ** -0.5)
    R.within(_attn_model(q, k, v, 32 ** -0.5), ref, bnd, "padded head")
    assert _rejects(_attn_model(q, k, v, 64 ** -0.5), ref, bnd)


def test_halo_bound_rejects_tap_shifted_by_one_pixel():
    g = _gen(5)
    B, H, W, C, N = 1, 9, 11, 64, 32
    xp = torch.randn(B, H + 2, W + 2, C, generator=g).half()
    w = (torch.randn(N, 9 * C, generator=g) / (9 * C) ** 0.5).half()
    bias = torch.randn(N, generator=g)
    ref, bnd = R.conv3x3_ref(xp, w, bias=bias)
    bnd = R.f16_out(ref, bnd)
    xt, wt = xp.float().permute(0, 3, 1, 2), w.float().view(N, 3, 3, C).permute(0, 3, 1, 2)
    good = (F.conv2d(xt, wt).permute(0, 2, 3, 1) + bias).half()
    R.within(good, ref, bnd, "f32 model of the halo conv")
    # tap (dy, dx) = (1, 2) reads pixel x + 1 (its column one further right, clamped at the edge)
    xs = torch.cat([xt[..., 1:], xt[..., -1:]], -1)
    wtap = torch.zeros_like(wt)
    wtap[:, :, 1, 2] = wt[:, :, 1, 2]
    shifted = (F.conv2d(xt, wt - wtap) + F.conv2d(xs, wtap)).permute(0, 2, 3, 1) + bias
    assert _rejects(shifted.half(), ref, bnd)


# ------------------------------------------------------------------------------------------------ CUDA-core kernels
def _ln_model(x, w, b, eps, n=None):
    """the LayerNorm kernels' arithmetic in f32: mean, two-pass variance, rsqrt, (x - m) rstd w + b"""
    x = x.float()
    n = x.shape[-1] if n is None else n
    m = x[:, :n].sum(-1, keepdim=True) / n
    d = x - m
    v = (d[:, :n] * d[:, :n]).sum(-1, keepdim=True) / n
    return d * torch.rsqrt(v + eps) * w + b


def test_layernorm_bound_rejects_dropped_row_of_a_warp():
    """rows = 4 k + 1 with four rows per warp: the last warp holds one live row; a kernel that skips it leaves the
    output's (zero) initial value there"""
    g = _gen(10)
    rows, dim = 13, 192
    x = (torch.randn(rows, dim, generator=g) * 3 + 1).half()
    w, b = torch.randn(dim, generator=g), torch.randn(dim, generator=g)
    ref, bnd = R.layernorm_ref(x, w, b, 1e-6)
    bnd16 = R.f16_out(ref, bnd)
    good = _ln_model(x, w, b, 1e-6)
    R.within(good, ref, bnd, "f32 model of layernorm_any (f32 out)")
    R.within(good.half(), ref, bnd16, "f32 model of layernorm_any (f16 out)")
    dropped = good.half().clone()
    dropped[-1] = 0
    assert _rejects(dropped, ref, bnd16)


def test_layernorm_bound_rejects_statistics_over_dim_instead_of_dim_valid():
    g = _gen(11)
    rows, dim, n = 40, 128, 96                             # a 96-channel map stored as 128 zero-padded columns
    x = torch.randn(rows, dim, generator=g).half()
    x[:, n:] = 0
    w, b = torch.randn(dim, generator=g), torch.randn(dim, generator=g)
    ref, bnd = R.layernorm_ref(x, w, b, 1e-5, n)
    bnd16 = R.f16_out(ref, bnd)
    R.within(_ln_model(x, w, b, 1e-5, n).half(), ref, bnd16, "f32 model, dim_valid")
    assert _rejects(_ln_model(x, w, b, 1e-5).half(), ref, bnd16)


def test_layernorm_split_output_and_s2d_quadrant_order():
    """split output: hi + lo inside the f32 bound; space-to-depth: columns ((y&1)*2 + (x&1))*C, a swapped quadrant order
    (x parity first) falls outside"""
    g = _gen(12)
    B, H, W, C = 1, 4, 6, 64
    x = torch.randn(B * H * W, C, generator=g) * 2
    w, b = torch.randn(C, generator=g), torch.randn(C, generator=g)
    ref, bnd = R.layernorm_ref(x, w, b, 1e-6)
    y = _ln_model(x, w, b, 1e-6)
    hi = y.half()
    lo = (y - hi.float()).half()
    bhi, bsum = R.split_out(ref, bnd, hi, lo)
    R.within(hi, ref, bhi, "split hi")
    R.within(hi.double() + lo.double(), ref, bsum, "split hi + lo")

    def s2d(t, swap):
        t = t.reshape(B, H // 2, 2, W // 2, 2, C)
        t = t.permute(0, 1, 3, 4, 2, 5) if swap else t.permute(0, 1, 3, 2, 4, 5)
        return t.reshape(B * (H // 2) * (W // 2), 4 * C)

    R.within(s2d(y, False), s2d(ref, False), s2d(bnd, False), "s2d")
    assert _rejects(s2d(y, True), s2d(ref, False), s2d(bnd, False))


def test_softmax_rows_bound_rejects_softmax_over_ld_in():
    g = _gen(13)
    rows, n_valid, ld_in = 20, 21, 32
    s = torch.randn(rows, ld_in, generator=g) * 4
    P, bnd = R.softmax_rows_ref(s, n_valid, 0.7)
    t = s * 0.7
    e = torch.exp(t[:, :n_valid] - t[:, :n_valid].amax(-1, keepdim=True))
    R.within((e / e.sum(-1, keepdim=True)).half(), P, bnd, "f32 model of softmax_rows")
    assert _rejects(torch.softmax(t, -1)[:, :n_valid].half(), P, bnd)


def _cross_attn_model(q, kv, nk, D, scale, empty_weight_one=False):
    """cross_attn_partial + merge in f32: 16 key splits of ceil(nk / 16) keys, partial (max, sum, weighted V), merge.
    empty_weight_one: a split without keys reports max 0 and sum 1 instead of -inf and 0"""
    qs = q.float() * scale
    k, v = kv[:, :D].float(), kv[:, D:].float()
    chunk = -(-nk // 16)
    parts = []
    for sp in range(16):
        j0, j1 = sp * chunk, min(nk, sp * chunk + chunk)
        if j1 <= j0:
            m = torch.zeros(q.shape[0]) if empty_weight_one else torch.full((q.shape[0],), -math.inf)
            parts.append((m, torch.ones_like(m) if empty_weight_one else torch.zeros_like(m), torch.zeros(q.shape[0], D)))
            continue
        sc = qs @ k[j0:j1].T
        m = sc.amax(-1)
        e = torch.exp(sc - m[:, None])
        parts.append((m, e.sum(-1), e @ v[j0:j1]))
    M = torch.stack([p[0] for p in parts]).amax(0)
    wgt = [torch.exp(p[0] - M) for p in parts]
    tot = sum(w_ * p[1] for w_, p in zip(wgt, parts))
    return sum(w_[:, None] * p[2] for w_, p in zip(wgt, parts)) / tot[:, None]


def test_cross_attention_bound_rejects_empty_split_merged_with_weight_one():
    """nk = 9 < 16 splits: seven splits get no key"""
    g = _gen(14)
    nq, nk, D = 3, 9, 256
    q = torch.randn(nq, D, generator=g)
    kv = torch.randn(nk, 2 * D, generator=g).half()
    scale = D ** -0.5
    s = (q.double() * scale) @ kv[:, :D].double().T
    ds = (D + 4) * R.U32 * ((q.double().abs() * scale) @ kv[:, :D].double().abs().T)
    ref, bnd = R.softmax_av_ref(s, ds, kv[:, D:], nk + 16)
    R.within(_cross_attn_model(q, kv, nk, D, scale), ref, bnd, "f32 model of the split cross attention")
    assert _rejects(_cross_attn_model(q, kv, nk, D, scale, empty_weight_one=True), ref, bnd)


def _aa_model(x, oh, ow, short=False):
    """aa_resize_nhwc_kernel in f32: ATen's window and triangle weights, renormalised; short: the window one tap short at
    the right edge"""
    def axis(in_size, out_size):
        scale = torch.tensor(in_size / out_size, dtype=torch.float32).item()
        Wm = torch.zeros(out_size, in_size)
        for i in range(out_size):
            c = torch.tensor(scale, dtype=torch.float32) * (i + 0.5)
            support = max(scale, 1.0)
            lo = max(int((c - support + 0.5).item()), 0)
            hi = min(int((c + support + 0.5).item()), in_size)
            if short and hi == in_size:
                hi -= 1
            inv = torch.tensor(1.0 / scale if scale >= 1.0 else 1.0, dtype=torch.float32)
            j = torch.arange(lo, hi, dtype=torch.float32)
            raw = (1 - ((j - c + 0.5) * inv).abs()).clamp(min=0)
            Wm[i, lo:hi] = raw * (1 / raw.sum())
        return Wm
    return torch.einsum("oh,bhwc,pw->bopc", axis(x.shape[1], oh), x.float(), axis(x.shape[2], ow))


def test_aa_resize_bound_rejects_window_one_tap_short_at_the_right_edge():
    g = _gen(15)
    x = (torch.randn(1, 23, 37, 8, generator=g) + 0.5).half()
    for oh, ow in ((9, 14), (40, 50)):                     # non-integer downscale and upscale
        ref, bnd = R.aa_resize_ref(x, oh, ow)
        R.within(_aa_model(x, oh, ow), ref, bnd, f"f32 model of aa_resize -> {oh}x{ow}")
        R.within(_aa_model(x, oh, ow).half(), ref, R.f16_out(ref, bnd), f"f32 model of aa_resize -> {oh}x{ow} f16")
        assert _rejects(_aa_model(x, oh, ow, short=True), ref, bnd)


def test_conv3x3_c1_bound_rejects_tap_shifted_at_the_border():
    g = _gen(16)
    B, H, W, C = 1, 5, 7, 64
    x = torch.randn(B, H, W, C, generator=g).half()
    w = torch.randn(9, C, generator=g) / 24
    ref, bnd = R.conv3x3_c1_ref(x, w, 0.1)
    xt, wt = x.float().permute(0, 3, 1, 2), w.t().reshape(1, C, 3, 3)
    good = torch.exp((F.conv2d(xt, wt, padding=1)[:, 0] + 0.1).clamp(-10, 10))
    R.within(good, ref, bnd, "f32 model of conv3x3_c1_exp")
    # reflect instead of zero padding at the border: only the edge pixels change
    refl = torch.exp((F.conv2d(F.pad(xt, (1, 1, 1, 1), mode="reflect"), wt)[:, 0] + 0.1).clamp(-10, 10))
    assert _rejects(refl, ref, bnd)


def test_small_linear_bound_rejects_dropped_k_tail():
    """K = 200 (one float per lane): a loop that stops at the last multiple of 32 drops 8 terms"""
    g = _gen(17)
    M, N, K = 5, 7, 200
    x, w = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / K ** 0.5
    bias, gamma, resid = torch.randn(N, generator=g), torch.rand(N, generator=g) + 0.5, torch.randn(M, N, generator=g)
    ref, bnd = R.small_linear_ref(x, w, bias=bias, act=R.ACT_GELU, gamma=gamma, resid=resid)
    model = lambda k: resid + gamma * F.gelu(x[:, :k] @ w[:, :k].T + bias)
    R.within(model(K), ref, bnd, "f32 model of small_linear")
    assert _rejects(model(192), ref, bnd)


def test_spatial_mean_bound_rejects_dropped_tail_pixels():
    """HW = 13: a loop over whole groups of 8 pixels drops the last 5"""
    g = _gen(18)
    x = torch.randn(2, 13, 40, generator=g) + 0.3
    ref, bnd = R.spatial_mean_ref(x)
    R.within(x.sum(1) / 13, ref, bnd, "f32 model of spatial_mean")
    assert _rejects(x[:, :8].sum(1) / 13, ref, bnd)


def test_upsample2x_bound_rejects_align_corners_source_index():
    g = _gen(19)
    x = torch.randn(1, 3, 6, 8, generator=g).half()
    ref, bnd = R.upsample2x_ref(x)
    bnd = R.f16_out(ref, bnd)
    up = lambda ac: F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=ac)
    R.within(up(False).permute(0, 2, 3, 1).half(), ref, bnd, "f32 model of upsample2x")
    assert _rejects(up(True).permute(0, 2, 3, 1).half(), ref, bnd)


def test_resize_ac_pad_bound_rejects_reflect_index_off_by_one():
    """reflect_idx(-1) = 1; an index one off repeats the edge pixel (replicate padding) instead"""
    g = _gen(20)
    x = torch.randn(2, 5, 7, 8, generator=g).half()
    ref, bnd = R.resize_ac_pad_ref(x, 2, 9, 1)
    bnd = R.f16_out(ref, bnd)
    rs = F.interpolate(x.float().permute(0, 3, 1, 2), size=(2, 9), mode="bilinear", align_corners=True)
    R.within(F.pad(rs, (1,) * 4, mode="reflect").permute(0, 2, 3, 1).half(), ref, bnd, "f32 model of resize_ac_pad")
    assert _rejects(F.pad(rs, (1,) * 4, mode="replicate").permute(0, 2, 3, 1).half(), ref, bnd)


def test_camera_attn4_bound_rejects_scale_of_the_full_width():
    """8 heads of 48 channels: scaling the logits by 1/sqrt(C) instead of 1/sqrt(C / heads)"""
    g = _gen(21)
    B, heads, Cc = 2, 8, 384
    q, pos, kv = torch.randn(B, 4, Cc, generator=g), torch.randn(4, Cc, generator=g), torch.randn(B, 4, 2 * Cc, generator=g)
    ref, bnd = R.camera_attn4_ref(q, pos, kv, heads)
    split = lambda t: t.reshape(B, 4, heads, Cc // heads).transpose(1, 2)
    Q, K, V = split(q + pos), split(kv[..., :Cc]), split(kv[..., Cc:])
    model = lambda sc: torch.softmax(Q @ K.transpose(-1, -2) * sc, -1) @ V
    R.within(model((Cc // heads) ** -0.5), ref, bnd, "f32 model of camera_attn4")
    assert _rejects(model(Cc ** -0.5), ref, bnd)


def test_landmark_mean_bound_rejects_equal_segments():
    """n = 300: 84 segments of 2 rows and 44 of 3; equal segments of n // 128 rows drop the remainder and shift the starts"""
    g = _gen(22)
    n = 300
    x = torch.randn(1, n, 64, generator=g).half()
    lens = R.nystrom_segments(n)
    ref, bnd = R.segment_mean_ref(x, lens)

    def model(ls):
        st = [sum(ls[:i]) for i in range(128)]
        return torch.stack([x[:, s0:s0 + ln].float().sum(1) / ln for s0, ln in zip(st, ls)], 1).half()

    R.within(model(lens), ref, bnd, "f32 model of nystrom_landmarks")
    assert _rejects(model([n // 128] * 128), ref, bnd)


def test_part_statistics_bound_rejects_whole_row_mean():
    """set_cls_rows_ln: {mean, M2} per part of 40 columns; centring each part on the mean of the whole row"""
    g = _gen(23)
    parts, pc = 11, 40
    v = (torch.randn(parts, pc, generator=g) * 2 + torch.arange(parts).view(-1, 1)).float()
    m, d, Q, dm, e, dQ = R.two_pass_stats(v.double(), pc)
    mean = v.sum(-1, keepdim=True) / pc
    R.within(mean, m, dm, "f32 model of the part means")
    R.within(((v - mean) ** 2).sum(-1, keepdim=True), Q, dQ, "f32 model of the part M2")
    assert _rejects(((v - v.mean()) ** 2).sum(-1, keepdim=True), Q, dQ)


def test_mean_maps_bound_rejects_one_level_one_tap_short():
    g = _gen(24)
    outs = [torch.rand(1, 4 << s, 6 << s, generator=g) + 0.5 for s in (1, 2, 3)]
    ref, bnd = R.mean_maps_ref(outs, 37, 53)
    lv = lambda o, short=False: _aa_model(o[..., None], 37, 53, short)[..., 0]
    R.within((lv(outs[0]) + lv(outs[1]) + lv(outs[2])) / 3, ref, bnd, "f32 model of v1_mean_maps")
    assert _rejects((lv(outs[0]) + lv(outs[1], True) + lv(outs[2])) / 3, ref, bnd)


def test_v1_points_bound_rejects_ray_through_the_pixel_corner():
    """back-projection through (X, Y) instead of the pixel centre (X + 0.5, Y + 0.5)"""
    g = _gen(25)
    H, W = 30, 40
    z = torch.rand(2, H, W, generator=g) + 1
    k4 = torch.tensor([[60.0, 58.0, 21.0, 13.0], [45.0, 47.0, 17.0, 16.0]])
    (xr, yr), (bx, by) = R.v1_points_ref(z, k4, H, W)

    def model(off):
        X = torch.arange(W, dtype=torch.float32).view(1, 1, W) + off
        Y = torch.arange(H, dtype=torch.float32).view(1, H, 1) + off
        dx, dy = (X - k4[:, 2].view(-1, 1, 1)) / k4[:, 0].view(-1, 1, 1), (Y - k4[:, 3].view(-1, 1, 1)) / k4[:, 1].view(-1, 1, 1)
        inv = 1 / torch.sqrt(dx * dx + dy * dy + 1)
        th, ph = torch.atan2(dx * inv, inv), torch.acos(dy * inv)
        return z * torch.tan(th), z / torch.tan(ph) / torch.cos(th)

    gx, gy = model(0.5)
    R.within(gx, xr, bx, "f32 model of the back-projection x")
    R.within(gy, yr, by, "f32 model of the back-projection y")
    bx_, by_ = model(0.0)
    assert _rejects(bx_, xr, bx) and _rejects(by_, yr, by)


def test_newton_schulz_bound_rejects_one_iteration_fewer():
    """kernel_2 of random landmarks; each of the six f32 iterations stays inside the bound of one float64 step from its
    predecessor, while a run with one iteration fewer (the fifth iterate reported as the sixth) falls outside"""
    g = _gen(26)
    ql, kl = (torch.randn(2, 128, 64, generator=g).half().double() for _ in range(2))
    k2 = torch.softmax(ql @ kl.transpose(-1, -2) * 0.125, -1).float()
    eye = torch.eye(128)
    Z = k2.transpose(-1, -2) * (1 / k2.sum(-2).amax(-1)[..., None, None])
    ref, bnd = R.pinv_init_ref(k2)
    R.within(Z, ref, bnd, "f32 model of the pseudo-inverse init")
    iterates = [Z]
    for t in range(6):
        KV = k2 @ Z
        Z = 0.25 * (Z @ (13 * eye - KV @ (15 * eye - KV @ (7 * eye - KV))))
        ref, bnd = R.newton_schulz_step_ref(k2, iterates[-1])
        R.within(Z, ref, bnd, f"f32 model of Newton-Schulz step {t + 1}")
        iterates.append(Z)
    ref, bnd = R.newton_schulz_step_ref(k2, iterates[5])
    assert _rejects(iterates[5], ref, bnd)
