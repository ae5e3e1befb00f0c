"""Float64 references and per-element error bounds for the wgmma GEMM, the attention kernel, the halo 3x3 convolution and
the CUDA-core kernels (LayerNorm, softmax-weighted sums, antialiased resampling, the single-output conv, the f32 dense layer).

One module, used by tests/test_kernel_conformance_gpu.py (kernel against reference) and tests/test_kernel_bounds_cpu.py
(the same bounds reject plausible kernel bugs).  Plain torch, any device.  Every reference takes the operands already
rounded to f16 exactly as the kernel reads them and computes in float64; the bound is per element.

Notation: u32 = 2^-24 and u16 = 2^-11 are the unit roundoffs of f32 and f16.

GEMM (and the convolutions, which are GEMMs with K = 9 C):  |got - ref| <= alpha * (|A| |W|^T)_ij + beta * mag_ij
  * A product of two f16 values has at most 22 significant bits, so it is exact in f32.  The tensor cores add the K
    products into an f32 accumulator.  Each addition loses at most one f32 ulp of the partial sum when the adder
    truncates instead of rounding (2^-23 relative), and every partial sum is bounded by S = sum_k |a_k| |w_k|.  Over K
    additions that is K 2^-23 S; alpha = K 2^-22 keeps a factor 2 for the block-wise alignment of the products inside
    one MMA step.
  * The f32 epilogue rounds at most four times (bias add, activation, gamma, residual add).  Each rounding costs
    u32 of its own result, so beta = 4 u32 with mag = |v| + |act(v)| |gamma| + |ref| (v = acc + bias).
  * The activation propagates the accumulator error with its Lipschitz constant: 1 for LeakyReLU, 1.13 for GELU; gamma
    scales it by |gamma|.  The epilogue's GELU is the Abramowitz-Stegun erf approximation; tests/test_numerics_claims_cpu.py
    bounds its absolute error by 2e-6 and its f32 evaluation adds at most 32 u32 |v|.
  * An f16 output adds its own rounding: u16 |ref| + 2^-25 (half the smallest f16 subnormal).

Attention, per query row:  |got - ref| <= gamma_row * sum_j P_j |v_j| + u16 |ref| + 2^-25
  (P = softmax(scale q k^T) in float64; the sum is taken per output column.)
  * Logits: q.k over 64 dims in the tensor cores, |ds_j| <= 64 2^-22 sum_d |q_d| |k_jd|.  The kernel works in base 2:
    scale log2(e) is rounded to f32, s sc - m is one rounded fma and ex2.approx is good to 2^-22.  So each exponent is
    off by at most  eps_j = scale |ds_j| + ln2 (2 u32 (|s_j sc| + |m|) + 2^-22)  (natural log units, m the row max).
    With D = max_j eps_j every weight carries a factor in [e^-D, e^D]; numerator and normaliser together move the
    output by at most (e^2D - 1) sum_j P_j |v_j|.
  * The kernel rounds P to f16 for the PV product but sums the row normaliser l from the f32 values: u16 sum_j P_j |v_j|.
    That is the cost of the f16 P, and it dominates gamma in every case here.  A weight below the f16 normal range
    (p < 2^-14, with p <= 1 and l = 1 / max_j P_j) is off by at most 2^-25 absolutely: + 2^-25 max_j P_j sum_j |v_j|.
  * PV accumulation over seq_k keys and the sum of l: (seq_k 2^-22 + seq_k u32) relative, plus a few u32 for the
    per-tile rescale and the final 1/l.
  gamma_row = u16 + (e^2D - 1) + seq_k (2^-22 + 2^-24) + 2^-20.
  The split (fp32) kernel keeps P in f32 and uses expf: the u16 term drops and its logits are f32 CUDA-core dots.

Fused 1x1 heads (GEMM HEAD store and the halo kernel's head):  head = exp(clamp(z, -8, 8) + add),
  z = sum_n hw_n leaky(v_n) + b.  |dz| <= sum_n |hw_n| bound(v_n) + 34 u32 sum_n |hw_n v_n| (the 32-term f32 dot), and
  |d head| <= |head| ((e^|dz| - 1) + 2 u32 |z + add| + 4 u32) (expf within 2 ulp).

CUDA-core kernels (elementwise.cu, v1_kernels.cu).  gamma_n = n u32 bounds n successive f32 roundings of a sum; a warp
reduction over 32 lanes adds 5 levels to the chain each lane runs; expf and rsqrtf are within 2 ulp (2^-22 relative).

LayerNorm (udb_layernorm, udb_layernorm_any; and the per-part {mean, M2} of udb_set_cls_rows_ln), n statistics columns:
  * mean: an f32 sum of n terms and one division, |dm| <= u32 (sum |x| + |m|) (gamma_(n-1) sum |x| / n <= u32 sum |x|).
  * deviations d_i = x_i - m~ are rounded once: e_i = dm + u32 (|d_i| + dm).
  * Q = sum d~^2: |dQ| <= sum e_i (2 |d_i| + e_i) + (n + 2) u32 sum (|d_i| + e_i)^2 (product and sum roundings).
  * var + eps after the division and the add: |dv| <= dQ / n + 3 u32 (v + eps); rsqrtf adds 2^-22, so rstd is off by the
    relative rho = x / (2 (1 - x)^1.5) + 2^-22 with x = dv / (v + eps).
  * y = (d~ rstd) w + b, three roundings: |dy| <= |w| rstd (|d| rho + e (1 + rho)) + 3 u32 (|d rstd w| + |y|).
  An f16 output adds f16_out; the split output stores hi = f16(y~) and lo = f16(y~ - hi) (the difference is exact in
  f32), so hi + lo is within the f32 bound plus lo's own rounding u16 |lo| + 2^-25.

Softmax-weighted sums (udb_softmax_rows, udb_camera_attn4_f32, udb_cross_attn_small, the Nystrom kernel_2):
  p = softmax(s) with s the exact scaled logits and ds_j a bound on the kernel's logit error.  Each exponent is off by
  eps_j = ds_j + 2 u32 (|s_j| + max |s|) (the rounded s - m and its scaling) and expf by 2^-22; with E = max eps_j + 2^-22
  every weight carries a factor in [e^-E, e^E], so numerator and normaliser together move p_j by at most
  (e^2E - 1) p_j.  The f32 sums of the n_acc weights and weighted values add 2 gamma_n_acc, the final division u32.
  Output bound: (e^2E - 1 + 2 (n_acc + 1) u32) sum_j p_j |v_j| + u32 |ref| (+ f16_out where the kernel stores f16).

Antialiased bilinear resampling (udb_aa_resize_nhwc_*, udb_v1_mean_maps, udb_v1_postprocess): the kernel evaluates
ATen's triangle weights in f32.  scale = in / out and center = scale (i + 0.5) carry 3 u32 |center|, the tap argument
((j - center + 0.5) / scale) another 2 u32 (|j| + center + 1) / scale + 3 u32 |arg|; the raw weight 1 - |arg| has slope 1,
so |draw_j| <= |darg_j| over the window widened by one tap each side (a tap that the f32 window adds or drops has a raw
weight below |darg|).  Renormalising by the f32 sum T of the raw weights: sum_j |dw_j| <= 2 sum_j |draw_j| / (T - dT)
+ (taps + 3) u32 per axis (E_y, E_x).  Out: (E_y + E_x) max |x| + (taps_y + taps_x + 2) u32 sum w_y w_x |x|.

Bilinear resamplers without antialias (udb_upsample2x_nhwc_f16, udb_resize_ac_pad_nhwc_f16): each output is
ly0 (lx0 a + lx1 b) + ly1 (lx0 c + lx1 d), three f32 roundings: 3 u32 sum w |x|.  For the 2x upsample the source index
0.5 (i + 0.5) - 0.5 is dyadic, so the weights (0, 1/4, 3/4, 1) are exact.  With align_corners the scale (H-1)/(oh-1) and
fy = sh Y carry 2 u32 fy <= 2 u32 H; ly1 = fy - y0 is exact, so each axis' two weights move by at most 2 u32 H each:
4 u32 (H + W) max |x| for both axes (the reflect pad only copies).

Single-output 3x3 conv (udb_conv3x3_c1_exp): each lane chains 9 taps x 8 channels = 72 fmaf, then log2(C/8) <= 5
shuffle adds and the bias: |dz| <= 78 u32 sum |x w| + u32 |z|.  clamp is 1-Lipschitz and expf adds 2^-22:
|d out| <= out (e^|dz| - 1 + 2^-22).

Small f32 dense layer (udb_small_linear_f32): every lane chains ceil(K/32) fmaf, then 5 shuffle levels; the GEMM epilogue
bound applies with K replaced by ceil(K/32) + 5 (its 2^-22 per term covers the u32 of an f32 rounding twice).

Spatial mean: 8 interleaved f32 partial sums of HW/8 terms, an 8-term sum and the division:
(ceil(HW/8) + 8) u32 sum |x| / HW + u32 |mean|.  The Nystrom landmark means: one f32 sum of len values and a division,
u32 sum |x| + u32 |mean| (gamma_(len-1) sum |x| / len <= u32 sum |x|), then the f16 store.

Logit error bounds ds for the softmax-weighted sums:
  * camera self-attention (udb_camera_attn4_f32): q + pos rounds once (u32), each lane chains ceil(d/32) fmaf and 5
    shuffle levels, then the product with rsqrtf(d) (2^-22) rounds: ds <= (d + 6) u32 sum |q'| |k| / sqrt(d)
    + (2^-22 + u32) |s|; n_acc = 4.
  * split cross attention (udb_cross_attn_small): q' = (q + pos) scale rounds twice, each lane chains D/32 fmaf and 5
    shuffle levels: ds <= (D + 4) u32 sum |q'| |k|; the merge rescales 16 partials, n_acc = nk + 16.
  * Nystrom kernel_2: 64 fmaf and the exact 1/8: ds <= 64 u32 sum |q| |k| / 8; the output is p itself.

V1 mean maps: three resizes, two f32 adds and the division by 3: the three bounds / 3 + 3 u32 sum |r| / 3 + u32 |ref|.
V1 back-projection (udb_v1_postprocess points, given the kernel's own z): x = z tan(theta), y = z / tan(phi) / cos(theta)
with theta = atan2(rx, rz), phi = acos(ry) of the unit ray (dx, dy, 1) / n.  dx, dy (a subtraction and an IEEE division)
and n (sqrtf of a 3-term sum, one division) leave rx, ry, rz within 7 u32 relative.  atan2f, acosf, tanf and cosf are
within 4 ulp (eps = 2^-21 relative): dtheta <= 7 u32 + eps |theta| (atan2 moves by |sin cos| <= 1/2 times the two
relative errors), dphi <= 7 u32 |ry| / sin(phi) + eps |phi|, d tan = (1 + tan^2) dtheta + eps |tan|,
d cot(phi) = dphi / sin^2(phi) + 2 eps |cot| (tanf and the division), d cos = |sin| dtheta + eps |cos|; then one (x) or
two (y) roundings.

Nystrom pseudo-inverse (udb_nystrom_k2_pinv).  Z0 = K^T / max_j sum_i K_ij: a 128-term f32 column sum, a reciprocal and
a product, (m + 3) u32 |Z0|.  A forward bound through all iterations grows like the product of the |T| matrices (about
1e14 after six steps) and says nothing, so every iteration is held to its own arithmetic: the launcher is deterministic,
so iters = t yields the t-th iterate of the same run, and step t is compared with one float64 step from the kernel's
Z_(t-1).  In that step each f32 matmul C = alpha A B + diag I over m = 128 terms adds
|alpha| (|A| E_B + E_A |B| + E_A E_B + m u32 (|A| + E_A)(|B| + E_B)) + 2 u32 (|alpha A B| + |C|) to the operand errors
E_A, E_B it inherits, and 7I - KV adds u32 |T1|.

Bit-exact kernels (asserted equal, not bounded; the GPU comparison itself is the guard): max_accum, add_f32 and its f16
copy, copy_rows, set_cls_rows, the reflect pads, and the K matrices of the camera-intrinsics kernels wherever their arithmetic is restated operation by
operation in f32 (IEEE division, one rounding per operation).
"""
import math

import torch
import torch.nn.functional as F

U32 = 2.0 ** -24
U16 = 2.0 ** -11
F16_FLOOR = 2.0 ** -25
ACT_NONE, ACT_GELU, ACT_LEAKY = 0, 1, 2
LIP = {ACT_NONE: 1.0, ACT_GELU: 1.13, ACT_LEAKY: 1.0}


def f64(t):
    return None if t is None else t.double()


def _act(v, act):
    if act == ACT_GELU:
        return 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))
    if act == ACT_LEAKY:
        return F.leaky_relu(v, 0.01)
    return v


def epilogue(acc, S, K, *, bias=None, act=ACT_NONE, gamma=None, resid=None):
    """ref and f32-output bound of  resid + gamma * act(acc + bias)  given the exact accumulator acc and S = |A||W|^T."""
    v = acc if bias is None else acc + f64(bias)
    av = _act(v, act)
    g = 1.0 if gamma is None else f64(gamma).abs()
    y = av if gamma is None else av * f64(gamma)
    ref = y if resid is None else y + f64(resid)
    bound = LIP[act] * g * (K * 2.0 ** -22) * S
    bound = bound + 4 * U32 * (v.abs() + av.abs() * g + ref.abs())
    if act == ACT_GELU:
        bound = bound + g * (2e-6 + 32 * U32 * v.abs())
    return ref, bound


def gemm_ref(a, w, **epi):
    """a [M, K] f16, w [N, K] f16 -> (ref, f32-output bound) of the matrix-mode GEMM."""
    a, w = f64(a), f64(w)
    return epilogue(a @ w.T, a.abs() @ w.abs().T, a.shape[1], **epi)


def f16_out(ref, bound):
    """bound for the same value stored as f16"""
    return bound * (1 + U16) + U16 * ref.abs() + F16_FLOOR


def conv3x3_ref(x, w, **epi):
    """x [B, H+2, W+2, C] f16 NHWC, already padded (zeros or reflection); w [N, 9C] ordered (dy, dx, c).
    Returns NHWC (ref, f32 bound)."""
    N, C = w.shape[0], x.shape[-1]
    xt = f64(x).permute(0, 3, 1, 2)
    wt = f64(w).view(N, 3, 3, C).permute(0, 3, 1, 2)
    acc = F.conv2d(xt, wt).permute(0, 2, 3, 1)
    S = F.conv2d(xt.abs(), wt.abs()).permute(0, 2, 3, 1)
    return epilogue(acc, S, 9 * C, **epi)


def convt_index(B, h, w, k, cout, pad, device="cpu"):
    """flat index into the [B, h k + 2 pad, w k + 2 pad, cout] map of GEMM element (m, n), n = (dy k + dx) cout + co
    (the CONVT store of udb_gemm_t)"""
    H2, W2 = h * k + 2 * pad, w * k + 2 * pad
    m = torch.arange(B * h * w, device=device)
    b, y, x = m // (h * w), (m % (h * w)) // w, m % w
    n = torch.arange(k * k * cout, device=device)
    dy, dx, co = n // (k * cout), (n // cout) % k, n % cout
    row = (b[:, None] * H2 + y[:, None] * k + dy[None] + pad) * W2 + x[:, None] * k + dx[None] + pad
    return row * cout + co[None]


def head_ref(v, vb, hw, hb, hadd):
    """fused head exp(clamp(sum_n hw_n leaky(v_n) + hb, -8, 8) + hadd) over the last dim of v (bound vb)"""
    hw = f64(hw)
    lv = F.leaky_relu(v, 0.01)
    z = (lv * hw).sum(-1) + hb
    zc = z.clamp(-8, 8) + hadd
    ref = torch.exp(zc)
    dz = (vb * hw.abs()).sum(-1) + 34 * U32 * (lv * hw).abs().sum(-1)
    return ref, ref * (torch.expm1(dz) + 2 * U32 * zc.abs() + 4 * U32)


def attention_ref(q, k, v, scale, *, f16_p=True):
    """q [B, H, Sq, 64], k / v [B, H, Sk, 64] (f16 values, or hi + lo sums for the split kernel) -> (ref, bound) of the
    f16 output [B, H, Sq, 64]."""
    q, k, v = f64(q), f64(k), f64(v)
    s = q @ k.transpose(-1, -2)
    P = torch.softmax(s * scale, -1)
    ref = P @ v
    Sk = k.shape[-2]
    if f16_p:   # wgmma logits, base-2 exponent arithmetic
        ds = 64 * 2.0 ** -22 * (q.abs() @ k.abs().transpose(-1, -2))
        sc = scale * math.log2(math.e)
        m = (s * sc).amax(-1, keepdim=True).abs()
        eps = scale * ds + math.log(2) * (2 * U32 * ((s * sc).abs() + m) + 2.0 ** -22)
        gamma = U16 + torch.expm1(2 * eps.amax(-1, keepdim=True)) + Sk * (2.0 ** -22 + U32) + 2.0 ** -20
    else:       # split kernel: f32 dots on the CUDA cores, exact expf, f32 P
        ds = 2 * 64 * U32 * (q.abs() @ k.abs().transpose(-1, -2))
        eps = scale * ds + 4 * U32 * (s * scale).abs()
        gamma = torch.expm1(2 * eps.amax(-1, keepdim=True)) + Sk * 2 * U32 + 2.0 ** -20
    bound = gamma * (P @ v.abs()) + U16 * ref.abs() + F16_FLOOR
    if f16_p:
        bound = bound + 2.0 ** -25 * P.amax(-1, keepdim=True) * v.abs().sum(-2, keepdim=True)
    return ref, bound


def attn_inputs(B, H, Sq, Sk, gen, q_gain=1.0, k_gain=1.0):
    """f16 q [B, H, Sq, 64], k, v [B, H, Sk, 64].  v has mean 0.5, so a key that wrongly enters the softmax (an unmasked
    zero-filled key, a key of the next image) moves the output by its weight times ~0.5 instead of averaging out."""
    q = (torch.randn(B, H, Sq, 64, generator=gen) * q_gain).half()
    k = (torch.randn(B, H, Sk, 64, generator=gen) * k_gain).half()
    v = (torch.randn(B, H, Sk, 64, generator=gen) + 0.5).half()
    return q, k, v


def isolation_inputs(B, Sq, Sk, gen, step=30.0, scale=0.125):
    """One head; every query of image b sees logits step*b + N(0, 1/4) against the keys of image b (q = 4 e_0), so the
    keys of image b+1 sit `step` above those of image b: any of them leaking into image b's last tile dominates."""
    q = torch.zeros(B, 1, Sq, 64)
    q[..., 0] = 4.0
    k = torch.randn(B, 1, Sk, 64, generator=gen) * 0.3
    k[..., 0] = (step * torch.arange(B).view(B, 1, 1) + 0.5 * torch.randn(B, 1, Sk, generator=gen)) / (4.0 * scale)
    v = torch.randn(B, 1, Sk, 64, generator=gen) + 0.5
    return q.half(), k.half(), v.half()


def ratio(got, ref, bound):
    """largest err / bound (inf when got has a NaN or Inf where ref is finite)"""
    err = (got.double() - ref).abs()
    r = err / bound
    r = torch.where(torch.isfinite(got.double()), r, torch.full_like(r, math.inf))
    return r.max().item()


def within(got, ref, bound, name):
    r = ratio(got, ref, bound)
    print(f"{name}: max err/bound {r:.3g}")
    assert r <= 1.0, (name, r)
    return r


# ------------------------------------------------------------------------------------------------ CUDA-core kernels
def _gamma(n):
    return n * U32


def two_pass_stats(x, n):
    """mean, centred sum of squares Q and their f32 two-pass error bounds over the first n columns of float64 rows x.
    Returns (m, d, Q, dm, e, dQ) with d = x - m over every column and e the bound on each rounded deviation."""
    xs = x[..., :n]
    m = xs.mean(-1, keepdim=True)
    dm = U32 * (xs.abs().sum(-1, keepdim=True) + m.abs())
    d = x - m
    e = dm + U32 * (d.abs() + dm)
    ds, es = d[..., :n], e[..., :n]
    Q = (ds * ds).sum(-1, keepdim=True)
    dQ = (es * (2 * ds.abs() + es)).sum(-1, keepdim=True) + (n + 2) * U32 * ((ds.abs() + es) ** 2).sum(-1, keepdim=True)
    return m, d, Q, dm, e, dQ


def layernorm_ref(x, w, b, eps, n=None):
    """x [rows, dim] as the kernel reads it (f16 / f32 values, plus the f32-rounded add table), statistics over the first
    n columns (dim_valid) -> (ref, f32-output bound) of (x - mean) rstd w + b over all dim columns"""
    x, w, b = f64(x), f64(w), f64(b)
    n = x.shape[-1] if n is None else n
    m, d, Q, dm, e, dQ = two_pass_stats(x, n)
    v = Q / n
    rstd = 1.0 / torch.sqrt(v + eps)
    xr = (dQ / n + 3 * U32 * (v + eps)) / (v + eps)
    rho = xr / (2 * (1 - xr) ** 1.5) + 2.0 ** -22
    y = d * rstd * w + b
    bound = w.abs() * rstd * (d.abs() * rho + e * (1 + rho)) + 3 * U32 * ((d * rstd * w).abs() + y.abs())
    return y, bound


def split_out(ref, bound, hi, lo):
    """checks for a split-f16 output: (hi bound, hi + lo bound)"""
    return f16_out(ref, bound), bound + U16 * lo.double().abs() + F16_FLOOR


def softmax_av_ref(s, ds, v, n_acc):
    """s [..., nq, nk] exact scaled logits, ds a bound on the kernel's logit error (same shape or broadcastable),
    v [..., nk, D] -> (ref, bound) of softmax(s) @ v accumulated in f32 over n_acc terms"""
    s, v = f64(s), f64(v)
    P = torch.softmax(s, -1)
    ref = P @ v
    E = (ds + 2 * U32 * (s.abs() + s.abs().amax(-1, keepdim=True))).amax(-1, keepdim=True) + 2.0 ** -22
    gamma = torch.expm1(2 * E) + 2 * (n_acc + 1) * U32
    return ref, gamma * (P @ v.abs()) + U32 * ref.abs()


def softmax_rows_ref(s, n_valid, scale):
    """udb_softmax_rows: f32 rows s (exact), softmax over the first n_valid columns of scale * s -> (P, f16 bound)"""
    s = f64(s)[..., :n_valid] * scale
    P = torch.softmax(s, -1)
    E = (2 * U32 * (s.abs() + s.abs().amax(-1, keepdim=True))).amax(-1, keepdim=True) + 2.0 ** -22
    bound = (torch.expm1(2 * E) + 2 * (n_valid + 1) * U32) * P
    return P, f16_out(P, bound)


def aa_weights(in_size, out_size):
    """ATen's antialiased bilinear weights of one axis in float64: W [out, in] (rows sum to 1), the f32 weight error
    budget E [out] (sum_j |dw_j|) and the tap count per output"""
    scale = in_size / out_size
    support = max(scale, 1.0)
    inv = 1.0 / scale if scale >= 1.0 else 1.0
    W = torch.zeros(out_size, in_size, dtype=torch.float64)
    E = torch.zeros(out_size, dtype=torch.float64)
    taps = torch.zeros(out_size, dtype=torch.float64)
    for i in range(out_size):
        c = scale * (i + 0.5)
        lo, hi = max(int(c - support + 0.5), 0), min(int(c + support + 0.5), in_size)
        j = torch.arange(lo, hi, dtype=torch.float64)
        raw = (1 - ((j - c + 0.5) * inv).abs()).clamp(min=0)
        T = raw.sum().item()
        W[i, lo:hi] = raw / T
        jw = torch.arange(max(lo - 1, 0), min(hi + 1, in_size), dtype=torch.float64)
        arg = ((jw - c + 0.5) * inv).abs()
        darg = inv * (3 * U32 * c + 2 * U32 * (jw.abs() + c + 1)) + 3 * U32 * arg
        draw = darg.sum().item()
        dT = draw + (hi - lo) * U32 * T
        E[i] = 2 * draw / (T - dT) + (hi - lo + 3) * U32
        taps[i] = hi - lo
    return W, E, taps


def aa_resize_ref(x, oh, ow):
    """x [B, H, W, C] NHWC -> (ref, f32 bound) of the antialiased bilinear resize to [B, oh, ow, C]"""
    x = f64(x)
    Wy, Ey, ty = aa_weights(x.shape[1], oh)
    Wx, Ex, tx = aa_weights(x.shape[2], ow)
    Wy, Ey, ty, Wx, Ex, tx = (t.to(x.device) for t in (Wy, Ey, ty, Wx, Ex, tx))
    ref = torch.einsum("oh,bhwc,pw->bopc", Wy, x, Wx)
    mag = torch.einsum("oh,bhwc,pw->bopc", Wy, x.abs(), Wx)
    xmax = x.abs().amax(dim=(1, 2), keepdim=True)
    bound = (Ey[None, :, None, None] + Ex[None, None, :, None]) * xmax
    bound = bound + (ty[None, :, None, None] + tx[None, None, :, None] + 2) * U32 * mag
    return ref, bound


def conv3x3_c1_ref(x, w, bias):
    """x [B, H, W, C] f16 NHWC, w [9, C] f32 ordered (dy, dx) -> (ref, bound) of exp(clamp(conv3x3 + bias, -10, 10))"""
    C = x.shape[-1]
    xt = f64(x).permute(0, 3, 1, 2)
    wt = f64(w).t().reshape(1, C, 3, 3)
    z = F.conv2d(xt, wt, padding=1)[:, 0] + bias
    S = F.conv2d(xt.abs(), wt.abs(), padding=1)[:, 0]
    ref = torch.exp(z.clamp(-10, 10))
    dz = 78 * U32 * S + U32 * z.abs()
    return ref, ref * (torch.expm1(dz) + 2.0 ** -22)


def small_linear_ref(x, w, **epi):
    """udb_small_linear_f32: x [M, K], w [N, K] f32 -> (ref, bound)"""
    x, w = f64(x), f64(w)
    K = x.shape[1]
    return epilogue(x @ w.T, x.abs() @ w.abs().T, -(-K // 32) + 5, **epi)


def upsample2x_ref(x):
    """x [B, H, W, C] NHWC -> (ref, f32 bound) of the 2x bilinear upsample (align_corners=False)"""
    up = lambda t: F.interpolate(t.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    return up(f64(x)), 3 * U32 * up(f64(x).abs())


def resize_ac_pad_ref(x, oh, ow, pad):
    """x [B, H, W, C] NHWC -> (ref, f32 bound) of the align_corners bilinear resize to (oh, ow) plus a reflect pad"""
    H, W = x.shape[1], x.shape[2]
    rs = lambda t: F.interpolate(t.permute(0, 3, 1, 2), size=(oh, ow), mode="bilinear", align_corners=True)
    ref, mag = rs(f64(x)), rs(f64(x).abs())
    if pad:
        ref, mag = F.pad(ref, (pad,) * 4, mode="reflect"), F.pad(mag, (pad,) * 4, mode="reflect")
    xmax = f64(x).abs().amax(dim=(1, 2), keepdim=True)
    return ref.permute(0, 2, 3, 1), 4 * U32 * (H + W) * xmax + 3 * U32 * mag.permute(0, 2, 3, 1)


def spatial_mean_ref(x):
    """x [B, HW, C] f32 -> (ref, bound) of the mean over HW"""
    x = f64(x)
    HW = x.shape[1]
    ref = x.mean(1)
    return ref, (-(-HW // 8) + 8) * U32 * x.abs().sum(1) / HW + U32 * ref.abs()


def segment_mean_ref(x, lens):
    """x [B, n, C] f16 values, consecutive segments of the given lengths -> (ref, f16 bound) of each segment's mean"""
    x = f64(x)
    starts = [sum(lens[:i]) for i in range(len(lens))]
    ref = torch.stack([x[:, s0:s0 + ln].mean(1) for s0, ln in zip(starts, lens)], 1)
    S = torch.stack([x[:, s0:s0 + ln].abs().sum(1) for s0, ln in zip(starts, lens)], 1)
    return ref, f16_out(ref, U32 * S + U32 * ref.abs())


def nystrom_segments(n, m=128):
    """landmark segment lengths: the first m - n % m segments have n // m rows, the rest one more"""
    return [n // m] * (m - n % m) + [n // m + 1] * (n % m)


def camera_attn4_ref(q, pos, kv, heads):
    """q [B, 4, C], pos [4, C], kv [B, 4, 2C] f32 -> (ref, bound) of the 4-token self-attention, as [B, heads, 4, d]"""
    B, _, Cc = q.shape
    d = Cc // heads
    split = lambda t: f64(t).reshape(B, 4, heads, d).transpose(1, 2)
    Q, K, V = split((q + pos).float()), split(kv[..., :Cc]), split(kv[..., Cc:])
    s = Q @ K.transpose(-1, -2) * d ** -0.5
    ds = (d + 6) * U32 * (Q.abs() @ K.abs().transpose(-1, -2)) * d ** -0.5 + (2.0 ** -22 + U32) * s.abs()
    return softmax_av_ref(s, ds, V, 4)


def mean_maps_ref(outs, net_h, net_w):
    """the three exp'ed maps [B, h, w] -> (ref, bound) of the mean of their antialiased resizes to (net_h, net_w)"""
    refs, bnds = zip(*(aa_resize_ref(o[..., None], net_h, net_w) for o in outs))
    ref = sum(refs) / 3
    bnd = sum(bnds) / 3 + 3 * U32 * sum(r.abs() for r in refs) / 3 + U32 * ref.abs()
    return ref[..., 0], bnd[..., 0]


def v1_points_ref(z, k4, H, W):
    """z [B, H, W] (the kernel's depth), k4 [B, 4] = fx, fy, cx, cy -> ((x, y) refs, bounds) of the back-projection"""
    z, k4 = f64(z), f64(k4)
    X = torch.arange(W, dtype=torch.float64, device=z.device).view(1, 1, W) + 0.5
    Y = torch.arange(H, dtype=torch.float64, device=z.device).view(1, H, 1) + 0.5
    fx, fy, cx, cy = (k4[:, i].view(-1, 1, 1) for i in range(4))
    dx, dy = (X - cx) / fx, (Y - cy) / fy
    n = torch.sqrt(dx * dx + dy * dy + 1)
    rx, ry, rz = dx / n, dy / n, 1 / n
    th, ph = torch.atan2(rx, rz), torch.acos(ry)
    eps = 2.0 ** -21
    dth = 7 * U32 + eps * th.abs()
    dph = 7 * U32 * ry.abs() / torch.sin(ph) + eps * ph.abs()
    tan, cot, cos = torch.tan(th), 1 / torch.tan(ph), torch.cos(th)
    dtan = (1 + tan * tan) * dth + eps * tan.abs()
    dcot = dph / torch.sin(ph) ** 2 + 2 * eps * cot.abs()
    dcos = torch.sin(th).abs() * dth + eps * cos.abs()
    x, y = z * tan, z * cot / cos
    bx = z.abs() * dtan + U32 * x.abs()
    by = z.abs() * (dcot / cos.abs() + cot.abs() * dcos / cos ** 2) + 2 * U32 * y.abs()
    return (x, y), (bx, by)


def pinv_init_ref(k2):
    """k2 [..., m, m] (the kernel's f32 kernel_2) -> (Z0, bound) of K^T / max_j sum_i K_ij"""
    K = f64(k2)
    m = K.shape[-1]
    Z = K.transpose(-1, -2) / K.sum(-2).amax(-1)[..., None, None]
    return Z, (m + 3) * U32 * Z.abs()


def newton_schulz_step_ref(k2, z_prev):
    """one Newton-Schulz step Z' = 0.25 Z (13I - KV (15I - KV (7I - KV))), KV = K Z, in float64 from the kernel's f32 K and
    Z_(t-1) -> (Z', bound of the f32 step)"""
    K, Z = f64(k2), f64(z_prev)
    m = K.shape[-1]
    eye = torch.eye(m, dtype=torch.float64, device=K.device)
    zero = torch.zeros_like(K)

    def mm(A, EA, B, EB, alpha, diag):
        P = A @ B
        Cm = alpha * P + diag * eye
        E = abs(alpha) * (A.abs() @ EB + EA @ B.abs() + EA @ EB + m * U32 * ((A.abs() + EA) @ (B.abs() + EB)))
        return Cm, E + 2 * U32 * (abs(alpha) * P.abs() + Cm.abs())

    KV, EKV = mm(K, zero, Z, zero, 1.0, 0.0)
    T1 = 7 * eye - KV
    ET1 = EKV + U32 * T1.abs()
    T2, ET2 = mm(KV, EKV, T1, ET1, -1.0, 15.0)
    T3, ET3 = mm(KV, EKV, T2, ET2, -1.0, 13.0)
    return mm(Z, zero, T3, ET3, 0.25, 0.0)
