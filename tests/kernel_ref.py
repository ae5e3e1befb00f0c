"""Float64 references and per-element error bounds for the wgmma GEMM, the attention kernel and the halo 3x3 convolution.

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
