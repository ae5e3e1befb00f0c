"""The per-element bounds of tests/kernel_ref.py, which tests/test_kernel_conformance_gpu.py holds the kernels to, on the
CPU: a float32 model of each kernel's arithmetic (f16 operands, f32 accumulation, f16 rounding where the kernel rounds)
stays inside them, and each of these plausible kernel bugs falls outside them:

  a dropped K-tail block, two adjacent output columns swapped, an off-by-one row map, an unmasked zero-filled key in the
  last tile, a key leaked from the next image, a padded head scaled by 1/sqrt(64) instead of 1/sqrt(true dim), and a
  halo tap read one pixel off."""
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
