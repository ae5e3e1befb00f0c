"""Python-side operator wrappers: torch tensors in, raw device pointers into the C ABI
(include/udb.h), launches on torch's current stream.  PyTorch is only the allocator / stream
provider here; all arithmetic happens in libudb.so.  No fallbacks."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _cabi as cabi
from ._cabi import (A_CONV3X3, A_MATRIX, ACT_GELU, ACT_LEAKY, ACT_NONE, STORE_CONVT, STORE_CONVTILE,
                    STORE_HEAD, STORE_ROWS)

f16, f32 = torch.float16, torch.float32

# When set to a list, the tensor-core ops append (kernel, algorithmic flops, start_event, end_event)
# for every launch (bench.py's per-kernel roofline); None in normal operation.
PROFILE = None


def _launch(kernel: str, flops: float, fn, nbytes: float = 0.0):
    """Run one C-ABI launch; with PROFILE set, bracket it with CUDA events and record the algorithmic flops / bytes."""
    if PROFILE is None:
        return fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    rc = fn()
    e.record()
    PROFILE.append((kernel, flops, s, e, nbytes))
    return rc


def _nb(*tensors):
    return float(sum(t.numel() * t.element_size() for t in tensors if t is not None))


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t: Optional[torch.Tensor]):
    if t is None:
        return None
    assert t.is_cuda, "udb ops need CUDA tensors (no CPU fallback)"
    return C.c_void_p(t.data_ptr())


def _unit_stride(*tensors):
    """The kernels address every operand as rows of contiguous elements (vector loads / stores along the last dim)."""
    for t in tensors:
        assert t is None or t.stride(-1) == 1, f"udb ops need stride(-1) == 1, got strides {tuple(t.stride())}"


def _is32(t):
    if t.dtype == f32:
        return 1
    assert t.dtype == f16, t.dtype
    return 0


def gemm(a: torch.Tensor, w: torch.Tensor, *, bias=None, act=ACT_NONE, gamma=None, resid=None,
         out: Optional[torch.Tensor] = None, out_dtype=f16, out2: Optional[torch.Tensor] = None, out2_leaky=True,
         rows_per_group=0, group_stride=0, row_offset=0, resid_mod=0, resid_row_offset=0,
         out_rows: Optional[int] = None, a_split_k: int = 0, out_split: bool = False,
         ln_stats_out=None, ln_stats_in=None, ln_c1=None, ln_parts: int = 0, ln_part_cols: int = 0, ln_eps: float = 0.0):
    """out[row(m), :] = resid + gamma * act(a @ w.T + bias).  a f16 [M,K], w f16 [N,K].
    Split-f16 mode (udb_gemm_t.a_split_k = K1): a is [M, 2*K1] = [hi | lo], w is [N, 3*K1] = [hi | hi | lo];
    out_split: the f16 output is written as [M, 2N] = [hi | lo]."""
    assert a.dtype == f16 and w.dtype == f16 and a.stride(-1) == 1 and w.stride(-1) == 1
    M, K = a.shape
    N = w.shape[0]
    if a_split_k:
        assert K == 2 * a_split_k and w.shape[1] == 3 * a_split_k
        K = 3 * a_split_k
    else:
        assert w.shape[1] == K
    if out is None:
        out = torch.empty((out_rows if out_rows is not None else M, 2 * N if out_split else N), device=a.device,
                          dtype=f16 if out_split else out_dtype)
    _unit_stride(out, out2, resid)
    g = cabi.Gemm()
    g.a, g.w = _ptr(a), _ptr(w)
    g.M, g.N, g.K = M, N, K
    g.lda, g.ldw = a.stride(0), w.stride(0)
    g.a_mode = A_MATRIX
    g.bias, g.gamma = _ptr(bias), _ptr(gamma)
    if resid is not None:
        g.resid, g.resid_f32, g.ldr = _ptr(resid), _is32(resid), resid.stride(0)
    g.out, g.out_f32, g.ldc = _ptr(out), _is32(out), out.stride(0)
    g.out2, g.out2_leaky = _ptr(out2), int(out2_leaky)
    g.act, g.store_mode = act, STORE_ROWS
    g.rows_per_group, g.group_stride, g.row_offset = rows_per_group, group_stride, row_offset
    g.resid_mod, g.resid_row_offset = resid_mod, resid_row_offset
    g.a_split_k, g.out_split = a_split_k, (N if out_split else 0)
    g.ln_stats_out, g.ln_stats_in, g.ln_c1 = _ptr(ln_stats_out), _ptr(ln_stats_in), _ptr(ln_c1)
    g.ln_parts, g.ln_part_cols, g.ln_eps = ln_parts, ln_part_cols, ln_eps
    cabi.check(_launch("gemm_f16_kernel", 2.0 * M * N * K, lambda: cabi.lib().udb_gemm_f16(C.byref(g), _stream())),
               "udb_gemm_f16")
    return out


def conv3x3(x: torch.Tensor, w: torch.Tensor, *, bias=None, act=ACT_NONE, gamma=None, resid=None,
            out: Optional[torch.Tensor] = None, out_dtype=f16, out2=None, out2_leaky=True, prepadded=False,
            head_w=None, head_b=0.0, head_add=0.0, tile=(8, 16), c_off=0, c_used=None):
    """3x3 convolution over an NHWC f16 image x [B,H,W,C] (or [B,H+2,W+2,C] if prepadded) with
    packed weights w [Cout, 9*C] ordered (dy,dx,c).  Zero padding unless prepadded.
    With head_w: fused LeakyReLU + 1x1 (32->1) + clamp/exp head, returns f32 [B,H,W]."""
    assert x.dtype == f16 and w.dtype == f16 and x.is_contiguous() and w.is_contiguous()
    B, inH, inW, Ctot = x.shape
    Cin = c_used if c_used is not None else Ctot        # channel slice [c_off, c_off + Cin) of the buffer
    H, W = (inH - 2, inW - 2) if prepadded else (inH, inW)
    N = w.shape[0]
    assert w.shape[1] == 9 * Cin and c_off + Cin <= Ctot
    _unit_stride(out, out2, resid)
    g = cabi.Gemm()
    g.a, g.w = _ptr(x), _ptr(w)
    g.M, g.N, g.K = B * H * W, N, 9 * Cin
    g.lda, g.ldw = Cin, 9 * Cin
    g.a_mode = A_CONV3X3
    g.conv_B, g.conv_H, g.conv_W, g.conv_C = B, H, W, Cin
    g.conv_inH, g.conv_inW = inH, inW
    g.conv_off = 0 if prepadded else -1
    g.conv_TH, g.conv_TW = tile
    g.conv_cstride, g.conv_coff = Ctot, c_off
    g.bias, g.gamma = _ptr(bias), _ptr(gamma)
    g.act = act
    if head_w is not None:
        if out is None:
            out = torch.empty((B, H, W), device=x.device, dtype=f32)
        g.store_mode = STORE_HEAD
        g.head_w, g.head_b, g.head_add = _ptr(head_w), float(head_b), float(head_add)
        g.out, g.out_f32, g.ldc = _ptr(out), 1, 1
    else:
        if out is None:
            out = torch.empty((B, H, W, N), device=x.device, dtype=out_dtype)
        g.store_mode = STORE_CONVTILE
        g.out, g.out_f32, g.ldc = _ptr(out), _is32(out), out.stride(2)
        if resid is not None:
            g.resid, g.resid_f32, g.ldr = _ptr(resid), _is32(resid), resid.stride(2)
        g.out2, g.out2_leaky = _ptr(out2), int(out2_leaky)
    cabi.check(_launch("gemm_f16_kernel", 2.0 * B * H * W * N * 9 * Cin,
                       lambda: cabi.lib().udb_gemm_f16(C.byref(g), _stream())), "udb_gemm_f16(conv3x3)")
    return out


def conv3x3_halo(x: torch.Tensor, w: torch.Tensor, *, bias, act=ACT_NONE, c_off=0, c_used=None, out=None,
                 head_w=None, head_b=0.0, head_add=0.0):
    """3x3 conv over a pre-padded NHWC f16 image x [B,H+2,W+2,Ctot] (channel slice), w [Cout, 9*C],
    Cout in {32, 64}, halo-reuse kernel.  Returns f16 [B,H,W,Cout] or (head_w given) f32 [B,H,W]."""
    assert x.dtype == f16 and w.dtype == f16 and x.is_contiguous() and w.is_contiguous()
    B, PH, PW, Ctot = x.shape
    Cin = c_used if c_used is not None else Ctot
    H, W, N = PH - 2, PW - 2, w.shape[0]
    assert w.shape[1] == 9 * Cin
    _unit_stride(out)
    c = cabi.ConvHalo()
    c.x, c.w, c.bias = _ptr(x), _ptr(w), _ptr(bias)
    c.B, c.H, c.W, c.C, c.cstride, c.coff, c.cout, c.act = B, H, W, Cin, Ctot, c_off, N, act
    if head_w is not None:
        if out is None:
            out = torch.empty((B, H, W), device=x.device, dtype=f32)
        c.head_w, c.head_b, c.head_add, c.head_out = _ptr(head_w), float(head_b), float(head_add), _ptr(out)
    else:
        if out is None:
            out = torch.empty((B, H, W, N), device=x.device, dtype=f16)
        c.out, c.ldc = _ptr(out), out.stride(2)
    cabi.check(_launch("conv3x3_halo_kernel", 2.0 * B * H * W * N * 9 * Cin,
                       lambda: cabi.lib().udb_conv3x3_halo_f16(C.byref(c), _stream())), "udb_conv3x3_halo_f16")
    return out


def conv_transpose_ks(x: torch.Tensor, w: torch.Tensor, k: int, cout: int, grid_hw, *, bias=None,
                      resid=None, out: Optional[torch.Tensor] = None, out_dtype=f16, out2=None, out2_leaky=True,
                      pad=0):
    """ConvTranspose2d with kernel == stride == k as a GEMM with a pixel-shuffle store.
    x f16 [B*h*w, Cin]; w f16 [k*k*cout, Cin] ordered (dy,dx,co); bias f32 [k*k*cout].
    out NHWC [B, h*k + 2*pad, w*k + 2*pad, cout] (+ resid of the same shape, may alias out); with
    pad > 0 only the interior is written (k == 1: a per-pixel linear layer into a padded buffer)."""
    h, ww = grid_hw
    M, K = x.shape
    B = M // (h * ww)
    if out is None:
        out = torch.empty((B, h * k + 2 * pad, ww * k + 2 * pad, cout), device=x.device, dtype=out_dtype)
    _unit_stride(x, w, out, out2, resid)
    g = cabi.Gemm()
    g.a, g.w = _ptr(x), _ptr(w)
    g.M, g.N, g.K = M, k * k * cout, K
    g.lda, g.ldw = x.stride(0), w.stride(0)
    g.a_mode = A_MATRIX
    g.bias = _ptr(bias)
    if resid is not None:
        g.resid, g.resid_f32 = _ptr(resid), _is32(resid)
    g.out, g.out_f32, g.ldc = _ptr(out), _is32(out), cout
    g.out2, g.out2_leaky = _ptr(out2), int(out2_leaky)
    g.store_mode = STORE_CONVT
    g.ct_k, g.ct_cout, g.ct_h, g.ct_w, g.ct_pad = k, cout, h, ww, pad
    cabi.check(_launch("gemm_f16_kernel", 2.0 * M * k * k * cout * K,
                       lambda: cabi.lib().udb_gemm_f16(C.byref(g), _stream())), "udb_gemm_f16(convT)")
    return out


def attention(q, k, v, out, *, B, heads, seq_q, seq_k, head_dim, q_col0=0, k_col0=0, v_col0=0, o_col0=0, scale=None,
              lo_off_in=0, lo_off_out=0):
    """lo_off_in > 0: split-f16 operands (lo halves lo_off_in columns to the right), fp32 CUDA-core kernel."""
    _unit_stride(q, k, v, out)
    a = cabi.Attn()
    a.q, a.k, a.v, a.out = _ptr(q), _ptr(k), _ptr(v), _ptr(out)
    a.B, a.heads, a.seq_q, a.seq_k, a.head_dim = B, heads, seq_q, seq_k, head_dim
    a.ldq, a.ldk, a.ldv, a.ldo = q.stride(0), k.stride(0), v.stride(0), out.stride(0)
    a.q_col0, a.k_col0, a.v_col0, a.o_col0 = q_col0, k_col0, v_col0, o_col0
    a.scale = head_dim ** -0.5 if scale is None else scale   # explicit scale: zero-padded narrower heads
    if lo_off_in:
        a.split, a.lo_off_q, a.lo_off_k, a.lo_off_v, a.lo_off_o = 1, lo_off_in, lo_off_in, lo_off_in, lo_off_out
    cabi.check(_launch("attn_fwd_kernel", 4.0 * B * heads * seq_q * seq_k * head_dim,
                       lambda: cabi.lib().udb_attention_f16(C.byref(a), _stream())), "udb_attention_f16")
    return out


def layernorm(x, weight, bias, eps, *, out=None, out_dtype=f16, rows=None, rows_per_group=0,
              group_stride=0, row_offset=0, dim_valid=0, out_split=False):
    dim = x.shape[-1]
    x2 = x.reshape(-1, dim)
    n_rows = rows if rows is not None else x2.shape[0]
    if out is None:
        out = torch.empty((n_rows, 2 * dim if out_split else dim), device=x.device, dtype=f16 if out_split else out_dtype)
    p = cabi.LayerNorm()
    p.inp, p.in_f32 = _ptr(x2), _is32(x2)
    p.out, p.out_f32 = _ptr(out), _is32(out)
    p.weight, p.bias = _ptr(weight), _ptr(bias)
    p.rows, p.dim = n_rows, dim
    p.ld_in, p.ld_out = x2.stride(0), out.stride(0)
    p.rows_per_group, p.group_stride, p.row_offset = rows_per_group, group_stride, row_offset
    p.eps = eps
    p.dim_valid = dim_valid
    p.out_split = dim if out_split else 0
    nbytes = float(n_rows * dim * (x2.element_size() + out.element_size()))
    cabi.check(_launch("layernorm_kernel", 0.0, lambda: cabi.lib().udb_layernorm(C.byref(p), _stream()), nbytes), "udb_layernorm")
    return out


def preprocess_patchify(rgb, paddings, net_hw, patches, normalize=True):
    B, _, H, W = rgb.shape
    assert rgb.is_contiguous() and rgb.dtype in (torch.uint8, f32)
    p = cabi.Preprocess()
    p.rgb, p.rgb_is_u8, p.normalize = _ptr(rgb), int(rgb.dtype == torch.uint8), int(normalize)
    p.B, p.H, p.W = B, H, W
    p.pad_l, p.pad_r, p.pad_t, p.pad_b = paddings
    p.net_h, p.net_w = net_hw
    p.patches, p.ldp = _ptr(patches), patches.stride(0)
    cabi.check(_launch("preprocess_patchify_kernel", 0.0, lambda: cabi.lib().udb_preprocess_patchify(C.byref(p), _stream()),
                       _nb(rgb, patches)), "udb_preprocess_patchify")
    return patches


def posembed_bicubic(grid, m, dim, gh, gw):
    out = torch.empty((gh * gw, dim), device=grid.device, dtype=f32)
    cabi.check(cabi.lib().udb_posembed_bicubic(_ptr(grid), m, dim, _ptr(out), gh, gw, _stream()), "udb_posembed_bicubic")
    return out


def set_cls_rows(x, cls_token, pos0, B, T, D):
    cabi.check(cabi.lib().udb_set_cls_rows(_ptr(x), _ptr(cls_token), _ptr(pos0), B, T, D, _stream()), "udb_set_cls_rows")


def small_linear(x, w, bias=None, act=ACT_NONE, gamma=None, resid=None, out=None):
    """fp32 y = resid + gamma * act(x @ w.T + bias); x / out / resid may be row-strided 2-D views."""
    M, K = x.shape
    N = w.shape[0]
    assert x.dtype == f32 and w.dtype == f32 and x.stride(1) == 1 and w.is_contiguous()
    if out is None:
        out = torch.empty((M, N), device=x.device, dtype=f32)
    assert out.stride(1) == 1 and (resid is None or resid.stride(1) == 1)
    p = cabi.SmallLinear()
    p.x, p.w, p.bias, p.gamma, p.resid, p.y = _ptr(x), _ptr(w), _ptr(bias), _ptr(gamma), _ptr(resid), _ptr(out)
    p.M, p.N, p.K, p.act = M, N, K, act
    p.ldx, p.ldy, p.ldr = x.stride(0), out.stride(0), (resid.stride(0) if resid is not None else 0)
    cabi.check(_launch("small_linear_kernel", 0.0, lambda: cabi.lib().udb_small_linear_f32(C.byref(p), _stream())), "udb_small_linear_f32")
    return out


def camera_attn4(q, kv, pos, B, C_, heads):
    out = torch.empty_like(q)
    cabi.check(cabi.lib().udb_camera_attn4_f32(_ptr(q), _ptr(kv), _ptr(pos), _ptr(out), B, C_, heads, _stream()),
               "udb_camera_attn4_f32")
    return out


def camera_intrinsics(x, B, net_hw, factor, pad_l, pad_t):
    intr4 = torch.empty((B, 4), device=x.device, dtype=f32)
    k_net = torch.empty((B, 3, 3), device=x.device, dtype=f32)
    k_out = torch.empty((B, 3, 3), device=x.device, dtype=f32)
    cabi.check(cabi.lib().udb_camera_intrinsics(_ptr(x), B, net_hw[0], net_hw[1], float(factor), pad_l, pad_t,
                                                _ptr(intr4), _ptr(k_net), _ptr(k_out), _stream()),
               "udb_camera_intrinsics")
    return intr4, k_net, k_out


def camera_rays(model, params, B, net_hw, paddings, factor):
    """GT-camera rays [B, net_h*net_w, 3] of a packed camera (udb_camera_rays; camera.pack_camera): params [B, CAM_STRIDE]
    f32 in input-image pixels, cropped by the paddings (l, r, t, b) and resized by `factor` in the kernel."""
    assert params.dtype == f32 and params.is_contiguous() and tuple(params.shape) == (B, cabi.CAM_STRIDE), params.shape
    nh, nw = net_hw
    out = torch.empty((B, nh * nw, 3), device=params.device, dtype=f32)
    pl, pr, pt, pb = paddings
    cabi.check(_launch("camera_rays_kernel", 0.0,
                       lambda: cabi.lib().udb_camera_rays(int(model), _ptr(params), B, nh, nw, pl, pr, pt, pb, float(factor),
                                                          _ptr(out), _stream()), _nb(out)), "udb_camera_rays")
    return out


def ray_embed(intr4, scales, B, net_hw, grid_hw, out_dtype=f32, rays_in=None):
    bands = scales.numel()
    out = torch.empty((B * grid_hw[0] * grid_hw[1], 2 * bands), device=scales.device, dtype=out_dtype)
    p = cabi.RayEmbed()
    p.intr4, p.rays_in, p.scales = _ptr(intr4), _ptr(rays_in), _ptr(scales)
    p.B, p.net_h, p.net_w, p.gh, p.gw, p.bands = B, net_hw[0], net_hw[1], grid_hw[0], grid_hw[1], bands
    p.out, p.out_f32 = _ptr(out), _is32(out)
    cabi.check(_launch("ray_embed_kernel", 0.0, lambda: cabi.lib().udb_ray_embed(C.byref(p), _stream()), _nb(out, rays_in)), "udb_ray_embed")
    return out


def upsample2x(x):
    B, H, W, Cc = x.shape
    out = torch.empty((B, 2 * H, 2 * W, Cc), device=x.device, dtype=f16)
    cabi.check(_launch("upsample2x_kernel", 0.0, lambda: cabi.lib().udb_upsample2x_nhwc_f16(_ptr(x), _ptr(out), B, H, W, Cc, _stream()),
                       _nb(x, out)),
               "udb_upsample2x_nhwc_f16")
    return out


def resize_ac_pad(x, oh, ow, pad):
    B, H, W, Cc = x.shape
    out = torch.empty((B, oh + 2 * pad, ow + 2 * pad, Cc), device=x.device, dtype=f16)
    cabi.check(_launch("resize_ac_pad_kernel", 0.0,
                       lambda: cabi.lib().udb_resize_ac_pad_nhwc_f16(_ptr(x), _ptr(out), B, H, W, Cc, oh, ow, pad, _stream()),
                       _nb(x, out)),
               "udb_resize_ac_pad_nhwc_f16")
    return out


def reflect_pad1(x):
    B, H, W, Cc = x.shape
    out = torch.empty((B, H + 2, W + 2, Cc), device=x.device, dtype=f16)
    cabi.check(cabi.lib().udb_reflect_pad1_nhwc_f16(_ptr(x), _ptr(out), B, H, W, Cc, _stream()), "udb_reflect_pad1_nhwc_f16")
    return out


def reflect_border_fill(buf):
    """In place: 1-pixel reflect border of a padded NHWC f16 buffer [B,H+2,W+2,C] from its interior."""
    B, PH, PW, Cc = buf.shape
    cabi.check(cabi.lib().udb_reflect_border_fill_nhwc_f16(_ptr(buf), B, PH - 2, PW - 2, Cc, _stream()),
               "udb_reflect_border_fill_nhwc_f16")
    return buf


def postprocess(radius, confidence, intr4, B, net_hw, padded_hw, pad_l, pad_t, out_hw, rays_in=None, mode="bilinear"):
    """Output assembly (udb_postprocess): resize points = rays*radius, confidence and rays from the network to the padded
    input size with F.interpolate(mode, align_corners=False) semantics, crop the paddings; mode "bilinear" or "bicubic"."""
    if mode not in cabi.INTERP_MODES:
        raise ValueError(f"postprocess: mode {mode!r} is not one of {sorted(cabi.INTERP_MODES)}")
    H, W = out_hw
    dev = radius.device
    outs = {
        "confidence": torch.empty((B, 1, H, W), device=dev, dtype=f32),
        "radius": torch.empty((B, 1, H, W), device=dev, dtype=f32),
        "depth": torch.empty((B, 1, H, W), device=dev, dtype=f32),
        "points": torch.empty((B, 3, H, W), device=dev, dtype=f32),
        "rays": torch.empty((B, 3, H, W), device=dev, dtype=f32),
    }
    p = cabi.Postprocess()
    p.radius, p.confidence, p.intr4, p.rays_in = _ptr(radius), _ptr(confidence), _ptr(intr4), _ptr(rays_in)
    p.B, p.net_h, p.net_w = B, net_hw[0], net_hw[1]
    p.padded_h, p.padded_w, p.pad_l, p.pad_t, p.H, p.W = padded_hw[0], padded_hw[1], pad_l, pad_t, H, W
    p.out_confidence, p.out_radius, p.out_depth = _ptr(outs["confidence"]), _ptr(outs["radius"]), _ptr(outs["depth"])
    p.out_points, p.out_rays = _ptr(outs["points"]), _ptr(outs["rays"])
    p.mode = cabi.INTERP_MODES[mode]
    kernel = "postprocess_bicubic_kernel" if mode == "bicubic" else "postprocess_kernel"
    cabi.check(_launch(kernel, 0.0, lambda: cabi.lib().udb_postprocess(C.byref(p), _stream()),
                       _nb(radius, confidence, rays_in, *outs.values())), "udb_postprocess")
    return outs


def _metric_operand(name, t, dtype):
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != dtype or not t.is_contiguous():
        raise ValueError(f"{name} must be a contiguous {dtype} CUDA tensor, got "
                         f"{t.dtype if isinstance(t, torch.Tensor) else type(t).__name__}"
                         f"{'' if not isinstance(t, torch.Tensor) else (' on ' + str(t.device))}")


def nearest_neighbor(x, y, lengths1=None, lengths2=None, both=True):
    """K = 1 squared-L2 nearest neighbours (udb_nearest_neighbor): x [N, P1, 3], y [N, P2, 3] f32 contiguous CUDA,
    lengths int64 [N] on the same device or None.  Returns (dist_x, idx_x, dist_y, idx_y); the y -> x pair is None
    unless `both`.  Lengths are assumed in [0, P] (the callers in validation.py check them)."""
    _metric_operand("x", x, f32)
    _metric_operand("y", y, f32)
    N, P1, _ = x.shape
    P2 = y.shape[1]
    for n, l in (("lengths1", lengths1), ("lengths2", lengths2)):
        if l is not None:
            _metric_operand(n, l, torch.int64)
    dev = x.device
    dist_x, idx_x = torch.empty((N, P1), device=dev, dtype=f32), torch.empty((N, P1), device=dev, dtype=torch.int64)
    dist_y = torch.empty((N, P2), device=dev, dtype=f32) if both else None
    idx_y = torch.empty((N, P2), device=dev, dtype=torch.int64) if both else None
    p = cabi.NearestNeighbor()
    p.x, p.y, p.lengths1, p.lengths2 = _ptr(x), _ptr(y), _ptr(lengths1), _ptr(lengths2)
    p.N, p.P1, p.P2 = N, P1, P2
    p.dist_x, p.idx_x, p.dist_y, p.idx_y = _ptr(dist_x), _ptr(idx_x), _ptr(dist_y), _ptr(idx_y)
    cabi.check(_launch("nn_kernel", 8.0 * N * P1 * P2, lambda: cabi.lib().udb_nearest_neighbor(C.byref(p), _stream())),
               "udb_nearest_neighbor")
    return dist_x, idx_x, dist_y, idx_y


def depth_metrics(gt, pred, mask, max_depth, thresholds, auc_thresholds, medians):
    """Per-image sums and counts of eval_depth (udb_depth_metrics): gt, pred [B, H, W] f32, mask [B, H, W] uint8,
    thresholds = (d1, d2, d3, tau) fp32 values, auc_thresholds [100] f32 ascending, medians [B, 2] f32 (median gt,
    median pred of the valid pixels).  Returns (out [B, DM_NACC] f64, ssi [B, 2] f32)."""
    _metric_operand("gt", gt, f32)
    _metric_operand("pred", pred, f32)
    _metric_operand("mask", mask, torch.uint8)
    _metric_operand("auc_thresholds", auc_thresholds, f32)
    _metric_operand("medians", medians, f32)
    B = gt.shape[0]
    HW = gt[0].numel()
    dev = gt.device
    partials = torch.empty((B, cabi.METRIC_MAX_BLOCKS, cabi.DM_NACC), device=dev, dtype=torch.float64)
    out = torch.empty((B, cabi.DM_NACC), device=dev, dtype=torch.float64)
    ssi = torch.empty((B, 2), device=dev, dtype=f32)
    p = cabi.DepthMetrics()
    p.gt, p.pred, p.mask, p.B, p.HW = _ptr(gt), _ptr(pred), _ptr(mask), B, HW
    p.use_max_depth = int(max_depth is not None)
    p.max_depth = float(max_depth) if max_depth is not None else 0.0
    p.thr_d1, p.thr_d2, p.thr_d3, p.thr_tau = thresholds
    p.auc_thresholds, p.medians = _ptr(auc_thresholds), _ptr(medians)
    p.partials, p.out, p.ssi = _ptr(partials), _ptr(out), _ptr(ssi)
    cabi.check(_launch("depth_metrics_kernel", 0.0, lambda: cabi.lib().udb_depth_metrics(C.byref(p), _stream()),
                       _nb(gt, pred, mask) * 2), "udb_depth_metrics")
    return out, ssi


def point_metrics(gt, pred, lengths, dist_x, dist_y, thresholds):
    """Per-cloud sums and F1 histograms of eval_3d (udb_point_metrics): gt, pred [N, P, 3] f32, lengths int64 [N] or
    None, dist_x, dist_y [N, P] f32, thresholds [T] f32 ascending.  Returns out [N, 2 + 2T] f64."""
    for n, t in (("gt", gt), ("pred", pred), ("dist_x", dist_x), ("dist_y", dist_y), ("thresholds", thresholds)):
        _metric_operand(n, t, f32)
    if lengths is not None:
        _metric_operand("lengths", lengths, torch.int64)
    N, P, _ = gt.shape
    T = thresholds.numel()
    dev = gt.device
    partials = torch.empty((N, cabi.METRIC_MAX_BLOCKS, 2 + 2 * T), device=dev, dtype=torch.float64)
    out = torch.empty((N, 2 + 2 * T), device=dev, dtype=torch.float64)
    p = cabi.PointMetrics()
    p.gt, p.pred, p.lengths, p.dist_x, p.dist_y, p.thresholds = (_ptr(gt), _ptr(pred), _ptr(lengths), _ptr(dist_x),
                                                                 _ptr(dist_y), _ptr(thresholds))
    p.N, p.P, p.n_thresholds = N, P, T
    p.partials, p.out = _ptr(partials), _ptr(out)
    cabi.check(_launch("point_metrics_kernel", 0.0, lambda: cabi.lib().udb_point_metrics(C.byref(p), _stream()),
                       _nb(gt, pred, dist_x, dist_y)), "udb_point_metrics")
    return out
