"""The CUDA-core kernels (elementwise.cu, v1_kernels.cu) on their own, at the shapes that select each template instance and
dispatch branch of their launchers, against float64 references with per-element bounds (derived in tests/kernel_ref.py)
or, where the kernel only copies, adds once or takes a maximum, against an exact restatement.  Every case

  * writes into a larger buffer filled with a NaN bit pattern (extra rows, a column offset or an extra image) and checks
    that every cell outside the written region still holds that pattern;
  * runs twice and requires bit-identical outputs;
  * prints its largest err / bound ratio (run with -s to see them)."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

import kernel_ref as R
from test_kernel_conformance_gpu import bits, sentinel, twice, untouched

pytestmark = pytest.mark.gpu

f16, f32 = torch.float16, torch.float32


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _lib():
    from unidepth_b200 import _cabi
    return _cabi, _cabi.lib()


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc, what):
    cabi, lib = _lib()
    cabi.check(rc, what)


def _mask(shape, dev, *index):
    m = torch.zeros(shape, dtype=torch.bool, device=dev)
    m[index] = True
    return m


def _exact(got, ref, name):
    got, ref = got.contiguous(), ref.contiguous()
    assert got.dtype == ref.dtype and torch.equal(bits(got), bits(ref)), f"{name}: not bit-exact"
    print(f"{name}: bit-exact")


# ------------------------------------------------------------------------------------------------ udb_layernorm
# general kernel (R = 1): dims 128 .. 1024, f16 / f32 in x f16 / f32 out, out_split, the row map
LN_CASES = [(128, True, True, False, False), (384, False, True, False, True), (640, True, False, True, False),
            (1024, False, False, False, True), (256, True, False, True, True), (896, True, False, False, False)]


@pytest.mark.parametrize("dim,in32,out32,split,rowmap", LN_CASES)
def test_layernorm_general(dim, in32, out32, split, rowmap):
    _, dev = _lib(), _dev()
    from unidepth_b200 import ops
    g = torch.Generator().manual_seed(dim + 7 * in32 + 3 * out32 + split)
    Bn, Np = 3, 37
    T = Np + 2 if rowmap else Np
    ld_in = dim + 64
    xb = (torch.randn(Bn * T, ld_in, generator=g) * 2 + 0.7).to(dev)
    xb = xb if in32 else xb.half()
    x = xb[:, :dim]
    w, b = torch.randn(dim, generator=g).to(dev), torch.randn(dim, generator=g).to(dev)
    rows = Bn * Np
    odt = f32 if out32 else f16
    width = 2 * dim if split else dim
    shape = (rows + 3, width + 16)
    mask = _mask(shape, dev, slice(1, 1 + rows), slice(8, 8 + width))
    kw = dict(rows_per_group=Np, group_stride=T, row_offset=1) if rowmap else {}

    def run():
        buf = sentinel(shape, odt, dev)
        ops.layernorm(x, w, b, 1e-6, out=buf[1:1 + rows, 8:8 + width], rows=rows, out_split=split, **kw)
        return [buf]

    name = f"layernorm dim{dim} {'f32' if in32 else 'f16'}->{'f32' if out32 else 'f16'}{' split' if split else ''}" \
           f"{' row map' if rowmap else ''}"
    buf, = twice(run, name)
    untouched(buf, mask, name)
    xin = torch.cat([x[bi * T + 1:bi * T + 1 + Np] for bi in range(Bn)]) if rowmap else x[:rows]
    ref, bnd = R.layernorm_ref(xin, w, b, 1e-6)
    got = buf[1:1 + rows, 8:8 + dim]
    if out32:
        R.within(got, ref, bnd, name)
    elif split:
        lo = buf[1:1 + rows, 8 + dim:8 + 2 * dim]
        bhi, bsum = R.split_out(ref, bnd, got, lo)
        R.within(got, ref, bhi, name + " hi")
        R.within(got.double() + lo.double(), ref, bsum, name + " hi + lo")
    else:
        R.within(got, ref, R.f16_out(ref, bnd), name)


@pytest.mark.parametrize("dim,dim_valid,rows", [(64, 0, 1), (64, 40, 37), (128, 96, 5), (128, 0, 67), (256, 0, 3),
                                                (256, 200, 130)])
def test_layernorm_f16_small(dim, dim_valid, rows):
    """layernorm_f16_small_kernel<8 / 16 / 32>: 4, 2 or 1 rows per warp, 32, 16 or 8 rows per block; row counts that
    leave warps and blocks partly empty; zero-padded rows with statistics over dim_valid columns"""
    _, dev = _lib(), _dev()
    from unidepth_b200 import ops
    g = torch.Generator().manual_seed(dim * 1000 + dim_valid + rows)
    xb = (torch.randn(rows, dim + 24, generator=g) * 1.5 - 0.3).half().to(dev)
    n = dim_valid or dim
    xb[:, n:dim] = 0
    x = xb[:, :dim]
    w, b = torch.randn(dim, generator=g).to(dev), torch.randn(dim, generator=g).to(dev)
    shape = (rows + 2, dim + 16)
    mask = _mask(shape, dev, slice(1, 1 + rows), slice(8, 8 + dim))

    def run():
        buf = sentinel(shape, f16, dev)
        ops.layernorm(x, w, b, 1e-5, out=buf[1:1 + rows, 8:8 + dim], dim_valid=dim_valid)
        return [buf]

    name = f"layernorm_f16_small dim{dim} dim_valid{dim_valid} rows{rows}"
    buf, = twice(run, name)
    untouched(buf, mask, name)
    ref, bnd = R.layernorm_ref(x, w, b, 1e-5, n)
    R.within(buf[1:1 + rows, 8:8 + dim], ref, R.f16_out(ref, bnd), name)


# ------------------------------------------------------------------------------------------------ udb_layernorm_any
# (dim, in32, out mode 0 f16 / 1 f32 / 2 split, add table, s2d): R = 4 up to 256 columns, 2 up to 768, 1 beyond
LN_ANY_CASES = [(64, True, 0, False, None), (192, False, 1, True, None), (256, True, 2, True, None),
                (320, False, 0, False, None), (768, True, 2, False, None), (512, False, 1, True, None),
                (1024, True, 0, True, None), (1536, False, 1, False, None), (1152, True, 2, False, None),
                (192, True, 0, False, (7, 9)), (128, False, 2, False, (5, 3)), (384, True, 1, False, (3, 5))]


@pytest.mark.parametrize("dim,in32,out,add,s2d", LN_ANY_CASES)
def test_layernorm_any(dim, in32, out, add, s2d):
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(dim * 10 + out + 100 * in32 + 1000 * add)
    if s2d:
        B, H, W = 2, *s2d
        rows = B * H * W
    else:
        rows = 8 * 4 * 3 + 5                          # not a multiple of 8 warps x R rows
    ld_in = dim + 32
    xb = (torch.randn(rows, ld_in, generator=g) * 2 + 0.5).to(dev)
    xb = xb if in32 else xb.half()
    w, bias = torch.randn(dim, generator=g).to(dev), torch.randn(dim, generator=g).to(dev)
    addt = torch.randn(11, dim, generator=g).to(dev) if add else None     # add_mod 11 does not divide rows
    odt = f32 if out == 1 else f16
    if s2d:
        orows, ocols = B * (H // 2) * (W // 2), 4 * dim
    else:
        orows, ocols = rows, dim
    ld_out = 2 * ocols + 16 if out == 2 else ocols + 8
    shape = (orows + 2, ld_out)
    mask = _mask(shape, dev, slice(1, 1 + orows), slice(0, ocols))
    if out == 2:
        mask[1:1 + orows, ld_out // 2:ld_out // 2 + ocols] = True

    def run():
        buf = sentinel(shape, odt, dev)
        p = cabi.LayerNormAny()
        p.inp, p.in_f32, p.out, p.out_f32, p.weight, p.bias = _p(xb), int(in32), _p(buf[1:]), out, _p(w), _p(bias)
        p.rows, p.dim, p.ld_in, p.ld_out, p.eps = rows, dim, ld_in, ld_out, 1e-6
        if add:
            p.add, p.add_mod = _p(addt), 11
        if s2d:
            p.s2d_h, p.s2d_w = H, W
        _check(lib.udb_layernorm_any(C.byref(p), _st()), "udb_layernorm_any")
        return [buf]

    name = f"layernorm_any dim{dim} {'f32' if in32 else 'f16'} out{out}{' add' if add else ''}{' s2d %dx%d' % s2d if s2d else ''}"
    buf, = twice(run, name)
    untouched(buf, mask, name)
    xin = xb[:, :dim].float()
    if add:
        xin = xin + addt[torch.arange(rows, device=dev) % 11]               # the kernel's one f32 add
    ref, bnd = R.layernorm_ref(xin, w, bias, 1e-6)
    if s2d:
        def s2d_map(t):
            t = t.reshape(B, H, W, dim)[:, :H // 2 * 2, :W // 2 * 2]
            return t.reshape(B, H // 2, 2, W // 2, 2, dim).permute(0, 1, 3, 2, 4, 5).reshape(orows, 4 * dim)
        ref, bnd = s2d_map(ref), s2d_map(bnd)
    got = buf[1:1 + orows, :ocols]
    if out == 1:
        R.within(got, ref, bnd, name)
    elif out == 2:
        lo = buf[1:1 + orows, ld_out // 2:ld_out // 2 + ocols]
        bhi, bsum = R.split_out(ref, bnd, got, lo)
        R.within(got, ref, bhi, name + " hi")
        R.within(got.double() + lo.double(), ref, bsum, name + " hi + lo")
    else:
        R.within(got, ref, R.f16_out(ref, bnd), name)


# ------------------------------------------------------------------------------------------------ cls rows
def test_set_cls_rows_and_ln_stats():
    """udb_set_cls_rows / udb_set_cls_rows_ln: rows b*T of x (f32) and x16 (f16) only; per-part {mean, M2} with 11 parts
    (not a multiple of the 8 warps) of 40 columns (not a multiple of 32)"""
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(5)
    B, T, parts, pc = 3, 5, 11, 40
    D = parts * pc
    cls, pos0 = (torch.randn(D, generator=g) * 2 + 1).to(dev), torch.randn(D, generator=g).to(dev)
    mask = torch.zeros(B * T, D, dtype=torch.bool, device=dev)
    mask[::T] = True
    smask = torch.zeros(B * T, parts, 2, dtype=torch.bool, device=dev)
    smask[::T] = True

    def run():
        x, x16, st = sentinel((B * T, D), f32, dev), sentinel((B * T, D), f16, dev), sentinel((B * T, parts, 2), f32, dev)
        xp = sentinel((B * T, D), f32, dev)
        _check(lib.udb_set_cls_rows_ln(_p(x), _p(x16), _p(st), _p(cls), _p(pos0), B, T, D, parts, pc, _st()), "cls_ln")
        _check(lib.udb_set_cls_rows(_p(xp), _p(cls), _p(pos0), B, T, D, _st()), "cls")
        return [x, x16, st, xp]

    x, x16, st, xp = twice(run, "set_cls_rows")
    for t, m, n in ((x, mask, "x"), (x16, mask, "x16"), (st, smask, "stats"), (xp, mask, "set_cls_rows x")):
        untouched(t, m, "set_cls_rows " + n)
    v = cls + pos0                                                          # the kernels' one f32 add
    for bi in range(B):
        _exact(x[bi * T], v, "set_cls_rows_ln x")
        _exact(x16[bi * T], v.half(), "set_cls_rows_ln x16")
        _exact(xp[bi * T], v, "set_cls_rows x")
    m, d, Q, dm, e, dQ = R.two_pass_stats(v.view(parts, pc).double(), pc)
    for bi in range(B):
        R.within(st[bi * T, :, 0], m[:, 0], dm[:, 0], "set_cls_rows_ln part mean")
        R.within(st[bi * T, :, 1], Q[:, 0], dQ[:, 0], "set_cls_rows_ln part M2")


# ------------------------------------------------------------------------------------------------ resamplers
AA_CASES = [(23, 37, 9, 14), (9, 14, 23, 37), (17, 19, 17, 19), (13, 11, 1, 1), (40, 7, 12, 3)]


@pytest.mark.parametrize("H,W,oh,ow", AA_CASES)
@pytest.mark.parametrize("dt", [f16, f32])
def test_aa_resize(H, W, oh, ow, dt):
    """non-integer downscale, upscale, identity, a 1-pixel output, mixed; C = 8 (one thread per pixel)"""
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(H * 100 + W + oh)
    B, Cc = 2, 8
    x = (torch.randn(B, H, W, Cc, generator=g) + 0.5).to(dev).to(dt)
    shape = (B + 1, oh, ow, Cc)
    mask = _mask(shape, dev, slice(0, B))
    fn = lib.udb_aa_resize_nhwc_f16 if dt == f16 else lib.udb_aa_resize_nhwc_f32

    def run():
        buf = sentinel(shape, dt, dev)
        _check(fn(_p(x), _p(buf), B, H, W, Cc, oh, ow, _st()), "aa_resize")
        return [buf]

    name = f"aa_resize {'f16' if dt == f16 else 'f32'} {H}x{W}->{oh}x{ow}"
    buf, = twice(run, name)
    untouched(buf, mask, name)
    ref, bnd = R.aa_resize_ref(x, oh, ow)
    R.within(buf[:B], ref, R.f16_out(ref, bnd) if dt == f16 else bnd, name)


@pytest.mark.parametrize("H,W", [(1, 5), (4, 1), (3, 6)])
def test_upsample2x(H, W):
    """H or W = 1: the source index clamps to the single row / column"""
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(H * 10 + W)
    B, Cc = 2, 16
    x = torch.randn(B, H, W, Cc, generator=g).half().to(dev)
    shape = (B + 1, 2 * H, 2 * W, Cc)
    mask = _mask(shape, dev, slice(0, B))

    def run():
        buf = sentinel(shape, f16, dev)
        _check(lib.udb_upsample2x_nhwc_f16(_p(x), _p(buf), B, H, W, Cc, _st()), "upsample2x")
        return [buf]

    name = f"upsample2x {H}x{W}"
    buf, = twice(run, name)
    untouched(buf, mask, name)
    ref, bnd = R.upsample2x_ref(x)
    R.within(buf[:B], ref, R.f16_out(ref, bnd), name)


@pytest.mark.parametrize("H,W,oh,ow,pad", [(5, 7, 2, 9, 1), (6, 3, 11, 2, 0), (9, 9, 4, 6, 1), (4, 5, 7, 8, 0)])
def test_resize_ac_pad(H, W, oh, ow, pad):
    """align_corners bilinear + reflect pad, pad 0 and 1, oh or ow = 2"""
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(H * 1000 + W * 100 + oh * 10 + ow)
    B, Cc = 2, 8
    x = torch.randn(B, H, W, Cc, generator=g).half().to(dev)
    shape = (B + 1, oh + 2 * pad, ow + 2 * pad, Cc)
    mask = _mask(shape, dev, slice(0, B))

    def run():
        buf = sentinel(shape, f16, dev)
        _check(lib.udb_resize_ac_pad_nhwc_f16(_p(x), _p(buf), B, H, W, Cc, oh, ow, pad, _st()), "resize_ac_pad")
        return [buf]

    name = f"resize_ac_pad {H}x{W}->{oh}x{ow} pad{pad}"
    buf, = twice(run, name)
    untouched(buf, mask, name)
    ref, bnd = R.resize_ac_pad_ref(x, oh, ow, pad)
    R.within(buf[:B], ref, R.f16_out(ref, bnd), name)


@pytest.mark.parametrize("H,W", [(2, 2), (2, 7), (5, 2)])
def test_reflect_pad_and_border_fill(H, W):
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(H * 10 + W)
    B, Cc = 2, 16
    x = torch.randn(B, H, W, Cc, generator=g).half().to(dev)
    ref = F.pad(x.permute(0, 3, 1, 2).float(), (1, 1, 1, 1), mode="reflect").permute(0, 2, 3, 1).half()
    shape = (B + 1, H + 2, W + 2, Cc)
    mask = _mask(shape, dev, slice(0, B))

    def run():
        buf = sentinel(shape, f16, dev)
        _check(lib.udb_reflect_pad1_nhwc_f16(_p(x), _p(buf), B, H, W, Cc, _st()), "reflect_pad1")
        fill = sentinel(shape, f16, dev)
        fill[:B, 1:H + 1, 1:W + 1] = x
        _check(lib.udb_reflect_border_fill_nhwc_f16(_p(fill), B, H, W, Cc, _st()), "reflect_border_fill")
        return [buf, fill]

    name = f"reflect pad {H}x{W}"
    buf, fill = twice(run, name)
    untouched(buf, mask, name)
    untouched(fill, mask, name + " border fill")
    _exact(buf[:B], ref, name)
    _exact(fill[:B], ref, name + " border fill")


@pytest.mark.parametrize("net_hw,pads,out_hw", [((37, 53), (3, 4, 2, 5), (61, 70)), ((37, 53), (1, 2, 3, 1), (13, 19))])
def test_v1_mean_maps_and_postprocess_depth(net_hw, pads, out_hw):
    """paddings on all four sides; output sizes above and below the cropped network size.  Depth is the resampled mean,
    points.z equals it bit for bit, and the x / y planes are the back-projection of the kernel's own depth"""
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(sum(out_hw))
    B, gh, gw = 2, 4, 6
    nh, nw = net_hw
    outs = [(torch.rand(B, gh << s, gw << s, generator=g) + 0.5).to(dev) for s in (1, 2, 3)]
    H, W = out_hw
    k4 = torch.tensor([[60.0, 58.0, 31.0, 33.0], [45.0, 47.0, 40.0, 22.0]], device=dev)

    def run():
        mean = sentinel((B + 1, nh, nw), f32, dev)
        _check(lib.udb_v1_mean_maps(_p(outs[0]), _p(outs[1]), _p(outs[2]), _p(mean), B, gh, gw, nh, nw, _st()), "mean_maps")
        od, op = sentinel((B + 1, H, W), f32, dev), sentinel((B + 1, 3, H, W), f32, dev)
        pp = cabi.V1Postprocess()
        pp.mean, pp.k4, pp.B, pp.net_h, pp.net_w = _p(mean), _p(k4), B, nh, nw
        pp.pad_l, pp.pad_r, pp.pad_t, pp.pad_b, pp.H, pp.W, pp.out_depth, pp.out_points = *pads, H, W, _p(od), _p(op)
        _check(lib.udb_v1_postprocess(C.byref(pp), _st()), "v1_postprocess")
        return [mean, od, op]

    name = f"v1 mean maps {nh}x{nw} pads {pads} -> {H}x{W}"
    mean, od, op = twice(run, name)
    for t in (mean, od, op):
        untouched(t, _mask(t.shape, dev, slice(0, B)), name)
    ref, bnd = R.mean_maps_ref(outs, nh, nw)
    R.within(mean[:B], ref, bnd, "v1_mean_maps " + name)
    pl, pr, pt, pb = pads
    crop = mean[:B, pt:nh - pb, pl:nw - pr]
    dref, dbnd = R.aa_resize_ref(crop[..., None], H, W)
    R.within(od[:B], dref[..., 0], dbnd[..., 0], "v1_postprocess depth " + name)
    _exact(op[:B, 2], od[:B], "v1_postprocess points.z")
    (xr, yr), (bx, by) = R.v1_points_ref(od[:B], k4, H, W)
    R.within(op[:B, 0], xr, bx, "v1_postprocess points.x " + name)
    R.within(op[:B, 1], yr, by, "v1_postprocess points.y " + name)


# ------------------------------------------------------------------------------------------------ small dense pieces
SOFTMAX_CASES = [(37, 5, 8, 8, 0.7, 1.0), (20, 64, 64, 64, 0.3, 4.0), (9, 40, 72, 48, 1.0, 2.0), (12, 300, 300, 320, 1.0, 30.0)]


@pytest.mark.parametrize("rows,n_valid,ld_in,ld_out,scale,gain", SOFTMAX_CASES)
def test_softmax_rows(rows, n_valid, ld_in, ld_out, scale, gain):
    """n_valid < 32; n_valid == ld_out; NaN in s beyond n_valid (never read); logits spanning > 80 after scaling"""
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(rows + n_valid)
    s = (torch.randn(rows, ld_in, generator=g) * gain).to(dev)
    s[:, n_valid:] = float("nan")
    if gain > 10:
        span = ((s[:, :n_valid].amax(-1) - s[:, :n_valid].amin(-1)) * scale).min().item()
        assert span > 80, span
    shape = (rows + 2, ld_out)
    mask = _mask(shape, dev, slice(1, 1 + rows))

    def run():
        buf = sentinel(shape, f16, dev)
        _check(lib.udb_softmax_rows(_p(s), _p(buf[1:]), rows, n_valid, ld_in, ld_out, scale, _st()), "softmax_rows")
        return [buf]

    name = f"softmax_rows {rows}x{n_valid} ld_in {ld_in} ld_out {ld_out}"
    buf, = twice(run, name)
    untouched(buf, mask, name)
    P, bnd = R.softmax_rows_ref(s, n_valid, scale)
    R.within(buf[1:1 + rows, :n_valid], P, bnd, name)
    assert (bits(buf[1:1 + rows, n_valid:]) == 0).all(), name


CROSS_CASES = [(1, 1, 256, True), (2, 9, 256, False), (3, 15, 512, True), (4, 16, 256, True), (4, 17, 512, False),
               (2, 45, 256, True), (4, 333, 512, True)]


@pytest.mark.parametrize("nq,nk,D,with_pos", CROSS_CASES)
def test_cross_attn_small(nq, nk, D, with_pos):
    """f16 keys / values: 1-4 queries; nk < 16 leaves splits without keys; nk not a multiple of 16"""
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(nq * 1000 + nk + D)
    B = 2
    q = torch.randn(B * nq, D, generator=g).to(dev)
    pos = torch.randn(nq, D, generator=g).to(dev) if with_pos else None
    kv = torch.randn(B * nk, 2 * D, generator=g).half().to(dev)
    scale = D ** -0.5
    shape = (B * nq + 2, D)
    mask = _mask(shape, dev, slice(1, 1 + B * nq))

    def run():
        buf = sentinel(shape, f32, dev)
        scratch = torch.full((B * 16 * nq * (D + 2),), float("nan"), device=dev)
        _check(lib.udb_cross_attn_small(_p(q), _p(pos), _p(kv), _p(buf[1:]), _p(scratch), B, nq, nk, D, scale, _st()), "cross")
        return [buf]

    name = f"cross_attn_small nq{nq} nk{nk} D{D}"
    buf, = twice(run, name)
    untouched(buf, mask, name)
    qq = (q.view(B, nq, D) + (pos if with_pos else 0)).double()            # (q + pos) scale: 2 u32 relative on q'
    k, v = kv.double().view(B, nk, 2 * D)[..., :D], kv.double().view(B, nk, 2 * D)[..., D:]
    s = (qq * scale) @ k.transpose(1, 2)
    ds = (D + 4) * R.U32 * ((qq.abs() * scale) @ k.abs().transpose(1, 2))
    ref, bnd = R.softmax_av_ref(s, ds, v, nk + 16)
    R.within(buf[1:1 + B * nq].view(B, nq, D), ref, bnd, name)


@pytest.mark.parametrize("heads,Cc", [(1, 64), (2, 512), (8, 384), (16, 256)])
def test_camera_attn4(heads, Cc):
    """head widths 64, 256, 48 (not a multiple of 32) and 16 (below 32)"""
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(heads * 1000 + Cc)
    B = 3
    q, pos = torch.randn(B, 4, Cc, generator=g).to(dev), torch.randn(4, Cc, generator=g).to(dev)
    kv = torch.randn(B, 4, 2 * Cc, generator=g).to(dev)
    shape = (B + 1, 4, Cc)
    mask = _mask(shape, dev, slice(0, B))

    def run():
        buf = sentinel(shape, f32, dev)
        _check(lib.udb_camera_attn4_f32(_p(q), _p(kv), _p(pos), _p(buf), B, Cc, heads, _st()), "camera_attn4")
        return [buf]

    name = f"camera_attn4 heads{heads} C{Cc}"
    buf, = twice(run, name)
    untouched(buf, mask, name)
    ref, bnd = R.camera_attn4_ref(q, pos, kv, heads)
    R.within(buf[:B].view(B, 4, heads, Cc // heads).transpose(1, 2), ref, bnd, name)


SL_CASES = [  # M, N, K, epilogue, x row offset (floats), strided
    (5, 33, 256, "plain", 0, False), (13, 6, 256, "bias_gelu", 0, True), (8, 12, 512, "gamma_resid", 0, True),
    (3, 7, 200, "bias", 0, False), (9, 20, 96, "gamma_resid", 0, True), (13, 33, 384, "bias_gelu", 0, True),
    (6, 10, 256, "gamma_resid", 1, True), (4, 9, 128, "bias", 3, False)]


@pytest.mark.parametrize("M,N,K,epi,xoff,strided", SL_CASES)
def test_small_linear(M, N, K, epi, xoff, strided):
    """both loops: 16-byte loads (K % 128 == 0, ldx % 4 == 0, x 16-byte aligned) and one float per lane (K % 128 != 0, or
    x a view 4 or 12 bytes into its buffer); M not a multiple of 8, N not a multiple of 4; strided x, out and resid"""
    _, dev = _lib(), _dev()
    from unidepth_b200 import ops
    g = torch.Generator().manual_seed(M * 10000 + N * 100 + K + xoff)
    ldx = K + (8 if strided else 0)                                         # ldx % 4 == 0 even where x is misaligned
    xb = torch.randn(M * ldx + 4, generator=g).to(dev)
    x = xb[xoff:xoff + M * ldx].view(M, ldx)[:, :K]
    assert (x.data_ptr() % 16 == 0) == (xoff == 0)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
    bias = torch.randn(N, generator=g).to(dev) if epi != "plain" else None
    act = ops.ACT_GELU if epi == "bias_gelu" else ops.ACT_NONE
    gamma = (torch.rand(N, generator=g) + 0.5).to(dev) if epi == "gamma_resid" else None
    resid = torch.randn(M, N + 5, generator=g).to(dev)[:, 2:2 + N] if epi == "gamma_resid" else None
    ldy = N + 7 if strided else N
    shape = (M + 2, ldy + 4)
    mask = _mask(shape, dev, slice(1, 1 + M), slice(4, 4 + N))

    def run():
        buf = sentinel(shape, f32, dev)
        ops.small_linear(x, w, bias=bias, act=act, gamma=gamma, resid=resid, out=buf[1:1 + M, 4:4 + N])
        return [buf]

    name = f"small_linear M{M} N{N} K{K} {epi} x+{4 * xoff}B{' strided' if strided else ''}"
    buf, = twice(run, name)
    untouched(buf, mask, name)
    ref, bnd = R.small_linear_ref(x, w, bias=bias, act=act, gamma=gamma, resid=resid)
    R.within(buf[1:1 + M, 4:4 + N], ref, bnd, name)


# ------------------------------------------------------------------------------------------------ Nystrom pieces
@pytest.mark.parametrize("n,heads", [(128, 1), (1000, 2), (300, 3), (131, 4)])
def test_nystrom_landmarks_k2_zk3(n, heads):
    """segment means (n % 128 != 0: the last segments one row longer), kernel_2 = softmax(ql kl^T / 8) against float64,
    and the (z . kernel_3) product for a given f32 z.  The pseudo-inverse itself: test_nystrom_pinv_newton_schulz."""
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(n * 10 + heads)
    B, m = 2, 128
    Cc = heads * 64
    qb = (torch.randn(B * n, Cc + 64, generator=g) * 0.7).half().to(dev)              # q in the first Cc columns
    kvb = (torch.randn(B * n, 2 * Cc, generator=g) * 0.7).half().to(dev)
    lshape = (B * m + 2, 2 * Cc)
    lmask = _mask(lshape, dev, slice(1, 1 + B * m))
    mm = B * heads * m * m
    z = (torch.randn(B * heads, m, m, generator=g) / m ** 0.5).to(dev)
    k3 = torch.randn(B * m, Cc, generator=g).half().to(dev)
    ldo = Cc + 16
    wshape = (B * m + 2, ldo)
    wmask = _mask(wshape, dev, slice(1, 1 + B * m), slice(0, Cc))

    def run():
        lm = sentinel(lshape, f16, dev)
        _check(lib.udb_nystrom_landmarks(_p(qb), Cc + 64, _p(kvb), 2 * Cc, _p(lm[1:]), B, n, heads, _st()), "landmarks")
        k2, zz = sentinel((mm + 64,), f32, dev), torch.empty(mm, device=dev)
        tmp = torch.empty(3 * mm, device=dev)
        _check(lib.udb_nystrom_k2_pinv(_p(lm[1:]), _p(k2), _p(zz), _p(tmp), B, heads, 0, _st()), "k2")
        w2 = sentinel(wshape, f16, dev)
        _check(lib.udb_nystrom_zk3(_p(z), _p(k3), Cc, _p(w2[1:]), ldo, B, heads, _st()), "zk3")
        return [lm, k2, w2]

    name = f"nystrom n{n} heads{heads}"
    lm, k2, w2 = twice(run, name)
    untouched(lm, lmask, name + " landmarks")
    untouched(k2, torch.arange(mm + 64, device=dev) < mm, name + " k2")
    untouched(w2, wmask, name + " zk3")
    # segments: the first m - n % m have n // m rows, the rest one more (n % m == 0: all equal)
    for which, src in (("q", qb[:, :Cc]), ("k", kvb[:, :Cc])):
        ref, bnd = R.segment_mean_ref(src.reshape(B, n, Cc), R.nystrom_segments(n))
        got = lm[1:1 + B * m].view(B, m, 2 * Cc)[..., :Cc] if which == "q" else lm[1:1 + B * m].view(B, m, 2 * Cc)[..., Cc:]
        R.within(got, ref, bnd, f"{name} {which} landmarks")
    lmd = lm[1:1 + B * m].view(B, m, 2, heads, 64).double()
    ql, kl = lmd[:, :, 0].transpose(1, 2), lmd[:, :, 1].transpose(1, 2)            # [B, heads, m, 64]
    s = ql @ kl.transpose(-1, -2) * 0.125
    ds = 64 * R.U32 * (ql.abs() @ kl.abs().transpose(-1, -2)) * 0.125
    eye = torch.eye(m, device=dev, dtype=torch.float64).expand(B, heads, m, m)
    P, bP = R.softmax_av_ref(s, ds, eye, m)
    R.within(k2[:mm].view(B, heads, m, m), P, bP, name + " kernel_2")
    zd = z.double().view(B, heads, m, m)
    k3d = k3.double().view(B, m, heads, 64).transpose(1, 2)
    ref = zd @ k3d
    bnd = R.f16_out(ref, m * R.U32 * (zd.abs() @ k3d.abs()))
    got = w2[1:1 + B * m, :Cc].view(B, m, heads, 64).transpose(1, 2)
    R.within(got, ref, bnd, name + " zk3")


def test_nystrom_pinv_newton_schulz():
    """udb_nystrom_k2_pinv with 0 .. 6 Newton-Schulz iterations (the engine runs 6): the launcher is deterministic, so
    iters = t yields the t-th iterate of the same run.  Z0 is checked against K^T / max column sum, every later iterate
    against one float64 step from the kernel's previous iterate (bounds in tests/kernel_ref.py); Z and the scratch sit in
    NaN-patterned buffers, kernel_2 is the same in every run"""
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(77)
    B, heads, m = 2, 2, 128
    lm = (torch.randn(B * m, 2 * heads * 64, generator=g) * 0.7).half().to(dev)
    mm = B * heads * m * m
    zshape = (mm + 64,)
    zmask = torch.arange(mm + 64, device=dev) < mm
    iterates, k2s = [], []
    for t in range(7):
        def run():
            k2, z = sentinel((mm,), f32, dev), sentinel(zshape, f32, dev)
            tmp = sentinel((3 * mm,), f32, dev)
            _check(lib.udb_nystrom_k2_pinv(_p(lm), _p(k2), _p(z), _p(tmp), B, heads, t, _st()), "k2_pinv")
            return [k2, z]

        k2, z = twice(run, f"nystrom pinv iters={t}")
        untouched(z, zmask, f"nystrom pinv iters={t}")
        iterates.append(z[:mm].view(B * heads, m, m))
        k2s.append(k2)
    for k2 in k2s[1:]:
        _exact(k2, k2s[0], "nystrom kernel_2 across runs")
    K = k2s[0].view(B * heads, m, m)
    ref, bnd = R.pinv_init_ref(K)
    R.within(iterates[0], ref, bnd, "nystrom pinv init Z0")
    for t in range(1, 7):
        ref, bnd = R.newton_schulz_step_ref(K, iterates[t - 1])
        R.within(iterates[t], ref, bnd, f"nystrom Newton-Schulz step {t}")


# ------------------------------------------------------------------------------------------------ V1 pieces
@pytest.mark.parametrize("Cc,B,H,W", [(64, 1, 3, 5), (64, 2, 5, 8), (128, 2, 7, 9), (256, 1, 6, 11), (64, 2, 1, 9),
                                     (256, 1, 9, 1)])
def test_conv3x3_c1_exp(Cc, B, H, W):
    """conv3x3_c1_kernel<8 / 16 / 32>: 4, 2 or 1 pixels per warp; pixel counts that leave warps partly empty; every border
    pixel of the map; logits past both clamps (+-10)"""
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(Cc * 100 + H * 10 + W)
    x = torch.randn(B, H, W, Cc, generator=g).half().to(dev)
    w = (torch.randn(9, Cc, generator=g) * (40.0 / (9 * Cc) ** 0.5)).to(dev)             # |z| well past 10 somewhere
    shape = (B + 1, H, W)
    mask = _mask(shape, dev, slice(0, B))

    def run():
        buf = sentinel(shape, f32, dev)
        _check(lib.udb_conv3x3_c1_exp(_p(x), _p(w), 0.25, _p(buf), B, H, W, Cc, _st()), "conv3x3_c1")
        return [buf]

    name = f"conv3x3_c1_exp C{Cc} {B}x{H}x{W}"
    buf, = twice(run, name)
    untouched(buf, mask, name)
    ref, bnd = R.conv3x3_c1_ref(x, w, 0.25)
    if B * H * W >= 30:                           # every instance: C = 64 at 2x5x8, 128 and 256
        assert (ref > math.exp(9.99)).any() and (ref < math.exp(-9.99)).any(), name     # both clamps active
    R.within(buf[:B], ref, bnd, name)


@pytest.mark.parametrize("first", [1, 0])
def test_max_accum(first):
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(first)
    n = 8 * 1001
    src = torch.randn(n, generator=g).to(dev)
    d0 = torch.randn(n, generator=g).to(dev)
    for dt, fn in ((f16, lib.udb_max_accum_f16), (f32, lib.udb_max_accum_f32)):
        s, dd = src.to(dt), d0.to(dt)

        def run():
            buf = sentinel((n + 24,), dt, dev)
            buf[8:8 + n] = dd
            _check(fn(_p(s), _p(buf[8:]), n, first, _st()), "max_accum")
            return [buf]

        name = f"max_accum {'f16' if dt == f16 else 'f32'} first={first}"
        buf, = twice(run, name)
        untouched(buf, _mask((n + 24,), dev, slice(8, 8 + n)), name)
        _exact(buf[8:8 + n], s if first else torch.maximum(s, dd), name)


@pytest.mark.parametrize("B,HW,Cc", [(2, 1, 64), (3, 13, 40), (1, 70, 96)])
def test_spatial_mean(B, HW, Cc):
    """HW = 1; HW not a multiple of the 8 row groups; C not a multiple of 32"""
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(B * 1000 + HW + Cc)
    x = (torch.randn(B, HW, Cc, generator=g) + 0.3).to(dev)

    def run():
        buf = sentinel((B + 1, Cc), f32, dev)
        _check(lib.udb_spatial_mean_f32(_p(x), _p(buf), B, HW, Cc, _st()), "spatial_mean")
        return [buf]

    name = f"spatial_mean B{B} HW{HW} C{Cc}"
    buf, = twice(run, name)
    untouched(buf, _mask((B + 1, Cc), dev, slice(0, B)), name)
    ref, bnd = R.spatial_mean_ref(x)
    R.within(buf[:B], ref, bnd, name)


@pytest.mark.parametrize("mode", ["f32", "f16", "both"])
def test_add_f32(mode):
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(len(mode))
    n = 4 * 777
    a, b = torch.randn(n, generator=g).to(dev), torch.randn(n, generator=g).to(dev)
    shape = (n + 16,)
    mask = _mask(shape, dev, slice(4, 4 + n))

    def run():
        o, o16 = sentinel(shape, f32, dev), sentinel(shape, f16, dev)
        _check(lib.udb_add_f32(_p(a), _p(b), _p(o[4:]) if mode != "f16" else None, _p(o16[4:]) if mode != "f32" else None, n,
                               _st()), "add_f32")
        return [o, o16]

    o, o16 = twice(run, f"add_f32 {mode}")
    r = a + b
    if mode != "f16":
        untouched(o, mask, "add_f32 out")
        _exact(o[4:4 + n], r, f"add_f32 {mode} f32")
    else:
        untouched(o, torch.zeros_like(mask), "add_f32 out (not requested)")
    if mode != "f32":
        untouched(o16, mask, "add_f32 out_f16")
        _exact(o16[4:4 + n], r.half(), f"add_f32 {mode} f16")
    else:
        untouched(o16, torch.zeros_like(mask), "add_f32 out_f16 (not requested)")


def test_copy_rows_f32_to_f16():
    """rows (g * dst_group_stride + dst_row0 + r): the cls tokens appended after each image's tokens"""
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(21)
    groups, rpg, D, stride, row0 = 3, 4, 72, 11, 6
    src = torch.randn(groups * rpg, D, generator=g).to(dev)
    shape = (groups * stride + 2, D)
    mask = torch.zeros(shape, dtype=torch.bool, device=dev)
    for gi in range(groups):
        mask[gi * stride + row0:gi * stride + row0 + rpg] = True

    def run():
        buf = sentinel(shape, f16, dev)
        _check(lib.udb_copy_rows_f32_to_f16(_p(src), _p(buf), groups, rpg, D, stride, row0, _st()), "copy_rows")
        return [buf]

    buf, = twice(run, "copy_rows")
    untouched(buf, mask, "copy_rows")
    for gi in range(groups):
        _exact(buf[gi * stride + row0:gi * stride + row0 + rpg], src[gi * rpg:(gi + 1) * rpg].half(), f"copy_rows group {gi}")


def _one_of(got, cands, name):
    """bit-equal to one of the candidate f32 evaluations (a * b + c may be contracted to one fma)"""
    ok = torch.zeros_like(got, dtype=torch.bool)
    for c in cands:
        ok |= bits(got.contiguous()) == bits(c.contiguous())
    assert ok.all(), name


@pytest.mark.parametrize("x4,gt_k,skip", [(True, False, 0), (True, True, 0), (True, True, 1), (False, True, 1), (False, True, 0)])
def test_v1_camera_intrinsics(x4, gt_k, skip):
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(4 * x4 + 2 * gt_k + skip)
    B, nh, nw, ratio, pl, pt = 3, 462, 616, 0.962, 5, 7
    xv = (torch.randn(B, 4, generator=g) * 0.5).to(dev) if x4 else None
    K = torch.tensor([[500.0, 0, 320.0], [0, 505.0, 240.0], [0, 0, 1]]).repeat(B, 1, 1)
    K[:, 0, 0] += torch.arange(B) * 13.5
    K = K.to(dev) if gt_k else None
    shapes = [(B + 1, 4), (B + 1, 3, 3), (B + 1, 4)]

    def run():
        bufs = [sentinel(s, f32, dev) for s in shapes]
        _check(lib.udb_v1_camera_intrinsics(_p(xv), _p(K), B, nh, nw, ratio, pl, pt, skip, *(_p(b) for b in bufs), _st()), "v1 K")
        return bufs

    name = f"v1_camera_intrinsics x4={x4} gt_k={gt_k} skip={skip}"
    ir, ko, kp = twice(run, name)
    for t in (ir, ko, kp):
        untouched(t, _mask(t.shape, dev, slice(0, B)), name)
    r32 = torch.tensor(ratio, dtype=f32, device=dev)
    if x4:
        half = max(nh, nw) / 2.0
        xd = xv.double()
        pred = torch.stack([half * xd[:, 0].exp(), half * xd[:, 1].exp(), nw * torch.sigmoid(xd[:, 2]),
                            nh * torch.sigmoid(xd[:, 3])], 1)
        pb = pred.abs() * (2.0 ** -22 + 4 * R.U32)                          # expf 2 ulp, then <= 3 roundings
    if gt_k:
        rf = [K[:, 0, 0] * r32, K[:, 1, 1] * r32]
        rc = [(K[:, 0, 2].double() * r32.double() + pl).float(), (K[:, 1, 2].double() * r32.double() + pt).float()]
        rc2 = [K[:, 0, 2] * r32 + pl, K[:, 1, 2] * r32 + pt]
        _exact(ir[:B, :2], torch.stack(rf, 1), name + " rays fx, fy")
        _one_of(ir[:B, 2:], [torch.stack(rc, 1), torch.stack(rc2, 1)], name + " rays cx, cy")
        _exact(kp[:B], ir[:B], name + " points K")
    else:
        R.within(ir[:B], pred, pb, name + " rays K")
    # the returned K is computed from the values in intr4_rays unless a GT K steers the rays while the prediction is returned
    if gt_k and x4 and not skip:
        back = torch.stack([ko[:B, 0, 0] * r32, ko[:B, 1, 1] * r32, ko[:B, 0, 2] * r32 + pl, ko[:B, 1, 2] * r32 + pt], 1)
        pads = torch.tensor([0.0, 0.0, pl, pt], device=dev, dtype=torch.float64)
        R.within(back, pred, pb + 4 * R.U32 * (pred.abs() + pads), name + " returned K (prediction)")
    else:
        fx, fy, cx, cy = ir[:B].unbind(1)
        kexp = torch.zeros(B, 3, 3, device=dev)
        kexp[:, 0, 0], kexp[:, 1, 1] = fx / r32, fy / r32
        kexp[:, 0, 2], kexp[:, 1, 2] = (cx - pl) / r32, (cy - pt) / r32
        kexp[:, 2, 2] = 1
        _exact(ko[:B], kexp, name + " returned K")
    z = ko[:B].clone()
    assert (z[:, [0, 1, 2, 2], [1, 0, 0, 1]] == 0).all() and (z[:, 2, 2] == 1).all(), name
    if not gt_k:
        _exact(kp[:B], torch.stack([ko[:B, 0, 0], ko[:B, 1, 1], ko[:B, 0, 2], ko[:B, 1, 2]], 1), name + " points K")


def test_camera_intrinsics_and_adjust_k():
    """udb_camera_intrinsics (V2 camera head tail) and udb_camera_adjust_k (infer(camera=K))"""
    _, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(31)
    B, nh, nw, factor, pl, pt = 3, 420, 560, 0.875, 6, 10
    x = (torch.randn(B, 4, generator=g) * 0.5).to(dev)

    def run():
        bufs = [sentinel((B + 1, 4), f32, dev), sentinel((B + 1, 3, 3), f32, dev), sentinel((B + 1, 3, 3), f32, dev)]
        _check(lib.udb_camera_intrinsics(_p(x), B, nh, nw, factor, pl, pt, *(_p(b) for b in bufs), _st()), "camera_intrinsics")
        return bufs

    i4, kn, ko = twice(run, "camera_intrinsics")
    for t in (i4, kn, ko):
        untouched(t, _mask(t.shape, dev, slice(0, B)), "camera_intrinsics")
    diag = torch.tensor(float(nh * nh + nw * nw), dtype=f32).sqrt()        # sqrtf: correctly rounded
    c07 = (torch.tensor(0.7, dtype=f32) * diag).double().item()            # 0.7f * diag, one rounding
    xd = x.double()
    ref = torch.stack([xd[:, 0].exp() * c07, xd[:, 1].exp() * c07, nw * torch.sigmoid(xd[:, 2]), nh * torch.sigmoid(xd[:, 3])], 1)
    R.within(i4[:B], ref, ref.abs() * (2.0 ** -22 + 4 * R.U32), "camera_intrinsics fx fy cx cy")
    fx, fy, cx, cy = i4[:B].unbind(1)
    zero = torch.zeros(B, device=dev)
    _exact(kn[:B].reshape(B, 9), torch.stack([fx, zero, cx, zero, fy, cy, zero, zero, zero + 1], 1), "camera_intrinsics K_net")
    fct = torch.tensor(factor, dtype=f32, device=dev)
    _exact(ko[:B].reshape(B, 9), torch.stack([fx / fct, zero, cx / fct - pl, zero, fy / fct, cy / fct - pt, zero, zero, zero + 1], 1),
           "camera_intrinsics K_out")
    K = (torch.rand(B, 3, 3, generator=g) * 500 + 100).to(dev)

    def run_adj():
        buf = sentinel((B + 1, 4), f32, dev)
        _check(lib.udb_camera_adjust_k(_p(K), B, factor, pl, pt, _p(buf), _st()), "camera_adjust_k")
        return [buf]

    a, = twice(run_adj, "camera_adjust_k")
    untouched(a, _mask(a.shape, dev, slice(0, B)), "camera_adjust_k")
    _exact(a[:B], torch.stack([K[:, 0, 0] * fct, K[:, 1, 1] * fct, (K[:, 0, 2] + pl) * fct, (K[:, 1, 2] + pt) * fct], 1),
           "camera_adjust_k")
