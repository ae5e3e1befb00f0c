"""UniDepthV1 precision = "split" on the GPU: the kernels the mode adds (split pre-processing and LayerNorm outputs, the f32
depthwise 7x7, f32 level taps, the f32 antialiased resize and the camera head's cross attention on f32 keys / values)
against torch restatements in f32 / f64 and, where an f16 kernel does the same work, bit for bit against it; then
UniDepthV1.infer in split mode on the four V1 goldens (north_star: intrinsics < 1e-4, depth ARel < 1e-3), printed as
`V1SPLITPARITY` lines."""
import copy
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
f16, f32 = torch.float16, torch.float32
WIDTHS = [64, 128, 192, 384, 768, 1536]          # the ConvNeXt-L widths and the small test arch's
MAPS = [(115, 154), (57, 77), (28, 38), (14, 19), (1, 1), (3, 5)]


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _lib():
    from unidepth_b200 import _cabi
    return _cabi, _cabi.lib()


def _check_lo(hi, lo):
    """lo = f16(v - f32(hi)) with hi = f16(v): at most half an f16 step of hi (2^-11 relative), or half the subnormal
    step, 2^-25, below f16's normal range.  (Recomputing lo from hi + lo is not exact: where v - hi rounds to exactly half
    a step, f16(hi + lo) may round to the other neighbour.)"""
    assert bool((lo.float().abs() <= 2.0 ** -11 * hi.float().abs() + 2.0 ** -25).all())


# ------------------------------------------------------------------------------------------------ pre-processing
def test_v1_preprocess_split_rows():
    cabi, lib = _lib()
    dev = _dev()
    import unidepth_v1_parts as P1
    g = torch.Generator().manual_seed(11)
    mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    for B, (H, W) in ((2, (480, 640)), (1, (375, 1242)), (3, (231, 309))):
        rgb = torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, generator=g)
        (rh, rw), ratio = P1.v1_shapes((H, W), (462, 616))
        pads = P1.v1_paddings((rh, rw), (462, 616))
        xr, _ = P1.v1_preprocess((rgb.float() / 255 - mean) / std, None, (rh, rw), pads, ratio)
        rd = rgb.to(dev)
        for patch, rows, cols, used in ((14, B * 33 * 44, 640, 588), (4, B * 115 * 154, 64, 48)):
            ref = F.unfold(xr[..., :115 * 4, :154 * 4] if patch == 4 else xr, kernel_size=patch, stride=patch)
            ref = ref.transpose(1, 2).reshape(-1, used)
            outs = []
            for fn, width in ((lib.udb_v1_preprocess, cols), (lib.udb_v1_preprocess_split, 2 * cols)):
                p = cabi.V1Preprocess()
                p.rgb, p.rgb_is_u8, p.scale255, p.normalize, p.B, p.H, p.W = _p(rd), 1, 1, 1, B, H, W
                p.rh, p.rw, p.pad_l, p.pad_t, p.net_h, p.net_w = rh, rw, pads[0], pads[2], 462, 616
                out = torch.full((rows, width), float("nan"), device=dev, dtype=f16)
                p.patches, p.patch = _p(out), patch
                cabi.check(fn(C.byref(p), _st()), "v1_preprocess")
                outs.append(out)
            plain, sp = outs
            assert torch.equal(sp[:, :cols], plain), patch                   # hi: the f16 mode's rows, bit for bit
            assert sp[:, used:cols].abs().max().item() == 0 and sp[:, cols + used:].abs().max().item() == 0
            v = sp[:, :used].float() + sp[:, cols:cols + used].float()
            _check_lo(sp[:, :used], sp[:, cols:cols + used])
            err_hi = (plain[:, :used].float().cpu() - ref).abs().max().item()
            err = (v.cpu() - ref).abs().max().item()
            print(f"v1_preprocess_split patch {patch}, B={B} {H}x{W}: hi+lo err {err:.2e} (hi alone {err_hi:.2e})")
            # torch's f32 antialiased resize and the kernel's agree to ~1.4e-4 (measured at 2 x 480x640, patch 14): that,
            # not the split operand, bounds this comparison, so it is asserted at the hi half's own rounding level
            assert err < 1e-3
    p = cabi.V1Preprocess()
    p.patch = 7
    assert lib.udb_v1_preprocess_split(C.byref(p), _st()) != 0 and b"patch 7" in lib.udb_last_error()


# ------------------------------------------------------------------------------------------------ LayerNorm, split output
def _ln_any(cabi, lib, x, out, out_f32, w, b, rows, dim, ld_out=0, add=None, add_mod=0, s2d=(0, 0), eps=1e-6):
    p = cabi.LayerNormAny()
    p.inp = _p(x)
    p.in_f32, p.out, p.out_f32, p.weight, p.bias = int(x.dtype == f32), _p(out), out_f32, _p(w), _p(b)
    p.rows, p.dim, p.ld_in, p.ld_out, p.eps = rows, dim, dim, ld_out or dim, eps
    p.add, p.add_mod, p.s2d_h, p.s2d_w = _p(add), add_mod, s2d[0], s2d[1]
    return lib.udb_layernorm_any(C.byref(p), _st())


@pytest.mark.parametrize("dim", WIDTHS + [320, 512])
def test_layernorm_any_split_output(dim):
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(dim)
    w = (torch.randn(dim, generator=g) * 0.3 + 1).to(dev)
    b = (torch.randn(dim, generator=g) * 0.1).to(dev)
    for rows in (1, 37, 1000):
        for in_dt in (f32, f16):
            x = (torch.randn(rows, dim, generator=g) * 3 + 0.5).to(dev, in_dt)
            add = (torch.randn(7, dim, generator=g)).to(dev) if in_dt == f32 else None
            h = torch.empty(rows, dim, device=dev, dtype=f16)
            sp = torch.full((rows, 2 * dim), float("nan"), device=dev, dtype=f16)
            assert _ln_any(cabi, lib, x, h, 0, w, b, rows, dim, add=add, add_mod=7) == 0
            assert _ln_any(cabi, lib, x, sp, 2, w, b, rows, dim, 2 * dim, add=add, add_mod=7) == 0, lib.udb_last_error()
            xin = x.double() + (add.double().repeat(rows // 7 + 1, 1)[:rows] if add is not None else 0)
            ref = F.layer_norm(xin, (dim,), w.double(), b.double(), 1e-6)
            assert torch.equal(sp[:, :dim], h), (rows, in_dt)
            v = sp[:, :dim].double() + sp[:, dim:].double()
            _check_lo(sp[:, :dim], sp[:, dim:])
            # f32 statistics: the error scales with the normalised values (|y| + 1), far below hi's 2^-11 rounding
            err = ((v - ref).abs() / (ref.abs() + 1)).max().item()
            assert err < 4e-6, (rows, in_dt, err)
    # space-to-depth (k2 s2 downsample) with ragged maps: hi where the f16 call writes, lo 4*dim further right
    for B, (H, W) in ((2, (5, 7)), (1, (14, 19)), (3, (2, 2))):
        rows = B * H * W
        x = (torch.randn(rows, dim, generator=g) * 2).to(dev)
        n = B * (H // 2) * (W // 2)
        h = torch.full((n, 4 * dim), float("nan"), device=dev, dtype=f16)
        sp = torch.full((n, 8 * dim), float("nan"), device=dev, dtype=f16)
        assert _ln_any(cabi, lib, x, h, 0, w, b, rows, dim, 4 * dim, s2d=(H, W)) == 0
        assert _ln_any(cabi, lib, x, sp, 2, w, b, rows, dim, 8 * dim, s2d=(H, W)) == 0
        assert torch.equal(sp[:, :4 * dim], h)
        y = F.layer_norm(x.double(), (dim,), w.double(), b.double(), 1e-6).reshape(B, H, W, dim)[:, :H // 2 * 2, :W // 2 * 2]
        y = y.reshape(B, H // 2, 2, W // 2, 2, dim).permute(0, 1, 3, 2, 4, 5).reshape(n, 4 * dim)
        v = sp[:, :4 * dim].double() + sp[:, 4 * dim:].double()
        _check_lo(sp[:, :4 * dim], sp[:, 4 * dim:])
        assert ((v - y).abs() / (y.abs() + 1)).max().item() < 4e-6
    # the split output needs room for both halves
    x = torch.zeros(4, dim, device=dev)
    sp = torch.zeros(4, 2 * dim, device=dev, dtype=f16)
    assert _ln_any(cabi, lib, x, sp, 2, w, b, 4, dim, dim) != 0 and b"split" in lib.udb_last_error()
    assert _ln_any(cabi, lib, x, sp, 2, w, b, 4, dim, 2 * dim, s2d=(2, 2)) != 0


# ------------------------------------------------------------------------------------------------ depthwise 7x7 in f32
@pytest.mark.parametrize("Cc", WIDTHS + [32, 96])
def test_dwconv7_f32(Cc):
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(Cc)
    for B in (1, 2):
        for H, W in MAPS:
            x = (torch.randn(B, H, W, Cc, generator=g) * 2).to(dev)
            w = (torch.randn(Cc, 1, 7, 7, generator=g) / 7).to(dev)
            bias = (torch.randn(Cc, generator=g) * 0.1).to(dev)
            wt = w.reshape(Cc, 49).t().contiguous()
            y = torch.full_like(x, float("nan"))
            assert lib.udb_dwconv7_nhwc_f32(_p(x), _p(wt), _p(bias), _p(y), B, H, W, Cc, _st()) == 0, lib.udb_last_error()
            xd = x.double().permute(0, 3, 1, 2)
            ref = F.conv2d(xd, w.double(), bias.double(), padding=3, groups=Cc).permute(0, 2, 3, 1)
            terms = F.conv2d(xd.abs(), w.double().abs(), bias.double().abs(), padding=3, groups=Cc).permute(0, 2, 3, 1)
            assert bool(((y.double() - ref).abs() <= 50 * 2.0 ** -24 * terms).all()), (B, H, W)
            if Cc % 64 == 0:
                # an input that is exactly f16: the f32 sums the f16 kernel rounds, so f16 of them is its output
                x16 = x.half()
                y16 = torch.empty_like(x16)
                assert lib.udb_dwconv7_nhwc_f16(_p(x16), _p(wt), _p(bias), _p(y16), B, H, W, Cc, _st()) == 0
                assert lib.udb_dwconv7_nhwc_f32(_p(x16.float()), _p(wt), _p(bias), _p(y), B, H, W, Cc, _st()) == 0
                assert torch.equal(y.half(), y16), (B, H, W)
    x = torch.zeros(1, 4, 4, 48, device=dev)
    assert lib.udb_dwconv7_nhwc_f32(_p(x), _p(x), _p(x), _p(x), 1, 4, 4, 48, _st()) != 0
    assert lib.udb_dwconv7_nhwc_f32(_p(x), _p(x), _p(x), _p(x), 1, 0, 4, 32, _st()) != 0


# ------------------------------------------------------------------------------------------------ f32 level taps
def test_f32_level_taps():
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(7)
    for B, N, D in ((2, 33 * 44, 1024), (3, 37, 64)):
        xs = [(3.0 * torch.randn(B, 1 + N, D, generator=g)).to(dev) for _ in range(4)]
        acc = torch.full((B * N, D), float("nan"), device=dev)
        acc16 = torch.full((B * N, D), float("nan"), device=dev, dtype=f16)
        cls = torch.zeros(B, D, device=dev)
        for i, x in enumerate(xs):
            cabi.check(lib.udb_vit_tap_f32(_p(x), _p(acc), _p(cls) if i == 1 else None, B, N, D, int(i == 0), _st()), "vit_tap_f32")
            cabi.check(lib.udb_vit_tap(_p(x), _p(acc16), None, B, N, D, int(i == 0), _st()), "vit_tap")
            ref = torch.stack([(y[:, 1:] + y[:, :1]) for y in xs[:i + 1]], -1).max(-1).values.reshape(B * N, D)
            assert torch.equal(acc, ref) and torch.equal(acc.half(), acc16), (B, N, D, i)
        assert torch.equal(cls, xs[1][:, 0])
    assert lib.udb_vit_tap_f32(_p(xs[0]), _p(acc), None, B, N, 60, 1, _st()) != 0
    # ConvNeXt: running max over a stage's block outputs
    for n in (4, 1000, 192 * 115 * 154):
        xs = [torch.randn(n, generator=g).to(dev) for _ in range(3)]
        acc = torch.full((n,), float("nan"), device=dev)
        for i, x in enumerate(xs):
            cabi.check(lib.udb_max_accum_f32(_p(x), _p(acc), n, int(i == 0), _st()), "max_accum_f32")
            assert torch.equal(acc, torch.stack(xs[:i + 1]).max(0).values)
    assert lib.udb_max_accum_f32(_p(acc), _p(acc), 6, 1, _st()) != 0


# ------------------------------------------------------------------------------------------------ antialiased resize in f32
@pytest.mark.parametrize("Cc", WIDTHS)
def test_aa_resize_f32(Cc):
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(Cc + 1)
    for B, (H, W), (oh, ow) in ((2, (115, 154), (28, 38)), (1, (57, 77), (28, 38)), (2, (14, 19), (28, 38)), (1, (5, 3), (2, 7))):
        x = (torch.randn(B, H, W, Cc, generator=g) * 2).to(dev)
        y = torch.full((B, oh, ow, Cc), float("nan"), device=dev)
        cabi.check(lib.udb_aa_resize_nhwc_f32(_p(x), _p(y), B, H, W, Cc, oh, ow, _st()), "aa_resize_f32")
        ref = F.interpolate(x.double().permute(0, 3, 1, 2), size=(oh, ow), mode="bilinear", align_corners=False,
                            antialias=True).permute(0, 2, 3, 1)
        scale = x.abs().max().item()
        assert (y.double() - ref).abs().max().item() < 1e-5 * scale, (B, H, W, oh, ow)
        x16 = x.half()
        y16 = torch.empty((B, oh, ow, Cc), device=dev, dtype=f16)
        cabi.check(lib.udb_aa_resize_nhwc_f16(_p(x16), _p(y16), B, H, W, Cc, oh, ow, _st()), "aa_resize_f16")
        cabi.check(lib.udb_aa_resize_nhwc_f32(_p(x16.float()), _p(y), B, H, W, Cc, oh, ow, _st()), "aa_resize_f32")
        assert torch.equal(y.half(), y16)
    assert lib.udb_aa_resize_nhwc_f32(_p(x), _p(y), 1, 4, 4, 12, 2, 2, _st()) != 0


# ------------------------------------------------------------------------------------------------ camera cross attention on f32 kv
def test_cross_attn_small_f32():
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(3)
    for B, nq, nk, D in ((1, 4, 4 * 396 + 4, 512), (3, 4, 4 * 1040 + 4, 512), (2, 3, 17, 256), (1, 1, 5, 512)):
        q = torch.randn(B * nq, D, generator=g).to(dev)
        qp = torch.randn(nq, D, generator=g).to(dev)
        kv = (torch.randn(B * nk, 2 * D, generator=g) * 2).to(dev)
        out = torch.full((B * nq, D), float("nan"), device=dev)
        scratch = torch.empty(B * 16 * nq * (D + 2), device=dev)
        s = 1.0 / D ** 0.5
        cabi.check(lib.udb_cross_attn_small_f32(_p(q), _p(qp), _p(kv), _p(out), _p(scratch), B, nq, nk, D, s, _st()), "cross_attn_f32")
        qq = ((q.double().reshape(B, nq, D) + qp.double()) * s)
        k, v = kv.double().reshape(B, nk, 2 * D).split(D, -1)
        ref = torch.softmax(qq @ k.transpose(1, 2), -1) @ v
        err = (out.double().reshape(B, nq, D) - ref).abs().max().item()
        assert err < 2e-5 * v.abs().max().item(), (B, nq, nk, err)
        kv16 = kv.half()
        out16 = torch.empty_like(out)
        cabi.check(lib.udb_cross_attn_small(_p(q), _p(qp), _p(kv16), _p(out16), _p(scratch), B, nq, nk, D, s, _st()), "cross_attn")
        cabi.check(lib.udb_cross_attn_small_f32(_p(q), _p(qp), _p(kv16.float()), _p(out), _p(scratch), B, nq, nk, D, s, _st()), "f32")
        assert torch.equal(out, out16)
    assert lib.udb_cross_attn_small_f32(_p(q), _p(qp), _p(kv), _p(out), _p(scratch), 1, 5, 4, 512, 1.0, _st()) != 0


# ------------------------------------------------------------------------------------------------ end to end
# depth max-rel of the f16 mode MEASURED on an H100 (tests/test_v1_gpu.py V1_MEASURED, tests/test_v1_vit_gpu.py
# V1VIT_MEASURED); the depth head runs the same f16 operands in split mode, so its max-rel is asserted at 1.5x these
F16_DEPTH_MAX = {
    "v1_cnvnxtl_480x640": 9.554e-4,
    "v1_cnvnxtl_gtK_375x1242": 6.032e-4,
    "v1_vitl14_480x640": 8.829e-4,
    "v1_vitl14_gtK_375x1242": 9.351e-4,
}
CASES = sorted(F16_DEPTH_MAX)


def _model(cfg, sd, precision="split"):
    from unidepth_b200 import UniDepthV1
    m = UniDepthV1(copy.deepcopy(cfg))
    m.load_state_dict(sd, strict=True)
    m = m.to(_dev()).eval()
    m.precision = precision
    return m


@pytest.mark.parametrize("name", CASES)
def test_v1_split_meets_north_star(name):
    from test_v1_fp8_cpu import v1_case, v1_errors
    cfg, sd, rgb, K, meta, ref = v1_case(name)
    m = _model(cfg, sd)
    out = m.infer(rgb, K, skip_camera=meta["skip_camera"])
    arel, dmax, kerr = v1_errors(out, ref, meta)
    m.precision = "f16"
    a16, d16, k16 = v1_errors(m.infer(rgb, K, skip_camera=meta["skip_camera"]), ref, meta)
    print(f"V1SPLITPARITY {name}: depth ARel {arel:.3e} max {dmax:.3e}; intrinsics rel {kerr:.3e} "
          f"(f16 mode: {a16:.3e} / {d16:.3e} / {k16:.3e})")
    assert kerr < 1e-4 and arel < 1e-3, (name, arel, dmax, kerr)
    assert dmax < 1.5 * F16_DEPTH_MAX[name], (name, dmax)


def test_switching_split_to_f16_is_bit_exact():
    from test_v1_fp8_cpu import v1_case
    for name in ("v1_cnvnxtl_480x640", "v1_vitl14_480x640"):
        cfg, sd, rgb, _, _, _ = v1_case(name)
        m = _model(cfg, sd, "f16")
        rgb2 = torch.cat([rgb, rgb.flip(-1)], 0)
        for use_graph in (True, False):
            m.use_cuda_graph = use_graph
            m.precision = "f16"
            ref = m.infer(rgb2)
            m.precision = "split"
            sp = m.infer(rgb2)
            assert not torch.equal(sp["intrinsics"], ref["intrinsics"])
            m.precision = "f16"
            back = m.infer(rgb2)
            for k in ref:
                assert torch.equal(back[k], ref[k]), (name, use_graph, k)


@pytest.mark.parametrize("name", ["v1_cnvnxtl_480x640", "v1_vitl14_480x640"])
def test_v1_split_batch_and_skip_camera(name):
    from test_v1_fp8_cpu import v1_case
    cfg, sd, rgb, _, _, _ = v1_case(name)
    m = _model(cfg, sd)
    g = torch.Generator().manual_seed(9)
    batch = torch.cat([rgb, torch.randint(0, 256, (2, 3, 480, 640), dtype=torch.uint8, generator=g)], 0)
    out = m.infer(batch)
    one = m.infer(rgb)
    for k in out:
        assert torch.equal(out[k][:1], one[k]), k
    K = torch.tensor([[[520.0, 0.0, 318.0], [0.0, 515.0, 242.0], [0.0, 0.0, 1.0]]])
    got = m.infer(rgb, K.clone(), skip_camera=True)
    assert torch.allclose(got["intrinsics"].cpu(), K, rtol=1e-6, atol=1e-4)       # the caller's K comes back
    assert torch.isfinite(got["depth"]).all() and (got["depth"] > 0).all()
    assert not torch.equal(got["depth"], one["depth"])              # the decoder's rays come from the given K


@pytest.mark.parametrize("name", ["v1_cnvnxtl_480x640", "v1_vitl14_480x640"])
def test_v1_split_launch_profile(name):
    """The split schedule's kernels: fp32 attention once per ViT block, the f32 depthwise conv once per ConvNeXt block,
    the split pre-processing and the f32 cross attention once, and no e4m3 GEMM."""
    from test_v1_fp8_cpu import v1_case
    from unidepth_b200 import _cabi
    cfg, sd, rgb, _, _, _ = v1_case(name)
    m = _model(cfg, sd)
    m.use_cuda_graph = False
    m.infer(rgb)
    prof = _cabi.profile(lambda: m.infer(rgb), _st())
    count = lambda k: sum(1 for n, *_ in prof if n == k)
    s = m.spec
    assert count("gemm_e4m3_kernel") == 0
    assert count("cross_attn_partial_f32_kernel") == 1 and count("cross_attn_partial_kernel") == 0
    if name.startswith("v1_vitl14"):
        assert count("attn_split_f32_kernel") == s.enc_depth
        assert count("v1_preprocess_split_kernel<14>") == 1 and count("vit_tap_f32_kernel") == s.enc_depth
        assert count("vit_tap_kernel") == 0
    else:
        assert count("dwconv7_f32_kernel") == sum(s.depths)
        assert count("v1_preprocess_split_kernel") == 1 and count("max_accum_f32_kernel") == sum(s.depths)
        assert count("max_accum_kernel") == 0 and count("aa_resize_nhwc_f32_kernel") == 3
        # the decoder's ConvNeXt blocks keep the f16 kernel: two per ConvUpsample
        assert count("dwconv7_kernel") == 6
