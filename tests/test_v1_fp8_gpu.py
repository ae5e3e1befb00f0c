"""UniDepthV1 precision = "fp8" on the GPU: the fused ConvNeXt block head (udb_dwconv7_ln_e4m3) against a torch model of
the same steps, the row quantiser at the ConvNeXt-L widths, and UniDepthV1.infer in fp8 mode (ConvNeXt-L and ViT-L)
against the reference goldens and against the CPU rounding model of tests/test_v1_fp8_cpu.py (ConvNeXt-L: bit for bit
the f16 mode, since no stage runs e4m3).

Tolerances follow tests/test_fp8_gpu.py: what was MEASURED on an H100 for each case, asserted with a 1.5x margin,
printed as `V1FP8PARITY` lines."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
E4M3 = torch.float8_e4m3fn
MARGIN = 1.5


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _lib():
    from unidepth_b200 import _cabi
    return _cabi.lib()


# ------------------------------------------------------------------------------------------------ udb_dwconv7_ln_e4m3
MAPS = [(115, 154), (57, 77), (28, 38), (14, 19), (1, 1), (3, 5)]


def _dwconv_ln_model(x, w, b, lw, lb):
    """The steps of the kernel in torch: conv in f64 -> f16 -> LayerNorm in f64 (eps 1e-6) -> f32 -> the kernels' row
    quantiser.  The f16 conv outputs fed to the LayerNorm are those udb_dwconv7_nhwc_f16 stores, because the fused kernel
    must see exactly the f16 mode's conv outputs; they are checked here against the f64 conv rounded to f16: equal, except
    one-ulp steps where the f64 value sits on an f16 rounding boundary that the kernels' f32 accumulation lands on the
    other side of, and near-cancelling sums within the f32 accumulation's error bound.  Returns (q, s, f16 conv outputs)."""
    from test_fp8_cpu import quantize_rows
    B, H, W, Cc = x.shape
    y16 = torch.empty_like(x)
    wt = w.reshape(Cc, 49).t().contiguous()
    assert _lib().udb_dwconv7_nhwc_f16(_ptr(x), _ptr(wt), _ptr(b), _ptr(y16), B, H, W, Cc, _stream()) == 0
    y64 = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), b.double(), padding=3, groups=Cc).permute(0, 2, 3, 1)
    d = (_ordinal16(y16) - _ordinal16(y64.half())).abs()
    # more than one ulp apart only where cancellation leaves the output far below its terms: there the f32 sum's own
    # error (<= 49 * 2^-24 of sum |terms|) spans several f16 steps
    terms = F.conv2d(x.double().abs().permute(0, 3, 1, 2), w.double().abs(), b.double().abs(), padding=3, groups=Cc)
    cancel = (y16.double() - y64).abs() <= 2.0 ** -18 * terms.permute(0, 2, 3, 1)
    assert bool(((d <= 1) | cancel).all()) and (d > 0).float().mean().item() < 1e-2, (int(d.max()), (d > 0).float().mean().item())
    y = F.layer_norm(y16.double(), (Cc,), lw.double(), lb.double(), 1e-6).float().reshape(-1, Cc)
    q, s = quantize_rows(y)
    return q, s.reshape(-1), y16


def _ordinal16(h):
    """f16 values on a signed integer scale on which neighbouring values differ by one (+0 and -0 are both 0)."""
    u = h.view(torch.int16).int() & 0xFFFF
    mag = u & 0x7FFF
    return torch.where(u >= 0x8000, -mag, mag)


def _ordinal(q):
    """e4m3 codes on a signed integer scale on which neighbouring values differ by one (+0 and -0 are both 0)."""
    u = q.view(torch.uint8).int()
    mag = u & 0x7F
    return torch.where(u >= 0x80, -mag, mag)


# the four ConvNeXt widths (every cluster block owns 3 channel chunks) and widths whose chunks do not split evenly:
# 64 / 128 (one block, 1-2 chunks), 320 (blocks own 3 and 2), 1472 (eight blocks, 3 or 2 chunks)
@pytest.mark.parametrize("Cc", [64, 128, 192, 320, 384, 768, 1472, 1536])
def test_dwconv7_ln_e4m3_against_torch_model(Cc):
    dev = _dev()
    lib = _lib()
    g = torch.Generator().manual_seed(Cc)
    worst = (0, 0.0)
    for B in (1, 3):
        for H, W in MAPS:
            x = (torch.randn(B, H, W, Cc, generator=g) * 2).half().to(dev)
            w = (torch.randn(Cc, 1, 7, 7, generator=g) / 7).to(dev)
            b = (torch.randn(Cc, generator=g) * 0.1).to(dev)
            lw = (torch.randn(Cc, generator=g) * 0.2 + 1).to(dev)
            lb = (torch.randn(Cc, generator=g) * 0.1).to(dev)
            rows = B * H * W
            q = torch.empty((rows, Cc), dtype=E4M3, device=dev)
            s = torch.empty(rows, device=dev)
            wt = w.reshape(Cc, 49).t().contiguous()
            rc = lib.udb_dwconv7_ln_e4m3(_ptr(x), _ptr(wt), _ptr(b), _ptr(lw), _ptr(lb), _ptr(q), _ptr(s), B, H, W, Cc, _stream())
            assert rc == 0, lib.udb_last_error().decode()
            q_ref, s_ref, _ = _dwconv_ln_model(x, w, b, lw, lb)
            # scales agree to the f32 rounding of the kernel's statistics
            srel = ((s - s_ref).abs() / s_ref).max().item()
            assert srel < 1e-5, (B, H, W, srel)
            # codes: identical except one-code steps where x * 448 / amax sits on an e4m3 rounding boundary (+-1 and 0
            # around zero count as neighbours)
            d = (_ordinal(q) - _ordinal(q_ref)).abs()
            near_zero = (_ordinal(q).abs() <= 1) & (_ordinal(q_ref).abs() <= 1)
            assert int(((d > 1) & ~near_zero).sum()) == 0, (B, H, W, Cc)
            frac = (d > 0).float().mean().item()
            worst = max(worst, (frac, srel))
            assert frac < 1e-3, (B, H, W, Cc, frac)
    print(f"DWCONVLN C={Cc}: worst share of one-code differences {worst[0]:.2e}, scale rel err {worst[1]:.2e}")


def test_dwconv7_ln_e4m3_rejects_bad_arguments():
    dev = _dev()
    lib = _lib()
    B, H, W, Cc = 1, 4, 5, 128
    x = torch.zeros((B, H, W, 1600), dtype=torch.float16, device=dev)
    w = torch.zeros((49, 1600), device=dev)
    v = torch.zeros(1600 + 8, device=dev)
    q = torch.empty((B * H * W, 1600 + 16), dtype=torch.uint8, device=dev)
    s = torch.empty(64, device=dev)

    def call(**kw):
        a = dict(x=_ptr(x), w=_ptr(w), bias=_ptr(v), ln_w=_ptr(v), ln_b=_ptr(v), out=_ptr(q), out_scale=_ptr(s), B=B, H=H, W=W, C=Cc)
        a.update(kw)
        rc = lib.udb_dwconv7_ln_e4m3(a["x"], a["w"], a["bias"], a["ln_w"], a["ln_b"], a["out"], a["out_scale"], a["B"], a["H"], a["W"],
                                     a["C"], _stream())
        return rc, lib.udb_last_error().decode()
    assert call()[0] == 0
    bad = [({"C": 100}, "C="), ({"C": 1600}, "C="), ({"C": 0}, "C="), ({"B": 0}, "B="), ({"H": 0}, "H="), ({"W": -1}, "W=")]
    for name, t in (("x", x), ("w", w), ("bias", v), ("ln_w", v), ("ln_b", v), ("out", q), ("out_scale", s)):
        bad.append(({name: C.c_void_p(t.data_ptr() + 4)}, f"`{name}`"))
        bad.append(({name: None}, f"`{name}`"))
    for kw, frag in bad:
        rc, msg = call(**kw)
        assert rc != 0 and frag in msg, (kw, msg)
    torch.cuda.synchronize()


@pytest.mark.parametrize("rows,cols", [(37, 4608), (300, 6144)])
def test_row_quantiser_at_convnext_widths(rows, cols):
    dev = _dev()
    lib = _lib()
    from test_fp8_cpu import quantize_rows
    g = torch.Generator().manual_seed(rows + cols)
    x = (torch.randn(rows, cols, generator=g) * torch.logspace(-3, 2, rows)[:, None]).half()
    x[rows // 2] = 0.0
    xd = x.to(dev)
    q = torch.empty((rows, cols), dtype=E4M3, device=dev)
    s = torch.empty(rows, device=dev)
    rc = lib.udb_quantize_rows_e4m3(_ptr(xd), cols, _ptr(q), cols, _ptr(s), rows, cols, _stream())
    assert rc == 0, lib.udb_last_error().decode()
    q_ref, s_ref = quantize_rows(x.float())
    assert torch.equal(s.cpu(), s_ref.reshape(-1))
    assert torch.equal(q.cpu().view(torch.uint8), q_ref.view(torch.uint8))
    wide = torch.empty((rows, 6152), dtype=torch.float16, device=dev)
    q2 = torch.empty((rows, 6152), dtype=torch.uint8, device=dev)
    assert lib.udb_quantize_rows_e4m3(_ptr(wide), 6152, _ptr(q2), 6152, _ptr(s), rows, 6152, _stream()) != 0
    assert "6144" in lib.udb_last_error().decode()


# ------------------------------------------------------------------------------------------------ end to end
# tag -> (depth ARel, depth max rel, intrinsics max rel) MEASURED on an H100 80GB HBM3 (700 W) in fp8 mode; asserted x1.5
MEASURED = {
    "golden_v1_vitl14_480x640": (7.145e-03, 3.677e-02, 1.585e-02),
    "golden_v1_vitl14_gtK_375x1242": (3.776e-03, 1.637e-02, 2.671e-02),
    "skip_camera_v1_vitl14_480x640": (4.168e-03, 2.135e-02, 1e-6),     # the caller's K comes back: 0 measured
}
CASES = ["v1_cnvnxtl_480x640", "v1_cnvnxtl_gtK_375x1242", "v1_vitl14_480x640", "v1_vitl14_gtK_375x1242"]


def _model(cfg, sd, precision="fp8"):
    import copy
    from unidepth_b200 import UniDepthV1
    m = UniDepthV1(copy.deepcopy(cfg))
    m.load_state_dict(sd, strict=True)
    m = m.to(_dev()).eval()
    m.precision = precision
    return m


def _check(tag, errs):
    arel, dmax, kerr = errs
    print(f"V1FP8PARITY {tag}: depth ARel {arel:.3e} max {dmax:.3e}; intrinsics rel {kerr:.3e}")
    m = MEASURED[tag]
    assert arel < MARGIN * m[0] and dmax < MARGIN * m[1] and kerr < MARGIN * m[2], (tag, errs, m)


@pytest.mark.parametrize("name", CASES)
def test_v1_fp8_infer_against_golden(name):
    from test_v1_fp8_cpu import V1_FP8_MODEL_ERROR, v1_case, v1_errors
    from unidepth_b200 import _cabi
    cfg, sd, rgb, K, meta, ref = v1_case(name)
    m = _model(cfg, sd)
    out = m.infer(rgb, K, skip_camera=meta["skip_camera"])
    if name.startswith("v1_cnvnxtl"):
        # no ConvNeXt stage runs e4m3 (FP8_STAGES): the fp8 mode computes exactly what the f16 mode does
        m.precision = "f16"
        f16 = m.infer(rgb, K, skip_camera=meta["skip_camera"])
        assert all(torch.equal(out[k], f16[k]) for k in out)
        m.precision = "fp8"
    else:
        _check("golden_" + name, v1_errors(out, ref, meta))
    errs = v1_errors(out, ref, meta)
    # the encoder's GEMMs run on e4m3 operands: 2 per ConvNeXt block of an fp8 stage, 4 per ViT block
    m.use_cuda_graph = False
    prof = _cabi.profile(lambda: m.infer(rgb, K, skip_camera=meta["skip_camera"]), _stream())
    from unidepth_b200.unidepthv1 import FP8_STAGES
    s = m.spec
    n8 = 4 * s.enc_depth if name.startswith("v1_vitl14") else 2 * sum(d for d, f in zip(s.depths, FP8_STAGES) if f)
    assert sum(1 for k, *_ in prof if k == "gemm_e4m3_kernel") == n8
    if name.startswith("v1_cnvnxtl"):
        assert sum(1 for k, *_ in prof if k == "dwconv7_ln_e4m3_kernel") == n8 // 2
    # consistent with the CPU rounding model: the same size of error as the model shows against the same goldens
    if name in V1_FP8_MODEL_ERROR:
        model = V1_FP8_MODEL_ERROR[name]
        assert 1 / 3 < errs[0] / model[0] < 3, (errs, model)


def test_v1_fp8_batch_float_input_and_skip_camera():
    import copy
    import unidepth_v1_vit_oracle as OV
    from test_v1_fp8_cpu import v1_case
    cfg, sd, rgb, _, meta, _ = v1_case("v1_vitl14_480x640")
    m = _model(cfg, sd)
    g = torch.Generator().manual_seed(9)
    batch = torch.cat([rgb, torch.randint(0, 256, (2, 3, 480, 640), dtype=torch.uint8, generator=g)], 0)
    out = m.infer(batch)
    one = m.infer(rgb)
    assert torch.equal(out["depth"][:1], one["depth"]) and torch.equal(out["intrinsics"][:1], one["intrinsics"])
    fl = m.infer(rgb.float() / 255.0)
    assert (fl["depth"] - one["depth"]).abs().max().item() < 2e-3 * one["depth"].max().item()
    K = torch.tensor([[[520.0, 0.0, 318.0], [0.0, 515.0, 242.0], [0.0, 0.0, 1.0]]])
    ref = OV.infer_v1_vit(sd, copy.deepcopy(cfg), rgb, K.clone(), skip_camera=True)
    got = m.infer(rgb.float() / 255.0, K.clone(), skip_camera=True)
    from test_v1_fp8_cpu import v1_errors
    _check("skip_camera_v1_vitl14_480x640", v1_errors(got, ref, {}))


def test_switching_precision_restores_f16():
    from test_v1_fp8_cpu import v1_case
    cfg, sd, rgb, _, _, _ = v1_case("v1_vitl14_480x640")
    m = _model(cfg, sd, "f16")
    rgb2 = torch.cat([rgb, rgb.flip(-1)], 0)
    for use_graph in (True, False):
        m.use_cuda_graph = use_graph
        m.precision = "f16"
        f16 = m.infer(rgb2)
        m.precision = "fp8"
        f8 = m.infer(rgb2)
        assert not torch.equal(f8["depth"], f16["depth"])
        m.precision = "f16"
        back = m.infer(rgb2)
        for k in f16:
            assert torch.equal(back[k], f16[k]), (use_graph, k)
