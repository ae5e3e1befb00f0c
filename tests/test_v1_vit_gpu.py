"""UniDepthV1 with the DINOv2 ViT-L/14 encoder (config_v1_vitl14.json) on the GPU: the two kernels this path adds (14x14
patch rows from the V1 pre-processing, the block-output tap) against PyTorch, and the whole `infer` (udb_infer_v1) against
outputs of the unmodified reference (tests/golden/v1_vitl14_*.npz, oracle/make_golden_v1_vit.py) and against the oracle."""
import copy
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
f16, f32 = torch.float16, torch.float32


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


def _preprocess(cabi, lib, rd, H, W, rh, rw, pads, patch, out):
    p = cabi.V1Preprocess()
    p.rgb, p.rgb_is_u8, p.scale255, p.normalize, p.B, p.H, p.W = _p(rd), 1, 1, 1, rd.shape[0], H, W
    p.rh, p.rw, p.pad_l, p.pad_t, p.net_h, p.net_w, p.patches = rh, rw, pads[0], pads[2], 462, 616, _p(out)
    p.patch = patch
    cabi.check(lib.udb_v1_preprocess(C.byref(p), _st()), f"v1_preprocess(patch={patch})")


def test_v1_preprocess_14x14_patch_rows():
    """V1 pre-processing into the DINOv2 patch-embedding rows vs torch: antialiased resize + zero pad (the oracle's
    v1_preprocess, itself pinned to the reference), then unfold 14x14 -> columns c*196 + py*14 + px, 588..639 zero."""
    cabi, lib = _lib()
    dev = _dev()
    import unidepth_v1_parts as P1
    g = torch.Generator().manual_seed(3)
    mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    for B, (H, W) in ((2, (480, 640)), (3, (375, 1242)), (2, (1001, 399)), (3, (231, 309))):
        rgb = torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, generator=g)
        (rh, rw), ratio = P1.v1_shapes((H, W), (462, 616))
        pads = P1.v1_paddings((rh, rw), (462, 616))
        xr, _ = P1.v1_preprocess((rgb.float() / 255 - mean) / std, None, (rh, rw), pads, ratio)
        ref = F.unfold(xr, kernel_size=14, stride=14).transpose(1, 2).reshape(-1, 588)
        rd = rgb.to(dev)
        patches = torch.full((B * 33 * 44, 640), float("nan"), device=dev, dtype=f16)
        _preprocess(cabi, lib, rd, H, W, rh, rw, pads, 14, patches)
        torch.cuda.synchronize()
        err = (patches[:, :588].float().cpu() - ref).abs().max().item()
        print(f"v1_preprocess patch 14, B={B} {H}x{W}: max abs err {err:.2e}")
        assert err < 3e-3 and patches[:, 588:].abs().max().item() == 0
        # the ConvNeXt stem layout: patch 0 and patch 4 are the same call, byte for byte
        p0 = torch.empty(B * 115 * 154, 64, device=dev, dtype=f16)
        p4 = torch.empty_like(p0)
        _preprocess(cabi, lib, rd, H, W, rh, rw, pads, 0, p0)
        _preprocess(cabi, lib, rd, H, W, rh, rw, pads, 4, p4)
        assert torch.equal(p0, p4)
    p = cabi.V1Preprocess()
    p.patch = 7
    assert lib.udb_v1_preprocess(C.byref(p), _st()) != 0 and b"patch 7" in lib.udb_last_error()


def test_vit_tap_kernel_is_bit_equal_to_f16_of_the_f32_max():
    """acc = f16(max over a slice of blocks of (patch tokens + cls token)), first block a plain store; raw cls capture."""
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(5)
    for B, N, D in ((2, 33 * 44, 1024), (3, 37, 64)):
        xs = [(3.0 * torch.randn(B, 1 + N, D, generator=g)).to(dev) for _ in range(4)]
        acc = torch.full((B * N, D), float("nan"), device=dev, dtype=f16)
        cls = torch.zeros(B, D, device=dev)
        for i, x in enumerate(xs):
            cabi.check(lib.udb_vit_tap(_p(x), _p(acc), _p(cls) if i == 2 else None, B, N, D, int(i == 0), _st()), "vit_tap")
            ref = torch.stack([(y[:, 1:] + y[:, :1]) for y in xs[:i + 1]], -1).max(-1).values.half().reshape(B * N, D)
            assert torch.equal(acc, ref), (B, N, D, i)
        assert torch.equal(cls, xs[2][:, 0])             # only the call that passed cls_out wrote it
    assert lib.udb_vit_tap(_p(xs[0]), _p(acc), None, B, N, 60, 1, _st()) != 0   # D % 8


def _model(cfg, sd):
    from unidepth_b200 import UniDepthV1
    m = UniDepthV1(copy.deepcopy(cfg))
    m.load_state_dict(sd, strict=True)
    return m.to("cuda:0").eval()


# measured on an H100 80GB HBM3 (700 W power limit; the tests print them as V1VITPARITY lines), asserted with a 1.5x margin:
# (depth ARel, depth max-rel, K rel).  Hard ceiling on the depth ARel whatever the table says: 1e-3.  The GT-K case's
# intrinsics (2.0e-4) exceed V2's 1e-4 bar: f16 operand rounding in the encoder alone reproduces it on the CPU
# (tests/test_v1_vit_numerics_cpu.py).
V1VIT_MEASURED = {
    "golden_v1_vitl14_480x640": (2.459e-4, 8.829e-4, 8.365e-5),
    "golden_v1_vitl14_gtK_375x1242": (3.532e-4, 9.351e-4, 1.988e-4),
    "skip_camera_480x640": (2.083e-4, 9.175e-4, 1e-6),
}


def _check(out, ref_depth, ref_K, ref_pts, tag, depth_stride=1, pts_stride=1, label=None):
    d, dr = out["depth"].float().cpu()[:, :, ::depth_stride, ::depth_stride], ref_depth
    rel = (d - dr).abs() / dr
    k, kr = out["intrinsics"].cpu(), ref_K
    kerr = max(((k[:, i, j] - kr[:, i, j]).abs() / kr[:, i, j].abs()).max().item() for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)))
    pts = out["points"].float().cpu()[:, :, ::pts_stride, ::pts_stride]
    perr = ((pts - ref_pts).abs() / ref_pts.abs().clamp(min=0.1 * ref_pts.abs().mean())).mean().item()
    print(f"V1VITPARITY {label or tag}: depth ARel {rel.mean().item():.3e} max {rel.max().item():.3e}; intrinsics rel {kerr:.3e}; "
          f"points mean rel {perr:.3e}")
    m = V1VIT_MEASURED[tag]
    assert rel.mean().item() < 1e-3
    assert rel.mean().item() < 1.5 * m[0] and rel.max().item() < 1.5 * m[1] and kerr < 1.5 * m[2], (tag, rel.mean().item(), rel.max().item(), kerr)
    assert perr < 5e-3


@pytest.mark.parametrize("name", ["v1_vitl14_480x640", "v1_vitl14_gtK_375x1242"])
def test_v1_vit_infer_against_reference_golden(name, golden_dir):
    _dev()
    import unidepth_v1_vit_oracle as OV
    from test_v1_vit_cpu import v1_vit_case_inputs
    cfg, sd, rgb, K, meta, z = v1_vit_case_inputs(golden_dir, name)
    m = _model(cfg, sd)
    out = m.infer(rgb, K, skip_camera=meta["skip_camera"])
    assert set(out) == {"intrinsics", "points", "depth"}
    # the reference's outputs, stored sub-sampled (oracle/make_golden_v1_vit.py) ...
    _check(out, torch.from_numpy(z["depth"]), torch.from_numpy(z["intrinsics"]), torch.from_numpy(z["points"]), "golden_" + name,
           meta["strides"]["depth"], meta["strides"]["points"])
    # ... and every pixel against the fp32 oracle, which those files pin to 5e-5 (tests/test_v1_vit_cpu.py): same bars
    ref = OV.infer_v1_vit(sd, copy.deepcopy(cfg), rgb, K, skip_camera=meta["skip_camera"])
    _check(out, ref["depth"], ref["intrinsics"], ref["points"], "golden_" + name, label="full_resolution_oracle_" + name)
    # graph replay and eager agree bit for bit
    again = m.infer(rgb, K, skip_camera=meta["skip_camera"])
    assert all(torch.equal(again[k], out[k]) for k in out)
    m.use_cuda_graph = False
    eager = m.infer(rgb, K, skip_camera=meta["skip_camera"])
    assert all(torch.equal(eager[k], out[k]) for k in out)


def test_v1_vit_batch_float_input_and_skip_camera(golden_dir):
    _dev()
    import unidepth_v1_vit_oracle as OV
    from test_v1_vit_cpu import v1_vit_case_inputs
    cfg, sd, rgb, _, meta, z = v1_vit_case_inputs(golden_dir, "v1_vitl14_480x640")
    m = _model(cfg, sd)
    g = torch.Generator().manual_seed(9)
    others = torch.randint(0, 256, (2, 3, 480, 640), dtype=torch.uint8, generator=g)
    batch = torch.cat([rgb, others], 0)
    out = m.infer(batch)
    for i in range(3):            # each image of a batch of 3 gets its single-image result, bit for bit
        one = m.infer(batch[i:i + 1])
        assert all(torch.equal(out[k][i:i + 1], one[k]) for k in out), i
    one = m.infer(rgb)
    # float input in [0, 1] takes the same path as uint8 (unidepthv1.py:301-308)
    fl = m.infer(rgb.float() / 255.0)
    assert (fl["depth"] - one["depth"]).abs().max().item() < 2e-3 * one["depth"].max().item()
    # skip_camera with GT intrinsics: the GT K comes back, rays / points use it
    K = torch.tensor([[[520.0, 0.0, 318.0], [0.0, 515.0, 242.0], [0.0, 0.0, 1.0]]])
    ref = OV.infer_v1_vit(sd, copy.deepcopy(cfg), rgb, K.clone(), skip_camera=True)
    got = m.infer(rgb, K.clone(), skip_camera=True)
    _check(got, ref["depth"], ref["intrinsics"], ref["points"], "skip_camera_480x640")
