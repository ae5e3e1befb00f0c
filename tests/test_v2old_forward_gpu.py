"""UniDepthV2old.forward on the GPU: the antialiased depth path of the output assembly against float64 torch, the patch rows
of a network-shaped input, and the whole network-only call (udb_infer_v2old, network_only = 1) against outputs of the
unmodified reference's `forward` (tests/golden/v2oldfwd_*.npz, oracle/make_golden_v2old_forward.py)."""
import ctypes as C
import glob
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
f16, f32, f64 = torch.float16, torch.float32, torch.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
FWD_GOLDENS = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "v2oldfwd_*.npz")))
IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)

# Parity bars of `forward` (f16 mode) against the reference's fp32 outputs on the seeded fixture, per backbone: depth ARel,
# depth max relative error, K max relative error, confidence max absolute error, depth_features max absolute error over
# the largest magnitude, points max absolute error over z.  Each is 1.5 times the largest value measured on an H100
# (80 GB HBM3, 700 W power limit) over the backbone's five goldens (V2OLDFWDPARITY lines; largest: ViT-L 3.18e-3 /
# 3.55e-2 / 4.04e-4 / 1.07e-3 / 8.53e-4 / 2.43e-2, ViT-S 1.91e-3 / 1.26e-2 / 2.13e-4 / 7.73e-4 / 9.07e-4 / 1.81e-2).  These
# are `infer`'s orders (tests/test_v2old_gpu.py); the points' x and y errors are the depth's times |tan theta|, up to 2
# at the borders of the wider ground truths, hence their bar above the depth's.
BARS = {"vitl14": (4.8e-3, 5.3e-2, 6.1e-4, 1.6e-3, 1.3e-3, 3.6e-2), "vits14": (2.9e-3, 1.9e-2, 3.2e-4, 1.2e-3, 1.4e-3, 2.7e-2)}


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


# ------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("B,net,HW", [(1, (588, 784), (240, 320)), (2, (294, 392), (480, 640)), (1, (70, 56), (211, 133)),
                                      (2, (294, 392), (294, 392))])
def test_postprocess_antialiased_depth_matches_float64(B, net, HW):
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(HW[0] + B)
    depth = 1 + torch.rand(B, 1, *net, generator=g)
    conf = torch.rand(B, 1, *net, generator=g)
    k4 = torch.stack([300 + 50 * torch.rand(B, generator=g), 310 + 50 * torch.rand(B, generator=g),
                      HW[1] / 2 + 10 * torch.rand(B, generator=g), HW[0] / 2 + 10 * torch.rand(B, generator=g)], 1)
    ref_d = F.interpolate(depth.double(), size=HW, mode="bilinear", align_corners=False, antialias=True)
    ref_c = F.interpolate(conf.double(), size=HW, mode="bilinear", align_corners=False, antialias=True)
    ys, xs = torch.meshgrid(torch.arange(HW[0], dtype=f64) + 0.5, torch.arange(HW[1], dtype=f64) + 0.5, indexing="ij")
    pts = []
    for b in range(B):
        fx, fy, cx, cy = k4[b].double()
        r = torch.stack([(xs - cx) / fx, (ys - cy) / fy, torch.ones_like(xs)], 0)
        r = r / r.norm(dim=0, keepdim=True)
        th, ph = torch.atan2(r[0], r[2]), torch.acos(r[1])
        z = ref_d[b, 0]
        pts.append(torch.stack([z * torch.tan(th), z / torch.tan(ph) / torch.cos(th), z]))
    ref_p = torch.stack(pts)
    dd, cd, kd = depth.to(dev), conf.to(dev), k4.contiguous().to(dev)
    od, oc, op = (torch.full((B, n, *HW), float("nan"), device=dev) for n in (1, 1, 3))
    p = cabi.V2oldPostprocess()
    p.depth, p.confidence, p.k4, p.B, p.net_h, p.net_w, p.H, p.W = _p(dd), _p(cd), _p(kd), B, net[0], net[1], HW[0], HW[1]
    p.mode, p.depth_aa = 2, 1                     # `mode` is not read on the antialiased path
    p.out_depth, p.out_confidence, p.out_points = _p(od), _p(oc), _p(op)
    cabi.check(lib.udb_v2old_postprocess(C.byref(p), _st()), "postprocess")
    torch.cuda.synchronize()
    # antialiased weights from f32 tap positions (aa_axis): a few e-5 relative
    assert ((od.double().cpu() - ref_d).abs() / ref_d).max().item() < 1e-4
    assert (oc.double().cpu() - ref_c).abs().max().item() < 2e-4
    assert ((op.double().cpu() - ref_p).abs() / ref_d.abs()).max().item() < 1e-4
    if tuple(net) == tuple(HW):
        # weights (1, 0) at equal sizes: the depth and the confidence are copied bit for bit
        assert torch.equal(od, dd) and torch.equal(oc, cd)
    p.depth_aa = 2
    assert lib.udb_v2old_postprocess(C.byref(p), _st()) != 0 and b"`depth_aa` 2" in lib.udb_last_error()


@pytest.mark.parametrize("split", [False, True])
def test_preprocess_of_a_network_shaped_input_is_the_f16_rounding(split):
    """At equal input and output sizes the antialiased resize has weights (1, 0): the patch rows of an f32 input with
    neither /255 nor normalisation are the f16 rounding of the input (split: hi = f16(v), lo = f16(v - hi)), bit for bit."""
    cabi, lib = _lib()
    dev = _dev()
    B, h, w = 2, 294, 392
    g = torch.Generator().manual_seed(3)
    x = (2.5 * torch.randn(B, 3, h, w, generator=g)).to(dev)
    gh, gw = h // 14, w // 14
    cols = x.reshape(B, 3, gh, 14, gw, 14).permute(0, 2, 4, 1, 3, 5).reshape(B * gh * gw, 588)
    out = torch.full((B * gh * gw, 640 * (2 if split else 1)), float("nan"), device=dev, dtype=f16)
    p = cabi.V1Preprocess()
    p.rgb, p.rgb_is_u8, p.scale255, p.normalize, p.B, p.H, p.W = _p(x), 0, 0, 0, B, h, w
    p.rh, p.rw, p.net_h, p.net_w, p.patch, p.patches = h, w, h, w, 14, _p(out)
    cabi.check((lib.udb_v1_preprocess_split if split else lib.udb_v1_preprocess)(C.byref(p), _st()), "preprocess")
    torch.cuda.synchronize()
    hi = cols.to(f16)
    assert torch.equal(out[:, :588], hi) and out[:, 588:640].abs().max().item() == 0
    if split:
        assert torch.equal(out[:, 640:1228], (cols - hi.float()).to(f16))


# ------------------------------------------------------------------------------------------ end to end
def _model(bb, seed, dev):
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    from make_golden_v2old import make_v2old_state_dict
    from unidepth_b200 import UniDepthV2old
    cfg = json.load(open(os.path.join(GOLDEN, f"config_v2old_{bb}.json")))
    m = UniDepthV2old(cfg)
    m.load_state_dict(make_v2old_state_dict(cfg, seed), strict=True)
    return m.to(dev).eval()


def _network_input(shape, seed):
    """The generator's input: ImageNet normalisation (/255, then (x - mean) / std in f32, as torchvision's normalize) of
    the seeded uint8 image."""
    g = torch.Generator().manual_seed(4321 + seed)
    b, h, w = shape
    rgb = torch.randint(0, 256, (b, 3, h, w), dtype=torch.uint8, generator=g)
    mean = torch.tensor(IMAGENET_MEAN, dtype=f32).view(1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD, dtype=f32).view(1, 3, 1, 1)
    return rgb.to(f32).div(255).sub(mean).div(std)


def _golden_case(name, dev):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["__meta__"]))
    x = _network_input(tuple(meta["shape"]), meta["seed"])
    s = meta["image_stride"]
    assert np.array_equal(x[:, :, ::s, ::s].numpy(), z["image_sample"]), "the network input differs from the generator's"
    inputs = {"image": x.to(dev), "depth": torch.zeros(meta["shape"][0], 1, *meta["gt_hw"], device=dev)}
    if meta["with_k"]:
        inputs["K"] = torch.from_numpy(z["K_in"]).to(dev)
    return z, meta, inputs


def _errors(out, z, meta):
    st = meta["strides"]
    d = out["depth"][:, :, ::st["depth"], ::st["depth"]].double().cpu().numpy()
    dr = z["depth"].astype(np.float64)
    arel, mrel = float(np.mean(np.abs(d - dr) / dr)), float(np.max(np.abs(d - dr) / dr))
    kr = z["K"].astype(np.float64)
    krel = float(np.max(np.abs(out["K"].double().cpu().numpy() - kr) / np.maximum(np.abs(kr), 1.0)))
    c = out["confidence"][:, :, ::st["confidence"], ::st["confidence"]].double().cpu().numpy()
    cerr = float(np.max(np.abs(c - z["confidence"])))
    p = out["points"][:, :, ::st["points"], ::st["points"]].double().cpu().numpy()
    pz = z["points"].astype(np.float64)
    prel = float(np.max(np.abs(p - pz) / pz[:, 2:3]))
    f = out["depth_features"][:, z["feat_idx"], ::meta["feat_ch_stride"]].double().cpu().numpy()
    fr = z["depth_features"].astype(np.float64)
    ferr = float(np.max(np.abs(f - fr)) / np.max(np.abs(fr)))
    return arel, mrel, krel, cerr, prel, ferr


@pytest.mark.parametrize("name", FWD_GOLDENS)
def test_forward_matches_reference_golden(name):
    dev = _dev()
    z, meta, inputs = _golden_case(name, dev)
    bb = meta["config"][len("config_v2old_"):-len(".json")]
    m = _model(bb, meta["seed"], dev)
    keys = {k: v.data_ptr() for k, v in inputs.items()}
    out = m(inputs, None)
    assert {k: v.data_ptr() for k, v in inputs.items()} == keys, "forward must not mutate the caller's inputs"
    B, (H, W) = meta["shape"][0], meta["gt_hw"]
    n = (meta["shape"][1] // 14) * (meta["shape"][2] // 14)
    assert out["depth"].shape == out["confidence"].shape == (B, 1, H, W) and out["points"].shape == (B, 3, H, W)
    assert out["K"].shape == (B, 3, 3) and out["depth_features"].shape == (B, n, 512)
    arel, mrel, krel, cerr, prel, ferr = _errors(out, z, meta)
    print(f"V2OLDFWDPARITY {name}: depth ARel {arel:.3e} max-rel {mrel:.3e} K max-rel {krel:.3e} confidence max-abs "
          f"{cerr:.3e} points max-rel {prel:.3e} depth_features max-abs/max {ferr:.3e}")
    bar_arel, bar_mrel, bar_k, bar_c, bar_f, bar_p = BARS[bb]
    assert arel < bar_arel and mrel < bar_mrel and krel < bar_k and cerr < bar_c and ferr < bar_f and prel < bar_p


def test_forward_graph_replay_equals_eager_and_keeps_out_of_infer():
    dev = _dev()
    z, meta, inputs = _golden_case("v2oldfwd_vits14_portraitK_560x420", dev)
    m = _model("vits14", meta["seed"], dev)
    m.output_buffers = {k: torch.zeros(1, device=dev) for k in ("intrinsics", "points", "depth", "confidence")}
    g1 = m(inputs, None)
    g2 = m(inputs, None)
    assert any(k[0] == "forward" for k in m._graphs) and all(v.numel() == 1 and v.item() == 0 for v in m.output_buffers.values())
    m.use_cuda_graph = False
    e = m(inputs, None)
    assert set(g1) == {"K", "depth", "confidence", "points", "depth_features"}
    for k in g1:
        assert g1[k].data_ptr() != g2[k].data_ptr()
        assert torch.equal(g1[k], g2[k]) and torch.equal(g1[k], e[k]), k


def test_forward_batch_slices_equal_single_image_runs():
    dev = _dev()
    for bb in ("vits14", "vitl14"):
        z, meta, inputs = _golden_case(f"v2oldfwd_{bb}_K2_294x392", dev)
        m = _model(bb, meta["seed"], dev)
        both = m(inputs, None)
        for b in range(2):
            one = m({k: v[b:b + 1] for k, v in inputs.items()}, None)
            for k in both:
                assert torch.equal(both[k][b:b + 1], one[k]), (bb, b, k)


@pytest.mark.parametrize("precision", ["split", "fp8"])
def test_forward_precision_modes(precision):
    from unidepth_b200 import _cabi
    dev = _dev()
    name = "v2oldfwd_vits14_eq_420x560"
    z, meta, inputs = _golden_case(name, dev)
    m = _model("vits14", meta["seed"], dev)
    f16_out = m(inputs, None)
    m.precision = precision
    n0 = _cabi.launch_count()
    out = m(inputs, None)
    torch.cuda.synchronize()
    assert _cabi.launch_count() > n0
    assert all(torch.isfinite(v).all() for v in out.values())
    assert not torch.equal(out["depth"], f16_out["depth"])
    arel, mrel, krel, cerr, prel, ferr = _errors(out, z, meta)
    print(f"V2OLDFWDPARITY {name} precision={precision}: depth ARel {arel:.3e} max-rel {mrel:.3e} K max-rel {krel:.3e} "
          f"confidence max-abs {cerr:.3e} depth_features max-abs/max {ferr:.3e}")
    if precision == "split":
        # split operands on the path to the intrinsics: the K error drops to V1's split order (DESIGN.md section 8)
        assert krel < 1e-4 and arel < BARS["vits14"][0]
    else:
        # e4m3 operands in the encoder: a coarse check only (DESIGN.md section 8 explains the size of the fp8 error)
        assert arel < 0.5
