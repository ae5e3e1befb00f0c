"""UniDepthV2old on the GPU: the kernels its decoder adds (pixel-shuffle depthwise conv, the ray Fourier features with the
ray appended, the depth / confidence convolutions over the resized levels, the depth tail, the output assembly, the
camera) against float64 torch references, and the whole `infer` (udb_infer_v2old) against outputs of the unmodified
reference (tests/golden/v2old_*.npz, oracle/make_golden_v2old.py)."""
import ctypes as C
import glob
import json
import math
import os
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
f16, f32, f64 = torch.float16, torch.float32, torch.float64
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")

# Parity bars of the f16 path against the reference's fp32 outputs on the seeded fixture, per backbone: depth ARel,
# depth max relative error, intrinsics max relative error, confidence max absolute error.  Each is 1.5 times the largest
# value measured on an H100 (80 GB HBM3) over the six goldens of the backbone (largest: ViT-L 2.54e-3 / 1.91e-2 /
# 2.46e-4 / 1.18e-3, ViT-S 2.29e-3 / 1.78e-2 / 2.90e-4 / 1.70e-3).  The depth bars are about ten times UniDepthV1's
# (DESIGN.md section 8): the intrinsics, whose path has no map-wide step, stay at V1's order.
BARS = {"vitl14": (3.8e-3, 2.9e-2, 3.7e-4, 1.8e-3), "vits14": (3.4e-3, 2.7e-2, 4.4e-4, 2.6e-3)}


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
@pytest.mark.parametrize("B,h,w,C,ldo", [(1, 7, 9, 512, 128), (2, 12, 11, 256, 64), (3, 5, 13, 128, 64)])
def test_pshuffle_dw7_relu_matches_float64(B, h, w, C, ldo):
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(B * 100 + h)
    x = torch.randn(B, h, w, C, generator=g).to(f16)
    wt = torch.randn(C // 4, 1, 7, 7, generator=g) / 7
    bias = 0.1 * torch.randn(C // 4, generator=g)
    ref = F.relu(F.conv2d(F.pixel_shuffle(x.double().permute(0, 3, 1, 2), 2), wt.double(), bias.double(), padding=3,
                          groups=C // 4)).permute(0, 2, 3, 1)
    out = torch.full((B, 2 * h, 2 * w, ldo), float("nan"), device=dev, dtype=f16)
    xd, wd, bd = x.to(dev), wt.reshape(C // 4, 49).t().contiguous().to(dev), bias.to(dev)
    cabi.check(lib.udb_pshuffle_dw7_relu(_p(xd), _p(wd), _p(bd), _p(out), B, h, w, C, ldo, _st()), "pshuffle")
    torch.cuda.synchronize()
    err = (out[..., :C // 4].double().cpu() - ref).abs().max().item()
    assert err < 2e-2 * max(1.0, ref.abs().max().item()), err
    assert ldo == C // 4 or out[..., C // 4:].abs().max().item() == 0


def test_pshuffle_dw7_relu_rejects_bad_arguments():
    cabi, lib = _lib()
    _dev()
    z = torch.zeros(64, device="cuda", dtype=f32)
    assert lib.udb_pshuffle_dw7_relu(_p(z), _p(z), _p(z), _p(z), 1, 4, 4, 66, 64, _st()) != 0
    assert b"C=66" in lib.udb_last_error()
    assert lib.udb_pshuffle_dw7_relu(_p(z), _p(z), _p(z), _p(z), 1, 4, 4, 256, 32, _st()) != 0
    assert b"ldo=32" in lib.udb_last_error()
    assert lib.udb_pshuffle_dw7_relu(_p(z), _p(z), _p(z), _p(z), 0, 4, 4, 256, 64, _st()) != 0
    assert b"B=0" in lib.udb_last_error()


def _ray_features_ref(K4, net_hw, grid_hw, scales):
    """flat_interpolate (antialiased bilinear) of the unit rays, normalise, Fourier features with the ray appended."""
    nh, nw = net_hw
    B = K4.shape[0]
    ys, xs = torch.meshgrid(torch.arange(nh, dtype=f64) + 0.5, torch.arange(nw, dtype=f64) + 0.5, indexing="ij")
    out = []
    for b in range(B):
        fx, fy, cx, cy = K4[b].double()
        r = torch.stack([(xs - cx) / fx, (ys - cy) / fy, torch.ones_like(xs)], 0)
        r = r / r.norm(dim=0, keepdim=True)
        r = F.interpolate(r[None], size=grid_hw, mode="bilinear", antialias=True)[0]
        r = F.normalize(r.permute(1, 2, 0).reshape(-1, 3), dim=-1)
        f = torch.sin(r[:, :, None] * scales.double() * math.pi).reshape(-1, 3 * scales.numel())
        out.append(torch.cat([f, r], -1))
    return torch.stack(out)


@pytest.mark.parametrize("B,net,grid", [(1, (588, 784), (42, 56)), (2, (378, 1246), (108, 356)), (3, (434, 350), (31, 25))])
def test_ray_embed_cat_orig_matches_float64(B, net, grid):
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(B)
    K4 = torch.stack([300 + 100 * torch.rand(B, generator=g), 300 + 100 * torch.rand(B, generator=g),
                      net[1] / 2 + 20 * torch.randn(B, generator=g), net[0] / 2 + 20 * torch.randn(B, generator=g)], 1)
    scales = 2.0 ** torch.linspace(0.0, math.log2(max(grid) // 2), 32, dtype=f32)
    out = torch.full((B, grid[0] * grid[1], 128), float("nan"), device=dev, dtype=f16)
    p = cabi.RayEmbed()
    k4d, sd = K4.contiguous().to(dev), scales.to(dev)
    p.intr4, p.scales, p.B, p.net_h, p.net_w, p.gh, p.gw, p.bands = _p(k4d), _p(sd), B, net[0], net[1], grid[0], grid[1], 32
    p.out, p.out_f32 = _p(out), 0
    cabi.check(lib.udb_ray_embed_cat_orig(C.byref(p), 128, _st()), "ray_embed_cat_orig")
    torch.cuda.synchronize()
    ref = _ray_features_ref(K4, net, grid, scales)
    err = (out[..., :99].double().cpu() - ref).abs().max().item()
    # f16 storage of values in [-1, 1] (5e-4) plus the f32 sine of arguments up to pi * max_freq
    assert err < 4e-3 and out[..., 99:].abs().max().item() == 0, err
    assert lib.udb_ray_embed_cat_orig(C.byref(p), 98, _st()) != 0 and b"ld_out=98" in lib.udb_last_error()


@pytest.mark.parametrize("B,gh,gw", [(1, 5, 7), (2, 9, 6)])
def test_v2old_heads_match_float64(B, gh, gw):
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(gh * gw)
    net = (14 * gh + 1, 14 * gw - 3)            # odd and not a multiple of the level grids
    levels = [torch.randn(B, (2 * gh) << i, (2 * gw) << i, 32, generator=g) for i in range(3)]
    w = torch.randn(2, 48, 49, generator=g) / 20
    bd, bc = 0.3, -0.2
    cat_d = torch.cat([F.interpolate(levels[i].double().permute(0, 3, 1, 2)[:, :16], size=net, mode="bilinear") for i in (2, 1, 0)], 1)
    cat_c = torch.cat([F.interpolate(levels[i].double().permute(0, 3, 1, 2)[:, 16:], size=net, mode="bilinear") for i in (2, 1, 0)], 1)
    ref_d = F.conv2d(F.pad(cat_d, (3, 3, 3, 3), mode="reflect"), w[0].double().reshape(1, 48, 7, 7)) + bd
    ref_c = torch.sigmoid(F.conv2d(F.pad(cat_c, (3, 3, 3, 3), mode="reflect"), w[1].double().reshape(1, 48, 7, 7)) + bc)
    lv = [t.to(dev) for t in levels]
    wd = w.to(dev)
    ld = torch.empty(B, *net, device=dev)
    cf = torch.empty(B, *net, device=dev)
    p = cabi.V2oldHeads()
    for i in range(3):
        p.levels[i] = lv[i].data_ptr()
    p.w, p.bias_depth, p.bias_conf, p.B, p.gh, p.gw, p.net_h, p.net_w = _p(wd), bd, bc, B, gh, gw, net[0], net[1]
    p.logdepth, p.confidence = _p(ld), _p(cf)
    cabi.check(lib.udb_v2old_heads(C.byref(p), _st()), "heads")
    torch.cuda.synchronize()
    assert (ld.double().cpu() - ref_d[:, 0]).abs().max().item() < 1e-4 * max(1.0, ref_d.abs().max().item())
    assert (cf.double().cpu() - ref_c[:, 0]).abs().max().item() < 1e-5
    p.net_h = 3
    assert lib.udb_v2old_heads(C.byref(p), _st()) != 0 and b"net_h=3" in lib.udb_last_error()


@pytest.mark.parametrize("B,h,w", [(1, 33, 47), (3, 588, 784)])
def test_v2old_depth_tail_matches_float64(B, h, w):
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(h)
    x = 0.5 * torch.randn(B, h * w, generator=g) + 1.0
    ss = torch.stack([0.3 * torch.randn(B, generator=g), 0.2 * torch.randn(B, generator=g)], 1)
    ref = F.softplus((F.layer_norm(x.double(), (h * w,)).exp() + ss[:, 1:].double()) * ss[:, :1].double().exp(), beta=10.0)
    d = x.to(dev)
    ssd = ss.to(dev)
    cabi.check(lib.udb_v2old_depth_tail(_p(d), _p(ssd), B, h * w, _st()), "tail")
    torch.cuda.synchronize()
    assert ((d.double().cpu() - ref).abs() / ref.abs().clamp_min(1e-3)).max().item() < 1e-4
    assert lib.udb_v2old_depth_tail(_p(d), None, B, h * w, _st()) != 0 and b"scale_shift" in lib.udb_last_error()


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("B,net,HW", [(1, (588, 784), (480, 640)), (2, (378, 1246), (375, 1241)), (1, (70, 56), (211, 133))])
def test_v2old_postprocess_matches_float64(mode, B, net, HW):
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(HW[0])
    depth = 1 + torch.rand(B, 1, *net, generator=g)
    conf = torch.rand(B, 1, *net, generator=g)
    k4 = torch.stack([300 + 50 * torch.rand(B, generator=g), 310 + 50 * torch.rand(B, generator=g),
                      HW[1] / 2 + 10 * torch.rand(B, generator=g), HW[0] / 2 + 10 * torch.rand(B, generator=g)], 1)
    ref_d = F.interpolate(depth, size=HW, mode="bilinear" if mode == 0 else "nearest-exact").double()
    ref_c = F.interpolate(conf.double(), size=HW, mode="bilinear", antialias=True)
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
    od, oc, op = (torch.empty(B, n, *HW, device=dev) for n in (1, 1, 3))
    p = cabi.V2oldPostprocess()
    p.depth, p.confidence, p.k4, p.B, p.net_h, p.net_w, p.H, p.W, p.mode = _p(dd), _p(cd), _p(kd), B, net[0], net[1], HW[0], HW[1], mode
    p.out_depth, p.out_confidence, p.out_points = _p(od), _p(oc), _p(op)
    cabi.check(lib.udb_v2old_postprocess(C.byref(p), _st()), "postprocess")
    torch.cuda.synchronize()
    assert (od.double().cpu() - ref_d).abs().max().item() < 1e-5
    # antialiased weights from f32 tap positions (V1's aa_axis): a few e-5 on values in [0, 1]
    assert (oc.double().cpu() - ref_c).abs().max().item() < 2e-4
    assert ((op.double().cpu() - ref_p).abs() / ref_d.abs()).max().item() < 1e-4
    p.mode = 2
    assert lib.udb_v2old_postprocess(C.byref(p), _st()) != 0 and b"`mode` 2" in lib.udb_last_error()


@pytest.mark.parametrize("with_k", [False, True])
def test_v2old_camera_matches_float64(with_k):
    cabi, lib = _lib()
    dev = _dev()
    B, nh, nw, ratio = 3, 378, 1246, 1.008
    g = torch.Generator().manual_seed(7)
    x4 = 0.3 * torch.randn(B, 4, generator=g)
    K = torch.tensor([[720.0, 0, 610], [0, 725, 180], [0, 0, 1]]).repeat(B, 1, 1) if with_k else None
    x = x4.double()
    half = max(nh, nw) / 2
    pk = torch.stack([half * x[:, 0].exp(), half * x[:, 1].exp(), x[:, 2].sigmoid() * nw, x[:, 3].sigmoid() * nh], 1)
    kout = torch.zeros(B, 3, 3, dtype=f64)
    kout[:, 0, 0], kout[:, 1, 1], kout[:, 0, 2], kout[:, 1, 2], kout[:, 2, 2] = *(pk / ratio).unbind(1)[:2], *(pk / ratio).unbind(1)[2:], 1
    gk = K[:, [0, 1, 0, 1], [0, 1, 2, 2]].double() if with_k else None
    i4, ko, k4 = torch.empty(B, 4, device=dev), torch.empty(B, 3, 3, device=dev), torch.empty(B, 4, device=dev)
    x4d, Kd = x4.to(dev), (K.to(dev) if with_k else None)
    cabi.check(lib.udb_v2old_camera(_p(x4d), _p(Kd), B, nh, nw, ratio, _p(i4), _p(ko), _p(k4), _st()), "camera")
    torch.cuda.synchronize()
    rel = lambda a, b: ((a.double().cpu() - b).abs() / b.abs().clamp_min(1.0)).max().item()
    assert rel(ko, kout) < 1e-6
    assert rel(i4, gk * ratio if with_k else pk) < 1e-6
    assert rel(k4, gk if with_k else pk / ratio) < 1e-6
    assert lib.udb_v2old_camera(_p(x4d), None, B, nh, nw, 0.0, _p(i4), _p(ko), _p(k4), _st()) != 0
    assert b"ratio=0" in lib.udb_last_error()


# ------------------------------------------------------------------------------------------ end to end
def _model(bb, seed, dev):
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))
    from make_golden_v2old import make_v2old_state_dict
    from unidepth_b200 import UniDepthV2old
    cfg = json.load(open(os.path.join(GOLDEN, f"config_v2old_{bb}.json")))
    m = UniDepthV2old(cfg)
    m.load_state_dict(make_v2old_state_dict(cfg, seed), strict=True)
    return m.to(dev).eval()


def _seeded_rgb(shape, seed):
    g = torch.Generator().manual_seed(4321 + seed)
    b, h, w = shape
    return torch.randint(0, 256, (b, 3, h, w), dtype=torch.uint8, generator=g)


GOLDENS = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "v2old_vit*.npz")))


@pytest.mark.parametrize("name", GOLDENS)
def test_infer_matches_reference_golden(name):
    dev = _dev()
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["__meta__"]))
    bb = meta["config"][len("config_v2old_"):-len(".json")]
    m = _model(bb, meta["seed"], dev)
    m.resolution_level = meta["resolution_level"]
    m.interpolation_mode = meta["interpolation_mode"]
    rgb = _seeded_rgb(tuple(meta["shape"]), meta["seed"])
    K = torch.from_numpy(z["K_in"]) if "K_in" in z else None
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = m.infer(rgb.to(dev), K)
    st = meta["strides"]
    d = out["depth"][:, :, ::st["depth"], ::st["depth"]].double().cpu().numpy()
    dr = z["depth"].astype(np.float64)
    arel = float(np.mean(np.abs(d - dr) / dr))
    mrel = float(np.max(np.abs(d - dr) / dr))
    kr = z["intrinsics"].astype(np.float64)
    krel = float(np.max(np.abs(out["intrinsics"].double().cpu().numpy() - kr) / np.maximum(np.abs(kr), 1.0)))
    c = out["confidence"][:, :, ::st["confidence"], ::st["confidence"]].double().cpu().numpy()
    cerr = float(np.max(np.abs(c - z["confidence"])))
    p = out["points"][:, :, ::st["points"], ::st["points"]].double().cpu().numpy()
    pz = z["points"].astype(np.float64)
    prel = float(np.max(np.abs(p - pz)[:, 2] / pz[:, 2]))
    print(f"{name}: depth ARel {arel:.3e} max-rel {mrel:.3e} K max-rel {krel:.3e} confidence max-abs {cerr:.3e} points-z max-rel {prel:.3e}")
    bar_arel, bar_mrel, bar_k, bar_c = BARS[bb]
    assert arel < bar_arel and mrel < bar_mrel and krel < bar_k and cerr < bar_c
    assert prel < bar_mrel


def test_graph_replay_equals_eager_and_batch_slices():
    dev = _dev()
    m = _model("vits14", 0, dev)
    m.resolution_level = 3
    rgb = torch.cat([_seeded_rgb((1, 300, 400), 0), _seeded_rgb((1, 300, 400), 1)]).to(dev)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        g1 = m.infer(rgb)
        g2 = m.infer(rgb)
        m.use_cuda_graph = False
        e = m.infer(rgb)
        one = m.infer(rgb[:1])
    for k in g1:
        assert torch.equal(g1[k], g2[k]) and torch.equal(g1[k], e[k]), k
        assert torch.equal(e[k][:1], one[k]), k


def test_cpu_resident_model_and_unknown_interpolation_raise():
    from unidepth_b200 import UniDepthV2old
    cfg = json.load(open(os.path.join(GOLDEN, "config_v2old_vits14.json")))
    m = UniDepthV2old(cfg)
    with pytest.raises(RuntimeError, match="CUDA device"):
        m.infer(torch.zeros(1, 3, 64, 64, dtype=torch.uint8))
    m.interpolation_mode = "bicubic"
    with pytest.raises(NotImplementedError, match="bicubic"):
        m.infer(torch.zeros(1, 3, 64, 64, dtype=torch.uint8))
