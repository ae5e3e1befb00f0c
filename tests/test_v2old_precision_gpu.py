"""UniDepthV2old precision = "split" and "fp8" on the GPU: the split output of the ray Fourier-feature kernel against a
float64 restatement and against its f16 output, both modes' `infer` against every V2old golden of the unmodified reference
(tests/golden/v2old_*.npz), and switching between the three modes.  tests/test_v2old_precision_cpu.py checks the packer
and the schedule without a GPU."""
import ctypes as C
import json
import math
import os
import warnings

import numpy as np
import pytest
import torch

from test_v2old_gpu import GOLDEN, GOLDENS, _dev, _lib, _model, _p, _ray_features_ref, _seeded_rgb, _st

pytestmark = pytest.mark.gpu
f16, f32, f64 = torch.float16, torch.float32, torch.float64

# Split-mode bars per backbone: depth ARel, depth max relative error, confidence max absolute error, each 1.5 times the
# largest value measured on an H100 80GB HBM3 (700 W) over the backbone's six goldens (ViT-L 9.9e-4 / 4.8e-3 / 4.2e-4,
# ViT-S 1.24e-3 / 8.7e-3 / 5.3e-4; intrinsics at most 7.8e-6); the intrinsics bar is the fixed 1e-4 of UniDepthV1's
# split mode.
SPLIT_BARS = {"vitl14": (1.5e-3, 7.2e-3, 6.3e-4), "vits14": (1.9e-3, 1.3e-2, 8.1e-4)}
SPLIT_K_BAR = 1e-4
# fp8-mode bars: depth ARel, depth max-rel, intrinsics max-rel, confidence max-abs, 1.5 times the largest value measured
# on the same card (ViT-L 0.225 / 3.21 / 2.67e-2 / 0.111, ViT-S 0.217 / 3.34 / 2.33e-2 / 0.113).  The seeded fixture
# amplifies e4m3 operand rounding far more than UniDepthV2's does; the CPU rounding model gives the same order.
FP8_BARS = {"vitl14": (0.34, 4.9, 4.0e-2, 0.17), "vits14": (0.33, 5.1, 3.5e-2, 0.17)}
# depth ARel the CPU rounding model of tests/test_v2old_precision_cpu.py predicts for fp8 mode (e4m3 operands in the
# encoder blocks' four linear layers, f32 elsewhere), for the golden it runs
CPU_MODEL_FP8_AREL = {"v2old_vits14_rl0_360x480": 1.057e-1}


# ------------------------------------------------------------------------------------------ the split ray features
@pytest.mark.parametrize("B,net,grid", [(1, (588, 784), (42, 56)), (2, (588, 784), (84, 112)), (2, (378, 1246), (27, 89)),
                                        (3, (434, 350), (31, 25))])
def test_ray_embed_cat_orig_split_output(B, net, grid):
    """hi + lo against the kernel's own f32 features (the value the split pair represents) and against the float64
    restatement; hi bit-equal to the f16 output; both halves zero past the 99 features; the ld_out check."""
    cabi, lib = _lib()
    dev = _dev()
    g = torch.Generator().manual_seed(B + grid[0])
    K4 = torch.stack([300 + 100 * torch.rand(B, generator=g), 300 + 100 * torch.rand(B, generator=g),
                      net[1] / 2 + 20 * torch.randn(B, generator=g), net[0] / 2 + 20 * torch.randn(B, generator=g)], 1)
    scales = 2.0 ** torch.linspace(0.0, math.log2(max(grid) // 2), 32, dtype=f32)
    k4d, sd = K4.contiguous().to(dev), scales.to(dev)
    n = grid[0] * grid[1]

    def run(out_f32, ld, dtype):
        out = torch.full((B, n, ld), float("nan"), device=dev, dtype=dtype)
        p = cabi.RayEmbed()
        p.intr4, p.scales, p.B, p.net_h, p.net_w, p.gh, p.gw, p.bands = _p(k4d), _p(sd), B, net[0], net[1], grid[0], grid[1], 32
        p.out, p.out_f32 = _p(out), out_f32
        cabi.check(lib.udb_ray_embed_cat_orig(C.byref(p), ld, _st()), "ray_embed_cat_orig")
        torch.cuda.synchronize()
        return out.cpu(), p

    y16, _ = run(0, 128, f16)
    y32, _ = run(1, 128, f32)
    sp, p = run(2, 256, f16)
    hi, lo = sp[..., :128], sp[..., 128:]
    assert torch.equal(hi, y16)
    assert hi[..., 99:].abs().max().item() == 0 and lo[..., 99:].abs().max().item() == 0
    rec = hi.double() + lo.double()
    y = y32.double()
    # hi carries 11 bits and lo the next 11: 2^-21 relative, with half the f16 subnormal step as the floor where lo is tiny
    assert ((rec - y).abs() <= 2.0 ** -21 * y.abs() + 2.0 ** -25).all(), (rec - y).abs().max().item()
    ref = _ray_features_ref(K4, net, grid, scales)
    err = (rec[..., :99] - ref).abs().max().item()
    err32 = (y[..., :99] - ref).abs().max().item()
    # the split pair is as close to float64 as the kernel's f32 arithmetic (the f32 sine of arguments up to pi * 112)
    assert err <= err32 + 2.0 ** -20, (err, err32)
    print(f"ray features split {grid}: hi+lo vs float64 {err:.3e} (f32 output {err32:.3e})")
    for bad in (197, 196, 100):      # odd; one feature short per half; room for one half only
        assert lib.udb_ray_embed_cat_orig(C.byref(p), bad, _st()) != 0
        assert f"ld_out={bad}".encode() in lib.udb_last_error() and b"both halves" in lib.udb_last_error()


# ------------------------------------------------------------------------------------------ end to end
def _run_golden(name, precision):
    dev = _dev()
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["__meta__"]))
    bb = meta["config"][len("config_v2old_"):-len(".json")]
    m = _model(bb, meta["seed"], dev)
    m.precision = precision
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
    kr = z["intrinsics"].astype(np.float64)
    c = out["confidence"][:, :, ::st["confidence"], ::st["confidence"]].double().cpu().numpy()
    errs = dict(arel=float(np.mean(np.abs(d - dr) / dr)), mrel=float(np.max(np.abs(d - dr) / dr)),
                krel=float(np.max(np.abs(out["intrinsics"].double().cpu().numpy() - kr) / np.maximum(np.abs(kr), 1.0))),
                cerr=float(np.max(np.abs(c - z["confidence"]))))
    return bb, errs


@pytest.mark.parametrize("name", GOLDENS)
def test_split_infer_matches_reference_golden(name):
    bb, e = _run_golden(name, "split")
    print(f"V2OLDSPLITPARITY {name}: depth ARel {e['arel']:.3e} max-rel {e['mrel']:.3e} intrinsics rel {e['krel']:.3e} "
          f"confidence max-abs {e['cerr']:.3e}")
    bar_arel, bar_mrel, bar_c = SPLIT_BARS[bb]
    assert e["krel"] < SPLIT_K_BAR
    assert e["arel"] < bar_arel and e["mrel"] < bar_mrel and e["cerr"] < bar_c


@pytest.mark.parametrize("name", GOLDENS)
def test_fp8_infer_matches_reference_golden(name):
    bb, e = _run_golden(name, "fp8")
    model = CPU_MODEL_FP8_AREL.get(name)
    print(f"V2OLDFP8PARITY {name}: depth ARel {e['arel']:.3e} max-rel {e['mrel']:.3e} intrinsics rel {e['krel']:.3e} "
          f"confidence max-abs {e['cerr']:.3e} (CPU rounding model depth ARel: {'%.3e' % model if model else 'not run'})")
    bar_arel, bar_mrel, bar_k, bar_c = FP8_BARS[bb]
    assert e["arel"] < bar_arel and e["mrel"] < bar_mrel and e["krel"] < bar_k and e["cerr"] < bar_c


def test_switching_modes_graphs_and_batch_slices():
    """f16 -> split -> fp8 -> f16 gives the first f16 outputs bit for bit; in each mode a graph replay equals the eager
    run and image 0 of a batch equals that image run alone."""
    dev = _dev()
    m = _model("vits14", 0, dev)
    m.resolution_level = 3
    rgb = torch.cat([_seeded_rgb((1, 300, 400), 0), _seeded_rgb((1, 300, 400), 1)]).to(dev)
    first = None
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for prec in ("f16", "split", "fp8", "f16"):
            m.precision = prec
            m.use_cuda_graph = True
            g1 = m.infer(rgb)
            g2 = m.infer(rgb)
            m.use_cuda_graph = False
            e = m.infer(rgb)
            one = m.infer(rgb[:1])
            for k in g1:
                assert torch.equal(g1[k], g2[k]) and torch.equal(g1[k], e[k]), (prec, k)
                assert torch.equal(e[k][:1], one[k]), (prec, k)
            if first is None:
                first = g1
            elif prec != "f16":
                assert not torch.equal(g1["depth"], first["depth"]), prec
    for k in first:
        assert torch.equal(first[k], g1[k]), k
