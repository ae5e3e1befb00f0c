"""UniDepthV2's evaluation forward, model(inputs, image_metas) = forward_test, on the GPU: the one engine call with the
ground-truth matching in its last kernel (udb_infer_v2_match, udb_match_gt) against the
unmodified reference (tests/golden/v2fwd_*.npz, oracle/make_golden_v2_forward.py), against torch's matching of
network_forward's outputs, through graph replay, new paddings, both camera paths, and the caller's inputs."""
import copy
import glob
import json
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
FWD_GOLDENS = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "v2fwd_*.npz")))

# Parity of forward_test (f16 mode) against the reference's fp32 outputs on the seeded fixture, per golden: depth ARel,
# depth max relative error, K max relative error, confidence max relative error.  MEASURED on an H100 80GB HBM3 (700 W
# power limit, V2FWDPARITY lines); asserted x1.5.
MEASURED = {
    "v2fwd_vitl14_pads2_224x294_300x400": (1.662e-04, 7.681e-04, 1.703e-04, 1.204e-03),
    "v2fwd_vits14_down_420x560_240x320": (1.463e-04, 7.627e-04, 8.658e-05, 7.818e-04),
    "v2fwd_vits14_eq_294x392": (1.520e-04, 7.579e-04, 7.268e-05, 8.694e-04),
    "v2fwd_vits14_eucm_294x392_480x640": (7.021e-04, 4.971e-03, 1.986e-04, 6.792e-03),
    "v2fwd_vits14_pads2_294x392_480x640": (1.253e-04, 8.702e-04, 2.739e-04, 8.070e-04),
    "v2fwd_vits14_pinhole_294x392_360x480": (1.369e-04, 7.337e-04, 1.639e-04, 9.857e-04),
}
# Largest difference between the engine's matched maps and validation.match_gt applied to network_forward's maps of the
# same input, in units in the last place of the pixel's largest channel (|z| for the points, the value itself for depth
# and confidence).  The interpolation is ATen's, term for term: the confidence, whose taps are read as stored, is bit-equal;
# the points' taps rays * radius can round differently where the compiler contracts the ray arithmetic differently in
# the two kernels (measured on an H100 80GB HBM3: 2.32 ulp at most).
MAX_ULP = 4


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _model(meta, dev):
    from fixture import make_state_dict
    from unidepth_b200 import UniDepthV2
    cfg = json.load(open(os.path.join(GOLDEN, meta["config"])))
    m = UniDepthV2(copy.deepcopy(cfg))
    m.load_state_dict(make_state_dict(cfg, meta["seed"]), strict=True)
    return m.to(dev).eval()


def _case(name, dev):
    from test_v2_forward_cpu import golden_case
    z, meta, inputs, metas = golden_case(name)
    inputs = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in inputs.items()}
    return z, meta, inputs, metas


def _errors(out, z, meta):
    st = meta["strides"]
    d = out["depth"][:, :, ::st["depth"], ::st["depth"]].double().cpu().numpy()
    dr = z["depth"].astype(np.float64)
    arel, mrel = float(np.mean(np.abs(d - dr) / dr)), float(np.max(np.abs(d - dr) / dr))
    kr = z["intrinsics"].astype(np.float64)
    krel = float(np.max(np.abs(out["intrinsics"].double().cpu().numpy() - kr) / np.maximum(np.abs(kr), 1.0)))
    c = out["confidence"][:, :, ::st["confidence"], ::st["confidence"]].double().cpu().numpy()
    cr = z["confidence"].astype(np.float64)
    crel = float(np.max(np.abs(c - cr) / cr))
    return arel, mrel, krel, crel


def _ulp(a, b):
    """Largest |a - b| per pixel over the f32 spacing (2^-23 relative) of the pixel's largest channel of b."""
    scale = b.double().abs().amax(dim=1, keepdim=True).clamp(min=1e-30) * 2.0 ** -23
    return float(((a.double() - b.double()).abs() / scale).max().item())


@pytest.mark.parametrize("name", FWD_GOLDENS)
def test_forward_matches_reference_golden(name):
    dev = _dev()
    z, meta, inputs, metas = _case(name, dev)
    m = _model(meta, dev)
    before = {k: (v.clone() if isinstance(v, torch.Tensor) else copy.deepcopy(v)) for k, v in inputs.items()}
    ptrs = {k: v.data_ptr() for k, v in inputs.items() if isinstance(v, torch.Tensor)}
    # the paddings travel in the metas only, as the reference's evaluation loop hands them over
    out = m(inputs, metas)
    assert set(inputs) == set(before) and {k: v.data_ptr() for k, v in inputs.items() if isinstance(v, torch.Tensor)} == ptrs
    for k, v in before.items():
        if isinstance(v, torch.Tensor):
            assert torch.equal(inputs[k], v), k
    B, (h, w), (H, W) = meta["shape"][0], meta["shape"][1:], meta["gt_hw"]
    assert set(out) == {"depth", "points", "confidence", "rays", "intrinsics"}
    assert out["depth"].shape == out["confidence"].shape == (B, 1, H, W) and out["points"].shape == (B, 3, H, W)
    assert out["rays"].shape == (B, 3, h, w) and out["intrinsics"].shape == (B, 3, 3)
    assert torch.equal(out["depth"], out["points"][:, 2:])
    arel, mrel, krel, crel = _errors(out, z, meta)
    print(f"V2FWDPARITY {name}: depth ARel {arel:.3e} max-rel {mrel:.3e} K max-rel {krel:.3e} confidence max-rel {crel:.3e}")
    bars = tuple(1.5 * v for v in MEASURED[name])
    assert arel <= bars[0] and mrel <= bars[1] and krel <= bars[2] and crel <= bars[3], (name, bars)


@pytest.mark.parametrize("name", ["v2fwd_vits14_pads2_294x392_480x640", "v2fwd_vits14_down_420x560_240x320",
                                  "v2fwd_vits14_eq_294x392", "v2fwd_vits14_pinhole_294x392_360x480"])
def test_matching_equals_torch_matching_of_network_forward(name):
    """The engine's matching against validation.match_gt / match_intrinsics on network_forward's outputs of the same
    input and camera: K bit for bit, the maps within MAX_ULP."""
    from unidepth_b200.camera import pack_camera
    from unidepth_b200.validation import match_gt, match_intrinsics
    dev = _dev()
    z, meta, inputs, metas = _case(name, dev)
    m = _model(meta, dev)
    out = m(inputs, metas)
    x = inputs["image"]
    B, _, h, w = x.shape
    rays = None
    if "camera" in inputs:
        assert pack_camera(inputs["camera"]) is not None
        rays = inputs["camera"].get_rays(shapes=(B, h, w)).to(dev).expand(B, 3, h, w)
    net = m._network_outputs(x, rays)
    pads = m._match_paddings(inputs, metas, B, h, w).tolist()
    gt = inputs["depth"]
    worst = {}
    for k in ("depth", "points", "confidence"):
        ref = match_gt(net[k], gt, padding1=pads, padding2=None)
        worst[k] = _ulp(out[k], ref)
    worst["rays"] = _ulp(out["rays"], net["rays"] / torch.norm(net["rays"], dim=1, keepdim=True).clip(min=1e-5))
    print(f"V2FWDULP {name}: " + ", ".join(f"{k} {v:.2f}" for k, v in worst.items()))
    assert torch.equal(out["intrinsics"], match_intrinsics(net["intrinsics"], x, gt, padding1=pads, padding2=None))
    # a Pinhole camera's rays come from the camera kernel here and from the object's get_rays in network_forward
    if "camera" not in inputs:
        assert max(worst.values()) <= MAX_ULP, worst


def test_graph_replay_equals_eager_and_new_paddings_replay():
    dev = _dev()
    z, meta, inputs, metas = _case("v2fwd_vits14_pads2_294x392_480x640", dev)
    m = _model(meta, dev)
    g1 = m(inputs, metas)
    n = len(m._graphs)
    g2 = m(inputs, metas)
    other = [{"paddings": (0, 0, 0, 0)}, {"paddings": (28, 14, 0, 7)}]
    g3 = m(inputs, other)
    assert len(m._graphs) == n == 1, "other paddings must replay the same graph"
    m.use_cuda_graph = False
    e1, e3 = m(inputs, metas), m(inputs, other)
    for k in g1:
        assert g1[k].data_ptr() != g2[k].data_ptr()
        assert torch.equal(g1[k], g2[k]) and torch.equal(g1[k], e1[k]) and torch.equal(g3[k], e3[k]), k
    for k in ("depth", "points", "confidence", "intrinsics"):
        assert not torch.equal(g1[k], g3[k]), k
    assert torch.equal(g1["rays"], g3["rays"])
    # the first image has zero paddings in `other`: its outputs equal those of a zero-padded call
    zero = m(dict(inputs, paddings=[(0, 0, 0, 0)] * 2), None)
    for k in ("depth", "points", "confidence", "intrinsics"):
        assert torch.equal(zero[k][0], g3[k][0]), k


def test_device_camera_rays_against_the_host_path():
    from test_camera_kernel_gpu import _HostOnly
    dev = _dev()
    # (depth ARel, depth max-rel) of the device path against the host path, MEASURED on an H100 80GB HBM3 (700 W);
    # asserted x1.5.  The host path asks the object for its rays as given, and the two ray sets differ by up to one f32
    # ulp here, unlike infer's EUCM case, where they are bit-identical; the f16 network amplifies that to the depth error
    # below.  The rays are held to test_camera_kernel_gpu.py's bound for infer's two paths (1.5 x 1.49e-7).
    for name, bound in (("v2fwd_vits14_pinhole_294x392_360x480", (8.684e-05, 5.347e-04)),
                        ("v2fwd_vits14_eucm_294x392_480x640", (3.723e-04, 2.938e-03))):
        z, meta, inputs, metas = _case(name, dev)
        m = _model(meta, dev)
        dev_out = m(inputs, metas)
        host_out = m(dict(inputs, camera=_HostOnly(inputs["camera"])), metas)
        assert len(m._graphs) == 2                   # one per camera source
        dr = host_out["depth"]
        rel = (dev_out["depth"] - dr).abs() / dr.abs().clamp(min=0.1 * dr.abs().mean().item())
        rmax = (dev_out["rays"] - host_out["rays"]).abs().max().item()
        print(f"V2FWDCAMERA {name}: depth ARel {rel.mean().item():.3e} max {rel.max().item():.3e} rays max {rmax:.3e}")
        assert rel.mean().item() <= 1.5 * bound[0] and rel.max().item() <= 1.5 * bound[1] and rmax <= 1.5 * 1.490e-7
        assert torch.equal(dev_out["intrinsics"], host_out["intrinsics"])
