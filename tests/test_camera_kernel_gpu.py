"""The GPU ray generator for camera objects (udb_camera_rays, ops.camera_rays) and the camera-conditioned `infer` it
serves, including CUDA-graph replay for every camera source.

Bounds of the kernel against the class's own `get_rays` (BatchCamera.from_camera(cam).crop(-pads).resize(f).get_rays,
fp32 torch on the same GPU), with u = 2^-24:
  * EUCM and Spherical: the kernel evaluates the class's expressions op for op with IEEE rounding (no FMA contraction),
    so the two differ only in how the final normalisations (one for EUCM, two for Spherical) sum three squares: at most
    2 u relative on the norm each, so 16 u per unit-vector component covers both.
  * Pinhole (torch.inverse vs the kernel's adjugate), OPENCV, Fisheye624 and MEI (the same fixed-step Newton solves,
    whose sums torch reduces in its own order): both sides carry the rounding error of an fp32 evaluation of the same
    function.  Against a float64 evaluation of the class (E32 = max |class_fp32 - class_fp64|, E_k the same for the
    kernel), |kernel - class| <= E_k + E32.  The kernel's own error E_k is of the class's size (largest E_k / E32
    measured on an H100: 1.64, opencv_strong at 14 x 14, where the corners sit close to the end of the monotonic
    range of its radial polynomial); asserted with an allowance of 3 E32 for it: max |kernel - class| <= 4 E32 + 16 u.
The measured maxima are printed as `RAYS` lines; the largest error / bound ratio measured is 0.64 for the Newton
models (opencv_strong), 0.16 for Pinhole with skew and 0 for EUCM and Spherical, which are bit-identical to the class.
"""
import copy
import ctypes as Ct
import json
import os

import numpy as np
import pytest
import torch

from unidepth_b200 import _cabi, ops
from unidepth_b200 import camera as C

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _p16(fx, fy, cx, cy, radial=(), tang=(0.0, 0.0), prism=(0.0, 0.0, 0.0, 0.0)):
    r = list(radial) + [0.0] * (6 - len(radial))
    return torch.tensor([[fx, fy, cx, cy, *r, *tang, *prism]], dtype=torch.float32)


# cameras in INPUT-image pixels for a 480 x 640 image; "strong" ones distort far into the corners
CAMERAS = {
    "pinhole": lambda: C.Pinhole(params=torch.tensor([[520.0, 515.0, 321.5, 238.25]])),
    "pinhole_skew": lambda: C.Pinhole(K=torch.tensor([[[520.0, 3.5, 321.5], [0.0, 515.0, 238.25], [0.0, 0.0, 1.0]]])),
    "eucm": lambda: C.EUCM(params=torch.tensor([[300.0, 302.0, 320.0, 241.0, 0.62, 1.05]])),
    "eucm_wide": lambda: C.EUCM(params=torch.tensor([[150.0, 150.0, 320.0, 240.0, 0.8, 1.4]])),
    "spherical": lambda: C.Spherical(params=torch.tensor([[100.0, 100.0, 320.0, 240.0, 640.0, 480.0, 3.0, 1.2]])),
    "opencv_strong": lambda: C.OPENCV(params=_p16(300.0, 302.0, 322.0, 236.0, (-0.2, 0.05, -0.005), (1.5e-3, -8e-4),
                                                  (2e-3, -1e-3, 1e-3, 5e-4))),
    "opencv_radial": lambda: C.OPENCV(params=_p16(500.0, 500.0, 320.0, 240.0, (-0.12, 0.03))),
    "opencv_plain": lambda: C.OPENCV(params=_p16(500.0, 500.0, 320.0, 240.0)),
    "fisheye_strong": lambda: C.Fisheye624(params=_p16(180.0, 181.0, 321.0, 239.0, (0.05, -0.012, 0.004, -6e-4, 4e-5, -1e-6),
                                                       (2e-3, -1e-3), (1e-3, -5e-4, 8e-4, -2e-4))),
    "fisheye_radial": lambda: C.Fisheye624(params=_p16(240.0, 240.0, 320.0, 240.0, (0.03, -0.004))),
    "fisheye_prism_only": lambda: C.Fisheye624(params=_p16(240.0, 240.0, 320.0, 240.0, (0.03,), (0.0, 0.0),
                                                           (3e-3, 0.0, -2e-3, 0.0))),
    "mei_strong": lambda: C.MEI(params=torch.tensor([[420.0, 421.0, 319.0, 241.0, -0.22, 0.06, 2e-3, -1e-3, 1.3]])),
    "mei_xi1": lambda: C.MEI(params=torch.tensor([[330.0, 330.0, 320.0, 240.0, -0.1, 0.01, 0.0, 0.0, 1.0]])),
    "mei_plain": lambda: C.MEI(params=torch.tensor([[330.0, 330.0, 320.0, 240.0, 0.0, 0.0, 0.0, 0.0, 0.8]])),
}
CLOSED = {"eucm", "eucm_wide", "spherical"}
# (net_h, net_w, paddings l r t b, factor)
GEOMS = [(14, 14, (0, 0, 80, 80), 0.021875), (14, 644, (0, 0, 80, 80), 1.0), (490, 14, (40, 40, 0, 0), 1.0),
         (490, 644, (0, 0, 0, 0), 1.0208), (490, 644, (0, 0, 13, 17), 0.73), (490, 644, (9, 7, 0, 0), 1.6), (30, 44, (3, 3, 5, 5), 0.73)]


def _class_rays(cam, pads, factor, nh, nw, dev, double=False):
    cam = copy.deepcopy(cam).to(dev)
    if double:
        if isinstance(cam, C.Pinhole):
            return _pinhole64(cam, pads, factor, nh, nw)
        cam.params, cam.K = cam.params.double(), cam.K.double()
    pl, pr, pt, pb = pads
    bc = C.BatchCamera.from_camera(cam).crop(left=-pl, top=-pt, right=-pr, bottom=-pb).resize(factor)
    r = bc.get_rays(shapes=(1, nh, nw))
    return r.permute(0, 2, 3, 1).reshape(r.shape[0], nh * nw, 3)


def _pinhole64(cam, pads, factor, nh, nw):
    """Pinhole.unproject inverts K in fp32 whatever its dtype: the float64 evaluation is restated here."""
    pl, _, pt, _ = pads
    K = cam.K.double().reshape(-1, 3, 3).clone()
    K[:, 0, 2] += pl
    K[:, 1, 2] += pt
    K[:, :2] *= factor
    uv = C.pixel_grid(1, nh, nw, homogeneous=True, device=K.device).double().reshape(1, 3, -1)
    xyz = torch.linalg.inv(K) @ uv
    xyz = xyz / xyz[:, 2:].clamp(min=1e-4)
    xyz = xyz / xyz.norm(dim=1, keepdim=True).clamp(min=1e-4)
    return xyz.transpose(1, 2)


def _kernel_rays(cam, pads, factor, nh, nw, B=1, dev=None):
    model, rows = C.pack_camera(cam)
    rows = rows.to(dev).expand(B, _cabi.CAM_STRIDE).contiguous() if rows.shape[0] == 1 else rows.to(dev).contiguous()
    return ops.camera_rays(model, rows, B, (nh, nw), pads, factor)


@pytest.mark.parametrize("name", sorted(CAMERAS))
def test_kernel_matches_class_get_rays(name):
    dev = _dev()
    worst = 0.0
    for nh, nw, pads, factor in GEOMS:
        cam = CAMERAS[name]()
        before = (cam.params.clone(), cam.K.clone())
        got = _kernel_rays(cam, pads, factor, nh, nw, dev=dev)
        assert torch.equal(cam.params, before[0]) and torch.equal(cam.K, before[1])
        ref = _class_rays(cam, pads, factor, nh, nw, dev)
        ref64 = _class_rays(cam, pads, factor, nh, nw, dev, double=True)
        assert got.shape == ref.shape == (1, nh * nw, 3)
        # pixels outside the model's domain (MEI with xi > 1 far off axis: no real lift) are NaN in every evaluation;
        # the kernel may only be non-finite there
        ok = torch.isfinite(ref64).all(-1)
        assert torch.isfinite(got).all(-1)[ok].all() and torch.isfinite(ref).all(-1)[ok].all()
        assert ok.float().mean().item() > 0.5, (name, nh, nw)
        err = (got - ref).abs()[ok].max().item()
        e32 = (ref.double() - ref64).abs()[ok].max().item()
        ek = (got.double() - ref64).abs()[ok].max().item()
        bound = 16 * U if name in CLOSED else 4 * e32 + 16 * U
        print(f"RAYS {name} {nh}x{nw} pads {pads} factor {factor}: |kernel-class| {err:.3e} (bound {bound:.3e}), "
              f"|class-f64| {e32:.3e}, |kernel-f64| {ek:.3e}")
        assert err <= bound, (name, nh, nw, pads, factor, err, bound)
        worst = max(worst, err / bound)
    print(f"RAYS {name}: largest error/bound {worst:.3f}")


def test_strong_distortion_reaches_the_corners():
    """The "strong" cameras really are far from pinhole at the corners of a 490 x 644 network input."""
    dev = _dev()
    for name in ("opencv_strong", "fisheye_strong", "mei_strong", "eucm_wide"):
        cam = CAMERAS[name]()
        r = _kernel_rays(cam, (0, 0, 0, 0), 1.0208, 490, 644, dev=dev).view(490, 644, 3)
        fx, fy, cx, cy = cam.params[0, :4].tolist()
        K = torch.tensor([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])
        pin = _kernel_rays(C.Pinhole(K=K[None]), (0, 0, 0, 0), 1.0208, 490, 644, dev=dev).view(490, 644, 3)
        d = (r[0, 0] - pin[0, 0]).abs().max().item()
        print(f"{name}: corner ray differs from the pinhole ray by {d:.3f}")
        assert d > 0.05, name


@pytest.mark.parametrize("name", ["pinhole_params", "eucm", "spherical", "opencv_radial", "opencv_full", "fisheye624",
                                  "fisheye624_radial", "mei", "mei_plain"])
def test_kernel_matches_reference_infer_rays(name):
    """tests/golden/cameras.npz `*/infer_rays`: the unmodified reference's crop(-pads).resize(0.73).get_rays at 30 x 44,
    at test_camera_cpu.py's bars (2e-6 closed forms, 1.5e-3 iterative models: the reference's own solver stops at 1e-3)."""
    dev = _dev()
    z = np.load(os.path.join(ROOT, "tests", "golden", "cameras.npz"))
    cls = {"pinhole_params": "Pinhole", "eucm": "EUCM", "spherical": "Spherical", "opencv_radial": "OPENCV",
           "opencv_full": "OPENCV", "fisheye624": "Fisheye624", "fisheye624_radial": "Fisheye624", "mei": "MEI",
           "mei_plain": "MEI"}[name]
    cam = getattr(C, cls)(params=torch.from_numpy(z[f"{name}/params"]).clone())
    got = _kernel_rays(cam, (3, 3, 5, 5), 0.73, 30, 44, dev=dev).cpu()
    want = torch.from_numpy(z[f"{name}/infer_rays"]).permute(0, 2, 3, 1).reshape(1, 30 * 44, 3)
    e = (got - want).abs().max().item()
    print(f"{name}: kernel vs reference infer_rays {e:.2e}")
    assert e < (2e-6 if cls in ("Pinhole", "EUCM", "Spherical") else 1.5e-3), e


def test_broadcast_batch_canary_and_determinism():
    dev = _dev()
    lib = _cabi.lib()
    nh, nw, pads, f = 490, 644, (0, 0, 13, 17), 0.73
    for name in ("fisheye_strong", "spherical", "pinhole_skew"):
        cam = CAMERAS[name]()
        one = _kernel_rays(cam, pads, f, nh, nw, B=1, dev=dev)
        four = _kernel_rays(cam, pads, f, nh, nw, B=4, dev=dev)
        for b in range(4):
            assert torch.equal(four[b], one[0]), (name, b)
        # per-image cameras: image b of a batch equals its own single run
        cams = [CAMERAS[name]() for _ in range(3)]
        for i, c in enumerate(cams):
            c.params[0, 0] += 10.0 * i
            if isinstance(c, C.Pinhole):
                c.K[0, 0, 0] += 10.0 * i
        model, rows = C.pack_camera(torch.cat([C.BatchCamera.from_camera(c) for c in cams]))
        batch = ops.camera_rays(model, rows.to(dev).contiguous(), 3, (nh, nw), pads, f)
        for i, c in enumerate(cams):
            assert torch.equal(batch[i], _kernel_rays(c, pads, f, nh, nw, dev=dev)[0]), (name, i)
        # NaN canary around the output; two runs bit-identical
        model, rows = C.pack_camera(cam)
        rows = rows.to(dev).expand(2, _cabi.CAM_STRIDE).contiguous()
        n = 2 * nh * nw * 3
        outs = []
        for _ in range(2):
            buf = torch.full((n + 128,), float("nan"), device=dev)
            st = Ct.c_void_p(torch.cuda.current_stream().cuda_stream)
            rc = lib.udb_camera_rays(model, Ct.c_void_p(rows.data_ptr()), 2, nh, nw, *pads, Ct.c_float(f),
                                     Ct.c_void_p(buf.data_ptr() + 64 * 4), st)
            assert rc == 0, lib.udb_last_error()
            torch.cuda.synchronize()
            assert torch.isnan(buf[:64]).all() and torch.isnan(buf[64 + n:]).all()
            assert torch.isfinite(buf[64:64 + n]).all()
            outs.append(buf[64:64 + n].clone())
        assert torch.equal(outs[0], outs[1])
        assert torch.equal(outs[0].view(2, nh * nw, 3)[0], one[0])


# ------------------------------------------------------------------------------------------------------ end to end
class _HostOnly:
    """A camera object the packer does not know: infer takes the host path (the object's own crop / resize / get_rays)."""

    def __init__(self, cam):
        self.cam = copy.deepcopy(cam)

    def to(self, device):
        self.cam = self.cam.to(device)
        return self

    def crop(self, left, top, right=None, bottom=None):
        self.cam = self.cam.crop(left, top, right, bottom)
        return self

    def resize(self, factor):
        self.cam = self.cam.resize(factor)
        return self

    def get_rays(self, shapes):
        return self.cam.get_rays(shapes)


@pytest.fixture(scope="module")
def shallow():
    from fixture import make_state_dict
    from test_infer_parity_gpu import _cfg
    cfg = _cfg(depth=4)
    return cfg, make_state_dict(cfg, 0)


def _model(cfg, sd):
    _dev()
    from unidepth_b200 import UniDepthV2
    m = UniDepthV2(copy.deepcopy(cfg))
    m.load_state_dict(sd, strict=True)
    return m.to("cuda:0").eval()


def _rgb(shape, seed):
    g = torch.Generator().manual_seed(1234 + seed)
    b, h, w = shape
    return torch.randint(0, 256, (b, 3, h, w), dtype=torch.uint8, generator=g)


# camera -> (depth ARel, depth max-rel, rays max) of the device path against the host path, MEASURED on an H100 80GB HBM3
# (700 W power limit); asserted x1.5.  EUCM and Spherical give bit-identical rays, so everything downstream is identical too.
# The intrinsics are predicted either way and must be bit-equal.
MEASURED_E2E = {
    "pinhole": (1.169e-04, 8.727e-04, 1.490e-07),
    "pinhole_skew": (1.155e-04, 8.469e-04, 2.086e-07),
    "eucm": (0.0, 0.0, 0.0),
    "spherical": (0.0, 0.0, 0.0),
    "opencv_strong": (1.144e-04, 7.826e-04, 2.086e-07),
    "fisheye_strong": (1.145e-04, 9.433e-04, 2.444e-05),
    "mei_strong": (1.101e-04, 7.664e-04, 1.192e-07),
    "mei_xi1": (1.113e-04, 8.591e-04, 1.192e-07),
}


@pytest.mark.parametrize("name", ["pinhole", "pinhole_skew", "eucm", "spherical", "opencv_strong", "fisheye_strong",
                                  "mei_strong", "mei_xi1"])
def test_infer_device_path_equals_host_path(shallow, name):
    cfg, sd = shallow
    m = _model(cfg, sd)
    m.resolution_level = None
    rgb = _rgb((2, 480, 640), 7)            # the image the cameras are defined for
    cam = CAMERAS[name]()
    before = (cam.params.clone(), cam.K.clone())
    dev_out = m.infer(rgb, camera=cam)
    host_out = m.infer(rgb, camera=_HostOnly(cam))
    assert torch.equal(cam.params, before[0]) and torch.equal(cam.K, before[1])
    # depth = points.z: relative to max(|depth|, 10 % of its mean) since wide cameras see rays with z near 0
    dr = host_out["depth"]
    rel = (dev_out["depth"] - dr).abs() / dr.abs().clamp(min=0.1 * dr.abs().mean().item())
    rmax = (dev_out["rays"] - host_out["rays"]).abs().max().item()
    print(f"E2E {name}: depth ARel {rel.mean().item():.3e} max {rel.max().item():.3e}, rays max {rmax:.3e}, intrinsics "
          f"{dev_out['intrinsics'][0].flatten().tolist()}")
    tol = tuple(1.5 * v for v in MEASURED_E2E[name])
    assert rel.mean().item() <= tol[0] and rel.max().item() <= tol[1] and rmax <= tol[2], (name, tol)
    assert torch.equal(dev_out["intrinsics"], host_out["intrinsics"])
    assert len(m._graphs) == 2                      # both replayed a graph, one per camera source


GOLDEN_CAMERA = ["vits_camK_120x160", "vits_campinhole_pad_96x288_rl3", "vits_cameucm_pad_200x70_rl0"]
# (depth ARel, depth max-rel, intrinsics max-rel) against the reference's goldens, MEASURED on an H100 80GB HBM3 (700 W);
# asserted x1.5 (MARGIN)
MEASURED_GOLDEN = {
    "vits_camK_120x160": (1.017e-04, 7.859e-04, 8.242e-05),
    "vits_campinhole_pad_96x288_rl3": (1.494e-04, 7.941e-04, 9.931e-05),
    "vits_cameucm_pad_200x70_rl0": (1.498e-04, 8.780e-04, 5.831e-05),
}


@pytest.mark.parametrize("name", GOLDEN_CAMERA)
def test_camera_goldens_through_the_device_path(name):
    """The unmodified reference's infer(rgb, camera=...) outputs (subsampled goldens) against the CUDA path, whose
    Pinhole / EUCM objects now take the device ray generator; bars as test_infer_parity_gpu (measured x1.5), and the
    rays themselves within 1e-5."""
    from fixture import make_state_dict
    from test_infer_parity_gpu import MARGIN, _check
    from test_oracle_golden import _rgb as golden_rgb, subsample_like_golden
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    meta = json.loads(str(z["__meta__"]))
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", meta["config"])))
    m = _model(cfg, make_state_dict(cfg, meta["seed"]))
    m.resolution_level = meta["resolution_level"]
    kind, params = meta["camera"]["kind"], meta["camera"]["params"]
    if kind == "K":
        cam = torch.tensor([[[params[0], 0.0, params[2]], [0.0, params[1], params[3]], [0.0, 0.0, 1.0]]])
    else:
        cam = getattr(C, kind)(params=torch.tensor([params], dtype=torch.float32))
        assert C.pack_camera(cam) is not None
    out = subsample_like_golden(dict(m.infer(golden_rgb(meta["shape"], meta["seed"]), camera=cam)), meta)
    ref = {k: torch.from_numpy(z[k]) for k in z.files if k != "__meta__"}
    meas = MEASURED_GOLDEN[name]
    _check(out, ref, name, tol=dict(arel=MARGIN * meas[0], dmax=MARGIN * meas[1], k=MARGIN * meas[2]))
    e = (out["rays"].cpu() - ref["rays"]).abs().max().item()
    print(f"{name}: rays vs reference {e:.2e}")
    assert e < 1e-5, e


class _KernelRays:
    """A camera object the packer does not know, whose rays are the device ray generator's (ops.camera_rays) for the
    paddings and factor infer crops and resizes it by: the same rays the engine generates for `cam` itself, entering
    through the rays source instead of the camera-model source."""

    def __init__(self, cam):
        self.cam = copy.deepcopy(cam)

    def crop(self, left, top, right=None, bottom=None):
        self.pads = (-left, -right, -top, -bottom)
        return self

    def resize(self, factor):
        self.factor = factor
        return self

    def get_rays(self, shapes):
        b, nh, nw = shapes
        rays = _kernel_rays(self.cam, self.pads, self.factor, nh, nw, B=b, dev=_dev())
        return rays.view(b, nh, nw, 3).permute(0, 3, 1, 2)


@pytest.mark.parametrize("use_graph", [False, True])
def test_engine_equals_python_schedule(shallow, use_graph):
    """Camera-model source (rays generated inside udb_infer_v2) against the rays source fed with the same kernel's rays
    generated from Python: udb_infer_v2 shares everything downstream of the rays, so the outputs are bit-identical."""
    cfg, sd = shallow
    m = _model(cfg, sd)
    m.resolution_level = 3
    m.use_cuda_graph = use_graph
    rgb = _rgb((2, 96, 288), 8)
    for name in ("pinhole_skew", "eucm", "spherical", "opencv_strong", "fisheye_strong", "mei_strong"):
        cam = CAMERAS[name]()
        outs = [m.infer(rgb, camera=cam), m.infer(rgb, camera=_KernelRays(cam))]
        for k in outs[0]:
            assert torch.equal(outs[0][k], outs[1][k]), (name, k, use_graph)


def test_graph_replay_reuse_and_source_switching(shallow):
    cfg, sd = shallow
    m = _model(cfg, sd)
    m.resolution_level = None
    rgb = _rgb((2, 240, 320), 9)
    a, b = CAMERAS["fisheye_strong"](), CAMERAS["fisheye_strong"]()
    b.params[0, 0] *= 1.1
    b.params[0, 4] = 0.07
    K = torch.tensor([[[300.0, 0.0, 170.0], [0.0, 310.0, 115.0], [0.0, 0.0, 1.0]]])
    sources = {"none": None, "K": K, "object": a, "object2": b, "duck": _HostOnly(a), "eucm": CAMERAS["eucm"]()}
    m.use_cuda_graph = False
    eager = {k: (m.infer(rgb, camera=v) if v is not None else m.infer(rgb)) for k, v in sources.items()}
    m.use_cuda_graph = True
    n0 = len(m._graphs)
    assert n0 == 0
    seen = set()
    for k in ("object", "object2", "K", "none", "duck", "object", "eucm", "K", "object2", "none", "duck"):
        before = (a.params.clone(), b.params.clone())
        v = sources[k]
        out = m.infer(rgb, camera=v) if v is not None else m.infer(rgb)
        assert torch.equal(a.params, before[0]) and torch.equal(b.params, before[1])
        for key in out:
            assert torch.equal(out[key], eager[k][key]), (k, key)
        seen.add({"object2": "object", "duck": "rays"}.get(k, k))
        assert len(m._graphs) == len(seen), (k, len(m._graphs), seen)   # object / object2 share one entry
    assert not torch.equal(eager["object"]["rays"], eager["object2"]["rays"])
    assert not torch.equal(eager["object"]["rays"], eager["eucm"]["rays"])
    # network_forward(rgbs, rays) replays too, with fresh rays every call
    x = torch.randn(1, 3, 224, 308, generator=torch.Generator().manual_seed(3)).cuda()
    r1 = _class_rays(a, (0, 0, 0, 0), 1.0, 224, 308, "cuda").transpose(1, 2).reshape(1, 3, 224, 308)
    r2 = _class_rays(b, (0, 0, 0, 0), 1.0, 224, 308, "cuda").transpose(1, 2).reshape(1, 3, 224, 308)
    m.use_cuda_graph = False
    e1, e2 = m.network_forward(x, r1), m.network_forward(x, r2)
    m.use_cuda_graph = True
    n = len(m._graphs)
    g1, g2 = m.network_forward(x, r1), m.network_forward(x, r2)
    assert len(m._graphs) == n + 1
    for u, w in ((e1, g1), (e2, g2)):
        for s, t in zip(u, w):
            assert torch.equal(s, t)
