"""Host side of the GPU ray generator for camera objects (udb_camera_rays, include/udb.h): which objects are packed for
it and how, the crop / resize rule the kernel applies to a packed row, and the argument checks of udb_camera_rays and
of the engine's camera fields.  CPU only: the C calls run in a fresh interpreter with no visible GPU and fake device
pointers, so nothing can launch."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from unidepth_b200 import _cabi
from unidepth_b200 import camera as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "cameras.npz")

# name in cameras.npz -> (class, UDB_CAM_* id)
CASES = {"pinhole_params": ("Pinhole", _cabi.CAM_PINHOLE), "eucm": ("EUCM", _cabi.CAM_EUCM),
         "spherical": ("Spherical", _cabi.CAM_SPHERICAL), "opencv_radial": ("OPENCV", _cabi.CAM_OPENCV),
         "opencv_full": ("OPENCV", _cabi.CAM_OPENCV), "fisheye624": ("Fisheye624", _cabi.CAM_FISHEYE624),
         "fisheye624_radial": ("Fisheye624", _cabi.CAM_FISHEYE624), "mei": ("MEI", _cabi.CAM_MEI),
         "mei_plain": ("MEI", _cabi.CAM_MEI)}


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def _make(gold, name):
    return getattr(C, CASES[name][0])(params=torch.from_numpy(gold[f"{name}/params"]).clone())


# ------------------------------------------------------------------------------------------------------------ packing
@pytest.mark.parametrize("name", sorted(CASES))
def test_each_class_packs_to_its_model_params_and_flags(gold, name):
    cam = _make(gold, name)
    before = (cam.params.clone(), cam.K.clone())
    model, rows = C.pack_camera(cam)
    assert model == CASES[name][1] and rows.shape == (1, _cabi.CAM_STRIDE) and rows.dtype == torch.float32
    if name.startswith("pinhole"):
        assert torch.equal(rows[0, :9], cam.K.reshape(9)) and not rows[0, 9:].any()
    else:
        n = cam.params.shape[1]
        assert torch.equal(rows[0, :n], cam.params[0]) and not rows[0, n:16].any()
        flags = [float(getattr(cam, f, False)) for f in ("use_radial", "use_tangential", "use_thin_prism")]
        assert rows[0, 16:19].tolist() == flags, (name, rows[0, 16:].tolist())
    assert rows[0, 19] == 0
    assert torch.equal(cam.params, before[0]) and torch.equal(cam.K, before[1])       # not mutated


def test_flags_follow_the_class_decision():
    """A part whose coefficients sum to <= 1e-6 is off, as the class decides it once on its parameters."""
    p = torch.zeros(1, 16)
    p[0, :4] = torch.tensor([300.0, 300.0, 320.0, 240.0])
    p[0, 4] = 0.1                       # radial on
    p[0, 10] = 4e-7                     # tangential below the threshold: off
    p[0, 12:16] = 1e-3                  # thin prism on
    _, rows = C.pack_camera(C.Fisheye624(params=p))
    assert rows[0, 16:19].tolist() == [1.0, 0.0, 1.0]
    q = torch.tensor([[300.0, 300.0, 320.0, 240.0, 0.0, 0.0, 0.02, 0.0, 0.9]])
    _, rows = C.pack_camera(C.MEI(params=q))
    assert rows[0, 16:19].tolist() == [0.0, 1.0, 0.0]


def test_batch_camera_of_one_model_packs_one_row_per_member(gold):
    cams = [_make(gold, "eucm"), _make(gold, "eucm")]
    cams[1].params[0, 0] += 7.0
    batch = torch.cat([C.BatchCamera.from_camera(c) for c in cams])
    model, rows = C.pack_camera(batch)
    assert model == _cabi.CAM_EUCM and rows.shape == (2, _cabi.CAM_STRIDE)
    for i, c in enumerate(cams):
        assert torch.equal(rows[i], C.pack_camera(c)[1][0])
    # a batched K is one object with B rows
    K = torch.tensor([[[300.0, 0.0, 160.0], [0.0, 310.0, 120.0], [0.0, 0.0, 1.0]]]).repeat(3, 1, 1)
    K[1, 0, 0] = 280.0
    model, rows = C.pack_camera(C.BatchCamera.from_camera(C.Pinhole(K=K)))
    assert model == _cabi.CAM_PINHOLE and rows.shape == (3, _cabi.CAM_STRIDE)
    assert torch.equal(rows[:, :9], K.reshape(3, 9))


class _Duck:
    """Any object with crop / resize / get_rays (the reference's own classes look like this from here)."""

    def __init__(self):
        self.K = torch.tensor([[[200.0, 0.0, 22.0], [0.0, 200.0, 15.0], [0.0, 0.0, 1.0]]])

    def crop(self, left, top, right=None, bottom=None):
        self.K[..., 0, 2] -= left
        self.K[..., 1, 2] -= top
        return self

    def resize(self, factor):
        self.K[..., :2, :] *= factor
        return self

    def get_rays(self, shapes):
        return C.Pinhole(K=self.K).get_rays(shapes)


class _MyPinhole(C.Pinhole):
    pass


def _host_objects(gold):
    p16 = torch.from_numpy(gold["fisheye624/params"]).clone()
    p15 = torch.cat([p16[:, :1], p16[:, 2:]], dim=1)            # single focal length
    mixed = torch.cat([C.BatchCamera.from_camera(_make(gold, "pinhole_params")),
                       C.BatchCamera.from_camera(_make(gold, "eucm"))])
    return {"duck": _Duck(), "mixed_batch": mixed, "fisheye_15_params": C.Fisheye624(params=p15),
            "opencv_15_params": C.OPENCV(params=torch.cat([p15[:, :7], torch.zeros(1, 3), p15[:, 10:]], dim=1)),
            "subclass": _MyPinhole(params=torch.tensor([[200.0, 200.0, 22.0, 15.0]])),
            "float64": C.EUCM(params=torch.from_numpy(gold["eucm/params"]).double())}


def test_everything_else_keeps_the_host_path(gold):
    """pack_camera declines; `_camera_source` then produces host rays with the object's own methods, and the same call
    with a packable object produces the packed rows instead."""
    from unidepth_b200.unidepthv2 import UniDepthV2
    geom = {"paddings": (3, 3, 5, 5), "factor": 0.73, "net_hw": (30, 44)}
    cpu = torch.device("cpu")
    for name, obj in _host_objects(gold).items():
        assert C.pack_camera(obj) is None, name
        src, t = UniDepthV2._camera_source(obj, None, 2, geom, cpu)
        assert src == "rays" and t["rays"].shape == (2, 30 * 44, 3), name
    src, t = UniDepthV2._camera_source(_make(gold, "mei"), None, 2, geom, cpu)
    assert src == ("model", _cabi.CAM_MEI) and t["params"].shape == (2, _cabi.CAM_STRIDE)
    assert torch.equal(t["params"][0], t["params"][1])                     # one camera, broadcast to the batch
    src, t = UniDepthV2._camera_source(torch.eye(3)[None], None, 2, geom, cpu)
    assert src == "K" and t["K"].shape == (2, 3, 3)
    assert UniDepthV2._camera_source(None, None, 2, geom, cpu) == (None, {})
    two = torch.cat([C.BatchCamera.from_camera(_make(gold, "eucm")) for _ in range(2)])
    with pytest.raises(ValueError, match="2 cameras for a batch of 3"):
        UniDepthV2._camera_source(two, None, 3, geom, cpu)


# ------------------------------------------------------------------------------------------------------- crop / resize
def _kernel_crop_resize(model, rows, pads, factor):
    """The rule udb_camera_rays applies to a packed row, restated in fp32 torch (camera.cu crop_resize)."""
    pl, pr, pt, pb = pads
    q = rows.clone()
    if model == _cabi.CAM_PINHOLE:
        q[:, 2] = q[:, 2] + pl
        q[:, 5] = q[:, 5] + pt
        q[:, :6] = q[:, :6] * factor
        return q
    q[:, 2] = q[:, 2] + pl
    q[:, 3] = q[:, 3] + pt
    if model == _cabi.CAM_SPHERICAL:
        W, H = q[:, 4].clone(), q[:, 5].clone()
        keep_w, keep_h = (W + pl + pr) / W, (H + pt + pb) / H
        q[:, 4] = W + (pl + pr)
        q[:, 5] = H + (pt + pb)
        q[:, 6] = q[:, 6] * keep_w
        q[:, 7] = q[:, 7] * keep_h
        q[:, :6] = q[:, :6] * factor
        return q
    q[:, :4] = q[:, :4] * factor
    return q


@pytest.mark.parametrize("name", sorted(CASES))
def test_crop_resize_rule_equals_the_class(gold, name):
    for pads in ((0, 0, 0, 0), (7, 9, 0, 0), (0, 0, 11, 4), (3, 3, 5, 5)):
        for factor in (0.73, 1.6):
            cam = _make(gold, name)
            model, rows = C.pack_camera(cam)
            pl, pr, pt, pb = pads
            edited = C.BatchCamera.from_camera(_make(gold, name)).crop(left=-pl, top=-pt, right=-pr, bottom=-pb)
            _, want = C.pack_camera(edited.resize(factor))
            got = _kernel_crop_resize(model, rows, pads, factor)
            assert torch.equal(got[:, :16], want[:, :16]), (name, pads, factor, got[:, :16], want[:, :16])
    if name == "spherical":       # the field of view follows the padding
        _, a = C.pack_camera(_make(gold, name))
        assert _kernel_crop_resize(_cabi.CAM_SPHERICAL, a, (10, 10, 0, 0), 1.0)[0, 6] > a[0, 6]


# ---------------------------------------------------------------------------------------------------------------- ABI
BASE = 1 << 28


def _child_main():
    """Runs in a fresh interpreter with no visible GPU; prints one JSON dict of results."""
    import ctypes as Ct
    lib = _cabi.lib()
    res = {}

    def rec(name, fn):
        n0 = lib.udb_launch_count()
        rc = fn()
        res[name] = {"rc": rc, "msg": lib.udb_last_error().decode(), "launched": lib.udb_launch_count() - n0}

    good = dict(model=_cabi.CAM_FISHEYE624, params=BASE, B=2, net_h=28, net_w=42, rays=BASE + (1 << 22))
    cases = {"model0": dict(good, model=0), "model7": dict(good, model=7), "model-1": dict(good, model=-1),
             "params_null": dict(good, params=0), "params_misaligned": dict(good, params=BASE + 4),
             "rays_null": dict(good, rays=0), "rays_misaligned": dict(good, rays=BASE + 2), "B0": dict(good, B=0),
             "net_h0": dict(good, net_h=0), "net_w0": dict(good, net_w=0), "valid": good}
    for name, a in cases.items():
        rec("rays:" + name, lambda a=a: lib.udb_camera_rays(a["model"], a["params"], a["B"], a["net_h"], a["net_w"],
                                                            1, 2, 3, 4, 0.5, a["rays"], None))

    cfg = _cabi.Config()
    cfg.embed_dim, cfg.depth, cfg.enc_heads, cfg.pos_grid = 384, 12, 6, 37
    for i, t in enumerate((3, 6, 9, 12)):
        cfg.taps[i] = t
    cfg.hidden, cfg.dec_heads, cfg.expansion, cfg.out_dim, cfg.n_stages = 256, 8, 4, 32, 3
    for i in range(3):
        cfg.dec_depths[i] = 2
    cfg.ratio_min, cfg.ratio_max, cfg.pixels_min, cfg.pixels_max = 0.5, 2.5, 200000.0, 600000.0
    h = Ct.c_void_p()
    assert lib.udb_create(Ct.byref(cfg), Ct.byref(h)) == 0
    infer = {"model9": dict(camera_model=9, camera_params=BASE), "model-1": dict(camera_model=-1, camera_params=BASE),
             "params_null": dict(camera_model=1), "params_misaligned": dict(camera_model=1, camera_params=BASE + 8),
             "with_k": dict(camera_model=2, camera_params=BASE, camera_k=BASE + 64),
             "with_rays": dict(camera_model=2, camera_params=BASE, camera_rays=BASE + 128),
             "valid": dict(camera_model=6, camera_params=BASE)}
    for name, extra in infer.items():
        a = _cabi.InferArgs()
        a.rgb, a.workspace, a.workspace_bytes = BASE, BASE + (1 << 24), 1 << 20
        a.B, a.H, a.W, a.resolution_level = 1, 120, 160, -1
        for i, f in enumerate(("confidence", "intrinsics", "radius", "depth", "points", "rays", "depth_features")):
            setattr(a, f, BASE + (1 << 25) + i * (1 << 22))
        for k, v in extra.items():
            setattr(a, k, v)
        rec("infer:" + name, lambda a=a: lib.udb_infer_v2(h, Ct.byref(a), None))
    lib.udb_destroy(h)
    json.dump(res, sys.stdout)


@pytest.fixture(scope="module")
def abi():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    code = "import sys; sys.path[:0] = ['tests']; import test_camera_kernel_cpu as t; t._child_main()"
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, check=True).stdout
    return json.loads(out)


@pytest.mark.parametrize("case,field", [("model0", "`model`"), ("model7", "`model`"), ("model-1", "`model`"),
                                        ("params_null", "`params`"), ("params_misaligned", "`params`"),
                                        ("rays_null", "`rays`"), ("rays_misaligned", "`rays`"), ("B0", "B=0"),
                                        ("net_h0", "net_h=0"), ("net_w0", "net_w=0")])
def test_camera_rays_rejects_before_launch(abi, case, field):
    r = abi["rays:" + case]
    print(case, r)
    assert r["rc"] != 0 and field in r["msg"] and r["launched"] == 0, r
    assert "CUDA" not in r["msg"] and "device" not in r["msg"], r


@pytest.mark.parametrize("case,fields", [("model9", ["`camera_model`"]), ("model-1", ["`camera_model`"]),
                                         ("params_null", ["`camera_params`"]), ("params_misaligned", ["`camera_params`"]),
                                         ("with_k", ["`camera_model`", "`camera_k`"]),
                                         ("with_rays", ["`camera_model`", "`camera_rays`"])])
def test_infer_rejects_camera_fields_before_launch(abi, case, fields):
    r = abi["infer:" + case]
    print(case, r)
    assert r["rc"] != 0 and r["launched"] == 0, r
    for f in fields:
        assert f in r["msg"], (f, r)


def test_valid_camera_calls_get_past_the_checks(abi):
    r = abi["rays:valid"]
    assert r["rc"] != 0 and r["launched"] == 0 and "`" not in r["msg"], r            # only the launch itself fails
    r = abi["infer:valid"]
    assert r["rc"] != 0 and "not prepared" in r["msg"] and r["launched"] == 0, r


def test_schedule_bytes_hold_the_generated_rays():
    """The dry run walks the camera stage with the real packed operands: the workspace it sizes holds the generated
    [B, net_h*net_w, 3] rays on top of everything the schedule needs anyway."""
    import ctypes as Ct
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_engine_schedule_cpu import _v2, _v2_engine
    lib = _cabi.lib()
    h, keep = _v2_engine(_v2("config_v2_vits14.json"))
    try:
        g = _cabi.Geometry()
        for B, H, W in ((1, 480, 640), (8, 480, 640), (2, 96, 288)):
            assert lib.udb_geometry(h, H, W, -1, Ct.byref(g)) == 0
            n, rays = lib.udb_schedule_bytes(h, B, H, W, -1), B * g.net_h * g.net_w * 12
            print(B, H, W, n, rays)
            assert n > rays, (B, H, W, n, rays)
    finally:
        lib.udb_destroy(h)
