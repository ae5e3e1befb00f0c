"""UniDepthV2old.forward (the reference's evaluation call, model(inputs, image_metas)) without a GPU: the argument checks
that run before anything touches the device, the engine's named refusals of a network-only call (checked before any
launch), the C layout of the two structs the mode extends, and, from the stored goldens alone
(tests/golden/v2oldfwd_*.npz, oracle/make_golden_v2old_forward.py), the rule that `forward`'s points use the predicted K
on the ground truth's grid."""
import ctypes as C
import glob
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from make_golden_v2old import make_v2old_state_dict  # noqa: E402
from unidepth_b200 import UniDepthV2old, _cabi  # noqa: E402

CPU = torch.device("cpu")
FWD_GOLDENS = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "v2oldfwd_*.npz")))


def _cfg(bb):
    return json.load(open(os.path.join(GOLDEN, f"config_v2old_{bb}.json")))


def _inputs(B=1, h=294, w=392, H=None, W=None, K=None):
    d = {"image": torch.zeros(B, 3, h, w), "depth": torch.zeros(B, 1, H or h, W or w)}
    if K is not None:
        d["K"] = K
    return d


def test_forward_argument_errors_before_the_device():
    m = UniDepthV2old(_cfg("vits14"))
    # a new module is in training mode: the training forward is out of scope
    with pytest.raises(NotImplementedError, match="eval mode"):
        m(_inputs(), None)
    m.eval()
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 3, 294, 392), None)
    with pytest.raises(ValueError, match="multiples of the patch size"):
        m(_inputs(h=300, w=392), None)
    with pytest.raises(ValueError, match="multiples of the patch size"):
        m(_inputs(h=294, w=400), None)
    with pytest.raises(ValueError, match="'depth'"):
        m({"image": torch.zeros(1, 3, 294, 392)}, None)
    with pytest.raises(ValueError, match="float"):
        m({"image": torch.zeros(1, 3, 294, 392, dtype=torch.uint8), "depth": torch.zeros(1, 1, 294, 392)}, None)
    with pytest.raises(ValueError, match=r"\[B, 3, 3\]"):
        m(_inputs(K=torch.eye(3)), None)
    with pytest.raises(ValueError, match=r"\[B, 3, 3\]"):
        m(_inputs(B=2, K=torch.eye(3).repeat(1, 1, 1)), None)
    with pytest.raises(ValueError, match="must be equal"):
        m(_inputs(H=480, W=640, K=torch.eye(3)[None]), None)
    # valid arguments reach the device check: this model is on the CPU
    with pytest.raises(RuntimeError, match="CUDA device"):
        m(_inputs(H=480, W=640), None)
    with pytest.raises(RuntimeError, match="CUDA device"):
        m(_inputs(K=torch.eye(3)[None]), {"anything": 1})


def _args(B, H, W, **kw):
    """udb_infer_v2old arguments whose pointers are never dereferenced: every call below is refused before any launch."""
    a = _cabi.InferV2oldArgs()
    a.rgb, a.workspace, a.workspace_bytes = 16, 16, 1 << 20
    a.out_intrinsics = a.out_points = a.out_depth = a.out_confidence = 16
    a.B, a.H, a.W = B, H, W
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_engine_refuses_bad_network_only_calls():
    lib = _cabi.lib()
    cfg = _cfg("vits14")
    m = UniDepthV2old(cfg)
    m.load_state_dict(make_v2old_state_dict(cfg, 0), strict=True)
    shape = (294, 392)
    T, S = m._pack_tensors(CPU, shape)
    h = C.c_void_p()
    _cabi.check(lib.udb_v2old_create(C.byref(m._engine_config(shape)), C.byref(h)), "udb_v2old_create")
    try:
        m._register(h, T, S)
        assert lib.udb_v2old_schedule_bytes(h, 2, *shape) > 0, lib.udb_last_error()
        cases = [
            (_args(1, 280, 392, network_only=1, out_h=280, out_w=392), b"network-only input is 280x392 but the engine's network shape is 294x392"),
            (_args(1, 294, 406, network_only=1, out_h=294, out_w=406), b"network shape is 294x392"),
            (_args(1, 294, 392, network_only=1, out_h=294, out_w=392, rgb_is_u8=1), b"must be f32 and already normalised"),
            (_args(1, 294, 392, network_only=1, out_h=294, out_w=392, normalize=1), b"must be f32 and already normalised"),
            (_args(1, 294, 392, network_only=1, out_h=294, out_w=392, scale255=1), b"must be f32 and already normalised"),
            (_args(1, 294, 392, network_only=1, out_h=0, out_w=392), b"output size 0x392"),
            (_args(1, 294, 392, network_only=1, out_h=480, out_w=640, intrinsics=16), b"a given K needs the output size 480x640"),
            (_args(1, 294, 392, network_only=2, out_h=294, out_w=392), b"`network_only` 2"),
            (_args(1, 294, 392, out_h=480, out_w=640), b"network-only mode only"),
            (_args(1, 294, 392, out_depth_features=16), b"network-only mode only"),
        ]
        for a, msg in cases:
            assert lib.udb_infer_v2old(h, C.byref(a), None) != 0
            assert msg in lib.udb_last_error(), (msg, lib.udb_last_error())
        # a valid network-only call gets past these checks and stops at the workspace, which no dry run has prepared
        a = _args(1, 294, 392, network_only=1, out_h=480, out_w=640, interpolation=7)
        assert lib.udb_infer_v2old(h, C.byref(a), None) != 0
        assert b"udb_v2old_workspace_bytes" in lib.udb_last_error(), lib.udb_last_error()
    finally:
        lib.udb_v2old_destroy(h)


def test_extended_structs_match_c_layout():
    structs = {"udb_infer_v2old_args_t": (_cabi.InferV2oldArgs, "out_depth_features"),
               "udb_v2old_postprocess_t": (_cabi.V2oldPostprocess, "depth_aa")}
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "udb.h"\nint main(){\n'
    for n, (_, last) in structs.items():
        src += f'printf("{n} %zu %zu\\n", sizeof({n}), offsetof({n}, {last}));\n'
    src += "return 0;}\n"
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        out = subprocess.check_output([os.path.join(d, "t")], text=True)
    for line in out.strip().splitlines():
        n, size, off = line.split()
        cs, last = structs[n]
        assert cs._fields_[-1][0] == last
        assert C.sizeof(cs) == int(size), (n, C.sizeof(cs), size)
        assert getattr(cs, last).offset == int(off), n


def test_forward_goldens_are_present():
    assert len(FWD_GOLDENS) == 10, FWD_GOLDENS
    for name in FWD_GOLDENS:
        assert 50e3 < os.path.getsize(os.path.join(GOLDEN, name + ".npz")) < 300e3, name


@pytest.mark.parametrize("name", FWD_GOLDENS)
def test_golden_points_use_the_predicted_K_on_the_gt_grid(name):
    """The stored points equal spherical_zbuffer_to_euclidean(generate_rays(stored K, (H, W)), stored depth) at the
    sampled pixels, restated in float64 numpy: the predicted K, unscaled, on the ground truth's grid, also where a GT K
    was given."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["__meta__"]))
    H, W = meta["gt_hw"]
    sp, sd = meta["strides"]["points"], meta["strides"]["depth"]
    K = z["K"].astype(np.float64)
    pts = z["points"].astype(np.float64)
    depth = z["depth"].astype(np.float64)[:, 0, ::sp // sd, ::sp // sd]
    ys, xs = np.meshgrid(np.arange(0, H, sp) + 0.5, np.arange(0, W, sp) + 0.5, indexing="ij")
    assert pts.shape[2:] == ys.shape == depth.shape[1:]
    for b in range(K.shape[0]):
        fx, fy, cx, cy = K[b, 0, 0], K[b, 1, 1], K[b, 0, 2], K[b, 1, 2]
        r = np.stack([(xs - cx) / fx, (ys - cy) / fy, np.ones_like(xs)])
        r /= np.linalg.norm(r, axis=0)
        theta, phi = np.arctan2(r[0], r[2]), np.arccos(r[1])
        d = depth[b]
        ref = np.stack([d * np.tan(theta), d / np.tan(phi) / np.cos(theta), d])
        assert np.max(np.abs(pts[b] - ref) / d) < 1e-4, name
    if meta["with_k"]:
        # the rule has teeth: the given K differs from the prediction
        assert np.max(np.abs(z["K_in"] - z["K"]) / z["K_in"].max()) > 1e-2


@pytest.mark.skipif(not os.path.isdir("/root/reference/unidepth"), reason="needs the reference sources")
def test_oracle_reproduces_a_forward_golden():
    """The generator's recipe (the unmodified reference's `forward` + the Nystrom restatement) reproduces a stored golden."""
    import copy
    import warnings
    sys.path[:0] = ["/root/reference", os.path.join(ROOT, "oracle", "ref_shims")]
    warnings.simplefilter("ignore")
    import unidepth.layers.nystrom_attention as NA
    from make_golden_v1 import OracleNystrom
    from make_golden_v2old_forward import CASES, network_input
    NA.NystromAttention = OracleNystrom
    from unidepth.models.unidepthv2.unidepthv2_old import UniDepthV2old as Ref
    name = "v2oldfwd_vits14_down_420x560_240x320"
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["__meta__"]))
    case = next(c for c in CASES if name.endswith(c[0]))
    cfg = _cfg("vits14")
    ref = Ref(copy.deepcopy(cfg)).eval()
    ref.load_state_dict(make_v2old_state_dict(cfg, meta["seed"]), strict=True)
    with torch.no_grad():
        out = ref({"image": network_input(case[2], case[1]), "depth": torch.zeros(1, 1, *case[3])}, None)
    s = meta["strides"]["depth"]
    np.testing.assert_allclose(out["depth"][:, :, ::s, ::s].numpy(), z["depth"], rtol=1e-5)
    np.testing.assert_allclose(out["K"].numpy(), z["K"], rtol=1e-5)
