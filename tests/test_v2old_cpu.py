"""UniDepthV2old without a GPU: the parameter table against the reference model's, the shape arithmetic of `infer` against
the reference's own functions (tests/golden/v2old_geometry.npz), the contract between the Python packer and the C
schedule (a dry run of udb_v2old_schedule_bytes, which walks every stage and launches nothing), hubconf, and the oracle
reproducing the goldens when the reference is at hand."""
import ctypes as C
import json
import os
import sys
import warnings

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from make_golden_v2old import geometry_grid, make_v2old_state_dict  # noqa: E402
from unidepth_b200 import UniDepthV2old, _cabi  # noqa: E402
from unidepth_b200.spec_v2old import check_ratio, check_resolution, param_shapes  # noqa: E402
from unidepth_b200.unidepthv2old import v2old_geometry  # noqa: E402

CPU = torch.device("cpu")
BACKBONES = ("vitl14", "vits14")


def _cfg(bb):
    return json.load(open(os.path.join(GOLDEN, f"config_v2old_{bb}.json")))


@pytest.mark.parametrize("bb", BACKBONES)
def test_state_dict_names_and_shapes_load_strict(bb):
    """The module's parameters are the spec's table (which the golden generator asserts equals the reference model's
    state dict), and the seeded fixture loads with strict=True."""
    cfg = _cfg(bb)
    m = UniDepthV2old(cfg)
    mine = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert mine == dict(param_shapes(cfg))
    m.load_state_dict(make_v2old_state_dict(cfg, 0), strict=True)
    d = 1024 if bb == "vitl14" else 384
    assert mine["pixel_decoder.input_adapter.input_adapters.0.1.weight"] == (512, d)
    assert mine["pixel_decoder.depth_layer.to_depth.weight"] == (1, 48, 7, 7)
    assert mine["pixel_decoder.global_layer.project_rays.weight"] == (512, 99)
    with pytest.raises(NotImplementedError):
        m.forward({}, {})


def test_geometry_matches_the_reference_functions():
    """Network shape, ratio and pixel count of ~1000 input shapes x resolution levels (None, clipped, in range) against
    the reference's `_check_resolution` / `_shapes`, and the warnings each one raises."""
    z = np.load(os.path.join(GOLDEN, "v2old_geometry.npz"))
    grid = geometry_grid()
    assert len(grid) == len(z["hw"])
    bounds = (1400, 2400)
    for i, (h, w, lv) in enumerate(grid):
        assert (h, w) == tuple(z["hw"][i]) and (-1 if lv is None else lv) == z["level"][i]
        with warnings.catch_warnings(record=True) as ws:
            warnings.simplefilter("always")
            level = check_resolution(lv)
            n_res = len(ws)
            check_ratio((h, w), (0.66, 2.0))
            n_ratio = len(ws) - n_res
        assert (n_res, n_ratio) == tuple(z["warnings"][i]), (h, w, lv)
        (nh, nw), ratio = v2old_geometry(h, w, level, bounds)
        assert (nh, nw) == tuple(z["net_hw"][i]) and ratio == z["ratio"][i], (h, w, lv, nh, nw, ratio)
        g = _cabi.V2oldGeometry()
        _cabi.check(_cabi.lib().udb_v2old_geometry(h, w, level, *bounds, C.byref(g)), "geometry")
        assert g.pixels == z["pixels"][i]
    assert _cabi.lib().udb_v2old_geometry(0, 10, 0, *bounds, C.byref(_cabi.V2oldGeometry())) != 0


def _engine(m, tensors, scalars, shape):
    h = C.c_void_p()
    _cabi.check(_cabi.lib().udb_v2old_create(C.byref(m._engine_config(shape)), C.byref(h)), "udb_v2old_create")
    m._register(h, tensors, scalars)
    return h


@pytest.mark.parametrize("bb", BACKBONES)
def test_packer_and_schedule_agree(bb):
    """The dry run accepts the packer's operands at two network shapes and batch sizes, and each operand the packer
    produces is one the schedule reads: without it, the dry run fails naming it."""
    lib = _cabi.lib()
    cfg = _cfg(bb)
    m = UniDepthV2old(cfg)
    m.load_state_dict(make_v2old_state_dict(cfg, 0), strict=True)
    for H, W, B in ((480, 640, 1), (375, 1242, 3)):
        shape, _ = v2old_geometry(H, W, 10, (1400, 2400))
        T, S = m._pack_tensors(CPU, shape)
        h = _engine(m, T, S, shape)
        try:
            n = lib.udb_v2old_schedule_bytes(h, B, H, W)
            assert n > 0, lib.udb_last_error().decode()
        finally:
            lib.udb_v2old_destroy(h)
    shape, _ = v2old_geometry(480, 640, 10, (1400, 2400))
    T, S = m._pack_tensors(CPU, shape)
    # every decoder operand, and the encoder's first and last block (ViT-L's middle blocks are the same loop)
    last = m.spec.enc_depth - 1
    names = [k for k in T if not k.startswith("blocks.") or k.startswith(("blocks.0.", f"blocks.{last}."))]
    for name in names:
        h = _engine(m, {k: v for k, v in T.items() if k != name}, S, shape)
        try:
            assert lib.udb_v2old_schedule_bytes(h, 1, 480, 640) == 0, name
            assert f"'{name}'" in lib.udb_last_error().decode(), (name, lib.udb_last_error())
        finally:
            lib.udb_v2old_destroy(h)
    for sname in S:
        h = _engine(m, T, {k: v for k, v in S.items() if k != sname}, shape)
        try:
            assert lib.udb_v2old_schedule_bytes(h, 1, 480, 640) == 0 and f"'{sname}'" in lib.udb_last_error().decode()
        finally:
            lib.udb_v2old_destroy(h)


def test_engine_rejects_bad_configs_and_small_shapes():
    lib = _cabi.lib()
    m = UniDepthV2old(_cfg("vits14"))
    h = C.c_void_p()
    cfg = m._engine_config((588, 784))
    cfg.hidden = 256
    assert lib.udb_v2old_create(C.byref(cfg), C.byref(h)) != 0 and b"hidden 256" in lib.udb_last_error()
    cfg = m._engine_config((588, 785))
    assert lib.udb_v2old_create(C.byref(cfg), C.byref(h)) != 0 and b"multiples of 14" in lib.udb_last_error()
    cfg = m._engine_config((140, 126))                 # 10 x 9 patches: fewer tokens than Nystrom's 128 landmarks
    _cabi.check(lib.udb_v2old_create(C.byref(cfg), C.byref(h)), "udb_v2old_create")
    try:
        assert lib.udb_v2old_schedule_bytes(h, 1, 140, 126) == 0 and b"128 landmarks" in lib.udb_last_error()
    finally:
        lib.udb_v2old_destroy(h)


def test_hubconf_builds_both_backbones_offline():
    sys.path.insert(0, ROOT)
    import hubconf
    for bb, d in (("vitl14", 1024), ("vits14", 384)):
        m = hubconf.UniDepth("v2old", bb, pretrained=False)
        assert isinstance(m, UniDepthV2old) and m.spec.embed_dim == d
        assert m.interpolation_mode == "bilinear" and m.resolution_level is None
        assert m.shape_constraints["pixels_bounds_ori"] == [1400, 2400]


@pytest.mark.skipif(not os.path.isdir("/root/reference/unidepth"), reason="needs the reference sources")
def test_oracle_reproduces_a_golden():
    """The generator's recipe (unmodified reference + the Nystrom restatement) reproduces a stored golden."""
    import copy
    sys.path[:0] = ["/root/reference", os.path.join(ROOT, "oracle", "ref_shims")]
    warnings.simplefilter("ignore")
    import unidepth.layers.nystrom_attention as NA
    from make_golden_v1 import OracleNystrom, seeded_rgb
    NA.NystromAttention = OracleNystrom
    from unidepth.models.unidepthv2.unidepthv2_old import UniDepthV2old as Ref
    z = np.load(os.path.join(GOLDEN, "v2old_vits14_rl0_360x480.npz"))
    meta = json.loads(str(z["__meta__"]))
    cfg = _cfg("vits14")
    ref = Ref(copy.deepcopy(cfg)).eval()
    ref.load_state_dict(make_v2old_state_dict(cfg, meta["seed"]), strict=True)
    ref.resolution_level = meta["resolution_level"]
    with torch.no_grad():
        out = ref.infer(seeded_rgb(tuple(meta["shape"]), meta["seed"]))
    np.testing.assert_allclose(out["depth"][:, :, ::4, ::4].numpy(), z["depth"], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(out["intrinsics"].numpy(), z["intrinsics"], rtol=1e-5)
