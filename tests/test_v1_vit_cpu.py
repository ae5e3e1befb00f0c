"""UniDepthV1 with the DINOv2 ViT-L/14 encoder (config_v1_vitl14.json), host side, no GPU:
  - the fp32 oracle (oracle/unidepth_v1_vit_oracle.py) against the unmodified reference's outputs (tests/golden/v1_vitl14_*.npz,
    oracle/make_golden_v1_vit.py) at the V1 bar;
  - the packer against the engine's dry-run schedule (names, shapes, workspace sizing; nothing is launched);
  - the spec: which encoders V1 accepts, and the pack-time position table against the oracle's."""
import copy
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from unidepth_b200 import UniDepthV1, _cabi
from unidepth_b200.spec_v1 import V1Spec, param_shapes

CPU = torch.device("cpu")
V1_VIT_CASES = ["v1_vitl14_480x640", "v1_vitl14_gtK_375x1242"]


def _cfg(golden_dir):
    return json.load(open(os.path.join(golden_dir, "config_v1_vitl14.json")))


def v1_vit_case_inputs(golden_dir, name):
    """(config, state dict, rgb, K or None, meta, golden arrays) of one tests/golden/v1_vitl14_*.npz case."""
    from unidepth_v1_vit_oracle import make_v1_vit_state_dict
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    meta = json.loads(str(z["__meta__"]))
    cfg = json.load(open(os.path.join(golden_dir, meta["config"])))
    g = torch.Generator().manual_seed(4321 + meta["seed"])
    b, h, w = meta["shape"]
    rgb = torch.randint(0, 256, (b, 3, h, w), dtype=torch.uint8, generator=g)
    K = torch.from_numpy(z["K_in"]) if meta["with_k"] else None
    return cfg, make_v1_vit_state_dict(cfg, meta["seed"]), rgb, K, meta, z


def like_golden(t, key, meta):
    """The sub-sampling oracle/make_golden_v1_vit.py applied to the stored `depth` / `points` maps."""
    s = meta["strides"].get(key, 1)
    return t[:, :, ::s, ::s] if t.ndim == 4 else t


@pytest.mark.parametrize("name", V1_VIT_CASES)
def test_v1_vit_oracle_matches_reference_golden(name, golden_dir):
    import unidepth_v1_vit_oracle as OV
    cfg, sd, rgb, K, meta, z = v1_vit_case_inputs(golden_dir, name)
    out = OV.infer_v1_vit(sd, cfg, rgb, K, skip_camera=meta["skip_camera"])
    assert set(out) == {"intrinsics", "points", "depth"}
    for k in ("intrinsics", "depth", "points"):
        ref = torch.from_numpy(z[k])
        got = like_golden(out[k], k, meta)
        assert got.shape == ref.shape, (k, got.shape, ref.shape)
        floor = 0.1 * ref.abs().mean().item()
        err = ((got - ref).abs() / ref.abs().clamp(min=floor)).max().item()
        print(name, k, "max rel err", err)
        assert err < 5e-5, (k, err)


def _model(golden_dir, seed=None):
    cfg = _cfg(golden_dir)
    m = UniDepthV1(copy.deepcopy(cfg)).eval()
    if seed is not None:
        from unidepth_v1_vit_oracle import make_v1_vit_state_dict
        m.load_state_dict(make_v1_vit_state_dict(cfg, seed), strict=True)
    return m


def _engine(m, T, S):
    h = C.c_void_p()
    _cabi.check(_cabi.lib().udb_v1_create(C.byref(m._engine_config()), C.byref(h)), "udb_v1_create")
    m._register(h, T, S)
    return h


def test_v1_vit_packer_and_schedule_agree(golden_dir):
    lib = _cabi.lib()
    m = _model(golden_dir)
    T, S = m._pack_tensors(CPU)
    assert T["patch_w"].shape == (1024, 640) and T["pos"].shape == (1 + 33 * 44, 1024)
    assert T["tokens_pos"].shape == (4 * 33 * 44, 512)
    assert not any(k.startswith(("stem", "s0.", "ds")) for k in T)       # no ConvNeXt operand
    h = _engine(m, T, S)
    try:
        sizes = {}
        for B in (1, 4, 16):
            for H, W in ((480, 640), (375, 1242), (1000, 400)):
                n = lib.udb_v1_workspace_bytes(h, B, H, W)
                assert n > 0, (B, H, W, lib.udb_last_error().decode())
                sizes[(B, H, W)] = n
        assert sizes[(1, 480, 640)] < sizes[(4, 480, 640)] < sizes[(16, 480, 640)]
        # the network input is fixed: the workspace does not depend on the image shape
        assert sizes[(4, 480, 640)] == sizes[(4, 375, 1242)] == sizes[(4, 1000, 400)]
        assert lib.udb_v1_workspace_bytes(h, 0, 480, 640) == 0
        a = _cabi.InferV1Args()
        assert lib.udb_infer_v1(h, C.byref(a), None) != 0                   # a dry run launches nothing and prepares no call
    finally:
        lib.udb_v1_destroy(h)
    del T


def test_v1_vit_schedule_names_the_missing_operand(golden_dir):
    lib = _cabi.lib()
    m = _model(golden_dir)
    T, S = m._pack_tensors(CPU)
    names = list(T)
    picks = {"patch_w", "patch_b", "cls", "pos", "blocks.0.qkv_w", "blocks.23.ls2", "tokens_pos"}
    picks |= set(names[:: max(1, len(names) // 10)])
    for name in sorted(picks):
        h = _engine(m, {k: v for k, v in T.items() if k != name}, S)
        try:
            assert lib.udb_v1_workspace_bytes(h, 1, 480, 640) == 0, name
            assert name in lib.udb_last_error().decode(), (name, lib.udb_last_error().decode())
        finally:
            lib.udb_v1_destroy(h)
    # a position table for another grid is refused by shape, not read out of bounds
    bad = dict(T)
    bad["pos"] = T["pos"][:-44].contiguous()
    h = _engine(m, bad, S)
    try:
        assert lib.udb_v1_workspace_bytes(h, 1, 480, 640) == 0
        assert "'pos'" in lib.udb_last_error().decode(), lib.udb_last_error().decode()
    finally:
        lib.udb_v1_destroy(h)


def test_v1_spec_encoders(golden_dir):
    cfg = _cfg(golden_dir)
    s = V1Spec(cfg)
    assert s.depths == (5, 7, 6, 6) and s.dims == (1024,) * 4 and s.output_idx == (5, 12, 18, 24)
    assert s.cls_dims == (1024,) * 4 and s.common_grid() == (33, 44)
    for name in ("dinov2_vits14", "dinov2_vitb14", "convnext2_large", "convnext2"):
        c = copy.deepcopy(cfg)
        c["model"]["pixel_encoder"]["name"] = name
        with pytest.raises(NotImplementedError):
            V1Spec(c)
    c = copy.deepcopy(cfg)
    c["data"]["image_shape"] = [460, 616]
    with pytest.raises(NotImplementedError):
        V1Spec(c)
    # the ConvNeXt table is untouched: 196.2 M parameters in the shipped ConvNeXt-L config
    cn = json.load(open(os.path.join(golden_dir, "config_v1_cnvnxtl.json")))
    assert V1Spec(cn).common_grid() == (28, 38)
    shapes = param_shapes(cfg)
    assert shapes["pixel_encoder.pos_embed"] == (1, 1370, 1024) and "pixel_encoder.stem.0.weight" not in shapes


def test_v1_vit_pack_time_position_table_matches_oracle(golden_dir):
    """The engine's "pos" operand (offset-0.1 bicubic resize folded at pack time) equals the oracle's position table,
    which the reference goldens pin."""
    from unidepth_v1_vit_oracle import interpolate_pos_embed_offset
    m = _model(golden_dir, seed=0)
    T, _ = m._pack_tensors(CPU)
    ref = interpolate_pos_embed_offset(m.state_dict()["pixel_encoder.pos_embed"].float(), 33, 44)[0]
    assert torch.equal(T["pos"], ref)
    # and it is NOT the offset-0 (size=) resize V2 uses: the two differ well above rounding
    import torch.nn.functional as F
    grid = m.state_dict()["pixel_encoder.pos_embed"][0, 1:].reshape(1, 37, 37, 1024).permute(0, 3, 1, 2)
    v2 = F.interpolate(grid, size=(33, 44), mode="bicubic", antialias=False).permute(0, 2, 3, 1).reshape(-1, 1024)
    assert float((v2 - ref[1:]).abs().max()) > 1e-3
