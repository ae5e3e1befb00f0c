"""UniDepthV1 at network shapes other than the config's (`model.image_shape`), without a GPU:
  - the oracles against the unmodified reference run at those shapes (tests/golden/v1_*_net*.npz, made by
    oracle/make_golden_v1_shapes.py);
  - the engine's dry run over a sweep of shapes per encoder, on a CPU packing with `image_shape` set: every operand is
    found with the right shape, or the one bound the grid breaks is named;
  - the two shape operands ("tokens_pos", "pos") against the oracle's tables;
  - the shapes `infer` refuses, before anything is packed or launched."""
import copy
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from unidepth_b200 import UniDepthV1, _cabi

CPU = torch.device("cpu")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# (golden, oracle module): ConvNeXt-L at 384x512, 470x630 (stem and downsample floors that do not divide evenly) and
# 448x448 (square); ViT-L/14 at 378x504 (27x36 patches), 518x686 (37x49) and 448x448 (32x32)
SHAPE_CASES = ["v1_cnvnxtl_net384x512_480x640", "v1_cnvnxtl_net470x630_480x640", "v1_cnvnxtl_net470x630_gtK_375x1242",
               "v1_cnvnxtl_net448x448_480x640", "v1_vitl14_net378x504_480x640", "v1_vitl14_net518x686_480x640",
               "v1_vitl14_net518x686_gtK_375x1242", "v1_vitl14_net448x448_480x640"]


def shape_case(name):
    """(config with the case's image_shape, state dict, rgb, K or None, meta, golden arrays) of one golden."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["__meta__"]))
    cfg = json.load(open(os.path.join(GOLDEN, meta["config"])))
    cfg["data"]["image_shape"] = list(meta["image_shape"])
    g = torch.Generator().manual_seed(4321 + meta["seed"])
    b, h, w = meta["shape"]
    rgb = torch.randint(0, 256, (b, 3, h, w), dtype=torch.uint8, generator=g)
    K = torch.from_numpy(z["K_in"]) if meta["with_k"] else None
    if "vitl14" in name:
        from unidepth_v1_vit_oracle import make_v1_vit_state_dict
        sd = make_v1_vit_state_dict(cfg, meta["seed"])
    else:
        from fixture import make_v1_state_dict
        sd = make_v1_state_dict(cfg, meta["seed"])
    return cfg, sd, rgb, K, meta, z


def oracle_infer(name, sd, cfg, rgb, K):
    if "vitl14" in name:
        import unidepth_v1_vit_oracle as OV
        return OV.infer_v1_vit(sd, cfg, rgb, K)
    import unidepth_v1_oracle as O1
    return O1.infer_v1(sd, cfg, rgb, K)


def sampled(t, key, meta):
    s = meta["strides"].get(key, 1)
    return t[:, :, ::s, ::s] if t.ndim == 4 else t


@pytest.mark.parametrize("name", SHAPE_CASES)
def test_oracle_matches_reference_at_network_shape(name):
    cfg, sd, rgb, K, meta, z = shape_case(name)
    out = oracle_infer(name, sd, cfg, rgb, K)
    assert tuple(out["depth"].shape[-2:]) == tuple(meta["shape"][1:])
    for k in ("intrinsics", "depth", "points"):
        ref = torch.from_numpy(z[k])
        got = sampled(out[k], k, meta)
        assert got.shape == ref.shape, (k, got.shape, ref.shape)
        floor = 0.1 * ref.abs().mean().item()
        err = ((got - ref).abs() / ref.abs().clamp(min=floor)).max().item()
        print(name, k, "max rel err", err)
        assert err < 2e-5, (k, err)       # measured: depth <= 1.4e-6, points <= 6.2e-6, intrinsics <= 3.5e-7


def _model(cfg_name):
    cfg = json.load(open(os.path.join(GOLDEN, cfg_name)))
    return UniDepthV1(copy.deepcopy(cfg)).eval()


def _dry_run(m, T, S, B=1, H=480, W=640):
    """udb_v1_workspace_bytes of an engine for m.image_shape with T / S registered: (bytes, error text)."""
    lib = _cabi.lib()
    h = C.c_void_p()
    _cabi.check(lib.udb_v1_create(C.byref(m._engine_config()), C.byref(h)), "udb_v1_create")
    try:
        m._register(h, T, S)
        n = lib.udb_v1_workspace_bytes(h, B, H, W)
        return n, (lib.udb_last_error().decode() if n == 0 else "")
    finally:
        lib.udb_v1_destroy(h)


# ConvNeXt: landscape and square shapes from 64x64 to 924x1232, with sides of every residue mod 4
CONVNEXT_SWEEP = [(64, 64), (64, 97), (90, 131), (96, 128), (127, 254), (201, 403), (384, 512), (462, 616), (448, 448),
                  (470, 630), (513, 771), (701, 702), (924, 1232)]
# ViT-L/14: multiples of 14 from 70x70 to 1036x1386
VIT_SWEEP = [(70, 70), (84, 84), (70, 1386), (98, 140), (378, 504), (448, 448), (462, 616), (518, 686), (1036, 1386)]


@pytest.mark.parametrize("cfg_name,sweep", [("config_v1_cnvnxtl.json", CONVNEXT_SWEEP), ("config_v1_vitl14.json", VIT_SWEEP)])
def test_dry_run_over_network_shapes(cfg_name, sweep):
    m = _model(cfg_name)
    W8, S = m._pack_weights(CPU)
    seen = []
    for shape in sweep:
        m.image_shape = list(shape)
        hc, wc = m.spec.common_grid(shape)
        ops = m._shape_operands(shape, CPU)
        assert ops["tokens_pos"].shape == (4 * hc * wc, 512)
        if "pos" in ops:
            assert ops["pos"].shape == (1 + hc * wc, 1024)
        n, err = _dry_run(m, {**W8, **ops}, S)
        if 4 * hc * wc <= 128:        # the 1/8 decoder level needs more tokens than Nystrom's 128 landmarks
            assert n == 0 and "Nystrom" in err and f"{shape[0]}x{shape[1]}" in err, (shape, err)
            continue
        assert n > 0, (shape, err)
        seen.append((hc * wc, n))
        # the operands of another shape are refused by shape, not read out of bounds
        other = m._shape_operands((shape[0], shape[1] + 28), CPU)
        n_bad, err = _dry_run(m, {**W8, **other}, S)
        assert n_bad == 0 and ("tokens_pos" in err or "'pos'" in err), (shape, err)
    assert len(seen) >= len(sweep) - 2
    # the workspace grows with the network grid
    seen.sort()
    assert all(a[1] <= b[1] for a, b in zip(seen, seen[1:]))
    # _pack_tensors at a set image_shape is the weights plus that shape's operands
    m.image_shape = [378, 504]
    T, _ = m._pack_tensors(CPU)
    assert set(T) == set(W8) | set(m._shape_operands((378, 504), CPU))


def test_shape_operands_match_oracle_tables():
    """"tokens_pos" (sine position of the common grid + level embedding) and "pos" (offset-0.1 bicubic resize of the
    37x37 table) at new shapes equal the oracles' tables."""
    import unidepth_v1_oracle as O1
    from unidepth_v1_vit_oracle import interpolate_pos_embed_offset, make_v1_vit_state_dict
    cfg = json.load(open(os.path.join(GOLDEN, "config_v1_vitl14.json")))
    m = UniDepthV1(copy.deepcopy(cfg)).eval()
    m.load_state_dict(make_v1_vit_state_dict(cfg, 0), strict=True)
    sd = m.state_dict()
    p = "pixel_decoder."
    le = torch.nn.functional.linear(torch.nn.functional.gelu(torch.nn.functional.linear(
        sd[p + "level_embeds"], sd[p + "level_embed_layer.0.weight"], sd[p + "level_embed_layer.0.bias"])),
        sd[p + "level_embed_layer.2.weight"], sd[p + "level_embed_layer.2.bias"])
    le = torch.nn.functional.layer_norm(le, (512,), sd[p + "level_embed_layer.3.weight"], sd[p + "level_embed_layer.3.bias"], 1e-5)
    for shape in ((378, 504), (518, 686), (448, 448)):
        gh, gw = shape[0] // 14, shape[1] // 14
        m.image_shape = list(shape)
        T, _ = m._pack_tensors(CPU)
        ref = interpolate_pos_embed_offset(sd["pixel_encoder.pos_embed"].float(), gh, gw)[0]
        assert torch.equal(T["pos"], ref), shape
        # decoder_v1: pos_embed + level_embed over the 4 levels of the common grid
        want = (O1.position_embedding_sine(gh, gw, 256)[None] + le[:, None, :]).reshape(4 * gh * gw, 512)
        assert torch.allclose(T["tokens_pos"], want, atol=1e-6, rtol=0), shape
    # ConvNeXt: the common grid is the stride-16 level, floors included (470x630 -> 117x157 -> 58x78 -> 29x39)
    mc = _model("config_v1_cnvnxtl.json")
    mc.image_shape = [470, 630]
    assert mc.spec.common_grid((470, 630)) == (29, 39)
    assert mc._shape_operands((470, 630), CPU)["tokens_pos"].shape == (4 * 29 * 39, 512)


@pytest.mark.parametrize("shape,exc,text", [
    ([0, 640], ValueError, "at least 64"), ([-462, 616], ValueError, "at least 64"), ([63, 616], ValueError, "at least 64"),
    ([462], ValueError, "two integers"), ([462.0, 616.0], ValueError, "two integers"), ("462x616", ValueError, "two integers"),
    ([True, 616], ValueError, "two integers"), ([616, 462], NotImplementedError, "portrait"),
    ([462, 620], NotImplementedError, "14-pixel patch"),
])
def test_invalid_image_shape_is_refused_before_anything_runs(shape, exc, text):
    cfg_name = "config_v1_vitl14.json" if "patch" in text else "config_v1_cnvnxtl.json"
    m = _model(cfg_name)
    m.image_shape = shape
    with pytest.raises(exc, match=text):
        m._network_shape()
    # infer validates before it looks at the device (a CPU model would otherwise fail for that), and packs nothing
    with pytest.raises(exc, match=text):
        m.infer(torch.zeros(1, 3, 480, 640, dtype=torch.uint8))
    assert m._packed is None and m._engine is None
    # the config's shape for this encoder is still valid
    m.image_shape = list(m.spec.image_shape)
    assert m._network_shape() == tuple(m.spec.image_shape)
