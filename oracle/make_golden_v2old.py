"""Generate tests/golden/v2old_{vitl14,vits14}_*.npz, tests/golden/v2old_geometry.npz and the two config copies: outputs
of the UNMODIFIED reference `UniDepthV2old.infer` (configs/config_v2old_{vitl14,vits14}.json), imported through
oracle/ref_shims, on a seeded fixture.  As for the UniDepthV1 goldens (make_golden_v1.py), the one substitution is
xformers' NystromAttention, replaced by the restatement in oracle/unidepth_v1_oracle.py.

The geometry file records, over a grid of input shapes and resolution levels, what the reference's own `_check_resolution`
and `_shapes` return and whether they warn, so the CPU tests pin unidepth_b200's arithmetic to them.

    python oracle/make_golden_v2old.py        (CPU; the GPU box only reads the .npz files)
TEST INFRASTRUCTURE ONLY."""
import copy
import json
import os
import sys
import warnings
from typing import Dict

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
sys.path[:0] = [REF, os.path.join(HERE, "ref_shims"), HERE, os.path.join(HERE, "..")]

from make_golden_v1 import OracleNystrom, seeded_rgb  # noqa: E402

BACKBONES = ("vitl14", "vits14")
K_WIDE = [[720.0, 0.0, 610.0], [0.0, 725.0, 180.0], [0.0, 0.0, 1.0]]
CASES = [
    # name, seed, (B,H,W), GT intrinsics, resolution_level, interpolation_mode
    ("480x640", 0, (1, 480, 640), None, None, "bilinear"),
    ("gtK_375x1242", 1, (1, 375, 1242), K_WIDE, 10, "bilinear"),
    ("rl0_360x480", 2, (1, 360, 480), None, 0, "bilinear"),
    ("rl5_600x800", 3, (1, 600, 800), None, 5, "bilinear"),
    ("nearest_480x640", 4, (1, 480, 640), None, 7, "nearest-exact"),
    ("ratio_600x250", 5, (1, 600, 250), None, 3, "bilinear"),
]


def make_v2old_state_dict(config: dict, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded fixture for UniDepthV2old: names / shapes from unidepth_b200.spec_v2old.param_shapes (asserted below to equal
    the reference model's), one generator per tensor seeded from (seed, index); the recipe of
    unidepth_v1_vit_oracle.make_v1_vit_state_dict."""
    from unidepth_b200.spec_v2old import param_shapes
    sd: Dict[str, torch.Tensor] = {}
    for idx, (key, shape) in enumerate(param_shapes(config).items()):
        g = torch.Generator().manual_seed(seed * 1_000_003 + idx)
        n = lambda *s: torch.randn(*s, generator=g)
        u = lambda *s: torch.rand(*s, generator=g)
        leaf = key.rsplit(".", 1)[-1]
        is_norm = ("norm" in key or key.endswith((".0.weight", ".0.bias")) and "input_adapters" in key
                   or "level_embed_layer.3." in key)
        if key.endswith(("mask_token", "register_tokens")):
            t = torch.zeros(*shape)                   # dead on the infer path
        elif key.endswith(("cls_token", "pos_embed")):
            t = 0.2 * n(*shape)
        elif key.endswith(("level_embeds", "latents_pos")):
            t = 0.5 * n(*shape)
        elif ".ls1.gamma" in key or ".ls2.gamma" in key:
            t = 0.3 * (0.5 + u(*shape))
        elif leaf == "gamma":
            t = 0.4 * (0.5 + u(*shape))
        elif is_norm and len(shape) == 1:
            t = 1.0 + 0.1 * n(*shape) if leaf == "weight" else 0.05 * n(*shape)
        elif leaf == "bias":
            t = 0.05 * n(*shape)
        elif leaf == "weight":
            fan_in = 1
            for s_ in shape[1:]:
                fan_in *= s_
            t = n(*shape) / fan_in ** 0.5
            if key.endswith(("camera_layer.out.proj2.weight", "global_layer.out.proj2.weight")):
                t = 0.3 * t
        else:
            raise KeyError(key)
        sd[key] = t.float().contiguous()
    return sd


def geometry_grid():
    """(H, W, level) triples: about 1000 input shapes across and beyond the ratio bounds, each with one level drawn from
    None, -2..12 (clipped), so every branch of `_check_resolution` and `_shapes` is visited."""
    g = torch.Generator().manual_seed(99)
    hs = torch.randint(8, 3000, (1000,), generator=g).tolist()
    ratios = (torch.rand(1000, generator=g) * 3.5 + 0.15).tolist()
    levels = torch.randint(-3, 13, (1000,), generator=g).tolist()
    out = []
    for h, r, lv in zip(hs, ratios, levels):
        w = max(8, int(round(h * r)))
        out.append((h, w, None if lv == -3 else lv))
    out += [(480, 640, None), (375, 1242, 10), (14, 14, 0), (4000, 4000, 10), (1000, 660, 4), (500, 1000, 6)]
    return out


def record_geometry(out_dir):
    from unidepth.models.unidepthv2 import unidepthv2_old as R
    rows, warned = [], []
    for h, w, lv in geometry_grid():
        sc = {"ratio_bounds": [0.66, 2.0], "pixels_bounds_ori": [1400, 2400], "patch_size": 14}
        with warnings.catch_warnings(record=True) as ws:
            warnings.simplefilter("always")
            sc = R._check_resolution(sc, lv)
            n_res = len(ws)
            (nh, nw), ratio = R._shapes((h, w), sc)
            n_ratio = len(ws) - n_res
        rows.append((h, w, -1 if lv is None else lv, sc["pixels_bounds"][0], nh, nw, ratio))
        warned.append((n_res, n_ratio))
    a = np.array(rows, dtype=np.float64)
    np.savez_compressed(os.path.join(out_dir, "v2old_geometry.npz"), hw=a[:, :2].astype(np.int64), level=a[:, 2].astype(np.int64),
                        pixels=a[:, 3].astype(np.int64), net_hw=a[:, 4:6].astype(np.int64), ratio=a[:, 6],
                        warnings=np.array(warned, dtype=np.int64))
    print("geometry", len(rows), "shapes")


def main():
    warnings.simplefilter("ignore")
    import unidepth.layers.nystrom_attention as NA
    NA.NystromAttention = OracleNystrom
    from unidepth.models.unidepthv2.unidepthv2_old import UniDepthV2old
    from unidepth_b200.spec_v2old import param_shapes
    out_dir = os.path.join(HERE, "..", "tests", "golden")
    pkg_dir = os.path.join(HERE, "..", "unidepth_b200", "configs")
    record_geometry(out_dir)
    only = sys.argv[1:]
    for bb in BACKBONES:
        cfg = json.load(open(os.path.join(REF, "configs", f"config_v2old_{bb}.json")))
        for d in (out_dir, pkg_dir):
            json.dump(cfg, open(os.path.join(d, f"config_v2old_{bb}.json"), "w"), indent=1)
        model = UniDepthV2old(copy.deepcopy(cfg)).eval()
        enc = model.pixel_encoder
        assert enc.use_norm and enc.interpolate_offset == 0.0 and enc.norm.eps == 1e-5, (enc.use_norm, enc.interpolate_offset)
        ref_shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
        mine = dict(param_shapes(cfg))
        assert ref_shapes == mine, (set(ref_shapes) ^ set(mine), [k for k in mine if k in ref_shapes and mine[k] != ref_shapes[k]])
        for case, seed, shape, K, level, mode in CASES:
            name = f"v2old_{bb}_{case}"
            if only and name not in only:
                continue
            model.load_state_dict(make_v2old_state_dict(cfg, seed), strict=True)
            model.resolution_level = level
            model.interpolation_mode = mode
            rgb = seeded_rgb(shape, seed)
            Kt = torch.tensor([K]) if K is not None else None
            with torch.no_grad():
                out = model.infer(rgb, Kt.clone() if Kt is not None else None)
            # sub-sampled maps (depth and confidence every 4th, points every 8th pixel per axis): full-resolution f32 maps
            # do not compress and would make each file megabytes
            arrays = {k: v.detach().cpu().numpy() for k, v in out.items()}
            arrays["depth"] = np.ascontiguousarray(arrays["depth"][:, :, ::4, ::4])
            arrays["confidence"] = np.ascontiguousarray(arrays["confidence"][:, :, ::4, ::4])
            arrays["points"] = np.ascontiguousarray(arrays["points"][:, :, ::8, ::8])
            meta = dict(config=f"config_v2old_{bb}.json", seed=seed, shape=list(shape), with_k=K is not None,
                        resolution_level=level, interpolation_mode=mode, strides=dict(depth=4, confidence=4, points=8))
            if Kt is not None:
                arrays["K_in"] = Kt.numpy()
            np.savez_compressed(os.path.join(out_dir, name + ".npz"), __meta__=json.dumps(meta), **arrays)
            d = arrays["depth"]
            print(name, "depth range", float(d.min()), float(d.max()), "K", arrays["intrinsics"][0].tolist(), flush=True)


if __name__ == "__main__":
    main()
