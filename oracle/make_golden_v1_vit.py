"""Generate tests/golden/v1_vitl14_*.npz and tests/golden/config_v1_vitl14.json: outputs of the UNMODIFIED reference
`UniDepthV1.infer` with the DINOv2 ViT-L/14 encoder (configs/config_v1_vitl14.json), imported through oracle/ref_shims,
on the seeded fixture of oracle/unidepth_v1_vit_oracle.py.  As for the ConvNeXt goldens (make_golden_v1.py), the one
substitution is xformers' NystromAttention, replaced by the restatement in oracle/unidepth_v1_oracle.py.

    python oracle/make_golden_v1_vit.py        (CPU, about 3 s per case; the GPU box only reads the .npz files)
TEST INFRASTRUCTURE ONLY."""
import copy
import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
sys.path[:0] = [REF, os.path.join(HERE, "ref_shims"), HERE, os.path.join(HERE, "..")]

from make_golden_v1 import OracleNystrom, seeded_rgb  # noqa: E402
from unidepth_v1_vit_oracle import make_v1_vit_state_dict  # noqa: E402

CASES = [
    # name, seed, (B,H,W), with GT intrinsics
    ("v1_vitl14_480x640", 0, (1, 480, 640), False),
    ("v1_vitl14_gtK_375x1242", 1, (1, 375, 1242), True),
]


def main():
    warnings.simplefilter("ignore")
    import unidepth.layers.nystrom_attention as NA
    NA.NystromAttention = OracleNystrom
    from unidepth.models import UniDepthV1
    from unidepth_b200.spec_v1 import param_shapes
    out_dir = os.path.join(HERE, "..", "tests", "golden")
    cfg = json.load(open(os.path.join(REF, "configs", "config_v1_vitl14.json")))
    keep = {"model": cfg["model"], "data": {"image_shape": cfg["data"]["image_shape"]}, "training": {}}
    json.dump(keep, open(os.path.join(out_dir, "config_v1_vitl14.json"), "w"), indent=1)
    model = UniDepthV1(copy.deepcopy(cfg)).eval()
    assert model.pixel_encoder.interpolate_offset == 0.1 and not model.pixel_encoder.use_norm
    ref_shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    mine = dict(param_shapes(cfg))
    assert ref_shapes == mine, (set(ref_shapes) ^ set(mine), [k for k in mine if k in ref_shapes and mine[k] != ref_shapes[k]])
    for name, seed, shape, with_k in CASES:
        sd = make_v1_vit_state_dict(cfg, seed)
        model.load_state_dict(sd, strict=True)
        rgb = seeded_rgb(shape, seed)
        K = None
        if with_k:
            K = torch.tensor([[[720.0, 0.0, 610.0], [0.0, 725.0, 180.0], [0.0, 0.0, 1.0]]])
        with torch.no_grad():
            out = model.infer(rgb, K.clone() if K is not None else None)
        # the maps are stored sub-sampled (depth every 4th, points every 8th pixel per axis): full-resolution f32 maps do not
        # compress and would make each file megabytes.  The full-resolution outputs are checked against the oracle, which
        # these files pin.
        arrays = {k: v.detach().cpu().numpy() for k, v in out.items()}
        arrays["depth"] = np.ascontiguousarray(arrays["depth"][:, :, ::4, ::4])
        arrays["points"] = np.ascontiguousarray(arrays["points"][:, :, ::8, ::8])
        meta = dict(config="config_v1_vitl14.json", seed=seed, shape=list(shape), with_k=with_k, skip_camera=False,
                    strides=dict(depth=4, points=8))
        if K is not None:
            arrays["K_in"] = K.numpy()
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), __meta__=json.dumps(meta), **arrays)
        d = arrays["depth"]
        print(name, "depth range", float(d.min()), float(d.max()), "K", arrays["intrinsics"][0].tolist())


if __name__ == "__main__":
    main()
