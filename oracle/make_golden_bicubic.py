"""Generate tests/golden/vits_bicubic_*.npz: `UniDepthV2.infer` of the UNMODIFIED reference with
`model.interpolation_mode = "bicubic"` (`_postprocess`, unidepthv2.py:80-89,311-329: F.interpolate(mode="bicubic",
align_corners=False) of confidence, points and rays to the padded input size).  The cases cover bicubic downsampling
(network input larger than the padded image), upsampling (smaller), a top/bottom padding crop and the GT-camera branch.
Pins the oracle's `interpolation_mode` argument (tests/test_bicubic_cpu.py) and the CUDA path (tests/test_bicubic_gpu.py).

Run where the reference is installed:   python oracle/make_golden_bicubic.py
TEST INFRASTRUCTURE ONLY.
"""
import copy
import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
sys.path[:0] = [REF, os.path.join(HERE, "ref_shims"), HERE]

from fixture import make_state_dict  # noqa: E402
from make_golden import seeded_rgb  # noqa: E402

# name, config, seed, (B,H,W), resolution_level, camera K as (fx, fy, cx, cy) or None,
# (depth stride, spatial stride, depth_features channel stride) -- see subsample_like_golden in tests/test_oracle_golden.py
CASES = [
    ("vits_bicubic_120x160", "config_v2_vits14.json", 10, (1, 120, 160), None, None, (1, 2, 16)),
    ("vits_bicubic_pad_96x288_rl3", "config_v2_vits14.json", 11, (1, 96, 288), 3, None, (1, 2, 16)),
    ("vits_bicubic_700x1000_rl0", "config_v2_vits14.json", 12, (1, 700, 1000), 0, None, (8, 16, 16)),
    ("vits_bicubic_camK_120x160", "config_v2_vits14.json", 13, (1, 120, 160), None, (125.0, 127.0, 79.0, 61.5), (1, 2, 16)),
]


def main():
    warnings.simplefilter("ignore")
    from unidepth.models import UniDepthV2
    out_dir = os.path.join(HERE, "..", "tests", "golden")
    for name, cfg_name, seed, shape, level, k4, (sd_, ss_, sc_) in CASES:
        cfg = json.load(open(os.path.join(REF, "configs", cfg_name)))
        model = UniDepthV2(copy.deepcopy(cfg)).eval()
        model.load_state_dict(make_state_dict(cfg, seed), strict=True)
        model.interpolation_mode = "bicubic"
        if level is not None:
            model.resolution_level = level
        rgb = seeded_rgb(shape, seed)
        if k4 is None:
            out = model.infer(rgb)
        else:
            fx, fy, cx, cy = k4
            out = model.infer(rgb, torch.tensor([[[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]]]))
        arrays = {k: v.detach().cpu().numpy() for k, v in out.items()}
        arrays["depth_features"] = arrays["depth_features"][:, ::sc_]
        arrays["depth"] = arrays["depth"][:, :, ::sd_, ::sd_]
        for k in ("confidence", "radius", "points", "rays"):
            arrays[k] = arrays[k][:, :, ::ss_, ::ss_]
        meta = dict(config=cfg_name, seed=seed, shape=list(shape), resolution_level=level, interpolation_mode="bicubic",
                    strides=dict(depth=sd_, spatial=ss_, depth_features=sc_))
        if k4 is not None:
            meta["camera"] = dict(kind="K", params=list(k4))
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), __meta__=json.dumps(meta), **arrays)
        d, c = arrays["depth"], arrays["confidence"]
        print(name, "depth range", float(d.min()), float(d.max()), "confidence range", float(c.min()), float(c.max()),
              "K out", arrays["intrinsics"][0].tolist())


if __name__ == "__main__":
    main()
