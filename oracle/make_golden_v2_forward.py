"""Generate tests/golden/v2fwd_*.npz: outputs of the UNMODIFIED reference `UniDepthV2.forward(inputs, image_metas)` in eval
mode (`forward_test`, unidepthv2.py:134-160, the call of the reference's evaluation loop unidepth/utils/validation.py),
imported from the reference sources, on the seeded ViT-S/14 and ViT-L/14 fixtures of make_golden.py.

The network input is the reference's own ImageNet normalisation of a seeded uint8 image, already at a shape whose sides
are multiples of 14, as the data pipeline hands it to `forward`.  The paddings travel in the metas as the data pipeline
writes them, (l, t, r, b) with "depth_paddings" beside them (the reference reads both); the cases cover paddings that
differ per image with a ground truth larger than the crop, a ground truth smaller than the crop, equal sizes with zero
paddings, a Pinhole and an EUCM camera object.  The files are named v2fwd_* so that no other test's pattern takes them in.

    python oracle/make_golden_v2_forward.py [name ...]       (CPU; the GPU box only reads the .npz files)
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

from fixture import make_state_dict  # noqa: E402
from make_golden import seeded_rgb  # noqa: E402

CONFIGS = {"vits14": "config_v2_vits14.json", "vitl14": "config_v2_vitl14.json"}
CASES = [
    # name, backbone, seed, (B, h, w) of the network input, (H, W) of the ground truth,
    # metas paddings (l, t, r, b) per image or None (no "paddings" in the metas: zeros), camera (class, params) or None
    ("v2fwd_vits14_pads2_294x392_480x640", "vits14", 20, (2, 294, 392), (480, 640), [(14, 0, 28, 7), (0, 21, 5, 0)], None),
    ("v2fwd_vits14_down_420x560_240x320", "vits14", 21, (1, 420, 560), (240, 320), [(0, 28, 0, 14)], None),
    ("v2fwd_vits14_eq_294x392", "vits14", 22, (1, 294, 392), (294, 392), [(0, 0, 0, 0)], None),
    ("v2fwd_vits14_pinhole_294x392_360x480", "vits14", 23, (1, 294, 392), (360, 480), [(7, 14, 7, 0)],
     ("Pinhole", [300.0, 305.0, 196.0, 150.0])),
    ("v2fwd_vits14_eucm_294x392_480x640", "vits14", 24, (1, 294, 392), (480, 640), None,
     ("EUCM", [180.0, 182.0, 196.0, 147.0, 0.6, 1.1])),
    ("v2fwd_vitl14_pads2_224x294_300x400", "vitl14", 25, (2, 224, 294), (300, 400), [(7, 0, 0, 14), (0, 0, 21, 0)], None),
]
# stored sub-samples: maps every STRIDES[k]-th pixel per axis, and every IMAGE_STRIDE-th pixel of the network input (the
# tests rebuild it and check it against these)
STRIDES = dict(depth=4, confidence=4, points=8, rays=8)
IMAGE_STRIDE = 14


def network_input(shape, seed):
    """The reference's normalisation (unidepthv2.py:280-290) of the seeded uint8 image: f32 [B, 3, h, w]."""
    import torchvision.transforms.functional as TF
    from unidepth.utils.constants import IMAGENET_DATASET_MEAN, IMAGENET_DATASET_STD
    rgb = seeded_rgb(shape, seed)
    return TF.normalize(rgb.to(torch.float32).div(255), mean=IMAGENET_DATASET_MEAN, std=IMAGENET_DATASET_STD)


def reference_forward(case):
    """(network input, metas, outputs) of the unmodified reference's eval-mode forward on one case."""
    from unidepth.models import UniDepthV2
    import unidepth.utils.camera as RC
    name, bb, seed, shape, gt_hw, pads, camera = case
    cfg = json.load(open(os.path.join(REF, "configs", CONFIGS[bb])))
    model = UniDepthV2(copy.deepcopy(cfg)).eval()
    model.load_state_dict(make_state_dict(cfg, seed), strict=True)
    x = network_input(shape, seed)
    inputs = {"image": x.clone(), "depth": torch.zeros(shape[0], 1, *gt_hw)}
    metas = [{"paddings": list(p), "depth_paddings": [0, 0, 0, 0]} for p in pads] if pads is not None else []
    if pads is None:
        inputs["paddings"] = torch.zeros(shape[0], 4, dtype=torch.int64)       # the reference needs the key
    if camera is not None:
        kind, params = camera
        p = torch.tensor([params], dtype=torch.float32)
        if kind == "Pinhole":
            fx, fy, cx, cy = params
            inputs["camera"] = RC.Pinhole(K=torch.tensor([[[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]]]))
        else:
            inputs["camera"] = getattr(RC, kind)(params=p)
    with torch.no_grad():
        out = model(inputs, metas)
    return x, metas, out


def main():
    warnings.simplefilter("ignore")
    out_dir = os.path.join(HERE, "..", "tests", "golden")
    only = sys.argv[1:]
    torch.set_num_threads(min(32, os.cpu_count()))
    for case in CASES:
        name, bb, seed, shape, gt_hw, pads, camera = case
        if only and name not in only:
            continue
        x, metas, out = reference_forward(case)
        arrays = {k: v.detach().float().cpu().numpy() for k, v in out.items()}
        for k, s in STRIDES.items():
            arrays[k] = np.ascontiguousarray(arrays[k][:, :, ::s, ::s])
        arrays["image_sample"] = np.ascontiguousarray(x[:, :, ::IMAGE_STRIDE, ::IMAGE_STRIDE].numpy())
        meta = dict(config=CONFIGS[bb], seed=seed, shape=list(shape), gt_hw=list(gt_hw),
                    metas_paddings=[list(p) for p in pads] if pads is not None else None,
                    camera=dict(kind=camera[0], params=camera[1]) if camera is not None else None,
                    strides=STRIDES, image_stride=IMAGE_STRIDE)
        path = os.path.join(out_dir, name + ".npz")
        np.savez_compressed(path, __meta__=json.dumps(meta), **arrays)
        d = arrays["depth"]
        print(name, f"{os.path.getsize(path) / 1e3:.0f} kB", "depth range", float(d.min()), float(d.max()),
              "K", arrays["intrinsics"][0].tolist(), flush=True)


if __name__ == "__main__":
    main()
