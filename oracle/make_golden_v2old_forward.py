"""Generate tests/golden/v2oldfwd_{vitl14,vits14}_*.npz: outputs of the UNMODIFIED reference `UniDepthV2old.forward(inputs,
image_metas)` in eval mode (the call of the reference's evaluation loop, unidepth/utils/validation.py), imported through
oracle/ref_shims, with the fixture and the Nystrom substitution of make_golden_v2old.py.

The network input is the reference's own ImageNet normalisation (`infer`'s /255 and TF.normalize) of a seeded uint8 image,
already at a shape whose sides are multiples of 14, as `forward` takes it.  The cases cover a ground truth of the image's
size, a batch of two with two different K, a ground truth larger and one smaller than the image, and a portrait image
with K.  The files are named v2oldfwd_* so that the `infer` goldens' v2old_vit* pattern does not take them in.

    python oracle/make_golden_v2old_forward.py        (CPU; the GPU box only reads the .npz files)
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
from make_golden_v2old import BACKBONES, make_v2old_state_dict  # noqa: E402

K_A = [[300.0, 0.0, 200.0], [0.0, 305.0, 150.0], [0.0, 0.0, 1.0]]
K_B = [[420.0, 0.0, 180.0], [0.0, 410.0, 140.0], [0.0, 0.0, 1.0]]
K_PORTRAIT = [[500.0, 0.0, 215.0], [0.0, 495.0, 275.0], [0.0, 0.0, 1.0]]
CASES = [
    # name, seed, (B, h, w) of the network input, (H, W) of the ground truth, K per image or None
    ("eq_420x560", 10, (1, 420, 560), (420, 560), None),
    ("K2_294x392", 11, (2, 294, 392), (294, 392), [K_A, K_B]),
    ("up_294x392_480x640", 12, (1, 294, 392), (480, 640), None),
    ("down_420x560_240x320", 13, (1, 420, 560), (240, 320), None),
    ("portraitK_560x420", 14, (1, 560, 420), (560, 420), [K_PORTRAIT]),
]
# stored sub-samples: maps every STRIDES[k]-th pixel per axis, FEAT_TOKENS tokens of depth_features every FEAT_CH-th
# channel, and every IMAGE_STRIDE-th pixel of the network input (the tests rebuild it and check it against these)
STRIDES = dict(depth=4, confidence=4, points=8)
FEAT_TOKENS, FEAT_CH, IMAGE_STRIDE = 32, 4, 14


def network_input(shape, seed):
    """The reference's normalisation (unidepthv2_old.py:211-218) of the seeded uint8 image: f32 [B, 3, h, w]."""
    import torchvision.transforms.functional as TF
    from unidepth.utils.constants import IMAGENET_DATASET_MEAN, IMAGENET_DATASET_STD
    rgb = seeded_rgb(shape, seed)
    return TF.normalize(rgb.to(torch.float32).div(255), mean=IMAGENET_DATASET_MEAN, std=IMAGENET_DATASET_STD)


def main():
    warnings.simplefilter("ignore")
    import unidepth.layers.nystrom_attention as NA
    NA.NystromAttention = OracleNystrom
    from unidepth.models.unidepthv2.unidepthv2_old import UniDepthV2old
    out_dir = os.path.join(HERE, "..", "tests", "golden")
    only = sys.argv[1:]
    for bb in BACKBONES:
        cfg = json.load(open(os.path.join(REF, "configs", f"config_v2old_{bb}.json")))
        model = UniDepthV2old(copy.deepcopy(cfg)).eval()
        for case, seed, shape, gt_hw, K in CASES:
            name = f"v2oldfwd_{bb}_{case}"
            if only and name not in only:
                continue
            model.load_state_dict(make_v2old_state_dict(cfg, seed), strict=True)
            x = network_input(shape, seed)
            inputs = {"image": x.clone(), "depth": torch.zeros(shape[0], 1, *gt_hw)}
            if K is not None:
                inputs["K"] = torch.tensor(K)
            with torch.no_grad():
                out = model(inputs, None)
            arrays = {k: v.detach().float().cpu().numpy() for k, v in out.items()}
            for k, s in STRIDES.items():
                arrays[k] = np.ascontiguousarray(arrays[k][:, :, ::s, ::s])
            n = arrays["depth_features"].shape[1]
            feat_idx = np.unique(np.linspace(0, n - 1, FEAT_TOKENS).round().astype(np.int64))
            arrays["depth_features"] = np.ascontiguousarray(arrays["depth_features"][:, feat_idx, ::FEAT_CH])
            arrays["feat_idx"] = feat_idx
            arrays["image_sample"] = np.ascontiguousarray(x[:, :, ::IMAGE_STRIDE, ::IMAGE_STRIDE].numpy())
            if K is not None:
                arrays["K_in"] = np.array(K, dtype=np.float32)
            meta = dict(config=f"config_v2old_{bb}.json", seed=seed, shape=list(shape), gt_hw=list(gt_hw), with_k=K is not None,
                        strides=STRIDES, feat_ch_stride=FEAT_CH, image_stride=IMAGE_STRIDE)
            path = os.path.join(out_dir, name + ".npz")
            np.savez_compressed(path, __meta__=json.dumps(meta), **arrays)
            d = arrays["depth"]
            print(name, f"{os.path.getsize(path) / 1e3:.0f} kB", "depth range", float(d.min()), float(d.max()),
                  "K", arrays["K"][0].tolist(), flush=True)


if __name__ == "__main__":
    main()
