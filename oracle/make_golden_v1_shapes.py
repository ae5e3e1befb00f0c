"""Generate tests/golden/v1_{cnvnxtl,vitl14}_net<H>x<W>_*.npz: outputs of the UNMODIFIED reference `UniDepthV1.infer` run
at a network shape other than the config's, set the way a user sets it (`model.image_shape = [H, W]`, which `infer` reads
on every call, unidepthv1.py:309-350).  Everything else is as in make_golden_v1.py (ConvNeXt-L) and make_golden_v1_vit.py
(ViT-L/14): the same seeded fixtures and inputs, and the one substitution, xformers' NystromAttention, replaced by the
restatement in oracle/unidepth_v1_oracle.py.  The maps are stored sub-sampled (depth every 4th, points every 8th pixel per
axis) so that each file stays small; the GPU tests check every pixel against the oracle, which these files pin.

    python oracle/make_golden_v1_shapes.py                      (every shape below; CPU, minutes per ConvNeXt-L case)
    python oracle/make_golden_v1_shapes.py --encoder vitl14 --image-shape 378 504 [--gt-k] [--out DIR]
TEST INFRASTRUCTURE ONLY."""
import argparse
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

CONFIGS = {"cnvnxtl": "config_v1_cnvnxtl.json", "vitl14": "config_v1_vitl14.json"}
# (encoder, network shape, with the GT-K case): ConvNeXt-L at 384x512, 470x630 (stem and downsample floors that do not
# divide evenly) and 448x448 (square); ViT-L/14 at 378x504 (27x36 patches), 518x686 (37x49) and 448x448 (32x32)
SHAPES = [("cnvnxtl", (384, 512), False), ("cnvnxtl", (470, 630), True), ("cnvnxtl", (448, 448), False),
          ("vitl14", (378, 504), False), ("vitl14", (518, 686), True), ("vitl14", (448, 448), False)]
K_IN = [[[720.0, 0.0, 610.0], [0.0, 725.0, 180.0], [0.0, 0.0, 1.0]]]
STRIDES = dict(depth=4, points=8)


def state_dict(encoder, cfg, seed):
    if encoder == "vitl14":
        from unidepth_v1_vit_oracle import make_v1_vit_state_dict
        return make_v1_vit_state_dict(cfg, seed)
    from fixture import make_v1_state_dict
    return make_v1_state_dict(cfg, seed)


def generate(encoder, image_shape, gt_k, out_dir):
    from unidepth.models import UniDepthV1
    cfg = json.load(open(os.path.join(REF, "configs", CONFIGS[encoder])))
    model = UniDepthV1(copy.deepcopy(cfg)).eval()
    model.image_shape = list(image_shape)
    net = f"v1_{encoder}_net{image_shape[0]}x{image_shape[1]}"
    # name, seed, (B,H,W), with GT intrinsics: the 480x640 input, and the GT-K 375x1242 one with `gt_k`
    cases = [(f"{net}_480x640", 0, (1, 480, 640), False)]
    if gt_k:
        cases.append((f"{net}_gtK_375x1242", 1, (1, 375, 1242), True))
    for name, seed, shape, with_k in cases:
        model.load_state_dict(state_dict(encoder, cfg, seed), strict=True)
        rgb = seeded_rgb(shape, seed)
        K = torch.tensor(K_IN) if with_k else None
        with torch.no_grad():
            out = model.infer(rgb, K.clone() if K is not None else None)
        arrays = {k: v.detach().cpu().numpy() for k, v in out.items()}
        for k, st in STRIDES.items():
            arrays[k] = np.ascontiguousarray(arrays[k][:, :, ::st, ::st])
        meta = dict(config=CONFIGS[encoder], seed=seed, shape=list(shape), with_k=with_k, skip_camera=False,
                    strides=STRIDES, image_shape=list(image_shape))
        if K is not None:
            arrays["K_in"] = K.numpy()
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), __meta__=json.dumps(meta), **arrays)
        d = arrays["depth"]
        print(name, "depth range", float(d.min()), float(d.max()), "K", arrays["intrinsics"][0].tolist())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--encoder", choices=sorted(CONFIGS), help="with --image-shape: one run instead of every shape")
    ap.add_argument("--image-shape", type=int, nargs=2, metavar=("H", "W"))
    ap.add_argument("--gt-k", action="store_true", help="with --image-shape: also the GT-intrinsics 375x1242 case")
    ap.add_argument("--out", default=os.path.join(HERE, "..", "tests", "golden"))
    args = ap.parse_args()
    if (args.encoder is None) != (args.image_shape is None):
        ap.error("--encoder and --image-shape go together")
    warnings.simplefilter("ignore")
    import unidepth.layers.nystrom_attention as NA
    NA.NystromAttention = OracleNystrom
    runs = [(args.encoder, tuple(args.image_shape), args.gt_k)] if args.encoder else SHAPES
    os.makedirs(args.out, exist_ok=True)
    for encoder, image_shape, gt_k in runs:
        generate(encoder, image_shape, gt_k, args.out)


if __name__ == "__main__":
    main()
