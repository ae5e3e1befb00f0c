"""Generate tests/golden/eval_metrics.npz from the UNMODIFIED reference evaluation code: unidepth/utils/evaluation_depth.py
(eval_depth, eval_3d) and its ChamferDistance, imported from the reference tree through oracle/ref_shims, with the
reference's KNN CPU extension (unidepth/ops/knn/src/knn_ext.cpp + knn_cpu.cpp) compiled into oracle/_ref/ and
registered as the `KNN` module that unidepth/ops/knn/functions/knn.py imports.

Inputs come from the seeded generators in oracle/eval_oracle.py, so only outputs are stored.  Besides the fp32
reference outputs, eval_depth is also run on float64 inputs (the reference code accepts them), and eval_3d's means
are also taken in float64 over the same per-point fp32 terms: the tests derive their tolerances from these
fp32-vs-fp64 differences.

Run on a machine with the reference tree:   python oracle/make_golden_eval.py [/path/to/reference]
TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
sys.path[:0] = [REF, os.path.join(HERE, "ref_shims"), HERE]


def load_knn():
    from torch.utils.cpp_extension import load
    src = os.path.join(REF, "unidepth", "ops", "knn", "src")
    build = os.path.join(HERE, "_ref")
    os.makedirs(build, exist_ok=True)
    mod = load("KNN", [os.path.join(src, "knn_ext.cpp"), os.path.join(src, "knn_cpu.cpp")], build_directory=build)
    sys.modules["KNN"] = mod
    return mod


def main():
    warnings.simplefilter("ignore")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    knn = load_knn()
    import eval_oracle as O
    from unidepth.utils import evaluation_depth as E
    out = {}

    gts, preds, masks = O.depth_case()
    for tag, md in (("nomax", None), ("max", 7.5)):
        r32 = E.eval_depth(gts, preds, masks, max_depth=md)
        r64 = E.eval_depth(gts.double(), preds.double(), masks, max_depth=md)
        assert list(r32) == O.KEYS, list(r32)
        for k in r32:
            out[f"depth/{tag}/{k}"] = r32[k].numpy()
            out[f"depth64/{tag}/{k}"] = r64[k].numpy()

    # "big": 32 images whose masks hold more than 240 x 320 points in all, so the batch-wide downscale branch runs; many
    # small images keep the reference's CPU KNN (about 165 ns per point pair here) to a couple of minutes
    for tag, case in (("big", O.points_case(B=32, H=48, W=60)), ("empty", O.points_case(seed=14, H=40, W=50, empty=1))):
        gts, preds, masks, thr = case
        r = E.eval_3d(gts, preds, masks, thresholds=thr)
        for k, v in r.items():
            out[f"e3d/{tag}/{k}"] = v.numpy()
        # fp64 means of the same per-point fp32 terms (MSE_3d, chamfer)
        ratio = min(1.0, (240 * 320 / masks.sum()) ** 0.5)
        h, w = int(gts.shape[-2] * ratio), int(gts.shape[-1] * ratio)
        out[f"e3d/{tag}/hw"] = np.array([h, w])
        F = torch.nn.functional
        g2 = F.interpolate(gts, size=(h, w), mode="nearest-exact")
        p2 = F.interpolate(preds, size=(h, w), mode="nearest-exact")
        m2 = F.interpolate(masks.float(), size=(h, w), mode="nearest-exact").bool()
        mse64, ch64 = [], []
        for g, p, m in zip(g2, p2, m2):
            if not m.any():
                continue
            a, b = g[:, m[0]], p[:, m[0]]
            mse64.append(torch.norm(a - b, dim=0, p=2).double().mean())
            d1, d2, _, _ = O.chamfer(a.T[None].contiguous(), b.T[None].contiguous())   # == the reference's (tested)
            ch64.append(((torch.sqrt(d1) + torch.sqrt(d2)) / 2).double().mean())
        out[f"e3d64/{tag}/MSE_3d"] = torch.stack(mse64).numpy()
        out[f"e3d64/{tag}/chamfer"] = torch.stack(ch64).numpy()
        print(tag, "downscaled to", h, w, {k: v.tolist() for k, v in r.items()})

    x, y, l1, l2 = O.knn_case()
    for tag, (a, b, la, lb) in (("xy", (x, y, l1, l2)), ("yx", (y, x, l2, l1))):
        idx, dist = knn.knn_points_idx(a, b, la, lb, 2, 1, -1)
        out[f"knn/{tag}/dist"] = dist[..., 0].numpy()
        out[f"knn/{tag}/idx"] = idx[..., 0].numpy()

    path = os.path.join(ROOT, "tests", "golden", "eval_metrics.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
