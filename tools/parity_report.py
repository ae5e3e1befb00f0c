"""Output parity report: CUDA path (unidepth_b200.UniDepthV2.infer, eager and CUDA graph) vs the CPU oracle on the
same seeded weights / input.  Test infrastructure (imports oracle/).  Usage on a GPU machine:
    python tools/parity_report.py [--depth N] [--batch B] [--hw H W] [--seed S] [--config NAME]
--depth N builds a shallow ViT-L-shaped encoder (arch_override) so the oracle runs in a second."""
import argparse
import copy
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import torch  # noqa: E402

import unidepth_oracle as O  # noqa: E402
from fixture import make_state_dict  # noqa: E402
from unidepth_b200 import UniDepthV2  # noqa: E402


def rel(got, ref):
    got, ref = got.float().cpu(), ref.float().cpu()
    floor = 0.1 * ref.abs().mean().item() + 1e-12
    r = (got - ref).abs() / ref.abs().clamp(min=floor)
    return r.max().item(), r.mean().item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=0)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--hw", type=int, nargs=2, default=[480, 640])
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--config", default="config_v2_vitl14.json")
    ap.add_argument("--camera", action="store_true")
    args = ap.parse_args()
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", args.config)))
    if args.depth:
        d = args.depth
        cfg["model"]["pixel_encoder"]["arch_override"] = {"depth": d}
        cfg["model"]["pixel_encoder"]["output_idx"] = [max(1, d * (i + 1) // 4) for i in range(4)]
    t0 = time.time()
    sd = make_state_dict(cfg, args.seed)
    print(f"weights: {time.time()-t0:.1f}s", flush=True)
    g = torch.Generator().manual_seed(1234 + args.seed)
    rgb = torch.randint(0, 256, (args.batch, 3, args.hw[0], args.hw[1]), dtype=torch.uint8, generator=g)
    torch.set_num_threads(os.cpu_count())
    t0 = time.time()
    ref = O.infer_v2(sd, copy.deepcopy(cfg), rgb)
    print(f"oracle: {time.time()-t0:.1f}s on {os.cpu_count()} cores", flush=True)

    model = UniDepthV2(copy.deepcopy(cfg))
    model.load_state_dict(sd, strict=True)
    model = model.to("cuda").eval()
    model.use_cuda_graph = False
    out = model.infer(rgb)
    print("---- outputs (max rel, mean rel; floor = 10% of mean |ref|)")
    for k in ["intrinsics", "depth", "radius", "points", "rays", "confidence", "depth_features"]:
        mx, mn = rel(out[k], ref[k])
        print(f"{k:14s} max {mx:.3e} mean {mn:.3e}")
    d, dr = out["depth"].cpu(), ref["depth"]
    print("depth ARel (mean |d-dref|/dref): %.3e   max: %.3e" % (((d - dr).abs() / dr).mean().item(), ((d - dr).abs() / dr).max().item()))
    K, Kr = out["intrinsics"].cpu(), ref["intrinsics"]
    for nm, (i, j) in dict(fx=(0, 0), fy=(1, 1), cx=(0, 2), cy=(1, 2)).items():
        print(f"{nm}: rel err {((K[:, i, j]-Kr[:, i, j]).abs()/Kr[:, i, j].abs()).max().item():.3e}")
    # CUDA graph capture and replay must equal the eager call
    model.use_cuda_graph = True
    o2 = model.infer(rgb)
    o3 = model.infer(rgb)
    for k in out:
        e = (o2[k].float() - out[k].float()).abs().max().item()
        e3 = (o3[k].float() - o2[k].float()).abs().max().item()
        print(f"graph vs eager {k}: {e:.3e}; replay vs replay {e3:.3e}")


if __name__ == "__main__":
    main()
