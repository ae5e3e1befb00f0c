"""What one evaluation step costs on one GPU, and where the time goes: `validation.validate` over a seeded UniDepthV2
ViT-L/14 (config_v2_vitl14, seeded weights) with batches of 8 normalised 3 x 490 x 644 network inputs and 480 x 640
ground truth (about 70 % valid pixels), alternating a Pinhole and a Fisheye624 camera.

    python tools/bench_validate.py [--batches 6] [--iters 20]

Prints the card and its power limit (read in the same run), then:
  * whole loop: images per second of validate end to end (forward, ground-truth points, metric accumulation, the final
    reduction), host clock around the loop, which ends in a device synchronise;
  * per batch: CUDA-event times of the forward, the ground-truth point map (validation.reconstruct), eval_depth and
    eval_3d, each timed on its own over the same batches;
  * reconstruct alone: udb_camera_reconstruct per camera model at 8 x 480 x 640 against camera.py's torch reconstruct of
    the same object on the same GPU."""
import argparse
import copy
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]

from unidepth_b200 import camera as C  # noqa: E402
from unidepth_b200 import validation as V  # noqa: E402

DEV = torch.device("cuda:0")
B, NET, GT = 8, (490, 644), (480, 640)


def smi(field):
    try:
        return subprocess.check_output(["nvidia-smi", "-i", "0", f"--query-gpu={field}", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:    # the numbers are still useful without it
        return f"unavailable ({e.__class__.__name__})"


def event_ms(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def cameras(kind, hw):
    h, w = hw
    if kind == "pinhole":
        return C.Pinhole(params=torch.tensor([[0.9 * w, 0.9 * w, w / 2, h / 2]]))
    return C.Fisheye624(params=torch.tensor([[0.5 * w, 0.5 * w, w / 2, h / 2, 0.03, -0.004, 0.001, 0.0, 0.0, 0.0,
                                              1e-3, -5e-4, 0.0, 0.0, 0.0, 0.0]]))


def make_batches(n):
    g = torch.Generator().manual_seed(0)
    mean = torch.tensor((0.485, 0.456, 0.406)).view(1, 3, 1, 1)
    std = torch.tensor((0.229, 0.224, 0.225)).view(1, 3, 1, 1)
    out = []
    for i in range(n):
        kind = ("pinhole", "fisheye")[i % 2]
        rgb = torch.randint(0, 256, (B, 3, *NET), generator=g).float().div(255).sub(mean).div(std)
        depth = torch.nn.functional.interpolate(torch.rand(B, 1, 30, 40, generator=g) * 9 + 1, size=GT, mode="bilinear")
        mask = torch.rand(B, 1, *GT, generator=g) < 0.7
        data = {"image": rgb[:, None], "depth": depth[:, None], "depth_mask": mask[:, None],
                "camera": cameras(kind, NET), "camera_original": cameras(kind, GT)}
        out.append({"data": data, "img_metas": [{"paddings": [[0, 0, 0, 0]]} for _ in range(B)]})
    return out


class Loader(list):
    dataset = None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=6)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_validate needs a GPU")
    from fixture import make_state_dict
    from unidepth_b200 import UniDepthV2
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "config_v2_vitl14.json")))
    model = UniDepthV2(copy.deepcopy(cfg))
    model.load_state_dict(make_state_dict(cfg, 0), strict=True)
    model = model.to(DEV).eval()
    print(f"card: {smi('name')}, power limit {smi('power.limit')}, max SM clock {smi('clocks.max.sm')}")

    batches = make_batches(args.batches)
    loader = Loader(batches)
    V.validate(model, {"warmup": loader})          # graphs, kernels and allocator warm
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = V.validate(model, {"bench": loader})
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    n_img = B * len(batches)
    print(f"whole loop: {n_img} images in {dt * 1e3:.1f} ms -> {n_img / dt:.1f} images/s ({len(res['bench'])} metrics)")

    # per batch, each stage on its own over the same (device-resident) batches
    dev_batches = []
    for b in batches:
        data = {k: (v.to(DEV).squeeze(1) if isinstance(v, torch.Tensor) else v.to(DEV)) for k, v in b["data"].items()}
        metas = [{k: v[0] for k, v in m.items()} for m in b["img_metas"]]
        with torch.no_grad():
            preds = model(data, metas)
        pts = V.reconstruct(data["camera_original"], data["depth"])
        dev_batches.append((data, metas, preds, pts))
    thr = torch.linspace(math.log(0.01), math.log(1000.0 / 20), steps=100, device=DEV).exp()
    stages = {
        "forward": lambda d, m, p, x: model(d, m),
        "reconstruct": lambda d, m, p, x: V.reconstruct(d["camera_original"], d["depth"]),
        "eval_depth": lambda d, m, p, x: V.eval_depth(d["depth"], p["depth"], d["depth_mask"], max_depth=1000.0),
        "eval_3d": lambda d, m, p, x: V.eval_3d(x, p["points"], d["depth_mask"], thresholds=thr),
    }
    with torch.no_grad():
        for name, fn in stages.items():
            per = [event_ms(lambda b=b: fn(*b), max(2, args.iters // 4)) for b in dev_batches]
            print(f"per batch of {B}: {name:12s} {sum(per) / len(per):9.3f} ms (min {min(per):.3f}, max {max(per):.3f})")

    # reconstruct alone at 8 x 480 x 640
    from test_camera_kernel_gpu import CAMERAS
    depth = (torch.rand(B, 1, *GT, generator=torch.Generator().manual_seed(1)) * 9 + 1).to(DEV)
    print(f"reconstruct alone, {B} x {GT[0]} x {GT[1]}: kernel vs camera.py's torch reconstruct")
    for name in ("pinhole", "eucm", "spherical", "opencv_strong", "fisheye_strong", "mei_strong"):
        cam = CAMERAS[name]().to(DEV)
        k = event_ms(lambda: V.reconstruct(cam, depth), args.iters)
        t = event_ms(lambda: cam.reconstruct(depth), max(2, args.iters // 4))
        gbs = (B * GT[0] * GT[1] * 16) / (k * 1e-3) / 1e9
        print(f"  {name:16s} kernel {k:8.3f} ms ({gbs:6.1f} GB/s of depth in + points out)   torch {t:9.3f} ms   "
              f"x{t / k:.1f}")


if __name__ == "__main__":
    main()
