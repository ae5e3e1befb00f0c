"""UniDepthV2's evaluation forward, old path against new, in one process on one GPU.

    python tools/bench_v2_forward.py [--steps 20] [--warmup 5] [--runs 3] [--batch 8] [--backbone vitl14|vits14] [--out DIR]

The workload is one evaluation step of the reference's loop at the benchmark's network size: a normalised B x 3 x 490 x 644
network input (what `infer` makes of a 480 x 640 image, default B = 8), a 480 x 640 ground truth and paddings that differ
per image, seeded fixture weights.
  old: the graphed network-only call (`network_forward`'s path) followed by `validation.match_gt` on depth, points and
       confidence and `match_intrinsics`, per image in torch, and the rays renormalised in torch (the parent's
       `forward_test`);
  new: `forward_test`, one graphed engine call whose last kernel writes the matched outputs.
The two alternate for --runs runs each, timed with CUDA events over --steps steps after --warmup.  The outputs of both are
compared.  The card's name, power limit and SM clocks are read in the same process.  Prints one JSON line, and writes it to
DIR/bench_v2_forward.json when --out is given."""
import argparse
import copy
import json
import os
import statistics
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools")]

import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from bench_fp8 import card  # noqa: E402
from fixture import make_state_dict  # noqa: E402
from unidepth_b200 import UniDepthV2  # noqa: E402
from unidepth_b200.validation import match_gt, match_intrinsics  # noqa: E402


def old_step(m, x, gt, pads):
    out = m._network_outputs(x)
    res = {k: match_gt(out[k], gt, padding1=pads, padding2=None) for k in ("depth", "points", "confidence")}
    res["rays"] = out["rays"] / torch.norm(out["rays"], dim=1, keepdim=True).clip(min=1e-5)
    res["intrinsics"] = match_intrinsics(out["intrinsics"], x, gt, padding1=pads, padding2=None)
    return res


def timed(fn, steps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--backbone", default="vitl14", choices=("vitl14", "vits14"))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_v2_forward needs a GPU")
    warnings.simplefilter("ignore")
    dev = torch.device("cuda:0")
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", f"config_v2_{args.backbone}.json")))
    m = UniDepthV2(copy.deepcopy(cfg))
    m.load_state_dict(make_state_dict(cfg, 0), strict=True)
    m = m.to(dev).eval()
    B, h, w, H, W = args.batch, 490, 644, 480, 640
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 3, h, w, generator=g).to(dev)
    gt = torch.zeros(B, 1, H, W, device=dev)
    pads = [(i % 3, (2 * i) % 5, i % 4, (3 * i) % 7) for i in range(B)]    # (l, r, t, b), one per image
    fns = {"old": lambda: old_step(m, x, gt, pads), "new": lambda: m({"image": x, "depth": gt, "paddings": pads}, [])}
    ref, new = fns["old"](), fns["new"]()
    torch.cuda.synchronize()
    diff = {k: (new[k] - ref[k]).abs().max().item() for k in ref}
    ms = {k: [] for k in fns}
    clocks = ClockSampler()
    clocks.start()
    for _ in range(args.runs):
        for k, fn in fns.items():
            for _ in range(args.warmup):
                fn()
            torch.cuda.synchronize()
            ms[k].append(timed(fn, args.steps))
    clk = clocks.stop()
    res = {"workload": f"{args.backbone} B={B} net {h}x{w} -> gt {H}x{W}", "card": card(), "clocks": clk,
           "ms_per_step": ms, "median_ms": {k: statistics.median(v) for k, v in ms.items()},
           "speedup_old_over_new": statistics.median(ms["old"]) / statistics.median(ms["new"]),
           "max_abs_diff_new_vs_old": diff}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "bench_v2_forward.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
