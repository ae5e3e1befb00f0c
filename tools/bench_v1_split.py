"""Time per step of UniDepthV1 with precision = "split" against precision = "f16", in one process on one GPU.

    python tools/bench_v1_split.py [--steps 10] [--warmup 3] [--runs 3] [--workloads v1,v1_vitl14] [--out DIR]

Workloads: UniDepthV1 ConvNeXt-L and UniDepthV1 ViT-L/14, each at 16 x 480x640 with the seeded synthetic weights
tools/bench_fp8.py uses.  The two precisions alternate for --runs runs each (CUDA-graph replay of `infer`, timed with CUDA
events over --steps steps after --warmup; switching precision repacks the weights, which the warm-up absorbs).  Split
mode is a parity / debugging mode, not a speed mode: this measures what it costs.  The card's name, power limit and SM
clocks are read in the same process.  Prints one JSON line per workload and writes them to DIR/bench_v1_split.json when
--out is given."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools")]

import torch  # noqa: E402

from bench_fp8 import build, card  # noqa: E402

WORKLOADS = {"v1": ("config_v1_cnvnxtl.json", 16, 480, 640), "v1_vitl14": ("config_v1_vitl14.json", 16, 480, 640)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_v1_split needs a CUDA GPU")
    dev = torch.device("cuda", 0)
    lines = []
    for wl in args.workloads.split(","):
        cfg_name, B, H, W = WORKLOADS[wl]
        torch.cuda.empty_cache()
        model = build(cfg_name, dev)
        g = torch.Generator().manual_seed(0)
        rgb = torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, generator=g).to(dev)
        ms = {"f16": [], "split": []}
        for _ in range(args.runs):
            for prec in ("f16", "split"):
                model.precision = prec
                for _ in range(args.warmup):
                    model.infer(rgb)
                torch.cuda.synchronize()
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(args.steps):
                    model.infer(rgb)
                t1.record()
                torch.cuda.synchronize()
                ms[prec].append(t0.elapsed_time(t1) / args.steps)
        med = {k: statistics.median(v) for k, v in ms.items()}
        line = {"workload": wl, "batch": B, "shape": [H, W], "ms_per_step": med, "runs_ms": ms,
                "split_over_f16": med["split"] / med["f16"], "card": card()}
        print(json.dumps(line), flush=True)
        lines.append(line)
        del model
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_v1_split.json"), "w") as fh:
            json.dump(lines, fh, indent=1)


if __name__ == "__main__":
    main()
