"""Throughput of UniDepthV1 at several network shapes (`model.image_shape`), in one process on one GPU.

    python tools/bench_v1_shapes.py [--steps 10] [--warmup 3] [--runs 2] [--workloads v1,v1_vitl14] [--out DIR]

Workloads: UniDepthV1 ConvNeXt-L and UniDepthV1 ViT-L/14, each on 16 x 3x480x640 uint8 images with the seeded synthetic
weights tools/bench_fp8.py uses.  The config's shape and the new shapes alternate for --runs rounds in one process; at
each switch the script records the wall time of the first `infer` (a new engine, its workspace and a CUDA-graph capture,
but no weight repack: a packed weight keeps its address, which is checked), then times --steps CUDA-graph replays after
--warmup with CUDA events.  The card's name and power limit and the SM clock sampled during the timed steps are read in
the same process.  Prints one JSON line per workload and writes them to DIR/bench_v1_shapes.json when --out is given."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools")]

import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from bench_fp8 import build, card  # noqa: E402

# (config, new network shapes): the shapes of the reference goldens at other network shapes (tests/golden/v1_*_net*)
WORKLOADS = {"v1": ("config_v1_cnvnxtl.json", [[384, 512], [470, 630], [448, 448]]),
             "v1_vitl14": ("config_v1_vitl14.json", [[378, 504], [518, 686], [448, 448]])}
B, H, W = 16, 480, 640


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_v1_shapes needs a CUDA GPU")
    dev = torch.device("cuda", 0)
    lines = []
    for wl in args.workloads.split(","):
        cfg_name, new_shapes = WORKLOADS[wl]
        torch.cuda.empty_cache()
        model = build(cfg_name, dev)
        shapes = [list(model.image_shape)] + new_shapes
        g = torch.Generator().manual_seed(0)
        rgb = torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, generator=g).to(dev)
        model.infer(rgb)
        weight = next(iter(model._packed[0].values()))
        ptr = weight.data_ptr()
        ms = {str(s): [] for s in shapes}
        first_s = {str(s): [] for s in shapes}
        clocks = ClockSampler(0)
        clocks.start()
        for _ in range(args.runs):
            for shape in shapes:
                model.image_shape = list(shape)
                torch.cuda.synchronize()
                t = time.perf_counter()
                model.infer(rgb)
                torch.cuda.synchronize()
                first_s[str(shape)].append(time.perf_counter() - t)
                for _ in range(args.warmup):
                    model.infer(rgb)
                torch.cuda.synchronize()
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(args.steps):
                    model.infer(rgb)
                t1.record()
                torch.cuda.synchronize()
                ms[str(shape)].append(t0.elapsed_time(t1) / args.steps)
        clock = clocks.stop()
        repacked = model._packed[0] is None or next(iter(model._packed[0].values())).data_ptr() != ptr
        res = {}
        for s in shapes:
            med = statistics.median(ms[str(s)])
            res[str(s)] = dict(ms_per_step=round(med, 3), images_per_s=round(B / (med * 1e-3), 1),
                               runs_ms=[round(v, 3) for v in ms[str(s)]],
                               first_infer_after_change_s=[round(v, 3) for v in first_s[str(s)]])
        line = {"workload": wl, "batch": B, "input": [H, W], "default_shape": shapes[0], "shapes": res,
                "weights_repacked_on_shape_change": repacked, "card": card(), "clocks_during_timing": clock}
        print(json.dumps(line), flush=True)
        lines.append(line)
        del model
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_v1_shapes.json"), "w") as fh:
            json.dump(lines, fh, indent=1)


if __name__ == "__main__":
    main()
