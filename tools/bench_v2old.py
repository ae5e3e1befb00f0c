"""Throughput of UniDepthV2old ViT-L/14 on one GPU.

    python tools/bench_v2old.py [--steps K] [--warmup W] [--batch B] [--backbone vitl14|vits14]

`infer` runs on a B x 3 x 480 x 640 uint8 batch (default B = 8; seeded fixture weights; resolution_level None, i.e. the
maximum, a 588 x 784 network input; CUDA-graph replays into fixed output buffers).  One JSON line is printed with:
  - images/s and ms per step, from CUDA events around each replay;
  - per-kernel time of one eager forward under the library's per-launch profile (udb_profile_begin / _end), split into
    GEMM, attention, the V2old kernels (pixel-shuffle depthwise conv, heads, tail, output assembly) and the rest, with the
    algorithmic FLOPs and bytes the launches declare;
  - the card name, power limit and SM clocks / throttle reasons sampled during the timed loop (bench.py's ClockSampler).
Nothing is written to disk."""
import argparse
import ctypes as C
import json
import os
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools")]

import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from bench_v1_vit import card  # noqa: E402
from make_golden_v2old import make_v2old_state_dict  # noqa: E402
from unidepth_b200 import UniDepthV2old, _cabi  # noqa: E402

V2OLD_KERNELS = ("pshuffle", "v2old", "ray_embed")


def kernel_split(m, rgb) -> dict:
    """One eager forward under the per-launch profile -> {category: ms, launches, GFLOP, GB, TFLOP/s, GB/s}."""
    m.use_cuda_graph = False
    torch.cuda.synchronize()
    torch.cuda._sleep(int(0.15 * 1.9e9))      # keeps the GPU busy while the host enqueues: events bracket kernels, not gaps
    prof = _cabi.profile(lambda: m.infer(rgb), C.c_void_p(torch.cuda.current_stream().cuda_stream), cap=16384)
    torch.cuda.synchronize()
    m.use_cuda_graph = True
    cats = {}
    for name, ms, flops, nbytes in prof:
        key = ("gemm" if name.startswith("gemm") else "attention" if name.startswith("attn") else
               "v2old_kernels" if name.startswith(V2OLD_KERNELS) else "other")
        a = cats.setdefault(key, dict(ms=0.0, launches=0, gflop=0.0, gb=0.0))
        a["ms"] += ms
        a["launches"] += 1
        a["gflop"] += flops / 1e9
        a["gb"] += nbytes / 1e9
    for a in cats.values():
        a["tflops"] = round(a["gflop"] / a["ms"], 1) if a["ms"] > 0 else None
        a["gbps"] = round(a["gb"] / a["ms"] * 1e3, 1) if a["ms"] > 0 else None
        for k in ("ms", "gflop", "gb"):
            a[k] = round(a[k], 3)
    return cats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--backbone", default="vitl14", choices=("vitl14", "vits14"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_v2old.py measures on a CUDA device; none is visible")
    warnings.simplefilter("ignore")       # resolution_level None warns on every call, as the reference does
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", f"config_v2old_{args.backbone}.json")))
    m = UniDepthV2old(cfg)
    m.load_state_dict(make_v2old_state_dict(cfg, 0), strict=True)
    m = m.to(dev).eval()
    g = torch.Generator().manual_seed(0)
    B = args.batch
    rgb = torch.randint(0, 256, (B, 3, 480, 640), dtype=torch.uint8, generator=g).to(dev)
    m.output_buffers = {"intrinsics": torch.empty(B, 3, 3, device=dev), "points": torch.empty(B, 3, 480, 640, device=dev),
                        "depth": torch.empty(B, 1, 480, 640, device=dev), "confidence": torch.empty(B, 1, 480, 640, device=dev)}
    for _ in range(args.warmup):
        m.infer(rgb)
    torch.cuda.synchronize()
    ms = 0.0
    sampler = ClockSampler(0)
    sampler.start()
    for _ in range(args.steps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        m.infer(rgb)
        e.record()
        e.synchronize()
        ms += s.elapsed_time(e)
    clocks = sampler.stop()
    net = m._engine_key
    print(json.dumps(dict(metric="images/s", model=f"v2old_{args.backbone}", batch=B, input="3x480x640 uint8",
                          net_input=f"{net[0]}x{net[1]}", steps=args.steps, warmup=args.warmup, card=card(0),
                          clocks_during_timing=clocks, images_per_s=round(args.steps * B / (ms / 1e3), 1),
                          ms_per_step=round(ms / args.steps, 3), kernels=kernel_split(m, rgb))))


if __name__ == "__main__":
    main()
