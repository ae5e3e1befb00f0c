"""Throughput of UniDepthV2old with precision = "f16", "split" and "fp8", in one process on one GPU.

    python tools/bench_v2old_precision.py [--steps 10] [--warmup 3] [--runs 3] [--batch 8] [--backbone vitl14|vits14] [--out DIR]

The workload is tools/bench_v2old.py's: B x 3 x 480 x 640 uint8 (default B = 8), seeded fixture weights, resolution_level
None (the maximum: a 588 x 784 network input).  The three precisions alternate for --runs runs each (CUDA-graph replay of
`infer` into fixed output buffers, timed with CUDA events over --steps steps after --warmup; switching precision repacks
the weights, which the warm-up absorbs).  After the timed runs, one eager `infer` per precision runs under the library's
per-launch profile; its first 1 + 4 * depth GEMM launches are the encoder's (patch embedding, then qkv, proj, fc1 and fc2
of every block), and their summed time is reported as the encoder-GEMM ms per step.  The card's name, power limit and SM
clocks are read in the same process.  Prints one JSON line, and writes it to DIR/bench_v2old_precision.json when --out
is given."""
import argparse
import ctypes as C
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
from make_golden_v2old import make_v2old_state_dict  # noqa: E402
from unidepth_b200 import UniDepthV2old, _cabi  # noqa: E402

PRECISIONS = ("f16", "split", "fp8")


def encoder_gemm_ms(m, rgb) -> dict:
    """One eager `infer` under the per-launch profile -> encoder GEMM ms and launches, and the step's total kernel ms."""
    m.use_cuda_graph = False
    m.infer(rgb)
    torch.cuda.synchronize()
    torch.cuda._sleep(int(0.15 * 1.9e9))      # keeps the GPU busy while the host enqueues: events bracket kernels, not gaps
    prof = _cabi.profile(lambda: m.infer(rgb), C.c_void_p(torch.cuda.current_stream().cuda_stream), cap=16384)
    torch.cuda.synchronize()
    m.use_cuda_graph = True
    n_enc = 1 + 4 * m.spec.enc_depth
    gemms = [ms for name, ms, _, _ in prof if name.startswith("gemm")][:n_enc]
    return dict(encoder_gemm_ms=round(sum(gemms), 3), encoder_gemm_launches=len(gemms),
                all_kernels_ms=round(sum(ms for _, ms, _, _ in prof), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--backbone", default="vitl14", choices=("vitl14", "vits14"))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_v2old_precision.py measures on a CUDA device; none is visible")
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
    ms = {p: [] for p in PRECISIONS}
    sampler = ClockSampler(0)
    sampler.start()
    for _ in range(args.runs):
        for prec in PRECISIONS:
            m.precision = prec
            for _ in range(args.warmup):
                m.infer(rgb)
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.steps):
                m.infer(rgb)
            t1.record()
            torch.cuda.synchronize()
            ms[prec].append(t0.elapsed_time(t1) / args.steps)
    clocks = sampler.stop()
    med = {p: statistics.median(v) for p, v in ms.items()}
    profiles = {}
    for prec in PRECISIONS:
        m.precision = prec
        profiles[prec] = encoder_gemm_ms(m, rgb)
    net = m._engine_key
    line = dict(model=f"v2old_{args.backbone}", batch=B, input="3x480x640 uint8", net_input=f"{net[0]}x{net[1]}",
                steps=args.steps, warmup=args.warmup, runs=args.runs, card=card(), clocks_during_timing=clocks,
                ms_per_step=med, runs_ms=ms, images_per_s={p: round(B / (v / 1e3), 1) for p, v in med.items()},
                over_f16={p: round(med[p] / med["f16"], 3) for p in PRECISIONS}, profile_eager=profiles)
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_v2old_precision.json"), "w") as fh:
            json.dump(line, fh, indent=1)


if __name__ == "__main__":
    main()
