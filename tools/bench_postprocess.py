"""Time the output assembly (udb_postprocess) in bilinear and bicubic mode, and the share it takes of a whole UniDepthV2 step.

Kernel: the three V2 shapes the benchmark and users run -- 8 x 480x640 (network 490x644), 4 x 1024x1536 (network 644x952,
upsampling) and 8 x 120x160 (network 392x518, downsampling) -- with analytic rays from intr4 as in a plain `infer`.  The two
modes alternate within one process; each measurement is `--iters` back-to-back launches between CUDA events, and the
median over `--rounds` is reported with its min-max range and the bytes the kernel must move (network maps read once,
nine f32 output planes written) per second.

Step: UniDepthV2 ViT-L/14 (fixture weights), 8 x 480x640, in each mode: images/s of CUDA-graph replays between events,
and one eager pass under the library's per-launch profile (udb_profile_begin / _end) for the postprocessing share.
Usage (GPU): python tools/bench_postprocess.py [--rounds 7] [--iters 50] [--steps 20] [--json OUT]"""
import argparse
import copy
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import torch  # noqa: E402

from unidepth_b200 import _cabi, ops, spec  # noqa: E402

MODES = ("bilinear", "bicubic")
KERNELS = {"bilinear": "postprocess_kernel", "bicubic": "postprocess_bicubic_kernel"}
SHAPES = {"default_8x480x640": (8, 480, 640), "hires_4x1024x1536": (4, 1024, 1536), "small_8x120x160": (8, 120, 160)}
BOUNDS = {"pixels_min": 200000, "pixels_max": 600000}


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # informational only
        return f"unavailable ({e})"


def kernel_case(B, H, W, dev):
    pads, padded = spec.get_paddings((H, W), (0.5, 2.5))
    _, (nh, nw) = spec.get_resize_factor(padded, spec.pixel_bounds(BOUNDS, None))
    g = torch.Generator(device=dev).manual_seed(0)
    radius = torch.rand(B, nh, nw, device=dev, generator=g) * 10 + 1
    conf = torch.rand(B, nh, nw, device=dev, generator=g) + 0.5
    intr4 = torch.tensor([[0.8 * nw, 0.8 * nw, nw / 2, nh / 2]] * B, device=dev)
    nbytes = 4.0 * B * (2 * nh * nw + 9 * H * W)
    return (lambda mode: ops.postprocess(radius, conf, intr4, B, (nh, nw), padded, pads[0], pads[2], (H, W), mode=mode)), \
        (nh, nw), nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"gpu_before": gpu_info(), "rounds": args.rounds, "iters": args.iters, "kernel": {}, "step": {}}

    def timed(fn, n):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(n):
            fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / n

    cases = {name: kernel_case(*shape, dev) for name, shape in SHAPES.items()}
    for fn, _, _ in cases.values():
        for mode in MODES:
            timed(lambda: fn(mode), 5)
    times = {(n, m): [] for n in cases for m in MODES}
    for _ in range(args.rounds):
        for n, (fn, _, _) in cases.items():
            for mode in MODES:
                times[(n, mode)].append(timed(lambda: fn(mode), args.iters))
    for n, (_, net, nbytes) in cases.items():
        row = {"net_hw": list(net), "bytes": nbytes}
        for mode in MODES:
            ts = times[(n, mode)]
            ms = statistics.median(ts)
            row[mode] = {"us": ms * 1e3, "min_us": min(ts) * 1e3, "max_us": max(ts) * 1e3, "gbs": nbytes / ms / 1e6}
        res["kernel"][n] = row
        bl, bc = row["bilinear"], row["bicubic"]
        print(f"{n} (network {net[0]}x{net[1]}, {nbytes / 1e6:.1f} MB): bilinear {bl['us']:.1f} us "
              f"({bl['min_us']:.1f}-{bl['max_us']:.1f}, {bl['gbs']:.0f} GB/s) | bicubic {bc['us']:.1f} us "
              f"({bc['min_us']:.1f}-{bc['max_us']:.1f}, {bc['gbs']:.0f} GB/s) | x{bc['us'] / bl['us']:.2f}", flush=True)

    # whole step, default workload
    from fixture import make_state_dict
    from unidepth_b200 import UniDepthV2
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "config_v2_vitl14.json")))
    m = UniDepthV2(copy.deepcopy(cfg))
    m.load_state_dict(make_state_dict(cfg, 0), strict=True)
    m = m.to(dev).eval()
    m.resolution_level = None
    B = 8
    rgb = torch.randint(0, 256, (B, 3, 480, 640), dtype=torch.uint8, generator=torch.Generator().manual_seed(0)).to(dev)
    for mode in MODES:
        m.interpolation_mode = mode
        for _ in range(3):
            m.infer(rgb)
    step = {mode: [] for mode in MODES}
    for _ in range(3):
        for mode in MODES:
            m.interpolation_mode = mode
            step[mode].append(timed(lambda: m.infer(rgb), args.steps))
    for mode in MODES:
        m.interpolation_mode = mode
        m.use_cuda_graph = False
        torch.cuda._sleep(int(0.15 * 1.9e9))      # keep the GPU busy while the eager pass is enqueued
        prof = _cabi.profile(lambda: m.infer(rgb), C.c_void_p(torch.cuda.current_stream().cuda_stream), cap=8192)
        torch.cuda.synchronize()
        m.use_cuda_graph = True
        tot = sum(p[1] for p in prof)
        post = sum(p[1] for p in prof if p[0] == KERNELS[mode])
        ms = statistics.median(step[mode])
        res["step"][mode] = {"graph_ms": ms, "graph_ms_runs": step[mode], "images_per_s": B / ms * 1e3,
                             "profiled_ms": tot, "postprocess_ms": post, "postprocess_share": post / tot,
                             "profiled_images_per_s": B / tot * 1e3}
        print(f"step {mode}: {B / ms * 1e3:.1f} images/s (graph, {ms:.2f} ms/step, runs {[round(t, 2) for t in step[mode]]}); "
              f"profiled eager pass {tot:.2f} ms ({B / tot * 1e3:.1f} images/s), {KERNELS[mode]} {post * 1e3:.1f} us "
              f"= {100 * post / tot:.3f} %", flush=True)
    res["gpu_after"] = gpu_info()
    print(f"GPU before: {res['gpu_before']}\nGPU after:  {res['gpu_after']}", flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
