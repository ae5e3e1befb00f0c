"""Throughput of UniDepthV1 ViT-L/14 next to UniDepthV1 ConvNeXt-L, measured in one process on one GPU.

    python tools/bench_v1_vit.py [--steps K] [--warmup W] [--batch B]

Both models run `infer` on the same 16 x 3 x 480 x 640 uint8 batch (seeded fixture weights, CUDA-graph replays).  The
timed loop alternates between the two models step by step, so clock or power drift hits both alike.  Warm-up and step
counts default to bench.py's.  One JSON line is printed with:
  - images/s of each model;
  - per-kernel time of one eager forward under the library's per-launch profile (udb_profile_begin / _end), split into
    GEMM, attention, the ViT tap kernel and the rest, with the algorithmic FLOPs and bytes the launches declare;
  - the card name, power limit and SM clock, read by nvidia-smi during the same run.
Nothing is written to disk."""
import argparse
import copy
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]

import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from unidepth_b200 import UniDepthV1, _cabi  # noqa: E402

MODELS = [("v1_vitl14", "config_v1_vitl14.json"), ("v1_cnvnxtl", "config_v1_cnvnxtl.json")]


def card(idx: int) -> dict:
    q = "name,power.limit,power.max_limit,clocks.sm,clocks.max.sm"
    try:
        f = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(idx)],
                           capture_output=True, text=True, timeout=20).stdout.strip().split(", ")
        return dict(name=f[0], power_limit_w=float(f[1]), power_max_limit_w=float(f[2]), sm_mhz_idle=float(f[3]),
                    sm_max_mhz=float(f[4]))
    except Exception as ex:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(idx), error=f"nvidia-smi: {ex}")


def build(cfg_name: str, dev):
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", cfg_name)))
    if "vitl14" in cfg_name:
        from unidepth_v1_vit_oracle import make_v1_vit_state_dict as make_sd
    else:
        from fixture import make_v1_state_dict as make_sd
    m = UniDepthV1(copy.deepcopy(cfg))
    m.load_state_dict(make_sd(cfg, 0), strict=True)
    return m.to(dev).eval()


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
               "vit_tap" if name.startswith("vit_tap") else "other")
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
    ap.add_argument("--batch", type=int, default=16)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    g = torch.Generator().manual_seed(0)
    rgb = torch.randint(0, 256, (args.batch, 3, 480, 640), dtype=torch.uint8, generator=g).to(dev)
    models = {name: build(cfg, dev) for name, cfg in MODELS}
    for m in models.values():          # outputs land in fixed buffers: no allocation inside the timed loop
        m.output_buffers = {"intrinsics": torch.empty(args.batch, 3, 3, device=dev),
                            "points": torch.empty(args.batch, 3, 480, 640, device=dev),
                            "depth": torch.empty(args.batch, 1, 480, 640, device=dev)}
        for _ in range(args.warmup):
            m.infer(rgb)
    torch.cuda.synchronize()
    ms = {name: 0.0 for name in models}
    sampler = ClockSampler(0)
    sampler.start()
    for _ in range(args.steps):
        for name, m in models.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            m.infer(rgb)
            e.record()
            e.synchronize()
            ms[name] += s.elapsed_time(e)
    clocks = sampler.stop()
    result = dict(metric="images/s", batch=args.batch, input="3x480x640 uint8", net_input="462x616", steps=args.steps,
                  warmup=args.warmup, card=card(0), clocks_during_timing=clocks, models={})
    for name, m in models.items():
        result["models"][name] = dict(images_per_s=round(args.steps * args.batch / (ms[name] / 1e3), 1),
                                      ms_per_step=round(ms[name] / args.steps, 3), kernels=kernel_split(m, rgb))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
