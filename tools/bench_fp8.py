"""UniDepthV2 ViT-L throughput with precision = "f16" against precision = "fp8", in one process on one GPU.

    python tools/bench_fp8.py [--steps 20] [--warmup 5] [--runs 3] [--out DIR]

For the default (8 x 480x640) and hires (4 x 1024x1536) workloads of bench.py, the two precisions alternate for --runs
runs each (CUDA-graph replay of `infer`, timed with CUDA events over --steps steps after --warmup).  It then profiles one
eager `infer` per precision with the library's per-launch profile (udb_profile_begin / _end) and reports the achieved
TF/s of the encoder blocks' four GEMMs (qkv, proj, fc1, fc2), from the flops each launcher declares.  The card's name,
power limit and SM clocks are read in the same process.  Prints one JSON line per workload and writes them to
DIR/bench_fp8.json when --out is given."""
import argparse
import copy
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

WORKLOADS = {"default": (8, 480, 640), "hires": (4, 1024, 1536)}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")])) if "," in out else {"query": out}


def encoder_gemms(model, rgb):
    """{layer: (ms, TF/s)} of the encoder blocks' qkv / proj / fc1 / fc2 GEMMs in one eager infer, from the profile."""
    from unidepth_b200 import _cabi
    s = model.spec
    model.use_cuda_graph = False
    model.infer(rgb)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    prof = _cabi.profile(lambda: model.infer(rgb), stream)
    model.use_cuda_graph = True
    gemms = [e for e in prof if e[0] in ("gemm_f16_kernel", "gemm_e4m3_kernel")]
    # the encoder's GEMMs are the 4 * depth launches after the patch embedding (the first GEMM), qkv / proj / fc1 / fc2
    # per block; in fp8 mode they are exactly the e4m3 launches
    if model.precision == "fp8":
        blocks = [e for e in gemms if e[0] == "gemm_e4m3_kernel"]
    else:
        blocks = gemms[1:1 + 4 * s.depth]
    res = {}
    assert len(blocks) == 4 * s.depth, len(blocks)
    for i, layer in enumerate(("qkv", "proj", "fc1", "fc2")):
        sel = blocks[i::4]
        ms = sum(e[1] for e in sel)
        fl = sum(e[2] for e in sel)
        res[layer] = dict(ms=round(ms, 3), tflops=round(fl / (ms * 1e-3) / 1e12, 1))
    res["encoder_gemms_ms"] = round(sum(e[1] for e in blocks), 3)
    res["all_kernels_ms"] = round(sum(e[1] for e in prof), 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8 needs a CUDA GPU")
    import warnings
    warnings.simplefilter("ignore")
    from unidepth_b200 import UniDepthV2
    from unidepth_b200.synthetic import synthetic_state_dict
    dev = torch.device("cuda", 0)
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "config_v2_vitl14.json")))
    model = UniDepthV2(copy.deepcopy(cfg))
    model.load_state_dict(synthetic_state_dict(cfg, 0, device=dev), strict=True)
    model = model.to(dev).eval()
    model.resolution_level = None
    info = card()
    lines = []
    for wl, (B, H, W) in WORKLOADS.items():
        g = torch.Generator().manual_seed(0)
        rgb = torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, generator=g).to(dev)
        ips = {"f16": [], "fp8": []}
        for _ in range(args.runs):
            for prec in ("f16", "fp8"):
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
                ips[prec].append(args.steps * B / (t0.elapsed_time(t1) / 1e3))
        prof = {}
        for prec in ("f16", "fp8"):
            model.precision = prec
            prof[prec] = encoder_gemms(model, rgb)
        line = dict(workload=wl, batch=B, input=f"{H}x{W}", steps=args.steps, runs=args.runs,
                    images_per_s={p: [round(v, 1) for v in ips[p]] for p in ips},
                    median_images_per_s={p: round(statistics.median(ips[p]), 1) for p in ips},
                    speedup=round(statistics.median(ips["fp8"]) / statistics.median(ips["f16"]), 3),
                    encoder_gemm_profile=prof, card=info)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_fp8.json"), "w") as fh:
            json.dump(lines, fh, indent=1)


if __name__ == "__main__":
    main()
