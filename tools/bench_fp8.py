"""Throughput with precision = "f16" against precision = "fp8", in one process on one GPU.

    python tools/bench_fp8.py [--steps 20] [--warmup 5] [--runs 3] [--workloads default,hires,v1,v1_vitl14] [--out DIR]

Workloads: UniDepthV2 ViT-L at bench.py's default (8 x 480x640) and hires (4 x 1024x1536) shapes, UniDepthV1 ConvNeXt-L
at bench.py's v1 shape (16 x 480x640) and UniDepthV1 ViT-L at the same shape (as tools/bench_v1_vit.py), all with seeded
synthetic weights.  For each, the two precisions alternate for --runs runs each (CUDA-graph replay of `infer`, timed with
CUDA events over --steps steps after --warmup) while nvidia-smi samples the SM clock.  It then profiles one eager `infer`
per precision with the library's per-launch profile (udb_profile_begin / _end) and reports, from the flops and bytes each
launcher declares:
  - ViT encoders: the achieved TF/s of the blocks' four GEMMs (qkv, proj, fc1, fc2);
  - ConvNeXt-L: per stage, the TF/s of the blocks' two MLP GEMMs, the time of the rest of the blocks, and the depthwise
    7x7 kernel's achieved GB/s (in fp8 mode the fused udb_dwconv7_ln_e4m3) against the H100's 3.35 TB/s.
The card's name, power limit and SM clocks are read in the same process.  Prints one JSON line per workload and writes
them to DIR/bench_fp8.json when --out is given."""
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

from bench import ClockSampler  # noqa: E402

# workload -> (config, batch, H, W)
WORKLOADS = {"default": ("config_v2_vitl14.json", 8, 480, 640), "hires": ("config_v2_vitl14.json", 4, 1024, 1536),
             "v1": ("config_v1_cnvnxtl.json", 16, 480, 640), "v1_vitl14": ("config_v1_vitl14.json", 16, 480, 640)}
HBM_GBPS = 3350.0                      # H100 SXM data sheet
GEMMS = ("gemm_f16_kernel", "gemm_e4m3_kernel")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")])) if "," in out else {"query": out}


def _profile(model, rgb):
    """[(kernel, ms, flops, bytes)] of one eager infer, after one warm-up call."""
    from unidepth_b200 import _cabi
    model.use_cuda_graph = False
    model.infer(rgb)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    prof = _cabi.profile(lambda: model.infer(rgb), stream, cap=16384)
    model.use_cuda_graph = True
    return prof


def encoder_gemms(model, rgb, depth):
    """{layer: (ms, TF/s)} of the ViT encoder blocks' qkv / proj / fc1 / fc2 GEMMs in one eager infer, from the profile."""
    prof = _profile(model, rgb)
    gemms = [e for e in prof if e[0] in GEMMS]
    # the encoder's GEMMs are the 4 * depth launches after the patch embedding (the first GEMM), qkv / proj / fc1 / fc2
    # per block; in fp8 mode they are exactly the e4m3 launches
    if model.precision == "fp8":
        blocks = [e for e in gemms if e[0] == "gemm_e4m3_kernel"]
    else:
        blocks = gemms[1:1 + 4 * depth]
    res = {}
    assert len(blocks) == 4 * depth, len(blocks)
    for i, layer in enumerate(("qkv", "proj", "fc1", "fc2")):
        sel = blocks[i::4]
        ms = sum(e[1] for e in sel)
        fl = sum(e[2] for e in sel)
        res[layer] = dict(ms=round(ms, 3), tflops=round(fl / (ms * 1e-3) / 1e12, 1))
    res["encoder_gemms_ms"] = round(sum(e[1] for e in blocks), 3)
    res["all_kernels_ms"] = round(sum(e[1] for e in prof), 3)
    return res


def convnext_stages(model, rgb):
    """Per ConvNeXt stage of one eager infer: the blocks' two MLP GEMMs (ms, TF/s), the depthwise 7x7 kernel (ms, achieved
    GB/s and its share of HBM bandwidth; the fused dwconv + LayerNorm + e4m3 kernel in fp8 mode) and the rest of the
    blocks (LayerNorm or quantiser, running max, cls means).  A block starts at its depthwise launch; the first two GEMMs
    after it are fc1 and fc2; the encoder's blocks are the first sum(depths) depthwise launches."""
    prof = _profile(model, rgb)
    depths = model.spec.depths
    stage_of = [i for i, d in enumerate(depths) for _ in range(d)]
    acc = [dict(gemm_ms=0.0, gemm_flops=0.0, dw_ms=0.0, dw_bytes=0.0, rest_ms=0.0) for _ in depths]
    blk, pending = -1, 0
    for name, ms, fl, by in prof:
        if name in ("dwconv7_kernel", "dwconv7_ln_e4m3_kernel"):
            blk += 1
            if blk == len(stage_of):
                break
            st = acc[stage_of[blk]]
            st["dw_ms"] += ms
            st["dw_bytes"] += by
            pending = 2
        elif blk < 0:
            continue
        elif name in GEMMS and pending:
            st["gemm_ms"] += ms
            st["gemm_flops"] += fl
            pending -= 1
        elif pending or name in ("max_accum_kernel", "spatial_mean_kernel"):
            st["rest_ms"] += ms
    res = {}
    for i, st in enumerate(acc):
        gbps = st["dw_bytes"] / (st["dw_ms"] * 1e-3) / 1e9
        res[f"stage{i}"] = dict(blocks=depths[i], width=model.spec.dims[i], mlp_gemm_ms=round(st["gemm_ms"], 3),
                                mlp_gemm_tflops=round(st["gemm_flops"] / (st["gemm_ms"] * 1e-3) / 1e12, 1),
                                dwconv_ms=round(st["dw_ms"], 3), dwconv_gbps=round(gbps, 1),
                                dwconv_share_of_hbm=round(gbps / HBM_GBPS, 3), rest_ms=round(st["rest_ms"], 3),
                                block_ms=round(st["gemm_ms"] + st["dw_ms"] + st["rest_ms"], 3))
    res["all_kernels_ms"] = round(sum(e[1] for e in prof), 3)
    return res


def build(cfg_name, dev):
    from unidepth_b200 import UniDepthV1, UniDepthV2
    from unidepth_b200.synthetic import synthetic_state_dict, synthetic_state_dict_v1
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", cfg_name)))
    if cfg_name.startswith("config_v1"):
        model = UniDepthV1(copy.deepcopy(cfg))
        if "vitl14" in cfg_name:          # tools/bench_v1_vit.py's weights
            from unidepth_v1_vit_oracle import make_v1_vit_state_dict
            model.load_state_dict(make_v1_vit_state_dict(cfg, 0), strict=True)
        else:
            model.load_state_dict(synthetic_state_dict_v1(cfg, 0, device=dev), strict=True)
        return model.to(dev).eval()
    model = UniDepthV2(copy.deepcopy(cfg))
    model.load_state_dict(synthetic_state_dict(cfg, 0, device=dev), strict=True)
    model = model.to(dev).eval()
    model.resolution_level = None
    return model


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8 needs a CUDA GPU")
    import warnings
    warnings.simplefilter("ignore")
    dev = torch.device("cuda", 0)
    info = card()
    lines = []
    models = {}
    for wl in args.workloads.split(","):
        cfg_name, B, H, W = WORKLOADS[wl]
        if cfg_name not in models:
            models.clear()                    # one model on the device at a time
            torch.cuda.empty_cache()
            models[cfg_name] = build(cfg_name, dev)
        model = models[cfg_name]
        g = torch.Generator().manual_seed(0)
        rgb = torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8, generator=g).to(dev)
        ips = {"f16": [], "fp8": []}
        clocks = ClockSampler(0)
        clocks.start()
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
        clock = clocks.stop()
        prof = {}
        for prec in ("f16", "fp8"):
            model.precision = prec
            if cfg_name == "config_v1_cnvnxtl.json":
                prof[prec] = convnext_stages(model, rgb)
            else:
                prof[prec] = encoder_gemms(model, rgb, model.spec.enc_depth if cfg_name.startswith("config_v1") else model.spec.depth)
        line = dict(workload=wl, config=cfg_name, batch=B, input=f"{H}x{W}", steps=args.steps, runs=args.runs,
                    images_per_s={p: [round(v, 1) for v in ips[p]] for p in ips},
                    median_images_per_s={p: round(statistics.median(ips[p]), 1) for p in ips},
                    speedup=round(statistics.median(ips["fp8"]) / statistics.median(ips["f16"]), 3),
                    encoder_profile=prof, card=info, clocks_during_timing=clock)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_fp8.json"), "w") as fh:
            json.dump(lines, fh, indent=1)


if __name__ == "__main__":
    main()
