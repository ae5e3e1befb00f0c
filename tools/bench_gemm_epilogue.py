"""Time the encoder's four GEMMs (ViT-L/14 at 8 x 480x640: M = 12888 tokens) on the general and on the TMA-store epilogue.

The two paths alternate within one process (UDB_GEMM_TMA_EPILOGUE=0 selects the general one), each measurement is
`--iters` back-to-back launches between CUDA events, and the median over `--rounds` is reported with its min-max range,
as TF/s and as GB/s of epilogue bytes (output + residual).
Usage (GPU): python tools/bench_gemm_epilogue.py [--rounds 7] [--iters 20] [--json OUT]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from unidepth_b200 import _cabi, ops

ENV = "UDB_GEMM_TMA_EPILOGUE"
M, D = 12888, 1024


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # informational only
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    x16 = torch.randn(M, D, device=dev, generator=g).half()
    mid = torch.randn(M, 4 * D, device=dev, generator=g).half()
    x32 = torch.randn(M, D, device=dev, generator=g)
    qkv = torch.empty(M, 3 * D, device=dev, dtype=torch.float16)
    h4 = torch.empty(M, 4 * D, device=dev, dtype=torch.float16)

    def w(n, k):
        return (torch.randn(n, k, device=dev, generator=g) / k ** 0.5).half()

    def vec(n):
        return torch.randn(n, device=dev, generator=g)

    wq, wp, w1, w2 = w(3 * D, D), w(D, D), w(4 * D, D), w(D, 4 * D)
    bq, bp, b1, b2, g1, g2 = vec(3 * D), vec(D), vec(4 * D), vec(D), vec(D) * 1e-3, vec(D) * 1e-3
    # name: (launch, N, K, epilogue bytes)
    gemms = {
        "qkv": (lambda: ops.gemm(x16, wq, bias=bq, out=qkv), 3 * D, D, M * 3 * D * 2),
        "proj": (lambda: ops.gemm(x16, wp, bias=bp, gamma=g1, resid=x32, out=x32), D, D, M * D * 8),
        "fc1": (lambda: ops.gemm(x16, w1, bias=b1, act=ops.ACT_GELU, out=h4), 4 * D, D, M * 4 * D * 2),
        "fc2": (lambda: ops.gemm(mid, w2, bias=b2, gamma=g2, resid=x32, out=x32), D, 4 * D, M * D * 8),
    }

    def time_path(fn, tma):
        os.environ[ENV] = "1" if tma else "0"
        fn()
        used = _cabi.lib().udb_gemm_tma_epilogue_used()
        assert used == int(tma), (tma, used)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(args.iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / args.iters

    for fn, *_ in gemms.values():            # warm both paths of every shape
        for tma in (False, True):
            for _ in range(3):
                time_path(fn, tma)
    times = {(n, t): [] for n in gemms for t in (False, True)}
    for _ in range(args.rounds):
        for n, (fn, *_) in gemms.items():
            for tma in (False, True):
                times[(n, tma)].append(time_path(fn, tma))
    os.environ.pop(ENV, None)

    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    res = {"gpu": info, "M": M, "rounds": args.rounds, "iters": args.iters, "gemms": {}}
    for n, (_, N, K, eb) in gemms.items():
        row = {}
        for tma in (False, True):
            ts = times[(n, tma)]
            ms = statistics.median(ts)
            row["tma" if tma else "general"] = {"ms": ms, "min_ms": min(ts), "max_ms": max(ts),
                                                "tflops": 2.0 * M * N * K / ms / 1e9, "epi_gbs": eb / ms / 1e6}
        gen, tm = row["general"], row["tma"]
        row["speedup"] = gen["ms"] / tm["ms"]
        res["gemms"][n] = row
        print(f"{n:5s} M{M} N{N} K{K}: general {gen['ms'] * 1e3:8.1f} us ({gen['min_ms'] * 1e3:.1f}-{gen['max_ms'] * 1e3:.1f}) "
              f"{gen['tflops']:6.1f} TF/s {gen['epi_gbs']:6.0f} GB/s | tma {tm['ms'] * 1e3:8.1f} us "
              f"({tm['min_ms'] * 1e3:.1f}-{tm['max_ms'] * 1e3:.1f}) {tm['tflops']:6.1f} TF/s {tm['epi_gbs']:6.0f} GB/s | "
              f"x{row['speedup']:.3f}", flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
