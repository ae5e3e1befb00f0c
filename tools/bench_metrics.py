"""Time the evaluation metrics on one GPU: the nearest-neighbour kernel (both directions in one pass) and eval_3d /
eval_depth end to end, against the same functions of oracle/eval_oracle.py run in torch on the same GPU.

    python tools/bench_metrics.py [--iters 10]

Prints the card, its power limit and SM clock (read while the NN kernel runs), then one table.  NN rate: point pairs
per second (one pair serves both directions).  Its share of the FP32-lane issue bound -- 132 SMs x 128 FP32 lanes x the
measured SM clock, in lane operations per second -- counts the 8 FP32 operations each pair needs (3 sub, 3 mul, 2 add);
the compares and selects of the two running minima are not counted, so 100 % is not reachable."""
import argparse
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import eval_oracle as O  # noqa: E402

from unidepth_b200 import ops, validation as V  # noqa: E402

DEV = "cuda:0"


def smi(field):
    try:
        return subprocess.check_output(["nvidia-smi", "-i", "0", f"--query-gpu={field}", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:    # the table is still useful without it
        return f"unavailable ({e.__class__.__name__})"


def timed(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def depth_inputs(B, H, W, g):
    gts = torch.rand(B, 1, H, W, generator=g) * 20 + 0.5
    preds = torch.nn.functional.interpolate(gts, size=(H // 2, W // 2), mode="area") * 1.05
    masks = torch.rand(B, 1, H, W, generator=g) < 0.6
    return gts.to(DEV), preds.to(DEV), masks.to(DEV)


def point_inputs(B, H, W, g):
    z = torch.rand(B, 1, H, W, generator=g) * 20 + 0.5
    gts = torch.cat([torch.randn(B, 2, H, W, generator=g) * z * 0.5, z], dim=1)
    preds = gts + 0.3 * torch.randn(gts.shape, generator=g)
    masks = torch.rand(B, 1, H, W, generator=g) < 0.6
    thr = torch.linspace(torch.log(torch.tensor(0.01)).item(), torch.log(torch.tensor(4.0)).item(), 100).exp()
    return gts.to(DEV), preds.to(DEV), masks.to(DEV), thr.to(DEV)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    print("card:", torch.cuda.get_device_name(0), "| power limit:", smi("power.limit"), "| max SM clock:",
          smi("clocks.max.sm"))
    g = torch.Generator().manual_seed(0)
    rows = []
    for N, P in ((1, 76800), (4, 19200)):
        x = (torch.randn(N, P, 3, generator=g) * 3).to(DEV)
        y = (x.cpu() + 0.1 * torch.randn(N, P, 3, generator=g)).to(DEV)
        ms = timed(lambda: ops.nearest_neighbor(x, y), a.iters)
        for _ in range(int(1500 / max(ms, 1e-3)) + 1):     # about 1.5 s of back-to-back launches to read the clock under
            ops.nearest_neighbor(x, y)
        time.sleep(0.5)
        clk = smi("clocks.sm")
        torch.cuda.synchronize()
        pairs = N * P * P
        mhz = float(clk.split()[0]) if clk[:1].isdigit() else float("nan")
        bound = 132 * 128 * mhz * 1e6
        rate = pairs / (ms * 1e-3)
        rows.append((f"NN both directions, {N} x {P}", ms, None,
                     f"{rate:.3e} pairs/s, SM clock {clk}, {100 * 8 * rate / bound:.1f} % of the FP32-lane issue bound"))
        oms = timed(lambda: (O.knn1(x, y, chunk=1024), O.knn1(y, x, chunk=1024)), 1, warmup=1)
        rows[-1] = rows[-1][:2] + (oms,) + rows[-1][3:]
    for name, (B, H, W) in (("NYU-like", (1, 480, 640)), ("KITTI-like", (4, 375, 1242))):
        gts, preds, masks, thr = point_inputs(B, H, W, g)
        ms = timed(lambda: V.eval_3d(gts, preds, masks, thr), a.iters)
        oms = timed(lambda: O.eval_3d(gts, preds, masks, thr), 1, warmup=1)
        rows.append((f"eval_3d {name} {B}x{H}x{W}", ms, oms, ""))
        gts, preds, masks = depth_inputs(B, H, W, g)
        ms = timed(lambda: V.eval_depth(gts, preds, masks, max_depth=15.0), a.iters)
        oms = timed(lambda: O.eval_depth(gts, preds, masks, max_depth=15.0), 2, warmup=1)
        rows.append((f"eval_depth {name} {B}x{H}x{W}", ms, oms, ""))
    print(f"| {'workload':<36} | {'kernel path ms':>14} | {'torch oracle ms':>15} | {'speed-up':>8} | notes")
    print(f"|{'-' * 38}|{'-' * 16}|{'-' * 17}|{'-' * 10}|------")
    for name, ms, oms, note in rows:
        print(f"| {name:<36} | {ms:>14.3f} | {oms:>15.1f} | {oms / ms:>7.1f}x | {note}")


if __name__ == "__main__":
    main()
