"""Time camera-conditioned UniDepthV2.infer, and the GT-camera ray generator (udb_camera_rays) on its own.

Calls: UniDepthV2 ViT-L/14 (fixture weights) on 480x640 uint8 images, B = 1 and B = 8.  Five cases alternate within one
process, round by round:
    none           no camera                                            CUDA graph
    K_eager        camera = K tensor                                    use_cuda_graph = False (launch by launch)
    K_graph        camera = K tensor                                    CUDA graph
    fisheye_host   Fisheye624 behind a thin duck-typed wrapper: rays    use_cuda_graph = False
                   from the object's own torch code on the host side
    fisheye_dev    Fisheye624 object: rays from udb_camera_rays         CUDA graph
Each call is timed with the host clock between two device synchronisations (what a caller waits for); the median over
all calls and its min-max range are reported.

Kernel: udb_camera_rays for each camera model at 8 x 490x644 (the network input of 8 x 480x640), `--iters` launches
between CUDA events per round, median over `--rounds`, and the 12 bytes per pixel it must write per second.
Usage (GPU): python tools/bench_camera.py [--rounds 7] [--calls 10] [--iters 50] [--json OUT]"""
import argparse
import copy
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import torch  # noqa: E402

from unidepth_b200 import _cabi  # noqa: E402
from unidepth_b200 import camera as cam_mod  # noqa: E402


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # informational only
        return f"unavailable ({e})"


def _p16(fx, fy, cx, cy, radial, tang, prism):
    return torch.tensor([[fx, fy, cx, cy, *radial, *tang, *prism]], dtype=torch.float32)


# cameras in input-image pixels for 480 x 640 images
MODELS = {
    "pinhole": lambda: cam_mod.Pinhole(params=torch.tensor([[520.0, 515.0, 321.5, 238.25]])),
    "eucm": lambda: cam_mod.EUCM(params=torch.tensor([[300.0, 302.0, 320.0, 241.0, 0.62, 1.05]])),
    "spherical": lambda: cam_mod.Spherical(params=torch.tensor([[100.0, 100.0, 320.0, 240.0, 640.0, 480.0, 3.0, 1.2]])),
    "opencv": lambda: cam_mod.OPENCV(params=_p16(260.0, 262.0, 322.0, 236.0, (-0.32, 0.11, -0.018, 0.0, 0.0, 0.0),
                                                 (1.5e-3, -8e-4), (2e-3, -1e-3, 1e-3, 5e-4))),
    "fisheye624": lambda: cam_mod.Fisheye624(params=_p16(180.0, 181.0, 321.0, 239.0,
                                                         (0.05, -0.012, 0.004, -6e-4, 4e-5, -1e-6), (2e-3, -1e-3),
                                                         (1e-3, -5e-4, 8e-4, -2e-4))),
    "mei": lambda: cam_mod.MEI(params=torch.tensor([[420.0, 421.0, 319.0, 241.0, -0.22, 0.06, 2e-3, -1e-3, 1.3]])),
}


class HostCamera:
    """Duck-typed wrapper: the packer does not know it, so infer generates its rays with the object's own methods."""

    def __init__(self, cam):
        self.cam = copy.deepcopy(cam)

    def to(self, device):
        self.cam = self.cam.to(device)
        return self

    def crop(self, left, top, right=None, bottom=None):
        self.cam = self.cam.crop(left, top, right, bottom)
        return self

    def resize(self, factor):
        self.cam = self.cam.resize(factor)
        return self

    def get_rays(self, shapes):
        return self.cam.get_rays(shapes)


def kernel_times(dev, rounds, iters):
    lib = _cabi.lib()
    B, nh, nw = 8, 490, 644
    pads, factor = (0, 0, 0, 0), 1.0208
    out = torch.empty(B * nh * nw * 3, device=dev)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    res = {}
    for name, make in MODELS.items():
        model, rows = cam_mod.pack_camera(make())
        rows = rows.to(dev).expand(B, _cabi.CAM_STRIDE).contiguous()

        def launch():
            _cabi.check(lib.udb_camera_rays(model, C.c_void_p(rows.data_ptr()), B, nh, nw, *pads, C.c_float(factor),
                                            C.c_void_p(out.data_ptr()), st), "udb_camera_rays")

        for _ in range(5):
            launch()
        ts = []
        for _ in range(rounds):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                launch()
            e.record()
            torch.cuda.synchronize()
            ts.append(s.elapsed_time(e) / iters)
        ms = statistics.median(ts)
        nbytes = 12.0 * B * nh * nw
        res[name] = {"us": ms * 1e3, "min_us": min(ts) * 1e3, "max_us": max(ts) * 1e3, "gbs": nbytes / ms / 1e6}
        r = res[name]
        print(f"udb_camera_rays {name} 8x490x644: {r['us']:.1f} us ({r['min_us']:.1f}-{r['max_us']:.1f}), "
              f"{r['gbs']:.0f} GB/s of ray writes", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_camera.py needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"gpu_before": gpu_info(), "rounds": args.rounds, "calls": args.calls}
    res["kernel"] = kernel_times(dev, args.rounds, args.iters)

    from fixture import make_state_dict
    from unidepth_b200 import UniDepthV2
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "config_v2_vitl14.json")))
    m = UniDepthV2(copy.deepcopy(cfg))
    m.load_state_dict(make_state_dict(cfg, 0), strict=True)
    m = m.to(dev).eval()
    m.resolution_level = None
    K = torch.tensor([[[520.0, 0.0, 321.5], [0.0, 515.0, 238.25], [0.0, 0.0, 1.0]]])
    fish = MODELS["fisheye624"]()
    cases = {"none": (None, True), "K_eager": (K, False), "K_graph": (K, True), "fisheye_host": (HostCamera(fish), False),
             "fisheye_dev": (fish, True)}
    res["infer"] = {}
    for B in (1, 8):
        rgb = torch.randint(0, 256, (B, 3, 480, 640), dtype=torch.uint8, generator=torch.Generator().manual_seed(0)).to(dev)

        def call(name):
            camera, graph = cases[name]
            m.use_cuda_graph = graph
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m.infer(rgb, camera=camera)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3

        for name in cases:            # warm-up: graphs captured, workspaces and allocator primed
            for _ in range(3):
                call(name)
        times = {n: [] for n in cases}
        for _ in range(args.rounds):
            for name in cases:
                times[name].extend(call(name) for _ in range(args.calls))
        row = {}
        for name, ts in times.items():
            row[name] = {"ms": statistics.median(ts), "min_ms": min(ts), "max_ms": max(ts)}
            print(f"B={B} {name:13s}: {row[name]['ms']:.2f} ms per call ({row[name]['min_ms']:.2f}-{row[name]['max_ms']:.2f}), "
                  f"{B / row[name]['ms'] * 1e3:.1f} images/s", flush=True)
        res["infer"][f"B{B}"] = row
    m.use_cuda_graph = True
    res["gpu_after"] = gpu_info()
    print(f"GPU before: {res['gpu_before']}\nGPU after:  {res['gpu_after']}", flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
