"""Evaluation over a test set on the GPU: the ground-truth point map kernel (udb_camera_reconstruct via
validation.reconstruct) against the camera classes and the reference, DatasetMetrics on the device against the
unmodified reference's accumulation (tests/golden/validate_metrics.npz), and `validate` end to end on UniDepthV2.

Bounds of the kernel against the class's own reconstruct (fp32 torch on the same GPU), per point relative to the point's
magnitude max(|p|, 1e-3), with u = 2^-24, as test_camera_kernel_gpu.py bounds the rays:
  * EUCM and Spherical evaluate the class's expressions op for op: 16 u.
  * Pinhole (torch.inverse against the adjugate) and the Newton models: 4 E32 + 16 u, E32 the class's own fp32 error
    against a float64 evaluation of the same function.
NaN only where the class gives NaN (MEI with xi > 1 far off axis).  The measured maxima are printed as `RECON` lines."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

from unidepth_b200 import _cabi
from unidepth_b200 import camera as C
from unidepth_b200 import validation as V

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
U = 2.0 ** -24


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _cameras():
    from test_camera_kernel_gpu import CAMERAS, CLOSED
    return CAMERAS, CLOSED


def _depth(B, H, W, seed, dev):
    g = torch.Generator().manual_seed(seed)
    d = torch.rand(B, 1, H, W, generator=g) * 9.5 + 0.5
    d.view(-1)[::97] = -1.0            # negative and tiny depths exercise each class's clamp
    d.view(-1)[1::89] = 3e-5
    return d.to(dev)


def _class64(cam, depth):
    """The class's reconstruct in float64 (Pinhole inverts K in fp32 whatever its dtype: restated)."""
    cam = copy.deepcopy(cam)
    d = depth.double()
    if isinstance(cam, C.Pinhole):
        B, _, H, W = d.shape
        uv = C.pixel_grid(1, H, W, homogeneous=True, device=d.device).double().reshape(1, 3, -1)
        xyz = torch.linalg.inv(cam.K.double()) @ uv
        xyz = (xyz / xyz[:, 2:].clamp(min=1e-4)).reshape(-1, 3, H, W)
        return xyz * d.clip(min=0.0)
    cam.params, cam.K = cam.params.double(), cam.K.double()
    return cam.reconstruct(d)


@pytest.mark.parametrize("name", sorted(_cameras()[0]))
def test_kernel_matches_class_reconstruct(name):
    dev = _dev()
    cameras, closed = _cameras()
    worst = 0.0
    for B, H, W, per_image in ((1, 14, 14, False), (2, 480, 640, False), (3, 37, 501, True), (2, 300, 17, True)):
        cams = [cameras[name]().to(dev) for _ in range(B if per_image else 1)]
        for i, c in enumerate(cams):           # per-image rows: each image its own focal length
            c.params[0, 0] += 3.0 * i
            if isinstance(c, C.Pinhole):
                c.K[0, 0, 0] += 3.0 * i
        cam = torch.cat([C.BatchCamera.from_camera(c) for c in cams]) if per_image else cams[0]
        depth = _depth(B, H, W, 10 + B + H, dev)
        assert C.pack_camera(cam) is not None
        n0 = _cabi.launch_count()
        got = V.reconstruct(cam, depth)
        assert _cabi.launch_count() == n0 + 1 and got.shape == (B, 3, H, W) and got.is_contiguous()
        ref = cam.reconstruct(depth)
        ref64 = torch.cat([_class64(c, depth[i:i + 1]) for i, c in enumerate(cams)]) if per_image else _class64(cam, depth)
        nan_got, nan_ref = torch.isnan(got), torch.isnan(ref)
        assert not (nan_got & ~nan_ref).any(), name            # NaN only where the class gives NaN
        ok = torch.isfinite(ref64).all(1, keepdim=True) & torch.isfinite(ref).all(1, keepdim=True)
        assert torch.isfinite(got)[ok.expand_as(got)].all()
        assert ok.float().mean().item() > 0.5
        scale = ref64.abs().amax(1, keepdim=True).clamp(min=1e-3)
        err = ((got.double() - ref.double()).abs() / scale)[ok.expand_as(got)].max().item()
        e32 = ((ref.double() - ref64).abs() / scale)[ok.expand_as(got)].max().item()
        ek = ((got.double() - ref64).abs() / scale)[ok.expand_as(got)].max().item()
        bound = 16 * U if name in closed else 4 * e32 + 16 * U
        print(f"RECON {name} B={B} {H}x{W} per-image={per_image}: |kernel-class| {err:.3e} (bound {bound:.3e}), "
              f"|class-f64| {e32:.3e}, |kernel-f64| {ek:.3e}, NaN {int(nan_got.sum())}/{int(nan_ref.sum())}")
        assert err <= bound, (name, B, H, W, err, bound)
        worst = max(worst, err / bound)
    print(f"RECON {name}: largest error/bound {worst:.3f}")


@pytest.mark.parametrize("name", ["pinhole_params", "eucm", "spherical", "opencv_radial", "opencv_full", "fisheye624",
                                  "fisheye624_radial", "mei", "mei_plain"])
def test_kernel_matches_reference_reconstruct(name):
    """tests/golden/cameras.npz `*/reconstruct`: the unmodified reference's reconstruct of a seeded depth, at
    test_camera_cpu.py's bars (2e-6 closed forms, 1.5e-3 iterative models, relative to the point)."""
    dev = _dev()
    z = np.load(os.path.join(ROOT, "tests", "golden", "cameras.npz"))
    cls = {"pinhole_params": "Pinhole", "eucm": "EUCM", "spherical": "Spherical", "opencv_radial": "OPENCV",
           "opencv_full": "OPENCV", "fisheye624": "Fisheye624", "fisheye624_radial": "Fisheye624", "mei": "MEI",
           "mei_plain": "MEI"}[name]
    cam = getattr(C, cls)(params=torch.from_numpy(z[f"{name}/params"]).clone())
    depth = torch.from_numpy(z["depth"][:1]).to(dev)           # the golden reconstructs the first map with the camera
    got = V.reconstruct(cam, depth).cpu().double()
    want = torch.from_numpy(z[f"{name}/reconstruct"]).double()
    e = ((got - want).abs() / want.abs().amax(1, keepdim=True).clamp(min=1e-3)).max().item()
    print(f"RECON {name}: kernel vs reference reconstruct {e:.2e}")
    assert e < (2e-6 if cls in ("Pinhole", "EUCM", "Spherical") else 1.5e-3), e


def test_mixed_batch_takes_the_host_path():
    dev = _dev()
    cameras, _ = _cameras()
    mixed = torch.cat([C.BatchCamera.from_camera(cameras[n]().to(dev)) for n in ("pinhole", "eucm", "mei_strong")])
    assert C.pack_camera(mixed) is None
    depth = _depth(3, 40, 56, 3, dev)
    n0 = _cabi.launch_count()
    got = V.reconstruct(mixed, depth)
    assert _cabi.launch_count() == n0
    assert torch.equal(got, mixed.reconstruct(depth))


# ------------------------------------------------------------------------------------------------ DatasetMetrics
COUNTS = {"d1", "d2", "d3", "tau", "d1_si", "tau_si"}


def test_dataset_metrics_on_the_device_match_the_reference():
    """GPU metrics and kernel point maps against the reference's store, at test_eval_metrics_gpu.py's bars: plain and si
    ratio counts exact, ssi counts and d_auc within 3 pixels, sums within 1e-5 relative plus the fp32-vs-f64 summation
    allowance; the 3D metrics within 5e-4 relative (the Fisheye624 batch: the reference's Newton loop stops at a
    residual of 1e-3, ours converges)."""
    dev = _dev()
    import validate_oracle as VO
    z = np.load(os.path.join(ROOT, "tests", "golden", "validate_metrics.npz"))
    m = V.DatasetMetrics(min_depth=VO.MIN_DEPTH, max_depth=VO.MAX_DEPTH)
    for inputs, preds, kf in VO.batches(C):
        inputs = {k: v.to(dev) for k, v in inputs.items()}
        preds = {k: v.to(dev) for k, v in preds.items()}
        m.accumulate_metrics(inputs=inputs, preds=preds, keyframe_idx=kf)
    for t, store in m.metrics_store.items():
        n = z[f"count/{t}"]
        for name, v in store.items():
            got, want = v.cpu().numpy(), z[f"store/{t}/{name}"]
            assert got.shape == want.shape and np.array_equal(np.isnan(got), np.isnan(want)), (t, name)
            ok = ~np.isnan(want)
            err = np.abs(got - want)[ok]
            if name in COUNTS:
                tol = np.zeros_like(err)
            elif name in ("MSE_3d", "chamfer", "F1"):
                tol = 5e-4 * np.abs(want[ok]) + 1e-6
            else:
                tol = 2e-5 * np.abs(want[ok]) + 1e-6
                if name in ("d1_ssi", "tau_ssi", "d_auc"):
                    tol = tol + 3.0 / np.maximum(n[: len(want)][ok], 1)
            print(f"DSMETRICS {t or '-'}/{name}: max err {err.max() if err.size else 0:.3e}")
            assert np.all(err <= tol), (t, name, got, want)
    ev = m.get_evaluation()
    assert list(ev) == list(z["eval_keys"])


# --------------------------------------------------------------------------------------------------- validate
# the fixtures with a camera: the accumulation builds the ground-truth points from inputs["camera"], as the reference's
V2FWD = ["v2fwd_vits14_pinhole_294x392_360x480", "v2fwd_vits14_eucm_294x392_480x640"]


def _loader_batches(dev):
    """One batch per v2fwd fixture (same seeded ViT-S weights), shaped as a loader hands them: a temporal axis of 1 on
    every tensor and list-wrapped metas; ground-truth depth from a smooth seeded field with about 70 % valid pixels."""
    from test_v2_forward_cpu import golden_case
    out = []
    for i, name in enumerate(V2FWD):
        z, meta, inputs, metas = golden_case(name)
        B, _, H, W = inputs["depth"].shape
        g = torch.Generator().manual_seed(100 + i)
        depth = 2.0 + torch.rand(B, 1, H, W, generator=g) * 4.0
        data = {"image": inputs["image"][:, None], "depth": depth[:, None],
                "depth_mask": (torch.rand(B, 1, 1, H, W, generator=g) < 0.7)}
        if "camera" in inputs:
            data["camera"] = inputs["camera"]
        out.append(({"data": data, "img_metas": [{k: [v] for k, v in mt.items()} for mt in metas]}, z, name))
    return out


class _Loader(list):
    def __init__(self, batches, dataset):
        super().__init__(batches)
        self.dataset = dataset


def test_validate_end_to_end_on_unidepthv2():
    dev = _dev()
    from test_v2_forward_cpu import golden_case
    from test_v2_forward_gpu import MEASURED, _model
    _, meta0, _, _ = golden_case(V2FWD[0])
    m = _model(meta0, dev)
    items = _loader_batches(dev)
    batches = [b for b, _, _ in items]
    res = V.validate(m, {"fixtures": _Loader(batches, object())})["fixtures"]
    # the same forward outputs fed to DatasetMetrics by hand: bit for bit
    acc = V.DatasetMetrics()
    fwd = []
    for b in batches:
        data = {k: (v.to(dev).squeeze(1) if isinstance(v, torch.Tensor) else v) for k, v in b["data"].items()}
        metas = [{k: v[0] for k, v in mt.items()} for mt in b["img_metas"]]
        with torch.no_grad():
            preds = m(data, metas)
        fwd.append((data, preds))
        acc.accumulate_metrics(data, preds)
    want = acc.get_evaluation()
    assert list(res) == list(want) and len(res) == 21
    for k in res:
        assert res[k] == want[k] or (np.isnan(res[k]) and np.isnan(want[k])), (k, res[k], want[k])
    # against the reference's golden forward outputs (subsampled in the goldens): depth metrics of our depth and of the
    # reference's on the same subsampled pixels.  With e the forward's max relative depth error (test_v2_forward_gpu's
    # measured value, x1.5), a pred p(1 + eps), |eps| <= e, moves rmse by <= e rmse(p) <= e (rmse + rms gt), arel and sqrel
    # by <= e (1 + arel) and 2e (sqrel + mean gt) to first order, and the log metrics by <= e (rmselog, log10) and 100 e
    # (silog) in absolute terms; asserted with a factor 2 on each.
    # Each fixture has its own seeded weights: its batch runs through its own model here.
    for (data, _), (_, z, name) in zip(fwd, items):
        meta = golden_case(name)[1]
        with torch.no_grad():
            preds = _model(meta, dev)(data, [{"paddings": p, "depth_paddings": [0, 0, 0, 0]} for p in meta["metas_paddings"]]
                                      if meta["metas_paddings"] else [])
        s = meta["strides"]["depth"]
        gt = data["depth"][:, :, ::s, ::s].contiguous()
        mask = data["depth_mask"][:, :, ::s, ::s].contiguous()
        ours = V.eval_depth(gt, preds["depth"][:, :, ::s, ::s].contiguous(), mask)
        ref = V.eval_depth(gt, torch.from_numpy(z["depth"]).to(dev), mask)
        e = 1.5 * MEASURED[name][1]
        g = gt[mask.bool()].double()
        allow = {"rmse": lambda r: e * (r + g.pow(2).mean().sqrt()), "arel": lambda r: e * (1 + r),
                 "sqrel": lambda r: 2 * e * (r + g.mean()), "rmselog": lambda r: e, "log10": lambda r: e,
                 "silog": lambda r: 100 * e}
        for k, fn in allow.items():
            a, r = ours[k].double(), ref[k].double()
            tol = 2 * fn(r) + 1e-6 + torch.zeros_like(r)
            print(f"VALIDATE {k}: ours {a.tolist()} reference-forward {r.tolist()} tol {tol.tolist()}")
            assert torch.all((a - r).abs() <= tol), k


# ------------------------------------------------------------------------------------------------------ two GPUs
def _rank_main(rank, world, port, q):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    from test_v2_forward_cpu import golden_case
    from test_v2_forward_gpu import _model
    from unidepth_b200 import validation as V2
    _, meta0, _, _ = golden_case(V2FWD[0])
    m = _model(meta0, torch.device("cuda", rank))
    batches = [b for b, _, _ in _loader_batches(None)]
    mine = batches[rank::world]
    res = V2.validate(m, {"fixtures": _Loader(mine, object())})
    q.put((rank, res))
    dist.destroy_process_group()


def test_two_rank_validate_equals_one_rank():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import socket
    import torch.multiprocessing as mp
    dev = _dev()
    from test_v2_forward_cpu import golden_case
    from test_v2_forward_gpu import _model
    _, meta0, _, _ = golden_case(V2FWD[0])
    m = _model(meta0, dev)
    batches = [b for b, _, _ in _loader_batches(dev)]
    order = batches[0::2] + batches[1::2]               # rank 0's batches, then rank 1's: the gather's order
    one = V.validate(m, {"fixtures": _Loader(order, object())})
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank_main, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=600) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for r in range(2):
        for k, v in one["fixtures"].items():
            w = res[r]["fixtures"][k]
            assert v == w or (np.isnan(v) and np.isnan(w)), (r, k, v, w)
