"""Seeded inputs of the evaluation-accumulation golden (tests/golden/validate_metrics.npz, made by
oracle/make_golden_validate.py): a sequence of batches as a test loader hands them to the reference's
BaseDataset.accumulate_metrics after the forward, i.e. `inputs` (ground-truth depth, masks, camera) and `preds`.

`batches(C)` builds the cameras with the classes of module C, so the same batches feed the reference's classes
(unidepth/utils/camera.py) and ours (unidepth_b200/camera.py).  The batches cover: different B and sizes; an image whose
mask is empty; pinhole, EUCM, Fisheye624 and Spherical BatchCameras and one mixed-model BatchCamera; a points_mask; a
keyframe index; ground truth above MAX_DEPTH (dropped by the depth metrics); pred keys that are and are not selected.
Every image holds at most a few thousand points, so the reference's CPU nearest-neighbour search stays fast.
TEST INFRASTRUCTURE ONLY.
"""
import torch

MIN_DEPTH, MAX_DEPTH = 0.01, 8.0

# (B, H, W, camera kind, keyframe_idx, empty image or None, points_mask?, extra pred keys)
PLAN = [
    (2, 36, 48, "pinhole", None, 1, False, ()),
    (3, 30, 44, "eucm", None, None, True, ("depth-aux",)),
    (2, 32, 40, "fisheye", None, None, False, ()),
    (3, 28, 36, "spherical", 1, None, False, ()),
    (3, 30, 40, "mixed", None, 2, True, ()),
]


def _cameras(C, kind, B, H, W, g):
    def pinhole():
        f = 0.9 * W + 4 * torch.rand(1, generator=g).item()
        return C.Pinhole(params=torch.tensor([[f, f * 1.02, W / 2 + 0.25, H / 2 - 0.5]]))

    def eucm():
        return C.EUCM(params=torch.tensor([[0.6 * W, 0.61 * W, W / 2, H / 2, 0.6, 1.1]]))

    def fisheye():
        return C.Fisheye624(params=torch.tensor([[0.55 * W, 0.56 * W, W / 2, H / 2, 0.03, -0.004, 0.0, 0.0, 0.0, 0.0,
                                                  0.0, 0.0, 0.0, 0.0, 0.0, 0.0]]))

    def spherical():
        return C.Spherical(params=torch.tensor([[1.0, 1.0, W / 2, H / 2, float(W), float(H), 1.4, 0.6]]))

    make = {"pinhole": pinhole, "eucm": eucm, "fisheye": fisheye, "spherical": spherical}
    if kind == "mixed":
        members = [pinhole(), eucm(), spherical()][:B]
    else:
        members = [make[kind]() for _ in range(B)]
    return torch.cat([C.BatchCamera.from_camera(c) for c in members])


def batches(C):
    """[(inputs, preds, keyframe_idx)] with f32 CPU tensors; depth is z (the range for Spherical members)."""
    g = torch.Generator().manual_seed(2024)
    out = []
    for B, H, W, kind, kf, empty, pmask, extra in PLAN:
        depth = torch.rand(B, 1, H, W, generator=g) * 9.5 + 0.5           # about 16 % above MAX_DEPTH
        mask = torch.rand(B, 1, H, W, generator=g) < 0.7
        if empty is not None:
            mask[empty] = False
        inputs = {"depth": depth, "depth_mask": mask.to(torch.uint8), "camera": _cameras(C, kind, B, H, W, g)}
        if pmask:
            inputs["points_mask"] = mask & (torch.rand(B, 1, H, W, generator=g) < 0.8)
        pred_depth = depth * (1 + 0.2 * (torch.rand(B, 1, H, W, generator=g) - 0.5)) + 0.05
        rays = torch.randn(B, 3, H, W, generator=g) * 0.2
        rays[:, 2] = 1.0
        preds = {"depth": pred_depth, "points": rays * pred_depth, "confidence": torch.rand(B, 1, H, W, generator=g),
                 "intrinsics": torch.eye(3).repeat(B, 1, 1)}
        for key in extra:
            preds[key] = _half_res(pred_depth, g)
        out.append((inputs, preds, kf))
    return out


def _half_res(depth, g):
    """A half-resolution depth prediction (eval_depth resizes it to the ground truth)."""
    coarse = torch.nn.functional.interpolate(depth, scale_factor=0.5, mode="area")
    return coarse * (1 + 0.3 * (torch.rand(coarse.shape, generator=g) - 0.5))
