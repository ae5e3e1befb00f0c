"""The reference's validation path (SURVEY.md section 8f rank 3): matching the network outputs to the ground-truth
frame, the depth and 3D evaluation metrics, the ground-truth point map, their accumulation over a test set and the
evaluation loop.

`match_gt`, `match_intrinsics` and `depth_metrics` are plain torch ops on small tensors (the network itself runs in
libudb.so, UniDepthV2.forward_test).  `eval_depth`, `eval_3d` and `chamfer_distance` run their per-pixel and per-point
work in libudb.so (udb_depth_metrics, udb_nearest_neighbor, udb_point_metrics); torch only resizes, compacts and turns
the per-image sums and counts into the metrics.

Reference: unidepth/utils/misc.py:596-642 (`match_gt`), :645-690 (`match_intrinsics`),
unidepth/utils/evaluation_depth.py (metrics), unidepth/utils/chamfer_distance.py:59-158 (`ChamferDistance`),
unidepth/datasets/base_dataset.py:155-275 (`accumulate_metrics`, `get_evaluation`), unidepth/utils/validation.py:64-91
(`validate`), unidepth/utils/distributed.py:153-176 (`sync_tensor_across_gpus`)."""
from __future__ import annotations

import contextlib
from math import log
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist
import torch.nn.functional as F


def _pad4(padding, i):
    return tuple(int(v) for v in padding[i]) if padding is not None else (0, 0, 0, 0)


def match_gt(pred: torch.Tensor, target: torch.Tensor, padding1: Optional[Sequence] = None,
             padding2: Optional[Sequence] = None, mode: str = "bilinear") -> torch.Tensor:
    """Per image: strip `padding1` (l, r, t, b) from `pred`, resize to `target`'s un-padded size, re-pad
    with `padding2`; interpolation happens in the target's dtype, the result returns to pred's dtype."""
    out = []
    for i in range(len(pred)):
        l1, r1, t1, b1 = _pad4(padding1, i)
        l2, r2, t2, b2 = _pad4(padding2, i)
        item = pred[i]
        core = item[:, t1:item.shape[1] - b1, l1:item.shape[2] - r1]
        size = (target[i].shape[1] - t2 - b2, target[i].shape[2] - l2 - r2)
        resized = F.interpolate(core.unsqueeze(0).to(target[i].dtype), size=size, mode=mode)
        out.append(F.pad(resized, (l2, r2, t2, b2)))
    return torch.cat(out).to(pred[0].dtype)


def match_intrinsics(K: torch.Tensor, image: torch.Tensor, target: torch.Tensor, padding1: Optional[Sequence] = None,
                     padding2: Optional[Sequence] = None) -> torch.Tensor:
    """Pinhole K of the (padded) network input -> K of the target frame: un-pad, scale each axis by the
    ratio of the un-padded sizes, re-pad."""
    out = K.clone()
    h1, w1 = image.shape[2], image.shape[3]
    h2, w2 = target.shape[2], target.shape[3]
    for i in range(K.shape[0]):
        l1, r1, t1, b1 = _pad4(padding1, i)
        l2, r2, t2, b2 = _pad4(padding2, i)
        sx = (w2 - l2 - r2) / (w1 - l1 - r1)
        sy = (h2 - t2 - b2) / (h1 - t1 - b1)
        out[i, 0, 0] *= sx
        out[i, 1, 1] *= sy
        out[i, 0, 2] = (K[i, 0, 2] - l1) * sx + l2
        out[i, 1, 2] = (K[i, 1, 2] - t1) * sy + t2
    return out


def depth_metrics(gt: torch.Tensor, pred: torch.Tensor, mask: Optional[torch.Tensor] = None) -> Dict[str, float]:
    """Scalar metrics of one image on the valid pixels (the subset of evaluation_depth.py's DICT_METRICS
    that needs no scale-alignment solver): d1/d2/d3, rmse, rmselog, arel, sqrel, log10, silog."""
    if mask is None:
        mask = gt > 0
    g, p = gt[mask].double(), pred[mask].double()
    ratio = torch.maximum(g / p, p / g)
    lg = torch.log(p) - torch.log(g)
    return {
        "d1": (ratio < 1.25).double().mean().item(),
        "d2": (ratio < 1.25 ** 2).double().mean().item(),
        "d3": (ratio < 1.25 ** 3).double().mean().item(),
        "rmse": torch.sqrt(((g - p) ** 2).mean()).item(),
        "rmselog": torch.sqrt((lg ** 2).mean()).item(),
        "arel": ((g - p).abs() / g).mean().item(),
        "sqrel": (((g - p) ** 2) / g).mean().item(),
        "log10": (torch.log10(p) - torch.log10(g)).abs().mean().item(),
        "silog": (100 * torch.std(lg)).item(),
    }


# ---------------------------------------------------------------------------------------------------- GPU metrics
# fp32 thresholds of delta (1.25 ** 1, 2, 3) and tau (1 + 0.03): torch compares the fp32 ratio with the scalar in fp32
_DELTA_TAU = (1.25 ** 1.0, 1.25 ** 2.0, 1.25 ** 3.0, 1.0 + 0.03)


def _require(name: str, t, dtypes) -> None:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor, got {type(t).__name__}")
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor (there is no CPU path), got one on {t.device}")
    if t.dtype not in dtypes:
        raise TypeError(f"{name} must have dtype {' or '.join(str(d) for d in dtypes)}, got {t.dtype}")


def _lower_median(vals: torch.Tensor, valid: torch.Tensor, n: torch.Tensor) -> torch.Tensor:
    """Per row, torch.median of vals[valid] (the lower median: element (n - 1) // 2 of the sorted values), NaN for an
    empty row; one batched sort instead of a compaction per image."""
    s = torch.where(valid, vals, torch.full_like(vals, float("inf"))).sort(dim=1).values
    m = s.gather(1, ((n - 1).clamp(min=0) // 2)[:, None])[:, 0]
    return torch.where(n > 0, m, torch.full_like(m, float("nan")))


def _counts_below(hist: torch.Tensor, perm: torch.Tensor) -> torch.Tensor:
    """Histogram over ascending thresholds (bin k: first threshold above the value is k) -> count of values below
    each threshold, in the caller's threshold order (perm: the sort permutation)."""
    cs = hist.cumsum(dim=-1)
    out = torch.empty_like(cs)
    out[:, perm] = cs
    return out


def eval_depth(gts: torch.Tensor, preds: torch.Tensor, masks: torch.Tensor,
               max_depth: Optional[float] = None) -> Dict[str, torch.Tensor]:
    """The reference's eval_depth (evaluation_depth.py:132-147): 18 per-image metrics as f32 tensors [B], in the
    reference's key order.  gts [B, 1, H, W] f32, preds [B, 1, h, w] f32 (resized to H x W with F.interpolate(bilinear)
    first, as the reference does), masks [B, 1, H, W] bool or uint8; all on the GPU.  With max_depth, pixels with
    gt > max_depth are dropped too.

    One udb_depth_metrics call computes every per-pixel term.  The si scale uses median(gt) and median(pred) of the
    valid pixels and medianlog uses median(log pred - log gt): these are torch.median's lower median, taken with one
    batched sort.  The ssi (scale, shift) is solved in f64 (the reference solves in f32), so the ssi metrics can differ
    from the reference's by a few pixels' worth.  An image whose mask is empty gets NaN for every key, as the reference
    gives on CPU."""
    _require("gts", gts, (torch.float32,))
    _require("preds", preds, (torch.float32,))
    _require("masks", masks, (torch.bool, torch.uint8))
    if gts.dim() != 4 or gts.shape[1] != 1 or preds.dim() != 4 or preds.shape[:2] != gts.shape[:2] \
            or masks.shape != gts.shape:
        raise ValueError(f"eval_depth: expected gts, masks [B, 1, H, W] and preds [B, 1, h, w], got "
                         f"{tuple(gts.shape)}, {tuple(masks.shape)}, {tuple(preds.shape)}")
    from . import _cabi as cabi
    from . import ops
    B = gts.shape[0]
    preds = F.interpolate(preds, gts.shape[-2:], mode="bilinear")
    g = gts.reshape(B, -1).contiguous()
    p = preds.reshape(B, -1).contiguous()
    m = masks.reshape(B, -1).contiguous()
    valid = m.bool() if max_depth is None else m.bool() & (g <= max_depth)
    n = valid.sum(dim=1)
    medians = torch.stack([_lower_median(g, valid, n), _lower_median(p, valid, n)], dim=1).contiguous()
    medlog = _lower_median(torch.log(p) - torch.log(g), valid, n)
    exponents = torch.linspace(0.01, 5.0, steps=cabi.DM_AUC_BINS, device=g.device)
    auc_thr, perm = torch.sort(1.25 ** exponents)
    out, _ = ops.depth_metrics(g, p, m.view(torch.uint8) if m.dtype == torch.bool else m, max_depth, _DELTA_TAU,
                               auc_thr.contiguous(), medians)
    nd, nf = out[:, cabi.DM_N], out[:, cabi.DM_N].float()
    frac = lambda k: out[:, k].float() / nf                    # the reference's f32 mean of 0/1 values
    mean = lambda k: (out[:, k] / nd).float()
    var = (out[:, cabi.DM_LG2] - out[:, cabi.DM_LG] ** 2 / nd) / (nd - 1)
    deltas = _counts_below(out[:, cabi.DM_AUC:cabi.DM_AUC + cabi.DM_AUC_BINS], perm).float() / nf[:, None]
    return {
        "d1_ssi": frac(cabi.DM_D1_SSI), "d1_si": frac(cabi.DM_D1_SI), "d1": frac(cabi.DM_D1),
        "d2": frac(cabi.DM_D2), "d3": frac(cabi.DM_D3),
        "rmse": torch.sqrt(out[:, cabi.DM_SQ] / nd).float(),
        "rmselog": torch.sqrt(out[:, cabi.DM_SQLOG] / nd).float(),
        "arel_ssi": mean(cabi.DM_AREL_SSI), "arel_si": mean(cabi.DM_AREL_SI), "arel": mean(cabi.DM_AREL),
        "sqrel": mean(cabi.DM_SQREL), "log10": mean(cabi.DM_LOG10),
        "silog": 100 * torch.sqrt(var).float(),
        "medianlog": 100 * medlog.abs(),
        "d_auc": torch.trapz(deltas, exponents, dim=-1) / 5.0,
        "tau_ssi": frac(cabi.DM_TAU_SSI), "tau_si": frac(cabi.DM_TAU_SI), "tau": frac(cabi.DM_TAU),
    }


def _check_lengths(name: str, lengths, N: int, P: int) -> None:
    _require(name, lengths, (torch.int64,))
    if lengths.shape != (N,):
        raise ValueError(f"{name} must have shape ({N},), got {tuple(lengths.shape)}")
    if bool(((lengths < 0) | (lengths > P)).any()):
        raise ValueError(f"{name} must lie in [0, {P}], got {lengths.tolist()}")


def chamfer_distance(x: torch.Tensor, y: torch.Tensor, x_lengths: Optional[torch.Tensor] = None,
                     y_lengths: Optional[torch.Tensor] = None
                     ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """ChamferDistance()(x, y, x_lengths, y_lengths) with its default arguments (chamfer_distance.py:59-158): returns
    (cham_x [N, P1], cham_y [N, P2], idx_x, idx_y), the squared distance of every point to its nearest neighbour in
    the other cloud and that neighbour's index (ties to the lowest index), 0 past a cloud's length.  x [N, P1, 3],
    y [N, P2, 3] f32 CUDA; lengths int64 [N] in [0, P] or None.  Both directions come from one udb_nearest_neighbor
    pass.  The reference's normals, weights and reduction options are not offered."""
    _require("x", x, (torch.float32,))
    _require("y", y, (torch.float32,))
    if x.dim() != 3 or y.dim() != 3 or x.shape[0] != y.shape[0] or x.shape[2] != 3 or y.shape[2] != 3:
        raise ValueError(f"chamfer_distance: expected x [N, P1, 3] and y [N, P2, 3], got {tuple(x.shape)}, "
                         f"{tuple(y.shape)}")
    N, P1, P2 = x.shape[0], x.shape[1], y.shape[1]
    if N == 0 or P1 == 0 or P2 == 0:
        raise ValueError(f"chamfer_distance: empty batch or cloud dimension, shapes {tuple(x.shape)}, {tuple(y.shape)}")
    for name, l, P in (("x_lengths", x_lengths, P1), ("y_lengths", y_lengths, P2)):
        if l is not None:
            _check_lengths(name, l, N, P)
    from . import ops
    dist_x, idx_x, dist_y, idx_y = ops.nearest_neighbor(x.contiguous(), y.contiguous(), x_lengths, y_lengths)
    return dist_x, dist_y, idx_x, idx_y


def eval_3d(gts: torch.Tensor, preds: torch.Tensor, masks: torch.Tensor,
            thresholds=None) -> Dict[str, torch.Tensor]:
    """The reference's eval_3d (evaluation_depth.py:150-170): {"MSE_3d", "chamfer", "F1"} as f32 tensors with one entry
    per image whose mask is not empty (images with an empty mask are skipped, so the tensors can be shorter than B,
    and with no valid image at all the dict is empty).  gts, preds [B, 3, H, W] f32 point maps, masks [B, 1, H, W]
    bool or uint8, thresholds: 1-D tensor or sequence of F1 thresholds; all on the GPU.

    As in the reference: the whole batch is first downscaled with nearest-exact so that at most about 240 x 320 valid
    points remain; MSE_3d is the mean of |gt - pred|_2 over the valid points; chamfer the mean of
    (sqrt(dist_x) + sqrt(dist_y)) / 2; and F1 compares the SQUARED nearest-neighbour distances with `thresholds`
    (a quirk of the reference, kept), then takes trapz(f1) / len(thresholds).  Every image goes through one batched
    udb_nearest_neighbor launch (both directions) and one udb_point_metrics launch."""
    if thresholds is None:
        raise ValueError("eval_3d needs F1 thresholds (the reference fails on thresholds=None)")
    _require("gts", gts, (torch.float32,))
    _require("preds", preds, (torch.float32,))
    _require("masks", masks, (torch.bool, torch.uint8))
    if gts.dim() != 4 or gts.shape[1] != 3 or preds.shape != gts.shape or masks.dim() != 4 or masks.shape[1] != 1 \
            or masks.shape[0] != gts.shape[0] or masks.shape[2:] != gts.shape[2:]:
        raise ValueError(f"eval_3d: expected gts, preds [B, 3, H, W] and masks [B, 1, H, W], got {tuple(gts.shape)}, "
                         f"{tuple(preds.shape)}, {tuple(masks.shape)}")
    from . import _cabi as cabi
    from . import ops
    thr = torch.as_tensor(thresholds, device=gts.device)
    if thr.is_floating_point():
        thr = thr.float()
    if thr.dim() != 1 or not 1 <= thr.numel() <= cabi.PM_MAX_THRESHOLDS or thr.dtype != torch.float32:
        raise ValueError(f"eval_3d: thresholds must be 1-D floats, 1 to {cabi.PM_MAX_THRESHOLDS} of them, "
                         f"got {tuple(thr.shape)} {thr.dtype}")
    ratio = min(1.0, (240 * 320 / masks.sum()) ** 0.5)       # evaluation_depth.py:154-157, same fp32 arithmetic
    h, w = int(gts.shape[-2] * ratio), int(gts.shape[-1] * ratio)
    gts = F.interpolate(gts, size=(h, w), mode="nearest-exact")
    preds = F.interpolate(preds, size=(h, w), mode="nearest-exact")
    valid = F.interpolate(masks.float(), size=(h, w), mode="nearest-exact").bool().reshape(gts.shape[0], -1)
    n = valid.sum(dim=1)
    n_host = n.tolist()
    keep = [i for i, v in enumerate(n_host) if v > 0]
    if not keep:
        return {}
    P = max(n_host)
    order = torch.argsort((~valid).to(torch.uint8), dim=1, stable=True)[:, :P]   # valid pixels first, in raster order
    idx = order[:, :, None].expand(-1, -1, 3)
    x = gts.reshape(gts.shape[0], 3, -1).transpose(1, 2).gather(1, idx).contiguous()
    y = preds.reshape(preds.shape[0], 3, -1).transpose(1, 2).gather(1, idx).contiguous()
    dist_x, _, dist_y, _ = ops.nearest_neighbor(x, y, n, n)
    thr_sorted, perm = torch.sort(thr)
    out = ops.point_metrics(x, y, n, dist_x, dist_y, thr_sorted.contiguous())
    T = thr.numel()
    nd, nf = n.double(), n.float()[:, None]
    precision = _counts_below(out[:, 2:2 + T], perm).float() / nf
    recall = _counts_below(out[:, 2 + T:], perm).float() / nf
    f1 = 2 * precision * recall / (precision + recall)
    f1 = torch.where(torch.isnan(f1), torch.zeros_like(f1), f1)
    res = {"MSE_3d": (out[:, 0] / nd).float(), "chamfer": (out[:, 1] / nd).float(),
           "F1": torch.trapz(f1, dim=-1) / T}
    if len(keep) < len(n_host):
        sel = torch.tensor(keep, device=gts.device)
        res = {k: v[sel] for k, v in res.items()}
    return res


# ------------------------------------------------------------------------------------------ ground-truth point map
def reconstruct(camera, depth: torch.Tensor) -> torch.Tensor:
    """The reference's `camera.reconstruct(depth)`: the ground-truth point map [B, 3, H, W] of a z-depth (range, for
    Spherical) map [B, 1, H, W], with each camera class's own rule.  A camera that `camera.pack_camera` accepts, with one
    row (broadcast to the batch) or one row per image, and an f32 CUDA depth map take the udb_camera_reconstruct kernel;
    anything else (mixed-model BatchCameras, the reference's own classes, duck-typed objects, the 15-parameter layout,
    CPU tensors) runs the object's own `reconstruct`."""
    from .camera import pack_camera
    packed = None
    if isinstance(depth, torch.Tensor) and depth.is_cuda and depth.dtype == torch.float32 and depth.dim() == 4 \
            and depth.shape[1] == 1:
        packed = pack_camera(camera)
    if packed is not None and packed[1].shape[0] in (1, depth.shape[0]):
        from . import ops
        model, rows = packed
        rows = rows.to(depth.device).expand(depth.shape[0], -1).contiguous()
        return ops.camera_reconstruct(model, rows, depth.contiguous())
    return camera.reconstruct(depth)


# ------------------------------------------------------------------------------------- accumulation over a test set
def gather_across_ranks(t: Optional[torch.Tensor], group=None) -> Optional[torch.Tensor]:
    """Concatenate every rank's 1-D (or leading-dimension) tensor in rank order, whatever each rank's length: gather
    the lengths, pad to the longest, all_gather, trim, concatenate (the reference's sync_tensor_across_gpus).  The
    tensor itself when torch.distributed is not initialised."""
    if t is None or not (dist.is_available() and dist.is_initialized()):
        return t
    t = torch.atleast_1d(t)
    world = dist.get_world_size(group)
    n = torch.tensor([t.shape[0]], device=t.device, dtype=torch.int64)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n, group=group)
    sizes = [int(v.item()) for v in sizes]
    longest = max(sizes)
    if longest > t.shape[0]:
        t = torch.cat([t, t.new_zeros((longest - t.shape[0],) + tuple(t.shape[1:]))])
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t.contiguous(), group=group)
    return torch.cat([p[:k] for p, k in zip(parts, sizes)])


def _index(x, index):
    """The reference's recursive_index: slice the tensors of a (nested) dict, leave everything else as it is."""
    if isinstance(x, dict):
        return {k: _index(v, index) for k, v in x.items()}
    if isinstance(x, torch.Tensor):
        return x[index]
    return x


def _no_autocast(fn):
    """The reference accumulates in fp32 whatever autocast context the caller opened."""
    return torch.autocast(device_type="cuda", enabled=False)(fn)


class DatasetMetrics:
    """Per-image evaluation metrics accumulated over a test set and reduced to its means, as the reference's
    BaseDataset does (accumulate_metrics, get_evaluation and their helpers, same names and attributes).  It can be used
    on its own or inherited as a mixin by a dataset class (which then calls DatasetMetrics.__init__ or sets
    `metrics_store`, `metrics_count`, `min_depth` and `max_depth` itself); a `keyframe_idx` attribute, if the object has
    one, selects the depth frame as in the reference.

    Kept from the reference: a metric is available when it is a substring of some key of both `inputs` and `preds`;
    `keyframe_idx` slices tensors only, and prepare_depth_eval slices again with the `keyframe_idx` attribute; a pred
    key containing "depth" is evaluated with eval_depth and one containing "points" with eval_3d (100 F1 thresholds
    log-spaced from min_depth to max_depth / 20) under the log name left by removing that word, so a pred dict with
    "depth" and "points" fills one store "" with 21 metrics; `metrics_count` is gathered but unused; a metric image whose
    mask is empty gives NaN depth metrics, which propagates to the mean.  Differences: the caller's `inputs` is not
    modified (the point map is added to a shallow copy), and a pred selected for depth that is not a float
    [B, 1, h, w] tensor raises ValueError naming it before any metric runs (the reference fails inside F.interpolate)."""

    eval_depth = staticmethod(eval_depth)
    eval_3d = staticmethod(eval_3d)

    def __init__(self, min_depth: float = 0.01, max_depth: float = 1000.0):
        self.min_depth = min_depth
        self.max_depth = max_depth
        self.metrics_store: Dict[str, Dict[str, torch.Tensor]] = {}
        self.metrics_count: Dict[str, torch.Tensor] = {}

    def add_points(self, inputs):
        inputs["points"] = reconstruct(inputs.get("camera_original", inputs["camera"]), inputs["depth"])
        return inputs

    def prepare_depth_eval(self, inputs, preds):
        keyframe_idx = getattr(self, "keyframe_idx", None)
        slice_idx = slice(keyframe_idx, keyframe_idx + 1 if keyframe_idx is not None else None)
        new_gts = inputs["depth"][slice_idx]
        new_masks = inputs["depth_mask"][slice_idx].bool()
        new_preds = {key: val[slice_idx] for key, val in preds.items() if "depth" in key}
        return new_gts, new_preds, new_masks

    def prepare_points_eval(self, inputs, preds):
        new_gts = inputs["points"]
        new_masks = inputs["points_mask"].bool() if "points_mask" in inputs else inputs["depth_mask"].bool()
        new_preds = {key: val for key, val in preds.items() if "points" in key}
        return new_gts, new_preds, new_masks

    @_no_autocast
    def accumulate_metrics(self, inputs, preds, keyframe_idx=None, metrics=("depth", "points", "flow_fwd", "pairwise")):
        if "depth" in inputs and "points" not in inputs:
            inputs = self.add_points(dict(inputs))
        available = [m for m in metrics if any(m in k for k in inputs) and any(m in k for k in preds)]
        if keyframe_idx is not None:
            inputs = _index(inputs, slice(keyframe_idx, keyframe_idx + 1))
            preds = _index(preds, slice(keyframe_idx, keyframe_idx + 1))
        if "depth" in available:
            gts, depth_preds, masks = self.prepare_depth_eval(inputs, preds)
            for key, val in depth_preds.items():
                if not isinstance(val, torch.Tensor) or not val.is_floating_point() or val.dim() != 4 \
                        or val.shape[:2] != (gts.shape[0], 1):
                    shape = tuple(val.shape) if isinstance(val, torch.Tensor) else type(val).__name__
                    raise ValueError(f"accumulate_metrics: pred {key!r} is selected for the depth metrics (its key "
                                     f"contains 'depth') but is not a float [B, 1, h, w] depth map with B = "
                                     f"{gts.shape[0]}: {shape}")
            self.accumulate_metrics_depth(gts, depth_preds, masks)
        if "points" in available:
            self.accumulate_metrics_3d(*self.prepare_points_eval(inputs, preds))

    def _append(self, log_name, gts, masks, values):
        store = self.metrics_store.setdefault(log_name, {})
        count = self.metrics_count.get(log_name, torch.tensor([], device=gts.device))
        self.metrics_count[log_name] = torch.cat([count, masks.view(gts.shape[0], -1).sum(dim=-1)])
        for k, v in values.items():
            store[k] = torch.cat([store.get(k, torch.tensor([], device=gts.device)), v])

    @_no_autocast
    def accumulate_metrics_depth(self, gts, preds, masks):
        for eval_type, pred in preds.items():
            log_name = eval_type.replace("depth", "").strip("-").strip("_")
            self._append(log_name, gts, masks, self.eval_depth(gts, pred, masks, max_depth=self.max_depth))

    @_no_autocast
    def accumulate_metrics_3d(self, gts, preds, masks):
        thresholds = torch.linspace(log(self.min_depth), log(self.max_depth / 20), steps=100, device=gts.device).exp()
        for eval_type, pred in preds.items():
            log_name = eval_type.replace("points", "").strip("-").strip("_")
            self._append(log_name, gts, masks, self.eval_3d(gts, pred, masks, thresholds=thresholds))

    def get_evaluation(self, metrics=None) -> Dict[str, float]:
        """{f"{eval_type}_{name}".strip("_"): mean over every rank's images, rounded to 5 decimals}; clears the stores.
        A store that was emptied by an earlier call and has had nothing added raises AssertionError, as in the
        reference."""
        values = {}
        for eval_type in metrics if metrics is not None else list(self.metrics_store.keys()):
            assert self.metrics_store[eval_type], f"no metrics accumulated for {eval_type!r}"
            gather_across_ranks(self.metrics_count[eval_type])
            for name, val in self.metrics_store[eval_type].items():
                mean = gather_across_ranks(val).mean()
                values[f"{eval_type}_{name}".strip("_")] = float(np.round(mean.cpu().item(), 5))
            self.metrics_store[eval_type] = {}
        self.metrics_count = {}
        return values


# --------------------------------------------------------------------------------------------------- evaluation loop
def _rank0() -> bool:
    return not (dist.is_available() and dist.is_initialized()) or dist.get_rank() == 0


def _barrier() -> None:
    if dist.is_available() and dist.is_initialized():
        dist.barrier()


def _dataset_metrics(dataset) -> DatasetMetrics:
    if isinstance(dataset, DatasetMetrics):
        return dataset
    return DatasetMetrics(min_depth=getattr(dataset, "min_depth", 0.01), max_depth=getattr(dataset, "max_depth", 1000.0))


def validate(model, test_loaders, step=None, context=None) -> Dict[str, Dict[str, float]]:
    """The reference's evaluation loop over {name: DataLoader}: for each batch, move `batch["data"]` to model.device and
    drop the loader's temporal axis (squeeze(1); an object without `squeeze`, such as a camera, is taken as already
    squeezed), unwrap the metas ({k: v[0]} of their list values), run `model(data, metas)` under torch.no_grad() and
    `context`, and accumulate the metrics with the first meta's keyframe_idx.  After each loader, every rank runs
    get_evaluation (which gathers across ranks), and rank 0 prints `Metrics/{name}/{metric} {value}` lines.  Returns
    {name: {metric: value}}.

    Each loader's accumulator is its dataset if that is a DatasetMetrics, else a DatasetMetrics with the dataset's
    min_depth / max_depth (0.01 / 1000 without them).  Differences from the reference: nothing is logged to wandb
    (`step` is accepted and unused); `original_image` is not run, since nothing the accumulation reads depends on it; a
    dataset's own accumulate_metrics override is only called when the dataset is a DatasetMetrics.  The caller's batches
    are not modified."""
    metrics_all = {}
    for name_ds, loader in test_loaders.items():
        acc = _dataset_metrics(loader.dataset)
        for batch in loader:
            with context if context is not None else contextlib.nullcontext(), torch.no_grad():
                data = {k: (v.to(model.device) if hasattr(v, "to") else v) for k, v in batch["data"].items()}
                data = {k: (v.squeeze(1) if hasattr(v, "squeeze") else v) for k, v in data.items()}
                metas = [{k: v[0] for k, v in meta.items() if isinstance(v, list)} for meta in batch["img_metas"]]
                preds = model(data, metas)
            acc.accumulate_metrics(inputs=data, preds=preds, keyframe_idx=metas[0].get("keyframe_idx") if metas else None)
        _barrier()
        metrics_all[name_ds] = acc.get_evaluation()
    _barrier()
    if _rank0():
        for name_ds, values in metrics_all.items():
            for name, v in values.items():
                print(f"Metrics/{name_ds}/{name} {round(v, 4)}")
    return metrics_all
