"""The reference's validation path (SURVEY.md section 8f rank 3): matching the network outputs to the ground-truth
frame, and the depth and 3D evaluation metrics.

`match_gt`, `match_intrinsics` and `depth_metrics` are plain torch ops on small tensors (the network itself runs in
libudb.so, UniDepthV2.forward_test).  `eval_depth`, `eval_3d` and `chamfer_distance` run their per-pixel and per-point
work in libudb.so (udb_depth_metrics, udb_nearest_neighbor, udb_point_metrics); torch only resizes, compacts and turns
the per-image sums and counts into the metrics.

Reference: unidepth/utils/misc.py:596-642 (`match_gt`), :645-690 (`match_intrinsics`),
unidepth/utils/evaluation_depth.py (metrics), unidepth/utils/chamfer_distance.py:59-158 (`ChamferDistance`)."""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import torch
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
