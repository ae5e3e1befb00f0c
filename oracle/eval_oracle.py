"""Pure-torch restatement of the reference's evaluation metrics, for the goldens' inputs and as the GPU tests' oracle.

- knn1: K = 1, L2 nearest neighbour of ops/knn (knn_cpu.cpp:13-69, knn.py:113-196): squared distance formed as
  ((dx*dx) + dy*dy) + dz*dz with dx = p1 - p2, each op rounded on its own (torch eager ops do not fuse), ties to the
  lowest index (the CPU code's strict `<`; torch.argmin returns the first minimum), zeros past lengths1 and where
  lengths2 == 0.  Chunked exact brute force, so it runs at sizes the goldens do not cover, on CPU or GPU.
- eval_depth: evaluation_depth.py:37-109 (delta, tau, ssi, si, d_auc, DICT_METRICS) and :132-147.
- eval_3d: evaluation_depth.py:12-18 (chamfer_dist), :74-90 (f1_score), :112-122 (DICT_METRICS_3D) and :150-170;
  ChamferDistance (chamfer_distance.py:104-158) with default arguments is chamfer() below.

Seeded input generators for the goldens live here too, so inputs are regenerated rather than stored.
TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


# ------------------------------------------------------------------------------------------------ nearest neighbour
def knn1(p1, p2, lengths1=None, lengths2=None, chunk=2048):
    """(dist [N, P1] f32, idx [N, P1] int64) like knn_points_idx(p1, p2, lengths1, lengths2, norm=2, K=1)."""
    N, P1, _ = p1.shape
    P2 = p2.shape[1]
    l1 = [P1] * N if lengths1 is None else [int(v) for v in lengths1]
    l2 = [P2] * N if lengths2 is None else [int(v) for v in lengths2]
    dist = torch.zeros(N, P1, dtype=torch.float32, device=p1.device)
    idx = torch.zeros(N, P1, dtype=torch.int64, device=p1.device)
    for n in range(N):
        if l2[n] == 0:
            continue
        ys = p2[n, :l2[n]]
        for s in range(0, l1[n], chunk):
            xs = p1[n, s:min(s + chunk, l1[n])]
            dx = xs[:, None, 0] - ys[None, :, 0]
            dy = xs[:, None, 1] - ys[None, :, 1]
            dz = xs[:, None, 2] - ys[None, :, 2]
            d = (dx * dx + dy * dy) + dz * dz
            m, i = d.min(dim=1)
            # torch.min(dim) on CUDA does not promise the first index among equal minima: take it explicitly
            i = torch.where(d == m[:, None], torch.arange(d.shape[1], device=d.device)[None], d.shape[1]).min(dim=1).values
            dist[n, s:s + xs.shape[0]] = m
            idx[n, s:s + xs.shape[0]] = i
    return dist, idx


def chamfer(x, y, x_lengths=None, y_lengths=None):
    """ChamferDistance()(x, y, x_lengths, y_lengths) -> (cham_x, cham_y, idx_x, idx_y)."""
    dx, ix = knn1(x, y, x_lengths, y_lengths)
    dy, iy = knn1(y, x, y_lengths, x_lengths)
    return dx, dy, ix, iy


# ------------------------------------------------------------------------------------------------------- eval_depth
def _delta(g, p, thr):
    inlier = torch.maximum(g / p, p / g)
    return (inlier < thr).to(torch.float32).mean()


def _ssi(g, p):
    stab = 1e-9 * torch.eye(2, device=g.device)
    A = torch.stack([p, torch.ones_like(p)], dim=1)
    scale, shift = (torch.inverse(A.T @ A + stab) @ (A.T @ g.unsqueeze(1))).squeeze().chunk(2, dim=0)
    return p * scale + shift


def _si(g, p):
    return p * torch.median(g) / torch.median(p)


def _d_auc(g, p):
    exponents = torch.linspace(0.01, 5.0, steps=100, device=g.device)
    deltas = torch.stack([_delta(g, p, 1.25 ** e) for e in exponents])
    return torch.trapz(deltas, exponents) / 5.0


METRICS = {
    "d1": lambda g, p: _delta(g, p, 1.25 ** 1.0),
    "d2": lambda g, p: _delta(g, p, 1.25 ** 2.0),
    "d3": lambda g, p: _delta(g, p, 1.25 ** 3.0),
    "rmse": lambda g, p: torch.sqrt(((g - p) ** 2).mean()),
    "rmselog": lambda g, p: torch.sqrt(((torch.log(g) - torch.log(p)) ** 2).mean()),
    "arel": lambda g, p: (torch.abs(g - p) / g).mean(),
    "sqrel": lambda g, p: (((g - p) ** 2) / g).mean(),
    "log10": lambda g, p: torch.abs(torch.log10(p) - torch.log10(g)).mean(),
    "silog": lambda g, p: 100 * torch.std(torch.log(p) - torch.log(g)),
    "medianlog": lambda g, p: 100 * (torch.log(p) - torch.log(g)).median().abs(),
    "d_auc": _d_auc,
    "tau": lambda g, p: _delta(g, p, 1.0 + 0.03),
}
KEYS = ["d1_ssi", "d1_si", "d1", "d2", "d3", "rmse", "rmselog", "arel_ssi", "arel_si", "arel", "sqrel", "log10",
        "silog", "medianlog", "d_auc", "tau_ssi", "tau_si", "tau"]


def eval_depth(gts, preds, masks, max_depth=None):
    out = {k: [] for k in KEYS}
    preds = F.interpolate(preds, gts.shape[-2:], mode="bilinear")
    for gt, pred, mask in zip(gts, preds, masks):
        mask = mask.bool()
        if max_depth is not None:
            mask = mask & (gt <= max_depth)
        g, p = gt[mask], pred[mask]
        for name, fn in METRICS.items():
            if name in ("tau", "d1", "arel"):
                out[name + "_ssi"].append(fn(g, _ssi(g, p)))
                out[name + "_si"].append(fn(g, _si(g, p)) if g.numel() else torch.tensor(float("nan"), device=g.device))
            out[name].append(fn(g, p) if g.numel() else torch.tensor(float("nan"), device=g.device))
    return {k: torch.stack(v) for k, v in out.items()}


# ---------------------------------------------------------------------------------------------------------- eval_3d
def eval_3d(gts, preds, masks, thresholds):
    ratio = min(1.0, (240 * 320 / masks.sum()) ** 0.5)
    h, w = int(gts.shape[-2] * ratio), int(gts.shape[-1] * ratio)
    gts = F.interpolate(gts, size=(h, w), mode="nearest-exact")
    preds = F.interpolate(preds, size=(h, w), mode="nearest-exact")
    masks = F.interpolate(masks.float(), size=(h, w), mode="nearest-exact").bool()
    out = {"MSE_3d": [], "chamfer": [], "F1": []}
    for gt, pred, mask in zip(gts, preds, masks):
        if not torch.any(mask):
            continue
        g, p = gt[:, mask.squeeze(0)], pred[:, mask.squeeze(0)]
        out["MSE_3d"].append(torch.norm(g - p, dim=0, p=2).mean())
        d1, d2, _, _ = chamfer(g.T[None].contiguous(), p.T[None].contiguous())
        out["chamfer"].append(((torch.sqrt(d1) + torch.sqrt(d2)) / 2).mean())
        prec = torch.stack([(d1 < t).sum() / d1.numel() for t in thresholds])
        rec = torch.stack([(d2 < t).sum() / d2.numel() for t in thresholds])
        f1 = 2 * prec * rec / (prec + rec)
        f1 = torch.where(torch.isnan(f1), torch.zeros_like(f1), f1)
        out["F1"].append(torch.trapz(f1) / len(thresholds))
    return {k: torch.stack(v) for k, v in out.items() if v}


# ------------------------------------------------------------------------------------------------- seeded inputs
def depth_case(seed=11, B=3, H=60, W=80):
    """gts [B,1,H,W] in (0.5, 10.5), preds [B,1,H/2,W/2] a noisy copy at half resolution, masks: image 0 dense
    (gt > 0.7), image 1 sparse (about 5 %), image B-1 empty."""
    g = torch.Generator().manual_seed(seed)
    gts = torch.rand(B, 1, H, W, generator=g) * 10 + 0.5
    coarse = F.interpolate(gts, size=(H // 2, W // 2), mode="area")
    preds = coarse * (1 + 0.25 * (torch.rand(coarse.shape, generator=g) - 0.5)) * 1.1 + 0.05
    masks = gts > 0.7
    masks[1] &= torch.rand(1, H, W, generator=g) < 0.05
    masks[B - 1] = False
    return gts, preds, masks


def points_case(seed=12, B=2, H=200, W=300, empty=None):
    """Point maps gts, preds [B,3,H,W] (pred = gt + noise), masks [B,1,H,W] about 90 % valid, F1 thresholds as the
    reference's datasets build them (base_dataset.py:237-242, min_depth 0.01, max_depth 80)."""
    g = torch.Generator().manual_seed(seed)
    z = torch.rand(B, 1, H, W, generator=g) * 8 + 1.0
    uv = torch.randn(B, 2, H, W, generator=g)
    gts = torch.cat([uv * z * 0.5, z], dim=1)
    preds = gts + 0.6 * torch.randn(B, 3, H, W, generator=g)
    masks = torch.rand(B, 1, H, W, generator=g) < 0.9
    if empty is not None:
        masks[empty] = False
    thresholds = torch.linspace(math.log(0.01), math.log(80 / 20), steps=100).exp()
    return gts, preds, masks, thresholds


def knn_case(seed=13):
    """Ragged clouds: P1 != P2, lengths below P, one zero length, duplicated y points (exact ties), coordinates on a
    coarse grid (many equal distances) and a cloud offset by 1e3."""
    g = torch.Generator().manual_seed(seed)
    N, P1, P2 = 3, 300, 257
    x = torch.randn(N, P1, 3, generator=g)
    y = torch.randn(N, P2, 3, generator=g)
    x[0], y[0] = (x[0] * 4).round() / 4, (y[0] * 4).round() / 4
    y[0, 100:150] = y[0, 0:50]
    y[2, 200:257] = y[2, 0:57]
    x[2] += 1e3
    y[2] += 1e3
    lengths1 = torch.tensor([300, 211, 57], dtype=torch.int64)
    lengths2 = torch.tensor([257, 0, 240], dtype=torch.int64)
    return x, y, lengths1, lengths2
