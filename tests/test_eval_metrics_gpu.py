"""Evaluation metrics on the GPU (udb_nearest_neighbor, udb_depth_metrics, udb_point_metrics through
unidepth_b200.validation) against the unmodified reference's outputs (tests/golden/eval_metrics.npz) and against the
exact same-order brute force of oracle/eval_oracle.py at sizes the goldens do not cover."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import eval_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "eval_metrics.npz"))


def _bits(t):
    return t.detach().cpu().numpy().view(np.uint32)


# ------------------------------------------------------------------------------------------------ nearest neighbour
def test_nn_matches_reference_cpu_knn_bit_for_bit(gold):
    from unidepth_b200.validation import chamfer_distance
    x, y, l1, l2 = (t.to(DEV) for t in O.knn_case())
    dx, dy, ix, iy = chamfer_distance(x, y, l1, l2)
    assert np.array_equal(_bits(dx), gold["knn/xy/dist"].view(np.uint32))
    assert np.array_equal(ix.cpu().numpy(), gold["knn/xy/idx"])
    assert np.array_equal(_bits(dy), gold["knn/yx/dist"].view(np.uint32))
    assert np.array_equal(iy.cpu().numpy(), gold["knn/yx/idx"])


def _cloud(g, N, P, grid=None):
    p = torch.randn(N, P, 3, generator=g) * 3
    if grid:
        p = (p * grid).round() / grid          # many exactly equal distances
    return p


@pytest.mark.parametrize("P1,P2", [(1, 1), (2, 2), (127, 127), (128, 128), (129, 129), (4097, 4097), (76800, 76800),
                                   (1, 300), (300, 1), (129, 4097), (4097, 130)])
def test_nn_exact_against_same_order_brute_force(P1, P2):
    from unidepth_b200 import ops
    g = torch.Generator().manual_seed(P1 * 7919 + P2)
    N = 1 if P1 * P2 > 1e8 else 2
    x = _cloud(g, N, P1, grid=8 if P1 < 5000 else None).to(DEV)
    y = _cloud(g, N, P2, grid=8 if P2 < 5000 else None).to(DEV)
    if P2 > 2:
        y[:, P2 // 2:P2 // 2 + 1] = y[:, :1]       # a duplicated reference point: a tie
    l1 = torch.tensor([P1, max(0, P1 - 3)][:N], device=DEV)
    l2 = torch.tensor([P2, max(1, P2 // 2)][:N], device=DEV)
    dx, ix, dy, iy = ops.nearest_neighbor(x, y, l1, l2)
    rdx, rix = O.knn1(x, y, l1.tolist(), l2.tolist(), chunk=1024)
    rdy, riy = O.knn1(y, x, l2.tolist(), l1.tolist(), chunk=1024)
    assert torch.equal(dx.view(torch.int32), rdx.view(torch.int32)) and torch.equal(ix, rix)
    assert torch.equal(dy.view(torch.int32), rdy.view(torch.int32)) and torch.equal(iy, riy)
    # one-direction launches give the same as the fused pass, and a second run is bit-identical
    dx1, ix1, n1, n2 = ops.nearest_neighbor(x, y, l1, l2, both=False)
    dy1, iy1, _, _ = ops.nearest_neighbor(y, x, l2, l1, both=False)
    assert n1 is None and n2 is None
    assert torch.equal(dx1.view(torch.int32), dx.view(torch.int32)) and torch.equal(ix1, ix)
    assert torch.equal(dy1.view(torch.int32), dy.view(torch.int32)) and torch.equal(iy1, iy)
    dx2, ix2, dy2, iy2 = ops.nearest_neighbor(x, y, l1, l2)
    assert all(torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32) if b.dtype == torch.float32 else b)
               for a, b in ((dx, dx2), (ix, ix2), (dy, dy2), (iy, iy2)))


def test_nn_overwrites_a_nan_canary_and_zeroes_empty_rows():
    from unidepth_b200 import _cabi as cabi
    g = torch.Generator().manual_seed(3)
    x, y = _cloud(g, 3, 200).to(DEV), _cloud(g, 3, 150).to(DEV)
    l1, l2 = torch.tensor([200, 17, 0], device=DEV), torch.tensor([0, 150, 99], device=DEV)
    dx, dy = torch.full((3, 200), float("nan"), device=DEV), torch.full((3, 150), float("nan"), device=DEV)
    ix, iy = torch.full((3, 200), -7, dtype=torch.int64, device=DEV), torch.full((3, 150), -7, dtype=torch.int64, device=DEV)
    p = cabi.NearestNeighbor(x=x.data_ptr(), y=y.data_ptr(), lengths1=l1.data_ptr(), lengths2=l2.data_ptr(), N=3, P1=200,
                             P2=150, dist_x=dx.data_ptr(), idx_x=ix.data_ptr(), dist_y=dy.data_ptr(), idx_y=iy.data_ptr())
    cabi.check(cabi.lib().udb_nearest_neighbor(ctypes.byref(p), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "udb_nearest_neighbor")
    torch.cuda.synchronize()
    assert not dx.isnan().any() and not dy.isnan().any() and (ix >= 0).all() and (iy >= 0).all()
    assert (dx[0] == 0).all() and (ix[0] == 0).all() and (dx[1, 17:] == 0).all() and (dx[2] == 0).all()
    assert (dy[0] == 0).all() and (dy[2] == 0).all() and (dy[1, :] > 0).all()
    rdx, rix = O.knn1(x, y, l1.tolist(), l2.tolist())
    assert torch.equal(dx, rdx) and torch.equal(ix, rix)


def test_chamfer_distance_batched_equals_per_cloud_and_rejects_bad_arguments():
    from unidepth_b200.validation import chamfer_distance
    g = torch.Generator().manual_seed(4)
    x, y = _cloud(g, 3, 500).to(DEV), _cloud(g, 3, 400).to(DEV)
    lx, ly = torch.tensor([500, 321, 1], device=DEV), torch.tensor([400, 7, 399], device=DEV)
    full = chamfer_distance(x, y, lx, ly)
    for n in range(3):
        one = chamfer_distance(x[n:n + 1, :int(lx[n])], y[n:n + 1, :int(ly[n])])
        assert torch.equal(one[0][0], full[0][n, :int(lx[n])]) and torch.equal(one[2][0], full[2][n, :int(lx[n])])
        assert torch.equal(one[1][0], full[1][n, :int(ly[n])]) and torch.equal(one[3][0], full[3][n, :int(ly[n])])
    with pytest.raises(ValueError, match=r"\[0, 500\]"):
        chamfer_distance(x, y, torch.tensor([500, 501, 0], device=DEV), None)
    with pytest.raises(ValueError, match=r"\[0, 400\]"):
        chamfer_distance(x, y, None, torch.tensor([-1, 3, 3], device=DEV))
    with pytest.raises(ValueError, match="shape"):
        chamfer_distance(x, y, torch.tensor([5, 5], device=DEV))
    with pytest.raises(TypeError, match="int64"):
        chamfer_distance(x, y, torch.tensor([5, 5, 5], device=DEV, dtype=torch.int32))
    with pytest.raises(TypeError, match="float32"):
        chamfer_distance(x.double(), y)
    with pytest.raises(ValueError):
        chamfer_distance(x[..., :2].contiguous(), y[..., :2].contiguous())


# ------------------------------------------------------------------------------------------------------ eval_depth
COUNTS = {"d1", "d2", "d3", "tau", "d1_si", "tau_si"}
SSI_COUNTS = {"d1_ssi", "tau_ssi"}


def depth_bound(key, r32, r64, n):
    """Allowed |GPU - reference fp32| per image.  The kernel sums in f64 where the reference sums in fp32, so the
    reference's own fp32-vs-fp64 difference (stored in the golden), doubled, bounds the sums, plus 1e-5 relative for
    the last-ulp differences of CUDA's logf / powf against the CPU's.  Counts of the plain and si ratios are exact.
    ssi solves its 2 x 2 system in f64 (the reference: fp32), which may move a few ratios across a threshold: 3 pixels
    (3 / n) for the ssi counts and for d_auc (whose 100 thresholds come from powf)."""
    if key in COUNTS:
        return np.zeros_like(r32)
    tol = 2 * np.abs(r32 - r64) + 1e-5 * np.abs(r32) + 1e-6
    if key in SSI_COUNTS or key == "d_auc":
        tol = tol + 3.0 / n
    return tol


@pytest.mark.parametrize("tag,max_depth", [("nomax", None), ("max", 7.5)])
def test_eval_depth_matches_reference(gold, tag, max_depth):
    from unidepth_b200.validation import eval_depth
    gts, preds, masks = O.depth_case()
    valid = masks & (gts <= max_depth) if max_depth is not None else masks
    n = valid.reshape(3, -1).sum(1).double().numpy()
    got = eval_depth(gts.to(DEV), preds.to(DEV), masks.to(DEV), max_depth=max_depth)
    assert list(got) == O.KEYS
    for k in O.KEYS:
        g = got[k].cpu().numpy()
        assert got[k].dtype == torch.float32 and g.shape == (3,)
        r32, r64 = gold[f"depth/{tag}/{k}"], gold[f"depth64/{tag}/{k}"]
        assert np.isnan(g[2]) and np.isnan(r32[2]), k                   # empty mask: NaN, as the reference on CPU
        err, tol = np.abs(g[:2] - r32[:2]), depth_bound(k, r32[:2], r64[:2], n[:2])
        print(tag, k, g[:2], r32[:2], err, tol)
        assert np.all(err <= tol), (k, g, r32, err, tol)


def test_eval_depth_batched_equals_per_image_and_rejects_bad_arguments():
    from unidepth_b200.validation import eval_depth
    gts, preds, masks = (t.to(DEV) for t in O.depth_case())
    full = eval_depth(gts, preds, masks.to(torch.uint8), max_depth=9.0)
    for i in range(3):
        one = eval_depth(gts[i:i + 1], preds[i:i + 1], masks[i:i + 1], max_depth=9.0)
        for k in O.KEYS:
            assert torch.equal(one[k], full[k][i:i + 1]) or (one[k].isnan().all() and full[k][i].isnan()), k
    with pytest.raises(TypeError, match="float32"):
        eval_depth(gts.double(), preds, masks)
    with pytest.raises(TypeError, match="bool"):
        eval_depth(gts, preds, masks.float())
    with pytest.raises(ValueError, match="CUDA"):
        eval_depth(gts, preds.cpu(), masks)


# --------------------------------------------------------------------------------------------------------- eval_3d
@pytest.mark.parametrize("tag,kw", [("big", dict(B=32, H=48, W=60)), ("empty", dict(seed=14, H=40, W=50, empty=1))])
def test_eval_3d_matches_reference(gold, tag, kw):
    """F1 comes from exact counts (precision and recall equal the reference's bit for bit); only trapz's summation
    order may differ (1e-6).  MSE_3d and chamfer: twice the reference's fp32-vs-fp64 difference, plus 1e-6 relative."""
    from unidepth_b200.validation import eval_3d
    gts, preds, masks, thr = O.points_case(**kw)
    got = eval_3d(gts.to(DEV), preds.to(DEV), masks.to(DEV), thresholds=thr.to(DEV))
    assert list(got) == ["MSE_3d", "chamfer", "F1"]
    for k in got:
        g, r32 = got[k].cpu().numpy(), gold[f"e3d/{tag}/{k}"]
        assert g.shape == r32.shape and got[k].dtype == torch.float32, (k, g.shape, r32.shape)
        tol = 1e-6 * np.abs(r32) + 1e-7 if k == "F1" else 2 * np.abs(r32 - gold[f"e3d64/{tag}/{k}"]) + 1e-6 * np.abs(r32)
        print(tag, k, np.abs(g - r32).max(), tol.min())
        assert np.all(np.abs(g - r32) <= tol), (k, g, r32)
    # thresholds as a list and in another order give the same result
    again = eval_3d(gts.to(DEV), preds.to(DEV), masks.to(DEV), thresholds=thr.flip(0).tolist())
    ref_flip = O.eval_3d(gts, preds, masks, thr.flip(0))
    assert np.allclose(again["F1"].cpu().numpy(), ref_flip["F1"].numpy(), rtol=1e-6, atol=1e-7)


def test_eval_3d_all_empty_and_bad_arguments():
    from unidepth_b200.validation import eval_3d
    gts, preds, masks, thr = O.points_case(seed=15, B=2, H=20, W=30)
    assert eval_3d(gts.to(DEV), preds.to(DEV), torch.zeros_like(masks).to(DEV), thr) == {}
    with pytest.raises(ValueError, match="thresholds"):
        eval_3d(gts.to(DEV), preds.to(DEV), masks.to(DEV), thresholds=None)
    with pytest.raises(ValueError, match="thresholds"):
        eval_3d(gts.to(DEV), preds.to(DEV), masks.to(DEV), thresholds=torch.ones(2, 3))
    with pytest.raises(TypeError, match="float32"):
        eval_3d(gts.double().to(DEV), preds.to(DEV), masks.to(DEV), thr)
