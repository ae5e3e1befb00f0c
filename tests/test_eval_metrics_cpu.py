"""Evaluation metrics on the CPU: the pure-torch oracle (oracle/eval_oracle.py) against the unmodified reference's
outputs in tests/golden/eval_metrics.npz (oracle/make_golden_eval.py), the argument checks of udb_nearest_neighbor,
udb_depth_metrics and udb_point_metrics (fresh interpreter, no visible GPU, fake device pointers, so nothing can
launch), their ctypes layouts, and the Python layer's refusals that need no GPU."""
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import eval_oracle as O  # noqa: E402

from unidepth_b200 import _cabi  # noqa: E402


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "eval_metrics.npz"))


# --------------------------------------------------------------------------------------------------------- oracle
def test_oracle_knn_is_bit_identical_to_reference_cpu_knn(gold):
    x, y, l1, l2 = O.knn_case()
    for tag, (a, b, la, lb) in (("xy", (x, y, l1, l2)), ("yx", (y, x, l2, l1))):
        d, i = O.knn1(a, b, la, lb, chunk=64)
        assert np.array_equal(d.numpy().view(np.uint32), gold[f"knn/{tag}/dist"].view(np.uint32)), tag
        assert np.array_equal(i.numpy(), gold[f"knn/{tag}/idx"]), tag
    assert (gold["knn/xy/dist"][1] == 0).all() and (gold["knn/xy/idx"][2, 57:] == 0).all()   # zero length / past length


@pytest.mark.parametrize("tag,max_depth", [("nomax", None), ("max", 7.5)])
def test_oracle_eval_depth_reproduces_reference(gold, tag, max_depth):
    got = O.eval_depth(*O.depth_case(), max_depth=max_depth)
    assert list(got) == O.KEYS
    for k in O.KEYS:
        ref = gold[f"depth/{tag}/{k}"]
        assert np.allclose(got[k].numpy(), ref, rtol=1e-6, atol=0, equal_nan=True), (k, got[k], ref)
        assert np.isnan(ref[-1]) and np.isnan(got[k][-1].item()), k          # the empty-mask image: NaN everywhere


@pytest.mark.parametrize("tag,kw", [("big", dict(B=32, H=48, W=60)), ("empty", dict(seed=14, H=40, W=50, empty=1))])
def test_oracle_eval_3d_reproduces_reference(gold, tag, kw):
    gts, preds, masks, thr = O.points_case(**kw)
    got = O.eval_3d(gts, preds, masks, thr)
    for k in ("MSE_3d", "chamfer", "F1"):
        ref = gold[f"e3d/{tag}/{k}"]
        assert got[k].shape == ref.shape and np.allclose(got[k].numpy(), ref, rtol=1e-6, atol=0), (k, got[k], ref)
    if tag == "big":       # the batch-wide downscale ran
        assert tuple(gold["e3d/big/hw"]) < (48, 60) and masks.sum() > 240 * 320
    else:
        assert gold["e3d/empty/F1"].shape == (1,)


def test_f32_vs_f64_reference_differences_are_small(gold):
    """The GPU tests bound each metric by 2 x |reference fp32 - reference fp64| plus a small relative term (see
    test_eval_metrics_gpu.depth_bound); this records that those differences are at the fp32 rounding level."""
    for tag in ("nomax", "max"):
        for k in O.KEYS:
            a, b = gold[f"depth/{tag}/{k}"][:-1], gold[f"depth64/{tag}/{k}"][:-1]
            assert np.all(np.abs(a - b) <= 2e-3 * np.abs(b) + 1e-4), (tag, k, a, b)
    for tag in ("big", "empty"):
        for k in ("MSE_3d", "chamfer"):
            a, b = gold[f"e3d/{tag}/{k}"], gold[f"e3d64/{tag}/{k}"]
            assert np.all(np.abs(a - b) <= 1e-5 * np.abs(b)), (tag, k, a, b)


# ------------------------------------------------------------------------------------------------------------ ABI
def test_ctypes_structs_match_c_layout():
    structs = {"udb_nn_t": (_cabi.NearestNeighbor, "idx_y"), "udb_depth_metrics_t": (_cabi.DepthMetrics, "ssi"),
               "udb_point_metrics_t": (_cabi.PointMetrics, "out")}
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "udb.h"\nint main(){\n'
    for n, (_, last) in structs.items():
        src += f'printf("{n} %zu %zu\\n", sizeof({n}), offsetof({n}, {last}));\n'
    src += ('printf("consts %d %d %d %d %d %d\\n", UDB_METRIC_MAX_BLOCKS, UDB_DM_AUC_BINS, UDB_DM_AUC, UDB_DM_AREL_SSI, '
            'UDB_DM_NACC, UDB_PM_MAX_THRESHOLDS);\nreturn 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        out = subprocess.check_output([os.path.join(d, "t")], text=True).strip().splitlines()
    for line in out[:-1]:
        n, size, off = line.split()
        cs, last = structs[n]
        assert ctypes.sizeof(cs) == int(size) and getattr(cs, last).offset == int(off), (n, ctypes.sizeof(cs), size)
    assert [int(v) for v in out[-1].split()[1:]] == [_cabi.METRIC_MAX_BLOCKS, _cabi.DM_AUC_BINS, _cabi.DM_AUC,
                                                     _cabi.DM_AREL_SSI, _cabi.DM_NACC, _cabi.PM_MAX_THRESHOLDS]


BASE = 1 << 28


def _child_main():
    """Runs in a fresh interpreter with no visible GPU; prints one JSON dict of results."""
    import ctypes as Ct
    lib = _cabi.lib()
    res = {}

    def rec(name, fn):
        n0 = lib.udb_launch_count()
        rc = fn()
        res[name] = {"rc": rc, "msg": lib.udb_last_error().decode(), "launched": lib.udb_launch_count() - n0}

    nn = dict(x=BASE, y=BASE + (1 << 20), lengths1=0, lengths2=0, N=2, P1=300, P2=257, dist_x=BASE + (2 << 20),
              idx_x=BASE + (3 << 20), dist_y=BASE + (4 << 20), idx_y=BASE + (5 << 20))
    cases = {"N0": dict(N=0), "P1_0": dict(P1=0), "P2_0": dict(P2=0), "x_null": dict(x=0), "x_misaligned": dict(x=BASE + 2),
             "y_null": dict(y=0), "lengths1_misaligned": dict(lengths1=BASE + 4), "lengths2_misaligned": dict(lengths2=BASE + 4),
             "dist_x_null": dict(dist_x=0), "idx_x_null": dict(idx_x=0), "idx_x_misaligned": dict(idx_x=BASE + (3 << 20) + 4),
             "dist_y_only": dict(idx_y=0), "idx_y_misaligned": dict(idx_y=BASE + (5 << 20) + 4), "valid": {}, "valid_one": dict(dist_y=0, idx_y=0)}
    for name, extra in cases.items():
        p = _cabi.NearestNeighbor(**dict(nn, **extra))
        rec("nn:" + name, lambda p=p: lib.udb_nearest_neighbor(Ct.byref(p), None))

    dm = dict(gt=BASE, pred=BASE + (1 << 20), mask=BASE + (2 << 20), B=2, HW=4800, auc_thresholds=BASE + (3 << 20),
              medians=BASE + (3 << 20) + 512, partials=BASE + (4 << 20), out=BASE + (5 << 20), ssi=BASE + (6 << 20))
    cases = {"B0": dict(B=0), "HW0": dict(HW=0), "gt_null": dict(gt=0), "pred_misaligned": dict(pred=BASE + (1 << 20) + 2),
             "mask_null": dict(mask=0), "auc_thresholds_null": dict(auc_thresholds=0), "medians_null": dict(medians=0),
             "partials_misaligned": dict(partials=BASE + (4 << 20) + 4), "out_null": dict(out=0), "ssi_null": dict(ssi=0),
             "valid": {}}
    for name, extra in cases.items():
        p = _cabi.DepthMetrics(**dict(dm, **extra))
        rec("dm:" + name, lambda p=p: lib.udb_depth_metrics(Ct.byref(p), None))

    pm = dict(gt=BASE, pred=BASE + (1 << 20), lengths=0, dist_x=BASE + (2 << 20), dist_y=BASE + (3 << 20),
              thresholds=BASE + (4 << 20), N=2, P=1000, n_thresholds=100, partials=BASE + (5 << 20), out=BASE + (6 << 20))
    cases = {"N0": dict(N=0), "P0": dict(P=0), "T0": dict(n_thresholds=0), "T_big": dict(n_thresholds=1025),
             "gt_null": dict(gt=0), "pred_null": dict(pred=0), "lengths_misaligned": dict(lengths=BASE + 4),
             "dist_x_null": dict(dist_x=0), "dist_y_null": dict(dist_y=0), "thresholds_null": dict(thresholds=0),
             "partials_null": dict(partials=0), "out_misaligned": dict(out=BASE + (6 << 20) + 4), "valid": {}}
    for name, extra in cases.items():
        p = _cabi.PointMetrics(**dict(pm, **extra))
        rec("pm:" + name, lambda p=p: lib.udb_point_metrics(Ct.byref(p), None))
    json.dump(res, sys.stdout)


@pytest.fixture(scope="module")
def abi():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    code = "import sys; sys.path[:0] = ['tests']; import test_eval_metrics_cpu as t; t._child_main()"
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, check=True).stdout
    return json.loads(out)


@pytest.mark.parametrize("case,field", [
    ("nn:N0", "N=0"), ("nn:P1_0", "P1=0"), ("nn:P2_0", "P2=0"), ("nn:x_null", "`x`"), ("nn:x_misaligned", "`x`"),
    ("nn:y_null", "`y`"), ("nn:lengths1_misaligned", "`lengths1`"), ("nn:lengths2_misaligned", "`lengths2`"),
    ("nn:dist_x_null", "`dist_x`"), ("nn:idx_x_null", "`idx_x`"), ("nn:idx_x_misaligned", "`idx_x`"),
    ("nn:dist_y_only", "`dist_y`"), ("nn:idx_y_misaligned", "`idx_y`"),
    ("dm:B0", "B=0"), ("dm:HW0", "HW=0"), ("dm:gt_null", "`gt`"), ("dm:pred_misaligned", "`pred`"),
    ("dm:mask_null", "`mask`"), ("dm:auc_thresholds_null", "`auc_thresholds`"), ("dm:medians_null", "`medians`"),
    ("dm:partials_misaligned", "`partials`"), ("dm:out_null", "`out`"), ("dm:ssi_null", "`ssi`"),
    ("pm:N0", "N=0"), ("pm:P0", "P=0"), ("pm:T0", "n_thresholds=0"), ("pm:T_big", "n_thresholds=1025"),
    ("pm:gt_null", "`gt`"), ("pm:pred_null", "`pred`"), ("pm:lengths_misaligned", "`lengths`"),
    ("pm:dist_x_null", "`dist_x`"), ("pm:dist_y_null", "`dist_y`"), ("pm:thresholds_null", "`thresholds`"),
    ("pm:partials_null", "`partials`"), ("pm:out_misaligned", "`out`")])
def test_metric_entry_points_reject_before_launch(abi, case, field):
    r = abi[case]
    print(case, r)
    assert r["rc"] != 0 and field in r["msg"] and r["launched"] == 0, r
    assert "CUDA" not in r["msg"] and "device" not in r["msg"], r


@pytest.mark.parametrize("case", ["nn:valid", "nn:valid_one", "dm:valid", "pm:valid"])
def test_valid_metric_calls_get_past_the_checks(abi, case):
    r = abi[case]
    assert r["rc"] != 0 and r["launched"] == 0 and "`" not in r["msg"], r            # only the launch itself fails


# --------------------------------------------------------------------------------------------------------- Python
def test_python_layer_refuses_cpu_tensors_and_missing_thresholds():
    from unidepth_b200 import validation as V
    g = torch.rand(2, 1, 8, 8) + 0.5
    m = torch.ones(2, 1, 8, 8, dtype=torch.bool)
    with pytest.raises(ValueError, match="CUDA"):
        V.eval_depth(g, g, m)
    pts = torch.rand(2, 3, 8, 8)
    with pytest.raises(ValueError, match="thresholds"):
        V.eval_3d(pts, pts, m, thresholds=None)
    with pytest.raises(ValueError, match="CUDA"):
        V.eval_3d(pts, pts, m, thresholds=[0.1, 0.2])
    x = torch.rand(2, 10, 3)
    with pytest.raises(ValueError, match="CUDA"):
        V.chamfer_distance(x, x)
    with pytest.raises(TypeError):
        V.chamfer_distance(x.numpy(), x)
