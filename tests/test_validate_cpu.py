"""Evaluation over a test set without a GPU: the argument checks of udb_camera_reconstruct, DatasetMetrics' key
selection / keyframe / threshold / NaN / clearing rules against the unmodified reference's accumulation
(tests/golden/validate_metrics.npz, made by oracle/make_golden_validate.py) with the metrics restated on the CPU
(oracle/eval_oracle.py), the cross-rank gather on a gloo group, and validate's batch handling."""
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from unidepth_b200 import _cabi
from unidepth_b200 import camera as C
from unidepth_b200 import validation as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "validate_metrics.npz")
sys.path.insert(0, os.path.join(ROOT, "oracle"))


# ---------------------------------------------------------------------------------------------------------------- ABI
BASE = 1 << 28


def _child_main():
    """Runs in a fresh interpreter with no visible GPU; prints one JSON dict of results."""
    lib = _cabi.lib()
    res = {}
    good = dict(model=_cabi.CAM_MEI, params=BASE, B=2, H=30, W=40, depth=BASE + (1 << 20), points=BASE + (1 << 22))
    cases = {"model0": dict(good, model=0), "model7": dict(good, model=7), "B0": dict(good, B=0),
             "B65536": dict(good, B=65536), "H0": dict(good, H=0), "W0": dict(good, W=0),
             "HW_big": dict(good, H=1 << 16, W=1 << 15), "params_null": dict(good, params=0),
             "params_misaligned": dict(good, params=BASE + 4), "depth_null": dict(good, depth=0),
             "depth_misaligned": dict(good, depth=BASE + (1 << 20) + 2), "points_null": dict(good, points=0),
             "points_misaligned": dict(good, points=BASE + (1 << 22) + 1), "valid": good}
    for name, a in cases.items():
        n0 = lib.udb_launch_count()
        rc = lib.udb_camera_reconstruct(a["model"], a["params"], a["B"], a["H"], a["W"], a["depth"], a["points"], None)
        res[name] = {"rc": rc, "msg": lib.udb_last_error().decode(), "launched": lib.udb_launch_count() - n0}
    json.dump(res, sys.stdout)


@pytest.fixture(scope="module")
def abi():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    code = "import sys; sys.path[:0] = ['tests']; import test_validate_cpu as t; t._child_main()"
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, check=True).stdout
    return json.loads(out)


@pytest.mark.parametrize("case,text", [("model0", "`model` 0"), ("model7", "`model` 7"), ("B0", "B=0"),
                                       ("B65536", "B=65536"), ("H0", "H=0"), ("W0", "W=0"), ("HW_big", "H * W exceeds 2^30"),
                                       ("params_null", "`params` is null"), ("params_misaligned", "`params` must be 16-byte"),
                                       ("depth_null", "`depth` is null"), ("depth_misaligned", "`depth` must be 4-byte"),
                                       ("points_null", "`points` is null"), ("points_misaligned", "`points` must be 4-byte")])
def test_camera_reconstruct_rejects_before_launch(abi, case, text):
    r = abi[case]
    print(case, r)
    assert r["rc"] != 0 and r["launched"] == 0, r
    assert r["msg"].startswith("udb_camera_reconstruct: ") and text in r["msg"], r


def test_valid_reconstruct_call_gets_past_the_checks(abi):
    r = abi["valid"]
    assert r["rc"] != 0 and r["launched"] == 0 and "`" not in r["msg"], r            # only the launch itself fails


# ----------------------------------------------------------------------------------------------- accumulation rules
class _CpuMetrics(V.DatasetMetrics):
    """DatasetMetrics with the metrics restated on the CPU; reconstruct takes the host path for CPU tensors."""
    import eval_oracle as _O
    eval_depth = staticmethod(_O.eval_depth)
    eval_3d = staticmethod(_O.eval_3d)


def _accumulate(cls=_CpuMetrics):
    import validate_oracle as VO
    m = cls(min_depth=VO.MIN_DEPTH, max_depth=VO.MAX_DEPTH)
    for inputs, preds, kf in VO.batches(C):
        keys = set(inputs)
        m.accumulate_metrics(inputs=inputs, preds=preds, keyframe_idx=kf)
        assert set(inputs) == keys                           # the caller's dict is not modified
    return m


def test_accumulation_reproduces_the_reference_store_and_evaluation():
    z = np.load(GOLD)
    m = _accumulate()
    want_stores = sorted(k for k in z.files if k.startswith("store/"))
    got_stores = sorted(f"store/{t}/{n}" for t, s in m.metrics_store.items() for n in s)
    assert got_stores == want_stores
    assert sorted(m.metrics_store) == ["", "aux"] and len(m.metrics_store[""]) == 21
    worst = {}
    for key in want_stores:
        _, t, n = key.split("/")
        got, want = m.metrics_store[t][n].numpy(), z[key]
        assert got.shape == want.shape, (key, got.shape, want.shape)
        assert np.array_equal(np.isnan(got), np.isnan(want)), key
        ok = ~np.isnan(want)
        e = np.abs(got[ok] - want[ok]).max() if ok.any() else 0.0
        worst[key] = e
        # the host Fisheye624 solves to convergence, the reference's loop stops at a residual of 1e-3: the points of
        # that batch, and so the 3D metrics, differ slightly (8.7e-5 at most measured); everything else is the same
        # fp32 arithmetic
        tol = (5e-4 if n in ("MSE_3d", "chamfer", "F1") else 1e-5) * max(1.0, np.abs(want[ok]).max())
        assert e <= tol, (key, e, tol)
    print("largest |store - reference| per metric:", {k: f"{v:.2e}" for k, v in worst.items()})
    for t in m.metrics_count:
        assert np.array_equal(m.metrics_count[t].numpy(), z[f"count/{t}"]), t
    ev = m.get_evaluation()
    assert list(ev) == list(z["eval_keys"])
    for k, v in ev.items():
        want = float(z[f"eval/{k}"])
        assert isinstance(v, float) and (np.isnan(v) == np.isnan(want)), k
        assert np.isnan(want) or abs(v - want) <= (5e-4 if k in ("MSE_3d", "chamfer", "F1") else 1e-5) * max(1.0, abs(want)), (k, v, want)
    assert all(np.isnan(ev[k]) for k in ("d1", "rmse", "silog"))           # an empty-mask image makes the mean NaN
    assert m.metrics_store == {"": {}, "aux": {}} and m.metrics_count == {}
    with pytest.raises(AssertionError):
        m.get_evaluation()                                                 # emptied stores, nothing added since


def test_available_metrics_and_keyframe_attribute():
    """No depth in the inputs: no point map and no metric at all; a key of preds that only contains "points" selects
    the 3D metrics alone; the dataset's keyframe_idx attribute slices the depth evaluation only."""
    g = torch.Generator().manual_seed(5)
    d = torch.rand(3, 1, 12, 16, generator=g) + 1.0
    cam = C.Pinhole(params=torch.tensor([[14.0, 14.0, 8.0, 6.0]]))
    m = _CpuMetrics()
    m.accumulate_metrics({"image": d, "camera": cam}, {"depth": d})
    assert m.metrics_store == {}
    inputs = {"depth": d, "depth_mask": torch.ones_like(d, dtype=torch.bool), "camera": cam}
    m.accumulate_metrics(inputs, {"points_final": torch.rand(3, 3, 12, 16, generator=g)})
    assert list(m.metrics_store) == ["final"] and m.metrics_store["final"]["F1"].shape == (3,)
    m = _CpuMetrics()
    m.keyframe_idx = 1
    m.accumulate_metrics(inputs, {"depth": d * 1.1, "points": torch.rand(3, 3, 12, 16, generator=g)})
    assert m.metrics_store[""]["d1"].shape == (1,) and m.metrics_store[""]["F1"].shape == (3,)


def test_documented_errors():
    m = _CpuMetrics()
    d = torch.rand(2, 1, 8, 8) + 1.0
    inputs = {"depth": d, "depth_mask": torch.ones_like(d), "points": torch.rand(2, 3, 8, 8)}
    with pytest.raises(ValueError, match="'depth_features'"):
        m.accumulate_metrics(inputs, {"depth": d, "depth_features": torch.rand(2, 64, 512)})
    assert m.metrics_store == {}                                           # raised before any metric ran
    with pytest.raises(AssertionError):
        m.metrics_store["x"] = {}
        m.metrics_count["x"] = torch.tensor([])
        m.get_evaluation()


# ------------------------------------------------------------------------------------------------------ cross-rank
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _local(rank):
    return torch.arange(3 + 2 * rank, dtype=torch.float32) + 100 * rank


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from unidepth_b200.validation import gather_across_ranks
    got = gather_across_ranks(_local(rank))
    scalar = gather_across_ranks(torch.tensor(float(rank)))
    q.put((rank, got.tolist(), scalar.tolist()))
    dist.destroy_process_group()


def test_gather_across_ranks_on_gloo():
    assert torch.equal(V.gather_across_ranks(_local(1)), _local(1))      # not initialised: unchanged
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = torch.cat([_local(r) for r in range(world)]).tolist()
    for rank, got, scalar in res:
        assert got == want, rank
        assert scalar == [0.0, 1.0]


# --------------------------------------------------------------------------------------------------------- validate
class _StubModel(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))
        self.calls = []

    @property
    def device(self):
        return self.w.device

    def forward(self, data, metas):
        self.calls.append((data, metas, torch.is_grad_enabled()))
        return {"depth": data["depth"] * 2.0}


class _Recorder(V.DatasetMetrics):
    def accumulate_metrics(self, inputs, preds, keyframe_idx=None, metrics=("depth", "points", "flow_fwd", "pairwise")):
        self.seen = getattr(self, "seen", []) + [(inputs, preds, keyframe_idx)]
        self.metrics_store.setdefault("", {})["n"] = torch.cat([self.metrics_store.get("", {}).get("n", torch.tensor([])),
                                                                torch.tensor([float(inputs["depth"].shape[0])])])
        self.metrics_count[""] = torch.tensor([1.0])


class _Loader(list):
    def __init__(self, batches, dataset):
        super().__init__(batches)
        self.dataset = dataset


class _NoSqueeze:
    def to(self, device):
        return self


def test_validate_batch_handling(capsys):
    model = _StubModel()
    rec = _Recorder()
    cam = _NoSqueeze()
    depth = torch.rand(2, 1, 1, 4, 5)
    batch = {"data": {"depth": depth, "camera": cam},
             "img_metas": [{"keyframe_idx": [1], "paddings": [(0, 0, 0, 0)], "dropped": 3}, {"keyframe_idx": [1]}]}
    out = V.validate(model, {"ds": _Loader([batch, batch], rec)})
    data, metas, grad = model.calls[0]
    assert data["depth"].shape == (2, 1, 4, 5) and data["camera"] is cam and not grad
    assert metas == [{"keyframe_idx": 1, "paddings": (0, 0, 0, 0)}, {"keyframe_idx": 1}]
    assert batch["data"]["depth"] is depth and isinstance(batch["img_metas"][0]["keyframe_idx"], list)   # unchanged
    assert [s[2] for s in rec.seen] == [1, 1] and torch.equal(rec.seen[0][1]["depth"], data["depth"] * 2.0)
    assert out == {"ds": {"n": 2.0}}
    assert "Metrics/ds/n 2.0" in capsys.readouterr().out


def test_validate_builds_metrics_from_the_dataset_limits(monkeypatch):
    made = []
    real = V.DatasetMetrics.__init__

    def spy(self, min_depth=0.01, max_depth=1000.0):
        made.append((min_depth, max_depth))
        real(self, min_depth, max_depth)

    monkeypatch.setattr(V.DatasetMetrics, "__init__", spy)
    monkeypatch.setattr(V.DatasetMetrics, "get_evaluation", lambda self, metrics=None: {})

    class _DS:
        min_depth, max_depth = 0.1, 80.0

    V.validate(_StubModel(), {"a": _Loader([], _DS()), "b": _Loader([], object())})
    assert made == [(0.1, 80.0), (0.01, 1000.0)]
