"""`interpolation_mode = "bicubic"` without a GPU: the oracle against the unmodified reference's bicubic outputs
(tests/golden/vits_bicubic_*.npz, made by oracle/make_golden_bicubic.py), and the host checks of the mode fields of
udb_postprocess_t and udb_infer_args_t (include/udb.h), which must reject an unknown mode before any launch."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import unidepth_oracle as O
from fixture import make_state_dict
from test_oracle_golden import _rgb, subsample_like_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BICUBIC_CASES = ["vits_bicubic_120x160", "vits_bicubic_pad_96x288_rl3", "vits_bicubic_700x1000_rl0", "vits_bicubic_camK_120x160"]


def golden_camera(meta):
    """The K tensor a bicubic golden was made with, or None."""
    cam = meta.get("camera")
    if cam is None:
        return None
    fx, fy, cx, cy = cam["params"]
    return torch.tensor([[[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]]])


@pytest.mark.parametrize("name", BICUBIC_CASES)
def test_oracle_bicubic_matches_reference_golden(name, golden_dir):
    """Same bars as test_oracle_golden.py: 3e-4 relative per tensor (floored at 10 % of its mean magnitude), depth 5e-5,
    intrinsics 1e-5."""
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    meta = json.loads(str(z["__meta__"]))
    assert meta["interpolation_mode"] == "bicubic"
    cfg = json.load(open(os.path.join(golden_dir, meta["config"])))
    sd = make_state_dict(cfg, meta["seed"])
    out = O.infer_v2(sd, cfg, _rgb(meta["shape"], meta["seed"]), resolution_level=meta["resolution_level"],
                     interpolation_mode="bicubic", camera=golden_camera(meta))
    out = subsample_like_golden(out, meta)
    assert set(out) == set(z.files) - {"__meta__"}
    for k, v in out.items():
        ref = torch.from_numpy(z[k])
        assert v.shape == ref.shape, (k, v.shape, ref.shape)
        floor = 0.1 * ref.abs().mean().item()
        err = ((v - ref).abs() / ref.abs().clamp(min=floor)).max().item()
        print(name, k, "max rel err", err)
        assert err < 3e-4, (k, err)
    dr = torch.from_numpy(z["depth"])
    assert ((out["depth"] - dr).abs() / dr.abs()).max().item() < 5e-5
    kk, kr = out["intrinsics"], torch.from_numpy(z["intrinsics"])
    for (i, j) in ((0, 0), (1, 1), (0, 2), (1, 2)):
        assert ((kk[:, i, j] - kr[:, i, j]).abs() / kr[:, i, j].abs()).max().item() < 1e-5
    # the mode took effect: the bilinear oracle on the same input differs
    lin = subsample_like_golden(O.infer_v2(sd, cfg, _rgb(meta["shape"], meta["seed"]), resolution_level=meta["resolution_level"],
                                           camera=golden_camera(meta)), meta)
    assert (lin["depth"] - dr).abs().max().item() > 1e-4


BASE = 1 << 28          # fake device addresses; CUDA_VISIBLE_DEVICES="" keeps every launch from reaching a device


def _child_main():
    """Runs in a fresh interpreter with no visible GPU; prints one JSON dict of results."""
    import ctypes as C

    from unidepth_b200 import _cabi
    lib = _cabi.lib()
    res = {}

    def post(mode):
        p = _cabi.Postprocess()
        for i, f in enumerate(("radius", "confidence", "intr4", "out_confidence", "out_radius", "out_depth", "out_points",
                               "out_rays")):
            setattr(p, f, BASE + i * (1 << 22))
        p.B, p.net_h, p.net_w, p.padded_h, p.padded_w, p.H, p.W = 1, 28, 42, 24, 32, 24, 32
        p.mode = mode
        n0 = lib.udb_launch_count()
        rc = lib.udb_postprocess(C.byref(p), None)
        return {"rc": rc, "msg": lib.udb_last_error().decode(), "launched": lib.udb_launch_count() - n0}

    for mode in (2, -1, 0, 1):
        res[f"post{mode}"] = post(mode)

    cfg = _cabi.Config()
    cfg.embed_dim, cfg.depth, cfg.enc_heads, cfg.pos_grid = 384, 12, 6, 37
    for i, t in enumerate((3, 6, 9, 12)):
        cfg.taps[i] = t
    cfg.hidden, cfg.dec_heads, cfg.expansion, cfg.out_dim, cfg.n_stages = 256, 8, 4, 32, 3
    for i in range(3):
        cfg.dec_depths[i] = 2
    cfg.ratio_min, cfg.ratio_max, cfg.pixels_min, cfg.pixels_max = 0.5, 2.5, 200000.0, 600000.0
    h = C.c_void_p()
    assert lib.udb_create(C.byref(cfg), C.byref(h)) == 0
    for mode in (2, 1):
        a = _cabi.InferArgs()
        a.rgb, a.workspace, a.workspace_bytes = BASE, BASE + (1 << 24), 1 << 20
        a.B, a.H, a.W, a.resolution_level, a.interpolation = 1, 120, 160, -1, mode
        for i, f in enumerate(("confidence", "intrinsics", "radius", "depth", "points", "rays", "depth_features")):
            setattr(a, f, BASE + (1 << 25) + i * (1 << 22))
        n0 = lib.udb_launch_count()
        rc = lib.udb_infer_v2(h, C.byref(a), None)
        res[f"infer{mode}"] = {"rc": rc, "msg": lib.udb_last_error().decode(), "launched": lib.udb_launch_count() - n0}
    lib.udb_destroy(h)
    json.dump(res, sys.stdout)


def test_unknown_mode_is_rejected_before_any_launch():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    code = "import sys; sys.path[:0] = ['tests', 'oracle']; import test_bicubic_cpu as t; t._child_main()"
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, check=True).stdout
    r = json.loads(out)
    print(r)
    for case, field in (("post2", "`mode`"), ("post-1", "`mode`"), ("infer2", "`interpolation`")):
        assert r[case]["rc"] != 0 and field in r[case]["msg"] and r[case]["launched"] == 0, (case, r[case])
        assert "CUDA" not in r[case]["msg"] and "device" not in r[case]["msg"], (case, r[case])
    # the two valid modes get past the check and fail only at the launch, which has no device to run on
    for case in ("post0", "post1"):
        assert r[case]["rc"] != 0 and "mode" not in r[case]["msg"] and r[case]["launched"] == 0, (case, r[case])
    assert r["infer1"]["rc"] != 0 and "not prepared" in r["infer1"]["msg"] and r["infer1"]["launched"] == 0


def test_infer_rejects_other_modes_before_any_launch():
    """Every mode but the two the reference's F.interpolate(align_corners=False) accepts raises NotImplementedError before
    the input is even moved to a device (so also on a CPU model, ahead of its "no CPU path" error)."""
    from unidepth_b200 import UniDepthV2, _cabi
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "config_v2_vits14.json")))
    m = UniDepthV2(cfg)
    n0 = _cabi.launch_count()
    for mode in ("nearest", "area", "nearest-exact", "linear", "trilinear", "Bicubic"):
        m.interpolation_mode = mode
        with pytest.raises(NotImplementedError, match="'bilinear' and 'bicubic'"):
            m.infer(torch.zeros(3, 64, 64, dtype=torch.uint8))
    assert _cabi.launch_count() == n0
    for mode in ("bilinear", "bicubic"):           # accepted: the CPU model then fails for want of a device
        m.interpolation_mode = mode
        with pytest.raises(RuntimeError, match="no CPU"):
            m.infer(torch.zeros(3, 64, 64, dtype=torch.uint8))
