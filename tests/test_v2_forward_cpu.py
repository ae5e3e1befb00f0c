"""UniDepthV2's evaluation forward, model(inputs, image_metas) = forward_test, without a GPU: where the paddings come from
(the metas, reordered, before inputs["paddings"]), the argument checks that run before anything touches the device, the
engine's named refusals of the match fields (before any launch), the C layout of the structs, the dry-run workspace with
matching, and the goldens of the unmodified reference (tests/golden/v2fwd_*.npz, oracle/make_golden_v2_forward.py)
against this repository's fp32 oracle."""
import copy
import ctypes as C
import glob
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from fixture import make_state_dict  # noqa: E402
from unidepth_b200 import UniDepthV2, _cabi  # noqa: E402

CPU = torch.device("cpu")
FWD_GOLDENS = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, "v2fwd_*.npz")))


def _model(bb="vits14", seed=0):
    cfg = json.load(open(os.path.join(GOLDEN, f"config_v2_{bb}.json")))
    m = UniDepthV2(copy.deepcopy(cfg))
    m.load_state_dict(make_state_dict(cfg, seed), strict=True)
    return m.eval()


def _inputs(B=2, h=294, w=392, H=480, W=640, **kw):
    return dict({"image": torch.zeros(B, 3, h, w), "depth": torch.zeros(B, 1, H, W)}, **kw)


def test_paddings_come_from_the_metas_reordered_then_from_inputs():
    mp = UniDepthV2._match_paddings
    metas = [{"paddings": (1, 2, 3, 4), "depth_paddings": (0, 0, 0, 0)}, {"paddings": [5, 6, 7, 8]}]
    # the metas hold (l, t, r, b); the result is (l, r, t, b), as encode_decode's [..., [0, 2, 1, 3]]
    want = torch.tensor([[1, 3, 2, 4], [5, 7, 6, 8]], dtype=torch.int32)
    assert torch.equal(mp(_inputs(), metas, 2, 294, 392), want)
    # the metas override inputs["paddings"]
    assert torch.equal(mp(_inputs(paddings=[(0, 0, 0, 0)] * 2), metas, 2, 294, 392), want)
    # without metas paddings: inputs["paddings"], a list of (l, r, t, b) or a [B, 4] tensor
    ins = _inputs(paddings=[(1, 2, 3, 4), (0, 0, 14, 0)])
    for metas in (None, [], [{"flip": False}, {"flip": True}]):
        assert mp(ins, metas, 2, 294, 392).tolist() == [[1, 2, 3, 4], [0, 0, 14, 0]]
    assert mp(_inputs(paddings=torch.tensor([[1, 2, 3, 4]] * 2)), None, 2, 294, 392).tolist() == [[1, 2, 3, 4]] * 2
    # neither: zeros (the reference raises KeyError here)
    out = mp(_inputs(), None, 2, 294, 392)
    assert out.dtype == torch.int32 and out.tolist() == [[0] * 4] * 2
    # a crop of one row and one column is allowed
    assert mp(_inputs(paddings=[(391, 0, 0, 293)] * 2), None, 2, 294, 392).tolist() == [[391, 0, 0, 293]] * 2


def test_forward_argument_errors_before_the_device():
    m = _model()
    bad = [
        (_inputs(paddings=[(0, 0, 0, 0)]), None, "one \\(l, r, t, b\\) per image"),
        (_inputs(paddings=torch.zeros(2, 3)), None, "one \\(l, r, t, b\\) per image"),
        (_inputs(), [{"paddings": (0, 0, 0, 0)}], "one \\(l, r, t, b\\) per image"),
        (_inputs(), [{"paddings": (0, 0, 0)}, {"paddings": (0, 0, 0)}], "4 values"),
        (_inputs(paddings=[(0, -1, 0, 0), (0, 0, 0, 0)]), None, ">= 0"),
        (_inputs(), [{"paddings": (0, 0, 0, 0)}, {"paddings": (0, -2, 0, 0)}], ">= 0"),
        (_inputs(paddings=[(0, 0, 147, 147), (0, 0, 0, 0)]), None, "no row or column"),
        (_inputs(paddings=[(0, 0, 0, 0), (200, 192, 0, 0)]), None, "no row or column"),
        (_inputs(paddings=[(0.5, 0, 0, 0), (0, 0, 0, 0)]), None, "whole pixels"),
        (_inputs(depth=torch.zeros(2, 480, 640)), None, "\\[B, 1, H, W\\]"),
        (_inputs(h=300), None, "multiple of 14"),
        ({"image": torch.zeros(2, 294, 392), "depth": torch.zeros(2, 1, 4, 4)}, None, "\\[B, 3, h, w\\]"),
    ]
    for inputs, metas, msg in bad:
        before = {k: (v.clone() if isinstance(v, torch.Tensor) else copy.deepcopy(v)) for k, v in inputs.items()}
        with pytest.raises(ValueError, match=msg):
            m(inputs, metas)
        assert set(inputs) == set(before)      # the caller's dict is left as it was
    # valid arguments reach the device check: this model is on the CPU
    with pytest.raises(RuntimeError, match="CUDA"):
        m(_inputs(paddings=[(0, 0, 0, 0), (14, 0, 0, 28)]), [])
    m.train()
    with pytest.raises(NotImplementedError):
        m(_inputs(), [])


def _args(**kw):
    """udb_infer_v2_match arguments whose pointers are never dereferenced: every call below is refused before any
    launch."""
    ma = _cabi.InferMatchArgs()
    a = ma.args
    a.rgb, a.workspace, a.workspace_bytes = 16, 16, 1 << 20
    for k in ("confidence", "intrinsics", "radius", "depth", "points", "rays", "depth_features"):
        setattr(a, k, 16)
    a.B, a.H, a.W, a.resolution_level = 1, 294, 392, -2
    for k, v in kw.items():
        setattr(ma if k.startswith("match_") else a, k, v)
    return ma


def test_engine_refuses_bad_match_fields_and_sizes_no_scratch_for_them():
    lib = _cabi.lib()
    m = _model()
    T, S = m._pack_tensors(CPU)
    h = C.c_void_p()
    _cabi.check(lib.udb_create(C.byref(m._engine_config()), C.byref(h)), "udb_create")
    try:
        m._register(h, T, S)
        cases = [
            (_args(resolution_level=-1, match_h=480, match_w=640, match_pads=16), b"UDB_LEVEL_NETWORK_ONLY (-2) only, not -1"),
            (_args(resolution_level=3, match_pads=16), b"only, not 3"),
            (_args(match_h=480, match_w=640), b"match_pads NULL"),
            (_args(match_pads=16), b"match_h 0, match_w 0"),
            (_args(match_h=480, match_pads=16), b"match_w 0"),
            (_args(match_h=-1, match_w=640, match_pads=16), b"match_h -1"),
            (_args(match_h=480, match_w=640, match_pads=16, depth=None), b"all output pointers but radius"),
            (_args(radius=None), b"all seven output pointers"),
        ]
        for a, msg in cases:
            assert lib.udb_infer_v2_match(h, C.byref(a), None) != 0
            assert msg in lib.udb_last_error(), (msg, lib.udb_last_error())
        assert lib.udb_infer_v2_match(h, None, None) != 0 and b"null argument" in lib.udb_last_error()
        # a valid matching call, radius NULL, gets past these checks and stops at the workspace no dry run has prepared;
        # all-zero match fields are udb_infer_v2's call, which needs radius
        for a in (_args(match_h=480, match_w=640, match_pads=16, radius=None), _args()):
            assert lib.udb_infer_v2_match(h, C.byref(a), None) != 0
            assert b"udb_workspace_bytes" in lib.udb_last_error(), lib.udb_last_error()
        # the match assembly writes straight into the outputs: the network-only workspace is what it was before matching
        # existed (the dry run's bytes for these shapes at the parent commit)
        for (B, hh, ww), n in (((1, 294, 392), 52948736), ((2, 294, 392), 105896192), ((8, 490, 644), 1154584064)):
            assert lib.udb_schedule_bytes(h, B, hh, ww, -2) == n, (B, hh, ww)
    finally:
        lib.udb_destroy(h)


def test_extended_structs_match_c_layout():
    structs = {"udb_infer_match_args_t": (_cabi.InferMatchArgs, "match_pads"), "udb_match_gt_t": (_cabi.MatchGt, "out_rays")}
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "udb.h"\nint main(){\n'
    for n, (cs, _) in structs.items():
        for f, _t in cs._fields_:
            src += f'printf("{n} {f} %zu %zu\\n", sizeof({n}), offsetof({n}, {f}));\n'
    src += "return 0;}\n"
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        out = subprocess.check_output([os.path.join(d, "t")], text=True)
    for line in out.strip().splitlines():
        n, f, size, off = line.split()
        cs, last = structs[n]
        assert cs._fields_[-1][0] == last
        assert C.sizeof(cs) == int(size), (n, C.sizeof(cs), size)
        assert getattr(cs, f).offset == int(off), (n, f)


def test_forward_goldens_are_present():
    assert len(FWD_GOLDENS) == 6, FWD_GOLDENS
    for name in FWD_GOLDENS:
        assert 50e3 < os.path.getsize(os.path.join(GOLDEN, name + ".npz")) < 500e3, name


# ------------------------------------------------------------------------------------------ goldens
def golden_case(name):
    """(golden arrays, meta, model-free inputs): the network input rebuilt from the seed, the ground truth placeholder,
    the metas as the data pipeline writes them, and this repository's camera object of the case."""
    from make_golden import seeded_rgb
    from unidepth_b200 import camera as cams
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["__meta__"]))
    rgb = seeded_rgb(tuple(meta["shape"]), meta["seed"])
    mean = torch.tensor((0.485, 0.456, 0.406)).view(1, 3, 1, 1)
    std = torch.tensor((0.229, 0.224, 0.225)).view(1, 3, 1, 1)
    x = rgb.to(torch.float32).div(255).sub(mean).div(std)
    s = meta["image_stride"]
    assert np.array_equal(x[:, :, ::s, ::s].numpy(), z["image_sample"]), "the network input differs from the generator's"
    inputs = {"image": x, "depth": torch.zeros(meta["shape"][0], 1, *meta["gt_hw"])}
    metas = [{"paddings": p, "depth_paddings": [0, 0, 0, 0]} for p in meta["metas_paddings"]] if meta["metas_paddings"] else []
    if meta["camera"]:
        kind, params = meta["camera"]["kind"], meta["camera"]["params"]
        if kind == "Pinhole":
            fx, fy, cx, cy = params
            inputs["camera"] = cams.Pinhole(K=torch.tensor([[[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]]]))
        else:
            inputs["camera"] = getattr(cams, kind)(params=torch.tensor([params], dtype=torch.float32))
    return z, meta, inputs, metas


def oracle_forward_test(name):
    """This repository's fp32 oracle (oracle/unidepth_oracle.py: encoder + decoder at the network size) followed by the
    reference's matching restated in torch: crop (l, r, t, b), bilinear resize to the ground truth, K scaled per axis."""
    import unidepth_oracle as O
    z, meta, inputs, metas = golden_case(name)
    cfg = json.load(open(os.path.join(GOLDEN, meta["config"])))
    sd = make_state_dict(cfg, meta["seed"])
    x = inputs["image"]
    B, _, h, w = x.shape
    H, W = meta["gt_hw"]
    feats, clss = O.vit_encoder(sd, O.ModelSpec(cfg), x)
    rays_gt = None
    if "camera" in inputs:
        rays_gt = inputs["camera"].get_rays(shapes=(B, h, w)).expand(B, 3, h, w).flatten(2).transpose(1, 2)
    dec = O.decoder(sd, O.ModelSpec(cfg), feats, clss, (h, w), rays_gt=rays_gt)
    rays = dec["rays"].transpose(1, 2).reshape(B, 3, h, w)
    pts = rays * dec["radius"]
    pads = UniDepthV2._match_paddings(inputs, metas, B, h, w).tolist()
    out = {"points": [], "confidence": []}
    K = dec["intrinsics"].clone()
    for b, (l, r, t, bo) in enumerate(pads):
        for k, v in (("points", pts), ("confidence", dec["confidence"])):
            out[k].append(F.interpolate(v[b:b + 1, :, t:h - bo, l:w - r], size=(H, W), mode="bilinear"))
        sx, sy = W / (w - l - r), H / (h - t - bo)
        K[b, 0, 0] *= sx
        K[b, 1, 1] *= sy
        K[b, 0, 2] = (dec["intrinsics"][b, 0, 2] - l) * sx
        K[b, 1, 2] = (dec["intrinsics"][b, 1, 2] - t) * sy
    out = {k: torch.cat(v) for k, v in out.items()}
    out["depth"] = out["points"][:, 2:]
    out["intrinsics"] = K
    out["rays"] = rays / torch.norm(rays, dim=1, keepdim=True).clip(min=1e-5)
    return z, meta, out


@pytest.mark.parametrize("name", [n for n in FWD_GOLDENS if "vits14" in n])
def test_oracle_matches_reference_forward_golden(name):
    torch.set_num_threads(min(32, os.cpu_count()))
    z, meta, out = oracle_forward_test(name)
    st = meta["strides"]
    for k in ("depth", "confidence", "points", "rays"):
        got, ref = out[k][:, :, ::st[k], ::st[k]], torch.from_numpy(z[k])
        assert got.shape == ref.shape, (k, got.shape, ref.shape)
        # floored at 10 % of the mean magnitude, as tests/test_oracle_golden.py, for the signed maps
        err = ((got - ref).abs() / ref.abs().clamp(min=0.1 * ref.abs().mean().item())).max().item()
        assert err < 3e-4, (k, err)
    kk, kr = out["intrinsics"], torch.from_numpy(z["intrinsics"])
    for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)):
        assert ((kk[:, i, j] - kr[:, i, j]).abs() / kr[:, i, j].abs()).max().item() < 1e-5


@pytest.mark.skipif(not os.path.isdir("/root/reference/unidepth"), reason="needs the reference sources")
@pytest.mark.parametrize("name", FWD_GOLDENS)
def test_generator_reproduces_forward_golden(name):
    """The generator's recipe (the unmodified reference's eval-mode forward) reproduces every stored golden to 1e-5."""
    import warnings
    warnings.simplefilter("ignore")
    sys.path[:0] = ["/root/reference", os.path.join(ROOT, "oracle", "ref_shims")]
    from make_golden_v2_forward import CASES, reference_forward
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["__meta__"]))
    _, _, out = reference_forward(next(c for c in CASES if c[0] == name))
    for k, s in meta["strides"].items():
        np.testing.assert_allclose(out[k][:, :, ::s, ::s].numpy(), z[k], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(out["intrinsics"].numpy(), z["intrinsics"], rtol=1e-5)
