"""UniDepthV1 precision = "fp8" without a GPU: the packer (ConvNeXt and DINOv2 ViT-L encoders), the contract between the
packer and the V1 engine's schedule (dry run: udb_v1_workspace_bytes), and a CPU model of the mode's rounding -- the fp32
V1 oracles with the operands of the encoder blocks' MLP (ConvNeXt) or four linear layers (ViT-L) rounded through
float8_e4m3fn with the same row / column scales the kernels use.  tests/test_v1_fp8_gpu.py compares the GPU mode with it."""
import contextlib
import copy
import ctypes as C
import json
import os

import pytest
import torch
import torch.nn.functional as F

from test_fp8_cpu import fp8_encoder
from unidepth_b200 import UniDepthV1, _cabi
from unidepth_b200.unidepthv1 import FP8_STAGES
from unidepth_b200._pack import pack_e4m3

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
CPU = torch.device("cpu")
E4M3 = torch.float8_e4m3fn
SMALL = {"depths": [1, 1, 2, 1], "dims": [64, 128, 192, 256]}
CNX_FP8 = ("w1_8", "w1_8s", "w2_8", "w2_8s")
VIT_FP8 = ("qkv_w8", "qkv_w8s", "proj_w8", "proj_w8s", "fc1_w8", "fc1_w8s", "fc2_w8", "fc2_w8s")


def _model(cfg_name, arch=None, seed=0, precision="f16"):
    cfg = json.load(open(os.path.join(GOLD, cfg_name)))
    if arch is not None:
        cfg["model"]["pixel_encoder"]["arch"] = arch
    m = UniDepthV1(copy.deepcopy(cfg)).eval()
    if seed is not None:
        if cfg_name == "config_v1_vitl14.json":
            from unidepth_v1_vit_oracle import make_v1_vit_state_dict as make
        else:
            from fixture import make_v1_state_dict as make
        m.load_state_dict(make(cfg, seed), strict=True)
    m.precision = precision
    return m


def _engine(m, T, S):
    h = C.c_void_p()
    _cabi.check(_cabi.lib().udb_v1_create(C.byref(m._engine_config()), C.byref(h)), "udb_v1_create")
    m._register(h, T, S)
    return h


def _bytes(m, T, S, B=1, H=480, W=640):
    """(workspace bytes, error text) of a dry run of the schedule with these operands."""
    lib = _cabi.lib()
    h = _engine(m, T, S)
    try:
        n = lib.udb_v1_workspace_bytes(h, B, H, W)
        return n, lib.udb_last_error().decode()
    finally:
        lib.udb_v1_destroy(h)


# ----------------------------------------------------------------------------------------------- packer
@pytest.mark.parametrize("arch", [SMALL, None], ids=["small", "convnext_l"])
def test_convnext_fp8_packer(arch):
    m = _model("config_v1_cnvnxtl.json", arch, seed=0 if arch else None)
    T16, S16 = m._pack_tensors(CPU)
    m.precision = "fp8"
    T, S = m._pack_tensors(CPU)
    assert S == dict(S16, precision=2.0) and "precision" not in S16
    sd = m.state_dict()
    expected = set(T16)
    for i, depth in enumerate(m.spec.depths):
        for j in range(depth):
            if FP8_STAGES[i]:
                expected -= {f"s{i}.b{j}.w1", f"s{i}.b{j}.w2"}
                expected |= {f"s{i}.b{j}.{k}" for k in CNX_FP8}
    assert set(T) == expected
    for i, depth in enumerate(m.spec.depths):
        C_ = m.spec.dims[i]
        for j in range(depth):
            if not FP8_STAGES[i]:
                continue
            p, src = f"s{i}.b{j}.", f"pixel_encoder.stages.{i}.blocks.{j}.mlp."
            for k, fc, shp in (("w1", "fc1", (4 * C_, C_)), ("w2", "fc2", (C_, 4 * C_))):
                w8, s = T[p + k + "_8"], T[p + k + "_8s"]
                ref8, refs = pack_e4m3(sd[src + fc + ".weight"])
                assert w8.dtype == E4M3 and tuple(w8.shape) == shp and s.dtype == torch.float32 and s.shape == (shp[0],)
                assert torch.equal(w8.view(torch.uint8), ref8.view(torch.uint8)) and torch.equal(s, refs)
    # every other operand -- stem, downsample layers, the blocks' other vectors, the decoder -- is the f16 packing's
    for k in T16:
        if k in T:
            assert T[k].dtype == T16[k].dtype and torch.equal(T[k], T16[k]), k
    m.precision = "fp16"
    with pytest.raises(ValueError, match="'f16' or 'fp8'"):
        m._pack_tensors(CPU)


def test_vit_fp8_packer():
    m = _model("config_v1_vitl14.json", seed=None)
    T16, S16 = m._pack_tensors(CPU)
    m.precision = "fp8"
    T, S = m._pack_tensors(CPU)
    assert S == dict(S16, precision=2.0)
    sd = m.state_dict()
    d = m.spec.embed_dim
    src = {"qkv": "attn.qkv", "proj": "attn.proj", "fc1": "mlp.fc1", "fc2": "mlp.fc2"}
    for i in range(m.spec.enc_depth):
        b = f"blocks.{i}."
        assert {k for k in T if k.startswith(b)} == ({k for k in T16 if k.startswith(b) and not k.endswith("_w")}
                                                     | {b + k for k in VIT_FP8})
    for k, shp in (("qkv", (3 * d, d)), ("proj", (d, d)), ("fc1", (4 * d, d)), ("fc2", (d, 4 * d))):
        for i in (0, m.spec.enc_depth - 1):
            ref8, refs = pack_e4m3(sd[f"pixel_encoder.blocks.{i}.{src[k]}.weight"])
            w8 = T[f"blocks.{i}.{k}_w8"]
            assert tuple(w8.shape) == shp and torch.equal(w8.view(torch.uint8), ref8.view(torch.uint8))
            assert torch.equal(T[f"blocks.{i}.{k}_w8s"], refs)
    for k in T16:
        if not k.startswith("blocks."):
            assert torch.equal(T[k], T16[k]), k


def test_precision_change_repacks():
    m = _model("config_v1_cnvnxtl.json", SMALL)
    key = m._fingerprint()
    m.precision = "fp8"
    assert m._fingerprint() != key and m._fingerprint()[0] == "fp8"


# ----------------------------------------------------------------------------------------------- dry run
SHAPES = ((480, 640), (375, 1242), (1000, 400))


@pytest.mark.parametrize("cfg_name,arch", [("config_v1_cnvnxtl.json", SMALL), ("config_v1_cnvnxtl.json", None),
                                           ("config_v1_vitl14.json", None)], ids=["small", "convnext_l", "vitl14"])
def test_schedule_accepts_exactly_the_fp8_operands(cfg_name, arch):
    vit = cfg_name == "config_v1_vitl14.json"
    m = _model(cfg_name, arch, seed=None)
    T16, S16 = m._pack_tensors(CPU)
    m.precision = "fp8"
    T, S = m._pack_tensors(CPU)
    for B in (1, 4):
        for H, W in SHAPES:
            n, msg = _bytes(m, T, S, B, H, W)
            assert n > 0, msg
            if not vit:
                # the e4m3 operands take the place of the f16 block's scratch: never a larger workspace
                n16, msg16 = _bytes(m, T16, S16, B, H, W)
                assert 0 < n <= n16, (n, n16, msg16)
    # a missing fp8 operand is named: first block, last block, the scales
    if vit:
        last = m.spec.enc_depth - 1
        names = ["blocks.0.qkv_w8", "blocks.0.fc2_w8", f"blocks.{last}.fc2_w8", "blocks.0.qkv_w8s", f"blocks.{last}.proj_w8s"]
        wrong = (("blocks.0.fc1_w8", "dtype"), ("blocks.0.fc2_w8", "expected"))
        first = "blocks.0.qkv_w8"
    else:
        # no ConvNeXt stage runs e4m3 (FP8_STAGES): the fp8 packing is the f16 one plus the precision scalar, and the
        # schedule takes either with precision 2 and sizes the same workspace
        assert not any(FP8_STAGES)
        assert set(T) == set(T16) and all(torch.equal(T[k], T16[k]) for k in T)
        for B in (1, 4):
            assert _bytes(m, T16, dict(S16, precision=2.0), B)[0] == _bytes(m, T16, S16, B)[0] > 0
        n, msg = _bytes(m, T16, dict(S16, precision=1.0))
        assert n == 0 and "precision" in msg, msg
        return
    for name in names:
        n, msg = _bytes(m, {k: v for k, v in T.items() if k != name}, S)
        assert n == 0 and name in msg, (name, msg)
    # a weight of the wrong dtype (f16 bytes) or a transposed one is refused, not read as e4m3 [N, K]
    for name, what in wrong:
        bad = dict(T)
        bad[name] = T[name].float().half() if what == "dtype" else T[name].t().contiguous()
        n, msg = _bytes(m, bad, S)
        assert n == 0 and name in msg and what in msg, msg
    # an f16 packing registered with precision 2 names the first e4m3 weight it lacks
    n, msg = _bytes(m, T16, dict(S16, precision=2.0))
    assert n == 0 and first in msg, msg
    # and a precision the V1 engine has no mode for is refused
    n, msg = _bytes(m, T16, dict(S16, precision=1.0))
    assert n == 0 and "precision" in msg, msg


# ----------------------------------------------------------------------------------------------- rounding model
def v1_errors(out, ref, meta):
    """(depth ARel, depth max rel, intrinsics max rel) against a golden case's stored (sub-sampled) outputs."""
    s = meta.get("strides", {}).get("depth", 1)
    d, dr = out["depth"].float().cpu()[:, :, ::s, ::s], ref["depth"]
    rel = (d - dr).abs() / dr
    k, kr = out["intrinsics"].float().cpu(), ref["intrinsics"]
    kerr = max(((k[:, i, j] - kr[:, i, j]).abs() / kr[:, i, j].abs()).max().item() for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)))
    return rel.mean().item(), rel.max().item(), kerr


def v1_case(name):
    """(config, state dict, rgb, K, meta, reference outputs) of a tests/golden/v1_*.npz case."""
    if name.startswith("v1_vitl14"):
        from test_v1_vit_cpu import v1_vit_case_inputs as inputs
    else:
        from test_oracle_golden import v1_case_inputs as inputs
    cfg, sd, rgb, K, meta, z = inputs(GOLD, name)
    ref = {k: torch.from_numpy(z[k]) for k in ("depth", "intrinsics")}
    return cfg, sd, rgb, K, meta, ref


def fp8_model_infer(name, cfg, sd, rgb, K, meta):
    """The CPU rounding model of precision "fp8" on one ViT-L case (ConvNeXt-L's fp8 mode has no e4m3 stage: FP8_STAGES)."""
    import unidepth_v1_vit_oracle as OV
    with fp8_encoder(OV):
        return OV.infer_v1_vit(sd, copy.deepcopy(cfg), rgb, K, skip_camera=meta["skip_camera"])


# The rounding model's error against the unmodified reference's outputs, recorded on this CPU model: (depth ARel, depth
# max rel, intrinsics max rel).  The fp32 oracles themselves are within 5e-5 of these goldens, so this is the e4m3
# rounding of the encoder's linear-layer operands alone, on seeded weights; on trained checkpoints it is not measured.
V1_FP8_MODEL_ERROR = {
    "v1_vitl14_480x640": (5.072e-03, 2.564e-02, 1.695e-02),
}


@pytest.mark.parametrize("name", sorted(V1_FP8_MODEL_ERROR))
def test_v1_fp8_rounding_model_error_against_golden(name):
    cfg, sd, rgb, K, meta, ref = v1_case(name)
    torch.set_num_threads(min(32, os.cpu_count()))
    out = fp8_model_infer(name, cfg, sd, rgb, K, meta)
    arel, dmax, kerr = v1_errors(out, ref, meta)
    print(f"V1FP8MODEL {name}: depth ARel {arel:.3e} max {dmax:.3e}; intrinsics rel {kerr:.3e}")
    exp = V1_FP8_MODEL_ERROR[name]
    for got, want in zip((arel, dmax, kerr), exp):
        assert 0.5 * want < got < 1.5 * want, (name, (arel, dmax, kerr), exp)
