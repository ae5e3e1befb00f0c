"""precision = "fp8" without a GPU: the e4m3 weight packer, the contract between the packer and the engine's schedule (dry
run), and a CPU model of the mode's rounding -- the fp32 oracle with the operands of the encoder blocks' four linear layers
rounded through float8_e4m3fn with the same row / column scales the kernels use.  The model predicts the error the GPU
mode shows against the reference goldens (tests/test_fp8_gpu.py compares the two)."""
import contextlib
import copy
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from fixture import make_state_dict  # noqa: E402
from unidepth_b200 import UniDepthV2, _cabi  # noqa: E402
from unidepth_b200._pack import pack_e4m3  # noqa: E402

CPU = torch.device("cpu")
E4M3 = torch.float8_e4m3fn
BLOCK_FP8 = ("qkv_w8", "qkv_w8s", "proj_w8", "proj_w8s", "fc1_w8", "fc1_w8s", "fc2_w8", "fc2_w8s")
BLOCK_COMMON = ("n1w", "n1b", "qkv_b", "proj_b", "ls1", "n2w", "n2b", "fc1_b", "fc2_b", "ls2")


# ----------------------------------------------------------------------------------------------- the rounding model
def quantize_rows(x: torch.Tensor):
    """Per-row e4m3 quantisation as the kernels do it (include/udb.h udb_quantize_rows_e4m3): (q, s), x ~= q * s."""
    x = x.float()
    amax = x.abs().amax(dim=-1, keepdim=True)
    nz = amax > 0
    one = torch.ones_like(amax)
    inv = torch.where(nz, torch.full_like(amax, 448.0) / torch.where(nz, amax, one), one)   # correctly rounded
    return (x * inv).to(E4M3), torch.where(nz, amax / 448.0, one)


_ENC_LINEARS = ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2")


@contextlib.contextmanager
def fp8_encoder(oracle):
    """Inside the block: the oracle's encoder blocks multiply e4m3-rounded operands (activations per row, weights per
    output channel, products and sums in f32), everything else stays fp32."""
    lin = oracle._lin

    def lin8(x, sd, prefix, bias=True):
        if not (prefix.startswith("pixel_encoder.blocks.") and prefix.endswith(_ENC_LINEARS)):
            return lin(x, sd, prefix, bias)
        q, s = quantize_rows(x)
        w8, ws = pack_e4m3(sd[prefix + ".weight"])
        y = F.linear(q.float() * s, w8.float() * ws[:, None])
        return y + sd[prefix + ".bias"] if bias else y

    oracle._lin = lin8
    try:
        yield
    finally:
        oracle._lin = lin


def depth_errors(out, ref):
    """(depth ARel, depth max rel, intrinsics max rel) as tests/test_infer_parity_gpu.py measures them."""
    d, dr = out["depth"].float().cpu(), ref["depth"]
    rel = (d - dr).abs() / dr
    k, kr = out["intrinsics"].cpu(), ref["intrinsics"]
    kerr = max(((k[:, i, j] - kr[:, i, j]).abs() / kr[:, i, j].abs()).max().item() for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)))
    return rel.mean().item(), rel.max().item(), kerr


def golden_case(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    meta = json.loads(str(z["__meta__"]))
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", meta["config"])))
    g = torch.Generator().manual_seed(1234 + meta["seed"])
    b, h, w = meta["shape"]
    rgb = torch.randint(0, 256, (b, 3, h, w), dtype=torch.uint8, generator=g)
    ref = {k: torch.from_numpy(z[k]) for k in z.files if k != "__meta__"}
    return cfg, make_state_dict(cfg, meta["seed"]), rgb, ref, meta


def fp8_model_infer(cfg, sd, rgb, meta):
    import unidepth_oracle as O
    with fp8_encoder(O):
        return O.infer_v2(sd, copy.deepcopy(cfg), rgb, resolution_level=meta["resolution_level"])


# ----------------------------------------------------------------------------------------------- tests
def test_pack_e4m3_values():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(96, 200, generator=g) * torch.logspace(-3, 1, 96)[:, None]
    w[7] = 0.0
    w8, s = pack_e4m3(w)
    assert w8.dtype == E4M3 and w8.shape == (96, 200) and s.dtype == torch.float32 and s.shape == (96,)
    amax = w.abs().amax(dim=1)
    nz = amax > 0
    assert torch.equal(s[nz], amax[nz] / 448.0) and s[7] == 1.0 and not w8[7].float().any()
    # every row's largest magnitude maps to +-448, and the rounding is e4m3's: relative 2^-4 for normal values,
    # absolute 2^-10 * s below the smallest normal (2^-6)
    assert torch.equal(w8.float().abs().amax(dim=1)[nz], torch.full((95,), 448.0))
    err = (w8.float() * s[:, None] - w).abs()
    assert (err <= torch.maximum(w.abs() * 2.0 ** -4, s[:, None] * 2.0 ** -10) * 1.0001).all()
    # the same values torch's own round-to-nearest-even cast gives
    inv = (torch.full_like(amax, 448.0) / amax).nan_to_num(1.0, 1.0, 1.0)
    assert torch.equal(w8.view(torch.uint8), (w * inv[:, None]).to(E4M3).view(torch.uint8))


def _v2(cfg_name, depth=None, **attrs):
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", cfg_name)))
    if depth is not None:
        cfg["model"]["pixel_encoder"]["arch_override"] = {"depth": depth}
        cfg["model"]["pixel_encoder"]["output_idx"] = [1, 2, 3, 4]
    m = UniDepthV2(copy.deepcopy(cfg))
    m.load_state_dict(make_state_dict(cfg, 0), strict=True)
    for k, v in attrs.items():
        setattr(m, k, v)
    return m.eval()


def _engine(m, tensors, scalars):
    h = C.c_void_p()
    _cabi.check(_cabi.lib().udb_create(C.byref(m._engine_config()), C.byref(h)), "udb_create")
    m._register(h, tensors, scalars)
    return h


def test_packer_gives_the_fp8_operand_set():
    m = _v2("config_v2_vits14.json", precision="fp8")
    T, S = m._pack_tensors(CPU)
    assert S["precision"] == 2.0 and S["fuse_ln"] == 0.0
    d = m.spec.embed_dim
    for i in range(m.spec.depth):
        blk = {k.split(".", 2)[2] for k in T if k.startswith(f"blocks.{i}.")}
        assert blk == set(BLOCK_FP8 + BLOCK_COMMON), blk
    shapes = {"qkv": (3 * d, d), "proj": (d, d), "fc1": (4 * d, d), "fc2": (d, 4 * d)}
    sd = m.state_dict()
    src = {"qkv": "attn.qkv", "proj": "attn.proj", "fc1": "mlp.fc1", "fc2": "mlp.fc2"}
    for k, shp in shapes.items():
        w8, s = T[f"blocks.0.{k}_w8"], T[f"blocks.0.{k}_w8s"]
        assert w8.dtype == E4M3 and tuple(w8.shape) == shp and s.shape == (shp[0],)
        ref8, refs = pack_e4m3(sd[f"pixel_encoder.blocks.0.{src[k]}.weight"])
        assert torch.equal(w8.view(torch.uint8), ref8.view(torch.uint8)) and torch.equal(s, refs)
    # the patch embedding and the decoder keep their f16 packing
    T16, _ = _v2("config_v2_vits14.json")._pack_tensors(CPU)
    for k in T16:
        if not k.startswith("blocks."):
            assert torch.equal(T[k], T16[k]), k
    # fuse_ln is ignored in fp8 mode, as in split mode
    m.fuse_ln = True
    assert m._pack_tensors(CPU)[1]["fuse_ln"] == 0.0
    m.precision = "fp16"
    with pytest.raises(ValueError, match="'f16', 'split' or 'fp8'"):
        m._pack_tensors(CPU)


@pytest.mark.parametrize("cfg_name,depth", [("config_v2_vits14.json", None), ("config_v2_vitb14.json", None),
                                            ("config_v2_vitl14.json", 4)])
def test_schedule_accepts_exactly_the_fp8_operands(cfg_name, depth):
    lib = _cabi.lib()
    m = _v2(cfg_name, depth, precision="fp8")
    T, S = m._pack_tensors(CPU)
    h = _engine(m, T, S)
    try:
        for (B, H, W, lvl) in ((1, 480, 640, -1), (2, 96, 288, 3), (1, 490, 644, -2)):
            assert lib.udb_schedule_bytes(h, B, H, W, lvl) > 0, lib.udb_last_error().decode()
    finally:
        lib.udb_destroy(h)
    # each fp8 operand of a block, and the vectors it shares with the f16 mode, is named when it is missing
    last = m.spec.depth - 1
    for name in [f"blocks.0.{k}" for k in BLOCK_FP8 + BLOCK_COMMON] + [f"blocks.{last}.fc2_w8s"]:
        h = _engine(m, {k: v for k, v in T.items() if k != name}, S)
        try:
            assert lib.udb_schedule_bytes(h, 1, 240, 320, -1) == 0
            assert name in lib.udb_last_error().decode(), (name, lib.udb_last_error().decode())
        finally:
            lib.udb_destroy(h)
    # a weight of the wrong dtype or shape is refused, not read as e4m3 bytes
    for name, fn, what in (("blocks.0.fc1_w8", lambda t: t.float().half(), "dtype"),
                           ("blocks.0.fc2_w8", lambda t: t.t().contiguous(), "expected")):
        bad = dict(T)
        bad[name] = fn(T[name])
        h = _engine(m, bad, S)
        try:
            assert lib.udb_schedule_bytes(h, 1, 240, 320, -1) == 0
            msg = lib.udb_last_error().decode()
            assert name in msg and what in msg, msg
        finally:
            lib.udb_destroy(h)
    # an f16 packing is not accepted as fp8 mode (precision 2 with f16 operands names the first missing e4m3 weight)
    T16, S16 = _v2(cfg_name, depth)._pack_tensors(CPU)
    h = _engine(m, T16, dict(S16, precision=2.0))
    try:
        assert lib.udb_schedule_bytes(h, 1, 240, 320, -1) == 0
        assert "blocks.0.qkv_w8" in lib.udb_last_error().decode()
    finally:
        lib.udb_destroy(h)


def test_quantize_rows_model():
    x = torch.randn(5, 384, dtype=torch.float64).float() * 3
    x[2] = 0.0
    q, s = quantize_rows(x)
    assert q.dtype == E4M3 and s.shape == (5, 1) and s[2, 0] == 1.0 and not q[2].float().any()
    assert torch.equal(q.float().abs().amax(dim=1)[[0, 1, 3, 4]], torch.full((4,), 448.0))
    assert ((q.float() * s - x).abs() <= x.abs() * 2.0 ** -4 + s * 2.0 ** -10).all()


# The rounding model's error against the unmodified reference's outputs (fp32 oracle arithmetic with e4m3 operands in
# the encoder's linear layers), recorded on this CPU model: (depth ARel, depth max rel, intrinsics max rel).  The same
# numbers for the fp32 oracle itself are <= 2e-6 (tests/test_oracle_golden.py), so this is the fp8 rounding alone.  The
# seeded fixture amplifies operand rounding (~50x a default-initialised network, SURVEY.md section 7), which is why the
# intrinsics error is percent-level here; what it is on trained checkpoints is not measured.
FP8_MODEL_ERROR = {
    "vits_120x160": (4.610e-03, 2.120e-02, 2.941e-02),
    "vitb_112x160": (3.292e-03, 2.198e-02, 1.401e-02),
}


@pytest.mark.parametrize("name", sorted(FP8_MODEL_ERROR))
def test_fp8_rounding_model_error_against_golden(name):
    cfg, sd, rgb, ref, meta = golden_case(name)
    from test_oracle_golden import subsample_like_golden
    out = subsample_like_golden(dict(fp8_model_infer(cfg, sd, rgb, meta)), meta)
    arel, dmax, kerr = depth_errors(out, ref)
    print(f"FP8MODEL {name}: depth ARel {arel:.3e} max {dmax:.3e}; intrinsics rel {kerr:.3e}")
    exp = FP8_MODEL_ERROR[name]
    # a model of the rounding, not of the kernels: deterministic on the CPU up to thread-count reordering
    for got, want in zip((arel, dmax, kerr), exp):
        assert 0.5 * want < got < 1.5 * want, (name, (arel, dmax, kerr), exp)
