"""UniDepthV2old precision = "split" and "fp8" without a GPU: the packer and the contract between the packer and the
V2old engine's schedule (dry run: udb_v2old_schedule_bytes), the `precision` attribute, and -- when the reference is at
hand -- a rounding model that runs the unmodified reference with operands rounded in chosen submodules, to locate where
V2old's depth error comes from.  tests/test_v2old_precision_gpu.py runs the modes on the GPU."""
import copy
import json
import os
import sys
import warnings

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from test_v2old_cpu import BACKBONES, GOLDEN, ROOT, _cfg, _engine
from make_golden_v2old import make_v2old_state_dict
from unidepth_b200 import UniDepthV2old, _cabi
from unidepth_b200._pack import pack_e4m3
from unidepth_b200.unidepthv2old import v2old_geometry

CPU = torch.device("cpu")
REFERENCE = "/root/reference"


def _model(bb):
    cfg = _cfg(bb)
    m = UniDepthV2old(cfg)
    m.load_state_dict(make_v2old_state_dict(cfg, 0), strict=True)
    return m


def _shape(H=480, W=640):
    return v2old_geometry(H, W, 10, (1400, 2400))[0]


def _bytes(m, T, S, B=1, H=480, W=640):
    lib = _cabi.lib()
    shape = _shape(H, W)
    h = _engine(m, T, S, shape)
    try:
        n = lib.udb_v2old_schedule_bytes(h, B, H, W)
        return n, ("" if n else lib.udb_last_error().decode())
    finally:
        lib.udb_v2old_destroy(h)


def _split_names(m):
    """Every operand the split packing stores as [N, 3K] (the encoder's first and last block stand for the others)."""
    last = m.spec.enc_depth - 1
    names = ["patch_w"] + [f"blocks.{i}.{k}_w" for i in (0, last) for k in ("qkv", "proj", "fc1", "fc2")]
    names += [f"adapt.{l}.w_cam" for l in range(4)] + ["cam.inf.w1", "cam.inf.w2", "cam.agg1.kv_w", "cam.agg2.kv_w"]
    return names + ["glob.rays_w", "glob.in_w", "glob.agg1.kv_w", "glob.agg2.kv_w"]


def _e4m3_names(m):
    last = m.spec.enc_depth - 1
    return [f"blocks.{i}.{k}_w8{s}" for i in (0, last) for k in ("qkv", "proj", "fc1", "fc2") for s in ("", "s")]


def _packs(bb):
    m = _model(bb)
    shape = _shape()
    out = {}
    for prec in ("f16", "split", "fp8"):
        m.precision = prec
        out[prec] = m._pack_tensors(CPU, shape)
    m.precision = "f16"
    return m, out


@pytest.mark.parametrize("bb", BACKBONES)
def test_split_and_fp8_packers(bb):
    m, P = _packs(bb)
    (T16, S16), (Ts, Ss), (T8, S8) = P["f16"], P["split"], P["fp8"]
    assert "precision" not in S16 and Ss == dict(S16, precision=1.0) and S8 == dict(S16, precision=2.0)
    split = _split_names(m)
    assert set(Ts) == set(T16) | {f"adapt.{l}.w_cam" for l in range(4)}
    for n in split:
        ref = T16[n.replace("_cam", "")]
        N, K = ref.shape
        assert Ts[n].dtype == torch.float16 and tuple(Ts[n].shape) == (N, 3 * K), n
        assert torch.equal(Ts[n][:, :K], ref) and torch.equal(Ts[n][:, K:2 * K], ref), n
    for k in T16:
        if k not in split and not (k.startswith("blocks.") and k.endswith(("qkv_w", "proj_w", "fc1_w", "fc2_w"))):
            assert torch.equal(Ts[k], T16[k]), k
    # fp8: the blocks' four weights become e4m3 + per-channel scales (pack_e4m3); every other operand is the f16 packing's
    for k in T16:
        if k.startswith("blocks.") and k.endswith(("qkv_w", "proj_w", "fc1_w", "fc2_w")):
            assert k not in T8 and T8[k + "8"].dtype == torch.float8_e4m3fn, k
            assert T8[k + "8s"].shape == (T16[k].shape[0],), k
        else:
            assert torch.equal(T8[k], T16[k]), k
    w = m.state_dict()["pixel_encoder.blocks.0.attn.qkv.weight"]
    w8, s = pack_e4m3(w)
    assert torch.equal(T8["blocks.0.qkv_w8"].view(torch.uint8), w8.view(torch.uint8)) and torch.equal(T8["blocks.0.qkv_w8s"], s)


@pytest.mark.parametrize("bb", BACKBONES)
@pytest.mark.parametrize("prec", ["split", "fp8"])
def test_schedule_accepts_exactly_the_new_operands(bb, prec):
    m, P = _packs(bb)
    T16, S16 = P["f16"]
    T, S = P[prec]
    for H, W, B in ((480, 640, 1), (375, 1242, 3)):
        shape = _shape(H, W)
        m.precision = prec
        Tx, Sx = m._pack_tensors(CPU, shape)
        n, msg = _bytes(m, Tx, Sx, B, H, W)
        assert n > 0, msg
    m.precision = "f16"
    names = _split_names(m) if prec == "split" else _e4m3_names(m)
    # dropping any of the mode's operands is reported by name
    for name in names:
        n, msg = _bytes(m, {k: v for k, v in T.items() if k != name}, S)
        assert n == 0 and f"'{name}'" in msg, (name, msg)
    # a mis-shaped (f16 layout) split operand, or an e4m3 operand holding f16 bytes, is refused by name
    for name in names[:2] + names[-6:]:
        bad = dict(T)
        if prec == "split":
            bad[name] = T16[name.replace("_cam", "")]
            want = "expected"
        elif name.endswith("_w8"):
            bad[name] = T16[name[:-1]]
            want = "e4m3"
        else:
            bad[name] = T[name][:-1].contiguous()
            want = "expected"
        n, msg = _bytes(m, bad, S)
        assert n == 0 and f"'{name}'" in msg and want in msg, (name, msg)
    # the mode's packing run as the f16 mode (no "precision" scalar) is refused naming an operand
    n, msg = _bytes(m, T, {k: v for k, v in S.items() if k != "precision"})
    assert n == 0 and ("'patch_w'" if prec == "split" else "'blocks.0.qkv_w'") in msg, msg
    # and the f16 packing run as this mode
    n, msg = _bytes(m, T16, dict(S16, precision=S["precision"]))
    if prec == "split":
        assert n == 0 and "precision 1" in msg and "split packing" in msg and "'patch_w'" in msg, msg
    else:
        assert n == 0 and "'blocks.0.qkv_w8'" in msg, msg
    n, msg = _bytes(m, T, dict(S, precision=3.0))
    assert n == 0 and "precision 3" in msg, msg


def test_precision_attribute():
    m = _model("vits14")
    assert m.precision == "f16"
    for bad in ("fp16", "bf16", "SPLIT", None):
        m.precision = bad
        with pytest.raises(ValueError, match="precision must be 'split', 'f16' or 'fp8'"):
            m._pack_tensors(CPU, _shape())
    keys = set()
    for prec in ("f16", "split", "fp8"):
        m.precision = prec
        keys.add(m._fingerprint())
        assert m._fingerprint()[0] == prec
    assert len(keys) == 3


# ------------------------------------------------------------------------------------------ rounding model
def _round_f16(t):
    return t.half().float()


def _round_e4m3_rows(t):
    """Per-row e4m3 with scale amax / 448, as the engine's activation quantiser and pack_e4m3 (per output channel)."""
    shp = t.shape
    w8, s = pack_e4m3(t.reshape(-1, shp[-1]))
    return (w8.float() * s[:, None]).reshape(shp)


class _Rounded(nn.Module):
    """nn.Linear / nn.Conv2d whose operands (input and weight) are rounded by `rnd` before an f32 product."""

    def __init__(self, mod, rnd):
        super().__init__()
        self.mod, self.rnd = mod, rnd

    def forward(self, x):
        m = self.mod
        if isinstance(m, nn.Linear):
            return F.linear(self.rnd(x), self.rnd(m.weight), m.bias)
        return m._conv_forward(self.rnd(x), self.rnd(m.weight), m.bias)      # f16 rounding only: elementwise


def _round_in(root, rnd, pred=lambda name: True):
    for name, mod in list(root.named_modules()):
        for cn, child in list(mod.named_children()):
            full = f"{name}.{cn}" if name else cn
            if isinstance(child, (nn.Linear, nn.Conv2d)) and pred(full):
                setattr(mod, cn, _Rounded(child, rnd))


@pytest.mark.skipif(not os.path.isdir(os.path.join(REFERENCE, "unidepth")), reason="needs the reference sources")
def test_rounding_model_locates_the_depth_error():
    """The unmodified reference UniDepthV2old on a seeded golden with operands rounded in chosen submodules: f16
    everywhere (the f16 mode), f16 in the depth head only (the split mode's prediction), f16 everywhere but the depth
    head, and e4m3 in the encoder blocks' four linear layers (the fp8 mode's prediction).  Only nn.Linear and nn.Conv2d
    operands are rounded; attention products and the map-wide steps stay f32.  Prints depth ARel / max-rel and intrinsics max-rel of each against the
    golden; asserts the ordering the experiment establishes."""
    sys.path[:0] = [REFERENCE, os.path.join(ROOT, "oracle", "ref_shims")]
    warnings.simplefilter("ignore")
    import unidepth.layers.nystrom_attention as NA
    from make_golden_v1 import OracleNystrom, seeded_rgb
    NA.NystromAttention = OracleNystrom
    from unidepth.models.unidepthv2.unidepthv2_old import UniDepthV2old as Ref

    name = "v2old_vits14_rl0_360x480"
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(z["__meta__"]))
    cfg = _cfg("vits14")
    sd = make_v2old_state_dict(cfg, meta["seed"])
    rgb = seeded_rgb(tuple(meta["shape"]), meta["seed"])
    st = meta["strides"]["depth"]
    dr = z["depth"].astype(np.float64)
    kr = z["intrinsics"].astype(np.float64)
    depth_head = "pixel_decoder.depth_layer."
    blocks = lambda n: n.startswith("pixel_encoder.blocks.") and n.endswith(("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2"))
    cases = {"f16 everywhere": (_round_f16, lambda n: True),
             "f16 depth head only (split prediction)": (_round_f16, lambda n: n.startswith(depth_head)),
             "f16 upstream of the depth head only": (_round_f16, lambda n: not n.startswith(depth_head)),
             "e4m3 encoder blocks (fp8 prediction)": (_round_e4m3_rows, blocks)}
    res = {}
    for label, (rnd, pred) in cases.items():
        ref = Ref(copy.deepcopy(cfg)).eval()
        ref.load_state_dict(sd, strict=True)
        ref.resolution_level = meta["resolution_level"]
        _round_in(ref, rnd, pred)
        with torch.no_grad():
            out = ref.infer(rgb)
        d = out["depth"][:, :, ::st, ::st].double().numpy()
        res[label] = (float(np.mean(np.abs(d - dr) / dr)), float(np.max(np.abs(d - dr) / dr)),
                      float(np.max(np.abs(out["intrinsics"].double().numpy() - kr) / np.maximum(np.abs(kr), 1.0))))
        print(f"V2OLDROUNDING {name} {label}: depth ARel {res[label][0]:.3e} max-rel {res[label][1]:.3e} "
              f"intrinsics rel {res[label][2]:.3e}")
    f16_all, head_only, upstream, fp8 = (res[k] for k in cases)
    # the depth head does not reach the intrinsics, and its f16 rounding is the smaller part of the f16 depth error: the
    # encoder and the camera / global heads upstream of it carry most of it
    assert head_only[2] == 0 and upstream[2] == f16_all[2]
    assert head_only[0] < upstream[0] and head_only[0] < f16_all[0]
    assert fp8[0] > f16_all[0]
