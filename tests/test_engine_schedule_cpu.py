"""Host logic of the two whole-path engines, without a GPU: pack a model's weights on the CPU with the product's own packer
(`_pack_tensors`), register them with a C engine (`udb_set_weight` only stores pointers) and let the engine DRY-RUN its
schedule (`udb_schedule_bytes`, `udb_v1_workspace_bytes`: every stage is walked, operand names and shapes are checked, the
bump allocator is sized; nothing is launched and no device is touched).  This pins the contract between the Python packers
and the C schedules for every packing mode (default f16, split precision, fused LayerNorm) and every shipped model size;
the GPU tests then only have to show that the kernels compute the right numbers."""
import copy
import ctypes as C
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from fixture import make_state_dict  # noqa: E402
from unidepth_b200 import UniDepthV1, UniDepthV2, _cabi  # noqa: E402

CPU = torch.device("cpu")


def _v2(cfg_name, depth=None, **attrs):
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", cfg_name)))
    if depth is not None:                       # ViT-L width, shallow: keeps the CPU packing small
        cfg["model"]["pixel_encoder"]["arch_override"] = {"depth": depth}
        cfg["model"]["pixel_encoder"]["output_idx"] = [1, 2, 3, 4]
    m = UniDepthV2(copy.deepcopy(cfg))
    m.load_state_dict(make_state_dict(cfg, 0), strict=True)
    for k, v in attrs.items():
        setattr(m, k, v)
    return m.eval()


def _v2_engine(m, drop=(), reshape=None, scalars_over=None):
    tensors, scalars = m._pack_tensors(CPU)
    scalars = dict(scalars, **(scalars_over or {}))
    cfg = m._engine_config()
    for name in drop:
        del tensors[name]
    if reshape:
        name, fn = reshape
        tensors[name] = fn(tensors[name]).contiguous()
    h = C.c_void_p()
    _cabi.check(_cabi.lib().udb_create(C.byref(cfg), C.byref(h)), "udb_create")
    m._register(h, tensors, scalars)
    return h, tensors          # the caller keeps `tensors` alive while the engine holds their pointers


@pytest.mark.parametrize("cfg_name,depth,attrs", [
    ("config_v2_vits14.json", None, {}),
    ("config_v2_vitb14.json", None, {}),
    ("config_v2_vitl14.json", 4, {}),
    ("config_v2_vitl14.json", 4, {"precision": "split"}),
    ("config_v2_vitl14.json", 4, {"fuse_ln": True}),
    ("config_v2_vits14.json", None, {"precision": "split"}),
])
def test_v2_packer_and_schedule_agree(cfg_name, depth, attrs):
    lib = _cabi.lib()
    m = _v2(cfg_name, depth, **attrs)
    h, keep = _v2_engine(m)
    try:
        sizes = {}
        for (B, H, W, lvl) in ((1, 480, 640, -1), (2, 480, 640, -1), (2, 96, 288, 3), (1, 1000, 400, 9), (1, 490, 644, -2)):
            n = lib.udb_schedule_bytes(h, B, H, W, lvl)
            assert n > 0, (B, H, W, lvl, lib.udb_last_error().decode())
            sizes[(B, H, W, lvl)] = n
        assert sizes[(2, 480, 640, -1)] > sizes[(1, 480, 640, -1)]                  # activations scale with the batch
        assert lib.udb_schedule_bytes(h, 1, 480, 640, 10) == 0                      # resolution_level out of range
        assert lib.udb_schedule_bytes(h, 1, 481, 640, -2) == 0                      # network-only input not a multiple of 14
        # a dry run prepares nothing: the real call still refuses the shape
        a = _cabi.InferArgs()
        assert lib.udb_infer_v2(h, C.byref(a), None) != 0
    finally:
        lib.udb_destroy(h)
    del keep


def test_v2_schedule_names_the_missing_or_misshapen_operand():
    lib = _cabi.lib()
    m = _v2("config_v2_vits14.json")
    names = list(m._pack_tensors(CPU)[0])
    # every registered tensor is needed: dropping any one of a spread of them is reported by name
    for name in names[:: max(1, len(names) // 12)]:
        h, keep = _v2_engine(m, drop=(name,))
        try:
            assert lib.udb_schedule_bytes(h, 1, 240, 320, -1) == 0
            assert name in lib.udb_last_error().decode(), (name, lib.udb_last_error().decode())
        finally:
            lib.udb_destroy(h)
    # a weight packed with the wrong shape (here: transposed) is rejected, not read with the wrong leading dimension
    h, keep = _v2_engine(m, reshape=("blocks.0.fc1_w", lambda t: t.t()))
    try:
        assert lib.udb_schedule_bytes(h, 1, 240, 320, -1) == 0
        msg = lib.udb_last_error().decode()
        assert "blocks.0.fc1_w" in msg and "expected" in msg, msg
    finally:
        lib.udb_destroy(h)


@pytest.mark.parametrize("precision,want", [
    (3.0, ("udb_infer_v2", "precision 3 unsupported")),                          # no such mode: refused, not run as f16
    (1.0, ("udb_infer_v2", "precision 1", "split packing", "'patch_w'")),       # the f16 packing named as such
])
def test_v2_schedule_checks_the_precision(precision, want):
    lib = _cabi.lib()
    h, keep = _v2_engine(_v2("config_v2_vits14.json"), scalars_over={"precision": precision})
    try:
        assert lib.udb_schedule_bytes(h, 1, 240, 320, -1) == 0
        msg = lib.udb_last_error().decode()
        assert all(w in msg for w in want), msg
    finally:
        lib.udb_destroy(h)
    del keep


def _v1(arch=None):
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", "config_v1_cnvnxtl.json")))
    if arch is not None:
        cfg["model"]["pixel_encoder"]["arch"] = arch
    return UniDepthV1(copy.deepcopy(cfg)).eval()


@pytest.mark.parametrize("arch", [{"depths": [1, 1, 2, 1], "dims": [64, 128, 192, 256]}, None])
def test_v1_packer_and_schedule_agree(arch):
    """`None` is the shipped ConvNeXt-L (BASELINE config 4: depths 3-3-27-3, dims 192..1536), default-initialised."""
    lib = _cabi.lib()
    m = _v1(arch)
    T, S = m._pack_tensors(CPU)
    h = C.c_void_p()
    _cabi.check(lib.udb_v1_create(C.byref(m._engine_config()), C.byref(h)), "udb_v1_create")
    try:
        m._register(h, T, S)
        n1 = lib.udb_v1_workspace_bytes(h, 1, 480, 640)
        assert n1 > 0, lib.udb_last_error().decode()
        n4 = lib.udb_v1_workspace_bytes(h, 4, 480, 640)
        assert n4 > n1
        assert lib.udb_v1_workspace_bytes(h, 1, 375, 1242) > 0 and lib.udb_v1_workspace_bytes(h, 1, 1000, 400) > 0
        assert lib.udb_v1_workspace_bytes(h, 0, 480, 640) == 0
    finally:
        lib.udb_v1_destroy(h)
    # one operand or scalar short (the output heads' biases included): reported by name
    for name in list(T)[:: max(1, len(T) // 10)] + list(S):
        h = C.c_void_p()
        _cabi.check(lib.udb_v1_create(C.byref(m._engine_config()), C.byref(h)), "udb_v1_create")
        try:
            m._register(h, {k: v for k, v in T.items() if k != name}, {k: v for k, v in S.items() if k != name})
            assert lib.udb_v1_workspace_bytes(h, 1, 480, 640) == 0
            assert name in lib.udb_last_error().decode(), (name, lib.udb_last_error().decode())
        finally:
            lib.udb_v1_destroy(h)
