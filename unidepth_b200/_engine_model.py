"""Host runtime shared by UniDepthV1, UniDepthV2 and UniDepthV2old: parameters under the reference's state-dict names,
checkpoint loading, weight packing per weight version, the C engine's lifetime, the engine of a network shape, the input
block of `infer`, and the workspace and CUDA-graph caches.

A model class supplies its packer (`_pack_weights`, plus `_shape_operands` for an engine per network shape; `_pack_tensors`
-> ({engine tensor name: tensor}, {scalar name: float}) joins the two; the shared packing code is `_pack.py`), its config
struct (`_engine_config`), the names of its engine's C entry points (`_ENGINE_FNS`, and `_INFER` for the UniDepthV1
family's infer call) and the calls that look up its engine and run it."""
from __future__ import annotations

import ctypes as C
import json
import os
from collections import OrderedDict

import torch
import torch.nn as nn

from . import _cabi as cabi
from .spec import PATCH

try:  # same mixin as the reference (unidepthv2.py:111-117)
    from huggingface_hub import PyTorchModelHubMixin
    _HAS_HF = True
except Exception:  # pragma: no cover
    _HAS_HF = False

    class PyTorchModelHubMixin:  # minimal stand-in: local directories only
        def __init_subclass__(cls, **kwargs):
            super().__init_subclass__()

# Class keywords of the hub mixin.  Each public model class lists the mixin and these itself: the mixin records the
# __init__ of the class it is declared on.
HUB_KWARGS = dict(library_name="UniDepth", repo_url="https://github.com/lpiccinelli-eth/UniDepth",
                  tags=["monocular-metric-depth-estimation"]) if _HAS_HF else {}

f16, f32 = torch.float16, torch.float32
# the accepted `precision` modes; a mode's index is the engine's "precision" scalar (engine_common.h encoder_precision)
PRECISIONS = ("f16", "split", "fp8")
_DTYPES = {f16: cabi.DT_F16, f32: cabi.DT_F32, torch.float8_e4m3fn: cabi.DT_E4M3}   # udb.h UDB_DT_*


def infer_inputs(rgbs: torch.Tensor, intrinsics, dev):
    """The input block of UniDepthV1.infer and UniDepthV2old.infer (unidepthv1.py:301-308, unidepthv2_old.py:211-218)
    -> (rgbs, K, scale255, normalize): the batch on `dev`, uint8 or f32, contiguous; "/255" when the data looks like
    0..255, ImageNet normalisation when it then lies in [0, 1] (uint8: both); K the intrinsics as [B, 3, 3] f32, one
    matrix per image, or None."""
    rgbs = rgbs.to(dev)
    B = rgbs.shape[0]
    if rgbs.dtype == torch.uint8:
        scale255, normalize = True, True
    else:
        rgbs = rgbs.float()
        mx, mn = float(rgbs.max()), float(rgbs.min())
        scale255 = mx > 5
        if scale255:
            mx, mn = mx / 255.0, mn / 255.0
        normalize = mn >= 0.0 and mx <= 1.0
    rgbs = rgbs.contiguous()
    K = None
    if intrinsics is not None:
        K = intrinsics.to(dev, f32).reshape(-1, 3, 3)
        if K.shape[0] != B:
            raise ValueError(f"intrinsics holds {K.shape[0]} matrices for a batch of {B} images")
        K = K.contiguous()
    return rgbs, K, scale255, normalize


class _Node(nn.Module):
    """Anonymous container used to reproduce the reference's dotted parameter names."""


class EngineModel(nn.Module):
    # include/udb.h entry points of the model's engine: (create, destroy, set_weight, set_scalar)
    _ENGINE_FNS: tuple

    def __init__(self, config: dict, eps: float, max_cached_workspaces: int):
        super().__init__()
        self.config = config
        self.eps = eps
        self.use_cuda_graph = True
        # optional dict of preallocated output tensors (same keys / shapes as infer's result): graph-mode infer copies its
        # static outputs there instead of cloning them (parallel.PeerGather.views(): the multi-GPU send slot)
        self.output_buffers = None
        # Bounded caches (LRU): the reference handles arbitrary shapes in constant memory, so a stream of
        # differently-sized images must not grow device memory without limit.  A captured graph keeps its own
        # reference to the workspace it was captured with, so evicting a workspace never frees memory a live
        # graph still replays into.
        self.max_cached_graphs = 8
        self.max_cached_workspaces = max_cached_workspaces
        self._graphs: "OrderedDict[tuple, dict]" = OrderedDict()
        self._workspaces: "OrderedDict[tuple, torch.Tensor]" = OrderedDict()
        self._last_ws = None
        self._packed = None          # (tensors, scalars) of the weight version `_packed_key`
        self._packed_key = None
        self._engine = self._engine_key = self._engine_device = None

    def _add_params(self, shapes: dict):
        """Zero f32 parameters under the reference's dotted state-dict names."""
        for dotted, shape in shapes.items():
            *path, leaf = dotted.split(".")
            mod = self
            for p in path:
                if p not in mod._modules:
                    mod.add_module(p, _Node())
                mod = mod._modules[p]
            mod.register_parameter(leaf, nn.Parameter(torch.zeros(shape, dtype=f32), requires_grad=False))

    # ------------------------------------------------------------------ reference-compatible API
    @property
    def device(self):
        return next(self.parameters()).device

    def _cuda_device(self):
        """The model's device, which packing and every engine call need to be a CUDA device."""
        dev = self.device
        if dev.type != "cuda":
            raise RuntimeError("unidepth_b200 has no CPU path: move the model to a CUDA device")
        return dev

    def load_pretrained(self, model_file: str):
        """unidepthv2.py:381-394 / unidepthv1.py:375-392: torch checkpoint, optional 'model' key, strip 'module.'."""
        sd = torch.load(model_file, map_location="cpu", weights_only=False)
        if "model" in sd:
            sd = sd["model"]
        sd = {k.replace("module.", ""): v for k, v in sd.items()}
        info = self.load_state_dict(sd, strict=False)
        print(f"Loaded from {model_file} for {self.__class__.__name__} results in:", info)

    if not _HAS_HF:
        @classmethod
        def from_pretrained(cls, path: str, **kwargs):
            config = json.load(open(os.path.join(path, "config.json")))
            model = cls(config=config.get("config", config))
            st = os.path.join(path, "model.safetensors")
            if os.path.exists(st):
                from safetensors.torch import load_file
                model.load_state_dict(load_file(st), strict=False)
            else:
                model.load_state_dict(torch.load(os.path.join(path, "pytorch_model.bin"), map_location="cpu"),
                                      strict=False)
            return model

    # ------------------------------------------------------------------ weight packing
    def _precision(self):
        """(split, fp8, code) of the model's `precision`, one of PRECISIONS: code is the engine's "precision" scalar."""
        if self.precision not in PRECISIONS:
            raise ValueError(f"precision must be 'split', 'f16' or 'fp8', not {self.precision!r}; the engine's \"precision\" "
                             "scalar numbers 'f16', 'split' or 'fp8' as 0, 1 or 2")
        code = PRECISIONS.index(self.precision)
        return code == 1, code == 2, code

    def _fingerprint(self):
        return (self.precision,) + tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _default_shape(self):
        """The network shape `_pack_tensors` and `_engine_config` take when given none; None: the model has no shape
        operands (its engine takes every network shape)."""
        return None

    def _pack_tensors(self, dev, shape=None):
        """({engine tensor name: tensor on `dev`}, {scalar name: float}): the weight operands (`_pack_weights`) and, for
        a model with one engine per network shape, the operands of `shape` (default `_default_shape()`).  The product
        packs the two parts separately (`_weights`, `_shape_engine`); the CPU tests run this to check, through the
        engine's dry run, that the packer registers exactly the operands the C schedule asks for."""
        T, S = self._pack_weights(dev)
        shape = shape or self._default_shape()
        if shape is not None:
            T.update(self._shape_operands(shape, dev))
        return T, S

    def _weights(self):
        """The packed (tensors, scalars), repacked once per weight version; a repack drops the engine and its caches."""
        if self._packed is None or self._packed_key != self._fingerprint():
            dev = self._cuda_device()
            torch.cuda.set_device(dev)      # callers hold the device context of `_run_graphed`
            self._drop_engine()             # it borrows the pointers of the tensors about to be replaced
            self._packed = self._pack_weights(dev)
            self._packed_key = self._fingerprint()
        return self._packed

    # ------------------------------------------------------------------ C engine
    def _register(self, handle, tensors: dict, scalars: dict):
        """set_weight / set_scalar for every packed operand (the engine borrows the pointers)."""
        _, _, set_weight, set_scalar = self._ENGINE_FNS
        lib = cabi.lib()
        for name, t in tensors.items():
            assert t.is_contiguous() and t.dtype in _DTYPES, name
            shape = (C.c_int64 * max(t.ndim, 1))(*t.shape)
            cabi.check(getattr(lib, set_weight)(handle, name.encode(), C.c_void_p(t.data_ptr()), shape, t.ndim,
                                                _DTYPES[t.dtype]), f"{set_weight}({name})")
        for name, v in scalars.items():
            cabi.check(getattr(lib, set_scalar)(handle, name.encode(), float(v)), f"{set_scalar}({name})")

    def _create_engine(self, cfg, key=None, tensors=None, check=None):
        """A new engine for the config struct `cfg`, with `tensors` (default: the packed weights) and the packed scalars
        registered; `key` is what the caller compares to decide when to rebuild it.  `check(handle)` may refuse the new
        engine by raising: it is destroyed and the current engine stays as it was.  Otherwise the new engine replaces the
        current one, which is dropped with its workspaces and graphs."""
        packed, scalars = self._weights()
        tensors = packed if tensors is None else tensors
        create, destroy = self._ENGINE_FNS[:2]
        handle = C.c_void_p()
        cabi.check(getattr(cabi.lib(), create)(C.byref(cfg), C.byref(handle)), create)
        try:
            for name, t in tensors.items():
                assert t.is_cuda, name
            self._register(handle, tensors, scalars)
            if check is not None:
                check(handle)
        except BaseException:
            getattr(cabi.lib(), destroy)(handle)
            raise
        self._drop_engine()
        self._engine, self._engine_key, self._engine_device = handle, key, self.device
        return handle

    def _shape_engine(self, shape, check=None):
        """The engine of the network shape `shape` (UniDepthV1, UniDepthV2old: one engine per shape).  A new shape makes
        a new engine for `_engine_config(shape)` with the packed weights and the shape's own operands
        (`_shape_operands`); `_create_engine` drops the previous one, with its workspaces and graphs, only once the new
        one has passed `check`."""
        T, _ = self._weights()
        if self._engine is not None and self._engine_key == shape:
            return self._engine
        ops = self._shape_operands(shape, self.device)
        handle = self._create_engine(self._engine_config(shape), shape, tensors={**T, **ops}, check=check)
        self._shape_ops = ops              # the engine borrows their pointers
        return handle

    def _drop_engine(self):
        """Destroy the engine AND everything that holds raw pointers into it: captured graphs replay kernels whose
        arguments point at the engine's tables and at the workspaces, so they go first."""
        self._graphs.clear()
        if self._engine is not None:
            torch.cuda.synchronize(self._engine_device)       # nothing may still be running out of the tables we free
            getattr(cabi.lib(), self._ENGINE_FNS[1])(self._engine)
        self._engine = self._engine_key = None
        self._workspaces.clear()

    def __del__(self):
        try:
            self._drop_engine()
        except Exception:
            pass

    def _workspace(self, key: tuple, nbytes) -> torch.Tensor:
        """The cached workspace for `key`, or a new one of `nbytes()` bytes (0: the engine refused the shape)."""
        ws = self._workspaces.get(key)
        if ws is None:
            n = nbytes()
            if n == 0:
                raise RuntimeError(f"engine workspace sizing failed: {cabi.lib().udb_last_error().decode()}")
            ws = torch.empty(n, device=self.device, dtype=torch.uint8)
            self._workspaces[key] = ws
            while len(self._workspaces) > self.max_cached_workspaces:
                self._workspaces.popitem(last=False)
        else:
            self._workspaces.move_to_end(key)
        self._last_ws = ws
        return ws

    def _infer_call(self, eng, rgb: torch.Tensor, K, scale255: bool = False, normalize: bool = False, **fields) -> dict:
        """One checked infer call of a UniDepthV1-family engine `eng` (`_INFER`: udb_infer_v1, udb_infer_v2old) on
        `rgb` [B, 3, H, W] with the intrinsics `K` [B, 3, 3] or None -> {"intrinsics", "points", "depth" and, where the
        args struct has it, "confidence"}, new tensors with their maps at (H, W), or at (`out_h`, `out_w`) when the
        caller sets them.  `fields` are the caller's own fields of the args struct (`_INFER`); this fills the ones
        InferV1Args and InferV2oldArgs share, with the cached workspace of (B, H, W)."""
        args, infer_fn, workspace_fn = self._INFER
        lib = cabi.lib()
        a = args(**fields)
        B, _, H, W = rgb.shape
        h, w = fields.get("out_h", H), fields.get("out_w", W)
        E = lambda *shape: torch.empty(shape, device=rgb.device, dtype=f32)
        out = {"intrinsics": E(B, 3, 3), "points": E(B, 3, h, w), "depth": E(B, 1, h, w)}
        if hasattr(a, "out_confidence"):
            out["confidence"] = E(B, 1, h, w)
            a.out_confidence = out["confidence"].data_ptr()
        # the workspaces go with their engine (_drop_engine), so (B, H, W) names one
        ws = self._workspace((B, H, W), lambda: getattr(lib, workspace_fn)(eng, B, H, W))
        a.rgb, a.rgb_is_u8, a.scale255, a.normalize = rgb.data_ptr(), int(rgb.dtype == torch.uint8), int(scale255), int(normalize)
        a.B, a.H, a.W = B, H, W
        a.intrinsics = K.data_ptr() if K is not None else None
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
        a.out_intrinsics, a.out_points, a.out_depth = out["intrinsics"].data_ptr(), out["points"].data_ptr(), out["depth"].data_ptr()
        cabi.check(getattr(lib, infer_fn)(eng, C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)), infer_fn)
        return out

    # ------------------------------------------------------------------ entry points
    def _infer(self, rgbs: torch.Tensor, intrinsics, shape, check=None, **fields) -> dict:
        """The body of UniDepthV1.infer and UniDepthV2old.infer: `rgbs` [B, 3, H, W] through the engine of the network
        shape `shape` (`_shape_engine` with `check`), with the class's own args-struct `fields` (`_infer_call`), which
        also key the CUDA graph."""
        dev = self._cuda_device()
        rgbs, K, scale255, normalize = infer_inputs(rgbs, intrinsics, dev)
        run = lambda eng, x, inputs: self._infer_call(eng, x, inputs.get("K"), scale255, normalize, **fields)
        key = (shape, tuple(rgbs.shape), rgbs.dtype, scale255, normalize, K is not None) + tuple(fields.values())
        return self._run_graphed(lambda: self._shape_engine(shape, check), run, rgbs, {} if K is None else {"K": K}, key)

    def _check_eval_call(self, inputs):
        """The evaluation call `model(inputs_dict, image_metas)` runs in eval mode only."""
        if self.training or not isinstance(inputs, dict):
            raise NotImplementedError(f"{type(self).__name__}.forward runs the evaluation call model(inputs_dict, "
                                      "image_metas) in eval mode only (model.eval()); the training forward is out of scope")

    @staticmethod
    def _network_input_shape(image: torch.Tensor):
        """(B, h, w) of a network input `image` [B, 3, h, w] (no resize or padding), whose sides are multiples of the
        patch size.  Raises before anything touches the device."""
        if image.ndim != 4 or image.shape[1] != 3:
            raise ValueError(f"the network input must be [B, 3, h, w], not {tuple(image.shape)}")
        B, _, h, w = image.shape
        if h % PATCH or w % PATCH:
            raise ValueError(f"network input {h}x{w} must be a multiple of {PATCH}: both sides must be multiples of the patch "
                             "size")
        return B, h, w

    # ------------------------------------------------------------------ CUDA graphs
    def _run_graphed(self, engine, run, rgb: torch.Tensor, inputs: dict, key: tuple, keep=None,
                     output_buffers: bool = True) -> dict:
        """`run(eng, rgb, inputs)` -> outputs on the engine `engine()` returns, eagerly or by replaying a CUDA graph
        cached under `key`.  Everything runs with the model's device current (streams, the engine's allocations, the
        per-device kernel attributes on the C side), so a model on cuda:1 works while cuda:0 is the process default.
        `engine()` packs the weights (`_weights()`): a repack drops every graph, so none replays stale weights.  The
        graph reads static copies of `rgb` and of the tensors in `inputs`, refreshed before every replay; `keep` is
        anything else a captured kernel reads, which the cache entry must own.  `output_buffers=False`: return fresh
        tensors even when `self.output_buffers` is set (it holds `infer`'s outputs only)."""
        with torch.cuda.device(self._cuda_device()):
            eng = engine()
            if not self.use_cuda_graph:
                return run(eng, rgb, inputs)
            entry = self._graphs.get(key)
            if entry is None:
                static_in = rgb.clone()
                static_inputs = {k: v.clone() for k, v in inputs.items()}
                # warm-up on a side stream (allocator, per-shape tables, workspace), then capture
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    run(eng, static_in, static_inputs)
                torch.cuda.current_stream().wait_stream(side)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    static_out = run(eng, static_in, static_inputs)
                # the entry owns everything whose address the captured kernels read
                entry = dict(graph=graph, inp=static_in, inputs=static_inputs, out=static_out, ws=self._last_ws, keep=keep)
                self._graphs[key] = entry
                while len(self._graphs) > self.max_cached_graphs:
                    self._graphs.popitem(last=False)
            else:
                self._graphs.move_to_end(key)
            entry["inp"].copy_(rgb, non_blocking=True)
            for k, v in inputs.items():
                entry["inputs"][k].copy_(v, non_blocking=True)
            entry["graph"].replay()
            bufs = self.output_buffers if output_buffers else None
            if bufs is not None:       # caller-provided destinations (e.g. the send slot of parallel.PeerGather): one copy, no clone
                for k, v in entry["out"].items():
                    bufs[k].copy_(v)
                return {k: bufs[k] for k in entry["out"]}
            return {k: v.clone() for k, v in entry["out"].items()}
