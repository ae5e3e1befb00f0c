"""UniDepthV1 (ConvNeXt-L or DINOv2 ViT-L/14 encoder) -- drop-in for the reference's inference API, running on libudb.so (sm_90a).

Mirrors `unidepth.models.UniDepthV1` for the inference path only (reference:
unidepth/models/unidepthv1/unidepthv1.py:96-110 constructor, :288-373 `infer`, :375-392 `load_pretrained`,
:418-420 `device`; HF-hub mixin `from_pretrained`):

    model = UniDepthV1.from_pretrained(dir_with_config_json_and_safetensors)    # or UniDepthV1(config)
    model = model.to("cuda").eval()
    out = model.infer(rgb_uint8, intrinsics=None, skip_camera=False)             # dict: intrinsics points depth

The module owns `nn.Parameter`s under exactly the reference's state-dict names (unidepth_b200/spec_v1.py), so reference
checkpoints load unchanged.  `infer` packs the weights once and makes ONE C call (`udb_infer_v1`, include/udb.h) that
enqueues the hand-written kernels on torch's current stream, optionally captured as a CUDA graph.  No CPU / eager fallback.

The 1/8 and 1/4 decoder levels use Nystrom attention (reference: xformers NystromAttention, absent here); this
implementation follows the published algorithm as restated in oracle/unidepth_v1_oracle.py -- parity for that one
function is unpinned (see DESIGN.md).
"""
from __future__ import annotations

import operator
from typing import Dict, Tuple

import torch

from . import _cabi as cabi
from ._pack import (adapter, attn_block, c32, convnext_block, cross_block, h16, latents, mlp, pack_vit_encoder,
                    pos_table_by_scale, split_weight, tokens_pos)
from .spec import PATCH
from .spec_v1 import (ENCODER_CONVNEXT, ENCODER_DINOV2, V1_INTERPOLATE_OFFSET, V1Spec, param_shapes, v1_paddings,
                      v1_shapes)
from ._engine_model import HUB_KWARGS, EngineModel, PyTorchModelHubMixin, f32

# ConvNeXt stages whose blocks run on e4m3 operands in precision "fp8" (engine_v1.cu kFp8Stage, the same fixed rule: a
# stage runs e4m3 only where that is measured faster, which on an H100 is none of them, DESIGN.md section 8)
FP8_STAGES = (False, False, False, False)


class UniDepthV1(EngineModel, PyTorchModelHubMixin, **HUB_KWARGS):
    _ENGINE_FNS = ("udb_v1_create", "udb_v1_destroy", "udb_v1_set_weight", "udb_v1_set_scalar")
    _INFER = (cabi.InferV1Args, "udb_infer_v1", "udb_v1_workspace_bytes")

    def __init__(self, config: dict, eps: float = 1e-6, **kwargs):
        super().__init__(config, eps, max_cached_workspaces=4)
        self.spec = V1Spec(config)
        self._add_params(param_shapes(config))
        # the network shape `infer` resizes and pads every input to (unidepthv1.py:443), read on every call as the
        # reference does: [height, width], landscape or square (see _network_shape)
        self.image_shape = list(self.spec.image_shape)
        # "f16" (default) or "fp8": speed mode -- the linear layers of the encoder blocks multiply FP8 E4M3 operands on the
        # e4m3 wgmma (include/udb.h udb_gemm_e4m3): weights with one scale per output channel, activations quantised per
        # row on the fly.  DINOv2 ViT-L: qkv, proj, fc1 and fc2, as UniDepthV2's fp8 mode.  ConvNeXt: the two MLP layers of
        # the blocks of the stages in FP8_STAGES, fed by a fused depthwise 7x7 + LayerNorm + quantisation kernel
        # (udb_dwconv7_ln_e4m3) -- an empty set, since no stage is faster that way, so ConvNeXt-L computes what "f16" does.  The stem, downsample layers, attention and the decoder stay f16.  Its accuracy is only measured on
        # seeded synthetic weights (tests/test_v1_fp8_gpu.py), not on trained checkpoints.
        # "split": parity / debugging mode, as UniDepthV2's -- every GEMM operand of the encoder and of the camera head's
        # context path (the adapters' camera copy, in_features, the aggregate block's kv) is a hi + lo pair fed through the
        # same wgmma GEMM (include/udb.h udb_gemm_t.a_split_k), the encoder levels and the camera context stay f32, and
        # ViT-L's attention runs in the fp32 kernel.  The depth head runs as in "f16".  Slower; not a speed mode.
        self.precision = "f16"

    def _network_shape(self) -> Tuple[int, int]:
        """`image_shape` as (net_h, net_w), checked before anything is packed or launched for it."""
        shp = self.image_shape
        try:
            h, w = shp
            if isinstance(h, bool) or isinstance(w, bool):
                raise TypeError
            h, w = operator.index(h), operator.index(w)
        except (TypeError, ValueError):
            raise ValueError(f"UniDepthV1.image_shape must be two integers [height, width], not {shp!r}") from None
        if h < 64 or w < 64:
            raise ValueError(f"UniDepthV1.image_shape {[h, w]}: each side must be at least 64 pixels")
        if self.spec.encoder == ENCODER_DINOV2 and (h % PATCH or w % PATCH):
            raise NotImplementedError(f"network shape {(h, w)} is not a multiple of the {PATCH}-pixel patch")
        if h > w:
            raise NotImplementedError(
                f"UniDepthV1.image_shape {[h, w]}: portrait network shapes are not supported.  The reference's decoder "
                "orders every token grid as sorted([h, w]) (decoder.py:384-396), so it runs a portrait shape as its "
                "transpose; use a landscape or square shape (height <= width)")
        return h, w

    _default_shape = _network_shape

    # ------------------------------------------------------------------ weight packing
    def _shape_operands(self, shape: Tuple[int, int], dev) -> Dict[str, torch.Tensor]:
        """The operands that depend on the network shape: "tokens_pos", the sine position embedding of the decoder's
        common grid plus the level embedding MLP of the four learned level vectors (decoder.py:410-433), and for DINOv2
        "pos", the patch grid's position table (dinov2.py:267-304)."""
        s = self.spec
        sd = self.state_dict()
        hc, wc = s.common_grid(shape)
        T: Dict[str, torch.Tensor] = {}
        if s.encoder == ENCODER_DINOV2:
            pos = c32(sd["pixel_encoder.pos_embed"].detach().reshape(-1, s.embed_dim))
            T["pos"] = c32(pos_table_by_scale(pos, hc, wc, V1_INTERPOLATE_OFFSET))
        T["tokens_pos"] = tokens_pos(sd, hc, wc, s.hidden, dev)
        return T

    def _pack_weights(self, dev):
        """The weight operands and scalars: everything but `_shape_operands`, so a change of network shape repacks
        nothing here."""
        s = self.spec
        split, fp8, code = self._precision()
        sd = {k: v.detach() for k, v in self.state_dict().items()}
        # GEMM weight of the split-precision mode's operands: [N, 3K] = [hi | hi | lo], or f16 in the other modes
        s16 = split_weight if split else h16
        T: Dict[str, torch.Tensor] = {}
        # an engine without "precision" runs the f16 mode, so the f16 packing registers exactly the scalars it always has
        S: Dict[str, float] = {"precision": float(code)} if code else {}
        pe, pd = "pixel_encoder.", "pixel_decoder."
        hid = s.hidden

        def zpad(t, rows, cols):
            out = torch.zeros((rows, cols), device=dev, dtype=f32)
            out[:t.shape[0], :t.shape[1]] = t
            return out

        def zpad1(t, n):
            out = torch.zeros(n, device=dev, dtype=f32)
            out[:t.shape[0]] = t
            return out

        # ---- encoder
        if s.encoder == ENCODER_DINOV2:
            # the V2 encoder's packing; the final norm, mask token and register tokens are never read (use_norm=False,
            # dinov2.py:173-178), and the position table is a shape operand
            T.update(pack_vit_encoder(sd, s.embed_dim, s.enc_depth, dev, split=split, fp8=fp8))
        for i, depth in enumerate(s.depths if s.encoder == ENCODER_CONVNEXT else ()):
            if i == 0:
                T["stem_w"] = s16(zpad(sd[pe + "stem.0.weight"].reshape(s.dims[0], 48), s.dims[0], 64))
                T["stem_b"] = c32(sd[pe + "stem.0.bias"])
                T["stem_ln_w"], T["stem_ln_b"] = c32(sd[pe + "stem.1.weight"]), c32(sd[pe + "stem.1.bias"])
            st = f"{pe}stages.{i}."
            if i > 0:
                w = sd[st + "downsample.1.weight"]                               # [C, Cp, 2, 2] -> [C, (dy,dx,ci)]
                T[f"ds{i}.ln_w"], T[f"ds{i}.ln_b"] = c32(sd[st + "downsample.0.weight"]), c32(sd[st + "downsample.0.bias"])
                T[f"ds{i}.w"], T[f"ds{i}.b"] = s16(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)), c32(sd[st + "downsample.1.bias"])
            for j in range(depth):
                convnext_block(T, sd, f"s{i}.b{j}.", f"{st}blocks.{j}.", ("conv_dw", "norm", "mlp.fc1", "mlp.fc2"),
                               fp8 and FP8_STAGES[i], s16)

        # ---- decoder: adapters, embeddings
        for l in range(4):
            a = f"{pd}input_adapter.input_adapters.{l}."
            adapter(T, sd, f"adapt.{l}.", a, h16)
            if split:       # the adapter's copy for the camera head, which reads it on split operands
                T[f"adapt.{l}.w_cam"] = split_weight(sd[a + "1.weight"])
            adapter(T, sd, f"tok.{l}.", f"{pd}token_adapter.input_adapters.{l}.", c32)

        cl = pd + "camera_layer."
        T["cam.cls.nw"], T["cam.cls.nb"] = c32(sd[cl + "cls_project.0.weight"]), c32(sd[cl + "cls_project.0.bias"])
        T["cam.cls.w1"], T["cam.cls.b1"] = c32(sd[cl + "cls_project.1.weight"]), c32(sd[cl + "cls_project.1.bias"])
        T["cam.cls.w2"], T["cam.cls.b2"] = c32(sd[cl + "cls_project.3.weight"]), c32(sd[cl + "cls_project.3.bias"])
        mlp(T, sd, "cam.inf", cl + "in_features", s16)
        T["cam.pos"] = c32(sd[cl + "latents_pos"].reshape(4, hid))
        cross_block(T, sd, "cam.agg.", cl + "aggregate.", s16)
        for i in range(2):
            cross_block(T, sd, f"cam.l{i}.", f"{cl}layers.{i}.", c32)
        mlp(T, sd, "cam.out", cl + "out", c32)

        dl = pd + "depth_layer."
        for name, outd in (("16", hid), ("8", hid // 2), ("4", hid // 4)):
            src = f"{dl}project_rays{name}"
            T[f"rays.{name}.ln_w"], T[f"rays.{name}.ln_b"] = zpad1(sd[src + ".norm.weight"].float(), 84), zpad1(sd[src + ".norm.bias"].float(), 84)
            T[f"rays.{name}.w1"] = h16(zpad(sd[src + ".proj1.weight"].float(), 384, 128))       # [324, 81] zero-extended
            T[f"rays.{name}.b1"] = zpad1(sd[src + ".proj1.bias"].float(), 384)
            T[f"rays.{name}.w2"] = h16(zpad(sd[src + ".proj2.weight"].float(), outd, 384))
            T[f"rays.{name}.b2"] = c32(sd[src + ".proj2.bias"])
        latents(T, sd, dl)
        attn_block(T, sd, "agg16.", dl + "aggregate_16.", True)
        attn_block(T, sd, "prompt.", dl + "prompt_camera.", True)
        for name, dst, n in (("layers_16", "l16", s.dec_depths[0]), ("layers_8", "l8", s.dec_depths[1]), ("layers_4", "l4", s.dec_depths[2])):
            for i in range(n):
                attn_block(T, sd, f"{dst}.{i}.", f"{dl}{name}.{i}.", False)
        for name in ("up8", "up4", "up2"):
            for j in range(2):
                convnext_block(T, sd, f"{name}.c{j}.", f"{dl}{name}.convs.{j}.", ("dwconv", "norm", "pwconv1", "pwconv2"))
            uw = sd[f"{dl}{name}.up.0.weight"]
            T[f"{name}.up_w"], T[f"{name}.up_b"] = h16(uw.reshape(uw.shape[0], uw.shape[1])), c32(sd[f"{dl}{name}.up.0.bias"])
            cw = sd[f"{dl}{name}.up.2.weight"]
            T[f"{name}.conv_w"] = h16(cw.permute(0, 2, 3, 1).reshape(cw.shape[0], -1))
            T[f"{name}.conv_b"] = c32(sd[f"{dl}{name}.up.2.bias"])
        for name in ("out8", "out4", "out2"):
            w = sd[f"{dl}{name}.weight"]                                             # [1, C, 3, 3] -> [9, C]
            T[f"{name}.w"] = c32(w.permute(0, 2, 3, 1).reshape(9, w.shape[1]))
            S[f"{name}.b"] = float(sd[f"{dl}{name}.bias"].item())
        return T, S

    # ------------------------------------------------------------------ engine
    def _engine_config(self, shape=None) -> "cabi.V1Config":
        """udb_v1_config_t of this model at the network shape `shape` (default: `image_shape`) (include/udb.h)."""
        s = self.spec
        cfg = cabi.V1Config()
        for i in range(4):
            cfg.depths[i], cfg.dims[i] = s.depths[i], s.dims[i]
        cfg.hidden, cfg.heads, cfg.expansion = s.hidden, s.heads, s.expansion
        for i in range(3):
            cfg.dec_depths[i] = s.dec_depths[i]
        cfg.net_h, cfg.net_w = shape or self._network_shape()
        cfg.encoder = s.encoder
        return cfg

    # ------------------------------------------------------------------ infer
    @torch.no_grad()
    def infer(self, rgbs: torch.Tensor, intrinsics=None, skip_camera: bool = False):
        """Same contract as the reference `UniDepthV1.infer` (unidepthv1.py:288-373)."""
        if rgbs.ndim == 3:
            rgbs = rgbs.unsqueeze(0)
        if intrinsics is not None and intrinsics.ndim == 2:
            intrinsics = intrinsics.unsqueeze(0)
        shape = self._network_shape()

        def check(handle):      # a dry run names any bound the shape breaks before anything is launched
            lib = cabi.lib()
            if lib.udb_v1_workspace_bytes(handle, 1, *shape) == 0:
                raise NotImplementedError(f"UniDepthV1.image_shape {list(shape)}: {lib.udb_last_error().decode()}")

        return self._infer(rgbs, intrinsics, shape, check, skip_camera=int(bool(skip_camera and intrinsics is not None)))

    def forward(self, *args, **kwargs):
        raise NotImplementedError("training / validation forward of UniDepthV1 is out of scope; use .infer()")
