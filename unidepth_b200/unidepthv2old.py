"""UniDepthV2old (DINOv2 ViT-L/14 or ViT-S/14 encoder) -- drop-in for the reference's inference API, running on libudb.so
(sm_90a).

Mirrors `unidepth.models.unidepthv2.unidepthv2_old.UniDepthV2old` for the inference and evaluation paths (reference:
unidepth/models/unidepthv2/unidepthv2_old.py:126-132 constructor, :134-196 `forward` in eval mode, :198-282 `infer`,
:284-300 `load_pretrained`, :302-304 `device`, :343-349 the `shape_constraints` / `interpolation_mode` /
`resolution_level` attributes; HF-hub mixin `from_pretrained`):

    model = UniDepthV2old.from_pretrained(dir_with_config_json_and_safetensors)     # or UniDepthV2old(config)
    model = model.to("cuda").eval()
    model.resolution_level = 5                                                       # None: the maximum (10), with a warning
    out = model.infer(rgb_uint8, intrinsics=None)       # dict: intrinsics points depth confidence
    out = model(inputs, image_metas)                    # the reference's evaluation forward (see `forward`)

The module owns `nn.Parameter`s under exactly the reference's state-dict names (unidepth_b200/spec_v2old.py), so
reference checkpoints load unchanged.  `infer` packs the weights once and makes ONE C call (`udb_infer_v2old`,
include/udb.h) that enqueues the hand-written kernels on torch's current stream, replayed as a CUDA graph per input
shape.  No CPU / eager fallback.  The network shape follows the input's aspect ratio and the resolution level, so the
engine (one per network shape, as UniDepthV1's) is rebuilt when that shape changes.

The first decoder level uses Nystrom attention (reference: xformers NystromAttention, absent here); this implementation
follows the published algorithm as restated in oracle/unidepth_v1_oracle.py, as UniDepthV1 does -- parity for that one
function is unpinned (see DESIGN.md).
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, Tuple

import torch

from . import _cabi as cabi
from ._engine_model import HUB_KWARGS, EngineModel, PyTorchModelHubMixin, f32
from ._pack import (adapter, attn_block, c32, convnext_block, cross_block, h16, latents, mlp, pack_vit_encoder,
                    pos_table_by_size, split_weight, tokens_pos)
from .spec import PATCH
from .spec_v2old import RAY_K, V2oldSpec, check_ratio, check_resolution, param_shapes


def v2old_geometry(H: int, W: int, level: int, pixels_bounds) -> Tuple[Tuple[int, int], float]:
    """((net_h, net_w), ratio) of an H x W input at the (clipped) resolution level: the engine's own arithmetic
    (udb_v2old_geometry, unidepthv2_old.py:45-92)."""
    g = cabi.V2oldGeometry()
    lo, hi = sorted(pixels_bounds)
    cabi.check(cabi.lib().udb_v2old_geometry(int(H), int(W), int(level), int(lo), int(hi), C.byref(g)), "udb_v2old_geometry")
    return (g.net_h, g.net_w), g.ratio


class UniDepthV2old(EngineModel, PyTorchModelHubMixin, **HUB_KWARGS):
    _ENGINE_FNS = ("udb_v2old_create", "udb_v2old_destroy", "udb_v2old_set_weight", "udb_v2old_set_scalar")
    _INFER = (cabi.InferV2oldArgs, "udb_infer_v2old", "udb_v2old_workspace_bytes")

    def __init__(self, config: dict, eps: float = 1e-6, **kwargs):
        super().__init__(config, eps, max_cached_workspaces=4)
        self.spec = V2oldSpec(config)
        self._add_params(param_shapes(config))
        # the reference's attributes (unidepthv2_old.py:343-349), read on every call
        sc = dict(config["data"]["shape_constraints"])
        sc["pixels_bounds_ori"] = list(sc.get("pixels_bounds", [1400, 2400]))
        self.shape_constraints = sc
        self.interpolation_mode = "bilinear"
        self.resolution_level = None
        # "f16" (default), "fp8" or "split", as UniDepthV1's.  "fp8": speed mode -- the encoder blocks' qkv, proj, fc1 and
        # fc2 multiply FP8 E4M3 operands (include/udb.h udb_gemm_e4m3) with per-output-channel weight scales and per-row
        # activation scales; the taps, heads and decoder run as in "f16".  "split": parity / debugging mode -- every GEMM
        # on the path from the image to the intrinsics and to the global (scale, shift) (patch embedding, encoder blocks,
        # the adapters' copy for the two heads, the camera head's in_features and kv, the global head's project_rays,
        # in_features and kv) multiplies hi + lo f16 operands (udb_gemm_t.a_split_k), the taps and the heads' contexts
        # are f32 and the encoder's attention runs in the fp32 kernel.  The depth head runs as in "f16".  Slower; not a
        # speed mode.  Changing it repacks the weights.
        self.precision = "f16"

    def _default_shape(self) -> Tuple[int, int]:
        """The network shape of a 480 x 640 input at the maximum level."""
        return v2old_geometry(480, 640, 10, self.shape_constraints["pixels_bounds_ori"])[0]

    # ------------------------------------------------------------------ weight packing
    def _shape_operands(self, shape: Tuple[int, int], dev) -> Dict[str, torch.Tensor]:
        """The operands that depend on the network shape: "pos", the DINOv2 position table resized (bicubic, to the
        patch grid's size: interpolate_offset 0, dinov2.py:267-304); "tokens_pos", the sine position embedding of the
        patch grid plus the level embedding MLP of the four learned level vectors (decoder_old.py:463-479); and
        "ray_scales.{i}", the 32 Fourier frequencies 2^linspace(0, log2(max(grid_i) // 2)) of the three decoder grids
        (positional_embedding.py:230-233), computed on the CPU as the reference computes them."""
        s = self.spec
        sd = self.state_dict()
        gh, gw = shape[0] // PATCH, shape[1] // PATCH
        to_dev = lambda t: t.to(dev, f32).contiguous()
        T: Dict[str, torch.Tensor] = {}
        pos = sd["pixel_encoder.pos_embed"].detach().float().reshape(-1, s.embed_dim)
        T["pos"] = to_dev(pos_table_by_size(pos, gh, gw))
        T["tokens_pos"] = tokens_pos(sd, gh, gw, s.hidden, dev)
        for i in range(3):
            mf = max(gh << i, gw << i) // 2
            T[f"ray_scales.{i}"] = to_dev(2.0 ** torch.linspace(0.0, math.log2(mf), steps=32, dtype=f32))
        return T

    def _pack_weights(self, dev):
        s = self.spec
        split, fp8, code = self._precision()
        # GEMM weight of the split mode's operands: [N, 3K] = [hi | hi | lo], or f16 in the other modes
        s16 = split_weight if split else h16
        sd = {k: v.detach() for k, v in self.state_dict().items()}
        T: Dict[str, torch.Tensor] = {}
        # an engine without "precision" runs the f16 mode, so the f16 packing registers exactly the scalars it always has
        S: Dict[str, float] = {"precision": float(code)} if code else {}
        pd, dl = "pixel_decoder.", "pixel_decoder.depth_layer."
        hid, D = s.hidden, s.embed_dim

        def kpad(w, k):
            out = torch.zeros((w.shape[0], k), dtype=f32, device=w.device)
            out[:, :w.shape[1]] = w.float()
            return out

        # ---- encoder: the shared DINOv2 packing; the position table is a shape operand
        T.update(pack_vit_encoder(sd, D, s.enc_depth, dev, split=split, fp8=fp8))
        T["norm_w"], T["norm_b"] = c32(sd["pixel_encoder.norm.weight"]), c32(sd["pixel_encoder.norm.bias"])

        # ---- adapters
        for l in range(4):
            a = f"{pd}input_adapter.input_adapters.{l}."
            adapter(T, sd, f"adapt.{l}.", a, h16)
            if split:       # the adapter's copy for the camera and global heads, which read it on split operands
                T[f"adapt.{l}.w_cam"] = split_weight(sd[a + "1.weight"])
        for dst, src, n in (("ctok", "camera_token_adapter", 4), ("gtok", "global_token_adapter", 2)):
            for i in range(n):
                adapter(T, sd, f"{dst}.{i}.", f"{pd}{src}.input_adapters.{i}.", c32)

        # ---- camera head
        cl = pd + "camera_layer."
        mlp(T, sd, "cam.cls", cl + "project_cls", c32)
        mlp(T, sd, "cam.inf", cl + "in_features", s16)
        T["cam.pos"] = c32(sd[cl + "latents_pos"].reshape(4, hid))
        cross_block(T, sd, "cam.agg1.", cl + "aggregate1.", s16)
        cross_block(T, sd, "cam.agg2.", cl + "aggregate2.", s16)
        mlp(T, sd, "cam.out", cl + "out", c32)

        # ---- global head
        gl = pd + "global_layer."
        mlp(T, sd, "glob.cls", gl + "project_cls", c32)
        T["glob.rays_w"], T["glob.rays_b"] = s16(kpad(sd[gl + "project_rays.weight"], RAY_K)), c32(sd[gl + "project_rays.bias"])
        T["glob.in_w"], T["glob.in_b"] = s16(sd[gl + "in_features.weight"]), c32(sd[gl + "in_features.bias"])
        cross_block(T, sd, "glob.agg1.", gl + "aggregate1.", s16)
        cross_block(T, sd, "glob.agg2.", gl + "aggregate2.", s16)
        mlp(T, sd, "glob.out", gl + "out", c32)

        # ---- depth head
        for i in range(3):
            T[f"rays.{i}.w"], T[f"rays.{i}.b"] = h16(kpad(sd[f"{dl}rays_layers.{i}.weight"], RAY_K)), c32(sd[f"{dl}rays_layers.{i}.bias"])
        latents(T, sd, dl)
        attn_block(T, sd, "agg16.", dl + "aggregate_16.", True)
        attn_block(T, sd, "prompt.", dl + "prompt_camera.", True)
        for j in range(s.dec_depths[0]):
            attn_block(T, sd, f"nys.{j}.", f"{dl}process_layers.0.{j}.", False)
        for i in range(3):
            c = hid >> i
            cq, c2 = c // 4, c // 2
            cqp = -(-cq // 64) * 64
            u, dst = f"{dl}ups.{i}.", f"up.{i}."
            for j in range(2):
                convnext_block(T, sd, f"{dst}c{j}.", f"{u}convs.{j}.", ("dwconv", "norm", "pwconv1", "pwconv2"))
            T[dst + "dw_w"], T[dst + "dw_b"] = c32(sd[u + "up.1.weight"].reshape(cq, 49).t()), c32(sd[u + "up.1.bias"])
            cw = torch.zeros((c2, 3, 3, cqp), dtype=f32, device=sd[u + "up.3.weight"].device)
            cw[..., :cq] = sd[u + "up.3.weight"].float().permute(0, 2, 3, 1)         # [C/2, C/4, 3, 3] -> [C/2, (ky, kx, ci)]
            T[dst + "conv_w"], T[dst + "conv_b"] = h16(cw.reshape(c2, 9 * cqp)), c32(sd[u + "up.3.bias"])
            T[dst + "res_w"], T[dst + "res_b"] = h16(sd[u + "residual.0.weight"].reshape(c2, c)), c32(sd[u + "residual.0.bias"])
            # depth_mlp / confidence_mlp: first layers apart, second layers as one block-diagonal [32, 2 * C/2] GEMM weight
            hm = f"hmlp.{i}."
            w2 = torch.zeros((32, c), dtype=f32, device=sd[u + "up.3.weight"].device)
            for k, nm in enumerate(("depth_mlp", "confidence_mlp")):
                src, p = f"{dl}{nm}.{i}.", hm + ("c." if k else "d.")
                T[p + "nw"], T[p + "nb"] = c32(sd[src + "norm.weight"]), c32(sd[src + "norm.bias"])
                T[p + "w1"], T[p + "b1"] = h16(sd[src + "proj1.weight"]), c32(sd[src + "proj1.bias"])
                w2[16 * k:16 * (k + 1), c2 * k:c2 * (k + 1)] = sd[src + "proj2.weight"].float()
            T[hm + "w2"] = h16(w2)
            T[hm + "b2"] = c32(torch.cat([sd[f"{dl}depth_mlp.{i}.proj2.bias"], sd[f"{dl}confidence_mlp.{i}.proj2.bias"]]))
        T["head_w"] = c32(torch.stack([sd[dl + "to_depth.weight"].reshape(48, 49), sd[dl + "to_confidence.weight"].reshape(48, 49)]))
        S["head_b_depth"] = float(sd[dl + "to_depth.bias"].item())
        S["head_b_conf"] = float(sd[dl + "to_confidence.bias"].item())
        return T, S

    # ------------------------------------------------------------------ engine
    def _engine_config(self, shape=None) -> "cabi.V2oldConfig":
        """udb_v2old_config_t of this model at the network shape `shape` (default: `_default_shape()`) (include/udb.h)."""
        s = self.spec
        cfg = cabi.V2oldConfig()
        cfg.embed_dim, cfg.enc_depth, cfg.enc_heads = s.embed_dim, s.enc_depth, s.enc_heads
        for i in range(4):
            cfg.output_idx[i] = s.output_idx[i]
        cfg.hidden, cfg.heads, cfg.expansion = s.hidden, s.heads, s.expansion
        cfg.nystrom_depth = s.dec_depths[0]
        cfg.net_h, cfg.net_w = shape or self._default_shape()
        return cfg

    # ------------------------------------------------------------------ infer
    @torch.no_grad()
    def infer(self, rgbs: torch.Tensor, intrinsics=None):
        """Same contract as the reference `UniDepthV2old.infer` (unidepthv2_old.py:198-282)."""
        if self.interpolation_mode not in cabi.V2OLD_INTERP_MODES:
            raise NotImplementedError(f"interpolation_mode {self.interpolation_mode!r}: only 'bilinear' and 'nearest-exact' "
                                      "are implemented")
        if rgbs.ndim == 3:
            rgbs = rgbs.unsqueeze(0)
        if intrinsics is not None and intrinsics.ndim == 2:
            intrinsics = intrinsics.unsqueeze(0)
        B, _, H, W = rgbs.shape
        level = check_resolution(self.resolution_level)
        check_ratio((H, W), self.shape_constraints["ratio_bounds"])
        shape, _ = v2old_geometry(H, W, level, self.shape_constraints["pixels_bounds_ori"])
        return self._infer(rgbs, intrinsics, shape, interpolation=cabi.V2OLD_INTERP_MODES[self.interpolation_mode])

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, inputs, image_metas=None):
        """The reference's evaluation call `model(inputs, image_metas)` (unidepthv2_old.py:134-196), in eval mode only:

            out = model({"image": x, "depth": gt, "K": K}, image_metas)    # "K" optional; image_metas is not read

        `inputs["image"]` is the network input itself: float [B, 3, h, w], already normalised, both sides multiples of 14
        (no resize, padding or normalisation here).  `inputs["depth"]` gives only its size (H, W).  A `inputs["K"]`
        [B, 3, 3] drives the rays as it is, which the reference allows only when (H, W) == (h, w).  Returns
          "K"              [B, 3, 3]   the predicted K at (h, w), also when K is given (`infer` returns the given K),
          "depth"          [B, 1, H, W] and "confidence" [B, 1, H, W], antialiased bilinear from (h, w),
          "points"         [B, 3, H, W] through the predicted K, unscaled, on the (H, W) grid, also when K is given,
          "depth_features" [B, (h/14)(w/14), 512] f32, the depth head's latents before its Nystrom blocks.
        Unlike the reference, the caller's `inputs` dict is left as it was: the reference adds "rays", "angles",
        "features", "tokens", "global_tokens" and "camera_tokens" to it.  `precision` applies as in `infer`; the outputs
        are new tensors (`output_buffers` holds `infer`'s only).  Training mode raises NotImplementedError: the training
        forward is out of scope."""
        self._check_eval_call(inputs)
        for k in ("image", "depth"):
            if k not in inputs:
                raise ValueError(f"inputs needs {k!r}: the network input and the ground truth whose size the outputs take")
        image = inputs["image"]
        B, h, w = self._network_input_shape(image)
        if not image.dtype.is_floating_point:
            raise ValueError(f"inputs['image'] must be a float tensor, not {image.dtype}")
        H, W = (int(v) for v in inputs["depth"].shape[-2:])
        K = inputs.get("K")
        if K is not None:
            if tuple(K.shape) != (B, 3, 3):
                raise ValueError(f"inputs['K'] must be [B, 3, 3] = [{B}, 3, 3], not {tuple(K.shape)}")
            if (H, W) != (h, w):
                raise ValueError(f"inputs['K'] with a ground truth of {H}x{W} and an image of {h}x{w}: the rays of K are "
                                 "reshaped to the image grid, so the two sizes must be equal")
        dev = self._cuda_device()
        x = image.to(dev, f32).contiguous()
        ins = {} if K is None else {"K": K.to(dev, f32).contiguous()}

        def run(eng, x, ins):
            # the network-only call of udb_infer_v2old on the normalised network input; maps at the ground truth's size
            feats = torch.empty((B, (h // PATCH) * (w // PATCH), self.spec.hidden), device=dev, dtype=f32)
            out = self._infer_call(eng, x, ins.get("K"), network_only=1, out_h=H, out_w=W,
                                   out_depth_features=feats.data_ptr())
            return {"K": out.pop("intrinsics"), **out, "depth_features": feats}

        key = ("forward", B, h, w, H, W, K is not None)
        return self._run_graphed(lambda: self._shape_engine((h, w)), run, x, ins, key, output_buffers=False)
