"""Torch-fp32 functional restatement of `UniDepthV1.infer()` with the DINOv2 ViT-L/14 encoder (configs/config_v1_vitl14.json),
and its seeded weight fixture.  TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/, never by the product path.

It reuses the pieces of the other two oracles -- the DINOv2 block arithmetic of unidepth_oracle.py and the whole V1
decoder / pre- / post-processing of unidepth_v1_oracle.py -- and adds what differs in V1's DINOv2 encoder
(file:line under /root/reference/unidepth):
  models/unidepthv1/unidepthv1.py:416-428  build: the encoder factory gets interpolate_offset 0.1
  models/backbones/dinov2.py:267-304       interpolate_pos_encoding: bicubic with scale_factor ((gh+0.1)/37, (gw+0.1)/37),
                                           height first (the function's `w, h` are H and W)
  models/backbones/dinov2.py:173-178       use_norm=False (the final norm is never applied), output_idx 5, 12, 18, 24,
                                           every block's output returned
  models/unidepthv1/unidepthv1.py:322-326  each block output gets its own cls token added before the decoder's max_stack
Pinned by tests/golden/v1_vitl14_*.npz (oracle/make_golden_v1_vit.py, the unmodified reference)."""
import os
import sys
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import unidepth_v1_oracle as O1  # noqa: E402
from unidepth_oracle import _lin, _ln, _sdpa  # noqa: E402
from unidepth_v1_parts import v1_paddings, v1_postprocess, v1_preprocess, v1_shapes  # noqa: E402

PATCH = 14
INTERPOLATE_OFFSET = 0.1


def interpolate_pos_embed_offset(pos_embed: torch.Tensor, gh: int, gw: int, offset: float = INTERPOLATE_OFFSET):
    """dinov2.py:267-304 with a nonzero interpolate_offset: [1, 1+M*M, D] -> [1, 1+gh*gw, D]."""
    n = pos_embed.shape[1] - 1
    m = int(round(n ** 0.5))
    assert m * m == n
    d = pos_embed.shape[-1]
    grid = pos_embed[:, 1:].reshape(1, m, m, d).permute(0, 3, 1, 2)
    grid = F.interpolate(grid, scale_factor=((gh + offset) / m, (gw + offset) / m), mode="bicubic", antialias=False)
    assert tuple(grid.shape[-2:]) == (gh, gw)
    return torch.cat([pos_embed[:, :1], grid.permute(0, 2, 3, 1).reshape(1, gh * gw, d)], dim=1)


def vit_encoder_v1(sd: Dict[str, torch.Tensor], image: torch.Tensor, depth: int = 24, heads: int = 16):
    """DINOv2 forward as UniDepthV1 runs it: every block's output, no final norm.  Returns (enc_outs, cls_all): per block
    the patch tokens plus that block's cls token [B, gh, gw, D] and the raw cls row [B, 1, D]."""
    p = "pixel_encoder."
    b, _, hh, ww = image.shape
    gh, gw = hh // PATCH, ww // PATCH
    d = sd[p + "cls_token"].shape[-1]
    x = F.conv2d(image, sd[p + "patch_embed.proj.weight"], sd[p + "patch_embed.proj.bias"], stride=PATCH)
    x = torch.cat([sd[p + "cls_token"].expand(b, -1, -1), x.flatten(2).transpose(1, 2)], dim=1)
    x = x + interpolate_pos_embed_offset(sd[p + "pos_embed"].float(), gh, gw)
    enc_outs, cls_all = [], []
    for i in range(depth):
        bp = f"{p}blocks.{i}."
        h1 = _ln(x, sd, bp + "norm1", 1e-6)
        qkv = _lin(h1, sd, bp + "attn.qkv").view(b, -1, 3, heads, d // heads).permute(2, 0, 3, 1, 4)
        a = _sdpa(qkv[0], qkv[1], qkv[2]).transpose(1, 2).reshape(b, -1, d)
        x = x + _lin(a, sd, bp + "attn.proj") * sd[bp + "ls1.gamma"]
        h2 = _lin(F.gelu(_lin(_ln(x, sd, bp + "norm2", 1e-6), sd, bp + "mlp.fc1")), sd, bp + "mlp.fc2")
        x = x + h2 * sd[bp + "ls2.gamma"]
        enc_outs.append((x[:, 1:] + x[:, :1]).reshape(b, gh, gw, d))
        cls_all.append(x[:, :1])
    return enc_outs, cls_all


@torch.no_grad()
def infer_v1_vit(sd: Dict[str, torch.Tensor], cfg: dict, rgbs: torch.Tensor, intrinsics: Optional[torch.Tensor] = None,
                 skip_camera: bool = False, taps: Optional[dict] = None) -> Dict[str, torch.Tensor]:
    """unidepthv1.py:288-373 for config_v1_vitl14 (same pre- / post-processing and decoder as the ConvNeXt path)."""
    if rgbs.ndim == 3:
        rgbs = rgbs.unsqueeze(0)
    if intrinsics is not None and intrinsics.ndim == 2:
        intrinsics = intrinsics.unsqueeze(0)
    B, _, H, W = rgbs.shape
    if rgbs.max() > 5 or rgbs.dtype == torch.uint8:
        rgbs = rgbs.to(torch.float32).div(255)
    if rgbs.min() >= 0.0 and rgbs.max() <= 1.0:
        mean = torch.tensor(O1.IMAGENET_MEAN, dtype=rgbs.dtype).view(1, 3, 1, 1)
        std = torch.tensor(O1.IMAGENET_STD, dtype=rgbs.dtype).view(1, 3, 1, 1)
        rgbs = (rgbs - mean) / std
    net_hw = tuple(cfg["data"]["image_shape"])
    (h, w), ratio = v1_shapes((H, W), net_hw)
    pads = v1_paddings((h, w), net_hw)
    x, gt_k = v1_preprocess(rgbs, intrinsics, (h, w), pads, ratio)
    enc_outs, cls_all = vit_encoder_v1(sd, x)
    if taps is not None:
        taps["image"], taps["enc_outs"], taps["cls_all"] = x, enc_outs, cls_all
    K, outs, _ = O1.decoder_v1(sd, enc_outs, cls_all, net_hw, (5, 12, 18, 24), cfg["model"]["num_heads"], gt_k=gt_k,
                               skip_camera=skip_camera and gt_k is not None)
    pred, K_out = v1_postprocess(outs, K.clone(), net_hw, pads, ratio, (H, W))
    use_k = gt_k if gt_k is not None else K_out          # unidepthv1.py:354-356, as in infer_v1
    angles = O1.generate_rays(use_k, (H, W))[1].transpose(1, 2).reshape(B, 2, H, W)
    pts = O1.spherical_zbuffer_to_euclidean(torch.cat((angles, pred), dim=1).permute(0, 2, 3, 1)).permute(0, 3, 1, 2)
    return {"intrinsics": K_out, "points": pts, "depth": pred[:, -1:]}


def make_v1_vit_state_dict(config: dict, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded fixture for UniDepthV1 ViT-L/14: names / shapes from unidepth_b200.spec_v1.param_shapes, one generator per
    tensor seeded from (seed, index).  The recipe is fixture.make_v1_state_dict's, plus the DINOv2 entries it has no rule
    for (cls / position / register tokens, as fixture.make_state_dict draws them for V2)."""
    from unidepth_b200.spec_v1 import param_shapes as v1_param_shapes
    sd: Dict[str, torch.Tensor] = {}
    for idx, (key, shape) in enumerate(v1_param_shapes(config).items()):
        g = torch.Generator().manual_seed(seed * 1_000_003 + idx)
        n = lambda *s: torch.randn(*s, generator=g)
        u = lambda *s: torch.rand(*s, generator=g)
        leaf = key.rsplit(".", 1)[-1]
        is_norm = ("norm" in key or key.endswith((".0.weight", ".0.bias")) and "input_adapters" in key
                   or "cls_project.0." in key or "level_embed_layer.3." in key)
        if key.endswith(("mask_token", "register_tokens")):
            t = torch.zeros(*shape)                   # dead on the infer path
        elif key.endswith(("cls_token", "pos_embed")):
            t = 0.2 * n(*shape)
        elif key.endswith(("level_embeds", "latents_pos")):
            t = 0.5 * n(*shape)
        elif ".ls1.gamma" in key or ".ls2.gamma" in key:
            t = 0.3 * (0.5 + u(*shape))
        elif leaf == "gamma":
            t = 0.4 * (0.5 + u(*shape))
        elif is_norm and len(shape) == 1:
            t = 1.0 + 0.1 * n(*shape) if leaf == "weight" else 0.05 * n(*shape)
        elif leaf == "bias":
            t = 0.05 * n(*shape)
        elif leaf == "weight":
            fan_in = 1
            for s_ in shape[1:]:
                fan_in *= s_
            t = n(*shape) / fan_in ** 0.5
            if key.endswith(("camera_layer.out.proj2.weight", "out2.weight", "out4.weight", "out8.weight")):
                t = 0.3 * t
        else:
            raise KeyError(key)
        sd[key] = t.float().contiguous()
    return sd
