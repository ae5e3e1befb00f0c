"""Static description of UniDepthV2old (DINOv2 ViT-L/14 or ViT-S/14 encoder) for the inference path: hyper-parameters
read from the reference's config format, the parameter table under the reference's state-dict names, and the shape
arithmetic of `infer` (reference: unidepth/models/unidepthv2/unidepthv2_old.py:33-92 `_check_ratio` /
`_check_resolution` / `_get_closes_num_pixels` / `_shapes`, :306-349 `build`; unidepthv2/decoder_old.py:528-585
`Decoder.build`, :89-146 `GlobalHead`, :149-229 `DepthHead`; layers/upsample.py:82-130 `ConvUpsampleShuffleResidual`)."""
from __future__ import annotations

import warnings
from collections import OrderedDict
from typing import Tuple

from .spec import PATCH, attn_decoder_shapes, vit_encoder_shapes

# encoder.py:139-193 (`dinov2_vits14`, `dinov2_vitl14`): width, blocks, heads
DINO_ARCHS = {
    "dinov2_vits14": dict(dim=384, depth=12, heads=6),
    "dinov2_vitl14": dict(dim=1024, depth=24, heads=16),
}
RESOLUTION_LEVELS = 10          # unidepthv2_old.py:29
CAMERA_DIM = 96                 # decoder_old.py:555,572: Fourier width of the ray features (32 bands x 3 axes)
RAY_FEATURES = CAMERA_DIM + 3   # cat_orig: the unit ray itself follows its Fourier features
RAY_K = 128                     # RAY_FEATURES zero-extended to the GEMM's 64-wide K step
HEAD_CHANNELS = 16              # decoder_old.py:211-222: width of each level's depth / confidence MLP output


class V2oldSpec:
    def __init__(self, config: dict):
        m = config["model"]
        enc = m["pixel_encoder"]
        name = enc["name"]
        if name not in DINO_ARCHS:
            raise NotImplementedError(f"UniDepthV2old encoder '{name}': only DINOv2 ViT-L/14 (config_v2old_vitl14.json) and "
                                      "ViT-S/14 (config_v2old_vits14.json) are implemented")
        a = DINO_ARCHS[name]
        self.encoder_name = name
        self.embed_dim, self.enc_depth, self.enc_heads = a["dim"], a["depth"], a["heads"]
        # stacking_fn "last" over the slices [0, i0), [i0, i1), ... keeps blocks output_idx - 1 (unidepthv2_old.py:236-243)
        self.output_idx = tuple(enc["output_idx"])
        if len(self.output_idx) != 4 or list(self.output_idx) != sorted(set(self.output_idx)) or self.output_idx[-1] != self.enc_depth:
            raise NotImplementedError(f"output_idx {list(self.output_idx)}: four increasing block indices ending at {self.enc_depth}")
        if enc.get("stacking_fn", "last") != "last":
            raise NotImplementedError(f"stacking_fn '{enc.get('stacking_fn')}': only 'last' is implemented")
        if not enc.get("use_norm", False):
            raise NotImplementedError("UniDepthV2old is implemented with use_norm=True (both shipped configs)")
        if enc.get("interpolate_offset", 0.0) or enc.get("num_register_tokens", 0):
            raise NotImplementedError("interpolate_offset and register tokens are not part of the shipped configs")
        dec = m["pixel_decoder"]
        self.hidden = dec["hidden_dim"]
        self.dec_depths = tuple(dec["depths"])           # Nystrom blocks per decoder level
        self.heads = m["num_heads"]
        self.expansion = m["expansion"]
        if self.hidden != 512 or self.heads != 8 or self.expansion != 4:
            raise NotImplementedError("decoder hidden_dim 512, num_heads 8, expansion 4 (both shipped configs)")
        if len(self.dec_depths) != 3 or any(d for d in self.dec_depths[1:]):
            raise NotImplementedError(f"decoder depths {list(self.dec_depths)}: Nystrom blocks at the first of three levels only")
        sc = config["data"]["shape_constraints"]
        self.ratio_bounds = tuple(sorted(sc["ratio_bounds"]))
        self.pixels_bounds = tuple(sorted(sc.get("pixels_bounds", [1400, 2400])))   # unidepthv2_old.py:344-346
        if sc.get("patch_size", PATCH) != PATCH:
            raise NotImplementedError(f"patch_size {sc['patch_size']}: DINOv2 uses {PATCH}")


def check_resolution(resolution_level) -> int:
    """unidepthv2_old.py:45-67: the level `infer` runs at, with the reference's warnings for None (level 10) and for a
    level outside [0, 10] (clipped).  The pixel count and network shape of that level are the engine's own arithmetic
    (include/udb.h udb_v2old_geometry)."""
    if resolution_level is None:
        warnings.warn("Resolution level is not set. Using max resolution. You can tradeoff resolution for speed by setting a "
                      "number in [0,10]. This can be achieved by setting model's `resolution_level` attribute.")
        resolution_level = RESOLUTION_LEVELS
    clipped = min(max(resolution_level, 0), RESOLUTION_LEVELS)
    if clipped != resolution_level:
        warnings.warn(f"Resolution level {resolution_level} is out of bounds ([0,{RESOLUTION_LEVELS}]). Clipping to {clipped}.")
    return int(clipped)


def check_ratio(image_hw: Tuple[int, int], ratio_bounds) -> None:
    """unidepthv2_old.py:33-42: an input aspect ratio outside `ratio_bounds` only warns."""
    h, w = image_hw
    image_ratio = w / h
    lo, hi = sorted(ratio_bounds)
    if image_ratio < lo or image_ratio > hi:
        warnings.warn(f"Input image ratio ({image_ratio:.3f}) is out of training distribution: {[lo, hi]}. This may lead to "
                      "unexpected results. Consider resizing/padding the image to match the training distribution.")


def param_shapes(config: dict) -> "OrderedDict[str, tuple]":
    """name -> shape of every parameter of the reference `UniDepthV2old(config)` state dict."""
    s = V2oldSpec(config)
    out: "OrderedDict[str, tuple]" = OrderedDict()
    vit_encoder_shapes(out, s.embed_dim, s.enc_depth)
    pd = "pixel_decoder."
    hid, ex, D = s.hidden, s.expansion, s.embed_dim
    ln, lin, mlp, attn_block = attn_decoder_shapes(out, ex)

    cl = pd + "camera_layer"
    attn_block(cl + ".aggregate1", hid)
    attn_block(cl + ".aggregate2", hid)
    out[cl + ".latents_pos"] = (1, 4, hid)
    mlp(cl + ".in_features", hid, 2)
    mlp(cl + ".project_cls", hid, 4)
    mlp(cl + ".out", hid, 2, 1)
    gl = pd + "global_layer"
    lin(gl + ".in_features", hid, hid)
    lin(gl + ".project_rays", hid, RAY_FEATURES)
    attn_block(gl + ".aggregate1", hid)
    attn_block(gl + ".aggregate2", hid)
    mlp(gl + ".project_cls", hid, 4)
    mlp(gl + ".out", hid, 2, 1)
    for adapter, n in (("input_adapter", 4), ("camera_token_adapter", 4), ("global_token_adapter", 2)):
        for i in range(n):
            ln(f"{pd}{adapter}.input_adapters.{i}.0", D)
            lin(f"{pd}{adapter}.input_adapters.{i}.1", hid, D)
    dl = pd + "depth_layer"
    mlp(dl + ".to_latents", hid, 2)
    lin(dl + ".features_channel_cat", hid, 4 * hid)
    attn_block(dl + ".aggregate_16", hid)
    attn_block(dl + ".prompt_camera", hid)
    for i, depth in enumerate(s.dec_depths):
        c = hid >> i
        for j in range(depth):
            attn_block(f"{dl}.process_layers.{i}.{j}", c)
        lin(f"{dl}.rays_layers.{i}", c, RAY_FEATURES)
        u = f"{dl}.ups.{i}"
        for j in range(2):
            b = f"{u}.convs.{j}"
            out[b + ".dwconv.weight"], out[b + ".dwconv.bias"] = (c, 1, 7, 7), (c,)
            ln(b + ".norm", c)
            lin(b + ".pwconv1", ex * c, c)
            lin(b + ".pwconv2", c, ex * c)
            out[b + ".gamma"] = (c,)
        out[u + ".up.1.weight"], out[u + ".up.1.bias"] = (c // 4, 1, 7, 7), (c // 4,)
        out[u + ".up.3.weight"], out[u + ".up.3.bias"] = (c // 2, c // 4, 3, 3), (c // 2,)
        out[u + ".residual.0.weight"], out[u + ".residual.0.bias"] = (c // 2, c, 1, 1), (c // 2,)
        mlp(f"{dl}.depth_mlp.{i}", c // 2, 1, HEAD_CHANNELS)
        mlp(f"{dl}.confidence_mlp.{i}", c // 2, 1, HEAD_CHANNELS)
    n_head = HEAD_CHANNELS * len(s.dec_depths)
    for nm in ("to_depth", "to_confidence"):
        out[f"{dl}.{nm}.weight"], out[f"{dl}.{nm}.bias"] = (1, n_head, 7, 7), (1,)
    out[pd + "level_embeds"] = (4, hid)
    lin(pd + "level_embed_layer.0", hid, hid)
    lin(pd + "level_embed_layer.2", hid, hid)
    ln(pd + "level_embed_layer.3", hid)
    return out
