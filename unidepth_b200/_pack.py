"""State dict -> engine operands, in the layouts the engines read (include/udb.h): the DINOv2 encoder packer and position
tables, and the decoder packers UniDepthV1 and UniDepthV2old share (their engines share engine_common.h's
dense_attn_block, mh_attn_block, cvnxt_block and cam_mlp).  A decoder packer writes into the operand dict `T` from the
state dict `sd`, under the engine name prefix `dst` from the state-dict prefix `src`."""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F

from ._engine_model import f16, f32


def h16(t: torch.Tensor) -> torch.Tensor:
    return t.to(f16).contiguous()


def c32(t: torch.Tensor) -> torch.Tensor:
    return t.to(f32).contiguous()


def split_weight(w: torch.Tensor) -> torch.Tensor:
    """GEMM weight [N, K] of the split-precision mode: [N, 3K] = [hi | hi | lo] f16 with hi = f16(w), lo = f16(w - hi)
    (include/udb.h udb_gemm_t.a_split_k)."""
    w = w.to(f32)
    hi = w.to(f16)
    lo = (w - hi.to(f32)).to(f16)
    return torch.cat([hi, hi, lo], dim=1).contiguous()


def pack_e4m3(w: torch.Tensor):
    """A GEMM weight [N, K] as FP8 E4M3 with one f32 scale per output channel: (w8, s) with s = amax / 448 (1 for an
    all-zero row) and w8 = e4m3(w * (448 / amax)), rounded to nearest even; w ~= w8 * s.  The same arithmetic as the
    engine's activation quantisers (include/udb.h udb_quantize_rows_e4m3)."""
    w = w.to(f32)
    amax = w.abs().amax(dim=1)
    nz = amax > 0
    one = torch.ones_like(amax)
    # a tensor division (correctly rounded, as on the device): `448.0 / amax` would be computed as amax.reciprocal() * 448
    inv = torch.where(nz, torch.full_like(amax, 448.0) / torch.where(nz, amax, one), one)
    s = torch.where(nz, amax / 448.0, one)
    return (w * inv[:, None]).to(torch.float8_e4m3fn).contiguous(), s.contiguous()


def pack_vit_encoder(sd: dict, d: int, depth: int, dev, split: bool = False, fuse: bool = False,
                     pe: str = "pixel_encoder.", fp8: bool = False) -> Dict[str, torch.Tensor]:
    """Operands of the DINOv2 encoder (patch embedding, cls token, `depth` blocks) from the reference state dict `sd`,
    under their engine names (`patch_w`, `cls`, `blocks.{i}.qkv_w`, ...) and in the layouts the engines' shared block
    loop reads (engine_common.h `vit_blocks`).  The position table is not among them: each model resizes the stored grid
    its own way (`pos_table_by_scale`, `pos_table_by_size`).  `split`: GEMM weights as `split_weight` pairs.  `fp8`: the
    blocks' four linear layers are packed as e4m3 weights with per-output-channel scales (`blocks.{i}.qkv_w8`,
    `qkv_w8s`, ...; `pack_e4m3`)."""
    enc16 = split_weight if split else h16

    def ln_fold(w, b, lnw, lnb):
        """LayerNorm folded into the Linear that follows it:  LN(x) W^T + b = rstd (x W'^T - mean c1) + c2  with
        W' = W diag(ln_w) (f16, what the MMA multiplies), c1 = row sums of the ROUNDED W', c2 = W ln_b + b."""
        w, b, lnw, lnb = w.float(), b.float(), lnw.float(), lnb.float()
        wf = (w * lnw.unsqueeze(0)).to(f16)
        return wf.contiguous(), wf.float().sum(dim=1).contiguous(), (w @ lnb + b).contiguous()

    T: Dict[str, torch.Tensor] = {}
    wpe = torch.zeros((d, 640), device=dev, dtype=f32)
    wpe[:, :588] = sd[pe + "patch_embed.proj.weight"].reshape(d, 588).to(f32)
    T["patch_w"], T["patch_b"] = enc16(wpe), c32(sd[pe + "patch_embed.proj.bias"])
    T["cls"] = c32(sd[pe + "cls_token"].reshape(d))
    for i in range(depth):
        b = f"{pe}blocks.{i}."
        if fuse:
            qw, qc1, qc2 = ln_fold(sd[b + "attn.qkv.weight"], sd[b + "attn.qkv.bias"], sd[b + "norm1.weight"], sd[b + "norm1.bias"])
            fw, fc1, fc2 = ln_fold(sd[b + "mlp.fc1.weight"], sd[b + "mlp.fc1.bias"], sd[b + "norm2.weight"], sd[b + "norm2.bias"])
            blk = dict(
                qkv_wf=qw, qkv_c1=qc1, qkv_c2=qc2, fc1_wf=fw, fc1_c1=fc1, fc1_c2=fc2,
                proj_w=h16(sd[b + "attn.proj.weight"]), proj_b=c32(sd[b + "attn.proj.bias"]), ls1=c32(sd[b + "ls1.gamma"]),
                fc2_w=h16(sd[b + "mlp.fc2.weight"]), fc2_b=c32(sd[b + "mlp.fc2.bias"]), ls2=c32(sd[b + "ls2.gamma"]))
        elif fp8:
            blk = dict(n1w=c32(sd[b + "norm1.weight"]), n1b=c32(sd[b + "norm1.bias"]), qkv_b=c32(sd[b + "attn.qkv.bias"]),
                       proj_b=c32(sd[b + "attn.proj.bias"]), ls1=c32(sd[b + "ls1.gamma"]),
                       n2w=c32(sd[b + "norm2.weight"]), n2b=c32(sd[b + "norm2.bias"]), fc1_b=c32(sd[b + "mlp.fc1.bias"]),
                       fc2_b=c32(sd[b + "mlp.fc2.bias"]), ls2=c32(sd[b + "ls2.gamma"]))
            for k, src in (("qkv", "attn.qkv"), ("proj", "attn.proj"), ("fc1", "mlp.fc1"), ("fc2", "mlp.fc2")):
                blk[k + "_w8"], blk[k + "_w8s"] = pack_e4m3(sd[b + src + ".weight"])
        else:
            blk = dict(
                n1w=c32(sd[b + "norm1.weight"]), n1b=c32(sd[b + "norm1.bias"]),
                qkv_w=enc16(sd[b + "attn.qkv.weight"]), qkv_b=c32(sd[b + "attn.qkv.bias"]),
                proj_w=enc16(sd[b + "attn.proj.weight"]), proj_b=c32(sd[b + "attn.proj.bias"]),
                ls1=c32(sd[b + "ls1.gamma"]),
                n2w=c32(sd[b + "norm2.weight"]), n2b=c32(sd[b + "norm2.bias"]),
                fc1_w=enc16(sd[b + "mlp.fc1.weight"]), fc1_b=c32(sd[b + "mlp.fc1.bias"]),
                fc2_w=enc16(sd[b + "mlp.fc2.weight"]), fc2_b=c32(sd[b + "mlp.fc2.bias"]),
                ls2=c32(sd[b + "ls2.gamma"]))
        for k, v in blk.items():
            T[f"blocks.{i}.{k}"] = v
    return T


# ---------------------------------------------------------------------------------------------- position tables
# DINOv2's interpolate_pos_encoding (dinov2.py:267-304) resizes the stored M x M grid to the gh x gw patch grid.  With a
# nonzero interpolate_offset (UniDepthV1) it passes scale factors, without one (UniDepthV2old) the target size; the two
# sample at different positions (DESIGN.md, V1 ViT table), so each model keeps its own.  Both map pos [1 + M*M, D] to
# [1 + gh*gw, D], cls row first, and are constants of the weights and the network shape.

def pos_table_by_scale(pos: torch.Tensor, gh: int, gw: int, offset: float) -> torch.Tensor:
    """Bicubic resize with scale factors ((gh + offset) / M, (gw + offset) / M), height first, so the sampling positions
    use 1 / scale_factor rather than M / gh."""
    D = pos.shape[1]
    M = math.isqrt(pos.shape[0] - 1)
    grid = pos[1:].float().reshape(1, M, M, D).permute(0, 3, 1, 2)
    g = F.interpolate(grid, scale_factor=((gh + offset) / M, (gw + offset) / M), mode="bicubic", antialias=False)
    if tuple(g.shape[-2:]) != (gh, gw):
        raise ValueError(f"position grid resized to {tuple(g.shape[-2:])}, expected {(gh, gw)}")
    return torch.cat([pos[:1].float(), g.permute(0, 2, 3, 1).reshape(gh * gw, D)], dim=0)


def pos_table_by_size(pos: torch.Tensor, gh: int, gw: int) -> torch.Tensor:
    """Bicubic resize to the size (gh, gw) (interpolate_offset 0)."""
    D = pos.shape[1]
    M = math.isqrt(pos.shape[0] - 1)
    grid = pos[1:].reshape(1, M, M, D).permute(0, 3, 1, 2)
    g = F.interpolate(grid, size=(gh, gw), mode="bicubic", antialias=False)
    return torch.cat([pos[:1], g.permute(0, 2, 3, 1).reshape(gh * gw, D)], dim=0)


# ---------------------------------------------------------------------------------------------- UniDepthV1-family decoder
def tokens_pos(sd: dict, h: int, w: int, hid: int, dev) -> torch.Tensor:
    """The operand "tokens_pos" [4*h*w, hid] f32 on `dev`: the sine position embedding of an all-valid h x w grid plus
    the level embedding MLP of the four learned level vectors (decoder.py:410-433, decoder_old.py:463-479).  The
    embedding is PositionEmbeddingSine(hid // 2, normalize=True) (layers/positional_encoding.py:15-59: y features then x
    features, sin on even / cos on odd feature indices).  A constant of the weights and the grid, evaluated when the
    engine for a network shape is made."""
    pd = "pixel_decoder."
    le = F.linear(F.gelu(F.linear(sd[pd + "level_embeds"].float(), sd[pd + "level_embed_layer.0.weight"].float(),
                                  sd[pd + "level_embed_layer.0.bias"].float())),
                  sd[pd + "level_embed_layer.2.weight"].float(), sd[pd + "level_embed_layer.2.bias"].float())
    le = F.layer_norm(le, (hid,), sd[pd + "level_embed_layer.3.weight"].float(), sd[pd + "level_embed_layer.3.bias"].float(), 1e-5)
    num_pos_feats, device = hid // 2, le.device
    eps, scale = 1e-6, 2 * math.pi
    y = torch.arange(1, h + 1, dtype=f32, device=device)[:, None].expand(h, w) / (h + eps) * scale
    x = torch.arange(1, w + 1, dtype=f32, device=device)[None, :].expand(h, w) / (w + eps) * scale
    dim_t = torch.arange(num_pos_feats, dtype=f32, device=device)
    dim_t = 10000.0 ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)
    px, py = x[..., None] / dim_t, y[..., None] / dim_t
    px = torch.stack((px[..., 0::2].sin(), px[..., 1::2].cos()), dim=3).flatten(2)
    py = torch.stack((py[..., 0::2].sin(), py[..., 1::2].cos()), dim=3).flatten(2)
    sine = torch.cat((py, px), dim=2).reshape(h * w, 2 * num_pos_feats)
    return (sine[None, :, :] + le[:, None, :]).reshape(4 * h * w, hid).to(dev, f32).contiguous()


def adapter(T, sd, dst, src, w16):
    """An input / token adapter (LayerNorm then Linear, `src` "0." and "1."): f32 LayerNorm and bias, the weight
    packed by `w16` (h16 for a GEMM operand, c32 for the CUDA-core path of the cls tokens)."""
    T[dst + "ln_w"], T[dst + "ln_b"] = c32(sd[src + "0.weight"]), c32(sd[src + "0.bias"])
    T[dst + "w"], T[dst + "b"] = w16(sd[src + "1.weight"]), c32(sd[src + "1.bias"])


def mlp(T, sd, dst, src, w16):
    """An Mlp (norm, proj1, GELU, proj2): f32 LayerNorm and biases, the two weights packed by `w16` (c32 for the
    CUDA-core path of the camera head, h16 or split_weight for a GEMM)."""
    T[dst + ".nw"], T[dst + ".nb"] = c32(sd[src + ".norm.weight"]), c32(sd[src + ".norm.bias"])
    T[dst + ".w1"], T[dst + ".b1"] = w16(sd[src + ".proj1.weight"]), c32(sd[src + ".proj1.bias"])
    T[dst + ".w2"], T[dst + ".b2"] = w16(sd[src + ".proj2.weight"]), c32(sd[src + ".proj2.bias"])


def cross_block(T, sd, dst, src, kv_w):
    """A single-head AttentionBlock of the camera / global head: f32 operands of the CUDA-core path; the (k | v) weight,
    which a GEMM over the long context may read, packed by `kv_w`."""
    for a, b in (("nxw", "norm_attnx.weight"), ("nxb", "norm_attnx.bias"), ("ncw", "norm_attnctx.weight"),
                 ("ncb", "norm_attnctx.bias"), ("q_w", "q.weight"), ("q_b", "q.bias"), ("kv_b", "kv.bias"),
                 ("out_w", "out.weight"), ("out_b", "out.bias"), ("ls1", "ls1.gamma"), ("ls2", "ls2.gamma")):
        T[dst + a] = c32(sd[src + b])
    T[dst + "kv_w"] = kv_w(sd[src + "kv.weight"])
    mlp(T, sd, dst + "mlp", src + "mlp", c32)


def attn_block(T, sd, dst, src, split_kv):
    """The depth head's AttentionBlock / NystromBlock (engine_common.h dense_attn_block, mh_attn_block): f16 weights,
    f32 norms, biases and layer scales."""
    for a, b in (("nxw", "norm_attnx.weight"), ("nxb", "norm_attnx.bias"), ("ncw", "norm_attnctx.weight"),
                 ("ncb", "norm_attnctx.bias"), ("q_b", "q.bias"), ("out_b", "out.bias"), ("ls1", "ls1.gamma"),
                 ("ls2", "ls2.gamma"), ("mnw", "mlp.norm.weight"), ("mnb", "mlp.norm.bias"), ("mb1", "mlp.proj1.bias"),
                 ("mb2", "mlp.proj2.bias")):
        T[dst + a] = c32(sd[src + b])
    for a, b in (("q_w", "q.weight"), ("out_w", "out.weight"), ("mw1", "mlp.proj1.weight"), ("mw2", "mlp.proj2.weight")):
        T[dst + a] = h16(sd[src + b])
    kvw, kvb = sd[src + "kv.weight"], sd[src + "kv.bias"]
    d = kvw.shape[1]
    if split_kv:       # dense single-head blocks: k and v projections are separate GEMM operands
        T[dst + "k_w"], T[dst + "k_b"] = h16(kvw[:d]), c32(kvb[:d])
        T[dst + "v_w"], T[dst + "v_b"] = h16(kvw[d:]), c32(kvb[d:])
    else:
        T[dst + "kv_w"], T[dst + "kv_b"] = h16(kvw), c32(kvb)


def convnext_block(T, sd, dst, src, conv_names, e4m3=False, enc16=h16):
    """ConvNeXt block operands: depthwise weights tap-major [49, C] f32, MLP weights f16 (`enc16`: split in the
    encoder's split mode), or e4m3 with per-output-channel scales (`w1_8` / `w1_8s`, `w2_8` / `w2_8s`; pack_e4m3) for
    a block of the fp8 mode.  `conv_names`: the state-dict names of the depthwise conv, norm and the two pointwise
    layers."""
    dw, norm, fc1, fc2 = conv_names
    w = sd[f"{src}{dw}.weight"]
    T[dst + "dw_w"] = c32(w.reshape(w.shape[0], 49).t())
    T[dst + "dw_b"] = c32(sd[f"{src}{dw}.bias"])
    T[dst + "ln_w"], T[dst + "ln_b"] = c32(sd[f"{src}{norm}.weight"]), c32(sd[f"{src}{norm}.bias"])
    T[dst + "b1"], T[dst + "b2"] = c32(sd[f"{src}{fc1}.bias"]), c32(sd[f"{src}{fc2}.bias"])
    if e4m3:
        T[dst + "w1_8"], T[dst + "w1_8s"] = pack_e4m3(sd[f"{src}{fc1}.weight"])
        T[dst + "w2_8"], T[dst + "w2_8s"] = pack_e4m3(sd[f"{src}{fc2}.weight"])
    else:
        T[dst + "w1"], T[dst + "w2"] = enc16(sd[f"{src}{fc1}.weight"]), enc16(sd[f"{src}{fc2}.weight"])
    T[dst + "gamma"] = c32(sd[f"{src}gamma"])


def latents(T, sd, dl):
    """The depth head's features_channel_cat and to_latents: f16 GEMM weights, f32 norms and biases."""
    T["fcc_w"], T["fcc_b"] = h16(sd[dl + "features_channel_cat.weight"]), c32(sd[dl + "features_channel_cat.bias"])
    mlp(T, sd, "lat", dl + "to_latents", h16)
