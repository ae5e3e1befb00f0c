"""UniDepthV2 -- drop-in for the reference's inference API, running on libudb.so (sm_90a).

Mirrors `unidepth.models.UniDepthV2` for the inference path only
(reference: unidepth/models/unidepthv2/unidepthv2.py:111-127 constructor, :239-339 `infer`,
:414-416 `device`, :381-394 `load_pretrained`; HF-hub mixin `from_pretrained`):

    model = UniDepthV2.from_pretrained(dir_with_config_json_and_safetensors)   # or UniDepthV2(config)
    model = model.to("cuda").eval()
    out = model.infer(rgb_uint8)        # dict: confidence intrinsics radius depth points rays depth_features

The module owns `nn.Parameter`s under exactly the reference's state-dict names, so reference
checkpoints (`model.safetensors` / `pytorch_model.bin`) load unchanged.  The forward itself is not
PyTorch: `infer` packs the weights once (f16 GEMM operands, f32 epilogue vectors) and drives the
hand-written kernels through the C ABI (include/udb.h) on torch's current stream, optionally as a
captured CUDA graph.  There is no CPU / eager fallback: a missing library or a CPU-resident model
raises.
"""
from __future__ import annotations

import ctypes as C
import math
import warnings
from typing import Dict, Optional

import torch

from . import _cabi as cabi
from ._engine_model import HUB_KWARGS, EngineModel, PyTorchModelHubMixin, f32
from ._pack import c32, h16, pack_vit_encoder
from ._pack import pack_e4m3  # noqa: F401  -- the fp8 weight quantiser stays importable from here, where callers import it
from .camera import pack_camera
from .spec import ModelSpec, PATCH, get_paddings, get_resize_factor, param_shapes, pixel_bounds


class UniDepthV2(EngineModel, PyTorchModelHubMixin, **HUB_KWARGS):
    _ENGINE_FNS = ("udb_create", "udb_destroy", "udb_set_weight", "udb_set_scalar")

    def __init__(self, config: dict, eps: float = 1e-6, **kwargs):
        super().__init__(config, eps, max_cached_workspaces=8)
        self.spec = ModelSpec(config)
        s = self.spec
        if not s.use_norm:
            raise NotImplementedError("pixel_encoder.use_norm=false is not used by any shipped UniDepthV2 config")
        self._add_params(param_shapes(config))
        self.shape_constraints = dict(s.shape_constraints)   # mutable, read by infer (unidepthv2.py:459)
        self.interpolation_mode = "bilinear"                 # unidepthv2.py:460
        # "f16": f16 GEMM / attention operands with f32 accumulation (the reference's own GPU dtype, unidepthv2.py:240).
        # "split": parity / debugging mode -- every f16 operand of the ENCODER is a hi + lo pair fed through the same
        # wgmma GEMM (three products hi.W_hi + lo.W_hi + hi.W_lo, include/udb.h udb_gemm_t.a_split_k) and attention
        # runs in fp32; ~4x slower.  It shows that the default mode's residual against the fp32 reference is operand
        # rounding: the intrinsics (fp32 camera head on the encoder's cls tokens) then meet north_star's 1e-4.
        # "fp8": speed mode -- the four linear layers of every encoder block (qkv, proj, fc1, fc2) multiply FP8 E4M3
        # operands on the e4m3 wgmma: weights with one scale per output channel, activations quantised per row on the
        # fly (include/udb.h udb_gemm_e4m3).  The patch embedding, attention and the decoder are unchanged.  Its
        # accuracy is only measured on seeded synthetic weights (tests/test_fp8_gpu.py), not on trained checkpoints.
        self.precision = "f16"
        # Fused LayerNorm (north_star: "fused LayerNorm + QKV projection"): norm1 / norm2 of the encoder blocks folded into
        # the qkv / fc1 GEMMs (include/udb.h udb_gemm_t.ln_*), no stand-alone LayerNorm pass.  f16 mode only.
        # OFF by default: it removes the LayerNorm kernels but the producers' extra f16 store + row statistics lengthen
        # the GEMM epilogues more than that saves -- measured on an H100 SXM (700 W, same run): 38.88 vs 37.74 ms per
        # 8-image ViT-L step (bench.py --fuse-ln).
        self.fuse_ln = False
        self.max_engine_shapes = 64       # per-(gh,gw) tables live inside the engine; beyond this everything is rebuilt
        self._scales_cache: Dict[tuple, torch.Tensor] = {}      # ray-embedding frequency tables: shape constants, never dropped
        self._engine_shapes: set = set()

    # ------------------------------------------------------------------ weight packing
    def _fuse(self) -> bool:
        return bool(self.fuse_ln and self.precision == "f16")

    def _fingerprint(self):
        return super()._fingerprint() + (self._fuse(),)

    def _pack_weights(self, dev):
        """({engine tensor name: tensor on `dev`}, {scalar name: float}) (names: include/udb.h, DESIGN.md 'packed
        tensors'): plain torch layout work, no kernel involved.  UniDepthV2 has no shape operands: its engine keeps its
        per-grid tables itself, so this is all of `_pack_tensors`."""
        s = self.spec
        if s.kernel_size != 3:
            raise NotImplementedError(f"pixel_decoder.kernel_size={s.kernel_size}: the residual conv units run as 3x3 "
                                      "convolutions (every shipped UniDepthV2 config sets 3)")
        sd = {k: v.detach() for k, v in self.state_dict().items()}
        split, fp8, code = self._precision()
        fuse = self._fuse()

        d, hid = s.embed_dim, s.hidden
        # The attention kernel works on 64-wide heads.  Narrower decoder heads (ViT-S: 256/8 = 32) are
        # zero-padded to 64 in the packed q / kv / out weights: padded q,k columns add 0 to q.k, padded
        # v columns produce zeros that meet zero columns of the out projection; the softmax scale stays
        # 1/sqrt(true head dim).
        hd = hid // s.dec_heads
        if d // s.enc_heads != 64 or hd > 64:
            raise NotImplementedError(f"head dims (encoder {d // s.enc_heads}, decoder {hd}) not supported")
        for cch in list(s.cur) + list(s.outd[:-1]):
            if cch % 64:
                raise NotImplementedError(f"decoder channel count {cch} is not a multiple of 64")
        # The last stage's output map (ViT-B: 96 channels) and the "lr" convs' outputs (48 / 32) are
        # zero-padded to multiples of 64 channels: zero weight rows produce zero channels, which meet
        # zero weight columns downstream; LayerNorm statistics use the real count (dim_valid).
        pad64 = lambda c: (c + 63) // 64 * 64
        c_hr_real, c_hr = s.outd[-1], pad64(s.outd[-1])
        if c_hr_real % 8 or c_hr > 256:
            raise NotImplementedError(f"high-resolution feature width {c_hr_real} not supported")
        pe = "pixel_encoder."
        T = pack_vit_encoder(sd, d, s.depth, dev, split, fuse, fp8=fp8)
        T["pos"] = c32(sd[pe + "pos_embed"].reshape(-1, d))      # the stored grid: the engine resizes it per shape
        S: Dict[str, float] = {"precision": float(code), "fuse_ln": 1.0 if fuse else 0.0}
        T["norm_w"], T["norm_b"] = c32(sd[pe + "norm.weight"]), c32(sd[pe + "norm.bias"])

        pd = "pixel_decoder."
        for l in range(4):
            a, c = f"{pd}input_adapter.input_adapters.{l}", f"{pd}camera_token_adapter.input_adapters.{l}"
            T[f"adapt.{l}.w"], T[f"adapt.{l}.b"] = h16(sd[a + ".weight"]), c32(sd[a + ".bias"])
            T[f"cam_adapt.{l}.w"], T[f"cam_adapt.{l}.b"] = c32(sd[c + ".weight"]), c32(sd[c + ".bias"])
        cl = pd + "camera_layer."

        def copy32(dst, src, names):
            for a, b in names:
                T[f"{dst}.{a}"] = c32(sd[f"{src}.{b}"])

        mlp_names = (("nw", "norm.weight"), ("nb", "norm.bias"), ("w1", "proj1.weight"), ("b1", "proj1.bias"),
                     ("w2", "proj2.weight"), ("b2", "proj2.bias"))
        T["cam.pos"] = c32(sd[cl + "latents_pos"].reshape(4, hid))
        copy32("cam.project", cl + "project", mlp_names)
        copy32("cam.pinhole", cl + "out_pinhole", mlp_names)
        for i in (1, 2):
            copy32(f"cam.agg{i}.mlp", f"{cl}aggregate{i}.mlp", mlp_names)
            copy32(f"cam.agg{i}", f"{cl}aggregate{i}", (
                ("kv", "kv.weight"), ("q", "q.weight"), ("nxw", "norm_attnx.weight"), ("nxb", "norm_attnx.bias"),
                ("ncw", "norm_attnctx.weight"), ("ncb", "norm_attnctx.bias"), ("out", "out.weight"), ("ls1", "ls1.gamma"),
                ("ls2", "ls2.gamma")))
        dl = pd + "depth_layer."
        nh_dec = s.dec_heads

        def pad_heads_rows(w):      # [heads*hd, K] -> [heads*64, K], zero rows for the padded head dims
            if hd == 64:
                return w
            out_w = torch.zeros((nh_dec, 64, w.shape[1]), device=w.device, dtype=w.dtype)
            out_w[:, :hd] = w.reshape(nh_dec, hd, w.shape[1])
            return out_w.reshape(nh_dec * 64, w.shape[1])

        def pad_heads_cols(w):      # [N, heads*hd] -> [N, heads*64]
            if hd == 64:
                return w
            out_w = torch.zeros((w.shape[0], nh_dec, 64), device=w.device, dtype=w.dtype)
            out_w[:, :, :hd] = w.reshape(w.shape[0], nh_dec, hd)
            return out_w.reshape(w.shape[0], nh_dec * 64)

        for l in range(4):
            p, dst = f"{dl}prompt_camera.{l}.layers.0", f"prompt.{l}"
            copy32(dst, p, (("nxw", "norm_attnx.weight"), ("nxb", "norm_attnx.bias"), ("ncw", "norm_attnctx.weight"),
                            ("ncb", "norm_attnctx.bias"), ("mnw", "mlp.norm.weight"), ("mnb", "mlp.norm.bias"),
                            ("b1", "mlp.proj1.bias"), ("b2", "mlp.proj2.bias")))
            kv = sd[p + ".kv.weight"]
            T[dst + ".q"] = h16(pad_heads_rows(sd[p + ".q.weight"]))
            T[dst + ".kv"] = h16(torch.cat([pad_heads_rows(kv[:hid]), pad_heads_rows(kv[hid:])], 0))
            T[dst + ".out"] = h16(pad_heads_cols(sd[p + ".out.weight"]))
            T[dst + ".w1"], T[dst + ".w2"] = h16(sd[p + ".mlp.proj1.weight"]), h16(sd[p + ".mlp.proj2.weight"])
        T["lat_w"], T["lat_b"] = h16(sd[dl + "to_latents.weight"]), c32(sd[dl + "to_latents.bias"])
        conv_pack = lambda w: h16(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1))   # [Cout,(dy,dx,ci)]
        for i in range(len(s.dec_depths)):
            k = max(1, 2 * i)
            wt = sd[f"{dl}process_features.{i}.weight"]                            # [Cin,Cout,k,k]
            cout = wt.shape[1]
            T[f"ups.{i}.ct_w"] = h16(wt.permute(2, 3, 1, 0).reshape(k * k * cout, wt.shape[0]))
            T[f"ups.{i}.ct_b"] = c32(sd[f"{dl}process_features.{i}.bias"].repeat(k * k))
            for j in range(s.dec_depths[i]):
                u, dst = f"{dl}ups.{i}.convs.{j}.", f"ups.{i}.rcu.{j}."
                T[dst + "w1"], T[dst + "b1"] = conv_pack(sd[u + "conv1.weight"]), c32(sd[u + "conv1.bias"])
                T[dst + "w2"], T[dst + "b2"] = conv_pack(sd[u + "conv2.weight"]), c32(sd[u + "conv2.bias"])
                T[dst + "gamma"] = c32(sd[u + "gamma"].reshape(-1))
            uw = sd[f"{dl}ups.{i}.up.0.weight"]
            uw, ub = uw.reshape(uw.shape[0], uw.shape[1]).float(), sd[f"{dl}ups.{i}.up.0.bias"].float()
            if uw.shape[0] % 64:            # last stage of ViT-B: 96 -> 128 output channels (zeros)
                extra = pad64(uw.shape[0]) - uw.shape[0]
                uw = torch.cat([uw, torch.zeros((extra, uw.shape[1]), device=dev)], 0)
                ub = torch.cat([ub, torch.zeros(extra, device=dev)], 0)
            T[f"ups.{i}.up_w"], T[f"ups.{i}.up_b"] = h16(uw), c32(ub)
        last = len(s.dec_depths) - 1
        # heads: LN(x) = xhat * w + b with the SAME xhat for depth and confidence, so the two
        # LN -> Linear pairs fold into one GEMM on xhat with W' = W * w (per input channel) and
        # b' = W b + bias, depth rows first then confidence rows (decoder.py:190-199, 288, 306-307)
        wm, bm = [], []
        zpad = lambda t, dim, n: t if t.shape[dim] == n else torch.cat(
            [t, torch.zeros(tuple(n - t.shape[dim] if i == dim else sz for i, sz in enumerate(t.shape)), device=dev)], dim)
        for i, (mlp_p, lr, hr, add) in enumerate(((f"{dl}depth_mlp.{last}", "to_depth_lr", "to_depth_hr", 2.0),
                                                  (f"{dl}confidence_mlp", "to_confidence_lr", "to_confidence_hr", 0.0))):
            lnw, lnb = sd[mlp_p + ".0.weight"].float(), sd[mlp_p + ".0.bias"].float()
            w, bb = sd[mlp_p + ".1.weight"].float(), sd[mlp_p + ".1.bias"].float()
            # [c_hr, c_hr] block of the merged GEMM: real rows / columns first, zero padding after
            wm.append(zpad(zpad(w * lnw.unsqueeze(0), 1, c_hr), 0, c_hr))
            bm.append(zpad(w @ lnb + bb, 0, c_hr))
            lr_w, lr_b, hr_w = sd[f"{dl}{lr}.weight"].float(), sd[f"{dl}{lr}.bias"].float(), sd[f"{dl}{hr}.0.weight"].float()
            lr_c = pad64(lr_w.shape[0])       # ViT-S: 32 -> 64, ViT-B: 48 -> 64 output channels of the lr conv
            lr_w = zpad(zpad(lr_w, 1, c_hr), 0, lr_c)
            lr_b = zpad(lr_b, 0, lr_c)
            hr_w = zpad(hr_w, 1, lr_c)
            dst = f"heads.{i}."
            T[dst + "lr_w"], T[dst + "lr_b"] = conv_pack(lr_w), c32(lr_b)
            T[dst + "hr_w"], T[dst + "hr_b"] = conv_pack(hr_w), c32(sd[f"{dl}{hr}.0.bias"])
            T[dst + "head_w"] = c32(sd[f"{dl}{hr}.2.weight"].reshape(32))
            S[dst + "head_b"], S[dst + "add"] = float(sd[f"{dl}{hr}.2.bias"].item()), add
        T["head_mlp_w"], T["head_mlp_b"] = h16(torch.cat(wm, 0)), c32(torch.cat(bm, 0))
        ones = torch.zeros(c_hr, device=dev, dtype=f32)
        ones[:c_hr_real] = 1.0               # padded channels: weight 0 -> normalised value 0
        T["ln_ones"] = ones
        T["ln_zeros"] = torch.zeros(c_hr, device=dev, dtype=f32)
        return T, S

    # ------------------------------------------------------------------ C engine (udb_create / udb_infer_v2)
    def _drop_engine(self):
        super()._drop_engine()
        self._engine_shapes = set()

    def _engine_config(self, shape=None) -> "cabi.Config":
        """udb_config_t of this model (include/udb.h).  The engine takes every network shape: `shape` is not read."""
        s, sc = self.spec, self.shape_constraints
        cfg = cabi.Config()
        cfg.embed_dim, cfg.depth, cfg.enc_heads = s.embed_dim, s.depth, s.enc_heads
        for i, t in enumerate(s.taps):
            cfg.taps[i] = t
        cfg.pos_grid = int(math.isqrt(self.pixel_encoder.pos_embed.numel() // s.embed_dim - 1))
        cfg.hidden, cfg.dec_heads, cfg.expansion, cfg.out_dim = s.hidden, s.dec_heads, s.expansion, s.out_dim
        cfg.n_stages = len(s.dec_depths)
        for i, dd in enumerate(s.dec_depths):
            cfg.dec_depths[i] = dd
        cfg.ratio_min, cfg.ratio_max = sc["ratio_bounds"]
        cfg.pixels_min, cfg.pixels_max = sc["pixels_min"], sc["pixels_max"]
        return cfg

    def _get_engine(self):
        """The engine of the current shape constraints, rebuilt when they change or once it holds the per-grid tables of
        more than `max_engine_shapes` grids (the rebuild frees them)."""
        self._weights()
        sc = self.shape_constraints
        key = (tuple(sc["ratio_bounds"]), sc["pixels_min"], sc["pixels_max"])
        if len(self._engine_shapes) > self.max_engine_shapes:
            self._drop_engine()
        if self._engine is not None and self._engine_key == key:
            return self._engine
        return self._create_engine(self._engine_config(), key)

    def _forward_engine(self, eng, rgb: torch.Tensor, geom: dict, normalize: bool, level, camera_k=None, rays_in=None,
                        camera_model=0, camera_params=None, match_pads=None):
        """The whole path as ONE C call (udb_infer_v2) of the engine `eng`: torch only allocates outputs / workspace.
        With `match_pads` (device int32 [B, 4], network-only level, geom["match_hw"]) the engine matches the outputs to
        the ground truth as `forward_test` returns them."""
        lib = cabi.lib()
        dev = rgb.device
        B, _, H, W = rgb.shape
        lvl = -1 if level is None else int(level)      # -2: network-only (identity geometry)
        g = cabi.Geometry()
        cabi.check(lib.udb_geometry(eng, H, W, lvl, C.byref(g)), "udb_geometry")
        assert (g.net_h, g.net_w) == tuple(geom["net_hw"]) and (g.pad_l, g.pad_r, g.pad_t, g.pad_b) == tuple(geom["paddings"])
        ws = self._workspace((B, H, W, lvl), lambda: lib.udb_workspace_bytes(eng, B, H, W, lvl))
        self._engine_shapes.add((g.gh, g.gw))
        hid = self.spec.hidden
        E = lambda *shape: torch.empty(shape, device=dev, dtype=f32)
        out = {"confidence": E(B, 1, H, W), "intrinsics": E(B, 3, 3), "radius": E(B, 1, H, W), "depth": E(B, 1, H, W),
               "points": E(B, 3, H, W), "rays": E(B, 3, H, W)}
        feats = E(B, g.gh, g.gw, hid)
        ma = cabi.InferMatchArgs()
        a = ma.args                        # a view into `ma`
        if match_pads is not None:
            Hm, Wm = geom["match_hw"]
            out = {"depth": E(B, 1, Hm, Wm), "points": E(B, 3, Hm, Wm), "confidence": E(B, 1, Hm, Wm),
                   "rays": E(B, 3, H, W), "intrinsics": E(B, 3, 3)}
            ma.match_h, ma.match_w, ma.match_pads = Hm, Wm, match_pads.data_ptr()
        a.rgb, a.rgb_is_u8, a.normalize = rgb.data_ptr(), int(rgb.dtype == torch.uint8), int(normalize)
        a.B, a.H, a.W, a.resolution_level = B, H, W, lvl
        a.interpolation = cabi.INTERP_MODES[geom.get("interpolation", "bilinear")]
        a.camera_k = camera_k.data_ptr() if camera_k is not None else None
        a.camera_rays = rays_in.data_ptr() if rays_in is not None else None
        a.camera_model = int(camera_model)
        a.camera_params = camera_params.data_ptr() if camera_params is not None else None
        a.ray_scales = geom["scales"].data_ptr()
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
        for k, v in out.items():
            setattr(a, k, v.data_ptr())
        a.depth_features = feats.data_ptr()
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        if match_pads is None:
            cabi.check(lib.udb_infer_v2(eng, C.byref(a), st), "udb_infer_v2")
        else:
            cabi.check(lib.udb_infer_v2_match(eng, C.byref(ma), st), "udb_infer_v2_match")
        if match_pads is None:
            out["depth_features"] = feats.permute(0, 3, 1, 2)
        return out

    @staticmethod
    def _camera_source(camera, rays_in, B, geom, dev):
        """The call's camera as (source, device tensors): source None (predicted rays), "K" ({"K": [B,3,3]}),
        ("model", UDB_CAM_*) ({"params": [B, CAM_STRIDE]}: a camera object whose rays the udb_camera_rays kernel
        generates) or "rays" ({"rays": [B, net_h*net_w, 3]}: network_forward's rays, or the host path of any other
        camera object).  Everything is validated here, before a graph is captured or replayed."""
        if camera is None:
            return (None, {}) if rays_in is None else ("rays", {"rays": rays_in})
        if isinstance(camera, torch.Tensor):
            # a (...,3,3) pinhole K (unidepthv2.py:267-279).  The reference wraps it in Pinhole/BatchCamera, shifts the
            # principal point by the paddings (`crop`, utils/camera.py:115-120) and scales it by the resize factor
            # (`resize`, :78-81); the engine does the same on the device (udb_camera_adjust_k) before its ray kernels
            # evaluate K^-1 [u,v,1] at pixel centres (Pinhole.unproject :252-263).
            assert camera.shape[-1] == 3 and camera.shape[-2] == 3, \
                "camera tensor should be of shape (..., 3, 3): assume pinhole"
            K = camera.to(dev, f32).reshape(-1, 3, 3)
            if K.shape[0] not in (1, B):
                raise ValueError(f"camera holds {K.shape[0]} intrinsics for a batch of {B} images (need 1 or {B})")
            if float(K[:, 0, 1].abs().max()) != 0.0:
                raise NotImplementedError("pinhole K with skew is not supported")
            return "K", {"K": K.expand(B, 3, 3).contiguous()}
        packed = pack_camera(camera)
        if packed is None:
            nh, nw = geom["net_hw"]
            return "rays", {"rays": UniDepthV2._camera_rays(camera, B, geom["paddings"], geom["factor"], (nh, nw), dev)}
        model, rows = packed
        if rows.shape[0] not in (1, B):
            raise ValueError(f"camera holds {rows.shape[0]} cameras for a batch of {B} images (need 1 or {B})")
        return ("model", model), {"params": rows.to(dev).expand(B, cabi.CAM_STRIDE).contiguous()}

    # ------------------------------------------------------------------ infer
    @staticmethod
    def _camera_rays(camera, B, paddings, factor, net_hw, dev):
        """`camera=` given as a camera OBJECT that `pack_camera` does not cover (the reference's `Camera` / `BatchCamera`
        family, utils/camera.py, or anything with the same three methods): the reference crops it by the
        paddings, resizes it by the factor and asks it for unit rays at network-input resolution
        (unidepthv2.py:299-303, :361-362); those rays replace the predicted ones (decoder.py:400).
        The object's own host/torch code generates the rays; they enter the kernels as a
        [B, net_h*net_w, 3] f32 tensor.  The caller's object is not mutated (the reference does)."""
        import copy
        for name in ("crop", "resize", "get_rays"):
            if not callable(getattr(camera, name, None)):
                raise TypeError(f"camera must be a (...,3,3) tensor or an object with crop/resize/get_rays (missing {name})")
        cam = copy.deepcopy(camera)
        if callable(getattr(cam, "to", None)):
            cam = cam.to(dev)
        pl, pr_, pt, pb = paddings
        cam = cam.crop(left=-pl, top=-pt, right=-pr_, bottom=-pb)
        cam = cam.resize(factor)
        nh, nw = net_hw
        rays = cam.get_rays(shapes=(B, nh, nw))
        if rays.ndim == 3:
            rays = rays.unsqueeze(0)
        assert rays.shape[-3:] == (3, nh, nw), f"camera.get_rays returned {tuple(rays.shape)}"
        if rays.shape[0] not in (1, B):
            raise ValueError(f"camera.get_rays returned {rays.shape[0]} ray maps for a batch of {B} images")
        if rays.shape[0] == 1 and B > 1:
            rays = rays.expand(B, 3, nh, nw)
        return rays.to(dev, f32).permute(0, 2, 3, 1).reshape(B, nh * nw, 3).contiguous()

    @torch.no_grad()
    def infer(self, rgb: torch.Tensor, camera=None, normalize: bool = True):
        """Same contract as the reference `UniDepthV2.infer` (unidepthv2.py:239-339)."""
        mode = self.interpolation_mode
        if mode not in cabi.INTERP_MODES:
            raise NotImplementedError(
                f"interpolation_mode {mode!r} is not supported: the reference resizes its outputs with "
                f"F.interpolate(..., align_corners=False), which accepts only 'bilinear' and 'bicubic'")
        level = getattr(self, "resolution_level", None)
        if level is None:
            warnings.warn("!! self.resolution_level not set, using default bounds !!")
        bounds = pixel_bounds(self.shape_constraints, level)
        if rgb.ndim == 3:
            rgb = rgb.unsqueeze(0)
        B, _, H, W = rgb.shape
        rgb = self._to_device_input(rgb)
        paddings, (ph, pw) = get_paddings((H, W), self.shape_constraints["ratio_bounds"])
        factor, (nh, nw) = get_resize_factor((ph, pw), bounds)
        geom = dict(paddings=paddings, padded_hw=(ph, pw), factor=factor, net_hw=(nh, nw), out_hw=(H, W), interpolation=mode)
        key = (level, tuple(self.shape_constraints["ratio_bounds"]), bounds, mode)
        return self._run(rgb, geom, level, normalize, camera, key)

    NETWORK_ONLY = -2      # udb.h: UDB_LEVEL_NETWORK_ONLY

    @torch.no_grad()
    def network_forward(self, rgbs: torch.Tensor, rays: Optional[torch.Tensor] = None):
        """The network alone, as the reference's ONNX wrappers expose it (unidepthv2/export.py:27-45 `forward(rgbs)`
        and :58-79 `forward(rgbs, rays)`): `rgbs` is the NORMALISED float network input [B,3,H,W] with H, W
        multiples of 14; no padding / resizing / cropping.  Returns (pts_3d [B,3,H,W], confidence [B,1,H,W],
        intrinsics [B,3,3])."""
        out = self._network_outputs(rgbs, rays)
        return out["points"], out["confidence"], out["intrinsics"]

    def _network_outputs(self, rgbs, rays=None):
        B, H, W = self._network_input_shape(rgbs)
        rgbs = self._to_device_input(rgbs.float())
        geom = dict(paddings=(0, 0, 0, 0), padded_hw=(H, W), factor=1.0, net_hw=(H, W), out_hw=(H, W))
        rays_in = None
        if rays is not None:
            assert tuple(rays.shape) == (B, 3, H, W), "rays must be [B,3,H,W] at the network resolution"
            rays_in = rays.to(rgbs.device, f32).permute(0, 2, 3, 1).reshape(B, H * W, 3).contiguous()
        return self._run(rgbs, geom, self.NETWORK_ONLY, False, None, ("network_only",), rays_in=rays_in)

    @staticmethod
    def _match_paddings(inputs: dict, image_metas, B: int, h: int, w: int) -> torch.Tensor:
        """The (l, r, t, b) paddings of each network input as a CPU int32 [B, 4] tensor, taken as the reference's
        `encode_decode` takes them (unidepthv2.py:344-357): the metas' "paddings" (l, t, r, b) reordered to (l, r, t, b)
        when the first meta has them, else inputs["paddings"] (4-tuples or a [B, 4] tensor), else zeros (where the
        reference raises KeyError).  Raises ValueError for a count other than B, a negative padding or a crop that
        leaves no row or column."""
        if image_metas is not None and len(image_metas) and "paddings" in image_metas[0]:
            rows = [torch.as_tensor(m["paddings"]).cpu() for m in image_metas]
            if any(r.shape != (4,) for r in rows):
                raise ValueError(f"image_metas paddings must be 4 values (l, t, r, b) each, got {[tuple(r.shape) for r in rows]}")
            pads, src = torch.stack(rows)[:, [0, 2, 1, 3]], "image_metas"
        elif inputs.get("paddings") is not None:
            pads, src = torch.as_tensor(inputs["paddings"]).cpu(), "inputs['paddings']"
        else:
            return torch.zeros((B, 4), dtype=torch.int32)
        if pads.ndim != 2 or pads.shape != (B, 4):
            raise ValueError(f"{src} holds {tuple(pads.shape)} paddings: need one (l, r, t, b) per image, [{B}, 4]")
        if pads.is_floating_point() and not torch.equal(pads, pads.trunc()):
            raise ValueError(f"{src}: paddings must be whole pixels, got {pads.tolist()}")
        pads = pads.to(torch.int64)
        if bool((pads < 0).any()):
            raise ValueError(f"{src}: paddings must be >= 0, got {pads.tolist()}")
        rows_left, cols_left = h - pads[:, 2] - pads[:, 3], w - pads[:, 0] - pads[:, 1]
        if bool((rows_left < 1).any() or (cols_left < 1).any()):
            raise ValueError(f"{src}: paddings {pads.tolist()} leave no row or column of the {h}x{w} network input")
        return pads.to(torch.int32)

    @torch.no_grad()
    def forward_test(self, inputs: dict, image_metas=None):
        """Validation forward of the reference (unidepthv2.py:134-160), on the engine: `inputs["image"]` is the data
        pipeline's normalised network input [B, 3, h, w], `inputs["depth"]` the ground truth [B, 1, H, W] whose size the
        predictions are matched to, the paddings of the network input come from the metas or `inputs["paddings"]`
        (`_match_paddings`), and an optional `inputs["camera"]` gives the rays (:361-362).  Returns depth, points and
        confidence at (H, W) (`match_gt`: crop the paddings, bilinear resize), the intrinsics of that frame
        (`match_intrinsics`) and the renormalised rays at (h, w), all from one udb_infer_v2 call.

        A camera object that `pack_camera` accepts gets its rays from the engine's camera kernel at (h, w), uncropped and
        unscaled (the reference calls get_rays(shapes=(B, h, w)) on it as given); any other object's own get_rays runs on
        the host.  CUDA graphs are cached per (B, h, w, H, W, camera source): the paddings are graph inputs, so a new
        batch with other paddings replays.  The caller's `inputs` is left unchanged."""
        image, gt = inputs["image"], inputs["depth"]
        B, h, w = self._network_input_shape(image)
        if gt.ndim != 4:
            raise ValueError(f"inputs['depth'] must be a [B, 1, H, W] ground truth, not {tuple(gt.shape)}")
        pads = self._match_paddings(inputs, image_metas, B, h, w)
        H, W = int(gt.shape[-2]), int(gt.shape[-1])
        cam, rays_in = inputs.get("camera", None), None
        if cam is not None and pack_camera(cam) is None:
            rays = cam.get_rays(shapes=(B, h, w))
            rays_in = rays.to(self._cuda_device(), f32).expand(B, 3, h, w).permute(0, 2, 3, 1).reshape(B, h * w, 3).contiguous()
            cam = None
        rgb = self._to_device_input(image.float())
        geom = dict(paddings=(0, 0, 0, 0), padded_hw=(h, w), factor=1.0, net_hw=(h, w), out_hw=(h, w), match_hw=(H, W))
        return self._run(rgb, geom, self.NETWORK_ONLY, False, cam, ("forward_test", H, W), rays_in=rays_in,
                         match_pads=pads)

    def forward(self, inputs=None, image_metas=None, *args, **kwargs):
        """Evaluation-mode `forward` of the reference dispatches to `forward_test` (unidepthv2.py:162-166);
        training is out of scope."""
        self._check_eval_call(inputs)
        return self.forward_test(inputs, image_metas)

    def _to_device_input(self, rgb):
        rgb = rgb.to(self._cuda_device())
        if rgb.dtype not in (torch.uint8, f32):
            rgb = rgb.float()
        return rgb.contiguous()

    def _run(self, rgb, geom, level, normalize, camera, key_extra, rays_in=None, match_pads=None):
        """Common tail of infer / network_forward / forward_test: camera handling, then the engine call on the CUDA graph
        cache (`_run_graphed`)."""
        B, _, H, W = rgb.shape
        dev = rgb.device
        nh, nw = geom["net_hw"]
        gh, gw = nh // PATCH, nw // PATCH
        bands = self.spec.hidden // 2
        # The frequency tables are never dropped and every graph entry owns the one it reads (`keep`), so the repack of
        # `_get_engine` below, which drops the graphs, frees none.  (A table that a repack once freed was replayed from
        # freed memory.)
        skey = (gh, gw, bands, dev.index)
        if skey not in self._scales_cache:
            # positional_embedding.py:231-233 -- computed with the same torch expression (host, once per grid)
            self._scales_cache[skey] = (2.0 ** torch.linspace(0.0, math.log2(max(gh, gw) // 2), steps=bands)).to(dev)
        scales = self._scales_cache[skey]
        geom["scales"] = scales

        source, cam = self._camera_source(camera, rays_in, B, geom, dev)
        model = source[1] if isinstance(source, tuple) else 0

        def run(eng, inp, cam):
            return self._forward_engine(eng, inp, geom, normalize, level, camera_k=cam.get("K"), rays_in=cam.get("rays"),
                                        camera_model=model, camera_params=cam.get("params"), match_pads=cam.get("pads"))

        if match_pads is not None:
            cam["pads"] = match_pads.to(dev)
        # The camera source is part of the key (a graph captured for one source reads other buffers); its values are not:
        # the entry owns static copies of the camera tensors (and of forward_test's paddings), refreshed before every
        # replay like the image.
        key = (B, H, W, rgb.dtype, bool(normalize)) + tuple(key_extra) + (source,)
        return self._run_graphed(self._get_engine, run, rgb, cam, key, keep=scales)
