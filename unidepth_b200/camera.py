"""Camera models accepted by `UniDepthV2.infer(rgb, camera=...)` (SURVEY section 8 rows a19 / f1).

Host-side mirror of the reference's `unidepth/utils/camera.py` interface: same class names, parameter layouts,
in-place `crop` / `resize` semantics and the same `get_rays` / `unproject` / `project` / `reconstruct` results, so
that the README's second usage (`model.infer(rgb, Pinhole(K=K))`, README.md:140-156) works unchanged:

    reference class (camera.py)      here           params
    Camera            :30-226        Camera         fx fy cx cy ...
    Pinhole           :229-273       Pinhole        fx fy cx cy                      (or K)
    EUCM              :276-328       EUCM           fx fy cx cy alpha beta
    Spherical         :331-409       Spherical      fx fy cx cy W H hfov/2 vfov/2    (equirectangular)
    OPENCV            :412-694       OPENCV         fx fy cx cy k1..k6 p1 p2 s1..s4  (k4..k6 must be 0)
    Fisheye624        :697-974       Fisheye624     fx fy cx cy k1..k6 p1 p2 s1..s4
    MEI               :977-1142      MEI            fx fy cx cy k1 k2 p1 p2 xi
    BatchCamera       :1145-1308     BatchCamera    a batch of the above, params padded to 16

The GT-camera branch of `infer` does not run the torch code below: `pack_camera` turns an object of these classes
(or a BatchCamera of one of them) into a model id and rows of parameters, and the `udb_camera_rays` kernel evaluates
the same crop / resize / unproject / get_rays arithmetic on the GPU.  Any other object (the reference's own classes,
duck-typed cameras, mixed-model batches, the 15-parameter layout, non-fp32 parameters) still goes through its own
methods on the host (`unidepthv2.py::_camera_rays`); every op below is a small torch op on the device the parameters
live on.  The closed-form models (Pinhole, EUCM, Spherical, every `project`) are pinned to
the reference's outputs (tests/golden/cameras.npz, made by oracle/make_golden_cameras.py).  The three models whose
`unproject` has no closed form (OPENCV, Fisheye624, MEI) invert the SAME forward distortion, but with one shared
damped-Newton solver run to convergence instead of the reference's per-class trust-region loops, which stop at a
residual of 1e-3 (camera.py:497,630; 779,906): they agree with the reference to within that stopping tolerance and
are additionally tested by the round trip project(unproject(uv)) == uv.
"""
from __future__ import annotations

import copy
import math
from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

__all__ = ["Camera", "Pinhole", "EUCM", "Spherical", "OPENCV", "Fisheye624", "MEI", "BatchCamera", "pixel_grid",
           "invert_pinhole", "pack_camera"]

_PAD = 16          # parameter vector length inside a BatchCamera (camera.py:156-167)


def pixel_grid(b: int, h: int, w: int, homogeneous: bool = False, device=None, noisy: bool = False) -> torch.Tensor:
    """[b, 2|3, h, w] pixel-centre coordinates (u + 0.5, v + 0.5[, 1]) (utils/coordinate.py:4-20)."""
    xs = torch.linspace(0.5, w - 0.5, w, device=device)
    ys = torch.linspace(0.5, h - 0.5, h, device=device)
    if noisy:                                  # +-0.5 px jitter per column / row
        xs = xs + torch.rand_like(xs) - 0.5
        ys = ys + torch.rand_like(ys) - 0.5
    planes = [xs[None, :].expand(h, w), ys[:, None].expand(h, w)]
    if homogeneous:
        planes.append(torch.ones(h, w, device=device))
    return torch.stack(planes, 0).float()[None].repeat(b, 1, 1, 1)


def invert_pinhole(K: torch.Tensor) -> torch.Tensor:
    """Analytic inverse of a skew-free pinhole matrix (camera.py:16-27)."""
    inv = torch.zeros_like(K)
    inv[..., 0, 0] = 1.0 / K[..., 0, 0]
    inv[..., 1, 1] = 1.0 / K[..., 1, 1]
    inv[..., 0, 2] = -K[..., 0, 2] / K[..., 0, 0]
    inv[..., 1, 2] = -K[..., 1, 2] / K[..., 1, 1]
    inv[..., 2, 2] = 1.0
    return inv


def _flat(x: torch.Tensor) -> Tuple[torch.Tensor, Tuple[int, int, int]]:
    """[B, C, H, W] -> [B, H*W, C]."""
    b, c, h, w = x.shape
    return x.permute(0, 2, 3, 1).reshape(b, h * w, c), (b, h, w)


def _unflat(x: torch.Tensor, bhw: Tuple[int, int, int]) -> torch.Tensor:
    b, h, w = bhw
    return x.reshape(b, h, w, x.shape[-1]).permute(0, 3, 1, 2)


def _no_autocast(fn):
    """The reference computes camera geometry in fp32 whatever autocast context `infer` opened (camera.py:238 etc.)."""
    return torch.autocast(device_type="cuda", enabled=False)(fn)


# ------------------------------------------------------------------------------------------------------------------
# Tangential + thin-prism distortion shared by OPENCV / Fisheye624 / MEI:  d(x, y) = (x, y) + tangential + prism
# with r2 = x^2 + y^2, tangential = ((2x^2 + r2) p0 + 2xy p1, (2y^2 + r2) p1 + 2xy p0), prism = (s0 r2 + s1 r2^2,
# s2 r2 + s3 r2^2)  (camera.py:449-476).
def _tan_prism(xy: torch.Tensor, p: torch.Tensor, s: Optional[torch.Tensor], jac: bool = False):
    """xy [B,N,2]; p [B,2]; s [B,4] or None.  Returns d(xy) and, if asked, its 2x2 Jacobian as (j00, j01, j10, j11)."""
    x, y = xy[..., 0], xy[..., 1]
    p0, p1 = p[:, 0:1], p[:, 1:2]
    r2 = x * x + y * y
    dx = x + (2.0 * x * x + r2) * p0 + 2.0 * x * y * p1
    dy = y + (2.0 * y * y + r2) * p1 + 2.0 * x * y * p0
    if s is not None:
        s0, s1, s2, s3 = (s[:, i:i + 1] for i in range(4))
        dx = dx + s0 * r2 + s1 * r2 * r2
        dy = dy + s2 * r2 + s3 * r2 * r2
    out = torch.stack([dx, dy], -1)
    if not jac:
        return out
    j00 = 1.0 + 6.0 * x * p0 + 2.0 * y * p1
    off = 2.0 * (x * p1 + y * p0)
    j01, j10 = off, off
    j11 = 1.0 + 6.0 * y * p1 + 2.0 * x * p0
    if s is not None:
        t1 = 2.0 * (s0 + 2.0 * s1 * r2)
        t2 = 2.0 * (s2 + 2.0 * s3 * r2)
        j00, j01 = j00 + x * t1, j01 + y * t1
        j10, j11 = j10 + x * t2, j11 + y * t2
    return out, (j00, j01, j10, j11)


def _undo_tan_prism(target: torch.Tensor, p: torch.Tensor, s: Optional[torch.Tensor], iters: int = 10) -> torch.Tensor:
    """Solve d(xy) = target by Newton from xy = target (the distortion is a small perturbation of the identity)."""
    xy = target.clone()
    for _ in range(iters):
        est, (a, b, c, d) = _tan_prism(xy, p, s, jac=True)
        ex, ey = target[..., 0] - est[..., 0], target[..., 1] - est[..., 1]
        det = a * d - b * c
        xy = xy + torch.stack([(d * ex - b * ey) / det, (a * ey - c * ex) / det], -1)
    return xy


def _undo_radial(rd: torch.Tensor, coeffs: torch.Tensor, iters: int = 25) -> torch.Tensor:
    """Solve t * (1 + sum_i c_i t^(2i+2)) = rd for t >= 0 (rd [B,N,1], coeffs [B,n]).  Newton steps, each clamped to
    +-0.25 and to t >= 0 so that a far-off-axis pixel of a strongly distorting lens cannot jump over the first
    extremum of the polynomial; converges quadratically everywhere the model is monotonic."""
    n = coeffs.shape[1]
    c = coeffs[:, None, :]                                                     # [B,1,n]
    odd = torch.arange(n, device=rd.device, dtype=rd.dtype) * 2.0 + 3.0        # d/dt of t^(2i+3)
    t = rd.clone()
    for _ in range(iters):
        t2 = t * t
        pw = torch.cumprod(t2.expand(-1, -1, n), dim=-1)                       # t^2, t^4, ...
        f = t * (1.0 + (pw * c).sum(-1, keepdim=True)) - rd
        df = 1.0 + (pw * c * odd).sum(-1, keepdim=True)
        df = torch.where(df.abs() < 1e-6, torch.full_like(df, 1e-6), df)
        t = (t - (f / df).clamp(-0.25, 0.25)).clamp(min=0.0)
    return t


class Camera:
    """Base class: parameter storage, the pixel-space edits `infer` applies (crop, resize), ray generation, and the
    torch.cat / torch.stack protocol that builds a BatchCamera (camera.py:30-226)."""

    def __init__(self, params: torch.Tensor, K: Optional[torch.Tensor] = None):
        params = torch.as_tensor(params)
        if params.ndim == 1:
            params = params[None]
        if K is None:
            K = torch.eye(3, device=params.device, dtype=params.dtype).repeat(params.shape[0], 1, 1)
            K[..., 0, 0], K[..., 1, 1] = params[..., 0], params[..., 1]
            K[..., 0, 2], K[..., 1, 2] = params[..., 2], params[..., 3]
        self.params = params
        self.K = K
        self.overlap_mask = None
        self.projection_mask = None

    # ---- model-specific
    def project(self, xyz: torch.Tensor) -> torch.Tensor:
        raise NotImplementedError

    def unproject(self, uv: torch.Tensor) -> torch.Tensor:
        raise NotImplementedError

    # ---- shared behaviour
    def get_projection_mask(self):
        return self.projection_mask

    def get_overlap_mask(self):
        return self.overlap_mask

    def get_rays(self, shapes: Sequence[int], noisy: bool = False) -> torch.Tensor:
        """Unit rays through the pixel centres of an (h, w) image: [b_cameras, 3, h, w] (camera.py:88-92)."""
        _, h, w = shapes
        rays = self.unproject(pixel_grid(1, h, w, device=self.K.device, noisy=noisy))
        return rays / rays.norm(dim=1, keepdim=True).clamp(min=1e-4)

    def get_pinhole_rays(self, shapes: Sequence[int], noisy: bool = False) -> torch.Tensor:
        b, h, w = shapes
        uv1 = pixel_grid(b, h, w, homogeneous=True, device=self.K.device, noisy=noisy)
        rays = (invert_pinhole(self.K) @ uv1.reshape(b, 3, -1)).reshape(b, 3, h, w)
        return rays / rays.norm(dim=1, keepdim=True).clamp(min=1e-4)

    def reconstruct(self, depth: torch.Tensor) -> torch.Tensor:
        """z-depth map -> points (assumes z > 0) (camera.py:69-76)."""
        rays = self.unproject(pixel_grid(1, depth.shape[-2], depth.shape[-1], device=depth.device))
        return rays / rays[:, -1:].clamp(min=1e-4) * depth.clamp(min=1e-4)

    def resize(self, factor: float) -> "Camera":
        self.K[..., :2, :] *= factor
        self.params[..., :4] *= factor
        return self

    def crop(self, left, top, right=None, bottom=None) -> "Camera":
        self.K[..., 0, 2] -= left
        self.K[..., 1, 2] -= top
        self.params[..., 2] -= left
        self.params[..., 3] -= top
        return self

    def flip(self, H, W, direction: str = "horizontal") -> "Camera":
        cx = W - self.params[:, 2] if direction == "horizontal" else self.params[:, 2]
        cy = H - self.params[:, 3] if direction == "vertical" else self.params[:, 3]
        self.params = torch.stack([self.params[:, 0], self.params[:, 1], cx, cy], dim=1)
        self.K[..., 0, 2], self.K[..., 1, 2] = cx, cy
        return self

    def to(self, device, non_blocking: bool = False) -> "Camera":
        self.params = self.params.to(device, non_blocking=non_blocking)
        self.K = self.K.to(device, non_blocking=non_blocking)
        return self

    def clone(self) -> "Camera":
        return copy.deepcopy(self)

    def get_new_fov(self, new_shape, original_shape):
        hf = 2 * torch.atan(self.params[..., 2] / self.params[..., 0] * new_shape[1] / original_shape[1])
        vf = 2 * torch.atan(self.params[..., 3] / self.params[..., 1] * new_shape[0] / original_shape[0])
        return hf, vf

    def mask_overlap_projection(self, projected: torch.Tensor) -> torch.Tensor:
        """Pixels whose projection flow folds over another part of the image (camera.py:132-154): sample the flow a
        tenth of the way along itself and flag where it is longer there than what is left of the local flow."""
        b, _, h, w = projected.shape
        ident = pixel_grid(b, h, w, device=projected.device)
        flow = projected - ident
        gamma = 0.1
        at = gamma * flow + ident
        grid = torch.stack([at[:, 0] / (w - 1) * 2 - 1, at[:, 1] / (h - 1) * 2 - 1], dim=-1)
        there = F.grid_sample(flow, grid, mode="bilinear", align_corners=False, padding_mode="border")
        here_n = flow.norm(dim=1, keepdim=True)
        return ((1 - gamma) * here_n < there.norm(dim=1, keepdim=True)) | (here_n < 1)

    def _set_projection_mask(self, uv: torch.Tensor, extra_invalid: Optional[torch.Tensor] = None):
        h, w = uv.shape[-2:]
        bad = (uv[:, 0] < 0) | (uv[:, 0] > w) | (uv[:, 1] < 0) | (uv[:, 1] > h)      # u == W / v == H still count as inside
        if extra_invalid is not None:
            bad = bad | extra_invalid
        self.projection_mask = (~bad).unsqueeze(1)

    def _padded_params(self) -> torch.Tensor:
        n = self.params.shape[1]
        if n >= _PAD:
            return self.params
        return torch.cat([self.params, self.params.new_zeros(self.params.shape[0], _PAD - n)], dim=1)

    # ---- torch.cat / torch.stack / torch.flatten over camera objects -> BatchCamera (camera.py:169-209)
    @staticmethod
    def flatten_cameras(cameras) -> List["Camera"]:
        flat: List[Camera] = []
        for cam in cameras:
            if isinstance(cam, BatchCamera):
                flat.extend(Camera.flatten_cameras(cam.cameras))
            elif isinstance(cam, (list, tuple)):
                flat.extend(cam)
            else:
                flat.append(cam)
        return flat

    @staticmethod
    def _merge(cameras, func, **kwargs) -> "BatchCamera":
        flat = Camera.flatten_cameras(cameras)
        K = func([c.K for c in flat], **kwargs)
        params = func([c._padded_params() for c in flat], **kwargs)
        return BatchCamera(params, K, [type(c).__name__ for c in flat], flat)

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func is torch.cat or func is torch.stack:
            return Camera._merge(args[0], func, **kwargs)
        if func is torch.flatten:
            return Camera._merge(args[0], torch.cat, **kwargs)
        return NotImplemented

    @property
    def device(self):
        return self.K.device

    @property
    def hfov(self):
        return 2 * torch.atan(self.params[..., 2] / self.params[..., 0])

    @property
    def vfov(self):
        return 2 * torch.atan(self.params[..., 3] / self.params[..., 1])

    @property
    def max_fov(self):
        return 150.0 / 180.0 * math.pi, 150.0 / 180.0 * math.pi


class Pinhole(Camera):
    """params fx fy cx cy, or a (..., 3, 3) K (used as given, skew included) (camera.py:229-273)."""

    def __init__(self, params: Optional[torch.Tensor] = None, K: Optional[torch.Tensor] = None):
        assert params is not None or K is not None, "Pinhole needs params or K"
        if params is None:
            params = torch.stack([K[..., 0, 0], K[..., 1, 1], K[..., 0, 2], K[..., 1, 2]], dim=-1)
        super().__init__(params=params, K=K)

    @_no_autocast
    def project(self, pcd: torch.Tensor) -> torch.Tensor:
        b, _, h, w = pcd.shape
        cam = self.K @ pcd.reshape(b, 3, -1)
        uv = (cam[:, :2] / cam[:, 2:].clamp(min=0.01)).reshape(b, 2, h, w)
        # NB parity: for Pinhole the reference stores the COMPLEMENT of the in-image test (camera.py:246-252: the
        # variable called `invalid` holds the in-bounds pixels and the mask is its negation); kept as is.
        inside = (uv[:, 0] >= 0) & (uv[:, 0] < w) & (uv[:, 1] >= 0) & (uv[:, 1] < h)
        self.projection_mask = (~inside).unsqueeze(1)
        return uv

    @_no_autocast
    def unproject(self, uv: torch.Tensor) -> torch.Tensor:
        b, _, h, w = uv.shape
        uv1 = torch.cat([uv.reshape(b, 2, -1), torch.ones(b, 1, h * w, device=uv.device)], dim=1)
        xyz = torch.inverse(self.K.float()) @ uv1
        xyz = (xyz / xyz[:, -1:].clip(min=1e-4)).reshape(-1, 3, h, w)
        self.unprojection_mask = xyz[:, -1:] > 1e-4
        return xyz

    @_no_autocast
    def reconstruct(self, depth: torch.Tensor) -> torch.Tensor:
        b, _, h, w = depth.shape
        return self.unproject(pixel_grid(b, h, w, device=depth.device)) * depth.clip(min=0.0)


class EUCM(Camera):
    """Enhanced unified camera model: params fx fy cx cy alpha beta (camera.py:276-328)."""

    def __init__(self, params: torch.Tensor):
        super().__init__(params=params, K=None)

    @_no_autocast
    def project(self, xyz: torch.Tensor) -> torch.Tensor:
        fx, fy, cx, cy, alpha, beta = (self.params[:, i].reshape(-1, 1, 1) for i in range(6))
        x, y, z = xyz.unbind(dim=1)
        d = torch.sqrt(beta * (x * x + y * y) + z * z)
        den = (alpha * d + (1 - alpha) * z).clip(min=1e-3)
        uv = torch.stack([fx * (x / den) + cx, fy * (y / den) + cy], dim=1)
        self._set_projection_mask(uv, extra_invalid=z < 0)
        return uv

    @_no_autocast
    def unproject(self, uv: torch.Tensor) -> torch.Tensor:
        fx, fy, cx, cy, alpha, beta = (self.params[:, i].reshape(-1, 1, 1) for i in range(6))
        mx, my = (uv[:, 0] - cx) / fx, (uv[:, 1] - cy) / fy
        r2 = mx * mx + my * my
        # outside this radius the model has no pre-image (only when alpha > 0.5)
        limit = torch.where(alpha < 0.5, torch.full_like(alpha, 1e6), 1 / (beta * (2 * alpha - 1)))
        root = (1 - (2 * alpha - 1) * beta * r2).clip(min=1e-5).sqrt()
        mz = (1 - beta * alpha * alpha * r2) / (alpha * root + (1 - alpha))
        inv_n = 1 / torch.sqrt(r2 + mz * mz + 1e-5)
        z = inv_n * mz
        self.unprojection_mask = (r2 < limit) & (z > 1e-3)
        return torch.stack([inv_n * mx, inv_n * my, z.clamp(1e-3)], dim=1)


class Spherical(Camera):
    """Equirectangular panorama: params fx fy cx cy W H hfov/2 vfov/2 (radians) (camera.py:331-409)."""

    def __init__(self, params: torch.Tensor):
        super().__init__(params=params, K=None)

    def resize(self, factor: float) -> "Spherical":
        self.K[..., :2, :] *= factor
        self.params[..., :6] *= factor            # the image size scales too, the angular extent does not
        return self

    def crop(self, left, top, right, bottom) -> "Spherical":
        self.K[..., 0, 2] -= left
        self.K[..., 1, 2] -= top
        self.params[..., 2] -= left
        self.params[..., 3] -= top
        W, H = self.params[..., 4], self.params[..., 5]
        keep_w, keep_h = (W - left - right) / W, (H - top - bottom) / H
        self.params[..., 4] -= left + right
        self.params[..., 5] -= top + bottom
        self.params[..., 6] *= keep_w             # the field of view shrinks (or grows, for padding) with the image
        self.params[..., 7] *= keep_h
        return self

    def _extent(self):
        p = self.params
        view = lambda t: t.reshape(-1, 1, 1)
        return view(p[..., 4]), view(p[..., 5]), view(2 * p[..., 6]), view(2 * p[..., 7])

    @_no_autocast
    def project(self, xyz: torch.Tensor) -> torch.Tensor:
        width, height, hfov, vfov = self._extent()
        lon = torch.atan2(xyz[:, 0], xyz[:, 2])
        lat = torch.asin(xyz[:, 1] / xyz.norm(dim=1).clamp(min=1e-5))
        return torch.stack([lon / hfov * (width - 1) + (width - 1) / 2, lat / vfov * (height - 1) + (height - 1) / 2], dim=1)

    @_no_autocast
    def unproject(self, uv: torch.Tensor) -> torch.Tensor:
        width, height, hfov, vfov = self._extent()
        lon = (uv[:, 0] - (width - 1) / 2) / (width - 1) * hfov
        lat = (uv[:, 1] - (height - 1) / 2) / (height - 1) * vfov
        sphere = torch.stack([torch.cos(lat) * torch.sin(lon), torch.sin(lat), torch.cos(lat) * torch.cos(lon)], dim=1)
        return sphere / sphere.norm(dim=1, keepdim=True).clip(min=1e-5)

    def reconstruct(self, depth: torch.Tensor) -> torch.Tensor:
        return self.unproject(pixel_grid(1, depth.shape[-2], depth.shape[-1], device=depth.device)) * depth

    def get_new_fov(self, new_shape, original_shape):
        return (2 * self.params[..., 6] * new_shape[1] / original_shape[1],
                2 * self.params[..., 7] * new_shape[0] / original_shape[0])

    @property
    def hfov(self):
        return 2 * self.params[..., 6]

    @property
    def vfov(self):
        return 2 * self.params[..., 7]

    @property
    def max_fov(self):
        return 2 * math.pi, 0.9 * math.pi


class _Distorted(Camera):
    """Common part of the Brown-Conrady style models: 16 params fx fy cx cy | 6 radial | 2 tangential | 4 thin prism
    (or 15 with a single focal length).  Sub-classes define how the radial polynomial acts."""

    n_radial = 6

    def __init__(self, params: torch.Tensor):
        super().__init__(params=params, K=None)
        p = self.params
        self.use_radial = bool(p[..., 4:10].abs().sum() > 1e-6)
        self.use_tangential = bool(p[..., 10:12].abs().sum() > 1e-6)
        self.use_thin_prism = bool(p[..., 12:].abs().sum() > 1e-6)

    def _focal_centre(self):
        p = self.params
        b = p.shape[0]
        if p.shape[-1] == 15:
            return p[..., 0].reshape(b, 1, 1), p[..., 1:3].reshape(b, 1, 2)
        return p[..., 0:2].reshape(b, 1, 2), p[..., 2:4].reshape(b, 1, 2)

    def _tan_prism_coeffs(self):
        return self.params[..., -6:-4], self.params[..., -4:]

    def _finish_project(self, xy: torch.Tensor, bhw) -> torch.Tensor:
        p, s = self._tan_prism_coeffs()
        f, c = self._focal_centre()
        uv = _unflat(_tan_prism(xy, p, s) * f + c, bhw)
        self._set_projection_mask(uv)
        self.overlap_mask = self.mask_overlap_projection(uv)
        return uv

    def _start_unproject(self, uv: torch.Tensor):
        flat, bhw = _flat(uv)
        f, c = self._focal_centre()
        xy = (flat - c) / f
        if self.use_tangential or self.use_thin_prism:
            p, s = self._tan_prism_coeffs()
            xy = _undo_tan_prism(xy, p, s if self.use_thin_prism else None)
        return xy, bhw


class OPENCV(_Distorted):
    """OpenCV rational model restricted to the polynomial numerator: r_d = r (1 + k1 r^2 + k2 r^4 + k3 r^6)
    (camera.py:412-694)."""

    def __init__(self, params: torch.Tensor):
        super().__init__(params)
        assert self.params[..., 7:10].abs().sum() == 0.0, "Do not support poly division model"

    @_no_autocast
    def project(self, xyz: torch.Tensor) -> torch.Tensor:
        flat, bhw = _flat(xyz)
        z = flat[..., 2:3]
        z = torch.where(z.abs() < 1e-9, 1e-9 * torch.sign(z), z)
        ab = flat[..., :2] / z
        r2 = (ab * ab).sum(-1, keepdim=True)
        k = self.params[:, 4:7][:, None, :]
        pw = torch.cat([r2, r2 * r2, r2 * r2 * r2], dim=-1)
        return self._finish_project(ab * (1 + (pw * k).sum(-1, keepdim=True)), bhw)

    @_no_autocast
    def unproject(self, uv: torch.Tensor, max_iters: int = 25) -> torch.Tensor:
        xy, bhw = self._start_unproject(uv)
        rd = xy.norm(dim=-1, keepdim=True)
        r = _undo_radial(rd, self.params[:, 4:7], max_iters) if self.use_radial else rd
        scale = torch.where(rd < 1e-6, torch.ones_like(rd), r / rd.clamp(min=1e-12))
        return _unflat(torch.cat([xy * scale, torch.ones_like(rd)], dim=-1), bhw)


class Fisheye624(_Distorted):
    """Kannala-Brandt style fisheye with 6 radial, 2 tangential, 4 thin-prism terms: theta = atan(r),
    r_d = theta + k1 theta^3 + ... + k6 theta^13 (camera.py:697-974)."""

    @_no_autocast
    def project(self, xyz: torch.Tensor) -> torch.Tensor:
        flat, bhw = _flat(xyz)
        z = flat[..., 2:3]
        z = torch.where(z.abs() < 1e-9, 1e-9 * torch.sign(z), z)
        ab = flat[..., :2] / z
        r = ab.norm(dim=-1, keepdim=True)
        th = torch.atan(r)
        direction = torch.where(r < 1e-9, torch.ones_like(ab), ab / r)
        k = self.params[:, 4:10][:, None, :]
        pw = torch.cat([th ** (3 + 2 * i) for i in range(6)], dim=-1)
        return self._finish_project((th + (pw * k).sum(-1, keepdim=True)) * direction, bhw)

    @_no_autocast
    def unproject(self, uv: torch.Tensor, max_iters: int = 25) -> torch.Tensor:
        xy, bhw = self._start_unproject(uv)
        rd = xy.norm(dim=-1, keepdim=True)
        th = _undo_radial(rd, self.params[:, 4:10], max_iters) if self.use_radial else rd
        scale = torch.where(rd < 1e-6, torch.ones_like(rd), torch.tan(th) / rd.clamp(min=1e-12))
        return _unflat(torch.cat([xy * scale, torch.ones_like(rd)], dim=-1), bhw)


class MEI(Camera):
    """Unified (Mei) omnidirectional model: params fx fy cx cy k1 k2 p1 p2 xi (camera.py:977-1142)."""

    def __init__(self, params: torch.Tensor):
        super().__init__(params=params, K=None)
        self.use_radial = bool(self.params[..., 4:6].abs().sum() > 1e-6)
        self.use_tangential = bool(self.params[..., 6:8].abs().sum() > 1e-6)

    @_no_autocast
    def project(self, xyz: torch.Tensor) -> torch.Tensor:
        is_map = xyz.ndim == 4
        flat, bhw = _flat(xyz) if is_map else (xyz, None)
        b = flat.shape[0]
        p = self.params
        xi = p[:, 8].reshape(b, 1, 1)
        ab = flat[..., :2] / (flat[..., 2:3] + xi * flat.norm(dim=-1, keepdim=True))
        r2 = (ab * ab).sum(-1, keepdim=True)
        xy = ab * (1 + p[:, 4].reshape(b, 1, 1) * r2 + p[:, 5].reshape(b, 1, 1) * r2 * r2)
        uv = _tan_prism(xy, p[:, 6:8], None) * p[:, 0:2].reshape(b, 1, 2) + p[:, 2:4].reshape(b, 1, 2)
        if not is_map:
            return uv
        uv = _unflat(uv, bhw)
        self._set_projection_mask(uv)
        return uv

    @_no_autocast
    def unproject(self, uv: torch.Tensor, max_iters: int = 25) -> torch.Tensor:
        flat, bhw = _flat(uv)
        b = flat.shape[0]
        p = self.params
        xy = (flat - p[:, 2:4].reshape(b, 1, 2)) / p[:, 0:2].reshape(b, 1, 2)
        if self.use_tangential:
            xy = _undo_tan_prism(xy, p[:, 6:8], None, iters=20)
        rd = xy.norm(dim=-1, keepdim=True)
        r = _undo_radial(rd, p[:, 4:6], max_iters) if self.use_radial else rd
        m = xy * torch.where(rd < 1e-6, torch.ones_like(rd), r / rd.clamp(min=1e-12))
        # lift the point of the normalised plane back onto the unit sphere shifted by xi
        xi = p[:, 8].reshape(b, 1, 1)
        rho2 = (m * m).sum(-1, keepdim=True)
        pz = 1.0 - xi * (rho2 + 1.0) / (xi + torch.sqrt(1.0 + (1.0 - xi * xi) * rho2))
        pz = torch.where(xi == 1.0, (1.0 - rho2) / 2.0, pz)
        return _unflat(torch.cat([m, pz], dim=-1), bhw)


class BatchCamera(Camera):
    """A batch of cameras of possibly different models; every call is delegated to the members (camera.py:1145-1308).
    Build it with `BatchCamera.from_camera(cam)` or `torch.cat([cam_a, cam_b, ...])`."""

    def __init__(self, params, K, original_class, cameras):
        super().__init__(params, K)
        self.original_class = original_class
        self.cameras = cameras

    @classmethod
    def from_camera(cls, camera: Camera) -> "BatchCamera":
        return cls(camera.params, camera.K, [type(camera).__name__], [camera])

    @_no_autocast
    def project(self, points_3d: torch.Tensor) -> torch.Tensor:
        return torch.cat([cam.project(points_3d[i:i + 1]) for i, cam in enumerate(self.cameras)])

    @_no_autocast
    def unproject(self, points_2d: torch.Tensor) -> torch.Tensor:
        return torch.cat([cam.unproject(points_2d) for cam in self.cameras])

    def crop(self, left, top, right=None, bottom=None) -> "BatchCamera":
        return torch.cat([cam.crop(left, top, right, bottom) for cam in self.cameras])

    def resize(self, ratio) -> "BatchCamera":
        return torch.cat([cam.resize(ratio) for cam in self.cameras])

    def reconstruct(self, depth: torch.Tensor) -> torch.Tensor:
        return torch.cat([cam.reconstruct(depth[i:i + 1]) for i, cam in enumerate(self.cameras)])

    def get_projection_mask(self):
        return torch.cat([cam.projection_mask for cam in self.cameras])

    def get_new_fov(self, new_shape, original_shape):
        return [cam.get_new_fov(new_shape, original_shape) for cam in self.cameras]

    def to(self, device, non_blocking: bool = False) -> "BatchCamera":
        super().to(device, non_blocking=non_blocking)
        self.cameras = [cam.to(device, non_blocking=non_blocking) for cam in self.cameras]
        return self

    def __len__(self) -> int:
        return len(self.cameras)

    def __getitem__(self, idx):
        if isinstance(idx, int):
            return self.cameras[idx]
        if isinstance(idx, slice):
            return BatchCamera(self.params[idx], self.K[idx], self.original_class[idx], self.cameras[idx])
        raise TypeError(f"Invalid index type: {type(idx)}")

    def __setitem__(self, idx, value):
        if isinstance(idx, int):
            self.cameras[idx] = value
            self.params[idx, :] = 0.0
            self.params[idx, : value.params.shape[1]] = value.params[0]
            self.K[idx] = value.K[0]
            self.original_class[idx] = getattr(value, "original_class", type(value).__name__)
        elif isinstance(idx, slice):
            self.params[idx] = value.params
            self.K[idx] = value.K
            self.original_class[idx] = value.original_class
            self.cameras[idx] = value.cameras
        else:
            raise TypeError(f"Invalid index type: {type(idx)}")

    def _members(self, kind) -> List[bool]:
        return [isinstance(cam, kind) for cam in self.cameras]

    @property
    def is_perspective(self):
        return self._members(Pinhole)

    @property
    def is_pinhole(self):
        return self._members(Pinhole)

    @property
    def is_spherical(self):
        return self._members(Spherical)

    @property
    def is_eucm(self):
        return self._members(EUCM)

    @property
    def is_fisheye(self):
        return self._members(Fisheye624)

    @property
    def hfov(self):
        return [cam.hfov for cam in self.cameras]

    @property
    def vfov(self):
        return [cam.vfov for cam in self.cameras]

    @property
    def max_fov(self):
        return [cam.max_fov for cam in self.cameras]


# ------------------------------------------------------------------------------------------------------------------
# Packing for the GPU ray generator (udb_camera_rays, include/udb.h)
_CAM_STRIDE = 20                          # udb.h UDB_CAM_STRIDE: 16 parameters + use_radial, use_tangential, use_thin_prism, 0
_MODEL_IDS = {"Pinhole": 1, "EUCM": 2, "Spherical": 3, "OPENCV": 4, "Fisheye624": 5, "MEI": 6}   # UDB_CAM_*
_MIN_PARAMS = {"EUCM": 6, "Spherical": 8, "OPENCV": 16, "Fisheye624": 16, "MEI": 9}


def _pack_one(cam) -> Optional[Tuple[int, torch.Tensor]]:
    name = type(cam).__name__
    if name not in _MODEL_IDS or type(cam) is not globals()[name]:      # exact classes only: a subclass may differ
        return None
    if name == "Pinhole":
        K = cam.K
        if not isinstance(K, torch.Tensor) or K.dtype != torch.float32 or K.shape[-2:] != (3, 3):
            return None
        vals = K.reshape(-1, 9)
        flags = (0.0, 0.0, 0.0)
    else:
        p = cam.params
        if p.dtype != torch.float32 or p.ndim != 2:
            return None
        n = p.shape[1]
        if n < _MIN_PARAMS[name] or (name in ("OPENCV", "Fisheye624") and n != 16) or n > 16:
            return None                       # the 15-parameter single-focal layout stays on the host
        vals = p
        flags = (float(getattr(cam, "use_radial", False)), float(getattr(cam, "use_tangential", False)),
                 float(getattr(cam, "use_thin_prism", False)))
    rows = vals.new_zeros(vals.shape[0], _CAM_STRIDE)
    rows[:, :vals.shape[1]] = vals
    rows[:, 16:19] = torch.tensor(flags, dtype=torch.float32)
    return _MODEL_IDS[name], rows


def pack_camera(camera) -> Optional[Tuple[int, torch.Tensor]]:
    """(UDB_CAM_* model id, [rows, 20] float32 params in input-image pixels) for a Pinhole / EUCM / Spherical /
    16-parameter OPENCV or Fisheye624 / MEI object, or a BatchCamera whose members are all one such model (one row per
    member row); None for anything else, which keeps the host path.  The rows carry the object's own use_radial /
    use_tangential / use_thin_prism decisions.  The caller's object is not modified."""
    members = camera.cameras if type(camera) is BatchCamera else [camera]
    model, rows = None, []
    for cam in members:
        packed = _pack_one(cam)
        if packed is None or (model is not None and packed[0] != model):
            return None
        model = packed[0]
        rows.append(packed[1])
    if model is None:
        return None
    return model, torch.cat([r.to(rows[0].device) for r in rows])
