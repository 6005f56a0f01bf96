"""Drop-in `GaussianAdapter` (SURVEY.md 8 row f-1): raw per-pixel network outputs -> world-space
Gaussians, as one fused CUDA kernel per direction (csrc/gaussian_adapter.cu) instead of the
reference's ~40 element-wise / tiny-matmul torch kernels.

Reference: /root/reference/src/model/encoder/common/gaussian_adapter.py:13-123 (same dataclasses,
constructor, `forward` signature, `get_scale_multiplier`, `d_sh`, `d_in`, non-persistent `sh_mask`
buffer) and gaussians.py:8-44.  The spherical-harmonics rotation (gaussian_adapter.py:84,
`rotate_sh` = e3nn Wigner-D of the camera-to-world rotation) uses pixelsplat_b200.sh, whose default
convention "e3nn" reproduces the reference's matrices; `sh_rotation_convention = "3dgs"` (attribute of
the module, not of the reference's cfg dataclass) opts into the rotation that is physically consistent
with the rasterizer's default basis instead.

The fused path covers the call shape EncoderEpipolar uses (encoder_epipolar.py:169-177): batch
dims (b, v, r, srf, spp) with extrinsics / intrinsics constant over (r, srf, spp) and coordinates /
raw features constant over spp.  Any other broadcast pattern takes the explicit torch path below
(same device, same formulas); CPU tensors are rejected -- this package has no CPU path.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass

import torch
from torch import Tensor, nn

from .. import _lib
from ..sh import camera_sh_rotations, rotate_sh


@dataclass
class Gaussians:
    means: Tensor         # [*batch, 3]
    covariances: Tensor   # [*batch, 3, 3]
    scales: Tensor        # [*batch, 3]
    rotations: Tensor     # [*batch, 4]  xyzw
    harmonics: Tensor     # [*batch, 3, d_sh]
    opacities: Tensor     # [*batch]


@dataclass
class GaussianAdapterCfg:
    gaussian_scale_min: float
    gaussian_scale_max: float
    sh_degree: int


def quaternion_to_matrix(quaternions: Tensor, eps: float = 1e-8) -> Tensor:
    """xyzw quaternions [..., 4] -> rotation matrices [..., 3, 3] (gaussians.py:8-30)."""
    i, j, k, r = torch.unbind(quaternions, dim=-1)
    two_s = 2 / ((quaternions * quaternions).sum(dim=-1) + eps)
    o = torch.stack((1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)), -1)
    return o.reshape(*quaternions.shape[:-1], 3, 3)


def build_covariance(scale: Tensor, rotation_xyzw: Tensor) -> Tensor:
    """R S S^T R^T (gaussians.py:33-44)."""
    rotation = quaternion_to_matrix(rotation_xyzw)
    rs = rotation * scale[..., None, :]
    return rs @ rs.transpose(-1, -2)


def world_rays(coordinates: Tensor, extrinsics: Tensor, intrinsics: Tensor) -> tuple[Tensor, Tensor]:
    """Broadcasting form of get_world_rays (/root/reference/src/geometry/projection.py:91-114)."""
    xy1 = torch.cat([coordinates, torch.ones_like(coordinates[..., :1])], dim=-1)
    d = torch.einsum("...ij,...j->...i", intrinsics.inverse(), xy1)
    d = d / d.norm(dim=-1, keepdim=True)
    d = torch.einsum("...ij,...j->...i", extrinsics[..., :3, :3], d)
    return extrinsics[..., :3, 3].broadcast_to(d.shape), d


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class _GaussianAdapterFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, extrinsics, intrinsics, sh_rotation, sh_mask, coordinates, depths, raw, image_shape,
                scale_min, scale_max, eps):
        nv, nr, ns = depths.shape
        n_sh = sh_mask.shape[0]
        h, w = image_shape
        dev = raw.device
        desc = _lib.AdapterDesc(nv, nr, ns, n_sh, h, w, scale_min, scale_max, eps, 0)
        tensors = [t.contiguous().float() for t in (extrinsics, intrinsics, sh_rotation, sh_mask, coordinates, depths, raw)]
        inputs = _lib.AdapterInputs(*[t.data_ptr() for t in tensors])
        means = torch.empty((nv, nr, ns, 3), dtype=torch.float32, device=dev)
        cov = torch.empty((nv, nr, ns, 3, 3), dtype=torch.float32, device=dev)
        harm = torch.empty((nv, nr, ns, 3, n_sh), dtype=torch.float32, device=dev)
        scales = torch.empty((nv, nr, ns, 3), dtype=torch.float32, device=dev)
        rot = torch.empty((nv, nr, 4), dtype=torch.float32, device=dev)
        stream = torch.cuda.current_stream(dev)
        rc = _lib.on_device(dev, _lib.lib.ps_gaussian_adapter_forward, ctypes.byref(desc), ctypes.byref(inputs), _p(means), _p(cov),
                                                  _p(harm), _p(scales), _p(rot), ctypes.c_void_p(stream.cuda_stream))
        _lib.check(rc, "ps_gaussian_adapter_forward")
        ctx.save_for_backward(*tensors)
        ctx.desc = desc
        ctx.out_shapes = (means.shape, cov.shape, harm.shape)
        # training reads scales and rotations only for a visualisation dump: their cotangents stay None and reach
        # the kernel as NULL instead of as zero tensors it would read for nothing
        ctx.set_materialize_grads(False)
        return means, cov, harm, scales, rot

    @staticmethod
    def backward(ctx, d_means, d_cov, d_harm, d_scales, d_rot):
        if all(g is None for g in (d_means, d_cov, d_harm, d_scales, d_rot)):
            return (None,) * 11
        tensors = ctx.saved_tensors
        desc = ctx.desc
        dev = tensors[-1].device
        inputs = _lib.AdapterInputs(*[t.data_ptr() for t in tensors])
        f = lambda t: t.contiguous().float()
        # the kernel requires these three; d_scales / d_rot may be NULL
        d_means, d_cov, d_harm = [f(t) if t is not None else torch.zeros(s, dtype=torch.float32, device=dev)
                                  for t, s in zip((d_means, d_cov, d_harm), ctx.out_shapes)]
        d_scales = f(d_scales) if d_scales is not None else None
        d_rot = f(d_rot) if d_rot is not None else None
        d_coord = torch.empty_like(tensors[4])
        d_depths = torch.empty_like(tensors[5])
        d_raw = torch.empty_like(tensors[6])
        stream = torch.cuda.current_stream(dev)
        rc = _lib.on_device(dev, _lib.lib.ps_gaussian_adapter_backward, ctypes.byref(desc), ctypes.byref(inputs), _p(d_means), _p(d_cov),
                                                   _p(d_harm), _p(d_scales), _p(d_rot), _p(d_coord), _p(d_depths),
                                                   _p(d_raw), ctypes.c_void_p(stream.cuda_stream))
        _lib.check(rc, "ps_gaussian_adapter_backward")
        return None, None, None, None, d_coord, d_depths, d_raw, None, None, None, None


class GaussianAdapter(nn.Module):
    cfg: GaussianAdapterCfg
    sh_rotation_convention: str = "e3nn"     # the reference's rotate_sh; "3dgs" = rasterizer-consistent (opt-in)

    def __init__(self, cfg: GaussianAdapterCfg):
        super().__init__()
        self.cfg = cfg
        self.register_buffer("sh_mask", torch.ones((self.d_sh,), dtype=torch.float32), persistent=False)
        for degree in range(1, self.cfg.sh_degree + 1):
            self.sh_mask[degree ** 2:(degree + 1) ** 2] = 0.1 * 0.25 ** degree

    # ---- fused path -------------------------------------------------------------------------
    def _fused_shapes(self, extrinsics, intrinsics, coordinates, depths, opacities, raw):
        """Returns (b, v, r, srf, spp) when the call has EncoderEpipolar's broadcast pattern, else None."""
        if opacities.dim() != 5 or depths.shape != opacities.shape or self.cfg.sh_degree > 4:
            return None
        b, v, r, srf, spp = opacities.shape
        ok = (extrinsics.dim() == 7 and tuple(extrinsics.shape[2:5]) == (1, 1, 1) and extrinsics.shape[0] in (1, b)
              and extrinsics.shape[1] in (1, v) and intrinsics.dim() == 7 and tuple(intrinsics.shape[2:5]) == (1, 1, 1)
              and intrinsics.shape[0] in (1, b) and intrinsics.shape[1] in (1, v)
              and coordinates.dim() == 6 and coordinates.shape[4] == 1 and coordinates.shape[-1] == 2
              and coordinates.shape[0] in (1, b) and coordinates.shape[1] in (1, v)
              and coordinates.shape[2] in (1, r) and coordinates.shape[3] in (1, srf)
              and raw.dim() == 6 and tuple(raw.shape[:5]) == (b, v, r, srf, 1) and raw.shape[-1] == self.d_in
              and 1 <= spp <= 8)
        return (b, v, r, srf, spp) if ok else None

    def forward(self, extrinsics: Tensor, intrinsics: Tensor, coordinates: Tensor, depths: Tensor,
                opacities: Tensor, raw_gaussians: Tensor, image_shape: tuple[int, int],
                eps: float = 1e-8) -> Gaussians:
        if not raw_gaussians.is_cuda:
            raise ValueError("pixelsplat_b200 has no CPU path: GaussianAdapter needs CUDA tensors")
        shp = self._fused_shapes(extrinsics, intrinsics, coordinates, depths, opacities, raw_gaussians)
        if shp is None:
            return self.forward_explicit(extrinsics, intrinsics, coordinates, depths, opacities, raw_gaussians,
                                         image_shape, eps)
        b, v, r, srf, spp = shp
        nv, nr = b * v, r * srf
        E = extrinsics.expand(b, v, 1, 1, 1, 4, 4).reshape(nv, 4, 4)
        K = intrinsics.expand(b, v, 1, 1, 1, 3, 3).reshape(nv, 3, 3)
        D = camera_sh_rotations(E, self.cfg.sh_degree, self.sh_rotation_convention)
        coords = coordinates.expand(b, v, r, srf, 1, 2).reshape(nv, nr, 2)
        means, cov, harm, scales, rot = _GaussianAdapterFn.apply(
            E.detach(), K.detach(), D, self.sh_mask, coords, depths.reshape(nv, nr, spp),
            raw_gaussians.reshape(nv, nr, self.d_in), tuple(image_shape), float(self.cfg.gaussian_scale_min),
            float(self.cfg.gaussian_scale_max), float(eps))
        lead = (b, v, r, srf, spp)
        return Gaussians(means=means.reshape(*lead, 3), covariances=cov.reshape(*lead, 3, 3),
                         harmonics=harm.reshape(*lead, 3, self.d_sh), opacities=opacities,
                         scales=scales.reshape(*lead, 3),
                         rotations=rot.reshape(b, v, r, srf, 1, 4).broadcast_to((*lead, 4)))

    # ---- explicit path: the reference's op sequence in torch (any broadcast pattern) ------------
    def forward_explicit(self, extrinsics, intrinsics, coordinates, depths, opacities, raw_gaussians,
                         image_shape, eps: float = 1e-8, rotate: bool = True) -> Gaussians:
        device = extrinsics.device
        scales, rotations, sh = raw_gaussians.split((3, 4, 3 * self.d_sh), dim=-1)
        scale_min, scale_max = self.cfg.gaussian_scale_min, self.cfg.gaussian_scale_max
        scales = scale_min + (scale_max - scale_min) * scales.sigmoid()
        h, w = image_shape
        wh = torch.cat([torch.full((1,), float(w), dtype=torch.float32, device=device),
                        torch.full((1,), float(h), dtype=torch.float32, device=device)])   # no H2D copy
        pixel_size = (1 / wh).to(intrinsics.dtype)
        multiplier = self.get_scale_multiplier(intrinsics, pixel_size)
        scales = scales * depths[..., None] * multiplier[..., None]
        rotations = rotations / (rotations.norm(dim=-1, keepdim=True) + eps)
        sh = sh.reshape(*sh.shape[:-1], 3, self.d_sh)
        sh = sh.broadcast_to((*opacities.shape, 3, self.d_sh)) * self.sh_mask
        covariances = build_covariance(scales, rotations)
        c2w = extrinsics[..., :3, :3]
        covariances = c2w @ covariances @ c2w.transpose(-1, -2)
        origins, directions = world_rays(coordinates, extrinsics, intrinsics)
        means = origins + directions * depths[..., None]
        return Gaussians(means=means, covariances=covariances,
                         harmonics=(rotate_sh(sh, c2w[..., None, :, :], self.sh_rotation_convention)
                                    if rotate else sh),
                         opacities=opacities, scales=scales,
                         rotations=rotations.broadcast_to((*scales.shape[:-1], 4)))

    def get_scale_multiplier(self, intrinsics: Tensor, pixel_size: Tensor, multiplier: float = 0.1) -> Tensor:
        xy = multiplier * torch.einsum("...ij,j->...i", intrinsics[..., :2, :2].inverse(), pixel_size)
        return xy.sum(dim=-1)

    @property
    def d_sh(self) -> int:
        return (self.cfg.sh_degree + 1) ** 2

    @property
    def d_in(self) -> int:
        return 7 + 3 * self.d_sh
