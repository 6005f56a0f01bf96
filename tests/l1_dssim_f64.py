"""A float64 restatement of ps_l1_dssim (csrc/l1_dssim.cu), 3DGS's loss (1 - lambda) L1 + lambda (1 - SSIM), and a
direct transcription of 3DGS's conv2d formulation to check it against.

`l1_dssim_f64` filters with the separable 11-tap window over zero-padded planes, written out as shifted slices, and
returns each image's loss with its two terms.  `l1_dssim_grad_f64` is the gradient of the summed losses in closed form:
the chain rule's per-pixel maps filtered back, as the kernel forms it (without the kernel's shift, which float64 does
not need).  `L1DssimF64` pairs the two, so gradcheck can test the closed form.  `loss_3dgs_torch` is 3DGS's
conv2d(padding=5, groups=C) SSIM and mean-absolute L1 in torch ops, for any dtype and device."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

RADIUS = 5
C1, C2 = 0.01 ** 2, 0.03 ** 2


def taps(dtype=torch.float64) -> torch.Tensor:
    k = torch.arange(-RADIUS, RADIUS + 1, dtype=torch.float64)
    g = torch.exp(-k * k / (2 * 1.5 ** 2))
    return (g / g.sum()).to(dtype)


def filter_zero(z: torch.Tensor) -> torch.Tensor:
    """'same'-size correlation of [..., h, w] with the 11x11 window over zero padding (separable, shifted slices)."""
    g = taps(z.dtype).to(z.device)
    h, w = z.shape[-2:]
    zp = F.pad(z, (RADIUS, RADIUS, 0, 0))
    rows = sum(g[k] * zp[..., :, k:k + w] for k in range(2 * RADIUS + 1))
    rp = F.pad(rows, (0, 0, RADIUS, RADIUS))
    return sum(g[k] * rp[..., k:k + h, :] for k in range(2 * RADIUS + 1))


def _terms(p: torch.Tensor, g: torch.Tensor):
    mg, mp = filter_zero(g), filter_zero(p)
    vg = filter_zero(g * g) - mg * mg
    vp = filter_zero(p * p) - mp * mp
    cov = filter_zero(g * p) - mg * mp
    a1, a2 = 2 * mg * mp + C1, 2 * cov + C2
    b1, b2 = mg * mg + mp * mp + C1, vg + vp + C2
    return mg, mp, a1, a2, b1, b2, a1 * a2 / (b1 * b2)


def l1_dssim_f64(p: torch.Tensor, g: torch.Tensor, lam: float):
    """[n, c, h, w] x 2 (float64) -> (loss [n], l1 [n], ssim [n])."""
    *_, s = _terms(p, g)
    l1 = (p - g).abs().mean(dim=(1, 2, 3))
    ssim = s.mean(dim=(1, 2, 3))
    return (1 - lam) * l1 + lam * (1 - ssim), l1, ssim


def l1_dssim_grad_f64(p: torch.Tensor, g: torch.Tensor, lam: float, magnitude: bool = False) -> torch.Tensor:
    """d(sum over images of loss)/dp, [n, c, h, w]: the maps a = dS/dmu_p - 2 mu_p b - mu_g c, b = dS/dvar,
    c = dS/dcov filtered back (the zero-padded correlation with a symmetric window is its own adjoint), plus the L1
    term with sign(0) = 0.  With `magnitude`, the same chain with every term replaced by its absolute value: the scale
    that a float32 evaluation's rounding error follows where the terms cancel (near a maximum of SSIM)."""
    mg, mp, a1, a2, b1, b2, s = _terms(p, g)
    area = p.shape[1] * p.shape[2] * p.shape[3]
    inv = 1 / (b1 * b2)
    b = -s / b2
    c = 2 * a1 * inv
    if magnitude:
        a = (2 * mg * a2 * inv).abs() + (2 * mp * s / b1).abs() + (2 * mp * b).abs() + (mg * c).abs()
        d_sum_s = filter_zero(a) + 2 * p.abs() * filter_zero(b.abs()) + g.abs() * filter_zero(c.abs())
        return (lam * d_sum_s + (1 - lam) * torch.sign(p - g).abs()) / area
    a = 2 * mg * a2 * inv - 2 * mp * s / b1 - 2 * mp * b - mg * c
    d_sum_s = filter_zero(a) + 2 * p * filter_zero(b) + g * filter_zero(c)
    return (-lam * d_sum_s + (1 - lam) * torch.sign(p - g)) / area


class L1DssimF64(torch.autograd.Function):
    """l1_dssim_f64's loss with l1_dssim_grad_f64 as its backward (in the prediction only)."""

    @staticmethod
    def forward(ctx, p, g, lam):
        ctx.save_for_backward(p, g)
        ctx.lam = lam
        return l1_dssim_f64(p, g, lam)[0]

    @staticmethod
    def backward(ctx, d_out):
        p, g = ctx.saved_tensors
        return l1_dssim_grad_f64(p, g, ctx.lam) * d_out.view(-1, 1, 1, 1), None, None


def loss_3dgs_torch(p: torch.Tensor, g: torch.Tensor, lam: float) -> torch.Tensor:
    """3DGS's per-image loss as its training code writes it: a 2D window (outer product of the 1D taps) applied with
    conv2d(padding=5, groups=C), mu1_sq / mu2_sq / mu1_mu2, sigma1_sq = conv(img1^2) - mu1_sq, ..., the SSIM map's
    mean (here per image), and the mean absolute difference.  -> [n]."""
    c = p.shape[1]
    g1 = taps(p.dtype).to(p.device)
    window = (g1[:, None] @ g1[None, :]).expand(c, 1, 2 * RADIUS + 1, 2 * RADIUS + 1).contiguous()
    conv = lambda z: F.conv2d(z, window, padding=RADIUS, groups=c)
    mu1, mu2 = conv(p), conv(g)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = conv(p * p) - mu1_sq
    sigma2_sq = conv(g * g) - mu2_sq
    sigma12 = conv(p * g) - mu1_mu2
    ssim_map = ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))
    l1 = (p - g).abs().mean(dim=(1, 2, 3))
    return (1.0 - lam) * l1 + lam * (1.0 - ssim_map.mean(dim=(1, 2, 3)))


def expon_lr(step: int, lr_init: float, lr_final: float, max_steps: int) -> float:
    """3DGS's get_expon_lr_func(lr_init, lr_final, max_steps=max_steps) at `step`, with no delay."""
    if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
        return 0.0
    t = min(max(step / max_steps, 0.0), 1.0)
    return math.exp(math.log(lr_init) * (1 - t) + math.log(lr_final) * t)
