"""Loss / metric of the training step (SURVEY.md 8 row f-4).

Drop-ins for /root/reference/src/loss/loss_mse.py:12-31 (`LossMse`, `LossMseCfg`, `LossMseCfgWrapper`) and
/root/reference/src/evaluation/metrics.py:11-19 (`compute_psnr`), plus the fused route: the compositor's
epilogue already returns, per view, sse = sum (C - t)^2 and sse_clipped = sum (clip C - clip t)^2
(`DecoderSplattingCUDA.forward_mse`), from which

    LossMse          = weight * sse.sum() / (b v 3 h w)                       (mse_from_sse)
    compute_psnr     = -10 log10(sse_clipped / (3 h w))                       (psnr_from_sse)

with the rendered image never re-read for the loss and dL/dC never written as a tensor.

`ssim` / `compute_ssim` score renders as /root/reference/src/evaluation/metrics.py:36-52 does (skimage's
structural_similarity with an 11-tap Gaussian window, sigma 1.5, data_range 1, sample covariance), on the GPU: the
sm_90a kernels of csrc/ssim.cu (`ps_ssim_forward` / `ps_ssim_backward`) instead of a device-to-host copy and a CPU
loop over images.  `ssim` is differentiable in both images (1 - ssim is the usual partner of the photometric loss);
`compute_ssim` is the no-grad metric.

`LossLpips` / `LossLpipsCfg` / `LossLpipsCfgWrapper` and `compute_lpips` are the drop-ins for
/root/reference/src/loss/loss_lpips.py and evaluation/metrics.py:22-33, on `pixelsplat_b200.lpips.Lpips` (VGG16 trunk
in torch, the distance head fused in csrc/lpips.cu).

`LossDepth` / `LossDepthCfg` / `LossDepthCfgWrapper` are the drop-in for /root/reference/src/loss/loss_depth.py: an
edge-aware smoothness penalty on the rendered depth map (`DecoderOutput.depth`), which the fused depth channel
(`DecoderSplattingCUDA.forward(depth_mode=...)`) provides.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass, fields

import torch
from torch import Tensor, nn


@dataclass
class LossMseCfg:
    weight: float


@dataclass
class LossMseCfgWrapper:
    mse: LossMseCfg


class LossMse(nn.Module):
    """Same constructor and forward signature as the reference's LossMse (prediction has `.color`,
    batch["target"]["image"] is the ground truth)."""

    def __init__(self, cfg: LossMseCfgWrapper) -> None:
        super().__init__()
        (field,) = fields(type(cfg))
        self.cfg = getattr(cfg, field.name)
        self.name = field.name

    def forward(self, prediction, batch, gaussians=None, global_step: int = 0) -> Tensor:
        delta = prediction.color - batch["target"]["image"]
        return self.cfg.weight * (delta ** 2).mean()

    def from_sse(self, sse: Tensor, image_shape: tuple[int, int]) -> Tensor:
        """The same number from the fused epilogue's per-view sums [b, v]."""
        return mse_from_sse(sse, image_shape, self.cfg.weight)


def mse_from_sse(sse: Tensor, image_shape: tuple[int, int], weight: float = 1.0) -> Tensor:
    h, w = image_shape
    return weight * sse.sum() / (sse.numel() * 3 * h * w)


@torch.no_grad()
def compute_psnr(ground_truth: Tensor, predicted: Tensor) -> Tensor:
    """[batch, c, h, w] x 2 -> [batch] (metrics.py:11-19)."""
    ground_truth = ground_truth.clip(min=0, max=1)
    predicted = predicted.clip(min=0, max=1)
    mse = ((ground_truth - predicted) ** 2).mean(dim=(1, 2, 3))
    return -10 * mse.log10()


@torch.no_grad()
def psnr_from_sse(sse_clipped: Tensor, image_shape: tuple[int, int], channels: int = 3) -> Tensor:
    h, w = image_shape
    return -10 * (sse_clipped / (channels * h * w)).log10()


def _ssim_check(ground_truth: Tensor, predicted: Tensor) -> None:
    if ground_truth.dim() != 4 or ground_truth.shape != predicted.shape:
        raise ValueError(f"ssim: expected two [batch, channel, height, width] tensors of one shape, got "
                         f"{tuple(ground_truth.shape)} and {tuple(predicted.shape)}")
    if ground_truth.dtype != torch.float32 or predicted.dtype != torch.float32:
        raise ValueError(f"ssim: expected float32 images, got {ground_truth.dtype} and {predicted.dtype}")
    if ground_truth.shape[-2] < 11 or ground_truth.shape[-1] < 11:
        raise ValueError(f"ssim: images must be at least 11 x 11 (the window), got {tuple(ground_truth.shape[-2:])}")
    if not (ground_truth.is_cuda and predicted.is_cuda) or ground_truth.device != predicted.device:
        raise ValueError(f"ssim: expected CUDA tensors on one device, got {ground_truth.device} and "
                         f"{predicted.device}; there is no CPU path")


def _ssim_workspace(n: int, h: int, w: int, device) -> Tensor:
    from . import _lib
    size = ctypes.c_size_t()
    _lib.check(_lib.lib.ps_ssim_workspace_bytes(n, h, w, ctypes.byref(size)), "ps_ssim_workspace_bytes")
    return torch.empty(size.value, dtype=torch.uint8, device=device)


class _SsimPlanes(torch.autograd.Function):
    """[n, h, w] x 2 -> [n] per-plane scores (x = ground truth, y = prediction)."""

    @staticmethod
    def forward(ctx, x: Tensor, y: Tensor) -> Tensor:
        from . import _lib
        n, h, w = x.shape
        ws = _ssim_workspace(n, h, w, x.device)
        out = torch.empty(n, dtype=torch.float32, device=x.device)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        rc = _lib.on_device(x.device, _lib.lib.ps_ssim_forward, n, h, w, x.data_ptr(), y.data_ptr(), out.data_ptr(),
                            ws.data_ptr(), ws.numel(), stream)
        _lib.check(rc, "ps_ssim_forward")
        ctx.save_for_backward(x, y)
        return out

    @staticmethod
    def backward(ctx, d_out: Tensor):
        from . import _lib
        x, y = ctx.saved_tensors
        n, h, w = x.shape
        d_out = d_out.contiguous().float()
        d_x = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        d_y = torch.empty_like(y)
        ws = _ssim_workspace(n, h, w, x.device)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        rc = _lib.on_device(x.device, _lib.lib.ps_ssim_backward, n, h, w, x.data_ptr(), y.data_ptr(),
                            d_out.data_ptr(), None if d_x is None else d_x.data_ptr(), d_y.data_ptr(), ws.data_ptr(),
                            ws.numel(), stream)
        _lib.check(rc, "ps_ssim_backward")
        return d_x, (d_y if ctx.needs_input_grad[1] else None)


def ssim(ground_truth: Tensor, predicted: Tensor) -> Tensor:
    """SSIM of each image, [batch, channel, h, w] x 2 float32 CUDA -> [batch]: the mean over channels of each
    plane's mean SSIM map on the crop [5, h-5) x [5, w-5), as skimage's structural_similarity(win_size=11,
    gaussian_weights=True, channel_axis=0, data_range=1.0) computes it.  Differentiable in both images (the ground
    truth gets a gradient only when it requires one).  Inputs are not clipped."""
    _ssim_check(ground_truth, predicted)
    b, c, h, w = predicted.shape
    planes = _SsimPlanes.apply(ground_truth.contiguous().view(b * c, h, w), predicted.contiguous().view(b * c, h, w))
    return planes.view(b, c).mean(dim=1)


@torch.no_grad()
def compute_ssim(ground_truth: Tensor, predicted: Tensor) -> Tensor:
    """[batch, c, h, w] x 2 -> [batch] (metrics.py:36-52), on the prediction's device, without a host copy."""
    return ssim(ground_truth, predicted).to(predicted.dtype)


@dataclass
class LossLpipsCfg:
    weight: float
    apply_after_step: int


@dataclass
class LossLpipsCfgWrapper:
    lpips: LossLpipsCfg


def convert_to_buffer(module: nn.Module, persistent: bool = True) -> None:
    """Re-registers every parameter and buffer of `module` and its children as a buffer of the given persistence
    (what the reference's misc/nn_module_tools.py does to its LPIPS network)."""
    for child in module.children():
        convert_to_buffer(child, persistent)
    for name, value in (*module.named_parameters(recurse=False), *module.named_buffers(recurse=False)):
        value = value.detach().clone()
        delattr(module, name)
        module.register_buffer(name, value, persistent=persistent)


class LossLpips(nn.Module):
    """Same constructor and forward signature as the reference's LossLpips: weight * LPIPS(prediction.color,
    batch["target"]["image"], normalize=True).mean() over the (b v) images, or a float32 zero on the image's device
    before `apply_after_step`.  The LPIPS network's tensors are non-persistent buffers, so the loss adds no
    state-dict keys (a checkpoint never held them).  `lpips` defaults to `Lpips.from_files()` (the weights already
    on disk; nothing is downloaded).  In train mode the head applies the package's dropout, as the reference's
    does when its LightningModule is in train mode."""

    def __init__(self, cfg: LossLpipsCfgWrapper, lpips=None) -> None:
        super().__init__()
        from .lpips import Lpips
        (field,) = fields(type(cfg))
        self.cfg = getattr(cfg, field.name)
        self.name = field.name
        self.lpips = lpips if lpips is not None else Lpips.from_files()
        convert_to_buffer(self.lpips, persistent=False)

    def forward(self, prediction, batch, gaussians=None, global_step: int = 0) -> Tensor:
        image = batch["target"]["image"]
        if global_step < self.cfg.apply_after_step:
            return torch.tensor(0, dtype=torch.float32, device=image.device)
        loss = self.lpips(prediction.color.flatten(0, 1), image.flatten(0, 1), normalize=True)
        return self.cfg.weight * loss.mean()


_LPIPS_BY_DEVICE: dict = {}


def get_lpips(device) -> nn.Module:
    """One eval-mode `Lpips.from_files()` per device, created on first use (metrics.py's get_lpips)."""
    from .lpips import Lpips
    device = torch.device(device)
    if device not in _LPIPS_BY_DEVICE:
        _LPIPS_BY_DEVICE[device] = Lpips.from_files().to(device)
    return _LPIPS_BY_DEVICE[device].eval()


@torch.no_grad()
def compute_lpips(ground_truth: Tensor, predicted: Tensor) -> Tensor:
    """[batch, 3, h, w] x 2 in [0, 1] -> [batch] (metrics.py:22-33), always in eval mode (no dropout)."""
    value = get_lpips(predicted.device).forward(ground_truth, predicted, normalize=True)
    return value[:, 0, 0, 0].to(predicted.dtype)


@dataclass
class LossDepthCfg:
    weight: float
    sigma_image: float | None
    use_second_derivative: bool


@dataclass
class LossDepthCfgWrapper:
    depth: LossDepthCfg


def depth_smoothness(depth: Tensor, near: Tensor, far: Tensor, image: Tensor | None, sigma_image: float | None,
                     second_derivative: bool) -> Tensor:
    """Mean absolute finite difference of the depth map along x plus the same along y (first or second order),
    each difference down-weighted by exp(-sigma * colour edge) when `sigma_image` is set.  The depth map [b, v, h, w]
    is first clamped to [log near, log far] and mapped to [0, 1] on that interval (near / far [b, v]; `image`
    [b, v, c, h, w] is the ground truth whose largest per-channel difference is the edge)."""
    lo, hi = near.log()[..., None, None], far.log()[..., None, None]
    d = (depth.minimum(hi).maximum(lo) - lo) / (hi - lo)
    order = 2 if second_derivative else 1
    dx, dy = d.diff(n=order, dim=-1), d.diff(n=order, dim=-2)
    if sigma_image is not None:
        ex = image.diff(dim=-1).amax(dim=-3)           # [b, v, h, w - 1]
        ey = image.diff(dim=-2).amax(dim=-3)           # [b, v, h - 1, w]
        if second_derivative:                          # the larger edge of the two differences a term spans
            ex = torch.maximum(ex[..., :, 1:], ex[..., :, :-1])
            ey = torch.maximum(ey[..., 1:, :], ey[..., :-1, :])
        dx = dx * torch.exp(-sigma_image * ex)
        dy = dy * torch.exp(-sigma_image * ey)
    return dx.abs().mean() + dy.abs().mean()


class LossDepth(nn.Module):
    """Same constructor and forward signature as the reference's LossDepth: prediction.depth [b, v, h, w],
    batch["target"]["near"] / ["far"] [b, v] and ["image"] [b, v, 3, h, w]."""

    def __init__(self, cfg: LossDepthCfgWrapper) -> None:
        super().__init__()
        (field,) = fields(type(cfg))
        self.cfg = getattr(cfg, field.name)
        self.name = field.name

    def forward(self, prediction, batch, gaussians=None, global_step: int = 0) -> Tensor:
        t = batch["target"]
        return self.cfg.weight * depth_smoothness(prediction.depth, t["near"], t["far"], t["image"],
                                                  self.cfg.sigma_image, self.cfg.use_second_derivative)
