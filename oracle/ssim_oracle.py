"""Restatements of the reference's SSIM (/root/reference/src/evaluation/metrics.py:36-52), test infrastructure only.

The reference calls skimage.metrics.structural_similarity(gt, hat, win_size=11, gaussian_weights=True,
channel_axis=0, data_range=1.0) on float32 [C, H, W] arrays.  With skimage's defaults (K1 = 0.01, K2 = 0.03,
sigma = 1.5, truncate = 3.5, use_sample_covariance=True) that is, per channel plane x (ground truth), y (prediction):

    g     the 11-tap Gaussian exp(-k^2 / (2 1.5^2)), k = -5..5, normalised (scipy.ndimage.gaussian_filter's kernel),
          G = g g^T, * = correlation with G (scipy filters with mode="reflect")
    mu_x = G*x,  mu_y = G*y,  var_x = n (G*x^2 - mu_x^2),  var_y = n (G*y^2 - mu_y^2),  cov = n (G*xy - mu_x mu_y)
    S    = (2 mu_x mu_y + C1)(2 cov + C2) / ((mu_x^2 + mu_y^2 + C1)(var_x + var_y + C2)),  n = 121/120,
          C1 = 0.01^2, C2 = 0.03^2
    score = mean of S over [5, H-5) x [5, W-5); the image's score is the mean over its channels.

skimage is not installed here, so these are restatements of that definition, not the library:
  - `ssim_numpy`: numpy, the filter written out as separable taps over np.pad(mode="symmetric") (scipy's "reflect"),
    in float64 or, to show how far a float32 evaluation drifts, in float32 arrays;
  - `ssim_torch`: torch float64, a valid-mode conv2d with G; its autograd gives the reference gradients.
Neither imports scipy.
"""
from __future__ import annotations

import numpy as np

RADIUS = 5
SIGMA = 1.5
C1 = 0.01 ** 2
C2 = 0.03 ** 2
COV_NORM = 121.0 / 120.0


def gaussian_taps() -> np.ndarray:
    """The 11 weights, float64, summing to 1."""
    k = np.arange(-RADIUS, RADIUS + 1, dtype=np.float64)
    g = np.exp(-0.5 * k * k / (SIGMA * SIGMA))
    return g / g.sum()


def gaussian_filter(a: np.ndarray) -> np.ndarray:
    """scipy.ndimage.gaussian_filter(a, sigma=1.5, truncate=3.5, mode="reflect") of a 2-D array, in a's dtype."""
    g = gaussian_taps().astype(a.dtype)
    out = a
    for axis in (0, 1):
        pad = [(0, 0), (0, 0)]
        pad[axis] = (RADIUS, RADIUS)
        p = np.pad(out, pad, mode="symmetric")
        n = out.shape[axis]
        acc = np.zeros_like(out)
        for k in range(2 * RADIUS + 1):
            acc += g[k] * (p[k:k + n] if axis == 0 else p[:, k:k + n])
        out = acc
    return out


def ssim_plane_numpy(x: np.ndarray, y: np.ndarray, dtype=np.float64) -> float:
    x, y = np.asarray(x, dtype), np.asarray(y, dtype)
    f = gaussian_filter
    mx, my = f(x), f(y)
    n = dtype(COV_NORM)
    vx = n * (f(x * x) - mx * mx)
    vy = n * (f(y * y) - my * my)
    cxy = n * (f(x * y) - mx * my)
    s = ((2 * mx * my + dtype(C1)) * (2 * cxy + dtype(C2))) / ((mx * mx + my * my + dtype(C1)) * (vx + vy + dtype(C2)))
    return float(s[RADIUS:-RADIUS, RADIUS:-RADIUS].astype(np.float64).mean())


def ssim_planes_numpy(x: np.ndarray, y: np.ndarray, dtype=np.float64) -> np.ndarray:
    """[..., H, W] x 2 -> [...] per-plane scores."""
    x, y = np.asarray(x), np.asarray(y)
    if x.shape[-2] < 2 * RADIUS + 1 or x.shape[-1] < 2 * RADIUS + 1:
        raise ValueError("ssim: images must be at least 11 x 11")
    lead = x.shape[:-2]
    xs, ys = x.reshape(-1, *x.shape[-2:]), y.reshape(-1, *y.shape[-2:])
    return np.array([ssim_plane_numpy(a, b, dtype) for a, b in zip(xs, ys)]).reshape(lead)


def ssim_numpy(ground_truth: np.ndarray, predicted: np.ndarray, dtype=np.float64) -> np.ndarray:
    """[batch, C, H, W] x 2 -> [batch], as the reference's compute_ssim."""
    return ssim_planes_numpy(ground_truth, predicted, dtype).mean(axis=-1)


def ssim_planes_torch(x, y):
    """[..., H, W] x 2 (any float dtype; float64 for a reference) -> [...] per-plane scores, differentiable."""
    import torch
    import torch.nn.functional as F
    g = torch.as_tensor(gaussian_taps(), dtype=x.dtype, device=x.device)
    w = (g[:, None] * g[None, :])[None, None]
    lead, (h, wd) = x.shape[:-2], x.shape[-2:]
    xs, ys = x.reshape(-1, 1, h, wd), y.reshape(-1, 1, h, wd)
    f = lambda a: F.conv2d(a, w)                       # valid windows only: exactly the crop
    mx, my = f(xs), f(ys)
    vx = COV_NORM * (f(xs * xs) - mx * mx)
    vy = COV_NORM * (f(ys * ys) - my * my)
    cxy = COV_NORM * (f(xs * ys) - mx * my)
    s = ((2 * mx * my + C1) * (2 * cxy + C2)) / ((mx * mx + my * my + C1) * (vx + vy + C2))
    return s.mean(dim=(1, 2, 3)).reshape(lead)


def ssim_torch(ground_truth, predicted):
    """[batch, C, H, W] x 2 -> [batch]."""
    return ssim_planes_torch(ground_truth, predicted).mean(dim=-1)
