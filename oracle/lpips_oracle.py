"""Restatements of the reference's LPIPS (the lpips package 0.1.x, LPIPS(net="vgg"), as
/root/reference/src/loss/loss_lpips.py and evaluation/metrics.py:22-33 call it), test infrastructure only.

The package is not installed here, so this restates its documented formula (unpinned against the package itself):

    x -> 2x - 1 (normalize=True), then (x - shift) / scale per channel, shift = (-0.030, -0.088, -0.188),
    scale = (0.458, 0.448, 0.450);
    torchvision vgg16().features split at the package's indices: slice1 = 0-3, slice2 = 4-8, slice3 = 9-15,
    slice4 = 16-22, slice5 = 23-29 (3x3 convolutions, padding 1, ReLU, 2x2 max-pool); outputs relu1_2 .. relu5_3;
    per layer l: f^ = f / (sqrt(sum_c f_c^2) + 1e-10) for each side, u = f^0 - f^1,
    d_l[n] = mean over pixels of sum_c w_{l,c} m u_c^2  (w: the bias-free 1x1 lin{l} weight; m: dropout, 1 in eval);
    value = sum_l d_l, shape [N, 1, 1, 1].

`trunk`, `head` and `lpips` evaluate this in torch in the dtype of their inputs (float64 for the reference values;
the float32 `head` is the unfused torch head the benchmark compares against).  `dropout_mask` is a numpy
restatement of the fused head's dropout hash (include/pixelsplat_b200.h, ps_lpips_desc).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)
EPS = 1e-10
# torchvision vgg16().features: index -> (in, out) channels of its 3x3 convolutions; 4, 9, 16, 23 are max-pools
CONVS = {0: (3, 64), 2: (64, 64), 5: (64, 128), 7: (128, 128), 10: (128, 256), 12: (256, 256), 14: (256, 256),
         17: (256, 512), 19: (512, 512), 21: (512, 512), 24: (512, 512), 26: (512, 512), 28: (512, 512)}
POOLS = (4, 9, 16, 23)
SLICES = ((0, 4), (4, 9), (9, 16), (16, 23), (23, 30))
CHANNELS = (64, 128, 256, 512, 512)
GOLDEN = 0x9E3779B97F4A7C15
_M64 = (1 << 64) - 1


def slice_of(index: int) -> int:
    """The 1-based slice that holds features[index]."""
    return next(k + 1 for k, (a, b) in enumerate(SLICES) if a <= index < b)


def random_state_dict(seed: int = 0) -> dict[str, torch.Tensor]:
    """A full Lpips state dict (the module's key names) of seeded random tensors: He-normal convolutions (so the
    activations keep their scale through the 13 layers), small biases and non-negative lin weights."""
    g = torch.Generator().manual_seed(seed)
    sd = {"scaling_layer.shift": torch.tensor(SHIFT)[None, :, None, None],
          "scaling_layer.scale": torch.tensor(SCALE)[None, :, None, None]}
    for i, (cin, cout) in CONVS.items():
        k = slice_of(i)
        sd[f"net.slice{k}.{i}.weight"] = torch.randn((cout, cin, 3, 3), generator=g) * (2.0 / (9 * cin)) ** 0.5
        sd[f"net.slice{k}.{i}.bias"] = 0.01 * torch.randn((cout,), generator=g)
    for k, c in enumerate(CHANNELS):
        sd[f"lin{k}.model.1.weight"] = 0.5 * torch.rand((1, c, 1, 1), generator=g)
    return sd


def trunk(x: torch.Tensor, sd: dict[str, torch.Tensor]) -> list[torch.Tensor]:
    """relu1_2 .. relu5_3 of the scaled input x [N, 3, H, W], in x's dtype."""
    outs = []
    for k, (a, b) in enumerate(SLICES, start=1):
        for i in range(a, b):
            if i in POOLS:
                x = F.max_pool2d(x, 2, 2)
            elif i in CONVS:
                x = F.conv2d(x, sd[f"net.slice{k}.{i}.weight"].to(x), sd[f"net.slice{k}.{i}.bias"].to(x), padding=1)
            else:
                x = F.relu(x)
        outs.append(x)
    return outs


def normalize_tensor(f: torch.Tensor) -> torch.Tensor:
    return f / (torch.sqrt(torch.sum(f * f, dim=1, keepdim=True)) + EPS)


def head(f0: list[torch.Tensor], f1: list[torch.Tensor], weights: list[torch.Tensor],
         masks: list[torch.Tensor] | None = None) -> torch.Tensor:
    """[N]: sum over layers of the mean over pixels of sum_c w_c m u_c^2 (weights [C] per layer; masks, if given,
    [N, C, H, W] per layer)."""
    total = 0
    for l, (a, b, w) in enumerate(zip(f0, f1, weights)):
        d = (normalize_tensor(a) - normalize_tensor(b)) ** 2
        if masks is not None:
            d = d * masks[l].to(d)
        total = total + (d * w.reshape(1, -1, 1, 1).to(d)).sum(dim=1).mean(dim=(1, 2))
    return total


def lpips(in0: torch.Tensor, in1: torch.Tensor, sd: dict[str, torch.Tensor], normalize: bool = False,
          masks: list[torch.Tensor] | None = None) -> torch.Tensor:
    """The package's LPIPS(net="vgg").forward(in0, in1, normalize) -> [N, 1, 1, 1], in the inputs' dtype."""
    if normalize:
        in0, in1 = 2 * in0 - 1, 2 * in1 - 1
    shift, scale = sd["scaling_layer.shift"].to(in0), sd["scaling_layer.scale"].to(in0)
    f0, f1 = trunk((in0 - shift) / scale, sd), trunk((in1 - shift) / scale, sd)
    weights = [sd[f"lin{k}.model.1.weight"].reshape(-1) for k in range(5)]
    return head(f0, f1, weights, masks)[:, None, None, None]


def _mix(z):
    """splitmix64's finaliser on numpy uint64 arrays (wrapping arithmetic)."""
    z = z ^ (z >> np.uint64(30))
    z = z * np.uint64(0xBF58476D1CE4E5B9)
    z = z ^ (z >> np.uint64(27))
    z = z * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def dropout_mask(seed: int, layer: int, shape: tuple[int, ...]) -> np.ndarray:
    """The fused head's dropout factors (0 or 2, float64) of layer `layer` [N, C, H, W] for the int64 seed."""
    key = int(_mix(np.array([(int(seed) + (layer + 1) * GOLDEN) & _M64], dtype=np.uint64))[0])
    i = np.arange(int(np.prod(shape)), dtype=np.uint64)
    h = _mix(np.uint64(key) + (i + np.uint64(1)) * np.uint64(GOLDEN))
    return np.where((h >> np.uint64(63)) == 1, 2.0, 0.0).reshape(shape)
