"""LPIPS with the VGG16 trunk: the analogue of the lpips package's `LPIPS(net="vgg")` (version 0.1, lpips=True,
spatial=False, use_dropout=True), which the reference uses as its second training loss and third test metric
(/root/reference/src/loss/loss_lpips.py, evaluation/metrics.py:22-33).

    x -> 2x - 1 (normalize=True);  (x - shift) / scale;  VGG16 features relu1_2 .. relu5_3 of both inputs;
    per layer: unit-normalise each side over channels, u = f^0 - f^1, the 1x1 `lin` weighting of u^2 (after
    dropout in train mode), mean over pixels;  sum over layers -> [N, 1, 1, 1].

The trunk is torch (`nn.Conv2d` / `ReLU` / `MaxPool2d` under `net.slice{k}.{i}`, run on cuDNN with torch's settings
as they stand).  The distance head is one sm_90a kernel over all five layers (csrc/lpips.cu, `ps_lpips_forward` /
`ps_lpips_backward`), forward and backward, with no float atomics.  In train mode the head applies the package's
Dropout(p = 0.5) to u^2: a counter-based hash of an int64 seed that each forward draws on the device from torch's
CUDA generator (so the forward can be captured in a CUDA graph), recomputed in the backward.

Weights are never downloaded.  `Lpips.from_files` reads torchvision's `vgg16-397923af.pth` and the package's
`weights/v0.1/vgg.pth` from where they already are on disk (the torch hub cache, the installed `lpips` package) or
from explicit paths.
"""
from __future__ import annotations

import ctypes
import importlib.util
from pathlib import Path

import torch
from torch import Tensor, nn

VGG16_FILE = "vgg16-397923af.pth"
SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)
CHANNELS = (64, 128, 256, 512, 512)
# torchvision vgg16().features indices of each slice (the package's split) and of the convolutions among them
SLICES = ((0, 4), (4, 9), (9, 16), (16, 23), (23, 30))
_POOLS = (4, 9, 16, 23)
_CONVS = {0: (3, 64), 2: (64, 64), 5: (64, 128), 7: (128, 128), 10: (128, 256), 12: (256, 256), 14: (256, 256),
          17: (256, 512), 19: (512, 512), 21: (512, 512), 24: (512, 512), 26: (512, 512), 28: (512, 512)}
MIN_SIZE = 16            # four 2x2 pools: relu5_3 is at least 1 x 1


class ScalingLayer(nn.Module):
    def __init__(self) -> None:
        super().__init__()
        self.register_buffer("shift", torch.tensor(SHIFT)[None, :, None, None])
        self.register_buffer("scale", torch.tensor(SCALE)[None, :, None, None])

    def forward(self, x: Tensor) -> Tensor:
        return (x - self.shift) / self.scale


class Vgg16(nn.Module):
    """torchvision's vgg16().features in the package's five slices; the modules keep their features index as name."""

    def __init__(self) -> None:
        super().__init__()
        for k, (a, b) in enumerate(SLICES, start=1):
            s = nn.Sequential()
            for i in range(a, b):
                if i in _POOLS:
                    m = nn.MaxPool2d(kernel_size=2, stride=2)
                elif i in _CONVS:
                    m = nn.Conv2d(*_CONVS[i], kernel_size=3, padding=1)
                else:
                    m = nn.ReLU(inplace=True)
                s.add_module(str(i), m)
            setattr(self, f"slice{k}", s)

    def forward(self, x: Tensor) -> list[Tensor]:
        outs = []
        for k in range(1, 6):
            x = getattr(self, f"slice{k}")(x)
            outs.append(x)
        return outs


class NetLinLayer(nn.Module):
    """The package's lin layer: Dropout(0.5) then a bias-free 1x1 convolution to one channel.  Only its weight is
    used (by the fused head); the key is `model.1.weight` as in the package."""

    def __init__(self, channels: int) -> None:
        super().__init__()
        self.model = nn.Sequential(nn.Dropout(0.5), nn.Conv2d(channels, 1, 1, bias=False))


class _LpipsHead(torch.autograd.Function):
    """(seed or None, n_layers, lin weights [C] x L, x0 features x L, x1 features x L) -> [N]."""

    @staticmethod
    def forward(ctx, seed, n_layers: int, *tensors):
        from . import _lib
        ws_, x0, x1 = tensors[:n_layers], tensors[n_layers:2 * n_layers], tensors[2 * n_layers:]
        desc = _desc(seed, ws_, x0, x1)
        dev = x0[0].device
        size = ctypes.c_size_t()
        _lib.check(_lib.lib.ps_lpips_workspace_bytes(ctypes.byref(desc), ctypes.byref(size)),
                   "ps_lpips_workspace_bytes")
        ws = torch.empty(size.value, dtype=torch.uint8, device=dev)
        out = torch.empty(x0[0].shape[0], dtype=torch.float32, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        rc = _lib.on_device(dev, _lib.lib.ps_lpips_forward, ctypes.byref(desc), out.data_ptr(), ws.data_ptr(),
                            ws.numel(), stream)
        _lib.check(rc, "ps_lpips_forward")
        ctx.n_layers = n_layers
        ctx.save_for_backward(*((seed,) if seed is not None else ()), *tensors)
        ctx.has_seed = seed is not None
        return out

    @staticmethod
    def backward(ctx, d_out: Tensor):
        from . import _lib
        saved = ctx.saved_tensors
        seed = saved[0] if ctx.has_seed else None
        tensors = saved[1:] if ctx.has_seed else saved
        L = ctx.n_layers
        ws_, x0, x1 = tensors[:L], tensors[L:2 * L], tensors[2 * L:]
        want0 = any(ctx.needs_input_grad[2 + L:2 + 2 * L])
        want1 = any(ctx.needs_input_grad[2 + 2 * L:])
        if not (want0 or want1):
            return (None,) * (2 + 3 * L)
        d0 = [torch.empty_like(t) if want0 else None for t in x0]
        d1 = [torch.empty_like(t) if want1 else None for t in x1]
        grads = _lib.LpipsGrads()
        for l in range(L):
            grads.d_x0[l] = None if d0[l] is None else d0[l].data_ptr()
            grads.d_x1[l] = None if d1[l] is None else d1[l].data_ptr()
        desc = _desc(seed, ws_, x0, x1)
        d_out = d_out.contiguous().float()
        dev = x0[0].device
        stream = torch.cuda.current_stream(dev).cuda_stream
        rc = _lib.on_device(dev, _lib.lib.ps_lpips_backward, ctypes.byref(desc), d_out.data_ptr(),
                            ctypes.byref(grads), stream)
        _lib.check(rc, "ps_lpips_backward")
        return (None, None) + (None,) * L + tuple(d0) + tuple(d1)


def _desc(seed, weights, x0, x1):
    from . import _lib
    desc = _lib.LpipsDesc()
    desc.n_layers = len(x0)
    desc.N = x0[0].shape[0] if x0 else 0
    for l, (w, a, b) in enumerate(zip(weights, x0, x1)):
        _, c, h, wd = a.shape
        desc.layers[l] = _lib.LpipsLayer(a.data_ptr(), b.data_ptr(), w.data_ptr(), c, h, wd)
    desc.dropout_seed = None if seed is None else seed.data_ptr()
    return desc


def _check_head(x0: list[Tensor], x1: list[Tensor], weights: list[Tensor]) -> None:
    if not 1 <= len(x0) <= 5 or len(x1) != len(x0) or len(weights) != len(x0):
        raise ValueError(f"lpips_head: expected 1 to 5 layers on each side with one weight each, got {len(x0)}, "
                         f"{len(x1)} and {len(weights)}")
    dev = x0[0].device
    for l, (a, b, w) in enumerate(zip(x0, x1, weights)):
        if a.dim() != 4 or a.shape != b.shape or a.shape[0] != x0[0].shape[0] or w.numel() != a.shape[1]:
            raise ValueError(f"lpips_head: layer {l}: expected two [N, C, H, W] features of one shape and a [C] "
                             f"weight, got {tuple(a.shape)}, {tuple(b.shape)} and {tuple(w.shape)}")
        if any(t.dtype != torch.float32 for t in (a, b, w)):
            raise ValueError(f"lpips_head: layer {l}: expected float32, got {a.dtype}, {b.dtype} and {w.dtype}")
        if not all(t.is_cuda and t.device == dev for t in (a, b, w)):
            raise ValueError(f"lpips_head: layer {l}: expected CUDA tensors on one device ({dev}), got {a.device}, "
                             f"{b.device} and {w.device}; there is no CPU path")


def lpips_head(x0: list[Tensor], x1: list[Tensor], weights: list[Tensor], seed: Tensor | None = None) -> Tensor:
    """The fused distance head: [N] = sum over layers of the mean over pixels of sum_c w_c m u_c^2, u the difference
    of the channel-normalised features x0[l], x1[l] [N, C, H, W] (float32 CUDA), weights[l] [C].  `seed` (a one-element
    int64 CUDA tensor) switches dropout on; None is eval.  Differentiable in the features of either side."""
    _check_head(x0, x1, weights)
    x0 = [t.contiguous() for t in x0]
    x1 = [t.contiguous() for t in x1]
    weights = [w.detach().reshape(-1).contiguous() for w in weights]
    return _LpipsHead.apply(seed, len(x0), *weights, *x0, *x1)


def _check_images(in0: Tensor, in1: Tensor) -> None:
    if in0.dim() != 4 or in0.shape != in1.shape or in0.shape[1] != 3:
        raise ValueError(f"lpips: expected two [N, 3, H, W] images of one shape, got {tuple(in0.shape)} and "
                         f"{tuple(in1.shape)}")
    if in0.dtype != torch.float32 or in1.dtype != torch.float32:
        raise ValueError(f"lpips: expected float32 images, got {in0.dtype} and {in1.dtype}")
    if in0.shape[-2] < MIN_SIZE or in0.shape[-1] < MIN_SIZE:
        raise ValueError(f"lpips: images must be at least {MIN_SIZE} x {MIN_SIZE} (relu5_3 is then 1 x 1), got "
                         f"{tuple(in0.shape[-2:])}")
    if not (in0.is_cuda and in1.is_cuda) or in0.device != in1.device:
        raise ValueError(f"lpips: expected CUDA tensors on one device, got {in0.device} and {in1.device}; there is "
                         f"no CPU path")


class Lpips(nn.Module):
    """LPIPS(net="vgg") of the lpips package: `forward(in0, in1, normalize=False) -> [N, 1, 1, 1]`.

    State-dict keys: `scaling_layer.shift/scale`, `net.slice{1..5}.{i}.weight/bias`, `lin{0..4}.model.1.weight`
    (the package's; its duplicate `lins.{k}.*` keys are accepted and dropped on load).  A new module has torch's
    default initialisation; `from_files` loads the real weights.  No parameter requires grad (as in the package);
    the lin weights feed the fused head, which computes no weight gradient.  `.train()` switches on the head's
    dropout, as the package's Dropout modules are switched on by a LightningModule's `.train()`."""

    def __init__(self) -> None:
        super().__init__()
        self.scaling_layer = ScalingLayer()
        self.net = Vgg16()
        for k, c in enumerate(CHANNELS):
            setattr(self, f"lin{k}", NetLinLayer(c))
        for p in self.parameters():
            p.requires_grad_(False)
        self._register_load_state_dict_pre_hook(_drop_duplicate_lins)

    def lin_weights(self) -> list[Tensor]:
        return [getattr(self, f"lin{k}").model[1].weight.reshape(-1) for k in range(5)]

    def features(self, x: Tensor, normalize: bool) -> list[Tensor]:
        if normalize:
            x = 2 * x - 1
        return self.net(self.scaling_layer(x))

    def forward(self, in0: Tensor, in1: Tensor, normalize: bool = False) -> Tensor:
        _check_images(in0, in1)
        feats = []
        for x in (in0, in1):
            if x.requires_grad or not torch.is_grad_enabled():
                feats.append(self.features(x, normalize))
            else:
                with torch.no_grad():
                    feats.append(self.features(x, normalize))
        seed = None
        if self.training:
            seed = torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64, device=in0.device)
        return lpips_head(feats[0], feats[1], self.lin_weights(), seed)[:, None, None, None]

    @classmethod
    def from_files(cls, vgg16_path: str | Path | None = None, lin_path: str | Path | None = None) -> "Lpips":
        """The module with torchvision's VGG16 weights (`features.{i}.*` keys of `vgg16-397923af.pth`) and the lpips
        package's lin weights (`lin{k}.model.1.weight` of `weights/v0.1/vgg.pth`).  An omitted path is looked up
        where those files already live: `torch.hub.get_dir()/checkpoints/vgg16-397923af.pth` and the installed
        `lpips` package's directory (found without importing it).  Nothing is downloaded: a missing file raises
        FileNotFoundError naming it and where it goes."""
        vgg16_path = Path(vgg16_path) if vgg16_path is not None else default_vgg16_path()
        lin_path = Path(lin_path) if lin_path is not None else default_lin_path()
        for path, what in ((vgg16_path, f"torchvision's VGG16 weights ({VGG16_FILE}; torchvision puts it in "
                                         f"torch.hub.get_dir()/checkpoints)"),
                           (lin_path, "the lpips package's lin weights (weights/v0.1/vgg.pth inside the installed "
                                      "lpips package)")):
            if path is None or not path.is_file():
                name = path if path is not None else "weights/v0.1/vgg.pth (no lpips package is installed)"
                raise FileNotFoundError(f"Lpips.from_files: {name} not found: it should hold {what}. Pass its path "
                                        f"explicitly; weights are never downloaded")
        vgg = torch.load(vgg16_path, map_location="cpu", weights_only=True)
        lin = torch.load(lin_path, map_location="cpu", weights_only=True)
        model = cls()
        sd = {k: v for k, v in model.state_dict().items() if k.startswith("scaling_layer.")}
        sd.update(vgg16_to_module_keys(vgg))
        sd.update({k: v for k, v in lin.items() if k.startswith("lin")})
        model.load_state_dict(sd)
        return model


def vgg16_to_module_keys(vgg: dict[str, Tensor]) -> dict[str, Tensor]:
    """torchvision vgg16 `features.{i}.weight/bias` -> `net.slice{k}.{i}.weight/bias` (classifier keys dropped)."""
    out = {}
    for name, v in vgg.items():
        parts = name.split(".")
        if parts[0] != "features" or len(parts) != 3:
            continue
        i = int(parts[1])
        if i not in _CONVS:
            continue
        k = next(j + 1 for j, (a, b) in enumerate(SLICES) if a <= i < b)
        out[f"net.slice{k}.{i}.{parts[2]}"] = v
    return out


def _drop_duplicate_lins(state_dict, prefix, *args) -> None:
    """The package's LPIPS also registers its lin layers as `lins.{k}`; those keys duplicate `lin{k}`."""
    for k in [k for k in state_dict if k.startswith(prefix + "lins.")]:
        del state_dict[k]


def default_vgg16_path() -> Path:
    return Path(torch.hub.get_dir()) / "checkpoints" / VGG16_FILE


def default_lin_path() -> Path | None:
    spec = importlib.util.find_spec("lpips")
    if spec is None or not spec.submodule_search_locations:
        return None
    return Path(list(spec.submodule_search_locations)[0]) / "weights" / "v0.1" / "vgg.pth"
