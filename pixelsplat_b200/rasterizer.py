"""Host side of the rasterizer: autograd glue over the C ABI (include/pixelsplat_b200.h) and the
drop-in `GaussianRasterizationSettings` / `GaussianRasterizer` pair that the reference imports
at /root/reference/src/model/decoder/cuda_splatting.py:5-8 and calls at :99-124.

PyTorch is plumbing here (device memory, the current stream, autograd bookkeeping); every
arithmetic step of the hot path runs in the CUDA library.  There is no CPU path: tensors that
are not on a CUDA device are rejected.
"""
from __future__ import annotations

import ctypes
import os
import threading
import warnings
import weakref
from typing import NamedTuple, Optional

import torch
from torch import Tensor

from . import _lib
from ._lib import PS_COV_3X3, PS_COV_TRIU6, PS_SH_M3, TILE
from .sh import convention_id

# ------------------------------------------------------------------ instance-capacity policy
# The binning buffers are sized for `capacity` (tile, Gaussian) instances.  The exact count is
# only known on the device; the forward returns it asynchronously through pinned memory.
#   "sync"     (default): wait for the count right after enqueueing the forward (one event wait
#              per *batch* of views -- upstream syncs once per view) and transparently re-run with
#              a larger buffer if it overflowed.  Always correct.
#   "deferred": a forward that will be followed by a backward (grad enabled, an input requires grad)
#              does not block; its count is verified when its backward starts AND at the start of the
#              next forward of the same shape, whichever comes first, and a RuntimeError is raised
#              if it had overflowed.  Forwards with no backward coming (inference) are always checked
#              synchronously, so a truncated image is never returned silently.
_CHECK_MODE = os.environ.get("PIXELSPLAT_B200_CAPACITY_CHECK", "sync")
_HEADROOM = 1.25        # capacity kept for the next call of a shape = headroom x the instances it needed
_capacity_hint: dict[tuple, int] = {}
_segment_hint: dict[tuple, int] = {}
_pending: dict[tuple, "weakref.ref"] = {}       # last deferred (unverified) state per shape key

# Pinned host slots for the asynchronous instance count: every RasterOutputState OWNS its slot for as
# long as it lives (a captured CUDA graph keeps writing to it on every replay) and hands it back to the
# pool when it is garbage collected -- no ring, no aliasing.
_PINNED_BLOCK = 64
_pinned_blocks: list[Tensor] = []
_pinned_free: list[Tensor] = []
_pool_lock = threading.Lock()

# SH convention the rasterizer evaluates coefficients in (include/pixelsplat_b200.h PS_SH_BASIS_*).
_SH_BASIS = convention_id(os.environ.get("PIXELSPLAT_B200_SH_BASIS", "3dgs"))


def set_capacity_check(mode: str) -> None:
    global _CHECK_MODE
    if mode not in ("sync", "deferred"):
        raise ValueError("mode must be 'sync' or 'deferred'")
    _CHECK_MODE = mode


def set_capacity_headroom(factor: float) -> None:
    """Head-room factor (>= 1) applied to the instance count a forward needed when sizing the binning buffers of
    the NEXT forward of the same shape (default 1.25).  A step captured into a CUDA graph freezes its capacity,
    so a training loop whose Gaussians move between replays should capture with a generous factor (the count is
    still checked after every replay: `RasterOutputState.verify`)."""
    global _HEADROOM
    if not factor >= 1.0:
        raise ValueError("headroom factor must be >= 1")
    _HEADROOM = float(factor)


def set_sh_basis(convention) -> None:
    """Process-wide default SH convention of the rasterizer: "3dgs" (upstream 3DGS basis, the default) or
    "e3nn" (the basis the reference's rotate_sh rotates in; see pixelsplat_b200/sh.py).  The drop-in
    `GaussianRasterizationSettings` has no field for it (it mirrors the extension's NamedTuple), hence a
    module switch; `rasterize_gaussians(sh_basis=...)` overrides it per call."""
    global _SH_BASIS
    _SH_BASIS = convention_id(convention)


def get_sh_basis() -> int:
    return _SH_BASIS


def _pinned_slot() -> Tensor:
    with _pool_lock:
        if not _pinned_free:
            block = torch.zeros(2 * _PINNED_BLOCK, dtype=torch.int64).pin_memory()
            _pinned_blocks.append(block)
            _pinned_free.extend(block[2 * i:2 * i + 2] for i in range(_PINNED_BLOCK))
        return _pinned_free.pop()


def _release_slot(slot: Tensor) -> None:
    with _pool_lock:
        _pinned_free.append(slot)


def _ptr(t: Optional[Tensor]):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _req(t: Tensor, name: str, shape: tuple) -> Tensor:
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor (pixelsplat_b200 has no CPU path)")
    if t.dtype != torch.float32:
        raise ValueError(f"{name} must be float32, got {t.dtype}")
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name} has shape {tuple(t.shape)}, expected {tuple(shape)}")
    return t.contiguous()


class RasterOutputState:
    """Opaque forward->backward state (the geom / binning / image byte buffers)."""

    def __init__(self, desc, geom, binning, image, n_host, event, hint_key=None):
        self.desc, self.geom, self.binning, self.image = desc, geom, binning, image
        self.n_host, self.event, self.hint_key = n_host, event, hint_key
        self.verified = False
        # the slot returns to the pool when this state dies; until then nothing else writes to it
        weakref.finalize(self, _release_slot, n_host)

    def raw_state(self) -> _lib.RasterState:
        return _lib.RasterState(self.geom.data_ptr(), self.geom.numel(), self.binning.data_ptr(),
                                self.binning.numel(), self.image.data_ptr(), self.image.numel())

    def num_instances(self) -> int:
        """Blocks until the forward's instance count has reached the host.  For a forward that was
        captured into a CUDA graph there is no event: the caller synchronises after a replay."""
        if self.event is not None:
            self.event.synchronize()
        if self.hint_key is not None:
            _segment_hint[self.hint_key] = max(int(self.n_host[1].item()), 1)
        return int(self.n_host[0].item())

    def verify(self) -> None:
        """Raises if the binning overflowed its buffer.  Inside a CUDA-graph capture nothing can be
        waited on, so the check is skipped there: call `verify()` again after replaying and
        synchronising (bench.py does)."""
        if self.verified:
            return
        if self.event is None and torch.cuda.is_current_stream_capturing():
            return
        n = self.num_instances()
        if n > self.desc.instance_capacity:
            if self.hint_key is not None:
                _capacity_hint[self.hint_key] = int(n * _HEADROOM) + 4096
            raise RuntimeError(
                f"rasterizer binning overflow: {n} instances needed, capacity was "
                f"{self.desc.instance_capacity}; the forward result of this call is invalid. "
                "Re-run (the capacity hint has been raised) or use the 'sync' capacity check.")
        self.verified = True

    # -- introspection for parity tests (bit-exact tile/bin indices) --
    def intermediates(self) -> dict:
        self.verify()
        d = self.desc
        lay = _lib.layout(d)
        vt = d.n_scenes * d.views_per_scene
        vp = vt * d.n_gaussians
        gx, gy = (d.width + TILE - 1) // TILE, (d.height + TILE - 1) // TILE
        tiles = gx * gy
        n = self.num_instances()

        def view(buf, off, dtype, count, shape):
            nbytes = count * torch.empty((), dtype=dtype).element_size()
            return buf[off:off + nbytes].view(dtype).reshape(shape)

        P = d.n_gaussians
        hw = d.height * d.width
        return dict(
            depth=view(self.geom, lay.depth, torch.float32, vp, (vt, P)),
            radii=view(self.geom, lay.radii, torch.int32, vp, (vt, P)),
            xy=view(self.geom, lay.xy, torch.float32, vp * 2, (vt, P, 2)),
            conic_opacity=view(self.geom, lay.conic_opacity, torch.float32, vp * 4, (vt, P, 4)),
            rgb=view(self.geom, lay.rgb, torch.float32, vp * 4, (vt, P, 4))[..., :3],
            rect=view(self.geom, lay.rect, torch.int16, vp * 4, (vt, P, 4)),
            clamped=view(self.geom, lay.clamped, torch.uint8, vp, (vt, P)),
            tile_count=view(self.geom, lay.tile_count, torch.int32, vt * tiles, (vt, tiles)),
            tile_start=view(self.geom, lay.tile_start, torch.int32, vt * tiles, (vt, tiles)),
            keys=view(self.binning, lay.keys, torch.int64, n, (n,)),
            final_T=view(self.image, lay.final_T, torch.float32, vt * hw, (vt, d.height, d.width)),
            n_contrib=view(self.image, lay.n_contrib, torch.int32, vt * hw, (vt, d.height, d.width)),
            color=view(self.image, lay.color, torch.float32, vt * 3 * hw, (vt, 3, d.height, d.width)),
            # (T, Cr, Cg, Cb) in front of list runs 1..3; written only when the forward cut lists into runs
            run_state=view(self.image, lay.run_state, torch.float32, vt * 3 * hw * 4, (vt, 3, d.height, d.width, 4)),
            # depth channel and the depth in front of list runs 1..3 (None when the forward had no depth channel)
            depth_image=view(self.image, lay.depth_image, torch.float32, vt * hw, (vt, d.height, d.width))
            if d.depth_mode else None,
            run_depth=view(self.image, lay.run_depth, torch.float32, vt * 3 * hw, (vt, 3, d.height, d.width))
            if d.depth_mode else None,
            # per on-screen pair: d(colour channel before the clamp) / d(normalised view direction), rows (x, y, z)
            # (None with precomputed colours)
            sh_jacobian=view(self.geom, lay.sh_jacobian, torch.float32, vp * 12, (vt, P, 3, 4))[..., :3]
            if d.sh_coeffs else None,
            num_instances=n,
        )

    def depth_image(self) -> Tensor:
        """The composited depth channel [S*V, H, W] (a view of the image state; depth forwards only)."""
        d = self.desc
        off = _lib.layout(d).depth_image
        n = d.n_scenes * d.views_per_scene * d.height * d.width
        return self.image[off:off + 4 * n].view(torch.float32).reshape(-1, d.height, d.width)


def _sync_deterministic() -> None:
    """Carries torch.use_deterministic_algorithms into the library's "deterministic" option (fixed-order composite
    backward and loss epilogue; include/pixelsplat_b200.h), setting it only when it differs.  Called before every
    forward and backward enqueues.  The legacy compositor (composite_impl = 1) has no fixed-order form; under the
    flag it is treated as torch treats an op without a deterministic implementation: RuntimeError, or with
    warn_only=True a warning and today's path."""
    want = 1 if torch.are_deterministic_algorithms_enabled() else 0
    if want and _lib.get_option("composite_impl") == 1:
        msg = ("pixelsplat_b200 rasterizer with the legacy compositor (composite_impl = 1) does not have a "
               "deterministic implementation, but you set 'torch.use_deterministic_algorithms(True)'. You can turn "
               "off determinism just for this operation, or you can use the 'warn_only=True' option, if that's "
               "acceptable for your application. Select the warp-task compositor (composite_impl = 2, the default) "
               "for deterministic rasterizer gradients.")
        if not torch.is_deterministic_algorithms_warn_only_enabled():
            raise RuntimeError(msg)
        warnings.warn(msg)
        want = 0
    if _lib.get_option("deterministic") != want:
        _lib.set_option("deterministic", want)


class _Config(NamedTuple):
    """The non-tensor settings of one rasterizer call: the ps_raster_desc fields the caller chooses, and whether
    the colour image is written."""
    S: int
    V: int
    P: int
    M: int
    degree: int
    sh_layout: int
    cov_layout: int
    H: int
    W: int
    sort_impl: int
    sh_basis: int
    depth_mode: int
    want_color: bool


def _raster_inputs(means, cov, opac, sh, cams) -> _lib.RasterInputs:
    opt = lambda k: cams[k].data_ptr() if cams.get(k) is not None else None
    return _lib.RasterInputs(
        means.data_ptr(), cov.data_ptr(), opac.data_ptr(), sh.data_ptr(),
        cams["viewmatrix"].data_ptr(), cams["projmatrix"].data_ptr(), cams["campos"].data_ptr(),
        cams["tanfov"].data_ptr(), cams["background"].data_ptr(), opt("scene_scale"), opt("near_far"))


def _forward(means, cov, opac, sh, cams, cfg: _Config, backward_follows: bool, target: Optional[Tensor]):
    """Enqueues the forward on the current stream of the Gaussians' device.  Returns (color | None, radii, state,
    sums | None): `sums` are the [S*V, 2, LOSS_SLOTS] partial sums of the loss epilogue, run when a `target` is
    given.  With cfg.depth_mode != 0 the state also holds the depth channel (RasterOutputState.depth_image)."""
    dev = means.device
    S, V, P, H, W = cfg.S, cfg.V, cfg.P, cfg.H, cfg.W
    key = (dev.index, S, V, P, H, W)
    with torch.cuda.device(dev):            # the library works on the CURRENT device
        capturing = torch.cuda.is_current_stream_capturing()
        prev = _pending.pop(key, None)
        if prev is not None and not capturing:
            prev = prev()
            if prev is not None:
                prev.verify()               # deferred check of the previous forward of this shape
        capacity = _capacity_hint.get(key)
        if capacity is None:
            capacity = max(4096, 3 * S * V * P)
        stream = torch.cuda.current_stream(dev)
        _sync_deterministic()               # before the sizes: the mode changes the image state
        while True:
            desc = _lib.RasterDesc(S, V, P, cfg.M, cfg.degree, cfg.sh_layout, cfg.cov_layout, H, W, cfg.sort_impl,
                                   min(_segment_hint.get(key, 0), 1 << 30), capacity, cfg.sh_basis, cfg.depth_mode)
            sz = _lib.sizes(desc)
            geom = torch.empty(sz.geom_bytes, dtype=torch.uint8, device=dev)
            binning = torch.empty(sz.binning_bytes, dtype=torch.uint8, device=dev)
            image = torch.empty(sz.image_bytes, dtype=torch.uint8, device=dev)
            color = torch.empty((S * V, 3, H, W), dtype=torch.float32, device=dev) if cfg.want_color else None
            radii = torch.empty((S * V, P), dtype=torch.int32, device=dev)
            n_host = _pinned_slot()
            inputs = _raster_inputs(means, cov, opac, sh, cams)
            state = _lib.RasterState(geom.data_ptr(), geom.numel(), binning.data_ptr(), binning.numel(),
                                     image.data_ptr(), image.numel())
            args = [ctypes.byref(desc), ctypes.byref(inputs), ctypes.byref(state)]
            if target is None:
                fn, sums = _lib.lib.ps_raster_forward, None
            else:
                fn = _lib.lib.ps_raster_forward_loss
                sums = torch.empty((S * V, 2, _lib.LOSS_SLOTS), dtype=torch.float32, device=dev)
                loss = _lib.RasterLoss(target.data_ptr(), sums.data_ptr())
                args.append(ctypes.byref(loss))
            rc = fn(*args, _ptr(color), _ptr(radii), ctypes.c_void_p(n_host.data_ptr()),
                    ctypes.c_void_p(stream.cuda_stream))
            _lib.check(rc, fn.__name__)
            if torch.cuda.is_current_stream_capturing():
                # CUDA-graph capture: shapes and capacity are frozen into the graph; the count still
                # lands in pinned memory on every replay and is checked by the caller afterwards
                if key not in _capacity_hint:
                    raise RuntimeError("run this shape once eagerly before capturing it in a CUDA graph "
                                       "(the binning capacity must be known)")
                return color, radii, RasterOutputState(desc, geom, binning, image, n_host, None, key), sums
            event = torch.cuda.Event()
            event.record(stream)
            st = RasterOutputState(desc, geom, binning, image, n_host, event, key)
            if _CHECK_MODE == "deferred" and key in _capacity_hint and backward_follows:
                _pending[key] = weakref.ref(st)
                return color, radii, st, sums
            n = st.num_instances()
            if n <= capacity:
                st.verified = True
                # keep ~25 % head-room for the next call of the same shape
                _capacity_hint[key] = max(_capacity_hint.get(key, 0), int(n * _HEADROOM) + 4096)
                return color, radii, st, sums
            capacity = int(n * _HEADROOM) + 4096
            _capacity_hint[key] = capacity


class _Rasterize(torch.autograd.Function):
    """One forward (+ backward) of S scenes x V views.  Optional parts of the same pass: the squared-error epilogue
    against `target` [S*V, 3, H, W] (SURVEY.md 8 row f-4) and the depth channel (cfg.depth_mode != 0).
    Outputs (color, depth, radii, sse, sse_clipped):
      color [S*V, 3, H, W]  differentiable without a target; detached with one (empty when not cfg.want_color);
      depth [S*V, H, W]     differentiable; None without the depth channel;
      sse [S*V]             sum over the view's pixels and channels of (C - target)^2, differentiable; its gradient
                            g reaches the composite backward as the per-view scale 2 g of (C - target), formed
                            in-kernel.  sse_clipped is the same on images clipped to [0, 1].  Both None without a
                            target.
    `means2d` [S*V, P, 3] is upstream's gradient holder: it takes no part in the forward and receives the gradient
    with respect to the projected means.  When no gradient reaches `depth` the backward is the colour-only one
    (ps_raster_backward without a target, ps_raster_backward_loss with one).
    The four camera arrays (viewmatrix, projmatrix, campos, tanfov; the same tensors as in `cams`) are inputs of the
    Function: when one of them requires grad the backward also returns the camera gradients (ps_raster_camera_grads,
    include/pixelsplat_b200.h); otherwise its launches and bits are those of the Gaussian-only backward.  When a
    camera array requires grad and none of means, cov, opac, sh and means2d does, the backward is the camera-only one:
    no Gaussian gradient is allocated or formed, and None is returned for each.  background, scene_scale and near_far
    are not differentiated."""

    @staticmethod
    def forward(ctx, means, cov, opac, sh, means2d, target, viewmatrix, projmatrix, campos, tanfov, cams,
                cfg: _Config, state_out):
        ctx.set_materialize_grads(False)
        backward_follows = any(ctx.needs_input_grad[:5]) or any(ctx.needs_input_grad[6:10])
        color, radii, st, sums = _forward(means, cov, opac, sh, cams, cfg, backward_follows, target)
        ctx.save_for_backward(means, cov, opac, sh, target)
        ctx.cams, ctx.st = cams, st
        if state_out is not None:
            state_out.append(st)
        depth = st.depth_image().clone() if cfg.depth_mode else None
        sse = sse_clipped = None
        if target is not None:
            totals = sums.sum(dim=-1)                                # [S*V, 2]
            sse, sse_clipped = totals[:, 0].contiguous(), totals[:, 1].contiguous()
            if color is None:
                color = torch.empty(0, device=means.device)
            ctx.mark_non_differentiable(color, sse_clipped)
        ctx.mark_non_differentiable(radii)
        return color, depth, radii, sse, sse_clipped

    @staticmethod
    def backward(ctx, d_color, d_depth, _d_radii, d_sse, _d_clip):
        means, cov, opac, sh, target = ctx.saved_tensors
        st: RasterOutputState = ctx.st
        st.verify()
        desc = st.desc
        dev = means.device
        VT = desc.n_scenes * desc.views_per_scene
        if target is None:
            # no dL/dC when only the depth reached the loss
            d_color = (torch.zeros((VT, 3, desc.height, desc.width), dtype=torch.float32, device=dev)
                       if d_color is None else d_color.to(torch.float32).contiguous())
            scale = None
        else:
            scale = (torch.zeros(VT, dtype=torch.float32, device=dev) if d_sse is None
                     else (2.0 * d_sse).to(torch.float32).contiguous())
        _sync_deterministic()               # before the sizes: the mode changes the backward scratch
        scratch = torch.empty(_lib.sizes(desc).backward_bytes, dtype=torch.uint8, device=dev)
        if any(ctx.needs_input_grad[:5]) or not any(ctx.needs_input_grad[6:10]):
            d_means, d_cov = torch.empty_like(means), torch.empty_like(cov)
            d_opac, d_sh = torch.empty_like(opac), torch.empty_like(sh)
            d_m2d = (torch.empty((VT, desc.n_gaussians, 3), dtype=torch.float32, device=dev)
                     if ctx.needs_input_grad[4] else None)
        else:
            # frozen Gaussians (test-time pose alignment): the camera-only backward forms no Gaussian gradient
            d_means = d_cov = d_opac = d_sh = d_m2d = None
        inputs = _raster_inputs(means, cov, opac, sh, ctx.cams)
        grads = _lib.RasterGrads(*[None if t is None else t.data_ptr() for t in (d_means, d_cov, d_opac, d_sh, d_m2d)])
        d_cams = [None] * 4                 # viewmatrix, projmatrix, campos, tanfov
        if any(ctx.needs_input_grad[6:10]):
            widths = (16, 16, 3, 2)
            d_cams = [torch.empty((VT, n), dtype=torch.float32, device=dev) if ctx.needs_input_grad[6 + i] else None
                      for i, n in enumerate(widths)]
            cam_ws = torch.empty(_lib.camera_workspace_bytes(desc), dtype=torch.uint8, device=dev)
            cam = _lib.RasterCameraGrads(*[None if t is None else t.data_ptr() for t in d_cams], cam_ws.data_ptr(),
                                         cam_ws.numel())
            grads.camera = ctypes.pointer(cam)
        state = st.raw_state()
        if d_depth is not None:
            d_depth = d_depth.to(torch.float32).contiguous()
            fn = _lib.lib.ps_raster_backward_depth
            args = (_ptr(d_color if target is None else None), _ptr(target), _ptr(scale), _ptr(d_depth))
        elif target is None:
            fn, args = _lib.lib.ps_raster_backward, (_ptr(d_color),)
        else:
            fn, args = _lib.lib.ps_raster_backward_loss, (_ptr(target), _ptr(scale))
        stream = torch.cuda.current_stream(dev)
        rc = _lib.on_device(dev, fn, ctypes.byref(desc), ctypes.byref(inputs), ctypes.byref(state), *args,
                            _ptr(scratch), scratch.numel(), ctypes.byref(grads), ctypes.c_void_p(stream.cuda_stream))
        _lib.check(rc, fn.__name__)
        return (d_means, d_cov, d_opac, d_sh, d_m2d, None, *d_cams, None, None, None)


def _rasterize(means, covariances, opacities, colors, *, viewmatrix, projmatrix, campos, tanfov, background,
               image_shape, views_per_scene, sh_degree, use_sh=True, sh_layout=PS_SH_M3, scene_scale=None,
               sort_impl=0, state_out=None, sh_basis=None, target=None, depth_mode=None, near_far=None,
               want_color=True, means2d=None):
    """Argument checks of every rasterizer entry point, then one _Rasterize: returns its (color, depth, radii, sse,
    sse_clipped).  `depth_mode` is a key of _lib.DEPTH_MODES (None: no depth channel)."""
    if means.dim() != 3 or means.shape[-1] != 3:
        raise ValueError(f"means must be [S, P, 3], got {tuple(means.shape)}")
    S, P, _ = means.shape
    V = int(views_per_scene)
    H, W = map(int, image_shape)
    means = _req(means, "means", (S, P, 3))
    if covariances.dim() == 4:
        cov_layout = PS_COV_3X3
        covariances = _req(covariances, "covariances", (S, P, 3, 3))
    else:
        cov_layout = PS_COV_TRIU6
        covariances = _req(covariances, "covariances", (S, P, 6))
    opacities = _req(opacities.reshape(S, P), "opacities", (S, P))
    if use_sh:
        if colors.dim() != 4:
            raise ValueError("SH colours must be [S, P, M, 3] or [S, P, 3, M]")
        M = colors.shape[2] if sh_layout == PS_SH_M3 else colors.shape[3]
        shape = (S, P, M, 3) if sh_layout == PS_SH_M3 else (S, P, 3, M)
        colors = _req(colors, "sh", shape)
    else:
        M = 0
        colors = _req(colors, "colors_precomp", (S, P, 3))
    VT = S * V
    cams = dict(
        viewmatrix=_req(viewmatrix.reshape(VT, 16), "viewmatrix", (VT, 16)),
        projmatrix=_req(projmatrix.reshape(VT, 16), "projmatrix", (VT, 16)),
        campos=_req(campos, "campos", (VT, 3)),
        tanfov=_req(tanfov, "tanfov", (VT, 2)),
        background=_req(background, "background", (VT, 3)),
        scene_scale=None if scene_scale is None else _req(scene_scale, "scene_scale", (VT,)),
    )
    if depth_mode not in _lib.DEPTH_MODES:
        raise ValueError(f"depth_mode must be one of {[k for k in _lib.DEPTH_MODES if k]}")
    mode = _lib.DEPTH_MODES[depth_mode]
    if near_far is not None:
        cams["near_far"] = _req(near_far, "near_far", (VT, 2))
    elif mode in (3, 4):
        raise ValueError("depth modes relative_disparity and log need near_far [S*V, 2]")
    if target is not None:
        target = _req(target, "target", (VT, 3, H, W))
    if means2d is not None and tuple(means2d.shape) != (VT, P, 3):
        raise ValueError(f"means2d must be [S*V, P, 3], got {tuple(means2d.shape)}")
    cfg = _Config(S, V, P, M, int(sh_degree), sh_layout, cov_layout, H, W, int(sort_impl),
                  _SH_BASIS if sh_basis is None else convention_id(sh_basis), mode, bool(want_color) or target is None)
    return _Rasterize.apply(means, covariances, opacities, colors, means2d, target, cams["viewmatrix"],
                            cams["projmatrix"], cams["campos"], cams["tanfov"], cams, cfg, state_out)


def rasterize_gaussians(
    means: Tensor,            # [S, P, 3]
    covariances: Tensor,      # [S, P, 6] (triu) or [S, P, 3, 3]
    opacities: Tensor,        # [S, P]
    colors: Tensor,           # SH [S, P, M, 3] / [S, P, 3, M], or precomputed RGB [S, P, 3]
    *,
    viewmatrix: Tensor,       # [S*V, 16] or [S*V, 4, 4], column-major flattening (see header)
    projmatrix: Tensor,       # same
    campos: Tensor,           # [S*V, 3]
    tanfov: Tensor,           # [S*V, 2]
    background: Tensor,       # [S*V, 3]
    image_shape: tuple[int, int],
    views_per_scene: int,
    sh_degree: int,
    use_sh: bool = True,
    sh_layout: int = PS_SH_M3,
    scene_scale: Optional[Tensor] = None,   # [S*V]
    sort_impl: int = 0,
    state_out: Optional[list] = None,
    means2d: Optional[Tensor] = None,       # [S*V, P, 3] gradient holder (upstream's means2D)
    sh_basis=None,                          # "3dgs" / "e3nn"; None = the module default (set_sh_basis)
) -> tuple[Tensor, Tensor]:
    """Batched differentiable rasterization: S scenes x V views in one set of launches.
    Returns (color [S*V, 3, H, W], radii [S*V, P] int32).  Differentiable with respect to the Gaussians and to
    viewmatrix, projmatrix, campos and tanfov (tanfov only through the focal lengths; see ps_raster_camera_grads);
    not with respect to background or scene_scale."""
    color, _, radii, _, _ = _rasterize(
        means, covariances, opacities, colors, viewmatrix=viewmatrix, projmatrix=projmatrix, campos=campos,
        tanfov=tanfov, background=background, image_shape=image_shape, views_per_scene=views_per_scene,
        sh_degree=sh_degree, use_sh=use_sh, sh_layout=sh_layout, scene_scale=scene_scale, sort_impl=sort_impl,
        state_out=state_out, sh_basis=sh_basis, means2d=means2d)
    return color, radii


def rasterize_gaussians_mse(means: Tensor, covariances: Tensor, opacities: Tensor, colors: Tensor, target: Tensor, *,
                            viewmatrix: Tensor, projmatrix: Tensor, campos: Tensor, tanfov: Tensor, background: Tensor,
                            image_shape: tuple[int, int], views_per_scene: int, sh_degree: int, use_sh: bool = True,
                            sh_layout: int = PS_SH_M3, scene_scale: Optional[Tensor] = None, sort_impl: int = 0,
                            state_out: Optional[list] = None, sh_basis=None, want_color: bool = True):
    """rasterize_gaussians + the loss epilogue: returns (sse [S*V] differentiable, sse_clipped [S*V], color
    [S*V, 3, H, W] detached (empty when want_color=False), radii).  `target` is [S*V, 3, H, W]."""
    color, _, radii, sse, sse_clipped = _rasterize(
        means, covariances, opacities, colors, viewmatrix=viewmatrix, projmatrix=projmatrix, campos=campos,
        tanfov=tanfov, background=background, image_shape=image_shape, views_per_scene=views_per_scene,
        sh_degree=sh_degree, use_sh=use_sh, sh_layout=sh_layout, scene_scale=scene_scale, sort_impl=sort_impl,
        state_out=state_out, sh_basis=sh_basis, target=target, want_color=want_color)
    return sse, sse_clipped, color, radii


def rasterize_gaussians_with_depth(
        means: Tensor, covariances: Tensor, opacities: Tensor, colors: Tensor, *, viewmatrix: Tensor,
        projmatrix: Tensor, campos: Tensor, tanfov: Tensor, background: Tensor, image_shape: tuple[int, int],
        views_per_scene: int, sh_degree: int, depth_mode: str, near_far: Optional[Tensor] = None,
        use_sh: bool = True, sh_layout: int = PS_SH_M3, scene_scale: Optional[Tensor] = None, sort_impl: int = 0,
        state_out: Optional[list] = None, sh_basis=None, target: Optional[Tensor] = None, want_color: bool = True):
    """rasterize_gaussians with a depth channel composited in the same pass: the Gaussians' camera-space depth in
    world units (view-space z / scene_scale), as `depth_mode` "depth" | "disparity" | "relative_disparity" | "log"
    (the values render_depth_cuda composites), blended with the colour's alphas over a zero background.
    `near_far` [S*V, 2] (world units) is needed by the last two modes.
    Returns (color [S*V, 3, H, W], depth [S*V, H, W], radii), both images differentiable.  With `target`
    [S*V, 3, H, W] the loss epilogue of rasterize_gaussians_mse runs too and the result is (sse [S*V]
    differentiable, sse_clipped, color detached (empty when want_color=False), depth differentiable, radii)."""
    if depth_mode is None:
        raise ValueError("rasterize_gaussians_with_depth needs a depth_mode")
    color, depth, radii, sse, sse_clipped = _rasterize(
        means, covariances, opacities, colors, viewmatrix=viewmatrix, projmatrix=projmatrix, campos=campos,
        tanfov=tanfov, background=background, image_shape=image_shape, views_per_scene=views_per_scene,
        sh_degree=sh_degree, use_sh=use_sh, sh_layout=sh_layout, scene_scale=scene_scale, sort_impl=sort_impl,
        state_out=state_out, sh_basis=sh_basis, target=target, depth_mode=depth_mode, near_far=near_far,
        want_color=want_color)
    if target is None:
        return color, depth, radii
    return sse, sse_clipped, color, depth, radii


# ------------------------------------------------------------------ drop-in extension surface
class GaussianRasterizationSettings(NamedTuple):
    """Field-for-field the NamedTuple the reference constructs by keyword at
    cuda_splatting.py:99-112."""
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: Tensor
    scale_modifier: float
    viewmatrix: Tensor
    projmatrix: Tensor
    sh_degree: int
    campos: Tensor
    prefiltered: bool
    debug: bool


def _cov_from_scale_rotation(scales: Tensor, rotations: Tensor, mod: float) -> Tensor:
    """Upstream computeCov3D: quaternion (r, x, y, z) used un-normalised; Sigma = (S R)^T (S R)."""
    r, x, y, z = rotations.unbind(-1)
    R = torch.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
    M = R * (mod * scales)[:, None, :]
    sigma = M @ M.transpose(1, 2)
    row, col = torch.triu_indices(3, 3, device=sigma.device)
    return sigma[:, row, col]


class GaussianRasterizer(torch.nn.Module):
    """Same constructor / forward signature and error behaviour as the extension class the
    reference instantiates at cuda_splatting.py:113."""

    def __init__(self, raster_settings: GaussianRasterizationSettings):
        super().__init__()
        self.raster_settings = raster_settings

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                rotations=None, cov3D_precomp=None):
        rs = self.raster_settings
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception("Please provide excatly one of either SHs or precomputed colors!")
        if ((scales is None or rotations is None) and cov3D_precomp is None) or (
                (scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception(
                "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
        if means3D.dim() != 2 or means3D.shape[-1] != 3:
            raise ValueError("means3D must have dimensions (num_points, 3)")
        P = means3D.shape[0]
        dev = means3D.device
        cov6 = cov3D_precomp if cov3D_precomp is not None else _cov_from_scale_rotation(
            scales, rotations, float(rs.scale_modifier))
        f32 = dict(dtype=torch.float32, device=dev)
        tanfov = torch.tensor([[float(rs.tanfovx), float(rs.tanfovy)]], **f32)
        color, radii = rasterize_gaussians(
            means3D[None], cov6[None], opacities.reshape(1, P),
            (shs if shs is not None else colors_precomp)[None],
            viewmatrix=rs.viewmatrix.reshape(1, 16).to(**f32),
            projmatrix=rs.projmatrix.reshape(1, 16).to(**f32),
            campos=rs.campos.reshape(1, 3).to(**f32), tanfov=tanfov,
            background=rs.bg.reshape(1, 3).to(**f32),
            image_shape=(int(rs.image_height), int(rs.image_width)), views_per_scene=1,
            sh_degree=int(rs.sh_degree), use_sh=shs is not None, sh_layout=PS_SH_M3,
            means2d=None if means2D is None else means2D[None])
        return color[0], radii[0]
