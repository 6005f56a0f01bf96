"""ctypes binding of include/pixelsplat_b200.h.

There is no fallback: if the CUDA library is missing, importing this module raises.  Build it
with `python -c "import __graft_entry__ as g; g.build()"` or `make -C pixelsplat_b200/csrc`.
"""
from __future__ import annotations

import ctypes
import os
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ.get("PIXELSPLAT_B200_LIB", _PKG / "_C" / "libpixelsplat_b200.so"))

PS_OK = 0
PS_SH_M3, PS_SH_3M = 0, 1
PS_COV_TRIU6, PS_COV_3X3 = 0, 1
PS_SH_BASIS_3DGS, PS_SH_BASIS_E3NN = 0, 1
PS_ERR_UNSUPPORTED = 3
# ps_raster_desc.depth_mode
DEPTH_MODES = {None: 0, "depth": 1, "disparity": 2, "relative_disparity": 3, "log": 4}
TILE = 16

_ERR_NAMES = {1: "PS_ERR_INVALID_ARGUMENT", 2: "PS_ERR_CUDA", 3: "PS_ERR_UNSUPPORTED"}


class RasterDesc(ctypes.Structure):
    _fields_ = [
        ("n_scenes", ctypes.c_int32), ("views_per_scene", ctypes.c_int32),
        ("n_gaussians", ctypes.c_int32), ("sh_coeffs", ctypes.c_int32),
        ("sh_degree", ctypes.c_int32), ("sh_layout", ctypes.c_int32),
        ("cov_layout", ctypes.c_int32), ("height", ctypes.c_int32), ("width", ctypes.c_int32),
        ("sort_impl", ctypes.c_int32), ("sort_segment_hint", ctypes.c_int32),
        ("instance_capacity", ctypes.c_int64),
        ("sh_basis", ctypes.c_int32), ("depth_mode", ctypes.c_int32),
    ]


class RasterInputs(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in (
        "means", "cov", "opacities", "sh", "viewmatrix", "projmatrix", "campos", "tanfov",
        "background", "scene_scale", "near_far")]


class RasterState(ctypes.Structure):
    _fields_ = [("geom", ctypes.c_void_p), ("geom_bytes", ctypes.c_size_t),
                ("binning", ctypes.c_void_p), ("binning_bytes", ctypes.c_size_t),
                ("image", ctypes.c_void_p), ("image_bytes", ctypes.c_size_t)]


class RasterSizes(ctypes.Structure):
    _fields_ = [(n, ctypes.c_size_t) for n in (
        "geom_bytes", "binning_bytes", "image_bytes", "backward_bytes")]


class RasterLayout(ctypes.Structure):
    _fields_ = [(n, ctypes.c_size_t) for n in (
        "depth", "radii", "xy", "conic_opacity", "rgb", "rect", "clamped", "tile_count",
        "tile_start", "tile_cursor", "n_instances", "vis_pairs", "vis_any", "keys", "keys_alt", "final_T",
        "n_contrib", "cull", "color", "block_hits", "run_hits", "run_state", "depth_image", "run_depth")]


class EpipolarDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in (
        "batch", "views", "grid_h", "grid_w", "samples", "channels", "heads", "pe_dim")]


class EpipolarInputs(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in (
        "features", "segments", "valid", "rel_disparity", "q_feat", "q_pe", "bias")]


class AdapterDesc(ctypes.Structure):
    _fields_ = [("n_views", ctypes.c_int32), ("n_rays", ctypes.c_int32), ("n_samples", ctypes.c_int32),
                ("sh_coeffs", ctypes.c_int32), ("image_h", ctypes.c_int32), ("image_w", ctypes.c_int32),
                ("scale_min", ctypes.c_float), ("scale_max", ctypes.c_float), ("eps", ctypes.c_float),
                ("reserved", ctypes.c_int32)]


class AdapterInputs(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in (
        "extrinsics", "intrinsics", "sh_rotation", "sh_mask", "coordinates", "depths", "raw")]


class RasterLoss(ctypes.Structure):
    _fields_ = [("target", ctypes.c_void_p), ("sums", ctypes.c_void_p)]


LOSS_SLOTS = 64
LPIPS_MAX_LAYERS = 5


class LpipsLayer(ctypes.Structure):
    _fields_ = [("x0", ctypes.c_void_p), ("x1", ctypes.c_void_p), ("weight", ctypes.c_void_p),
                ("C", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32)]


class LpipsDesc(ctypes.Structure):
    _fields_ = [("n_layers", ctypes.c_int32), ("N", ctypes.c_int32), ("layers", LpipsLayer * LPIPS_MAX_LAYERS),
                ("dropout_seed", ctypes.c_void_p)]


class LpipsGrads(ctypes.Structure):
    _fields_ = [("d_x0", ctypes.c_void_p * LPIPS_MAX_LAYERS), ("d_x1", ctypes.c_void_p * LPIPS_MAX_LAYERS)]


class ResampleDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("n_images", "in_h", "in_w", "out_h", "out_w", "taps_h", "taps_v")] + \
        [(n, ctypes.c_void_p) for n in ("images", "flip", "bounds_h", "weights_h", "bounds_v", "weights_v")]


PS_EVAL_RENDER, PS_EVAL_FRAME = 0, 1
EVAL_MAX_IMAGES = 32


class EvalDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("mode", "n_images", "height", "width")] + \
        [(n, ctypes.c_void_p) for n in ("render", "frame_in", "target", "frame_out", "planes", "sse")]


CLIP_ADAM_CHUNK = 4096
CLIP_ADAM_SEGMENT_FIELDS = ("param", "grad", "exp_avg", "exp_avg_sq", "count", "first_chunk")   # 6 x 8 bytes a row


class ClipAdamDesc(ctypes.Structure):
    _fields_ = [("n_segments", ctypes.c_int32), ("reserved", ctypes.c_int32), ("n_chunks", ctypes.c_int64),
                ("warm_up_steps", ctypes.c_int64)] + \
        [(n, ctypes.c_double) for n in ("lr", "beta1", "beta2", "eps", "max_norm")]


class ClipAdamState(ctypes.Structure):
    _fields_ = [("step", ctypes.c_void_p), ("grad_norm", ctypes.c_void_p)]


PS_PLY_REFERENCE, PS_PLY_VIEWER = 0, 1
PLY_SH_TRANSFORM_FLOATS = 84


class PlyDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("mode", "sh_degree", "sh_coeffs", "reserved")] + \
        [("n_gaussians", ctypes.c_int64), ("frame", ctypes.c_double * 9),
         ("sh_transform", ctypes.c_float * PLY_SH_TRANSFORM_FLOATS)] + \
        [(n, ctypes.c_void_p) for n in ("means", "covariances", "scales", "rotations", "harmonics", "opacities",
                                        "center", "scale")]


PLY_IMPORT_MAX_PROPERTIES, PLY_IMPORT_MAX_COEFFS = 512, 25


class PlyImportDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("sh_degree", "sh_coeffs", "n_props", "reserved")] + \
        [("n_gaussians", ctypes.c_int64), ("col_xyz", ctypes.c_int32 * 3), ("col_dc", ctypes.c_int32 * 3),
         ("col_rest", ctypes.c_int32 * 45), ("col_opacity", ctypes.c_int32), ("col_scale", ctypes.c_int32 * 3),
         ("col_rot", ctypes.c_int32 * 4), ("reserved2", ctypes.c_int32), ("frame", ctypes.c_double * 9),
         ("center", ctypes.c_double * 3), ("scale", ctypes.c_double),
         ("sh_transform", ctypes.c_float * PLY_SH_TRANSFORM_FLOATS)] + \
        [(n, ctypes.c_void_p) for n in ("records", "means", "covariances", "harmonics", "opacities")]


PLY_REFINE_MAX_PROPERTIES = 256


class PlyRefineDesc(ctypes.Structure):
    _fields_ = [("unpack", PlyImportDesc), ("step", ctypes.c_int64)] + \
        [(n, ctypes.c_double) for n in ("beta1", "beta2", "eps")] + \
        [("lr", ctypes.c_double * PLY_REFINE_MAX_PROPERTIES)] + \
        [(n, ctypes.c_void_p) for n in ("records_out", "exp_avg", "exp_avg_sq", "d_means", "d_covariances",
                                        "d_harmonics", "d_opacities", "d_records")]


class PlyDensifyDesc(ctypes.Structure):
    _fields_ = [("n_gaussians", ctypes.c_int64), ("n_props", ctypes.c_int32), ("prune_world", ctypes.c_int32),
                ("col_xyz", ctypes.c_int32 * 3), ("col_opacity", ctypes.c_int32), ("col_scale", ctypes.c_int32 * 3),
                ("col_rot", ctypes.c_int32 * 4), ("reserved", ctypes.c_int32)] + \
        [(n, ctypes.c_double) for n in ("grad_threshold", "percent_dense", "min_opacity", "extent")]


class RasterCameraGrads(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("d_viewmatrix", "d_projmatrix", "d_campos", "d_tanfov", "workspace")] + \
        [("workspace_bytes", ctypes.c_size_t)]


class RasterGrads(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in (
        "d_means", "d_cov", "d_opacities", "d_sh", "d_means2d")] + [("camera", ctypes.POINTER(RasterCameraGrads))]


EXPORTS = ("ps_version", "ps_last_error", "ps_raster_sizes_query", "ps_raster_layout_query",
           "ps_raster_forward", "ps_raster_backward", "ps_camera_setup", "ps_launch_count",
           "ps_timing_enable", "ps_timing_read", "ps_epipolar_geometry",
           "ps_epipolar_attention_forward", "ps_epipolar_attention_backward",
           "ps_self_attention_forward", "ps_gaussian_adapter_forward", "ps_gaussian_adapter_backward",
           "ps_sh_rotation_matrices", "ps_set_option", "ps_raster_forward_loss", "ps_raster_backward_loss",
           "ps_self_attention_forward_stats", "ps_self_attention_backward", "ps_get_option",
           "ps_raster_backward_depth", "ps_ssim_workspace_bytes", "ps_ssim_forward", "ps_ssim_backward",
           "ps_epipolar_attention_backward_workspace_bytes", "ps_epipolar_attention_backward_deterministic",
           "ps_raster_camera_workspace_bytes", "ps_camera_setup_backward", "ps_lpips_workspace_bytes",
           "ps_lpips_forward", "ps_lpips_backward", "ps_vit_attention_forward",
           "ps_vit_attention_backward_workspace_bytes", "ps_vit_attention_backward", "ps_image_resample",
           "ps_eval_images_workspace_bytes", "ps_eval_images", "ps_clip_adam_segment_chunks",
           "ps_clip_adam_workspace_bytes", "ps_clip_adam_step", "ps_ply_pack", "ps_ply_unpack", "ps_view_overlap",
           "ps_ply_refine_step", "ps_ply_densify_workspace_bytes", "ps_ply_densify_stats", "ps_ply_densify_count",
           "ps_ply_densify_apply", "ps_l1_dssim_workspace_bytes", "ps_l1_dssim")


class NativeLibraryMissing(ImportError):
    pass


def _load() -> ctypes.CDLL:
    if not LIB_PATH.exists():
        raise NativeLibraryMissing(
            f"{LIB_PATH} not found: the sm_90a CUDA library is not built. Run "
            f"`make -C {_PKG / 'csrc'}` (or __graft_entry__.build()). There is no CPU fallback.")
    lib = ctypes.CDLL(str(LIB_PATH))
    lib.ps_version.restype = ctypes.c_int
    lib.ps_last_error.restype = ctypes.c_char_p
    P = ctypes.POINTER
    lib.ps_raster_sizes_query.argtypes = [P(RasterDesc), P(RasterSizes)]
    lib.ps_raster_layout_query.argtypes = [P(RasterDesc), P(RasterLayout)]
    lib.ps_raster_forward.argtypes = [P(RasterDesc), P(RasterInputs), P(RasterState), ctypes.c_void_p,
                                      ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.ps_raster_backward.argtypes = [P(RasterDesc), P(RasterInputs), P(RasterState), ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_size_t, P(RasterGrads), ctypes.c_void_p]
    lib.ps_raster_forward_loss.argtypes = [P(RasterDesc), P(RasterInputs), P(RasterState), P(RasterLoss),
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.ps_raster_backward_loss.argtypes = [P(RasterDesc), P(RasterInputs), P(RasterState), ctypes.c_void_p,
                                            ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, P(RasterGrads),
                                            ctypes.c_void_p]
    lib.ps_raster_backward_depth.argtypes = [P(RasterDesc), P(RasterInputs), P(RasterState)] + [ctypes.c_void_p] * 5 + \
        [ctypes.c_size_t, P(RasterGrads), ctypes.c_void_p]
    lib.ps_raster_backward_depth.restype = ctypes.c_int
    lib.ps_raster_forward_loss.restype = ctypes.c_int
    lib.ps_raster_backward_loss.restype = ctypes.c_int
    lib.ps_camera_setup.argtypes = [ctypes.c_int32] + [ctypes.c_void_p] * 4 + [ctypes.c_int32] + \
        [ctypes.c_void_p] * 6
    lib.ps_camera_setup.restype = ctypes.c_int
    lib.ps_camera_setup_backward.argtypes = [ctypes.c_int32] + [ctypes.c_void_p] * 4 + [ctypes.c_int32] + \
        [ctypes.c_void_p] * 7
    lib.ps_camera_setup_backward.restype = ctypes.c_int
    lib.ps_raster_camera_workspace_bytes.argtypes = [P(RasterDesc), P(ctypes.c_size_t)]
    lib.ps_raster_camera_workspace_bytes.restype = ctypes.c_int
    lib.ps_launch_count.restype = ctypes.c_ulonglong
    lib.ps_timing_enable.argtypes = [ctypes.c_int]
    lib.ps_timing_enable.restype = None
    lib.ps_timing_read.argtypes = [ctypes.POINTER(ctypes.c_float)]
    lib.ps_timing_read.restype = ctypes.c_int
    lib.ps_epipolar_geometry.argtypes = [ctypes.c_int32] * 5 + [ctypes.c_void_p] * 9
    lib.ps_epipolar_geometry.restype = ctypes.c_int
    lib.ps_view_overlap.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 2 + [ctypes.c_int32] * 3 + \
        [ctypes.c_void_p] * 2
    lib.ps_view_overlap.restype = ctypes.c_int
    lib.ps_epipolar_attention_forward.argtypes = [P(EpipolarDesc), P(EpipolarInputs)] + [ctypes.c_void_p] * 5
    lib.ps_epipolar_attention_forward.restype = ctypes.c_int
    lib.ps_epipolar_attention_backward.argtypes = [P(EpipolarDesc), P(EpipolarInputs)] + [ctypes.c_void_p] * 10
    lib.ps_epipolar_attention_backward.restype = ctypes.c_int
    lib.ps_epipolar_attention_backward_workspace_bytes.argtypes = [P(EpipolarDesc), P(ctypes.c_size_t)]
    lib.ps_epipolar_attention_backward_workspace_bytes.restype = ctypes.c_int
    lib.ps_epipolar_attention_backward_deterministic.argtypes = [P(EpipolarDesc), P(EpipolarInputs)] + \
        [ctypes.c_void_p] * 10 + [ctypes.c_size_t, ctypes.c_void_p]
    lib.ps_epipolar_attention_backward_deterministic.restype = ctypes.c_int
    lib.ps_self_attention_forward.argtypes = [ctypes.c_int32] * 4 + [ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p,
                                                                      ctypes.c_int32, ctypes.c_void_p]
    lib.ps_self_attention_forward.restype = ctypes.c_int
    lib.ps_self_attention_forward_stats.argtypes = [ctypes.c_int32] * 4 + [ctypes.c_void_p, ctypes.c_float,
                                                                            ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.ps_self_attention_forward_stats.restype = ctypes.c_int
    lib.ps_self_attention_backward.argtypes = [ctypes.c_int32] * 4 + [ctypes.c_void_p] * 4 + [ctypes.c_float,
                                                                                             ctypes.c_void_p, ctypes.c_void_p]
    lib.ps_self_attention_backward.restype = ctypes.c_int
    lib.ps_gaussian_adapter_forward.argtypes = [P(AdapterDesc), P(AdapterInputs)] + [ctypes.c_void_p] * 6
    lib.ps_gaussian_adapter_forward.restype = ctypes.c_int
    lib.ps_gaussian_adapter_backward.argtypes = [P(AdapterDesc), P(AdapterInputs)] + [ctypes.c_void_p] * 9
    lib.ps_gaussian_adapter_backward.restype = ctypes.c_int
    lib.ps_sh_rotation_matrices.argtypes = [ctypes.c_int32] * 4 + [ctypes.c_void_p] * 5
    lib.ps_sh_rotation_matrices.restype = ctypes.c_int
    lib.ps_set_option.argtypes = [ctypes.c_char_p, ctypes.c_int]
    lib.ps_set_option.restype = ctypes.c_int
    lib.ps_get_option.argtypes = [ctypes.c_char_p, ctypes.POINTER(ctypes.c_int)]
    lib.ps_get_option.restype = ctypes.c_int
    lib.ps_ssim_workspace_bytes.argtypes = [ctypes.c_int32] * 3 + [P(ctypes.c_size_t)]
    lib.ps_ssim_workspace_bytes.restype = ctypes.c_int
    lib.ps_ssim_forward.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 4 + [ctypes.c_size_t, ctypes.c_void_p]
    lib.ps_ssim_forward.restype = ctypes.c_int
    lib.ps_ssim_backward.argtypes = [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 6 + [ctypes.c_size_t, ctypes.c_void_p]
    lib.ps_ssim_backward.restype = ctypes.c_int
    lib.ps_l1_dssim_workspace_bytes.argtypes = [ctypes.c_int32] * 4 + [P(ctypes.c_size_t)]
    lib.ps_l1_dssim_workspace_bytes.restype = ctypes.c_int
    lib.ps_l1_dssim.argtypes = [ctypes.c_int32] * 4 + [ctypes.c_void_p] * 2 + [ctypes.c_float] + \
        [ctypes.c_void_p] * 5 + [ctypes.c_size_t, ctypes.c_void_p]
    lib.ps_l1_dssim.restype = ctypes.c_int
    lib.ps_lpips_workspace_bytes.argtypes = [P(LpipsDesc), P(ctypes.c_size_t)]
    lib.ps_lpips_workspace_bytes.restype = ctypes.c_int
    lib.ps_lpips_forward.argtypes = [P(LpipsDesc), ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.ps_lpips_forward.restype = ctypes.c_int
    lib.ps_lpips_backward.argtypes = [P(LpipsDesc), ctypes.c_void_p, P(LpipsGrads), ctypes.c_void_p]
    lib.ps_lpips_backward.restype = ctypes.c_int
    lib.ps_vit_attention_forward.argtypes = [ctypes.c_int32] * 4 + [ctypes.c_void_p, ctypes.c_float] + \
        [ctypes.c_void_p] * 3
    lib.ps_vit_attention_forward.restype = ctypes.c_int
    lib.ps_vit_attention_backward_workspace_bytes.argtypes = [ctypes.c_int32] * 4 + [P(ctypes.c_size_t)]
    lib.ps_vit_attention_backward_workspace_bytes.restype = ctypes.c_int
    lib.ps_vit_attention_backward.argtypes = [ctypes.c_int32] * 4 + [ctypes.c_void_p] * 4 + \
        [ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.ps_vit_attention_backward.restype = ctypes.c_int
    lib.ps_image_resample.argtypes = [P(ResampleDesc), ctypes.c_void_p, ctypes.c_void_p]
    lib.ps_image_resample.restype = ctypes.c_int
    lib.ps_eval_images_workspace_bytes.argtypes = [ctypes.c_int32] * 3 + [P(ctypes.c_size_t)]
    lib.ps_eval_images_workspace_bytes.restype = ctypes.c_int
    lib.ps_eval_images.argtypes = [P(EvalDesc), ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.ps_eval_images.restype = ctypes.c_int
    lib.ps_clip_adam_segment_chunks.argtypes = [ctypes.c_void_p, ctypes.c_int64]
    lib.ps_clip_adam_segment_chunks.restype = ctypes.c_int64
    lib.ps_clip_adam_workspace_bytes.argtypes = [P(ClipAdamDesc), P(ctypes.c_size_t)]
    lib.ps_clip_adam_workspace_bytes.restype = ctypes.c_int
    lib.ps_clip_adam_step.argtypes = [P(ClipAdamDesc), ctypes.c_void_p, P(ClipAdamState), ctypes.c_void_p,
                                      ctypes.c_size_t, ctypes.c_void_p]
    lib.ps_clip_adam_step.restype = ctypes.c_int
    lib.ps_ply_pack.argtypes = [P(PlyDesc), ctypes.c_void_p, ctypes.c_void_p]
    lib.ps_ply_pack.restype = ctypes.c_int
    lib.ps_ply_unpack.argtypes = [P(PlyImportDesc), ctypes.c_void_p]
    lib.ps_ply_unpack.restype = ctypes.c_int
    lib.ps_ply_refine_step.argtypes = [P(PlyRefineDesc), ctypes.c_void_p]
    lib.ps_ply_refine_step.restype = ctypes.c_int
    lib.ps_ply_densify_workspace_bytes.argtypes = [ctypes.c_int64, P(ctypes.c_size_t)]
    lib.ps_ply_densify_workspace_bytes.restype = ctypes.c_int
    lib.ps_ply_densify_stats.argtypes = [ctypes.c_int64, ctypes.c_int32] + [ctypes.c_void_p] * 5
    lib.ps_ply_densify_stats.restype = ctypes.c_int
    lib.ps_ply_densify_count.argtypes = [P(PlyDensifyDesc)] + [ctypes.c_void_p] * 4 + [ctypes.c_size_t] + \
        [ctypes.c_void_p] * 2
    lib.ps_ply_densify_count.restype = ctypes.c_int
    lib.ps_ply_densify_apply.argtypes = [P(PlyDensifyDesc)] + [ctypes.c_void_p] * 5 + [ctypes.c_size_t] + \
        [ctypes.c_void_p] * 5
    lib.ps_ply_densify_apply.restype = ctypes.c_int
    for f in ("ps_raster_sizes_query", "ps_raster_layout_query", "ps_raster_forward", "ps_raster_backward"):
        getattr(lib, f).restype = ctypes.c_int
    return lib


lib = _load()


class NativeError(RuntimeError):
    pass


def check(rc: int, what: str) -> None:
    if rc != PS_OK:
        msg = lib.ps_last_error().decode("utf-8", "replace")
        exc = ValueError if rc == 1 else NativeError
        raise exc(f"{what}: {_ERR_NAMES.get(rc, rc)}: {msg}")


def on_device(device, fn, *args) -> int:
    """Calls a library entry point with `device` as the CURRENT CUDA device: the library creates its side
    stream / events and sets kernel attributes on the current device, so a tensor living on another GPU than
    the caller's current one must switch first (torch.cuda.device is a no-op when it already is current)."""
    import torch
    with torch.cuda.device(device):
        return fn(*args)


def set_option(name: str, value: int) -> None:
    check(lib.ps_set_option(name.encode(), int(value)), "ps_set_option")


def get_option(name: str) -> int:
    """The value of a compositor option in force (set through set_option or the environment)."""
    v = ctypes.c_int()
    check(lib.ps_get_option(name.encode(), ctypes.byref(v)), "ps_get_option")
    return v.value


def epipolar_backward_workspace_bytes(desc: EpipolarDesc) -> int:
    """Workspace of ps_epipolar_attention_backward_deterministic for `desc` (no device needed)."""
    out = ctypes.c_size_t()
    check(lib.ps_epipolar_attention_backward_workspace_bytes(ctypes.byref(desc), ctypes.byref(out)),
          "ps_epipolar_attention_backward_workspace_bytes")
    return out.value


def sizes(desc: RasterDesc) -> RasterSizes:
    out = RasterSizes()
    check(lib.ps_raster_sizes_query(ctypes.byref(desc), ctypes.byref(out)), "ps_raster_sizes_query")
    return out


def camera_workspace_bytes(desc: RasterDesc) -> int:
    out = ctypes.c_size_t()
    check(lib.ps_raster_camera_workspace_bytes(ctypes.byref(desc), ctypes.byref(out)),
          "ps_raster_camera_workspace_bytes")
    return out.value


def layout(desc: RasterDesc) -> RasterLayout:
    out = RasterLayout()
    check(lib.ps_raster_layout_query(ctypes.byref(desc), ctypes.byref(out)), "ps_raster_layout_query")
    return out
