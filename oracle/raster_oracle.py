"""ctypes front-end of oracle/raster_oracle.c (CPU restatement of the tile rasterizer).

TEST INFRASTRUCTURE ONLY -- see the header of raster_oracle.c.  PARITY UNPINNED: the
reference's rasterizer (diff-gaussian-rasterization-modified, requirements.txt:17) is an
un-vendored, un-pinned dependency with no golden vectors; this oracle restates the published
algorithm (SURVEY.md Appendix A) and follows the reference call site
src/model/decoder/cuda_splatting.py:99-124 for every argument convention.

Nothing under pixelsplat_b200/ imports this module.
"""
from __future__ import annotations

import ctypes
import subprocess
from dataclasses import dataclass
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIBS: dict[str, ctypes.CDLL] = {}
TILE = 16


def build(force: bool = False) -> None:
    """Compile the two oracle libraries with gcc (seconds)."""
    targets = [_HERE / "_build" / "liboracle_f32.so", _HERE / "_build" / "liboracle_f64.so"]
    src = _HERE / "raster_oracle.c"
    if not force and all(t.exists() and t.stat().st_mtime >= src.stat().st_mtime for t in targets):
        return
    subprocess.run(["make", "-C", str(_HERE), "-s"] + (["-B"] if force else []), check=True)


def _lib(dtype) -> ctypes.CDLL:
    name = "f64" if np.dtype(dtype) == np.float64 else "f32"
    if name not in _LIBS:
        path = _HERE / "_build" / f"liboracle_{name}.so"
        if not path.exists():
            build()
        lib = ctypes.CDLL(str(path))
        lib.orc_bin.restype = ctypes.c_int64
        assert lib.orc_real_bytes() == (8 if name == "f64" else 4)
        _LIBS[name] = lib
    return _LIBS[name]


class sh_basis:
    """Context manager: evaluate SH in the given convention (0 = 3DGS default, 1 = e3nn) in the C oracle
    (both precisions) and in raster_torch for the duration of the block."""

    def __init__(self, convention: int):
        self.convention = int(convention)

    def _set(self, c: int) -> None:
        from . import raster_torch
        for dt in (np.float32, np.float64):
            _lib(dt).orc_set_sh_basis(ctypes.c_int(c))
        raster_torch.set_sh_basis(c)

    def __enter__(self):
        self._set(self.convention)
        return self

    def __exit__(self, *exc):
        self._set(0)
        return False


def _p(a: np.ndarray | None):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(ctypes.c_void_p)


def _real(dtype):
    return ctypes.c_double if np.dtype(dtype) == np.float64 else ctypes.c_float


@dataclass
class Preprocessed:
    depth: np.ndarray          # [P]
    radii: np.ndarray          # [P] int32
    xy: np.ndarray             # [P,2]
    conic_opacity: np.ndarray  # [P,4]
    rgb: np.ndarray            # [P,3]
    clamped: np.ndarray        # [P,3] uint8
    rect: np.ndarray           # [P,4] int32 (minx, miny, maxx, maxy) in tiles
    tiles_touched: np.ndarray  # [P] uint32


@dataclass
class Binned:
    keys: np.ndarray    # [N] uint64 = tile << 32 | float_bits(depth)
    values: np.ndarray  # [N] uint32 Gaussian index
    ranges: np.ndarray  # [tiles, 2] uint32


@dataclass
class Forward:
    pre: Preprocessed
    binned: Binned
    color: np.ndarray      # [3,H,W]
    final_T: np.ndarray    # [H,W]
    n_contrib: np.ndarray  # [H,W] uint32


@dataclass
class Backward:
    dL_dmeans: np.ndarray     # [P,3]
    dL_dcov6: np.ndarray      # [P,6]
    dL_dsh: np.ndarray | None  # [P,M,3]
    dL_dcolors: np.ndarray    # [P,3]  (gradient of the post-SH rgb, or of colors_precomp)
    dL_dopacity: np.ndarray   # [P]
    dL_dmean2D: np.ndarray    # [P,2]
    dL_dconic: np.ndarray     # [P,3]


def preprocess(means, cov6, opac, sh, colors, viewmatrix, projmatrix, campos, tanfovx, tanfovy,
               W, H, sh_degree, dtype=np.float32) -> Preprocessed:
    """viewmatrix/projmatrix: 16 floats, column-major (element [4*col+row]) -- i.e. the flattened
    row-major transpose built at cuda_splatting.py:85-87."""
    lib = _lib(dtype)
    c = lambda a: np.ascontiguousarray(a, dtype=dtype)
    means, cov6, opac = c(means), c(cov6), c(opac).reshape(-1)
    P = means.shape[0]
    if sh is not None:
        shc = c(sh)
        M = shc.shape[1]
        assert shc.shape == (P, M, 3)
    else:
        shc = c(colors)
        M = 0
        assert shc.shape == (P, 3)
    vm, pm, cp = c(viewmatrix).reshape(16), c(projmatrix).reshape(16), c(campos).reshape(3)
    out = Preprocessed(
        np.zeros(P, dtype), np.zeros(P, np.int32), np.zeros((P, 2), dtype), np.zeros((P, 4), dtype),
        np.zeros((P, 3), dtype), np.zeros((P, 3), np.uint8), np.zeros((P, 4), np.int32),
        np.zeros(P, np.uint32))
    R = _real(dtype)
    lib.orc_preprocess(P, M, int(sh_degree), _p(means), _p(cov6), _p(opac), _p(shc), _p(vm), _p(pm),
                       _p(cp), R(tanfovx), R(tanfovy), int(W), int(H), _p(out.depth), _p(out.radii),
                       _p(out.xy), _p(out.conic_opacity), _p(out.rgb), _p(out.clamped), _p(out.rect),
                       _p(out.tiles_touched))
    return out


def bin_tiles(pre: Preprocessed, W, H) -> Binned:
    dtype = pre.depth.dtype
    lib = _lib(dtype)
    P = pre.depth.shape[0]
    N = int(pre.tiles_touched.astype(np.int64).sum())
    tiles = ((W + TILE - 1) // TILE) * ((H + TILE - 1) // TILE)
    keys = np.zeros(max(N, 1), np.uint64)
    values = np.zeros(max(N, 1), np.uint32)
    ranges = np.zeros((tiles, 2), np.uint32)
    n = lib.orc_bin(P, _p(pre.depth), _p(pre.radii), _p(pre.rect), int(W), int(H), _p(keys),
                    _p(values), _p(ranges))
    assert n == N
    return Binned(keys[:N], values[:N], ranges)


def forward(means, cov6, opac, sh, colors, viewmatrix, projmatrix, campos, tanfovx, tanfovy, bg,
            W, H, sh_degree, dtype=np.float32) -> Forward:
    lib = _lib(dtype)
    pre = preprocess(means, cov6, opac, sh, colors, viewmatrix, projmatrix, campos, tanfovx,
                     tanfovy, W, H, sh_degree, dtype)
    binned = bin_tiles(pre, W, H)
    color = np.zeros((3, H, W), dtype)
    final_T = np.zeros((H, W), dtype)
    n_contrib = np.zeros((H, W), np.uint32)
    bgc = np.ascontiguousarray(bg, dtype=dtype).reshape(3)
    values = binned.values if binned.values.size else np.zeros(1, np.uint32)
    lib.orc_composite_fwd(int(W), int(H), _p(binned.ranges), _p(values), _p(pre.xy),
                          _p(pre.conic_opacity), _p(pre.rgb), _p(bgc), _p(color), _p(final_T),
                          _p(n_contrib))
    return Forward(pre, binned, color, final_T, n_contrib)


def backward(fwd: Forward, dL_dcolor_img, means, cov6, sh, viewmatrix, projmatrix, campos, tanfovx,
             tanfovy, bg, W, H, sh_degree) -> Backward:
    dtype = fwd.color.dtype
    lib = _lib(dtype)
    c = lambda a: np.ascontiguousarray(a, dtype=dtype)
    P = fwd.pre.depth.shape[0]
    dpix = c(dL_dcolor_img)
    assert dpix.shape == (3, H, W)
    bgc = c(bg).reshape(3)
    d_mean2D = np.zeros((P, 2), np.float64)
    d_conic = np.zeros((P, 3), np.float64)
    d_opac = np.zeros(P, np.float64)
    d_color = np.zeros((P, 3), np.float64)
    values = fwd.binned.values if fwd.binned.values.size else np.zeros(1, np.uint32)
    lib.orc_composite_bwd(P, int(W), int(H), _p(fwd.binned.ranges), _p(values), _p(fwd.pre.xy),
                          _p(fwd.pre.conic_opacity), _p(fwd.pre.rgb), _p(bgc), _p(fwd.final_T),
                          _p(fwd.n_contrib), _p(dpix), _p(d_mean2D), _p(d_conic), _p(d_opac),
                          _p(d_color))
    means, cov6 = c(means), c(cov6)
    M = 0
    shc = None
    if sh is not None:
        shc = c(sh)
        M = shc.shape[1]
    d_means = np.zeros((P, 3), dtype)
    d_cov6 = np.zeros((P, 6), dtype)
    d_sh = np.zeros((P, M, 3), dtype) if M else None
    vm, pm, cp = c(viewmatrix).reshape(16), c(projmatrix).reshape(16), c(campos).reshape(3)
    R = _real(dtype)
    m2, cn, cl = c(d_mean2D), c(d_conic), c(d_color)
    lib.orc_preprocess_bwd(P, M, int(sh_degree), _p(means), _p(cov6), _p(shc), _p(vm), _p(pm), _p(cp),
                           R(tanfovx), R(tanfovy), int(W), int(H), _p(fwd.pre.radii),
                           _p(fwd.pre.clamped), _p(m2), _p(cn), _p(cl), _p(d_means), _p(d_cov6),
                           _p(d_sh))
    return Backward(d_means, d_cov6, d_sh, cl, c(d_opac), m2, cn)


@dataclass
class Margins:
    """Per pixel [H, W]: the smallest distance of a decision value from its threshold over the entries the forward
    looked at (orc_composite_margins).  `alpha` and `T` are relative to the threshold (1/255, 1e-4).  `power` is
    |power| of the entries whose sign test could go either way (positive, or zero to within rounding of the products
    it is a difference of); it is absolute because its threshold is 0 and an implementation may test a fixed
    distance above 0 instead, as the warp-task compositor does.  NO_MARGIN where no entry reached the decision."""
    alpha: np.ndarray
    T: np.ndarray
    power: np.ndarray


NO_MARGIN = 1.0e30
POWER_DELTA = 1.0e-4     # absolute; covers the warp-task compositor's `log2-power > 1e-4` form of `power > 0`


def decision_margins(fwd: Forward, W, H) -> Margins:
    """The decision margins of `fwd`'s composite, in fwd's precision, from its per-Gaussian records and list."""
    dtype = fwd.color.dtype
    m = Margins(*(np.zeros((H, W), dtype) for _ in range(3)))
    values = fwd.binned.values if fwd.binned.values.size else np.zeros(1, np.uint32)
    _lib(dtype).orc_composite_margins(int(W), int(H), _p(fwd.binned.ranges), _p(values), _p(fwd.pre.xy),
                                      _p(fwd.pre.conic_opacity), _p(m.alpha), _p(m.T), _p(m.power))
    return m


def unsettled_kinds(m: Margins, delta: float, power_delta: float = POWER_DELTA) -> dict:
    """{"alpha", "T", "power"} -> bool [H, W]: the pixels with a decision of that kind within the margin."""
    return dict(alpha=m.alpha <= delta, T=m.T <= delta, power=m.power <= power_delta)


def settled_mask(m: Margins, delta: float, power_delta: float = POWER_DELTA) -> np.ndarray:
    """bool [H, W]: every decision the pixel's walk took is further than `delta` (relative; `power_delta`
    absolute for `power > 0`) from its threshold, so an implementation whose decision values agree with the
    oracle's to within that takes the same branches and must agree on n_contrib and, to rounding, on the rest."""
    k = unsettled_kinds(m, delta, power_delta)
    return ~(k["alpha"] | k["T"] | k["power"])


def composite64_on_records(fwd: Forward, bg, W, H) -> Forward:
    """The float64 composite on `fwd`'s (float32) per-Gaussian records and binned list, widened: a high-precision
    reference of the composite alone that shares every front-end decision (radii, tile rectangles, list order,
    colour clamps) with whatever produced those records."""
    w = lambda a: np.ascontiguousarray(a, np.float64)
    p = fwd.pre
    pre = Preprocessed(w(p.depth), p.radii, w(p.xy), w(p.conic_opacity), w(p.rgb), p.clamped, p.rect,
                       p.tiles_touched)
    color, final_T, n_contrib = np.zeros((3, H, W)), np.zeros((H, W)), np.zeros((H, W), np.uint32)
    values = fwd.binned.values if fwd.binned.values.size else np.zeros(1, np.uint32)
    _lib(np.float64).orc_composite_fwd(int(W), int(H), _p(fwd.binned.ranges), _p(values), _p(pre.xy),
                                       _p(pre.conic_opacity), _p(pre.rgb), _p(w(bg).reshape(3)), _p(color),
                                       _p(final_T), _p(n_contrib))
    return Forward(pre, fwd.binned, color, final_T, n_contrib)


def upstream_key_list(binned: Binned):
    """(keys, values) exactly as upstream's sorted binning buffers hold them."""
    return binned.keys, binned.values
