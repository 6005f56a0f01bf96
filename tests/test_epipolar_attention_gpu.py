"""The fused epipolar attention kernels (csrc/epipolar_attention.cu: k_epi_attn_fwd, k_epi_attn_bwd and the
fixed-order d(feature map) of ps_epipolar_attention_backward_deterministic) against the float64 restatement
tests/epipolar_attention_f64.py, across the descriptor space the C ABI accepts.  `_EpipolarAttentionFn` is called
directly and all eight tensors are compared: z, e, mass, lse, dqt, dpq, dbias, dfeat.

  1. A pairwise sweep: heads 1-4; S in {1, 3, 4, 5, 8, 9, 17, 31, 32} (the forward's sub-chunks of 8 and the
     backward's of 4, full and with a partial tail); pe_dim 0 / 2 / 20, 24 at heads 4 and 32 at heads 3 (all 96 e /
     dpq lanes); v in {2, 3, 5, 9, 33}; b in {1, 2}; grids 1x1, 1x7, 2x3, 6x10, 8x8; bias and a mass cotangent in
     all four combinations.  Geometry from real rigs (epipolar_geometry on the generic / parallel / diverging rigs of
     golden_util.camera_rig) and hand-built segments: ends on texel centres and on the map edges 0 and 1, samples
     one texel apart on texel centres, partly and wholly off the map, one tap inside, zero length (every sample in
     one cell: the backward's register merge), +-1e4 long (the tap clamp); valid and invalid rays mixed, one query
     with every ray invalid, rel_disparity with exact 0 and 1.  One case takes non-contiguous inputs and cotangents.
     Every case runs with torch.use_deterministic_algorithms off (float-atomic d(feature map)) and on (fixed order);
     both meet the same bars.
  2. A structured case: texel values encode (b, view, y, x, channel) and a sharp qt selects one known texel per
     (query, head), so z must equal that texel: catches head, view (v >= 4) and batch mix-ups a norm-wise bar hides.
  3. The SUB = 4 forward (PIXELSPLAT_B200_EPI_SUB_FWD=4, read once per process) on a subset of the sweep, in a
     subprocess.
  4. The mass cotangent reaches dqt, dpq and d(feature map) without a bias, at one library launch per backward.

Bars, each against the float64 restatement, over the whole tensor and per slice (z / e per head, mass per (head,
other view)):
  z, e, mass  max |got - ref| / max |ref|                     <= FWD_BAR
  lse         max |got - ref| / (1 + |ref|)                   <= LSE_BAR
  dqt, dpq, dbias  ||got - ref||_2 / ||ref||_2 <= GRAD_L2_BAR and max-norm as above <= GRAD_MAX_BAR
  dfeat       ||got - ref||_2 / ||ref||_2                      <= DFEAT_L2_BAR
dbias with one other view, and dqt / dpq where every sample of a row is alike, vanish by construction (the score
gradient a (da - D) sums to zero); such a tensor is held to ||got||_2 <= ZERO_BAR times the norm of the same sum taken
over a (|da| + |D|), the size of the terms float32 rounds (epipolar_attention_f64.forward_backward).

Measured on an NVIDIA H100 80GB HBM3 at a 400 W power limit, worst over the 22 cases and both modes (the two modes
differ in dfeat only): z 4.2e-6, e 3.5e-6, mass 1.9e-6, lse 1.8e-6; dqt 2.6e-6 / 3.1e-6 (norm-wise / max-norm),
dpq 3.3e-6 / 2.4e-6, dbias 2.4e-6 / 3.5e-6; dfeat 2.1e-6; vanishing tensors 7.6e-8.  The SUB = 4 forward: z 2.9e-6,
e 3.3e-6, mass 1.9e-6, lse 1.8e-6.  The bars are these with a margin of 3.4x-4x.  The whole file takes about 25 s.
"""
import json
import os
import subprocess
import sys
from functools import lru_cache
from pathlib import Path

import pytest
import torch

from tests import epipolar_attention_f64 as ref
from tests import golden_util as gu

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = Path(__file__).resolve().parents[1]
C = 128

FWD_BAR, LSE_BAR = 1.5e-5, 6e-6
GRAD_L2_BAR, GRAD_MAX_BAR, DFEAT_L2_BAR = 1.2e-5, 1.2e-5, 8e-6
ZERO_BAR = 3e-7


@pytest.fixture(params=[False, True], ids=["atomic", "deterministic"])
def det_mode(request):
    """torch's deterministic flag off or on for the test; the flag and the cuBLAS workspace setting torch asks for
    under the flag are restored afterwards, also when the test fails."""
    flag, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    cublas = os.environ.get("CUBLAS_WORKSPACE_CONFIG")
    os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
    torch.use_deterministic_algorithms(request.param)
    try:
        yield request.param
    finally:
        torch.use_deterministic_algorithms(flag, warn_only=warn_only)
        if cublas is None:
            os.environ.pop("CUBLAS_WORKSPACE_CONFIG", None)
        else:
            os.environ["CUBLAS_WORKSPACE_CONFIG"] = cublas


# (b, v, (h, w), S, heads, pe_dim, geometry, bias, mass cotangent)
CASES = {
    "h1-s1-pe0-v2-1x1-hand": (1, 2, (1, 1), 1, 1, 0, "hand", False, False),
    "h1-s3-pe2-v3-1x7-generic": (2, 3, (1, 7), 3, 1, 2, "generic", True, True),
    "h1-s9-pe20-v5-6x10-hand": (1, 5, (6, 10), 9, 1, 20, "hand", False, True),
    "h1-s31-pe20-v9-8x8-parallel": (2, 9, (8, 8), 31, 1, 20, "parallel", True, False),
    "h1-s32-pe0-v2-8x8-hand": (2, 2, (8, 8), 32, 1, 0, "hand", False, True),
    "h2-s4-pe0-v9-1x7-hand": (1, 9, (1, 7), 4, 2, 0, "hand", True, True),
    "h2-s5-pe20-v2-8x8-generic": (2, 2, (8, 8), 5, 2, 20, "generic", False, False),
    "h2-s17-pe2-v3-6x10-diverging": (2, 3, (6, 10), 17, 2, 2, "diverging", True, False),
    "h2-s32-pe20-v5-1x1-hand": (2, 5, (1, 1), 32, 2, 20, "hand", False, True),
    "h2-s8-pe2-v2-6x10-hand": (2, 2, (6, 10), 8, 2, 2, "hand", True, False),
    "h3-s8-pe32-v3-8x8-generic": (2, 3, (8, 8), 8, 3, 32, "generic", False, True),
    "h3-s31-pe32-v5-6x10-hand": (1, 5, (6, 10), 31, 3, 32, "hand", True, True),
    "h3-s1-pe2-v9-1x1-hand": (2, 9, (1, 1), 1, 3, 2, "hand", False, False),
    "h3-s17-pe0-v2-1x7-parallel": (1, 2, (1, 7), 17, 3, 0, "parallel", True, True),
    "h3-s4-pe20-v2-8x8-hand": (1, 2, (8, 8), 4, 3, 20, "hand", True, False),
    "h4-s9-pe24-v2-6x10-generic": (2, 2, (6, 10), 9, 4, 24, "generic", True, True),
    "h4-s3-pe24-v5-8x8-hand": (2, 5, (8, 8), 3, 4, 24, "hand", False, True),
    "h4-s4-pe20-v3-8x8-diverging": (1, 3, (8, 8), 4, 4, 20, "diverging", False, False),
    "h4-s32-pe24-v9-6x10-generic": (1, 9, (6, 10), 32, 4, 24, "generic", True, False),
    "h4-s5-pe2-v33-2x3-hand": (1, 33, (2, 3), 5, 4, 2, "hand", True, True),
    "h4-s17-pe20-v9-1x7-hand": (2, 9, (1, 7), 17, 4, 20, "hand", False, False),
    "h4-s31-pe0-v3-8x8-hand-noncontig": (2, 3, (8, 8), 31, 4, 0, "hand", True, True),
}
# the SUB = 4 forward's subset: every head count, partial and full chunks of 4 and 8, the widest e
SUB4_CASES = ["h1-s9-pe20-v5-6x10-hand", "h2-s17-pe2-v3-6x10-diverging", "h3-s31-pe32-v5-6x10-hand",
              "h4-s9-pe24-v2-6x10-generic", "h4-s5-pe2-v33-2x3-hand", "h2-s32-pe20-v5-1x1-hand"]


def _hand_geometry(b, v, grid, S, seed):
    """Segments built by hand, one kind per ray (seeded), valid with ~15 % invalid rays and every ray of the first
    query invalid, rel_disparity in [0, 1] with exact 0 and 1."""
    from pixelsplat_b200.encoder.attention_fused import EpipolarGeometry
    h, w = grid
    shape = (b, v, v - 1, h * w)
    g = torch.Generator().manual_seed(seed)
    U = lambda lo=0.0, hi=1.0: lo + (hi - lo) * torch.rand(shape, generator=g, dtype=torch.float64)
    cx = lambda: (torch.randint(0, w, shape, generator=g).double() + 0.5) / w           # texel centres
    cy = lambda: (torch.randint(0, h, shape, generator=g).double() + 0.5) / h
    edge = lambda: torch.randint(0, 2, shape, generator=g).double()             # the map edges 0 and 1
    sign = lambda: torch.randint(0, 2, shape, generator=g).double() * 2 - 1
    out_x = lambda: torch.where(sign() > 0, 1 + 0.25 / w, -0.25 / w).double()   # one tap column inside
    out_y = lambda: torch.where(sign() > 0, 1 + 0.25 / h, -0.25 / h).double()
    x0c, y0c = cx(), cy()
    p, q = cx(), cy()
    ox, oy, oy2 = out_x(), out_y(), out_y()
    kinds = [
        (U(-0.3, 1.3), U(-0.3, 1.3), U(-0.3, 1.3), U(-0.3, 1.3)),              # random, partly off the map
        (x0c, y0c, p, q),                                                       # ends on texel centres
        (edge(), U(), U(), edge()),                                             # ends on the map edges
        (x0c - 0.5 / w, y0c, x0c - 0.5 / w + S / w, y0c),                       # samples on texel centres
        (x0c, y0c, x0c, y0c),                                                   # zero length on a texel centre
        (p + U(-0.4, 0.4) / w, q, p + U(-0.4, 0.4) / w, q),                     # short: a few cells at most
        (ox, oy, ox, oy),                                                       # one tap inside, zero length
        (U(), oy2, U(), oy2),                                                   # along an edge, one tap row in
        (U(1.2, 3.0), U(), U(1.2, 3.0), U(-2.0, -0.2)),                         # wholly off the map
        (-1e4 * sign(), -1e4 * sign(), U(), U()),                               # long: the tap clamp
        (torch.full(shape, -1e4, dtype=torch.float64), U(), torch.full(shape, 1e4, dtype=torch.float64), U()),
    ]
    kind = torch.randint(0, len(kinds), shape, generator=g)
    seg = torch.zeros((*shape, 4), dtype=torch.float64)
    for k, ends in enumerate(kinds):
        m = kind == k
        for i, t in enumerate(ends):
            seg[..., i][m] = t.expand(shape)[m]
    valid = torch.rand(shape, generator=g) > 0.15
    valid[0, 0, :, 0] = False
    rd = torch.rand((*shape, S), generator=g, dtype=torch.float64)
    rd[torch.rand(rd.shape, generator=g) < 0.1] = 0.0
    rd[torch.rand(rd.shape, generator=g) < 0.1] = 1.0
    return EpipolarGeometry(seg.float().to(DEV), valid.to(torch.uint8).to(DEV), rd.float().to(DEV),
                            torch.zeros((*shape, 2), device=DEV), grid, S)


def _geometry(b, v, grid, S, kind, seed):
    if kind == "hand":
        return _hand_geometry(b, v, grid, S, seed)
    from pixelsplat_b200.encoder.attention_fused import epipolar_geometry
    ext, K, near, far = [t.to(DEV, torch.float32) for t in gu.camera_rig(b, v, kind)]
    return epipolar_geometry(ext, K, near, far, grid, S)


@lru_cache(maxsize=None)
def _prepared(name):
    """(geometry, heads, inputs and cotangents, float64 results) of a sweep case; the same for both modes."""
    b, v, grid, S, heads, npe, kind, bias, dmass = CASES[name]
    seed = sorted(CASES).index(name)
    geom = _geometry(b, v, grid, S, kind, 100 + seed)
    h, w = grid
    n, ov = b * v * h * w, v - 1
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(s, generator=g) * scale).to(DEV)
    x = dict(qt=r(n, heads, C, scale=0.3), pq=r(n, heads, npe, scale=0.3), bias=r(n, heads, ov) if bias else None,
             feat=r(b, v, h, w, C), dz=r(n, heads, C), de=r(n, heads, npe), dmass=r(n, heads, ov) if dmass else None)
    if name.endswith("noncontig"):
        # cotangents as autograd may deliver them: broadcast over the heads (stride 0) and a strided view
        x["dz"] = x["dz"][:, :1].expand_as(x["dz"])
        x["de"] = torch.stack([x["de"], torch.randn_like(x["de"])], -1).flatten(-2)[..., 0::2]
    want = ref.forward_backward(x["feat"], geom.segments, geom.valid.bool(), geom.rel_disparity, x["qt"], x["pq"],
                                x["bias"], heads, x["dz"], x["de"], x["dmass"])
    return geom, heads, x, want


def _run(geom, heads, x, noncontig=False):
    """One _EpipolarAttentionFn forward and backward in the flag's current mode: the eight tensors.  noncontig: qt
    is a strided view of a wider leaf (and the case's cotangents are non-contiguous, see _prepared)."""
    from pixelsplat_b200.encoder.attention_fused import _EpipolarAttentionFn
    leaves = {k: x[k].clone().requires_grad_(True) for k in ("pq", "bias", "feat") if x[k] is not None}
    if noncontig:
        wide = torch.stack([x["qt"], torch.randn_like(x["qt"])], -1).flatten(-2).requires_grad_(True)
        qt = wide[..., 0::2]
        assert not (qt.is_contiguous() or x["dz"].is_contiguous() or (x["de"].numel() and x["de"].is_contiguous()))
        leaves = {"qt": wide, **leaves}
    else:
        qt = leaves["qt"] = x["qt"].clone().requires_grad_(True)
    z, e, mass = _EpipolarAttentionFn.apply(qt, leaves["pq"], leaves.get("bias"), leaves["feat"], geom, heads)
    lse = z.grad_fn.saved_tensors[-1]      # not an output of the Function: the forward saves it for the backward
    outs, cots = [z, e], [x["dz"], x["de"]]
    if x["dmass"] is not None:
        outs.append(mass)
        cots.append(x["dmass"])
    grads = dict(zip(leaves, torch.autograd.grad(outs, list(leaves.values()), cots)))
    if noncontig:
        assert not grads["qt"][..., 1::2].any()
        grads["qt"] = grads["qt"][..., 0::2]
    return dict(z=z.detach(), e=e.detach(), mass=mass.detach(), lse=lse, dqt=grads["qt"], dpq=grads["pq"],
                dbias=grads.get("bias"), dfeat=grads["feat"])


def _max_rel(got, want):
    got, want = got.double(), want.double()
    if want.numel() == 0:
        return 0.0
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-30))


def _l2_rel(got, want):
    got, want = got.double(), want.double()
    if want.numel() == 0:
        return 0.0
    return float((got - want).norm() / want.norm().clamp_min(1e-30))


def _forward_errors(got, want):
    """Worst error of z / e / mass over the whole tensor and every (head) or (head, other view) slice; lse's."""
    err = {}
    for k in ("z", "e"):
        err[k] = max([_max_rel(got[k], want[k])] + [_max_rel(got[k][:, hd], want[k][:, hd])
                                                   for hd in range(got[k].shape[1])])
    err["mass"] = max([_max_rel(got["mass"], want["mass"])] +
                      [_max_rel(got["mass"][:, hd, o], want["mass"][:, hd, o])
                       for hd in range(got["mass"].shape[1]) for o in range(got["mass"].shape[2])])
    err["lse"] = float(((got["lse"].double() - want["lse"]).abs() / (1 + want["lse"].abs())).max())
    return err


def _check_forward(got, want, name):
    err = _forward_errors(got, want)
    assert err["z"] <= FWD_BAR and err["e"] <= FWD_BAR and err["mass"] <= FWD_BAR, (name, err)
    assert err["lse"] <= LSE_BAR, (name, err)
    return err


@pytest.mark.parametrize("name", list(CASES))
def test_kernels_match_float64(det_mode, name):
    geom, heads, x, want = _prepared(name)
    got = _run(geom, heads, x, noncontig=name.endswith("noncontig"))
    for k in ("z", "e", "mass", "lse", "dqt", "dpq", "dfeat"):
        assert got[k].shape == want[k].shape and bool(torch.isfinite(got[k]).all()), k
    assert (got["dbias"] is None) == (x["bias"] is None)
    err = _forward_errors(got, want)
    for k in ("dqt", "dpq", "dbias"):
        if got[k] is None or got[k].numel() == 0:
            continue
        scale = want[k + "_scale"].norm()
        if want[k].norm() > 1e-9 * scale:
            err[k + "_l2"], err[k + "_max"] = _l2_rel(got[k], want[k]), _max_rel(got[k], want[k])
        else:                  # zero by construction up to float64 round-off: bounded by the terms' size instead
            err[k + "_zero"] = float(got[k].double().norm() / scale.clamp_min(1e-30))
    err["dfeat_l2"] = _l2_rel(got["dfeat"], want["dfeat"])
    print("errors", name, "deterministic" if det_mode else "atomic", json.dumps({k: f"{e:.2e}" for k, e in err.items()}))
    assert err["z"] <= FWD_BAR and err["e"] <= FWD_BAR and err["mass"] <= FWD_BAR, err
    assert err["lse"] <= LSE_BAR, err
    for k in ("dqt", "dpq", "dbias"):
        if k + "_l2" in err:
            assert err[k + "_l2"] <= GRAD_L2_BAR and err[k + "_max"] <= GRAD_MAX_BAR, (k, err)
        if k + "_zero" in err:
            assert err[k + "_zero"] <= ZERO_BAR, (k, err)
    assert err["dfeat_l2"] <= DFEAT_L2_BAR, err
    if CASES[name][6] == "hand":
        # the first query has no valid ray: z is exactly 0; the PE and the bias still spread mass (and e)
        assert not got["z"][0].any() and bool((got["mass"][0] > 0).all())
        if x["pq"].shape[-1] > 0:
            assert bool((got["e"][0].abs() > 0).any())


STRUCTURED = {"b2-v5-4x4-h4-s5": (2, 5, (4, 4), 5, 4), "b1-v33-2x3-h3-s3": (1, 33, (2, 3), 3, 3),
              "b2-v9-1x7-h2-s9": (2, 9, (1, 7), 9, 2)}


@pytest.mark.parametrize("name", list(STRUCTURED))
def test_sharp_query_selects_the_known_texel(name):
    """Texel (b, view, y, x) holds (((b V + view) h + y) w + x) 128 + c over the texel count in channel c < 124 and a
    per-head key (a permutation of the texels) in channel 124 + head.  Every ray of every query is a zero-length
    segment on one texel centre of its other view, and qt_h = beta e_{124+h}: head h's soft-max picks, of the query's
    v - 1 texels, the one with the largest key by a score gap of >= 60.  z_h must equal that texel to 1e-5 and the
    mass sit on its other view."""
    from pixelsplat_b200.encoder.attention_fused import EpipolarGeometry, _EpipolarAttentionFn
    b, v, (h, w), S, heads = STRUCTURED[name]
    ov, R = v - 1, h * w
    n, T = b * v * R, b * v * R
    g = torch.Generator().manual_seed(7)
    feat = (torch.arange(T * C, dtype=torch.float64) / (T * C)).reshape(b, v, h, w, C)
    keys = torch.stack([torch.randperm(T, generator=g).double() / T for _ in range(heads)], -1).reshape(b, v, h, w,
                                                                                                       heads)
    feat[..., 124:124 + heads] = keys
    ty = torch.randint(0, h, (b, v, ov, R), generator=g)
    tx = torch.randint(0, w, (b, v, ov, R), generator=g)
    cx, cy = (tx + 0.5) / w, (ty + 0.5) / h
    seg = torch.stack([cx, cy, cx, cy], -1)
    geom = EpipolarGeometry(seg.float().to(DEV), torch.ones((b, v, ov, R), dtype=torch.uint8, device=DEV),
                            torch.rand((b, v, ov, R, S), generator=g).to(DEV), torch.zeros((b, v, ov, R, 2), device=DEV),
                            (h, w), S)
    beta = 60.0 * T
    qt = torch.zeros(n, heads, C)
    for hd in range(heads):
        qt[:, hd, 124 + hd] = beta
    pq = 0.01 * torch.randn(n, heads, 4, generator=g)
    z, e, mass = _EpipolarAttentionFn.apply(qt.to(DEV), pq.to(DEV), None, feat.float().to(DEV), geom, heads)
    # the expected winner per (query, head), restated on the host
    other = torch.tensor(ref.other_views(v))                                        # [v, ov]
    bi = torch.arange(b)[:, None, None, None].expand(b, v, ov, R)
    src = other[None, :, :, None].expand(b, v, ov, R)
    cand = keys[bi, src, ty, tx]                                                    # [b, v, ov, R, heads]
    win = cand.argmax(2)                                                            # [b, v, R, heads]
    win_q = win.reshape(n, heads)                                                   # queries in (b, v, r) order
    texel = feat[bi, src, ty, tx].permute(0, 1, 3, 2, 4).reshape(n, ov, C)         # [n, ov, C]
    want = torch.stack([texel[torch.arange(n), win_q[:, hd]] for hd in range(heads)], 1)   # [n, heads, C]
    d = float((z.double().cpu() - want).abs().max())
    assert d < 1e-5, (name, d)
    onehot = torch.nn.functional.one_hot(win_q, ov).double()
    assert float((mass.double().cpu() - onehot).abs().max()) < 1e-5


def test_sub4_forward_matches_float64(tmp_path):
    """PIXELSPLAT_B200_EPI_SUB_FWD=4 is read once per process: a subprocess runs the forward of a subset of the
    sweep with it set.  It meets the same bars, and its z differs from the default forward's in the last bits (so
    the SUB = 4 kernel really ran)."""
    code = ("import sys, json, torch; sys.path.insert(0, sys.argv[1]);"
            "from tests import test_epipolar_attention_gpu as t;"
            "out = {}\n"
            "for name in t.SUB4_CASES:\n"
            "    geom, heads, x, want = t._prepared(name)\n"
            "    got = t._run(geom, heads, x)\n"
            "    out[name] = t._check_forward(got, want, name)\n"
            "    torch.save(got['z'].cpu(), sys.argv[2] + '/' + name + '.pt')\n"
            "print(json.dumps(out))\n")
    env = {**os.environ, "PIXELSPLAT_B200_EPI_SUB_FWD": "4"}
    res = subprocess.run([sys.executable, "-c", code, str(ROOT), str(tmp_path)], env=env, cwd=ROOT,
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    print("SUB=4 errors", res.stdout.strip().splitlines()[-1])
    differs = 0
    for name in SUB4_CASES:
        geom, heads, x, want = _prepared(name)
        got = _run(geom, heads, x)
        z4 = torch.load(tmp_path / f"{name}.pt")
        differs += not torch.equal(z4, got["z"].cpu())
    assert differs >= 3, differs


@pytest.mark.parametrize("dmass", [False, True])
def test_mass_gradient_without_bias(dmass):
    """Without a bias the mass output still depends on qt, pq and the features: its cotangent must reach their
    gradients (it once was dropped), and the backward stays one library launch either way."""
    from pixelsplat_b200 import _lib
    geom, heads, x, _ = _prepared("h1-s9-pe20-v5-6x10-hand")
    x = {**x, "dmass": x["dmass"] if dmass else None}
    flag = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(False)
        _run(geom, heads, x)                                       # warm-up
        torch.cuda.synchronize()
        l0 = _lib.lib.ps_launch_count()
        got = _run(geom, heads, x)
        torch.cuda.synchronize()
        launches = _lib.lib.ps_launch_count() - l0
    finally:
        torch.use_deterministic_algorithms(flag)
    assert launches == 2, launches                                  # k_epi_attn_fwd + k_epi_attn_bwd
    want = ref.forward_backward(x["feat"], geom.segments, geom.valid.bool(), geom.rel_disparity, x["qt"], x["pq"],
                                None, heads, x["dz"], x["de"], x["dmass"])
    for k in ("dqt", "dpq", "dfeat"):
        assert _l2_rel(got[k], want[k]) <= GRAD_L2_BAR, (k, _l2_rel(got[k], want[k]))
