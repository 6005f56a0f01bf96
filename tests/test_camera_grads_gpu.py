"""Camera gradients on the GPU (ps_raster_camera_grads, ps_camera_setup_backward) against float64 autograd of the
rasterizer restatement (tests/camera_grads_f64.py), with the project's gradient bar: the norm-wise distance to
float64 is at most 1.5x the float32 restatement's own distance, or 1e-5, whichever is larger; entries the forward
never reads are exact zeros.  The floor: a camera gradient is one sum over every on-screen Gaussian of terms that
largely cancel, so where the float32 restatement lands within a few ulps of float64 (d_tanfov, two entries per view,
has been seen at 7.6e-7), a different but equally valid float32 summation order is ~2e-6 away."""
import math

import numpy as np
import pytest
import torch

from oracle import raster_torch as rt
from pixelsplat_b200 import _lib, synthetic
from pixelsplat_b200.decoder.cuda_splatting import camera_setup, render_views, render_views_mse
from pixelsplat_b200.rasterizer import _rasterize
from tests import util
from tests.camera_grads_f64 import camera_chain, render_view

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _scenes(kind):
    """-> (list of S scenes, V views per scene, image (H, W))."""
    if kind == "cfg0":
        return [synthetic.scene_random_frustum(seed=0)], 1, (64, 64)
    if kind == "re10k64":
        sc = synthetic.scene_re10k_like(seed=0, image_hw=(64, 64), target_views=1)
        return [sc], 1, (64, 64)
    if kind == "ragged":
        return [synthetic.scene_random_frustum(seed=3, image_hw=(50, 70), num_gaussians=600)], 1, (50, 70)
    if kind == "s2v2":
        out = []
        for s in range(2):
            sc = synthetic.scene_random_frustum(seed=10 + s, num_gaussians=500)   # 500: warps straddle the scenes
            ext = torch.eye(4)[None].repeat(2, 1, 1)
            ext[1, :3, 3] = torch.tensor([0.15, -0.05, 0.1])
            c, sn = math.cos(0.04), math.sin(0.04)
            ext[1, :3, :3] = torch.tensor([[c, 0, sn], [0, 1, 0], [-sn, 0, c]])
            sc.extrinsics, sc.intrinsics = ext, sc.intrinsics.repeat(2, 1, 1)
            sc.near, sc.far = sc.near.repeat(2), sc.far.repeat(2)
            out.append(sc)
        return out, 2, (64, 64)
    raise KeyError(kind)


def _stack(scenes, V, use_sh):
    f = lambda k: torch.stack([getattr(s, k) for s in scenes]).to(DEV)
    S = len(scenes)
    ext, K = f("extrinsics").reshape(S, V, 4, 4), f("intrinsics").reshape(S, V, 3, 3)
    near, far = f("near").reshape(S, V), f("far").reshape(S, V)
    sh = f("harmonics")
    return ext, K, near, far, f("means"), f("covariances"), sh if use_sh else sh[..., :1], f("opacities")


def _errors(got, ref64, ref32):
    e = lambda a: float(np.linalg.norm(np.asarray(a, np.float64) - ref64) / max(np.linalg.norm(ref64), 1e-30))
    return e(got), e(ref32)


def _oracle(scenes, V, hw, use_sh, scale_invariant, cams, dtype, dC, dD, depth_mode, loss_scale=None, target=None,
            through_setup=False):
    """float64 / float32 autograd of the restatement, per view.  `cams`: the four arrays [S*V, .] (float32 values,
    widened) or, with through_setup, (extrinsics, intrinsics) -> their gradients."""
    H, W = hw
    out = []
    for s, sc in enumerate(scenes):
        row, col = torch.triu_indices(3, 3)
        means, cov6 = sc.means.to(dtype), sc.covariances.to(dtype)[:, row, col]
        opac = sc.opacities.to(dtype)
        shs = sc.harmonics.to(dtype).permute(0, 2, 1).contiguous()
        deg = math.isqrt(shs.shape[1]) - 1
        for v in range(V):
            vid = s * V + v
            nr, fr = float(sc.near[v]), float(sc.far[v])
            if through_setup:
                e = sc.extrinsics[v].to(dtype).clone().requires_grad_(True)
                k = sc.intrinsics[v].to(dtype).clone().requires_grad_(True)
                vm, pm, cp, tf, scale = camera_chain(e, k, nr, fr, scale_invariant)
                leaves = [e, k]
            else:
                leaves = [cams[i][vid].detach().cpu().to(dtype).clone().requires_grad_(True) for i in range(4)]
                vm, pm, cp, tf = leaves
                scale = 1.0 / nr if scale_invariant else 1.0
            bg = sc.background.to(dtype)
            c, d = render_view(means, cov6, opac, shs if use_sh else None, None if use_sh else shs[:, 0],
                               vm, pm, cp, tf, bg, W, H, deg, scale=scale, depth_mode=depth_mode, near=nr, far=fr)
            if target is None:
                loss = (c * dC[vid].to(dtype)).sum()
            else:
                loss = float(loss_scale[vid]) * ((c - target[vid].to(dtype)) ** 2).sum()
            if d is not None:
                loss = loss + (d * dD[vid].to(dtype)).sum()
            grads = torch.autograd.grad(loss, leaves, allow_unused=True)
            out.append([np.zeros(tuple(l.shape)) if g is None else g.double().numpy() for g, l in zip(grads, leaves)])
    return [np.stack([o[i] for o in out]) for i in range(len(out[0]))]


CASES = [
    # kind, use_sh, sh_basis, scale_invariant, loss, depth_mode, (segments, hit_lists)
    ("cfg0", True, "3dgs", True, "color", None, (0, 2)),
    ("re10k64", True, "3dgs", True, "color", None, (0, 2)),
    ("ragged", True, "3dgs", True, "color", None, (1, 0)),
    ("ragged", True, "3dgs", True, "color", None, (2, 1)),
    ("ragged", True, "3dgs", True, "color", None, (4, 1)),
    ("s2v2", True, "3dgs", True, "color", None, (0, 2)),
    ("cfg0", True, "3dgs", False, "color", None, (0, 2)),
    ("cfg0", True, "e3nn", True, "color", None, (0, 2)),
    ("cfg0", False, "3dgs", True, "color", None, (0, 2)),
    ("s2v2", True, "3dgs", True, "sse", None, (0, 2)),
    ("cfg0", True, "3dgs", True, "color", "depth", (0, 2)),
    ("cfg0", True, "3dgs", True, "color", "disparity", (0, 2)),
    ("cfg0", True, "3dgs", True, "color", "relative_disparity", (0, 2)),
    ("cfg0", True, "3dgs", True, "sse", "log", (0, 2)),
]


def _check(name, got, ref64, ref32):
    eg, e32 = _errors(got, ref64, ref32)
    assert eg <= max(1.5 * e32, 1e-5), f"{name}: norm-wise error {eg:.3e} vs float32 restatement {e32:.3e}"
    return eg, e32


@pytest.mark.parametrize("kind,use_sh,basis,scale_invariant,loss,depth_mode,variant", CASES)
def test_camera_gradients_match_float64(kind, use_sh, basis, scale_invariant, loss, depth_mode, variant):
    scenes, V, hw = _scenes(kind)
    S, H, W = len(scenes), hw[0], hw[1]
    rt.set_sh_basis(1 if basis == "e3nn" else 0)
    try:
        ext, K, near, far, means, cov, sh, opac = _stack(scenes, V, use_sh)
        n = S * V
        g = torch.Generator().manual_seed(5)
        dC = torch.randn(n, 3, H, W, generator=g)
        dD = torch.randn(n, H, W, generator=g) if depth_mode else None
        target = torch.rand(n, 3, H, W, generator=g) if loss == "sse" else None
        gs = torch.rand(n, generator=g) + 0.5
        bg = torch.stack([sc.background for sc in scenes for _ in range(V)]).to(DEV)
        cams = camera_setup(ext.reshape(n, 4, 4), K.reshape(n, 3, 3), near.reshape(n), far.reshape(n), scale_invariant)
        leaves = [cams[k].detach().clone().requires_grad_(True) for k in ("viewmatrix", "projmatrix", "campos", "tanfov")]
        colors = sh if use_sh else sh[..., 0]
        layout = _lib.PS_SH_3M if use_sh else _lib.PS_SH_M3
        nf = torch.stack([near.reshape(n), far.reshape(n)], -1)
        with util.composite_variant(2, *variant):
            color, depth, _, sse, _ = _rasterize(
                means, cov, opac, colors, viewmatrix=leaves[0], projmatrix=leaves[1], campos=leaves[2],
                tanfov=leaves[3], background=bg, image_shape=hw, views_per_scene=V,
                sh_degree=math.isqrt(sh.shape[-1]) - 1, use_sh=use_sh, sh_layout=layout,
                scene_scale=cams["scene_scale"] if scale_invariant else None, sh_basis=basis,
                target=None if target is None else target.to(DEV), depth_mode=depth_mode,
                near_far=nf if depth_mode else None)
            L = (sse * gs.to(DEV)).sum() if target is not None else (color * dC.to(DEV)).sum()
            if depth is not None:
                L = L + (depth * dD.to(DEV)).sum()
            L.backward()
        torch.cuda.synchronize()
        got = [l.grad.cpu().numpy() for l in leaves]
        args = (scenes, V, hw, use_sh, scale_invariant, leaves)
        kw = dict(dC=dC, dD=dD, depth_mode=depth_mode, loss_scale=gs, target=target)
        r64 = _oracle(*args, torch.float64, **kw)
        r32 = _oracle(*args, torch.float32, **kw)
        for i, name in enumerate(("d_viewmatrix", "d_projmatrix", "d_campos", "d_tanfov")):
            if use_sh or i != 2:
                for vid in range(n):
                    _check(f"{name}[{vid}]", got[i][vid], r64[i][vid], r32[i][vid])
        assert (got[0][:, [3, 7, 11, 15]] == 0).all() and (got[1][:, [2, 6, 10, 14]] == 0).all()
        if not use_sh:
            assert (got[2] == 0).all()

        # the same loss through the camera set-up: d_extrinsics, d_intrinsics
        e_leaf, k_leaf = ext.clone().requires_grad_(True), K.clone().requires_grad_(True)
        with util.composite_variant(2, *variant):
            if depth_mode is None and target is None:
                out = render_views(e_leaf, k_leaf, near, far, hw, bg.reshape(S, V, 3), means, cov, sh, opac,
                                   scale_invariant, use_sh=use_sh) if basis == "3dgs" else None
                if out is not None:
                    (out.reshape(n, 3, H, W) * dC.to(DEV)).sum().backward()
        if basis == "3dgs" and depth_mode is None and target is None:
            torch.cuda.synchronize()
            r64 = _oracle(scenes, V, hw, use_sh, scale_invariant, None, torch.float64, dC, dD, None,
                          through_setup=True)
            r32 = _oracle(scenes, V, hw, use_sh, scale_invariant, None, torch.float32, dC, dD, None,
                          through_setup=True)
            ge, gk = e_leaf.grad.reshape(n, 4, 4).cpu().numpy(), k_leaf.grad.reshape(n, 3, 3).cpu().numpy()
            for vid in range(n):
                _check(f"d_extrinsics[{vid}]", ge[vid], r64[0][vid], r32[0][vid])
                _check(f"d_intrinsics[{vid}]", gk[vid], r64[1][vid], r32[1][vid])
    finally:
        rt.set_sh_basis(0)


def _frozen_scene():
    sc = synthetic.scene_random_frustum(seed=0)
    t = lambda x: x.to(DEV)[None]
    return sc, t(sc.extrinsics), t(sc.intrinsics), t(sc.near), t(sc.far), t(sc.means), t(sc.covariances), \
        t(sc.harmonics), t(sc.opacities)


def test_fused_depth_extrinsics_gradient_equals_the_two_pass_route():
    from pixelsplat_b200.decoder.cuda_splatting import render_depth_views, render_views_with_depth
    sc, ext, K, near, far, means, cov, sh, opac = _frozen_scene()
    g = torch.Generator().manual_seed(0)
    dD = torch.randn(1, 1, 64, 64, generator=g).to(DEV)
    grads = []
    for fused in (True, False):
        e = ext.clone().requires_grad_(True)
        if fused:
            _, d = render_views_with_depth(e, K, near, far, (64, 64), torch.zeros(1, 1, 3, device=DEV), means, cov,
                                           sh, opac, mode="depth")
        else:
            d = render_depth_views(e, K, near, far, (64, 64), means, cov, opac, mode="depth")
        (d * dD).sum().backward()
        grads.append(e.grad.double().cpu())
    err = float((grads[0] - grads[1]).norm() / grads[1].norm())
    assert err < 1e-3, err


def test_orthographic_and_shim_deliver_camera_gradients():
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    from pixelsplat_b200.decoder.cuda_splatting import render_cuda_orthographic
    sc, ext, K, near, far, means, cov, sh, opac = _frozen_scene()
    e = ext[0].clone()
    e[:, :3, 3] = torch.tensor([0.0, 0.0, -1.0], device=DEV)
    e = e.requires_grad_(True)
    img = render_cuda_orthographic(e, torch.tensor([12.0], device=DEV), torch.tensor([12.0], device=DEV), near[0],
                                   far[0], (64, 64), torch.zeros(1, 3, device=DEV), means, cov, sh, opac)
    img.square().sum().backward()
    assert e.grad is not None and torch.isfinite(e.grad).all() and e.grad.abs().sum() > 0
    # the shim: settings built from extrinsics that require grad
    e2 = ext[0, 0].clone().requires_grad_(True)
    vm, pm, cp, tf, _ = camera_chain(e2, K[0, 0], float(sc.near[0]), float(sc.far[0]), scale_invariant=False)
    rs = GaussianRasterizationSettings(64, 64, float(tf[0]), float(tf[1]), torch.zeros(3, device=DEV), 1.0,
                                       vm.reshape(4, 4), pm.reshape(4, 4), 4, cp, False, False)
    row, col = torch.triu_indices(3, 3)
    color, _ = GaussianRasterizer(rs)(means[0], None, opac[0][:, None], shs=sh[0].permute(0, 2, 1).contiguous(),
                                      cov3D_precomp=cov[0][:, row, col])
    color.square().sum().backward()
    assert e2.grad is not None and torch.isfinite(e2.grad).all() and e2.grad.abs().sum() > 0


def test_no_camera_grad_keeps_the_launch_count_and_the_bits():
    sc, ext, K, near, far, means, cov, sh, opac = _frozen_scene()
    leaves = [t.clone().requires_grad_(True) for t in (means, cov, sh, opac)]
    counts, outs = [], []
    for cam_grad in (False, True, False):
        for l in leaves:
            l.grad = None
        e = ext.clone().requires_grad_(cam_grad)
        torch.cuda.synchronize()
        c0 = _lib.lib.ps_launch_count()
        img = render_views(e, K, near, far, (64, 64), torch.zeros(1, 1, 3, device=DEV), *leaves)
        img.square().mean().backward()
        torch.cuda.synchronize()
        counts.append(_lib.lib.ps_launch_count() - c0)
        outs.append([l.grad.clone() for l in leaves])
    # camera gradients add the finish kernel and the set-up backward; without them the count is the parent's
    assert counts[0] == counts[2] and counts[1] == counts[0] + 2
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for cam_grad in (False, True, True, True):
            for l in leaves:
                l.grad = None
            e = ext.clone().requires_grad_(cam_grad)
            img = render_views(e, K, near, far, (64, 64), torch.zeros(1, 1, 3, device=DEV), *leaves)
            img.square().mean().backward()
            runs.append(([l.grad.clone() for l in leaves], None if e.grad is None else e.grad.clone()))
        for gg, _ in runs[1:]:
            assert all(torch.equal(a, b) for a, b in zip(runs[0][0], gg))
        assert torch.equal(runs[1][1], runs[2][1]) and torch.equal(runs[1][1], runs[3][1])
    finally:
        torch.use_deterministic_algorithms(False)


def _twist(xi):
    """6-vector (rotation, translation) -> 4x4 rigid transform (exponential map of the rotation)."""
    w, t = xi[:3], xi[3:]
    z = torch.zeros((), dtype=xi.dtype, device=xi.device)
    W = torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])
    R = torch.linalg.matrix_exp(W)
    top = torch.cat([R, t[:, None]], 1)
    return torch.cat([top, torch.tensor([[0.0, 0.0, 0.0, 1.0]], device=xi.device)], 0)


def test_pose_alignment_through_render_views_mse():
    sc = synthetic.scene_re10k_like(seed=1, image_hw=(64, 64), target_views=1)
    t = lambda x: x.to(DEV)[None]
    ext, K, near, far = t(sc.extrinsics), t(sc.intrinsics), t(sc.near), t(sc.far)
    means, cov, sh, opac = t(sc.means), t(sc.covariances), t(sc.harmonics), t(sc.opacities)
    bg = torch.zeros(1, 1, 3, device=DEV)
    with torch.no_grad():
        target = render_views(ext, K, near, far, (64, 64), bg, means, cov, sh, opac)
    delta = torch.tensor([0.03, -0.04, 0.02, 0.02, -0.015, 0.01], device=DEV)   # ~3 degrees, ~2-4 % of the baseline
    xi = torch.zeros(6, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([xi], lr=2e-3)

    def errors(x):
        rel = _twist(x.detach()) @ _twist(delta)
        rot = float(torch.arccos(((rel[:3, :3].trace() - 1) / 2).clamp(-1, 1)))
        return rot, float(rel[:3, 3].norm())

    r0, t0 = errors(xi)
    for _ in range(150):
        opt.zero_grad()
        pose = ext[0, 0] @ _twist(xi) @ _twist(delta)
        sse, _, _ = render_views_mse(pose[None, None], K, near, far, (64, 64), bg, means, cov, sh, opac, target,
                                     want_color=False)
        sse.sum().backward()
        opt.step()
    r1, t1 = errors(xi)
    assert r1 * 5 <= r0 and t1 * 5 <= t0, (r0, r1, t0, t1)
