"""Test-time pose alignment on the GPU: the camera-only rasterizer backward (frozen Gaussians) against the full
backward's camera gradients and against float64 autograd of the rasterizer restatement, its determinism, launch
count and CUDA-graph replay, and pixelsplat_b200.pose.align_poses end to end."""
import math

import numpy as np
import pytest
import torch

from oracle import raster_torch as rt
from pixelsplat_b200 import _lib, synthetic
from pixelsplat_b200.decoder.cuda_splatting import camera_setup, render_views, render_views_mse
from pixelsplat_b200.pose import align_poses, alignment_loss, twist_to_transform
from pixelsplat_b200.rasterizer import _rasterize
from tests import util
from tests.test_camera_grads_gpu import CASES, _check, _oracle, _scenes, _stack

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CAM_NAMES = ("d_viewmatrix", "d_projmatrix", "d_campos", "d_tanfov")


def _camera_grads(case, frozen, deterministic):
    """One forward + backward of a camera-gradient case: -> (the four camera gradients [S*V, .], the Gaussian leaves,
    the launches of the backward).  `frozen`: the Gaussians do not require grad (camera-only backward)."""
    kind, use_sh, basis, scale_invariant, loss, depth_mode, variant = case
    scenes, V, hw = _scenes(kind)
    S, H, W = len(scenes), hw[0], hw[1]
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
    gauss = [t.clone().requires_grad_(not frozen) for t in (means, cov, opac, colors)]
    layout = _lib.PS_SH_3M if use_sh else _lib.PS_SH_M3
    nf = torch.stack([near.reshape(n), far.reshape(n)], -1)
    torch.use_deterministic_algorithms(deterministic)
    try:
        with util.composite_variant(2, *variant):
            color, depth, _, sse, _ = _rasterize(
                *gauss, viewmatrix=leaves[0], projmatrix=leaves[1], campos=leaves[2],
                tanfov=leaves[3], background=bg, image_shape=hw, views_per_scene=V,
                sh_degree=math.isqrt(sh.shape[-1]) - 1, use_sh=use_sh, sh_layout=layout,
                scene_scale=cams["scene_scale"] if scale_invariant else None, sh_basis=basis,
                target=None if target is None else target.to(DEV), depth_mode=depth_mode,
                near_far=nf if depth_mode else None)
            L = (sse * gs.to(DEV)).sum() if target is not None else (color * dC.to(DEV)).sum()
            if depth is not None:
                L = L + (depth * dD.to(DEV)).sum()
            torch.cuda.synchronize()
            c0 = _lib.lib.ps_launch_count()
            L.backward()
            torch.cuda.synchronize()
            launches = _lib.lib.ps_launch_count() - c0
    finally:
        torch.use_deterministic_algorithms(False)
    oracle_args = (scenes, V, hw, use_sh, scale_invariant, leaves)
    oracle_kw = dict(dC=dC, dD=dD, depth_mode=depth_mode, loss_scale=gs, target=target)
    return [l.grad.detach().clone() for l in leaves], gauss, launches, (oracle_args, oracle_kw)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}-{c[1]}-{c[2]}-{c[3]}-{c[4]}-{c[5]}-{c[6]}" for c in CASES])
def test_camera_only_matches_the_full_path_and_float64(case):
    kind, use_sh, basis, *_ = case
    rt.set_sh_basis(1 if basis == "e3nn" else 0)
    try:
        r64 = r32 = None
        for det in (False, True):
            full, _, n_full, _ = _camera_grads(case, frozen=False, deterministic=det)
            got, gauss, n_cam, (oargs, okw) = _camera_grads(case, frozen=True, deterministic=det)
            assert all(t.grad is None for t in gauss)
            assert n_cam == n_full, (n_cam, n_full)
            errs = [_rel(got[i], full[i]) for i in range(4) if use_sh or i != 2]
            print(f"camera-only vs full [{kind} det={det}]: " + " ".join(f"{e:.2e}" for e in errs))
            assert max(errs) <= 1e-6, errs
            if r64 is None:
                r64 = _oracle(*oargs, torch.float64, **okw)
                r32 = _oracle(*oargs, torch.float32, **okw)
            for i, name in enumerate(CAM_NAMES):
                if use_sh or i != 2:
                    for vid in range(got[i].shape[0]):
                        _check(f"{name}[{vid}]", got[i][vid].cpu().numpy(), r64[i][vid], r32[i][vid])
            assert (got[0][:, [3, 7, 11, 15]] == 0).all() and (got[1][:, [2, 6, 10, 14]] == 0).all()
            if not use_sh:
                assert (got[2] == 0).all()
    finally:
        rt.set_sh_basis(0)


@pytest.mark.parametrize("kind", ["re10k64", "s2v2"])
def test_camera_only_is_bit_identical_under_the_deterministic_flag(kind):
    # re10k64 (24 576 Gaussians): the finish spreads each view over several CTAs
    case = next(c for c in CASES if c[0] == kind)
    runs = [_camera_grads(case, frozen=True, deterministic=True)[0] for _ in range(3)]
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], r))


def _re10k(S, V, hw=(64, 64), seed=0):
    """S re10k-like scenes with V target views each, stacked for render_views."""
    scenes = [synthetic.scene_re10k_like(seed=seed + s, image_hw=hw, target_views=V) for s in range(S)]
    f = lambda k: torch.stack([getattr(sc, k) for sc in scenes]).to(DEV)
    return (f("extrinsics"), f("intrinsics"), f("near"), f("far"), torch.zeros(S, V, 3, device=DEV),
            f("means"), f("covariances"), f("harmonics"), f("opacities"))


def test_camera_only_backward_has_a_fixed_launch_count():
    ext, K, near, far, bg, *gauss = _re10k(1, 2)
    counts = {}
    for frozen in (True, False, True, True):
        leaves = [t.clone().requires_grad_(not frozen) for t in gauss]
        e = ext.clone().requires_grad_(True)
        img = render_views(e, K, near, far, (64, 64), bg, *leaves)
        torch.cuda.synchronize()
        c0 = _lib.lib.ps_launch_count()
        img.square().mean().backward()
        torch.cuda.synchronize()
        counts.setdefault(frozen, []).append(_lib.lib.ps_launch_count() - c0)
    # k_clear_pair_grads, k_composite_bwd2, k_camera_bwd, k_camera_finish, k_camera_setup_backward
    assert counts[True] == [5, 5, 5], counts
    assert counts[False] == [5], counts


def _rotation_translation_error(E, E_true):
    rel = torch.linalg.inv(E_true.double()) @ E.double()
    cos = ((rel[..., 0, 0] + rel[..., 1, 1] + rel[..., 2, 2] - 1) / 2).clamp(-1, 1)
    return torch.arccos(cos), rel[..., :3, 3].norm(dim=-1)


def _perturbations(S, V, seed=0):
    """Per-view twists: rotation of ~3 degrees about a random axis, translation of 2-4 % of the 1.0 baseline."""
    g = torch.Generator().manual_seed(seed)
    axis = torch.randn(S, V, 3, generator=g)
    axis = axis / axis.norm(dim=-1, keepdim=True)
    ang = math.radians(3.0) * (0.8 + 0.4 * torch.rand(S, V, 1, generator=g))
    d = torch.randn(S, V, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True) * (0.02 + 0.02 * torch.rand(S, V, 1, generator=g))
    return torch.cat([axis * ang, d], -1).to(DEV)


def test_align_poses_converges_and_leaves_the_gaussians_untouched():
    S, V = 2, 3
    ext, K, near, far, bg, *gauss = _re10k(S, V)
    with torch.no_grad():
        target = render_views(ext, K, near, far, (64, 64), bg, *gauss)
    E0 = ext @ twist_to_transform(_perturbations(S, V))
    leaves = [t.clone().requires_grad_(True) for t in gauss]
    before = [t.detach().clone() for t in leaves]
    out = align_poses(E0, K, near, far, bg, *leaves, target, steps=150)
    torch.cuda.synchronize()
    assert all(t.grad is None for t in leaves)
    assert all(torch.equal(a.detach(), b) for a, b in zip(leaves, before))
    r0, t0 = _rotation_translation_error(E0, ext)
    r1, t1 = _rotation_translation_error(out.extrinsics, ext)
    print("rotation error (rad) before / after:", r0.flatten().tolist(), r1.flatten().tolist())
    print("translation error before / after:", t0.flatten().tolist(), t1.flatten().tolist())
    print("final per-view MSE:", out.loss.flatten().tolist())
    assert (r1 * 5 <= r0).all() and (t1 * 5 <= t0).all()
    assert out.loss.shape == (S, V) and torch.isfinite(out.loss).all()
    # each view aligned alone reaches the pose it reaches inside the batch
    for s in range(S):
        for v in range(V):
            one = align_poses(E0[s:s + 1, v:v + 1], K[s:s + 1, v:v + 1], near[s:s + 1, v:v + 1],
                              far[s:s + 1, v:v + 1], bg[s:s + 1, v:v + 1], *[t[s:s + 1] for t in gauss],
                              target[s:s + 1, v:v + 1], steps=150)
            dr, dt = _rotation_translation_error(one.extrinsics[0, 0], out.extrinsics[s, v])
            print(f"alone vs batch ({s}, {v}): rotation {float(dr):.2e} rad, translation {float(dt):.2e}")
            assert float(dr) <= 2e-3 and float(dt) <= 2e-3, (s, v, float(dr), float(dt))


def test_alignment_step_replays_in_a_cuda_graph():
    ext, K, near, far, bg, *gauss = _re10k(1, 2)
    with torch.no_grad():
        target = render_views(ext, K, near, far, (64, 64), bg, *gauss)
    E0 = ext @ twist_to_transform(_perturbations(1, 2, seed=3))
    xi = torch.zeros(1, 2, 6, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([xi], lr=2e-3, capturable=True)
    states = []

    def step():
        opt.zero_grad(set_to_none=False)
        sse = alignment_loss(xi, E0, K, near, far, bg, *gauss, target)
        sse.sum().backward()
        opt.step()

    torch.use_deterministic_algorithms(True)
    try:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):          # eager warm-up: Adam state, the rasterizer's capacity for this shape
                step()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        snap = [xi.detach().clone()] + [opt.state[xi][k].clone() for k in ("step", "exp_avg", "exp_avg_sq")]

        def restore():
            with torch.no_grad():
                xi.copy_(snap[0])
                for k, t in zip(("step", "exp_avg", "exp_avg_sq"), snap[1:]):
                    opt.state[xi][k].copy_(t)

        graph = torch.cuda.CUDAGraph()
        import pixelsplat_b200.rasterizer as rz
        captured = []
        orig = rz._forward

        def spy(*a, **k):
            out = orig(*a, **k)
            captured.append(out[2])
            return out

        rz._forward = spy
        try:
            with torch.cuda.graph(graph):
                step()
        finally:
            rz._forward = orig
        restore()
        for _ in range(4):
            graph.replay()
        torch.cuda.synchronize()
        for st in captured:
            st.verify()                  # the instance count of the replayed forward, checked after the replay
            assert st.num_instances() <= st.desc.instance_capacity
        replayed = xi.detach().clone()
        restore()
        for _ in range(4):
            step()
        torch.cuda.synchronize()
        assert torch.equal(replayed, xi.detach()), (replayed - xi.detach()).abs().max()
        assert not torch.equal(replayed, snap[0])
    finally:
        torch.use_deterministic_algorithms(False)
