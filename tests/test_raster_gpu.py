"""GPU parity tests of the rasterizer: CUDA path (through the C ABI) vs the CPU oracle on the same
seeded inputs.  Bars (BASELINE.json north_star):
  * bit-exact: depth keys, radii, tile rectangles, per-tile counts/offsets, the sorted
    (key, Gaussian) list;  preprocess float outputs (compiled without FMA) are also bit-exact;
  * fp32 tolerance for images: |diff| <= 2e-5 on >= 99.9 % of pixels and PSNR > 60 dB; a pixel may
    differ more only where an alpha sits on the 1/255 or T < 1e-4 decision boundary (the GPU uses
    ex2.approx; the oracle libm expf), bounded by 1e-2;
  * gradients: relative max error <= 2e-3 of the largest entry (atomic summation order differs).
"""
import numpy as np
import pytest
import torch

from pixelsplat_b200 import synthetic
from tests import util

pytestmark = pytest.mark.gpu

DEV = util.DEV
L2_BAR = util.L2_BAR
_native, _check_forward, _check_backward = util.native, util.check_forward, util.check_backward


@pytest.mark.parametrize("sort_impl", [0, 1])
def test_config0_forward(sort_impl):
    """BASELINE configs[0]: 64x64, 1k random Gaussians, 1 view."""
    sc = synthetic.scene_random_frustum(seed=0)
    _check_forward(util.view_args(sc), (0.0, 0.0, 0.0), *sc.image_shape, sort_impl=sort_impl)


def test_config0_backward_nonzero_background():
    sc = synthetic.scene_random_frustum(seed=3)
    _check_backward(util.view_args(sc), (0.1, 0.2, 0.3), *sc.image_shape)


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_lower_sh_degrees(deg):
    sc = synthetic.scene_random_frustum(seed=4, sh_degree=deg)
    a = util.view_args(sc)
    _check_forward(a, (0.0, 0.0, 0.0), *sc.image_shape)
    _check_backward(a, (0.0, 0.0, 0.0), *sc.image_shape)


@pytest.mark.parametrize("deg", [1, 2, 4])
def test_e3nn_sh_basis_matches_oracle(deg):
    """PS_SH_BASIS_E3NN (y polar, no Condon-Shortley sign: the basis the reference's rotate_sh rotates in,
    sh_rotation.py:18-22): rgb stays bit-exact against the oracle evaluated in the same convention, gradients
    within the usual bar; and it is a different image from the default basis."""
    from oracle import raster_oracle as ro
    sc = synthetic.scene_random_frustum(seed=40 + deg, sh_degree=deg)
    sc.harmonics *= 3.0
    a = util.view_args(sc)
    with ro.sh_basis(1):
        _, color_e = _check_forward(a, (0.0, 0.0, 0.0), *sc.image_shape, sh_basis="e3nn")
        _check_backward(a, (0.0, 0.0, 0.0), *sc.image_shape, sh_basis="e3nn")
    color_g, _, _, _ = _native(a, (0.0, 0.0, 0.0), *sc.image_shape)
    assert np.abs(color_e - color_g).max() > 1e-2
    with pytest.raises(ValueError, match="unknown SH convention"):
        _native(a, (0.0, 0.0, 0.0), *sc.image_shape, sh_basis="opengl")


def test_colors_precomp_path():
    sc = synthetic.scene_random_frustum(seed=5, sh_degree=0)
    a = util.view_args(sc, use_sh=False)
    _check_forward(a, (0.2, 0.0, 0.1), *sc.image_shape)
    _check_backward(a, (0.2, 0.0, 0.1), *sc.image_shape)


def test_ragged_image_size_and_dense_stack():
    """70x50 (partial tiles) with 4k opaque Gaussians: exercises early termination."""
    sc = synthetic.scene_random_frustum(seed=6, image_hw=(50, 70), num_gaussians=4000, z_range=(1.0, 4.0))
    a = util.view_args(sc)
    f, _ = _check_forward(a, (0.0, 0.0, 0.0), 50, 70)
    assert (f.final_T < 1e-3).mean() > 0.05, "scene should saturate some pixels"
    _check_backward(a, (0.0, 0.0, 0.0), 50, 70)


def test_long_tiles_use_every_sort_path():
    """One 16x16 image, 30k Gaussians on it: the single tile exceeds the shared-memory sort
    capacities (2048 / 12288) and takes the global ping-pong path."""
    sc = synthetic.scene_random_frustum(seed=7, image_hw=(16, 16), num_gaussians=30000, z_range=(2.0, 30.0))
    a = util.view_args(sc)
    f, _ = _check_forward(a, (0.0, 0.0, 0.0), 16, 16)
    assert f.binned.keys.size > 12288
    sc = synthetic.scene_random_frustum(seed=8, image_hw=(32, 32), num_gaussians=14000, z_range=(2.0, 30.0))
    f, _ = _check_forward(util.view_args(sc), (0.0, 0.0, 0.0), 32, 32)
    cnt = f.binned.ranges[:, 1] - f.binned.ranges[:, 0]
    assert cnt.max() > 2048


def test_empty_and_single():
    """Nothing visible (all behind the camera) and a single Gaussian."""
    sc = synthetic.scene_random_frustum(seed=9, num_gaussians=64)
    sc.means[:, 2] = -sc.means[:, 2]
    a = util.view_args(sc)
    f, color = _check_forward(a, (0.3, 0.4, 0.5), *sc.image_shape)
    assert f.binned.keys.size == 0
    assert np.allclose(color, np.array([0.3, 0.4, 0.5], np.float32)[:, None, None])
    d_img = np.ones((3, 64, 64), np.float32)
    _, _, _, g = _native(a, (0.3, 0.4, 0.5), 64, 64, 0, d_img)
    assert all(np.all(v == 0) for v in g.values())
    sc1 = synthetic.scene_random_frustum(seed=10, num_gaussians=1)
    sc1.means[0] = torch.tensor([0.0, 0.0, 3.0])
    _check_forward(util.view_args(sc1), (0.0, 0.0, 0.0), *sc1.image_shape)
    _check_backward(util.view_args(sc1), (0.0, 0.0, 0.0), *sc1.image_shape)


def test_capacity_overflow_reruns():
    from pixelsplat_b200 import rasterizer
    sc = synthetic.scene_random_frustum(seed=11, num_gaussians=3000)
    a = util.view_args(sc)
    H, W = sc.image_shape
    rasterizer._capacity_hint[(0, 1, 1, 3000, H, W)] = 16   # far too small
    _check_forward(a, (0.0, 0.0, 0.0), H, W)
    assert rasterizer._capacity_hint[(0, 1, 1, 3000, H, W)] > 16


def test_config1_full_size():
    """BASELINE configs[1]: 2 context views -> 1 target, 256x256, 3 Gaussians/pixel (P = 393 216)."""
    sc = synthetic.scene_re10k_like(seed=0)
    a = util.view_args(sc)
    f, color = _check_forward(a, (0.0, 0.0, 0.0), 256, 256)
    print("config1: N =", f.binned.keys.size, "visible =", int((f.pre.radii > 0).sum()))
    _check_backward(a, (0.0, 0.0, 0.0), 256, 256, fwd=f)


def test_config4_high_res_tile_stress():
    """BASELINE configs[4] (one scene of it): 3 context views, 512x512 target, P = 2 359 296."""
    sc = synthetic.scene_re10k_like(seed=1, image_hw=(512, 512), context_views=3)
    a = util.view_args(sc)
    f, _ = _check_forward(a, (0.0, 0.0, 0.0), 512, 512)
    print("config4: N =", f.binned.keys.size)
    # backward at full size against the float64 oracle (norm-wise + percentile bars)
    _check_backward(a, (0.0, 0.0, 0.0), 512, 512, with_f64=False, fwd=f)
    torch.cuda.synchronize()
    print("config4: peak device memory %.2f GiB" % (torch.cuda.max_memory_allocated() / 2 ** 30))


def test_batched_scenes_and_views_against_the_oracle():
    """S = 2 scenes x V = 4 target views at 256x256 in ONE call (the training shape: 4 views per scene share the
    scene's Gaussians) against the ORACLE view by view: images, and the view-summed gradients of scene 0 (float32
    oracle, composite sums in float64; bars of _check_backward)."""
    from concurrent.futures import ThreadPoolExecutor

    from pixelsplat_b200.decoder import render_views
    S, V, H, W = 2, 4, 256, 256
    scs = [synthetic.scene_re10k_like(seed=60 + i, image_hw=(H, W), target_views=V) for i in range(S)]
    t = lambda x: x.to(DEV)
    st = lambda name: torch.stack([t(getattr(s, name)) for s in scs])
    leaves = [st("means").requires_grad_(True), st("covariances").requires_grad_(True),
              st("harmonics").requires_grad_(True), st("opacities").requires_grad_(True)]
    bg = torch.zeros(S, V, 3, device=DEV)
    out = render_views(st("extrinsics"), st("intrinsics"), st("near"), st("far"), (H, W), bg, *leaves)
    d_img = np.random.default_rng(5).standard_normal((S, V, 3, H, W)).astype(np.float32)
    (out * torch.as_tensor(d_img, device=DEV)).sum().backward()
    got = out.detach().cpu().numpy()

    def view_job(sv):
        s, v = sv
        a = util.view_args(scs[s], view=v)
        f = util.oracle_forward(a, (0.0, 0.0, 0.0), W, H)
        b64 = util.oracle_backward(f, a, d_img[s, v], (0.0, 0.0, 0.0), W, H) if s == 0 else None
        return s, v, f.color, b64, float(scs[s].near[v])

    with ThreadPoolExecutor(8) as ex:          # the C oracle releases the GIL
        jobs = list(ex.map(view_job, [(s, v) for s in range(S) for v in range(V)]))
    acc = None
    for s, v, color, b64, near in jobs:
        diff = np.abs(got[s, v] - color)
        assert (diff <= 1e-4).mean() >= 0.995 and util.psnr(got[s, v], color) > 50.0, (s, v, diff.max())
        if b64 is not None:
            # the oracle differentiates w.r.t. the RESCALED scene (means * 1/near, cov * 1/near^2): chain rule
            sc_ = 1.0 / near
            terms = dict(means=b64.dL_dmeans * sc_, cov6=b64.dL_dcov6 * sc_ * sc_, sh=b64.dL_dsh, opac=b64.dL_dopacity)
            acc = terms if acc is None else {k: acc[k] + terms[k] for k in acc}
    row, col = np.triu_indices(3)
    g_cov = leaves[1].grad[0].cpu().numpy()
    assert not np.tril(g_cov, -1).any()                       # only the upper triangle is read / receives gradient
    rep = dict(means=util.grad_errors(leaves[0].grad[0].cpu().numpy(), acc["means"]),
               cov=util.grad_errors(g_cov[:, row, col], acc["cov6"]),
               sh=util.grad_errors(leaves[2].grad[0].cpu().numpy(), np.transpose(acc["sh"], (0, 2, 1))),
               opac=util.grad_errors(leaves[3].grad[0].cpu().numpy(), acc["opac"]))
    print("S2xV4 grad errors vs oracle:", {k: {m: f"{v:.2e}" for m, v in r.items()} for k, r in rep.items()})
    for k, r in rep.items():
        assert r["l2"] <= L2_BAR and r["q999"] <= 1.0, (k, rep)


def test_render_cuda_api_matches_oracle():
    """Through the reference-facing Python API (render_cuda signature, native layouts, fused
    scale-invariant rescale, on-device camera set-up): tolerance only, since the matrices are
    computed on the device."""
    from pixelsplat_b200.decoder import render_cuda
    sc = synthetic.scene_re10k_like(seed=2, image_hw=(128, 128))
    t = lambda x: x.to(DEV)
    img = render_cuda(t(sc.extrinsics), t(sc.intrinsics), t(sc.near), t(sc.far), sc.image_shape,
                      t(sc.background)[None], t(sc.means)[None], t(sc.covariances)[None],
                      t(sc.harmonics)[None], t(sc.opacities)[None])
    f = util.oracle_forward(util.view_args(sc), (0.0, 0.0, 0.0), 128, 128)
    got = img[0].cpu().numpy()
    assert util.psnr(got, f.color) > 50.0
    assert (np.abs(got - f.color) <= 1e-4).mean() > 0.995


def test_shared_gaussians_multi_view_and_gradient_sum():
    """S=2 scenes x V=3 views in one call == six single-view calls; gradients sum over views."""
    from pixelsplat_b200.decoder import render_views
    scs = [synthetic.scene_re10k_like(seed=20 + i, image_hw=(64, 64), target_views=3) for i in range(2)]
    t = lambda x: x.to(DEV)
    st = lambda name: torch.stack([t(getattr(s, name)) for s in scs])
    leaves = [st("means").requires_grad_(True), st("covariances").requires_grad_(True),
              st("harmonics").requires_grad_(True), st("opacities").requires_grad_(True)]
    bg = torch.zeros(2, 3, 3, device=DEV)
    out = render_views(st("extrinsics"), st("intrinsics"), st("near"), st("far"), (64, 64), bg, *leaves)
    w = torch.randn_like(out)
    (out * w).sum().backward()
    g_batched = [l.grad.clone() for l in leaves]
    for l in leaves:
        l.grad = None
    total = 0
    for s in range(2):
        for v in range(3):
            o = render_views(st("extrinsics")[s:s + 1, v:v + 1], st("intrinsics")[s:s + 1, v:v + 1],
                             st("near")[s:s + 1, v:v + 1], st("far")[s:s + 1, v:v + 1], (64, 64),
                             bg[s:s + 1, v:v + 1], *[l[s:s + 1] for l in leaves])
            assert torch.allclose(o[0, 0], out[s, v], atol=1e-6)
            total = total + (o[0, 0] * w[s, v]).sum()
    total.backward()
    for gb, l in zip(g_batched, leaves):
        assert util.rel_err(gb.cpu().numpy(), l.grad.cpu().numpy()) < 1e-3


def test_gaussian_rasterizer_dropin_surface():
    """The extension classes the reference imports (cuda_splatting.py:5-8): argument checks and a
    render through them."""
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    sc = synthetic.scene_random_frustum(seed=12)
    a = util.view_args(sc)
    t = lambda x: x.to(DEV)
    H, W = sc.image_shape
    settings = GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=a["tanfovx"], tanfovy=a["tanfovy"],
        bg=torch.zeros(3, device=DEV), scale_modifier=1.0, viewmatrix=t(a["vm"]).reshape(4, 4),
        projmatrix=t(a["pm"]).reshape(4, 4), sh_degree=a["sh_degree"], campos=t(a["campos"]),
        prefiltered=False, debug=False)
    r = GaussianRasterizer(settings)
    m2d = torch.zeros_like(t(a["means"]), requires_grad=True)
    img, radii = r(means3D=t(a["means"]), means2D=m2d, shs=t(a["sh"]), colors_precomp=None,
                   opacities=t(a["opac"])[:, None], cov3D_precomp=t(a["cov6"]))
    f = util.oracle_forward(a, (0, 0, 0), W, H)
    assert img.shape == (3, H, W) and radii.dtype == torch.int32
    assert util.psnr(img.detach().cpu().numpy(), f.color) > 60
    img.sum().backward()
    assert m2d.grad is not None and m2d.grad.shape == m2d.shape
    with pytest.raises(Exception, match="SHs or precomputed colors"):
        r(means3D=t(a["means"]), means2D=m2d, opacities=t(a["opac"])[:, None], cov3D_precomp=t(a["cov6"]))
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(means3D=t(a["means"]), means2D=m2d, shs=t(a["sh"]), opacities=t(a["opac"])[:, None])
    with pytest.raises(ValueError, match="CUDA tensor"):
        r(means3D=a["means"], means2D=None, shs=a["sh"], opacities=a["opac"][:, None], cov3D_precomp=a["cov6"])


def test_idempotent_and_deterministic_forward():
    """Size-independent property: the forward (including the atomic scatter + sort) is
    bit-reproducible run to run."""
    sc = synthetic.scene_re10k_like(seed=5, image_hw=(128, 128))
    a = util.view_args(sc)
    c1, r1, s1, _ = _native(a, (0, 0, 0), 128, 128)
    c2, r2, s2, _ = _native(a, (0, 0, 0), 128, 128)
    assert np.array_equal(c1, c2) and np.array_equal(r1, r2)
    assert torch.equal(s1.intermediates()["keys"], s2.intermediates()["keys"])


def test_known_answers_on_the_gpu():
    """The hand-derived cases of tests/test_oracle_raster.py, through the CUDA path: a Gaussian
    centred on a pixel, front-to-back order of two overlapping Gaussians given far-first, the
    z <= 0.2 cull boundary, and the four-tile corner case."""
    from oracle import raster_torch as rt
    from pixelsplat_b200.rasterizer import rasterize_gaussians
    W = H = 64
    K = torch.tensor([[0.88, 0, 0.5], [0, 0.88, 0.5], [0, 0, 1.0]])
    vm, pm, cp, tx, ty = rt.camera_from_c2w(torch.eye(4), K, 0.5, 100.0, torch.float32)
    C0 = 0.28209479177387814

    def pt(i, j, z):
        return [((2 * i + 1) / W - 1) * tx * z, ((2 * j + 1) / H - 1) * ty * z, z]

    def iso(s):
        return [s * s, 0, 0, s * s, 0, s * s]

    def run(means, cov6, opac, sh, bg=(0.0, 0.0, 0.0)):
        t = lambda x: torch.tensor(x, dtype=torch.float32, device=DEV)
        states = []
        color, radii = rasterize_gaussians(
            t(means)[None], t(cov6)[None], t(opac)[None], t(sh)[None], viewmatrix=vm.to(DEV)[None],
            projmatrix=pm.to(DEV)[None], campos=cp.to(DEV)[None], tanfov=t([[tx, ty]]), background=t([list(bg)]),
            image_shape=(H, W), views_per_scene=1, sh_degree=0, state_out=states)
        return color[0].cpu().numpy(), radii[0].cpu().numpy(), states[0].intermediates()

    # one Gaussian on a pixel centre: alpha = min(0.99, opacity), colour = C0 * sh0 + 0.5
    for opacity in (0.5, 1.0):
        color, _, im = run([pt(20, 30, 5.0)], [iso(0.05)], [opacity], [[[1.0, -0.5, 0.2]]])
        alpha = min(0.99, opacity)
        expect = np.maximum(C0 * np.array([1.0, -0.5, 0.2]) + 0.5, 0) * alpha
        assert np.allclose(color[:, 30, 20], expect, atol=1e-5)
        assert abs(float(im["final_T"][0, 30, 20]) - (1 - alpha)) < 1e-5 and int(im["n_contrib"][0, 30, 20]) == 1
    # two overlapping Gaussians, far one listed first
    sh = [[[(1.0 - 0.5) / C0] * 3], [[(0.25 - 0.5) / C0] * 3]]
    color, _, im = run([pt(10, 10, 4.0), pt(10, 10, 2.0)], [iso(0.1), iso(0.05)], [0.8, 0.6], sh, bg=(0.5, 0.5, 0.5))
    expect = 0.25 * 0.6 + 1.0 * 0.8 * 0.4 + 0.5 * 0.4 * 0.2
    assert np.allclose(color[:, 10, 10], expect, atol=1e-5)
    assert (im["keys"][:2].cpu().numpy() & 0xFFFFFFFF).tolist() == [1, 0]
    # cull boundary
    z_above = float(np.nextafter(np.float32(0.2), np.float32(1)))
    _, radii, _ = run([[0, 0, 0.2], [0, 0, z_above]], [iso(0.001)] * 2, [0.5, 0.5], [[[0.0] * 3]] * 2)
    assert radii[0] == 0 and radii[1] > 0
    # tile corner -> exactly four tiles
    z = 5.0
    p = [((2 * 15.5 + 1) / W - 1) * tx * z, ((2 * 15.5 + 1) / H - 1) * ty * z, z]
    _, _, im = run([p], [iso(0.02)], [0.9], [[[0.0] * 3]])
    assert im["num_instances"] == 4 and im["tile_count"][0].cpu().numpy().nonzero()[0].tolist() == [0, 1, 4, 5]


def test_equal_depth_ties_are_broken_by_index():
    """All Gaussians on one plane parallel to the image (identical depth bits): the per-tile order
    must fall back to ascending Gaussian index -- short runs, and a run long enough (> 64) to take
    the sort's fallback path."""
    sc = synthetic.scene_random_frustum(seed=13, image_hw=(32, 32), num_gaussians=900)
    sc.means[:, 2] = 3.0
    sc.means[:300, 2] = 5.0
    _check_forward(util.view_args(sc), (0.0, 0.0, 0.0), 32, 32)


def test_depth_and_orthographic_entry_points():
    """render_depth_cuda (all four modes) against an oracle render with depth as colour, and
    render_cuda_orthographic against an oracle render with the same far-away narrow camera
    (cuda_splatting.py:130-269)."""
    from oracle import raster_torch as rt
    from pixelsplat_b200.decoder import render_cuda_orthographic, render_depth_cuda
    sc = synthetic.scene_re10k_like(seed=30, image_hw=(64, 64))
    t = lambda x: x.to(DEV)
    H = W = 64
    w2c = torch.linalg.inv(sc.extrinsics[0])
    z = (w2c[2, :3] * sc.means).sum(-1) + w2c[2, 3]
    near, far = sc.near[0], sc.far[0]
    fakes = {"depth": z, "disparity": 1 / z,
             "relative_disparity": 1 - (1 / (z + 1e-10) - 1 / (far + 1e-10)) / (1 / (near + 1e-10) - 1 / (far + 1e-10) + 1e-10),
             "log": z.minimum(near).maximum(far).log()}
    for mode, fake in fakes.items():
        got = render_depth_cuda(t(sc.extrinsics), t(sc.intrinsics), t(sc.near), t(sc.far), (H, W), t(sc.means)[None],
                                t(sc.covariances)[None], t(sc.opacities)[None], mode=mode)
        a = rt.prepare_view(sc.means, sc.covariances, fake[:, None, None].expand(-1, 3, 1).contiguous(), sc.opacities,
                            sc.extrinsics[0], sc.intrinsics[0], near, far, use_sh=False)
        f = util.oracle_forward(a, (0, 0, 0), W, H)
        ref = f.color.mean(0)
        assert got.shape == (1, H, W)
        err = np.abs(got[0].cpu().numpy() - ref)
        assert np.quantile(err, 0.995) <= 1e-3 * max(1.0, np.abs(ref).max()), (mode, err.max())
    # orthographic: compare with the oracle given the same "moved back" camera
    dump = {}
    bg = torch.zeros(1, 3, device=DEV)
    width, height = torch.tensor([2.0], device=DEV), torch.tensor([2.0], device=DEV)
    ext = torch.eye(4)[None]
    ext[0, 2, 3] = -1.0
    img = render_cuda_orthographic(t(ext), width, height, torch.tensor([0.0], device=DEV),
                                   torch.tensor([50.0], device=DEV), (H, W), bg, t(sc.means)[None],
                                   t(sc.covariances)[None], t(sc.harmonics)[None], t(sc.opacities)[None], dump=dump)
    assert img.shape == (1, 3, H, W) and torch.isfinite(img).all()
    assert set(dump) == {"extrinsics", "fov_x", "fov_y", "near", "far"}
    assert img.abs().sum() > 0
