"""The colour-direction Jacobian the SH forward stores for each on-screen (view, Gaussian) pair
(ps_raster_layout.sh_jacobian, RasterOutputState.intermediates()["sh_jacobian"]), which the preprocess backward and
the camera-only backward read instead of the SH coefficients.

  * the stored rows against a float64 restatement of d(sum_k Y_k c_k) / d(direction), per SH degree, basis and
    coefficient layout, on scenes whose channels clamp: per entry within 2e-5 of the sum of its terms' magnitudes
    (sum_k |c_k| |dY_k / d direction|), which bounds float32 rounding of the sum and of the direction;
  * with precomputed colours there is no such region;
  * the backwards that read it -- several views per scene with the coefficients in either layout, and the camera-only
    backward with several views in the e3nn basis -- against the oracle."""

import numpy as np
import pytest
import torch

from oracle import raster_torch as rt
from pixelsplat_b200 import _lib, synthetic
from pixelsplat_b200.rasterizer import rasterize_gaussians
from tests import util

pytestmark = pytest.mark.gpu
DEV = util.DEV
JAC_BAR = 2e-5


def _forward(a, H, W, layout, basis):
    """One view of view_args `a` through rasterize_gaussians with the SH rows in `layout`: -> intermediates."""
    t = lambda x: x.to(DEV)[None]
    sh = a["sh"] if layout == _lib.PS_SH_M3 else a["sh"].transpose(1, 2).contiguous()
    states = []
    rasterize_gaussians(t(a["means"]), t(a["cov6"]), t(a["opac"]), t(sh), viewmatrix=t(a["vm"]),
                        projmatrix=t(a["pm"]), campos=t(a["campos"]),
                        tanfov=torch.tensor([[a["tanfovx"], a["tanfovy"]]], device=DEV),
                        background=torch.zeros(1, 3, device=DEV), image_shape=(H, W), views_per_scene=1,
                        sh_degree=a["sh_degree"], sh_layout=layout, state_out=states, sh_basis=basis)
    return {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in states[0].intermediates().items()}


def _jacobian64(a, basis):
    """float64 d(colour before the clamp) / d(direction) [P, 3 channels, 3] and the magnitude of its terms."""
    deg = a["sh_degree"]
    nb = (deg + 1) ** 2
    d = (a["means"].double() - a["campos"].double())
    d = (d / d.norm(dim=-1, keepdim=True)).requires_grad_(True)
    rt.set_sh_basis(1 if basis == "e3nn" else 0)
    try:
        y = rt.sh_basis(deg, d)                                     # [P, nb]
    finally:
        rt.set_sh_basis(0)
    dy = torch.stack([torch.autograd.grad(y[:, k].sum(), d, retain_graph=True)[0] for k in range(nb)], 1)
    c = a["sh"][:, :nb, :].double()                                 # [P, nb, 3]
    return torch.einsum("pkj,pkc->pcj", dy, c), torch.einsum("pkj,pkc->pcj", dy.abs(), c.abs())


@pytest.mark.parametrize("layout", ["M3", "3M"])
@pytest.mark.parametrize("basis", ["3dgs", "e3nn"])
@pytest.mark.parametrize("deg", [0, 1, 2, 3, 4])
def test_stored_jacobian_matches_float64(deg, basis, layout):
    sc = synthetic.scene_random_frustum(seed=70 + deg, sh_degree=deg)
    sc.harmonics *= 3.0                                             # a good share of the channels clamp
    a = util.view_args(sc)
    H, W = sc.image_shape
    im = _forward(a, H, W, _lib.PS_SH_M3 if layout == "M3" else _lib.PS_SH_3M, basis)
    vis = im["radii"][0] > 0
    cl = im["clamped"][0][vis].numpy()
    clamped = np.stack([(cl >> c) & 1 for c in range(3)], -1).astype(bool)
    assert vis.sum() > 300 and clamped.any(axis=0).all() and not clamped.all(), (int(vis.sum()), clamped.mean(0))
    got = im["sh_jacobian"][0][vis].double()
    if deg == 0:                                                    # a constant colour
        assert torch.equal(got, torch.zeros_like(got))
        return
    ref, mag = _jacobian64(a, basis)
    ref, mag = ref[vis], mag[vis]
    ratio = ((got - ref).abs() / (JAC_BAR * mag)).nan_to_num(nan=0.0, posinf=np.inf)
    worst = float(ratio.max())
    print(f"deg {deg} {basis} {layout}: {int(vis.sum())} pairs, {clamped.mean():.2f} of the channels clamp, "
          f"worst error / bar {worst:.3f}")
    assert worst <= 1.0, worst
    # the stored rows hold for clamped and unclamped channels alike (the backward masks dL/dcolour, not the rows)
    assert float(got.abs().max()) > 0.1


def test_precomputed_colours_have_no_jacobian_region():
    sc = synthetic.scene_random_frustum(seed=5, sh_degree=0)
    a = util.view_args(sc, use_sh=False)
    _, _, st, _ = util.native(a, (0.0, 0.0, 0.0), *sc.image_shape)
    assert st.intermediates()["sh_jacobian"] is None
    assert _lib.layout(st.desc).sh_jacobian == 0


@pytest.mark.parametrize("layout", ["M3", "3M"])
def test_multi_view_backward_against_the_oracle(layout):
    """S = 2 scenes x V = 3 views in one call: the view-summed Gaussian gradients of each scene against the float32
    oracle with the bars of util.check_backward (the dL/dSH rows are staged once per Gaussian, the direction terms
    of three views are added to one mean)."""
    S, V, H, W = 2, 3, 64, 64
    scs = [synthetic.scene_re10k_like(seed=80 + s, image_hw=(H, W), target_views=V) for s in range(S)]
    args = [[util.view_args(sc, view=v, scale_invariant=False) for v in range(V)] for sc in scs]
    st = lambda k: torch.stack([args[s][0][k] for s in range(S)]).to(DEV)
    cam = lambda k: torch.stack([args[s][v][k] for s in range(S) for v in range(V)]).to(DEV)
    sh = st("sh") if layout == "M3" else st("sh").transpose(2, 3).contiguous()
    leaves = [st("means").requires_grad_(True), st("cov6").requires_grad_(True), st("opac").requires_grad_(True),
              sh.requires_grad_(True)]
    tanfov = torch.tensor([[args[s][v]["tanfovx"], args[s][v]["tanfovy"]] for s in range(S) for v in range(V)],
                          device=DEV)
    color, _ = rasterize_gaussians(*leaves, viewmatrix=cam("vm"), projmatrix=cam("pm"), campos=cam("campos"),
                                   tanfov=tanfov, background=torch.zeros(S * V, 3, device=DEV), image_shape=(H, W),
                                   views_per_scene=V, sh_degree=args[0][0]["sh_degree"],
                                   sh_layout=_lib.PS_SH_M3 if layout == "M3" else _lib.PS_SH_3M)
    d_img = np.random.default_rng(3).standard_normal((S * V, 3, H, W)).astype(np.float32)
    (color * torch.as_tensor(d_img, device=DEV)).sum().backward()
    for s in range(S):
        acc = None
        for v in range(V):
            a = args[s][v]
            f = util.oracle_forward(a, (0.0, 0.0, 0.0), W, H)
            b = util.oracle_backward(f, a, d_img[s * V + v], (0.0, 0.0, 0.0), W, H)
            terms = dict(means=b.dL_dmeans, cov=b.dL_dcov6, opac=b.dL_dopacity, sh=b.dL_dsh)
            acc = terms if acc is None else {k: acc[k] + terms[k] for k in acc}
        g_sh = leaves[3].grad[s].cpu().numpy()
        got = dict(means=leaves[0].grad[s].cpu().numpy(), cov=leaves[1].grad[s].cpu().numpy(),
                   opac=leaves[2].grad[s].cpu().numpy(), sh=g_sh if layout == "M3" else np.swapaxes(g_sh, 1, 2))
        rep = {k: util.grad_errors(got[k], acc[k]) for k in got}
        print(f"S{S}xV{V} {layout} scene {s}:", {k: {m: f"{x:.2e}" for m, x in r.items()} for k, r in rep.items()})
        for k, r in rep.items():
            assert r["max"] <= 2e-3 and r["l2"] <= util.L2_BAR and r["q999"] <= 1.0, (k, rep)


def test_camera_only_backward_with_views_and_e3nn_against_float64():
    """The camera-only backward (frozen Gaussians) for 2 scenes x 2 views in the e3nn basis: its campos gradient is
    the stored Jacobian contracted with dL/dcolour.  Against the full backward's camera gradients and float64."""
    from tests.test_camera_grads_gpu import _check, _oracle
    from tests.test_pose_alignment_gpu import CAM_NAMES, _camera_grads, _rel
    case = ("s2v2", True, "e3nn", True, "color", None, (0, 2))
    rt.set_sh_basis(1)
    try:
        full, _, n_full, _ = _camera_grads(case, frozen=False, deterministic=True)
        got, gauss, n_cam, (oargs, okw) = _camera_grads(case, frozen=True, deterministic=True)
        assert all(t.grad is None for t in gauss) and n_cam == n_full
        errs = [_rel(got[i], full[i]) for i in range(4)]
        assert max(errs) <= 1e-6, errs
        r64, r32 = _oracle(*oargs, torch.float64, **okw), _oracle(*oargs, torch.float32, **okw)
        for i, name in enumerate(CAM_NAMES):
            for vid in range(got[i].shape[0]):
                _check(f"{name}[{vid}]", got[i][vid].cpu().numpy(), r64[i][vid], r32[i][vid])
        assert float(got[2].abs().max()) > 0
    finally:
        rt.set_sh_basis(0)
