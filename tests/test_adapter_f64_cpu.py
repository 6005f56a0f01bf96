"""CPU tests of the float64 adapter restatement (tests/adapter_f64.py) and of its per-entry bars, before they are
pointed at the fused kernels (tests/test_adapter_sweep_gpu.py).

  * The restatement, fed D = sh.sh_rotation_matrices(...) in float64, equals GaussianAdapter.forward_explicit in
    float64 and the reference module's float64 golden (tests/golden/adapter_v2.npz) at the bars of
    test_adapter_cpu.py::test_explicit_adapter_path_matches_reference_f64.
  * torch.autograd.gradcheck on a tiny case; the zero-quaternion limit d_raw = d_rot / eps.
  * Sensitivity: planted errors that today's max-norm bars (the golden test's max(4 own, 1e-6) and the explicit-path
    sweep's 5e-6 / 2e-5, tests/test_adapter_gpu.py) accept and the per-entry bars reject.  Measured here (float64):
      (1) the degree-4 block of d_raw off by 1 % (golden case): max-norm error 3.7e-7 against the golden test's bar
          1.4e-6 and the sweep's 2e-5 -- both accept; the per-entry d_raw_sh bar sees 10000x its bar.
      (2) the degree-4 harmonics of the second block's rays off by 0.5 % (3 views x 161 rays): max-norm error 2.0e-6,
          accepted by the sweep's 5e-6 (the golden test's 1e-6 happens to catch it); per-entry 5700x.
      (3) the covariances of the nearest 5 % of Gaussians off by 1 %: max-norm error 1.4e-5 (both old bars reject it
          on this case, whose depths reach only 0.29); per-entry 2500x.
      (4) two neighbouring rays of the second block swapped: every old bar rejects it as well; per-entry 5.7e6x.
    And no per-entry bar is looser than the max-norm bar it replaces: on both cases every entry's allowance is at
    most 0.8 of the old one (covariances 0.8, d_raw 0.55, the others 0.1-0.33).
"""
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import adapter_f64 as af
from tests import golden_util as gu
from tests.util import rel_err

GOLD = np.load(Path(__file__).resolve().parent / "golden" / "adapter_v2.npz")
IMAGE_SHAPE = (48, 64)


def _abi(c, n_sh=25):
    """adapter_case inputs in the ABI's layout, with the golden loss's weights as cotangents (the rotations' cotangent
    summed over the samples the module broadcasts them to)."""
    b, v, r, srf, spp = c["depths"].shape
    nv, nr = b * v, r * srf
    w = c["weights"]
    cot = dict(d_means=w["means"].reshape(nv, nr, spp, 3), d_cov=1e3 * w["covariances"].reshape(nv, nr, spp, 3, 3),
               d_harm=w["harmonics"].reshape(nv, nr, spp, 3, n_sh), d_scales=10.0 * w["scales"].reshape(nv, nr, spp, 3),
               d_rot=w["rotations"].reshape(nv, nr, spp, 4).sum(2))
    E = c["extrinsics"].reshape(nv, 4, 4)
    from pixelsplat_b200 import sh
    D = sh.sh_rotation_matrices(E[:, :3, :3], af.sh_degree(n_sh))
    args = (E, c["intrinsics"].reshape(nv, 3, 3), D, af.sh_mask(n_sh), c["coordinates"].reshape(nv, nr, 2),
            c["depths"].reshape(nv, nr, spp), c["raw"].reshape(nv, nr, 7 + 3 * n_sh), IMAGE_SHAPE, 0.5, 15.0, 1e-8)
    return args, cot


def _golden(case, k, shape):
    return torch.from_numpy(GOLD[f"{case}_f64_{k}"]).reshape(shape)


@pytest.mark.parametrize("case", ["generic", "diverging"])
def test_restatement_equals_explicit_path_and_reference_f64(case):
    from pixelsplat_b200.encoder.gaussian_adapter import GaussianAdapter, GaussianAdapterCfg
    c = gu.adapter_case(case=case)
    args, cot = _abi(c)
    got = af.forward_backward(*args, cot)
    # the product's torch path, float64
    leaves = {k: c[k].clone().requires_grad_(True) for k in ("coordinates", "depths", "opacities", "raw")}
    ad = GaussianAdapter(GaussianAdapterCfg(0.5, 15.0, 4)).double()
    ad.sh_mask = ad.sh_mask.double()
    assert torch.equal(ad.sh_mask, af.sh_mask(25))
    g = ad.forward_explicit(c["extrinsics"], c["intrinsics"], leaves["coordinates"], leaves["depths"],
                            leaves["opacities"], leaves["raw"], IMAGE_SHAPE)
    gu.adapter_loss(g, c["weights"]).backward()
    for k in ("means", "covariances", "harmonics", "scales"):
        e = getattr(g, k).detach().reshape(got[k].shape)
        assert rel_err(got[k].numpy(), e.numpy()) < 1e-13, k
        assert rel_err(got[k].numpy(), _golden(case, k, got[k].shape).numpy()) < 1e-11, k
    rot = g.rotations.detach()[..., 0, :].reshape(got["rotations"].shape)
    assert rel_err(got["rotations"].numpy(), rot.numpy()) < 1e-14
    assert rel_err(got["rotations"].numpy(), _golden(case, "rotations", rot.shape).numpy()) < 1e-12
    for k, leaf in (("d_coordinates", "coordinates"), ("d_depths", "depths"), ("d_raw", "raw")):
        e = leaves[leaf].grad.reshape(got[k].shape)
        assert rel_err(got[k].numpy(), e.numpy()) < 1e-12, k
        assert rel_err(got[k].numpy(), _golden(case, "d_" + leaf, got[k].shape).numpy()) < 1e-9, k
    # the restatement held to its own bars: every ratio is float64 round-off
    assert max(af.check(got, got, tag=case).values()) == 0.0


def _tiny(seed=0, n_sh=4, nv=2, nr=3, ns=2):
    """A generic small call: random rotations and origins, a skewed K and a generic one, coordinates off the image."""
    from pixelsplat_b200 import sh
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(nv, 4, generator=g, dtype=torch.float64)
    from pixelsplat_b200.encoder.gaussian_adapter import quaternion_to_matrix
    E = torch.eye(4, dtype=torch.float64).repeat(nv, 1, 1)
    E[:, :3, :3] = quaternion_to_matrix(q / q.norm(dim=-1, keepdim=True), eps=0.0)
    E[:, :3, 3] = torch.randn(nv, 3, generator=g, dtype=torch.float64)
    K = torch.tensor([[1.1, 0.07, 0.45], [0.0, 0.8, 0.55], [0.0, 0.0, 1.0]], dtype=torch.float64).repeat(nv, 1, 1)
    K[1:] += 0.05 * torch.randn(nv - 1, 3, 3, generator=g, dtype=torch.float64)
    D = sh.sh_rotation_matrices(E[:, :3, :3], af.sh_degree(n_sh))
    coords = -0.5 + 2 * torch.rand(nv, nr, 2, generator=g, dtype=torch.float64)
    depths = 0.5 + 20 * torch.rand(nv, nr, ns, generator=g, dtype=torch.float64)
    raw = torch.randn(nv, nr, 7 + 3 * n_sh, generator=g, dtype=torch.float64)
    cot = dict(d_means=torch.randn(nv, nr, ns, 3, generator=g, dtype=torch.float64),
               d_cov=torch.randn(nv, nr, ns, 3, 3, generator=g, dtype=torch.float64),
               d_harm=torch.randn(nv, nr, ns, 3, n_sh, generator=g, dtype=torch.float64),
               d_scales=torch.randn(nv, nr, ns, 3, generator=g, dtype=torch.float64),
               d_rot=torch.randn(nv, nr, 4, generator=g, dtype=torch.float64))
    return (E, K, D, af.sh_mask(n_sh), coords, depths, raw, (5, 7), 0.3, 9.0, 1e-8), cot


def test_gradcheck():
    args, _ = _tiny()
    E, K, D, mask, coords, depths, raw, hw, smin, smax, eps = args
    fn = lambda c, d, r: tuple(af.forward(E, K, D, mask, c, d, r, hw, smin, smax, eps).values())
    leaves = [t.clone().requires_grad_(True) for t in (coords, depths, raw)]
    assert torch.autograd.gradcheck(fn, leaves, eps=1e-6, atol=1e-7, rtol=1e-5)


def test_zero_quaternion_gradient_is_d_rot_over_eps():
    """At qr = 0 the rotation matrix is the identity, flat to first order (every entry is quadratic in q), so the only
    gradient reaching qr is the rotations output's: d_raw[3:7] = d_rot / eps, the kernel's corr = 0 branch."""
    args, cot = _tiny(seed=1)
    raw = args[6].clone()
    raw[0, 1, 3:7] = 0.0
    raw[1, 2, 3:7] = 0.0
    args = args[:6] + (raw,) + args[7:]
    eps = args[-1]
    res = af.forward_backward(*args, cot)
    for v, r in ((0, 1), (1, 2)):
        assert torch.equal(res["rotations"][v, r], torch.zeros(4, dtype=torch.float64))
        want = cot["d_rot"][v, r] / eps
        assert torch.allclose(res["d_raw"][v, r, 3:7], want, rtol=1e-12, atol=0), (res["d_raw"][v, r, 3:7], want)
        C = args[0][v, :3, :3]
        s2 = res["scales"][v, r] ** 2
        assert torch.allclose(res["covariances"][v, r], C @ torch.diag_embed(s2) @ C.T, rtol=1e-12, atol=1e-15)
    assert torch.isfinite(res["d_raw"]).all() and (res["d_raw"][0, 0, 3:7].abs() < 1e3).all()


def _old_golden_bar(key, err):
    """The golden test's bar (test_adapter_gpu.py::test_fused_adapter_matches_reference): max(4 own, 1e-6) and 2e-5,
    own = the reference's float32 error on the golden case."""
    own = rel_err(GOLD[f"generic_f32_{key}"], GOLD[f"generic_f64_{key}"])
    bar = min(max(4 * own, 1e-6), 2e-5)
    return err < bar, bar


def test_planted_errors_pass_the_max_norm_bars_and_fail_the_per_entry_ones():
    OLD_SWEEP = dict(means=5e-6, covariances=5e-6, harmonics=5e-6, scales=5e-6, rotations=5e-6, d_raw=2e-5,
                     d_depths=2e-5, d_coordinates=2e-5)
    golden_key = dict(means="means", covariances="covariances", harmonics="harmonics", scales="scales",
                      rotations="rotations", d_raw="d_raw", d_depths="d_depths", d_coordinates="d_coordinates")
    args, cot = _abi(gu.adapter_case(case="generic"))
    ref_g = af.forward_backward(*args, cot)
    args, cot = _abi(gu.adapter_case(b=1, v=3, r=161, srf=1, spp=3, case="diverging"))
    ref_s = af.forward_backward(*args, cot)
    af.check(ref_g, ref_g, "clean")
    af.check(ref_s, ref_s, "clean")

    def plant(ref, edit):
        got = {k: ref[k].clone() for k in af.OUTPUTS + af.GRADIENTS}
        edit(got)
        return got

    def deg4_draw(g):
        for c in range(3):
            g["d_raw"][..., 7 + 25 * c + 16:7 + 25 * c + 25] *= 1.01

    def deg4_harm(g):
        g["harmonics"][:, 128:161, ..., 16:25] *= 1.005

    depth = args[5]
    near = depth <= torch.quantile(depth.flatten(), 0.05)

    def near_cov(g):
        g["covariances"][near] *= 1.01

    def swap(g):
        for k in af.OUTPUTS:
            g[k][:, [130, 131]] = g[k][:, [131, 130]]

    # no per-entry bar is looser than the max-norm bar it replaces, on either case
    for ref in (ref_g, ref_s):
        looser = {k: float((af.allowed(k, ref["scale"][k]) / (OLD_SWEEP[k] * ref[k].abs().max())).max())
                  for k in af.OUTPUTS + af.GRADIENTS}
        print("NEW_OVER_OLD_BAR", {k: f"{v:.3f}" for k, v in looser.items()})
        assert max(looser.values()) <= 1.0, looser
    planted = [("(1) d_raw degree 4 x 1.01", ref_g, deg4_draw, "d_raw", "d_raw_sh", True),
               ("(2) harmonics degree 4, second block x 1.005", ref_s, deg4_harm, "harmonics", "harmonics", True),
               ("(3) covariances of the nearest 5 % x 1.01", ref_s, near_cov, "covariances", "covariances", False),
               ("(4) rays 130 and 131 swapped", ref_s, swap, "means", "means", False)]
    for name, ref, edit, key, bar, old_must_pass in planted:
        got = plant(ref, edit)
        err = rel_err(got[key].numpy(), ref[key].numpy())
        ok_golden, golden_bar = _old_golden_bar(golden_key[key], err)
        ok_sweep = err < OLD_SWEEP[key]
        rep = af.ratios(got, ref)
        worst = max(rep.items(), key=lambda kv: kv[1][0])
        print(f"PLANTED {name}: max-norm {key} error {err:.2e}; golden bar {golden_bar:.2e} "
              f"{'accepts' if ok_golden else 'rejects'}, sweep bar {OLD_SWEEP[key]:.0e} "
              f"{'accepts' if ok_sweep else 'rejects'}; per-entry bars reject: {worst[0]} at {worst[1][1]} "
              f"{worst[1][0]:.3g}x its bar")
        if old_must_pass:
            assert ok_sweep, (name, err)
            if key == "d_raw":
                assert ok_golden, (name, err, golden_bar)
        assert rep[bar][0] > 10.0, (name, rep[bar])
        with pytest.raises(AssertionError, match="its bar"):
            af.check(got, ref, name)
