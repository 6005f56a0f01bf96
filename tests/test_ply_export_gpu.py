"""PLY export on the GPU (csrc/ply_export.cu behind pixelsplat_b200.ply_export):
  1. the reference format against the reference's own export_ply (tests/golden/ply_export_v1.npz);
  2. the viewer format round trip: the file read back and rendered by the float64 oracle from the camera moved into
     the export frame equals the original render (band 4 zeroed) on every settled pixel;
  3. the covariance factorisation of the viewer format on crafted covariances and on encoder output;
  4. the command line on re10k_tiny."""
import math

import numpy as np
import pytest
import torch

from oracle import raster_oracle as ro
from oracle import raster_torch as rt
from pixelsplat_b200 import ply_export as pe
from pixelsplat_b200 import rasterizer, synthetic
from pixelsplat_b200.decoder import Gaussians
from tests import dataset_golden as dg
from tests import golden_util as gu
from tests import ply_util
from tests import util

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = np.load(dg.GOLDEN / "ply_export_v1.npz")


def frame(e: torch.Tensor) -> torch.Tensor:
    """M from its definition, float64."""
    c, s = math.cos(-math.pi / 4), math.sin(-math.pi / 4)
    rz = torch.tensor([[c, -s, 0], [s, c, 0], [0, 0, 1]], dtype=torch.float64)
    up = torch.tensor([[0, 0, 1], [-1, 0, 0], [0, -1, 0]], dtype=torch.float64)
    return rz @ up @ torch.linalg.inv(e.double().cpu()[:3, :3])


def centre_and_scale(means: torch.Tensor) -> tuple[torch.Tensor, float]:
    m = means.to(DEV)
    center = m.median(dim=0).values
    return center.double().cpu(), float((m - center).abs().quantile(0.95, dim=0).max())


def quat_to_matrix(q: np.ndarray) -> np.ndarray:
    """wxyz (normalised here) -> [n, 3, 3], as 3DGS's build_rotation."""
    q = q.astype(np.float64)
    w, x, y, z = (q / np.linalg.norm(q, axis=-1, keepdims=True)).T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def read_viewer(path, degree=3):
    """The file as a 3DGS viewer loads it: positions, harmonics [n, 3, (d+1)^2], sigmoid opacity, covariance
    R diag(exp(scale))^2 R^T, all float64."""
    names, rec = ply_util.read_ply(path)
    assert names == pe.ply_properties(degree)
    rec = rec.astype(np.float64)
    k = (degree + 1) ** 2 - 1
    col = {n: i for i, n in enumerate(names)}
    rest = rec[:, 9:9 + 3 * k].reshape(-1, 3, k)
    harmonics = np.concatenate([rec[:, 6:9, None], rest], axis=-1)
    opacity = 1 / (1 + np.exp(-rec[:, col["opacity"]]))
    scale = np.exp(rec[:, col["scale_0"]:col["scale_0"] + 3])
    r = quat_to_matrix(rec[:, col["rot_0"]:col["rot_0"] + 4])
    cov = r @ (scale[:, :, None] ** 2 * np.swapaxes(r, -1, -2))
    return dict(means=rec[:, :3], harmonics=harmonics, opacities=opacity, covariances=cov, scale=scale, rot=r,
                records=rec)


def render64(means, cov, harmonics, opac, ext, k, near, far, hw):
    a = rt.prepare_view(torch.as_tensor(means), torch.as_tensor(cov), torch.as_tensor(harmonics),
                        torch.as_tensor(opac), torch.as_tensor(ext), torch.as_tensor(k), near, far,
                        dtype=torch.float64)
    return a, util.oracle_forward64(a, (0.0, 0.0, 0.0), hw[1], hw[0])


def round_trip(tmp_path, g: Gaussians, context_ext, ext, k, near, far, hw, tag, sh_degree=3, basis="3dgs"):
    """Exports `g` (CPU float32, one scene), reads the file back and renders it from the camera (ext, k, near, far)
    moved into the export frame; the original is rendered with its harmonics truncated to the exported degree."""
    path = tmp_path / f"{tag}.ply"
    old = rasterizer.get_sh_basis()
    rasterizer.set_sh_basis(basis)
    try:
        pe.export_gaussians_ply(Gaussians(*(t[None].to(DEV) for t in (g.means, g.covariances, g.harmonics,
                                                                       g.opacities))),
                                context_ext.to(DEV), path, sh_degree=sh_degree)
    finally:
        rasterizer.set_sh_basis(old)
    d = min(sh_degree, 3, math.isqrt(g.harmonics.shape[-1]) - 1)
    back = read_viewer(path, d)
    m = frame(context_ext)
    center, s = centre_and_scale(g.means)
    want_pos = ((g.means.double() - center) / s) @ m.T
    assert float((torch.from_numpy(back["means"]) - want_pos).abs().max()) <= 2e-6 * max(1.0, float(want_pos.abs().max()))

    n = (d + 1) ** 2
    with ro.sh_basis(0 if basis == "3dgs" else 1):
        a, orig = render64(g.means.double(), g.covariances.double(), g.harmonics.double()[..., :n], g.opacities.double(),
                           ext.double(), k.double(), float(near), float(far), hw)
        settled = util.SettledRef(a, (0.0, 0.0, 0.0), hw[0], hw[1]).settled
    e2 = torch.eye(4, dtype=torch.float64)
    e2[:3, :3] = m @ ext.double()[:3, :3]
    e2[:3, 3] = m @ ((ext.double()[:3, 3] - center) / s)
    _, got = render64(back["means"], back["covariances"], back["harmonics"], back["opacities"], e2, k.double(),
                      float(near) / s, float(far) / s, hw)
    diff = np.abs(got.color - orig.color).max(0)
    print(f"ROUND_TRIP {tag}: settled max diff {float(diff[settled].max()):.2e}, unsettled {int((~settled).sum())} "
          f"of {settled.size} (max diff there {float(diff[~settled].max()) if (~settled).any() else 0.0:.2e}), "
          f"covered {int((orig.final_T < 0.99).sum())}")
    assert (orig.final_T < 0.99).sum() > settled.size // 4, "the view sees too little of the scene"
    assert float(diff[settled].max()) <= 1e-4, tag
    return back


# ---- 1. reference format


@pytest.mark.parametrize("case", [c[0] for c in ply_util.PLY_CASES])
def test_reference_format_matches_the_reference(case, tmp_path):
    c = {k: v.to(DEV) for k, v in ply_util.ply_case(case).items()}
    want = GOLDEN[case]
    rec, names = pe.pack_reference(c["extrinsics"], c["means"], c["scales"], c["rotations"], c["harmonics"],
                                   c["opacities"])
    got = rec.cpu().numpy()
    assert names == list(GOLDEN["names"]) and got.shape == want.shape
    assert np.abs(got[:, :3] - want[:, :3]).max() <= 2e-6
    assert np.array_equal(got[:, 3:6], want[:, 3:6]) and np.array_equal(got[:, 6:10], want[:, 6:10])   # n, DC, opacity
    assert np.abs(got[:, 10:13] - want[:, 10:13]).max() <= 2e-6
    q, qw = got[:, 13:17], want[:, 13:17]
    assert np.minimum(np.abs(q - qw).max(-1), np.abs(q + qw).max(-1)).max() <= 2e-6
    # the file holds exactly these records
    pe.export_ply(c["extrinsics"], c["means"], c["scales"], c["rotations"], c["harmonics"], c["opacities"],
                  tmp_path / "sub" / f"{case}.ply")
    file_names, file_rec = ply_util.read_ply(tmp_path / "sub" / f"{case}.ply")
    assert file_names == names and np.array_equal(file_rec, got)


def test_inputs_are_checked():
    c = {k: v.to(DEV) for k, v in ply_util.ply_case("identity_tail").items()}
    args = [c["extrinsics"], c["means"], c["scales"], c["rotations"], c["harmonics"], c["opacities"], "x.ply"]
    for i, name, bad in ((1, "means", c["means"][:0]), (2, "scales", c["scales"][:-1]),
                         (3, "rotations", c["rotations"][:, :3]), (4, "harmonics", c["harmonics"][..., :24]),
                         (5, "opacities", c["opacities"].double()), (0, "extrinsics", c["extrinsics"][:3])):
        with pytest.raises(ValueError, match=f"`{name}`"):
            pe.export_ply(*args[:i], bad, *args[i + 1:])
    g = Gaussians(c["means"], torch.eye(3, device=DEV).expand(129, 3, 3), c["harmonics"], c["opacities"])
    with pytest.raises(ValueError, match="`gaussians.covariances`"):
        pe.export_gaussians_ply(Gaussians(g.means, g.covariances[:, :2], g.harmonics, g.opacities), c["extrinsics"],
                                "x.ply")
    with pytest.raises(ValueError, match="`sh_degree`"):
        pe.export_gaussians_ply(g, c["extrinsics"], "x.ply", sh_degree=-1)


# ---- 2. viewer format round trip


def _context_extrinsics():
    e = torch.eye(4, dtype=torch.float64)
    e[:3, :3] = gu.rotation(0.3, -0.5, 1.1)
    e[:3, 3] = torch.tensor([0.4, -1.2, 2.5], dtype=torch.float64)
    return e.float()


@pytest.mark.parametrize("sh_degree", [3, 4])
def test_round_trip_synthetic(sh_degree, tmp_path):
    sc = synthetic.scene_random_frustum(seed=3, num_gaussians=1000, sh_degree=sh_degree)
    g = Gaussians(sc.means, sc.covariances, sc.harmonics, sc.opacities)
    round_trip(tmp_path, g, _context_extrinsics(), sc.extrinsics[0], sc.intrinsics[0], sc.near[0], sc.far[0],
               sc.image_shape, f"synthetic_deg{sh_degree}", sh_degree=4)


def test_round_trip_e3nn_basis(tmp_path):
    sc = synthetic.scene_random_frustum(seed=4, num_gaussians=1000, sh_degree=3)
    g = Gaussians(sc.means, sc.covariances, sc.harmonics, sc.opacities)
    round_trip(tmp_path, g, _context_extrinsics(), sc.extrinsics[0], sc.intrinsics[0], sc.near[0], sc.far[0],
               sc.image_shape, "synthetic_e3nn", basis="e3nn")


def _encoder_scene():
    """The re10k preset's encoder with seeded random weights on two 64 x 64 views."""
    from pixelsplat_b200.evaluation import presets as ev
    encoder, _ = ev.build_model("re10k", ev.dataset_cfg("/data", "/index.json"))
    torch.manual_seed(0)
    encoder = encoder.to(DEV).eval()
    ext, k, near, far = [t.to(DEV, torch.float32) for t in gu.camera_rig(1, 2, "generic")]
    image = torch.rand(1, 2, 3, 64, 64, generator=torch.Generator().manual_seed(1)).to(DEV)
    dump = {}
    with torch.no_grad():
        g = encoder(dict(image=image, extrinsics=ext, intrinsics=k, near=near, far=far), 0, visualization_dump=dump)
    return g, dump, ext[0], k[0], near[0], far[0]


def test_round_trip_encoder(tmp_path):
    g, dump, ext, k, near, far = _encoder_scene()
    one = Gaussians(*(t[0].cpu() for t in (g.means, g.covariances, g.harmonics, g.opacities)))
    back = round_trip(tmp_path, one, ext[0].cpu(), ext[1].cpu(), k[1].cpu(), near[1].cpu(), far[1].cpu(), (64, 64),
                      "encoder")
    # the exported scales are the adapter's scales / s, up to the float32 rounding of the covariance it formed
    _, s = centre_and_scale(one.means)
    want = np.sort(dump["scales"][0].double().cpu().numpy() / s, axis=-1)
    got = np.sort(back["scale"], axis=-1)
    bar = 1e-5 + 4 * np.finfo(np.float32).eps * (want[:, 2:] / want) ** 2
    ratio = np.abs(got / want - 1) / bar
    print(f"ENCODER_SCALES worst ratio {float(ratio.max()):.3f}, anisotropy up to {float((want[:, 2] / want[:, 0]).max()):.1f}")
    assert float(ratio.max()) <= 1.0


# ---- 3. covariance factorisation


def crafted_covariances() -> dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(5)
    n = 300
    q = torch.randn(n, 4, generator=g, dtype=torch.float64)
    r = synthetic._quat_to_rot(q / q.norm(dim=-1, keepdim=True))

    def rotated(lam):
        return r @ torch.diag_embed(lam) @ r.transpose(-1, -2)

    base = torch.rand(n, 1, generator=g, dtype=torch.float64) * 0.1 + 0.01
    aniso = 10 ** (3 * torch.rand(n, 3, generator=g, dtype=torch.float64))      # scale ratios up to 1e3
    return {"isotropic": rotated(base.expand(n, 3).square()),
            "two_equal": rotated(torch.cat([base, base, 3 * base], -1).square()),
            "axis_aligned": torch.diag_embed((base * torch.rand(n, 3, generator=g, dtype=torch.float64) + 1e-3).square()),
            "anisotropic": rotated((base * aniso / 1e3).square()),
            "near_zero_axis": rotated(torch.cat([base, 0.5 * base, 1e-7 * base], -1).square())}


@pytest.mark.parametrize("family", list(crafted_covariances()))
def test_covariance_factorisation(family, tmp_path):
    cov = crafted_covariances()[family].float()
    n = cov.shape[0]
    means = gu.seeded_like("ply.factor.means", (n, 3), 1.0).float()
    harmonics = gu.seeded_like("ply.factor.harmonics", (n, 3, 16), 1.0).float()
    g = Gaussians(means[None].to(DEV), cov[None].to(DEV), harmonics[None].to(DEV), torch.full((1, n), 0.5, device=DEV))
    e = _context_extrinsics()
    pe.export_gaussians_ply(g, e.to(DEV), tmp_path / "f.ply")
    back = read_viewer(tmp_path / "f.ply")
    m = frame(e).numpy()
    _, s = centre_and_scale(means)
    want = m @ cov.double().numpy() @ m.T / (s * s)
    err = np.linalg.norm(back["covariances"] - want, axis=(1, 2)) / np.linalg.norm(want, axis=(1, 2))
    print(f"FACTOR {family}: worst relative Frobenius error {float(err.max()):.2e}")
    assert float(err.max()) <= 1e-5
    assert np.allclose(np.linalg.det(back["rot"]), 1.0, atol=1e-6)
    assert (back["records"][:, pe.ply_properties(3).index("rot_0")] >= 0).all()


# ---- 4. command line


def test_command_line_on_re10k_tiny(tmp_path):
    from pixelsplat_b200.evaluation import __main__ as cli
    from pixelsplat_b200.evaluation import presets as ev
    from pixelsplat_b200.evaluation.checkpoint import save_checkpoint
    encoder, _ = ev.build_model("re10k", ev.dataset_cfg(dg.DATA, dg.DATA / "evaluation_index.json"))
    ckpt = save_checkpoint(tmp_path / "random.ckpt", encoder, 0)
    base = ["export-ply", "--dataset-root", str(dg.DATA), "--index", str(dg.DATA / "evaluation_index.json"),
            "--checkpoint", str(ckpt), "--preset", "re10k", "--num-workers", "0"]
    scenes = [w["scene"] for w in dg.expected("test")]
    written = cli.export_ply(base[1:] + ["--output", str(tmp_path / "viewer")])
    assert sorted(p.name for p in (tmp_path / "viewer").iterdir()) == sorted(f"{s}.ply" for s in scenes)
    assert [p.stem for p in written] == scenes
    count = 2 * 256 * 256 * 3                     # views x h x w x gaussians_per_pixel
    for p in written:
        names, rec = ply_util.read_ply(p)
        assert names == pe.ply_properties(3) and rec.shape == (count, 62) and np.isfinite(rec).all()
    cli.main(base + ["--output", str(tmp_path / "ref"), "--format", "reference", "--scene", scenes[-1]])
    (only,) = (tmp_path / "ref").iterdir()
    names, rec = ply_util.read_ply(only)
    assert only.name == f"{scenes[-1]}.ply" and names == pe.ply_properties(None) and rec.shape == (count, 17)
    with pytest.raises(SystemExit, match="no test scene named zzz"):
        cli.main(base + ["--output", str(tmp_path / "none"), "--scene", "zzz"])
