"""PLY export without a GPU: the header and property order of both formats, the export frame M, the per-scene SH
matrix checked from its definition with sh_basis, input validation, the ABI's refusals and the command line."""
import ctypes
import math
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from pixelsplat_b200 import _lib, ply_export as pe
from pixelsplat_b200.sh import sh_basis
from tests import golden_util as gu
from tests import ply_util

ROOT = Path(__file__).resolve().parents[1]
REFERENCE_PROPERTIES = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2", "opacity", "scale_0", "scale_1",
                        "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]


def extrinsics(dtype=torch.float64) -> torch.Tensor:
    e = torch.eye(4, dtype=torch.float64)
    e[:3, :3] = gu.rotation(0.3, -0.5, 1.1)
    e[:3, 3] = torch.tensor([0.4, -1.2, 2.5], dtype=torch.float64)
    return e.to(dtype)


def frame_from_definition(e: torch.Tensor) -> torch.Tensor:
    c, s = math.cos(-math.pi / 4), math.sin(-math.pi / 4)
    rz = torch.tensor([[c, -s, 0], [s, c, 0], [0, 0, 1]], dtype=torch.float64)
    up = torch.tensor([[0, 0, 1], [-1, 0, 0], [0, -1, 0]], dtype=torch.float64)
    return rz @ up @ torch.linalg.inv(e.double()[:3, :3])


@pytest.mark.parametrize("degree", [None, 0, 1, 2, 3, 4])
def test_properties_and_header(degree):
    names = pe.ply_properties(degree)
    rest = 0 if degree is None else 3 * ((min(degree, 3) + 1) ** 2 - 1)
    assert names == REFERENCE_PROPERTIES[:9] + [f"f_rest_{i}" for i in range(rest)] + REFERENCE_PROPERTIES[9:]
    header = pe.ply_header(names, 12345).decode("ascii")
    assert header == ("ply\nformat binary_little_endian 1.0\nelement vertex 12345\n"
                      + "".join(f"property float {n}\n" for n in names) + "end_header\n")


def test_fixture_has_the_reference_properties():
    g = np.load(ROOT / "tests" / "golden" / "ply_export_v1.npz")
    assert list(g["names"]) == pe.ply_properties(None) == REFERENCE_PROPERTIES
    for name, _, n in ply_util.PLY_CASES:
        assert g[name].shape == (n, 17) and g[name].dtype == np.float32


def test_reader_round_trips_a_written_header(tmp_path):
    names = pe.ply_properties(2)
    rec = np.arange(3 * len(names), dtype=np.float32).reshape(3, len(names))
    path = tmp_path / "x.ply"
    path.write_bytes(pe.ply_header(names, 3) + rec.astype("<f4").tobytes())
    got_names, got = ply_util.read_ply(path)
    assert got_names == names and np.array_equal(got, rec)


@pytest.mark.parametrize("rotated", [False, True])
def test_export_frame(rotated):
    e = extrinsics() if rotated else torch.eye(4, dtype=torch.float64)
    m = pe.viewer_frame(e)
    assert torch.allclose(m, frame_from_definition(e), atol=1e-15, rtol=0)
    assert torch.allclose(m @ m.T, torch.eye(3, dtype=torch.float64), atol=1e-14) and abs(float(m.det()) - 1) < 1e-14
    # the camera looks along (1, -1, 0) / sqrt 2 (the viewer's 45 degree start), its up (-y in OpenCV) is +z
    r = e[:3, :3]
    h = math.sqrt(0.5)
    assert torch.allclose(m @ r @ torch.tensor([0, 0, 1.0], dtype=torch.float64),
                          torch.tensor([h, -h, 0], dtype=torch.float64), atol=1e-14)
    assert torch.allclose(m @ r @ torch.tensor([0, -1.0, 0], dtype=torch.float64),
                          torch.tensor([0, 0, 1.0], dtype=torch.float64), atol=1e-14)
    # the reference's float32 M: the same matrix, to float32 rounding
    ref = pe.reference_frame(e.float())
    assert ref.dtype == torch.float32 and torch.allclose(ref.double(), m, atol=3e-7, rtol=0)


@pytest.mark.parametrize("basis", ["3dgs", "e3nn"])
@pytest.mark.parametrize("degree", [0, 1, 2, 3])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_sh_transform_from_its_definition(basis, degree, dtype):
    """sum_i c'_i Y_3dgs,i(M d) = sum_i c_i Y_basis,i(d) for random directions d, degree by degree."""
    e = extrinsics(dtype)
    m = frame_from_definition(e)
    t = pe.sh_transform(pe.viewer_frame(e), degree, basis)
    n = (degree + 1) ** 2
    assert t.shape == (n, n) and t.dtype == torch.float64
    g = torch.Generator().manual_seed(degree)
    d = torch.randn(500, 3, generator=g, dtype=torch.float64)
    d = d / d.norm(dim=-1, keepdim=True)
    c = torch.randn(n, 7, generator=g, dtype=torch.float64)
    md = d @ m.T
    lhs = sh_basis(md / md.norm(dim=-1, keepdim=True), degree, "3dgs") @ (t @ c)
    rhs = sh_basis(d, degree, basis) @ c
    # float32 extrinsics: R_c2w^-1 is a rotation to ~1e-7 only
    tol = 1e-11 if dtype == torch.float64 else 2e-6
    assert float((lhs - rhs).abs().max()) <= tol * float(c.abs().max())
    for l in range(degree + 1):                  # block diagonal: no degree mixes with another
        s = slice(l * l, (l + 1) ** 2)
        off = t[s].clone()
        off[:, s] = 0
        assert float(off.abs().max()) < 1e-12


def test_inputs_are_checked_on_the_host():
    c = ply_util.ply_case("identity_tail")
    with pytest.raises(ValueError, match="`means` must be a CUDA tensor"):
        pe.export_ply(c["extrinsics"], c["means"], c["scales"], c["rotations"], c["harmonics"], c["opacities"],
                      "x.ply")
    with pytest.raises(ValueError, match="`means` must be a torch.Tensor"):
        pe.export_ply(c["extrinsics"], c["means"].numpy(), c["scales"], c["rotations"], c["harmonics"],
                      c["opacities"], "x.ply")
    from pixelsplat_b200.decoder import Gaussians
    g = Gaussians(c["means"], torch.eye(3).expand(129, 3, 3), c["harmonics"], c["opacities"])
    with pytest.raises(ValueError, match="`gaussians.means` must be a CUDA tensor"):
        pe.export_gaussians_ply(g, c["extrinsics"], "x.ply")
    batch = Gaussians(*(t[None].expand(2, *t.shape) for t in (g.means, g.covariances, g.harmonics, g.opacities)))
    with pytest.raises(ValueError, match="batch of 2 scenes"):
        pe.export_gaussians_ply(batch, c["extrinsics"], "x.ply")


def test_desc_layout_matches_the_header(tmp_path):
    """sizeof / offsetof of ps_ply_desc from a C probe compiled against the header, against the ctypes mirror."""
    src = tmp_path / "probe.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "pixelsplat_b200.h"\n'
                   'int main(void){printf("%zu %zu %zu %zu %zu\\n", sizeof(ps_ply_desc), offsetof(ps_ply_desc, frame),'
                   'offsetof(ps_ply_desc, sh_transform), offsetof(ps_ply_desc, means), offsetof(ps_ply_desc, scale));'
                   'return 0;}\n')
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    d = _lib.PlyDesc
    assert got == [ctypes.sizeof(d), d.frame.offset, d.sh_transform.offset, d.means.offset, d.scale.offset]


def _refused(desc, out=16) -> str:
    rc = _lib.lib.ps_ply_pack(ctypes.byref(desc) if desc is not None else None, ctypes.c_void_p(out), None)
    assert rc == 1, rc                                          # PS_ERR_INVALID_ARGUMENT, before any launch
    return _lib.lib.ps_last_error().decode()


def test_pack_refuses_bad_descriptors_before_launching():
    """Every refusal of ps_ply_pack comes before the library touches a device (the pointers are never read)."""
    def desc(**kw):
        d = _lib.PlyDesc(mode=_lib.PS_PLY_VIEWER, sh_degree=3, sh_coeffs=25, n_gaussians=10)
        for k in ("means", "covariances", "harmonics", "opacities", "center", "scale"):
            setattr(d, k, 256)
        for k, v in kw.items():
            setattr(d, k, v)
        return d
    assert "desc is NULL" in _refused(None)
    assert "out is NULL" in _refused(desc(), out=0)
    assert "unknown mode 2" in _refused(desc(mode=2))
    assert "n_gaussians 0" in _refused(desc(n_gaussians=0))
    assert "sh_degree 4 outside [0, 3]" in _refused(desc(sh_degree=4))
    assert "sh_degree 1 outside [0, 0]" in _refused(desc(mode=_lib.PS_PLY_REFERENCE, sh_degree=1))
    assert "sh_coeffs 9 < (sh_degree + 1)^2 = 16" in _refused(desc(sh_coeffs=9))
    assert "covariances is NULL" in _refused(desc(covariances=None))
    assert "scales is NULL" in _refused(desc(mode=_lib.PS_PLY_REFERENCE, sh_degree=0))
    assert "center is NULL" in _refused(desc(center=None))
    assert "not 16-byte aligned" in _refused(desc(), out=20)


def test_command_line_parses():
    from pixelsplat_b200.evaluation import __main__ as cli
    base = ["--dataset-root", "d", "--index", "i", "--checkpoint", "c.ckpt", "--output", "o"]
    a = cli.parse_export_ply(base)
    assert (a.format, a.scene, a.preset, a.output) == ("viewer", None, "re10k", Path("o"))
    a = cli.parse_export_ply(base + ["--scene", "aaa", "--scene", "bbb", "--format", "reference", "--preset", "acid"])
    assert (a.format, a.scene, a.preset) == ("reference", ["aaa", "bbb"], "acid")
    with pytest.raises(SystemExit):
        cli.parse_export_ply(base + ["--format", "splat"])
    with pytest.raises(SystemExit):
        cli.main(["export-ply", "--dataset-root", "d", "--index", "i", "--checkpoint", "c"])   # no --output
