"""PLY import without a GPU: the header parser (accepted layouts and every refusal), the body size checks, the
float64 restatement of the unpack against a direct reading of hand-built files, the inverse SH blocks, the frame
file, the ABI's descriptor layout and refusals, the spin trajectory against the reference's generate_spin and the
command line."""
import ctypes
import json
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from pixelsplat_b200 import _lib, ply_export as pe, ply_import as pi, video
from tests import golden_util as gu
from tests import ply_import_f64 as f64

ROOT = Path(__file__).resolve().parents[1]
SPIN = np.load(ROOT / "tests" / "golden" / "spin_trajectory_v1.npz")


def records(names, n=5, seed=0):
    return np.random.default_rng(seed).standard_normal((n, len(names))).astype(np.float32)


def body_of(path):
    """(layout, records) as the importer's parser reads them; the body is copied by numpy here, since the importer's
    pinned buffer needs a CUDA driver."""
    data = Path(path).read_bytes()
    layout = pi.parse_header(data)
    return layout, np.frombuffer(data[layout.body_offset:], "<f4").reshape(layout.count, -1)


# ---- header


@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_parser_accepts_every_degree_shuffled_with_extra_properties(degree, tmp_path):
    names = f64.gs_properties(degree) + ["extra_a", "semantic_id"]
    order = np.random.default_rng(degree).permutation(len(names))
    names = [names[i] for i in order]
    rec = records(names, 7, degree)
    path = f64.write_ply(tmp_path / "x.ply", names, rec, extra_header="comment written by a test\n")
    layout, body = body_of(path)
    assert (layout.count, layout.properties, layout.sh_degree) == (7, tuple(names), degree)
    assert np.array_equal(body, rec)


def test_parser_accepts_the_exporters_header():
    for d in range(4):
        names = pe.ply_properties(d)
        layout = pi.parse_header(pe.ply_header(names, 3))
        assert layout.sh_degree == d and layout.properties == tuple(names)


def _header(fmt="binary_little_endian", elements=None, names=None, count=4):
    names = f64.gs_properties(1) if names is None else names
    elements = elements if elements is not None else \
        f"element vertex {count}\n" + "".join(f"property float {n}\n" for n in names)
    return f"ply\nformat {fmt} 1.0\n{elements}end_header\n".encode("ascii")


@pytest.mark.parametrize("header, match", [
    (_header(fmt="ascii"), "format 'ascii 1.0' is not supported"),
    (_header(fmt="binary_big_endian"), "format 'binary_big_endian 1.0' is not supported"),
    (_header(elements="element vertex 4\n" + "".join(f"property float {n}\n" for n in f64.gs_properties(0))
             + "element face 2\nproperty list uchar int vertex_indices\n"), "only float properties"),
    (_header(elements="element vertex 4\n" + "".join(f"property float {n}\n" for n in f64.gs_properties(0))
             + "element face 2\n"), r"elements \['vertex', 'face'\]"),
    (_header(elements="element point 4\n" + "".join(f"property float {n}\n" for n in f64.gs_properties(0))),
     r"elements \['point'\]"),
    (_header(names=f64.gs_properties(0)).replace(b"property float z", b"property double z"),
     "property 'z' of element 'vertex' is 'double'"),
    (_header(names=[n for n in f64.gs_properties(0) if n != "rot_3"]), r"missing required properties \['rot_3'\]"),
    (_header(names=f64.gs_properties(0) + [f"f_rest_{i}" for i in range(10)]), "10 f_rest properties"),
    (_header(names=f64.gs_properties(0) + [f"f_rest_{i}" for i in range(1, 10)]), "no f_rest_0"),
    (_header(count=0), "count of 0"),
    (b"plx\n", "not a PLY file"),
    (_header()[:-11], "no 'end_header'"),
])
def test_parser_rejects_malformed_headers(header, match):
    with pytest.raises(pi.PlyFormatError, match=match):
        pi.parse_header(header)


@pytest.mark.parametrize("delta", [-4, -1, 1, 4])
def test_body_of_the_wrong_length_is_rejected(delta, tmp_path):
    names = f64.gs_properties(2)
    path = f64.write_ply(tmp_path / "x.ply", names, records(names, 9))
    data = path.read_bytes()
    path.write_bytes(data[:delta] if delta < 0 else data + b"\0" * delta)
    with pytest.raises(pi.PlyFormatError, match=f"holds {9 * len(names) * 4 + delta} bytes; 9 vertices of "
                                                f"{len(names)} floats need {9 * len(names) * 4}"):
        pi.read_ply_body(path, "cuda:0")


# ---- the float64 restatement against a direct reading


def _direct(means, quats_wxyz, log_scales, logits, sh, rotation=None, center=None, scale=1.0):
    """What a file of these values means, built from scipy and numpy independently of the restatement."""
    m = np.eye(3) if rotation is None else rotation
    c = np.zeros(3) if center is None else center
    rot = Rotation.from_quat(quats_wxyz[:, [1, 2, 3, 0]]).as_matrix()
    cov_file = rot @ np.apply_along_axis(np.diag, 1, np.exp(log_scales) ** 2) @ np.swapaxes(rot, 1, 2)
    return dict(means=means @ m * scale + c, covariances=scale ** 2 * np.swapaxes(m, 0, 1) @ cov_file @ m,
                opacities=1 / (1 + np.exp(-logits)), harmonics=sh)


@pytest.mark.parametrize("with_frame", [False, True])
@pytest.mark.parametrize("degree", [0, 3])
def test_restatement_matches_a_direct_reading(with_frame, degree, tmp_path):
    g = np.random.default_rng(7 + degree)
    n, nc = 33, (degree + 1) ** 2
    means = g.standard_normal((n, 3)).astype(np.float32).astype(np.float64)
    quats = g.standard_normal((n, 4)).astype(np.float32).astype(np.float64)
    log_scales = (g.standard_normal((n, 3)) - 3).astype(np.float32).astype(np.float64)
    logits = (3 * g.standard_normal(n)).astype(np.float32).astype(np.float64)
    sh = g.standard_normal((n, 3, nc)).astype(np.float32).astype(np.float64)
    names = f64.gs_properties(degree)[::-1]
    rec = np.zeros((n, len(names)))
    col = {k: i for i, k in enumerate(names)}
    for i, k in enumerate("xyz"):
        rec[:, col[k]] = means[:, i]
    for i in range(4):
        rec[:, col[f"rot_{i}"]] = quats[:, i]
    for i in range(3):
        rec[:, col[f"scale_{i}"]] = log_scales[:, i]
        rec[:, col[f"f_dc_{i}"]] = sh[:, i, 0]
        for k in range(1, nc):
            rec[:, col[f"f_rest_{i * (nc - 1) + k - 1}"]] = sh[:, i, k]
    rec[:, col["opacity"]] = logits
    path = f64.write_ply(tmp_path / "h.ply", names, rec.astype(np.float32))
    layout, body = body_of(path)
    frame = {}
    if with_frame:
        frame = dict(rotation=pe.viewer_frame(torch.eye(4, dtype=torch.float64)).numpy()
                     @ gu.rotation(0.2, 0.4, -0.9).numpy(), center=np.array([0.5, -2.0, 3.0]), scale=1.75)
    identity = [np.eye(2 * l + 1) for l in range(degree + 1)]
    got = f64.unpack_f64(body, list(layout.properties), layout.sh_degree, nc + 2, identity, **frame)
    want = _direct(means, quats, log_scales, logits, sh, **frame)
    for k in ("means", "covariances", "opacities"):
        assert np.allclose(got[k][0], want[k], rtol=1e-12, atol=1e-15 * np.abs(want[k]).max()), k
    assert np.array_equal(got["harmonics"][0][..., :nc], sh) and not got["harmonics"][0][..., nc:].any()


def test_restatement_zero_quaternion_is_the_identity():
    names = f64.gs_properties(0)
    rec = np.zeros((2, len(names)), dtype=np.float32)
    rec[:, names.index("scale_0")], rec[:, names.index("scale_1")], rec[:, names.index("scale_2")] = 0.0, -1.0, 1.0
    rec[1, names.index("rot_0"):names.index("rot_0") + 4] = [1e-30, 0, 0, 0]
    cov, _ = f64.unpack_f64(rec, names, 0, 1, [np.eye(1)])["covariances"]
    assert np.allclose(cov, np.diag(np.exp(2 * np.array([0.0, -1.0, 1.0])))[None], rtol=1e-15, atol=0)


# ---- SH blocks and the frame file


@pytest.mark.parametrize("basis", ["3dgs", "e3nn"])
@pytest.mark.parametrize("degree", [0, 1, 2, 3])
@pytest.mark.parametrize("with_frame", [False, True])
def test_inverse_sh_blocks_undo_the_exporters_matrix(basis, degree, with_frame):
    e = torch.eye(4, dtype=torch.float64)
    e[:3, :3] = gu.rotation(0.3, -0.5, 1.1)
    m = pe.viewer_frame(e) if with_frame else None
    forward = pe.sh_transform(torch.eye(3, dtype=torch.float64) if m is None else m, degree, basis)
    for l, inv in enumerate(pi.import_sh_blocks(m, degree, basis)):
        s = slice(l * l, (l + 1) ** 2)
        assert inv.dtype == torch.float64
        assert float((inv @ forward[s, s] - torch.eye(2 * l + 1, dtype=torch.float64)).abs().max()) <= 1e-12


def test_frame_json_holds_the_float32_values_exactly(tmp_path):
    means = torch.from_numpy(np.random.default_rng(3).standard_normal((101, 3)).astype(np.float32)) * 3
    e = torch.eye(4)
    e[:3, :3] = gu.rotation(0.3, -0.5, 1.1).float()
    frame = pe.export_frame(means, e)
    pe.write_frame_json(frame, tmp_path / "s.frame.json")
    back = pi.read_frame_json(tmp_path / "s.frame.json", "cpu")
    assert torch.equal(back.center, frame.center) and torch.equal(back.scale, frame.scale)
    assert torch.equal(back.rotation, frame.rotation) and back.rotation.dtype == torch.float64
    assert set(json.loads((tmp_path / "s.frame.json").read_text())) == {"center", "scale", "rotation"}
    # a degenerate scene (every mean equal) gets s = 1, as pack_viewer uses
    assert float(pe.export_frame(torch.ones(5, 3), e).scale[0]) == 1.0


# ---- ABI


def test_import_desc_layout_matches_the_header(tmp_path):
    src = tmp_path / "probe.c"
    fields = ("col_xyz", "col_rest", "col_rot", "frame", "center", "scale", "sh_transform", "records", "opacities")
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "pixelsplat_b200.h"\n'
                   'int main(void){printf("%zu' + " %zu" * len(fields) + '\\n", sizeof(ps_ply_import_desc)'
                   + "".join(f", offsetof(ps_ply_import_desc, {f})" for f in fields) + ');return 0;}\n')
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    d = _lib.PlyImportDesc
    assert got == [ctypes.sizeof(d)] + [getattr(d, f).offset for f in fields]


def test_unpack_refuses_bad_descriptors_before_launching():
    def desc(**kw):
        d = _lib.PlyImportDesc(sh_degree=3, sh_coeffs=16, n_props=62, n_gaussians=10)
        names = f64.gs_properties(3)
        d.col_xyz[:] = [0, 1, 2]
        d.col_dc[:] = [6, 7, 8]
        d.col_rest[:] = list(range(9, 54))
        d.col_opacity = 54
        d.col_scale[:] = [55, 56, 57]
        d.col_rot[:] = [58, 59, 60, 61]
        assert len(names) == 62
        for k in ("records", "means", "covariances", "harmonics", "opacities"):
            setattr(d, k, 256)
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    def refused(d):
        rc = _lib.lib.ps_ply_unpack(ctypes.byref(d) if d is not None else None, None)
        assert rc == 1, rc
        return _lib.lib.ps_last_error().decode()
    assert "desc is NULL" in refused(None)
    assert "n_gaussians 0 < 1" in refused(desc(n_gaussians=0))
    assert "sh_degree 4 outside [0, 3]" in refused(desc(sh_degree=4))
    assert "sh_coeffs 9 outside [(sh_degree + 1)^2 = 16, 25]" in refused(desc(sh_coeffs=9))
    assert "sh_coeffs 26 outside" in refused(desc(sh_coeffs=26))
    assert "n_props 513 outside [1, 512]" in refused(desc(n_props=513))
    assert "col_rest[44] = 62 outside [0, n_props = 62)" in refused(desc(col_rest=(ctypes.c_int32 * 45)(*range(18, 63))))
    assert "col_opacity[0] = -1" in refused(desc(col_opacity=-1))
    assert "harmonics is NULL" in refused(desc(harmonics=None))
    assert "records is not 16-byte aligned" in refused(desc(records=260))
    # a degree-0 file reads no f_rest column, whatever col_rest holds
    assert "col_rest" not in refused(desc(sh_degree=0, sh_coeffs=1, n_gaussians=0,
                                          col_rest=(ctypes.c_int32 * 45)(*([-1] * 45))))


def test_records_are_checked_on_the_host():
    names = f64.gs_properties(0)
    with pytest.raises(ValueError, match="`records` must be a CUDA float32"):
        pi.unpack_records(torch.zeros(3, len(names)), names, 0)


# ---- spin


@pytest.mark.parametrize("case", sorted({k.split("/")[0] for k in SPIN.files}))
def test_generate_spin_is_the_references(case):
    got = video.generate_spin(int(SPIN[f"{case}/num_frames"]), "cpu", float(SPIN[f"{case}/elevation"]),
                              float(SPIN[f"{case}/radius"]))
    assert got.dtype == torch.float32 and np.array_equal(got.numpy(), SPIN[f"{case}/extrinsics"])


@pytest.mark.parametrize("elevation", [-60.0, 0.0, 20.0, 85.0])
def test_spin_orbits_plus_z_looking_at_the_origin(elevation):
    ext, k, near, far = video.spin_trajectory(48, 2.5, elevation)
    assert ext.shape == (48, 4, 4) and k.shape == (48, 3, 3) and near.shape == far.shape == (48,)
    e = ext.double()
    up = -e[:, :3, 1]
    assert (up[:, 2] > 0).all()
    origin, look = e[:, :3, 3], e[:, :3, 2]
    assert torch.allclose(origin.norm(dim=-1), torch.full((48,), 2.5, dtype=torch.float64), atol=1e-6)
    assert torch.allclose(origin + 2.5 * look, torch.zeros(48, 3, dtype=torch.float64), atol=1e-5)
    # the orbit's height is the elevation: sin(elevation) of the radius, the same for every frame
    assert torch.allclose(origin[:, 2], torch.full((48,), 2.5 * np.sin(np.deg2rad(elevation)), dtype=torch.float64),
                          atol=1e-5)
    assert torch.equal(k[0], torch.tensor([[0.5, 0, 0.5], [0, 0.5, 0.5], [0, 0, 1.0]]))
    assert float(near[0]) == pytest.approx(0.025) and float(far[0]) == 5.0


# ---- command line


def test_command_line_parses():
    from pixelsplat_b200.evaluation import __main__ as cli
    a = cli.parse_render_ply(["--ply", "p", "--output", "o", "--dataset-root", "d", "--index", "i"])
    assert (a.ply, a.spin, a.dataset_root) == (Path("p"), None, Path("d"))
    a = cli.parse_render_ply(["--ply", "p.ply", "--output", "o.mp4", "--spin", "30", "--radius", "3",
                              "--elevation", "-10", "--resolution", "128", "96"])
    assert (a.spin, a.radius, a.elevation, a.resolution) == (30, 3.0, -10.0, [128, 96])
    for bad in (["--ply", "p", "--output", "o"], ["--ply", "p", "--output", "o", "--spin", "0"],
                ["--ply", "p", "--output", "o", "--spin", "5", "--radius", "-1"]):
        with pytest.raises(SystemExit):
            cli.parse_render_ply(bad)
    base = ["--dataset-root", "d", "--index", "i", "--checkpoint", "c.ckpt", "--output", "o"]
    assert cli.parse_export_ply(base).write_frame is False
    assert cli.parse_export_ply(base + ["--write-frame"]).write_frame is True
    with pytest.raises(SystemExit):
        cli.parse_export_ply(base + ["--write-frame", "--format", "reference"])
