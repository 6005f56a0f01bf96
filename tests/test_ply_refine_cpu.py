"""PLY refinement without a GPU: the float64 restatement of the step (tests/ply_refine_f64.py) against torch's own
autograd and Adam, the step's descriptor checks, the refine-ply arguments and the steps=0 copy."""
import ctypes
from pathlib import Path

import numpy as np
import pytest
import torch

from pixelsplat_b200 import _lib, ply_refine as pr
from tests import ply_import_f64 as f64
from tests import ply_refine_f64 as rf

pytestmark = pytest.mark.filterwarnings("ignore::UserWarning")


def random_case(n: int, degree: int, seed: int, normals: bool = True):
    """Records in a shuffled property order with an extra property, moderate log scales, some zero quaternions and
    random SH blocks; gradients N(0, 1) for every unpack output, with 16 coefficients per channel."""
    g = np.random.default_rng(seed)
    names = f64.gs_properties(degree, normals) + ["extra"]
    names = [names[i] for i in g.permutation(len(names))]
    rec = g.standard_normal((n, len(names)))
    col = {k: i for i, k in enumerate(names)}
    rec[:, [col[f"scale_{i}"] for i in range(3)]] = g.uniform(-2, 1, (n, 3))
    rec[::5, [col[f"rot_{i}"] for i in range(4)]] = 0.0
    blocks = [g.standard_normal((2 * l + 1, 2 * l + 1)) for l in range(degree + 1)]
    grads = {"means": g.standard_normal((n, 3)), "covariances": g.standard_normal((n, 3, 3)),
             "harmonics": g.standard_normal((n, 3, 16)), "opacities": g.standard_normal(n)}
    return rec, names, blocks, grads, col


def frame_of(seed: int):
    g = np.random.default_rng(seed)
    q, _ = np.linalg.qr(g.standard_normal((3, 3)))
    return q * np.sign(np.linalg.det(q)), g.standard_normal(3), float(10 ** g.uniform(-1, 1))


@pytest.mark.parametrize("with_frame", [False, True])
@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_backward_matches_torch_autograd(degree, with_frame):
    rec, names, blocks, grads, col = random_case(40, degree, 10 * degree + with_frame)
    rotation, center, scale = frame_of(degree) if with_frame else (None, None, 1.0)
    records = torch.from_numpy(rec).requires_grad_(True)
    out = rf.unpack_torch(rf.split(records, names, degree), degree, 16, blocks, rotation, center, scale)
    sum(torch.sum(torch.from_numpy(grads[k]) * out[k]) for k in out).backward()
    got, mag = rf.record_grad_f64(rec, names, degree, blocks, grads, rotation, center, scale)
    want = records.grad.numpy()
    assert np.all(np.abs(got - want) <= 1e-12 * (mag + 1e-300)), float(np.max(np.abs(got - want) / (mag + 1e-300)))
    assert np.all(mag >= np.abs(got))
    # the columns the unpack does not read, and the zero quaternions, get exactly 0
    unread = [col[k] for k in names if pr.group_of(k, degree) is None]
    assert unread and not got[:, unread].any() and not want[:, unread].any()
    zero = [col[f"rot_{i}"] for i in range(4)]
    assert not got[::5][:, zero].any() and not want[::5][:, zero].any()
    assert got[1::5][:, zero].any()


@pytest.mark.parametrize("degree", [0, 3])
def test_backward_passes_gradcheck(degree):
    rec, names, blocks, _, _ = random_case(6, degree, 7 + degree)
    rotation, center, scale = frame_of(3)
    records = torch.from_numpy(rec).requires_grad_(True)
    assert torch.autograd.gradcheck(
        lambda r: rf.UnpackF64.apply(r, names, degree, 16, blocks, rotation, center, scale), (records,),
        eps=1e-6, atol=1e-7, rtol=1e-5)


def test_adam_matches_torch_adam_with_a_group_per_property_group():
    degree, n, steps = 2, 30, 5
    rec, names, _, _, _ = random_case(n, degree, 3)
    cols = rf.group_columns(names, degree)
    lr = {"xyz": 1e-3, "f_dc": 2e-3, "f_rest": 3e-4, "opacity": 5e-2, "scale": 5e-3, "rot": 1e-3}
    params = {k: torch.tensor(rec[:, c], requires_grad=True) for k, c in cols.items()}
    opt = torch.optim.Adam([{"params": [params[k]], "lr": lr[k]} for k in rf.GROUPS], lr=0.0, eps=pr.EPS,
                           betas=pr.BETAS)
    col_lr = np.array(pr.column_lr(names, degree, lr))
    p, m, v = rec.copy(), np.zeros_like(rec), np.zeros_like(rec)
    g = np.random.default_rng(4)
    read = col_lr > 0
    for t in range(1, steps + 1):
        grad = g.standard_normal(rec.shape) * read
        for k, c in cols.items():
            params[k].grad = torch.from_numpy(grad[:, c].copy())
        opt.step()
        (p2, m, v), _ = rf.adam_f64(p, grad, m, v, col_lr, t, pr.BETAS, pr.EPS)
        p = np.where(read, p2, p)
    for k, c in cols.items():
        np.testing.assert_allclose(p[:, c], params[k].detach().numpy(), rtol=1e-14, atol=1e-15)
        np.testing.assert_allclose(m[:, c], opt.state[params[k]]["exp_avg"].numpy(), rtol=1e-14, atol=1e-16)
        np.testing.assert_allclose(v[:, c], opt.state[params[k]]["exp_avg_sq"].numpy(), rtol=1e-14, atol=1e-18)


def test_column_learning_rates():
    names = f64.gs_properties(1) + ["filter_3D"]
    lr = pr.column_lr(names, 1, {"f_rest": 0.5})
    by = dict(zip(names, lr))
    assert by["x"] == pr.DEFAULT_LR["xyz"] and by["f_rest_8"] == 0.5 and by["rot_3"] == pr.DEFAULT_LR["rot"]
    assert by["nx"] == 0.0 and by["filter_3D"] == 0.0
    with pytest.raises(ValueError, match="unknown learning-rate group 'xy'"):
        pr.column_lr(names, 1, {"xy": 1.0})
    with pytest.raises(ValueError, match="must be a finite number >= 0"):
        pr.column_lr(names, 1, {"rot": -1.0})


# ---- ABI


def test_refine_desc_layout_matches_the_header(tmp_path):
    import subprocess
    root = Path(__file__).resolve().parents[1]
    fields = ("step", "beta1", "eps", "lr", "records_out", "exp_avg_sq", "d_harmonics", "d_records")
    src = tmp_path / "probe.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "pixelsplat_b200.h"\n'
                   'int main(void){printf("%zu' + " %zu" * len(fields) + '\\n", sizeof(ps_ply_refine_desc)'
                   + "".join(f", offsetof(ps_ply_refine_desc, {f})" for f in fields) + ');return 0;}\n')
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", str(root / "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    d = _lib.PlyRefineDesc
    assert got == [ctypes.sizeof(d)] + [getattr(d, f).offset for f in fields]


def test_refine_step_refuses_bad_descriptors_before_launching():
    def desc(**kw):
        d = _lib.PlyRefineDesc(step=1, beta1=0.9, beta2=0.999, eps=1e-15)
        u = d.unpack
        u.sh_degree, u.sh_coeffs, u.n_props, u.n_gaussians = 3, 16, 62, 10
        u.col_xyz[:] = [0, 1, 2]
        u.col_dc[:] = [6, 7, 8]
        u.col_rest[:] = list(range(9, 54))
        u.col_opacity = 54
        u.col_scale[:] = [55, 56, 57]
        u.col_rot[:] = [58, 59, 60, 61]
        for k in ("records", "means", "covariances", "harmonics", "opacities"):
            setattr(u, k, 256)
        for k in ("records_out", "exp_avg", "exp_avg_sq", "d_means", "d_covariances", "d_harmonics", "d_opacities"):
            setattr(d, k, 512)
        d.lr[:62] = [1e-3] * 62
        for k, v in kw.items():
            if k.startswith("u_"):
                setattr(u, k[2:], v)
            else:
                setattr(d, k, v)
        return d

    def refused(d):
        rc = _lib.lib.ps_ply_refine_step(ctypes.byref(d) if d is not None else None, None)
        assert rc == 1, rc
        msg = _lib.lib.ps_last_error().decode()
        assert msg.startswith("ps_ply_refine_step: "), msg
        return msg

    assert "desc is NULL" in refused(None)
    assert "n_gaussians 0 < 1" in refused(desc(u_n_gaussians=0))
    assert "sh_degree 4 outside [0, 3]" in refused(desc(u_sh_degree=4))
    assert "sh_coeffs 9 outside" in refused(desc(u_sh_coeffs=9))
    assert "n_props 513 outside [1, 512]" in refused(desc(u_n_props=513))
    assert "n_props 300 above 256" in refused(desc(u_n_props=300))
    assert "col_rot[3] = 62 outside [0, n_props = 62)" in refused(desc(u_col_rot=(ctypes.c_int32 * 4)(58, 59, 60, 62)))
    assert "column 0 is read as two fields" in refused(desc(u_col_opacity=0))
    for name in ("records", "means", "covariances", "harmonics", "opacities"):
        assert f"{name} is NULL" in refused(desc(**{f"u_{name}": None}))
    assert "records is not 16-byte aligned" in refused(desc(u_records=260))
    for name in ("records_out", "exp_avg", "exp_avg_sq", "d_means", "d_covariances", "d_harmonics", "d_opacities"):
        assert f"{name} is NULL" in refused(desc(**{name: None}))
        assert f"{name} is not 16-byte aligned" in refused(desc(**{name: 516}))
    assert "d_records is not 16-byte aligned" in refused(desc(d_records=516))
    assert "step 0 < 1" in refused(desc(step=0))
    assert "betas 1 0.999 outside [0, 1)" in refused(desc(beta1=1.0))
    assert "betas 0.9 -0.5 outside" in refused(desc(beta2=-0.5))
    assert "eps -1 not finite" in refused(desc(eps=-1.0))
    lr = (ctypes.c_double * _lib.PLY_REFINE_MAX_PROPERTIES)(*([1e-3] * _lib.PLY_REFINE_MAX_PROPERTIES))
    lr[57] = -1.0
    assert "lr[57] = -1 is negative or not finite" in refused(desc(lr=lr))
    lr[57] = float("nan")
    assert "lr[57] = nan is negative or not finite" in refused(desc(lr=lr))


# ---- command line and file


def test_refine_ply_arguments_parse():
    from pixelsplat_b200.evaluation import __main__ as cli
    base = ["--ply", "p", "--dataset-root", "d", "--index", "i", "--output", "o"]
    a = cli.parse_refine_ply(base)
    assert (a.ply, a.dataset_root, a.index, a.output, a.scene, a.steps) == (Path("p"), Path("d"), Path("i"),
                                                                            Path("o"), None, 100)
    assert a.lr == pr.DEFAULT_LR
    a = cli.parse_refine_ply(base + ["--scene", "a", "--scene", "b", "--steps", "0", "--lr-xyz", "1e-3",
                                     "--lr-f-dc", "0.1", "--lr-f-rest", "0", "--lr-opacity", "0.2",
                                     "--lr-scale", "0.3", "--lr-rot", "0.4"])
    assert a.scene == ["a", "b"] and a.steps == 0
    assert a.lr == {"xyz": 1e-3, "f_dc": 0.1, "f_rest": 0.0, "opacity": 0.2, "scale": 0.3, "rot": 0.4}
    for bad in (["--steps", "-1"], ["--lr-xyz", "-1e-3"], ["--lr-rot", "nan"], ["--steps", "1.5"]):
        with pytest.raises(SystemExit):
            cli.parse_refine_ply(base + bad)
    with pytest.raises(SystemExit):
        cli.parse_refine_ply(["--ply", "p", "--output", "o"])


def test_refine_ply_with_no_steps_copies_the_file(tmp_path):
    names = f64.gs_properties(2) + ["filter_3D"]
    rec = np.random.default_rng(0).standard_normal((37, len(names))).astype(np.float32)
    src = f64.write_ply(tmp_path / "in.ply", names, rec, extra_header="comment made by a test\n")
    out = tmp_path / "out" / "refined.ply"
    z = torch.zeros(2, 3, 8, 8)
    got = pr.refine_ply(src, None, extrinsics=torch.eye(4)[None].expand(2, 4, 4), intrinsics=torch.eye(3)[None],
                        near=torch.ones(2), far=torch.ones(2), images=z, background_color=torch.zeros(3), steps=0,
                        out_path=out)
    assert got is None and out.read_bytes() == src.read_bytes()


def test_refine_step_needs_cuda_tensors():
    names = f64.gs_properties(0)
    rec = torch.zeros(4, len(names))
    step = pr.RefineStep(names, 0, 4)
    with pytest.raises(ValueError, match="`records` must be a CUDA tensor"):
        step(rec, torch.zeros_like(rec), torch.zeros_like(rec), [torch.zeros(4, 3), torch.zeros(4, 3, 3),
             torch.zeros(4, 3, 1), torch.zeros(4)], None, 1)
