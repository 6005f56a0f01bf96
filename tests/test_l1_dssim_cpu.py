"""CPU tests of 3DGS's L1 + D-SSIM loss and the refinement options built on it: the float64 restatement
(tests/l1_dssim_f64.py) against a direct transcription of 3DGS's conv2d SSIM + L1, its closed-form gradient against
autograd and gradcheck; the position rate's decay against 3DGS's get_expon_lr_func; the refine-ply flags and
refine.json's keys; the C ABI's and the Python layer's refusals, which happen before anything reaches a device."""
import ctypes
import math

import pytest
import torch

from pixelsplat_b200 import _lib, ply_refine as pr
from tests import l1_dssim_f64 as lf


def _pair(kind: str, shape, seed: int = 0):
    g = torch.Generator().manual_seed(seed)
    r = lambda: torch.rand(shape, generator=g, dtype=torch.float64)
    if kind == "noise":
        return r(), r()
    if kind == "flat_bright":
        return 0.95 + 0.002 * (2 * r() - 1), 0.95 + 0.002 * (2 * r() - 1)
    if kind == "outside":
        return 1.6 * r() - 0.3, 1.4 * r() - 0.2
    if kind == "ties":
        p, q = r(), r()
        q[..., : shape[-2] // 2, :] = p[..., : shape[-2] // 2, :]
        return p, q
    raise KeyError(kind)


SHAPES = [(1, 3, 1, 1), (1, 3, 5, 7), (1, 3, 11, 11), (2, 3, 17, 45), (1, 1, 30, 12)]


@pytest.mark.parametrize("kind", ["noise", "flat_bright", "outside", "ties"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_restatement_matches_the_3dgs_transcription(shape, kind):
    p, g = _pair(kind, shape, sum(shape))
    for lam in (0.0, 0.2, 1.0):
        got, l1, ssim = lf.l1_dssim_f64(p, g, lam)
        want = lf.loss_3dgs_torch(p, g, lam)
        assert got.shape == (shape[0],)
        assert (got - want).abs().max() <= 1e-12, (lam, got, want)
        assert torch.allclose((1 - lam) * l1 + lam * (1 - ssim), got, rtol=0, atol=1e-15)


def test_known_answers():
    x = torch.rand((2, 3, 9, 13), generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    loss, l1, ssim = lf.l1_dssim_f64(x, x, 0.2)
    assert torch.all(l1 == 0) and torch.allclose(ssim, torch.ones(2, dtype=torch.float64), rtol=0, atol=1e-14)
    assert loss.abs().max() <= 1e-14
    # a constant image against another: the zero padding makes the border windows see a smaller mean, so the SSIM
    # map is not the interior's constant; the interior value is (2ab + C1) / (a^2 + b^2 + C1)
    a, b = 0.3, 0.7
    _, _, _, _, _, _, s = lf._terms(torch.full((1, 1, 40, 40), b, dtype=torch.float64),
                                    torch.full((1, 1, 40, 40), a, dtype=torch.float64))
    want = (2 * a * b + lf.C1) / (a * a + b * b + lf.C1)
    assert abs(float(s[0, 0, 20, 20]) - want) <= 1e-12 and abs(float(s[0, 0, 0, 0]) - want) > 1e-3


@pytest.mark.parametrize("shape", [(1, 3, 1, 1), (2, 3, 6, 9), (1, 2, 13, 12)], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("kind", ["noise", "flat_bright", "outside"])
def test_closed_form_gradient_matches_autograd(shape, kind):
    p, g = _pair(kind, shape, 7 + sum(shape))
    w = torch.randn(shape[0], generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    for lam in (0.0, 0.2, 1.0):
        pg = p.clone().requires_grad_(True)
        (lf.l1_dssim_f64(pg, g, lam)[0] * w).sum().backward()
        got = lf.l1_dssim_grad_f64(p, g, lam) * w.view(-1, 1, 1, 1)
        assert (got - pg.grad).abs().max() <= 1e-12 * max(1.0, float(pg.grad.abs().max())), lam


def test_closed_form_gradient_passes_gradcheck():
    for shape, lam in (((2, 3, 6, 9), 0.2), ((1, 1, 12, 13), 1.0), ((1, 2, 1, 3), 0.5)):
        p, g = _pair("noise", shape, sum(shape))
        p.requires_grad_(True)
        assert torch.autograd.gradcheck(lambda a: lf.L1DssimF64.apply(a, g, lam), (p,), eps=1e-6, atol=1e-8)


def test_the_l1_gradient_is_zero_at_ties():
    p, g = _pair("ties", (1, 3, 16, 20), 5)
    tie = p == g
    assert tie.any() and (~tie).any()
    d = lf.l1_dssim_grad_f64(p, g, 0.0)
    assert torch.all(d[tie] == 0) and torch.all(d[~tie].abs() == 1 / (3 * 16 * 20))


# ---- the position rate's decay


@pytest.mark.parametrize("decay_steps", [1, 7, 30, 30_000])
def test_decay_matches_3dgs_schedule(decay_steps):
    lr0, lr1 = 1.6e-4, 1.6e-6
    for t in list(range(0, 40)) + [decay_steps - 1, decay_steps, decay_steps + 1, 10 * decay_steps]:
        got, want = pr.xyz_lr_at(t, lr0, lr1, decay_steps), lf.expon_lr(t, lr0, lr1, decay_steps)
        assert abs(got - want) <= 1e-15 * want, (t, got, want)
    assert pr.xyz_lr_at(0, lr0, lr1, decay_steps) == pytest.approx(lr0, rel=1e-15)
    assert pr.xyz_lr_at(decay_steps, lr0, lr1, decay_steps) == pytest.approx(lr1, rel=1e-15)
    assert pr.xyz_lr_at(decay_steps + 5, lr0, lr1, decay_steps) == pytest.approx(lr1, rel=1e-15)


def test_decay_arguments_are_checked():
    kw = dict(extrinsics=None, intrinsics=None, near=None, far=None, images=None, background_color=None, steps=1)
    rec = torch.zeros(1, 14)
    names = ["x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2", "opacity", "scale_0", "scale_1", "scale_2", "rot_0",
             "rot_1", "rot_2", "rot_3"]
    for bad, match in ((dict(lr_xyz_final=0.0), "lr_xyz_final"), (dict(lr_xyz_final=math.inf), "lr_xyz_final"),
                       (dict(lr_xyz_steps=10), "needs `lr_xyz_final`"),
                       (dict(lr_xyz_final=1e-6, lr_xyz_steps=0), "lr_xyz_steps"),
                       (dict(lr_xyz_final=1e-6, lr={"xyz": 0.0}), "xyz rate > 0"),
                       (dict(loss="l2"), "`loss` must be one of"), (dict(lambda_dssim=1.5), "lambda_dssim"),
                       (dict(lambda_dssim=math.nan), "lambda_dssim")):
        with pytest.raises(ValueError, match=match):
            pr.refine_records(rec, names, 0, **kw, **bad)


def test_refine_step_sets_only_the_position_rates():
    names = ["rot_0", "x", "f_dc_0", "f_dc_1", "f_dc_2", "y", "opacity", "scale_0", "scale_1", "scale_2", "z",
             "rot_1", "rot_2", "rot_3", "extra"]
    step = pr.RefineStep(names, 0, 10)
    assert [names[c] for c in step.xyz_columns] == ["x", "y", "z"]
    assert list(step.desc.lr[:len(names)]) == pr.column_lr(names, 0)


# ---- command line


def test_refine_ply_loss_flags_parse():
    from pixelsplat_b200.evaluation import __main__ as cli
    base = ["--ply", "p", "--dataset-root", "d", "--index", "i.json", "--output", "o"]
    a = cli.parse_refine_ply(base)
    assert (a.loss, a.lambda_dssim, a.lr_xyz_final, a.lr_xyz_steps) == ("mse", 0.2, None, None)
    a = cli.parse_refine_ply(base + ["--loss", "l1-dssim", "--lambda-dssim", "0.5", "--lr-xyz-final", "1.6e-6",
                                     "--lr-xyz-steps", "30000"])
    assert (a.loss, a.lambda_dssim, a.lr_xyz_final, a.lr_xyz_steps) == ("l1_dssim", 0.5, 1.6e-6, 30000)
    assert cli._refine_options(a) == dict(loss="l1_dssim", lambda_dssim=0.5, lr_xyz_final=1.6e-6, lr_xyz_steps=30000)
    for bad in (["--loss", "l2"], ["--lambda-dssim", "1.5"], ["--lr-xyz-final", "0"], ["--lr-xyz-steps", "100"],
                ["--lr-xyz-final", "1e-6", "--lr-xyz-steps", "0"], ["--lr-xyz", "0", "--lr-xyz-final", "1e-6"]):
        with pytest.raises(SystemExit):
            cli.parse_refine_ply(base + bad)


def test_refine_json_keys():
    from pixelsplat_b200.evaluation import __main__ as cli
    base = ["--ply", "p", "--dataset-root", "d", "--index", "i.json", "--output", "o", "--steps", "3"]
    result = pr.RefineResult(torch.zeros(2, 14), torch.tensor([4.0, 3.0, 2.0, 1.0]))
    a = cli.parse_refine_ply(base)
    scene = cli._refine_scene_report(a, result)
    assert scene == {"mse_before": 4.0, "mse_after": 1.0, "steps": 3}
    assert list(cli._refine_report(a, {"s": scene})) == ["steps", "lr", "scenes"]
    a = cli.parse_refine_ply(base + ["--loss", "l1-dssim", "--lr-xyz-final", "1e-6"])
    dssim = pr.RefineResult(torch.zeros(2, 14), torch.tensor([0.4, 0.3, 0.2, 0.1]), mse=torch.tensor([5.0, 0.5]))
    scene = cli._refine_scene_report(a, dssim)
    assert scene == pytest.approx({"mse_before": 5.0, "mse_after": 0.5, "steps": 3, "loss_before": 0.4,
                                   "loss_after": 0.1})
    report = cli._refine_report(a, {"s": scene})
    assert list(report) == ["steps", "lr", "scenes", "loss", "lambda_dssim", "lr_xyz_final", "lr_xyz_steps"]
    assert (report["loss"], report["lambda_dssim"], report["lr_xyz_final"], report["lr_xyz_steps"]) == \
        ("l1_dssim", 0.2, 1e-6, 3)


# ---- the C ABI and the Python layer


def test_abi_refuses_before_launching():
    L = _lib.lib
    fake = 1 << 20                        # never dereferenced: every call below is refused first
    ws = ctypes.c_size_t()
    assert L.ps_l1_dssim_workspace_bytes(2, 3, 1, 1, ctypes.byref(ws)) == 0 and ws.value == 256
    assert L.ps_l1_dssim_workspace_bytes(4, 3, 256, 256, ctypes.byref(ws)) == 0
    assert ws.value == 2 * 4 * 3 * 8 * 16 * 4
    assert L.ps_l1_dssim_workspace_bytes(1, 1, 8, 8, None) == 1
    need = ws.value

    def call(n=4, c=3, h=256, w=256, pred=fake, gt=fake, lam=0.2, out=fake, d=fake, work=fake, nbytes=need):
        return L.ps_l1_dssim(n, c, h, w, pred, gt, lam, out, None, None, d, work, nbytes, None)

    for kw in (dict(n=0), dict(c=0), dict(h=0), dict(w=-1), dict(n=1 << 20, c=1 << 10),
               dict(lam=-0.01), dict(lam=1.01), dict(lam=math.nan), dict(lam=math.inf),
               dict(pred=None), dict(gt=None), dict(out=None), dict(work=None), dict(nbytes=need - 1)):
        assert call(**kw) == 1, kw                               # PS_ERR_INVALID_ARGUMENT, not a CUDA error
    for n, c, h, w in ((0, 3, 4, 4), (1, 3, 0, 4), (1 << 20, 1 << 10, 17, 32)):
        assert L.ps_l1_dssim_workspace_bytes(n, c, h, w, ctypes.byref(ws)) == 1


def test_python_checks_before_the_device():
    from pixelsplat_b200.loss import l1_dssim
    x = torch.rand(2, 3, 8, 8)
    for args, match in (((x, x[:1]), "one shape"), ((x[0], x[0]), "one shape"), ((x.double(), x), "float32"),
                        ((x, x), "no CPU path"), ((x[:, :, :0], x[:, :, :0]), "empty")):
        with pytest.raises(ValueError, match=match):
            l1_dssim(*args)
    for lam in (-0.1, 1.5, math.nan, True):
        with pytest.raises(ValueError, match="lambda_dssim"):
            l1_dssim(x, x, lam)
