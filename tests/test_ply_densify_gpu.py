"""PLY densification on the GPU (csrc/ply_densify.cu behind pixelsplat_b200.ply_refine):
  1. the three kernels against the float64 restatement (tests/ply_densify_f64.py) with the same draws and the same
     float32 statistics, across counts, SH degrees, extra columns and mixes (mixed, all pruned but one, all split):
     identical decisions and order, copied columns and moments bit for bit, split positions and log-scales within
     1 ulp, untouched NaN tails, repeatable bits;
  2. the loop without densification is the loop of the plain refinement, bit for bit and launch for launch;
  3. densification on a synthetic scene: a coarse start with planted transparent rows;
  4. the command line on re10k_tiny: export-ply --write-frame, refine-ply with densification, render-ply."""
import json
import math

import numpy as np
import pytest
import torch

from pixelsplat_b200 import _lib, ply_import as pi, ply_refine as pr
from tests import dataset_golden as dg
from tests import ply_densify_f64 as df
from tests import ply_import_f64 as f64
from tests.test_ply_refine_gpu import CONVERGE_LR, synthetic_views

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def case_records(n: int, degree: int, extras: bool, mix: str, g: np.random.Generator):
    """Shuffled columns; log-scales U(-7, -1.5) (big above log 0.01), zero quaternions every 7th row, opacity
    logits N(0, 4); `mix` 'one': every opacity at -20 but row 0's; 'split': every row big, opaque and selected."""
    names = f64.gs_properties(degree, extras) + (["extra_0", "extra_1"] if extras else [])
    names = [names[i] for i in g.permutation(len(names))]
    c = df.columns(names)
    rec = g.standard_normal((n, len(names))).astype(np.float32)
    rec[:, c["scale"]] = g.uniform(-7, -1.5, (n, 3))
    rec[::7, c["rot"]] = 0.0
    rec[:, c["opacity"]] = 4 * g.standard_normal(n)
    if mix == "one":
        rec[0, c["opacity"]] = abs(rec[0, c["opacity"]])
        rec[0, c["scale"]] = -5.0
        rec[1:, c["opacity"]] = -20.0
    if mix == "split":
        rec[:, c["scale"][0]] = g.uniform(-4, -3, n)
        rec[:, c["opacity"]] = np.abs(rec[:, c["opacity"]])
    return torch.from_numpy(rec), names


def ulps(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    return (a.view(torch.int32).long() - b.view(torch.int32).long()).abs()


@pytest.mark.parametrize("degree", [0, 1, 2, 3])
@pytest.mark.parametrize("n", [1, 63, 64, 65, 4133, 393_216])
def test_kernels_match_the_restatement(n, degree):
    g = np.random.default_rng(100 + 10 * degree + n % 997)
    views = 2
    for extras, mix, prune_world in ((True, "mixed", False), (False, "mixed", True), (True, "one", True),
                                     (False, "split", False)):
        rec, names = case_records(n, degree, extras, mix, g)
        p = len(names)
        cfg = pr.DensifyConfig()
        # statistics: two views, about a third of the rows off-screen in each; NaN where a view is off-screen, as
        # the backward leaves those rows of d_means2d unwritten
        d2 = torch.from_numpy((g.standard_normal((views, n, 3)) * 3e-4).astype(np.float32))
        radii = torch.from_numpy(g.integers(-2, 4, (views, n)).astype(np.int32))
        d2[radii <= 0] = math.nan
        if mix == "split":
            radii[:] = 1
            d2[..., :2] = 1e-2
        accum0 = torch.from_numpy(g.uniform(0, 1e-3, n).astype(np.float32)) * (mix != "split")
        count0 = torch.from_numpy(g.integers(0, 3, n).astype(np.int32))
        runs = []
        for _ in range(2):
            accum, count = accum0.to(DEV), count0.to(DEV)
            pr.densify_stats(d2.to(DEV), radii.to(DEV), accum, count)
            runs.append((accum.cpu(), count.cpu()))
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
        accum, count = runs[0]
        want_a, want_c = df.stats_f64(torch.nan_to_num(d2), radii, accum0, count0)
        assert torch.equal(count, want_c)
        rel = ((accum.double() - want_a).abs() / want_a.clamp(min=1e-30)).max().item()
        assert rel <= 1e-6, rel

        m = torch.from_numpy(g.standard_normal((n, p)).astype(np.float32))
        v = torch.from_numpy(g.uniform(0, 1, (n, p)).astype(np.float32))
        eps = torch.from_numpy(g.standard_normal((2, n, 3)).astype(np.float32))
        want = df.densify_f64(rec, m, v, accum, count, names, cfg, prune_world, eps)
        keep, clone, split = df.flags(rec, accum, count, names, cfg, prune_world)
        n_new = want[0].shape[0]
        if mix == "one":
            assert n_new >= 1 and keep[1:].sum() + clone[1:].sum() + split[1:].sum() == 0
        if mix == "split":
            assert split.all() and n_new == 2 * n
        if n_new == 0:      # a small mixed case can prune every row
            with pytest.raises(ValueError, match="every Gaussian would be pruned"):
                pr.densify_records(rec.to(DEV), m.to(DEV), v.to(DEV), accum.to(DEV), count.to(DEV), names, cfg,
                                   prune_world=prune_world, eps=eps.to(DEV))
            continue
        outs = []
        for _ in range(2):
            bufs = [torch.full((2 * n + 5, p), math.nan, device=DEV) for _ in range(3)]
            got = pr.densify_records(rec.to(DEV), m.to(DEV), v.to(DEV), accum.to(DEV), count.to(DEV), names, cfg,
                                     prune_world=prune_world, eps=eps.to(DEV), out=bufs)
            assert all(t.shape == (n_new, p) for t in got)
            for b in bufs:
                assert b[n_new:].isnan().all(), "a row past n_new was written"
            outs.append([t.cpu() for t in got])
        for a, b in zip(*outs):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "reruns differ"
        got = outs[0]
        c = df.columns(names)
        moved = torch.zeros((n_new, p), dtype=torch.bool)
        first = int(keep.sum()) + int(clone.sum())
        moved[first:, c["xyz"] + c["scale"]] = True
        d = ulps(got[0], want[0])
        assert (d[~moved] == 0).all(), "a copied column differs"
        assert (d[moved] <= 1).all(), f"split copies off by {d[moved].max()} ulp"
        assert torch.equal(got[1].view(torch.int32), want[1].view(torch.int32))
        assert torch.equal(got[2].view(torch.int32), want[2].view(torch.int32))
        print(f"DENSIFY n={n} degree={degree} {mix}: {n} -> {n_new} (keep {int(keep.sum())}, clone "
              f"{int(clone.sum())}, split {int(split.sum())}); worst split ulp {int(d[moved].max()) if moved.any() else 0}")


def test_densification_refuses_an_empty_result_and_bad_tensors():
    rec, names = case_records(100, 1, False, "one", np.random.default_rng(1))
    rec[0, names.index("opacity")] = -20.0
    rec = rec.to(DEV)
    z = torch.zeros_like(rec)
    a, c = torch.zeros(100, device=DEV), torch.zeros(100, dtype=torch.int32, device=DEV)
    eps = torch.zeros(2, 100, 3, device=DEV)
    before = rec.clone()
    with pytest.raises(ValueError, match="every Gaussian would be pruned"):
        pr.densify_records(rec, z, z, a, c, names, pr.DensifyConfig(), prune_world=False, eps=eps)
    assert torch.equal(rec, before)
    with pytest.raises(ValueError, match="`eps` must be a dense float32"):
        pr.densify_records(rec, z, z, a, c, names, pr.DensifyConfig(), prune_world=False, eps=eps[:, :50])
    with pytest.raises(ValueError, match="`count` must be a dense int32"):
        pr.densify_records(rec, z, z, a, c.float(), names, pr.DensifyConfig(), prune_world=False, eps=eps)
    with pytest.raises(ValueError, match="`radii` must be a dense int32"):
        pr.densify_stats(torch.zeros(2, 100, 3, device=DEV), torch.zeros(2, 100, device=DEV), a, c)


# ---- the refinement loop


def plain_refinement(records, names, frame, views, steps, lr):
    """The refinement loop as it is without densification: render, backward, ps_ply_refine_step; then the final
    loss's render."""
    from pixelsplat_b200.decoder import Gaussians
    from pixelsplat_b200.decoder.cuda_splatting import render_views_mse
    n, v = records.shape[0], views["images"].shape[0]
    h, w = views["images"].shape[-2:]
    cam = [views[k][None] for k in ("extrinsics", "intrinsics", "near", "far")]
    bg = views["background_color"].reshape(1, 1, 3).expand(1, v, 3)
    leaves = [torch.empty((1, n, 3), device=DEV), torch.empty((1, n, 3, 3), device=DEV),
              torch.empty((1, n, 3, 16), device=DEV), torch.empty((1, n), device=DEV)]
    out = Gaussians(*(t[0] for t in leaves))
    work = records.clone()
    pi.unpack_records(work, names, 3, frame=frame, out=out)
    m, v2 = torch.zeros_like(work), torch.zeros_like(work)
    step = pr.RefineStep(names, 3, n, sh_coeffs=16, frame=frame, lr=lr)
    for leaf in leaves:
        leaf.requires_grad_(True)
    for t in range(1, steps + 1):
        sse, _, _ = render_views_mse(*cam, (h, w), bg, *leaves, target=views["images"][None], want_color=False)
        (sse.sum() / (v * 3 * h * w)).backward()
        grads = [leaf.grad[0].contiguous() for leaf in leaves]
        for leaf in leaves:
            leaf.grad = None
        step(work, m, v2, grads, out, t)
    with torch.no_grad():
        render_views_mse(*cam, (h, w), bg, *leaves, target=views["images"][None], want_color=False)
    return work, m, v2


def test_without_densification_the_loop_is_unchanged():
    records, names, frame, views = synthetic_views(3, seed=8, num_gaussians=1500)
    steps = 6
    runs = {}
    for name, fn in (("plain", lambda: plain_refinement(records, names, frame, views, steps, CONVERGE_LR)),
                     ("none", lambda: pr.refine_records(records, names, 3, frame=frame, steps=steps, lr=CONVERGE_LR,
                                                        **views)),
                     ("until 0", lambda: pr.refine_records(records, names, 3, frame=frame, steps=steps,
                                                           lr=CONVERGE_LR, densify=pr.DensifyConfig(until_step=0),
                                                           **views))):
        torch.cuda.synchronize()
        before = _lib.lib.ps_launch_count()
        res = fn()
        torch.cuda.synchronize()
        launches = _lib.lib.ps_launch_count() - before
        runs[name] = ((res[0], res[1], res[2]) if isinstance(res, tuple) else
                      (res.records, res.exp_avg, res.exp_avg_sq), launches, res)
    for name in ("none", "until 0"):
        for a, b in zip(runs[name][0], runs["plain"][0]):
            assert torch.equal(a, b), name
    assert runs["none"][1] == runs["plain"][1]
    assert runs["until 0"][1] == runs["none"][1]
    assert runs["none"][2].gaussians is None and runs["until 0"][2].gaussians == [1500] * (steps + 1)


def coarse_start(records, names, g: torch.Generator, planted: int = 100):
    """Every fourth record with scales doubled, plus `planted` copies of random records at opacity logit -8; a
    marker column (1 on the planted rows) travels with the records."""
    c = df.columns(names)
    coarse = records[::4].clone()
    coarse[:, c["scale"]] += math.log(2.0)
    idx = torch.randint(0, coarse.shape[0], (planted,), generator=g, device=DEV)
    dead = coarse[idx].clone()
    dead[:, c["opacity"]] = -8.0
    rec = torch.cat([coarse, dead])
    marker = torch.cat([torch.zeros(coarse.shape[0], device=DEV), torch.ones(planted, device=DEV)])
    return torch.cat([rec, marker[:, None]], 1).contiguous(), names + ["marker"]


# a coarse start (every fourth of 6 000 Gaussians, scales doubled, 100 planted transparent rows), 6 views, 400 steps
# at equal rates, densifying every 50 steps before step 300; the threshold is set for the fused MSE of 6 views, whose
# gradients are smaller than 3DGS's single-view ones.  Measured on an H100 80GB HBM3 (DESIGN.md section 10j):
# 1 600 -> 7 077 Gaussians, final context MSE with densification 0.031 of the MSE without; the bar keeps a 3x margin
E2E_STEPS, E2E_DENSIFY = 400, pr.DensifyConfig(from_step=0, until_step=300, every=50, grad_threshold=2e-6,
                                               opacity_reset_every=0)
E2E_FRACTION = 0.1


def test_densification_improves_a_coarse_start():
    records, names, frame, views = synthetic_views(6, seed=12, num_gaussians=6000)
    start, names2 = coarse_start(records, names, torch.Generator(DEV).manual_seed(0))
    n0 = start.shape[0]
    first = E2E_DENSIFY.from_step + E2E_DENSIFY.every
    early = pr.refine_records(start, names2, 3, frame=frame, steps=first, lr=CONVERGE_LR, densify=E2E_DENSIFY,
                              **views)
    assert early.records.shape[0] == early.gaussians[-1] and early.gaussians[:first] == [n0] * first
    assert not early.records[:, -1].any(), "a planted transparent row survived the first densification"
    on = pr.refine_records(start, names2, 3, frame=frame, steps=E2E_STEPS, lr=CONVERGE_LR, densify=E2E_DENSIFY,
                           **views)
    off = pr.refine_records(start, names2, 3, frame=frame, steps=E2E_STEPS, lr=CONVERGE_LR, **views)
    a, b = on.loss[-1].item(), off.loss[-1].item()
    print(f"E2E: {n0} -> {on.gaussians[-1]} Gaussians (after each densification: "
          f"{sorted(set(on.gaussians), key=on.gaussians.index)}); context MSE {on.loss[0]:.4e} -> with "
          f"densification {a:.4e}, without {b:.4e} ({a / b:.3f})")
    assert on.gaussians[-1] > n0
    assert a <= E2E_FRACTION * b


# ---- command line


def test_command_line_with_densification_on_re10k_tiny(tmp_path, monkeypatch):
    from pixelsplat_b200.evaluation import __main__ as cli
    from pixelsplat_b200.evaluation import presets as ev
    from pixelsplat_b200.evaluation.checkpoint import save_checkpoint
    from tests.test_evaluation_gpu import _seeded_lpips
    index = dg.DATA / "evaluation_index.json"
    encoder, _ = ev.build_model("re10k", ev.dataset_cfg(dg.DATA, index))
    ckpt = save_checkpoint(tmp_path / "random.ckpt", encoder, 0)
    data = ["--dataset-root", str(dg.DATA), "--index", str(index), "--num-workers", "0"]
    cli.main(["export-ply"] + data + ["--checkpoint", str(ckpt), "--preset", "re10k", "--output",
                                      str(tmp_path / "ply"), "--write-frame"])
    scenes = [w["scene"] for w in dg.expected("test")]
    cli.main(["refine-ply"] + data + ["--ply", str(tmp_path / "ply"), "--output", str(tmp_path / "refined"),
                                      "--steps", "30", "--densify-from", "5", "--densify-until", "25",
                                      "--densify-every", "10", "--densify-grad", "1e-7"])
    report = json.loads((tmp_path / "refined" / "refine.json").read_text())
    assert sorted(report["scenes"]) == sorted(scenes) and report["densify"]["until_step"] == 25
    for s, r in report["scenes"].items():
        print(f"REFINE_PLY_DENSIFY {s}: {r['gaussians_before']} -> {r['gaussians_after']} Gaussians, context MSE "
              f"{r['mse_before']:.5f} -> {r['mse_after']:.5f}")
        original = (tmp_path / "ply" / f"{s}.ply").read_bytes()
        refined = (tmp_path / "refined" / f"{s}.ply").read_bytes()
        lo, lr_ = pi.parse_header(original), pi.parse_header(refined)
        assert lo.count == r["gaussians_before"] and lr_.count == r["gaussians_after"] != r["gaussians_before"]
        assert lr_.properties == lo.properties
        assert refined[:lr_.body_offset] == pr.rewrite_vertex_count(original[:lo.body_offset], lr_.count)
        assert len(refined) == lr_.body_offset + 4 * lr_.count * len(lr_.properties)
        g = pi.load_gaussians_ply(tmp_path / "refined" / f"{s}.ply", DEV,
                                  frame=tmp_path / "refined" / f"{s}.frame.json")
        assert g.means.shape[1] == r["gaussians_after"]
        assert all(torch.isfinite(getattr(g, k)).all() for k in ("means", "covariances", "harmonics", "opacities"))
    monkeypatch.setattr(cli, "_lpips", lambda args, device: _seeded_lpips())
    out = cli.render_ply(["--ply", str(tmp_path / "refined"), "--output", str(tmp_path / "rendered")] + data)
    assert sorted(out["scenes"]) == sorted(scenes) and (tmp_path / "rendered" / "metrics.json").exists()
