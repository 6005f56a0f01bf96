"""PLY densification on the CPU: the float64 restatement (tests/ply_densify_f64.py) against a direct transcription of
3DGS's masked and concatenated densify_and_clone / densify_and_split / prune on hand-built records that reach every
branch, the configuration and its schedule, the header rewrite, the command line, and the ABI's layout and
refusals."""
import ctypes
import math
from pathlib import Path

import numpy as np
import pytest
import torch

from pixelsplat_b200 import _lib, ply_refine as pr
from tests import ply_densify_f64 as df
from tests import ply_import_f64 as f64

THR = np.float32(2e-4)


def transcription(records, exp_avg, exp_avg_sq, accum, count, names, cfg, prune_world, eps):
    """3DGS's densify_and_prune on the records, step by step: clone (concatenated), split on the grown set with the
    clones' gradients padded with zeros (copies concatenated, the originals removed), then the prune mask over the
    result."""
    c = df.columns(names)
    zeros = lambda k: torch.zeros((k, records.shape[1]))
    g = df.mean_grad(accum, count)
    thr = torch.tensor(cfg.grad_threshold, dtype=torch.float32)
    smax = records[:, c["scale"]].double().exp().amax(-1)
    clone = (g >= thr) & (smax <= cfg.percent_dense * cfg.extent)
    rec = torch.cat([records, records[clone]])
    m, v = torch.cat([exp_avg, zeros(int(clone.sum()))]), torch.cat([exp_avg_sq, zeros(int(clone.sum()))])
    origin = torch.cat([torch.arange(len(records)), torch.nonzero(clone)[:, 0]])
    padded = torch.cat([g, torch.zeros(int(clone.sum()))])
    split = (padded >= thr) & (rec[:, c["scale"]].double().exp().amax(-1) > cfg.percent_dense * cfg.extent)
    sel, idx = rec[split], origin[split]
    rot = df.rotation_f64(sel[:, c["rot"]])
    copies = []
    for k in range(2):
        copy = sel.clone()
        for i in range(len(sel)):
            s = sel[i, c["scale"]].double().exp() * eps[k, idx[i]].double()
            copy[i, c["xyz"]] = (sel[i, c["xyz"]].double() + rot[i] @ s).float()
            copy[i, c["scale"]] = (sel[i, c["scale"]].double() - math.log(1.6)).float()
        copies.append(copy)
    ns = len(sel)
    rec = torch.cat([rec] + copies)[torch.cat([~split, torch.ones(2 * ns, dtype=torch.bool)])]
    m = torch.cat([m, zeros(2 * ns)])[torch.cat([~split, torch.ones(2 * ns, dtype=torch.bool)])]
    v = torch.cat([v, zeros(2 * ns)])[torch.cat([~split, torch.ones(2 * ns, dtype=torch.bool)])]
    prune = 1.0 / (1.0 + torch.exp(-rec[:, c["opacity"]].double())) < cfg.min_opacity
    if prune_world:
        prune |= rec[:, c["scale"]].double().exp().amax(-1) > 0.1 * cfg.extent
    return rec[~prune], m[~prune], v[~prune]


def hand_built(degree: int = 1):
    """One row per branch (see ROWS); the remaining columns random."""
    names = f64.gs_properties(degree, True) + ["extra_0"]
    c = df.columns(names)
    n = len(ROWS)
    g = np.random.default_rng(3)
    rec = torch.from_numpy(g.standard_normal((n, len(names))).astype(np.float32))
    accum, count = torch.zeros(n), torch.ones(n, dtype=torch.int32)
    small, big, huge = math.log(0.005), math.log(0.05), math.log(0.12)
    for i, (grad, scale, opacity) in enumerate(ROWS.values()):
        rec[i, c["scale"]] = torch.tensor([scale, scale - 1.0, scale - 2.0]) if scale is not None else \
            torch.tensor([small, small, small])
        rec[i, c["opacity"]] = opacity
        accum[i] = grad
    rec[list(ROWS).index("zero quaternion"), c["rot"]] = 0.0
    count[list(ROWS).index("count 0")] = 0
    m = torch.from_numpy(g.standard_normal(rec.shape).astype(np.float32))
    v = torch.from_numpy(g.uniform(0, 1, rec.shape).astype(np.float32))
    eps = torch.from_numpy(g.standard_normal((2, n, 3)).astype(np.float32))
    return names, rec, m, v, accum, count, eps, (small, big, huge)


_big, _huge = math.log(0.05), math.log(0.12)
# name: (accum with count 1, largest log-scale or None for small, opacity logit)
ROWS = {
    "keep": (1e-5, None, 0.0),
    "clone": (1e-3, None, 0.0),
    "split": (1e-3, _big, 0.0),
    "pruned original": (1e-5, None, -8.0),
    "pruned clone": (1e-3, None, -8.0),
    "pruned split": (1e-3, _big, -8.0),
    "world-size": (1e-5, _huge, 0.0),
    "world-size split": (1e-3, _huge, 0.0),       # the copies' scale, / 1.6, is below 0.1
    "count 0": (1.0, None, 0.0),
    "1 ulp above": (float(np.nextafter(THR, np.float32(1))), None, 0.0),
    "at the threshold": (float(THR), None, 0.0),
    "1 ulp below": (float(np.nextafter(THR, np.float32(0))), None, 0.0),
    "zero quaternion": (1e-3, _big, 0.0),
}


@pytest.mark.parametrize("prune_world", [False, True])
def test_restatement_matches_the_transcription_on_every_branch(prune_world):
    names, rec, m, v, accum, count, eps, _ = hand_built()
    cfg = pr.DensifyConfig()
    keep, clone, split = df.flags(rec, accum, count, names, cfg, prune_world)
    row = {k: i for i, k in enumerate(ROWS)}
    want_keep = {"keep", "clone", "count 0", "1 ulp above", "at the threshold", "1 ulp below"} | \
        (set() if prune_world else {"world-size"})
    want_clone = {"clone", "1 ulp above", "at the threshold"}
    want_split = {"split", "world-size split", "zero quaternion"}
    assert {k for k in ROWS if keep[row[k]]} == want_keep
    assert {k for k in ROWS if clone[row[k]]} == want_clone
    assert {k for k in ROWS if split[row[k]]} == want_split

    got = df.densify_f64(rec, m, v, accum, count, names, cfg, prune_world, eps)
    want = transcription(rec, m, v, accum, count, names, cfg, prune_world, eps)
    for a, b in zip(got, want):
        assert a.shape == b.shape and torch.equal(a, b)
    n_keep, n_new = int(keep.sum()), int(clone.sum()) + 2 * int(split.sum())
    assert got[0].shape[0] == n_keep + n_new
    assert torch.equal(got[1][:n_keep], m[keep]) and torch.equal(got[2][:n_keep], v[keep])
    assert not got[1][n_keep:].any() and not got[2][n_keep:].any(), "new rows must start with zero moments"


def test_split_copies_of_a_zero_quaternion_use_the_identity():
    names, rec, m, v, accum, count, eps, _ = hand_built()
    c = df.columns(names)
    i = list(ROWS).index("zero quaternion")
    first, second = df.split_copies(rec, names, eps)
    for k, copy in enumerate((first, second)):
        want = (rec[i, c["xyz"]].double() + rec[i, c["scale"]].double().exp() * eps[k, i].double()).float()
        assert torch.equal(copy[i, c["xyz"]], want)
        assert torch.equal(copy[i, c["scale"]], (rec[i, c["scale"]].double() - math.log(1.6)).float())
        other = [j for j in range(len(names)) if j not in c["xyz"] + c["scale"]]
        assert torch.equal(copy[i, other], rec[i, other])


def test_statistics_and_opacity_reset():
    g = torch.Generator().manual_seed(0)
    d = torch.randn(3, 10, 3, generator=g)
    radii = torch.randint(-1, 3, (3, 10), generator=g, dtype=torch.int32)
    accum, count = torch.rand(10, generator=g), torch.randint(0, 5, (10,), generator=g, dtype=torch.int32)
    a, c = df.stats_f64(d, radii, accum, count)
    for i in range(10):
        on = [k for k in range(3) if radii[k, i] > 0]
        assert c[i] == count[i] + len(on)
        assert a[i] == pytest.approx(float(accum[i]) + sum(math.hypot(d[k, i, 0], d[k, i, 1]) for k in on), rel=1e-12)
    names = f64.gs_properties(0)
    rec = torch.randn(20, len(names), generator=g) * 6
    m, v = torch.randn(20, len(names), generator=g), torch.rand(20, len(names), generator=g)
    r2, m2, v2 = df.reset_opacity_f64(rec, m, v, names)
    o = names.index("opacity")
    assert torch.equal(r2[:, o], torch.clamp(rec[:, o], max=np.float32(math.log(0.01 / 0.99))))
    assert (r2[:, o] <= -4.59).all() and not m2[:, o].any() and not v2[:, o].any()
    keep = [j for j in range(len(names)) if j != o]
    assert torch.equal(r2[:, keep], rec[:, keep]) and torch.equal(m2[:, keep], m[:, keep])
    # the host's in-place reset is the restatement's
    r3, m3, v3 = rec.clone(), m.clone(), v.clone()
    pr.reset_opacity(r3, m3, v3, names)
    assert torch.equal(r3, r2) and torch.equal(m3, m2) and torch.equal(v3, v2)


def test_config_defaults_schedule_and_checks():
    d = pr.DensifyConfig()
    assert (d.from_step, d.until_step, d.every, d.grad_threshold, d.percent_dense, d.min_opacity,
            d.opacity_reset_every, d.extent, d.seed) == (500, 15000, 100, 2e-4, 0.01, 0.005, 3000, 1.0, 0)
    assert [t for t in range(1, 1001) if d.densifies_at(t)] == list(range(600, 1001, 100))
    assert not d.densifies_at(500) and not d.densifies_at(15000) and d.densifies_at(14900)
    assert d.resets_at(3000) and not d.resets_at(15000) and not d.resets_at(2999)
    assert not d.prunes_world_at(3000) and d.prunes_world_at(3001)
    assert d.stats_at(14999) and not d.stats_at(15000)
    off = pr.DensifyConfig(opacity_reset_every=0)
    assert not any(off.resets_at(t) or off.prunes_world_at(t) for t in range(1, 20000))
    zero = pr.DensifyConfig(until_step=0)
    assert not any(zero.stats_at(t) or zero.densifies_at(t) or zero.resets_at(t) for t in range(1, 20000))
    for bad in (dict(every=0), dict(from_step=-1), dict(until_step=1.5), dict(grad_threshold=-1.0),
                dict(min_opacity=float("nan")), dict(extent=0.0), dict(percent_dense=float("inf")), dict(seed=True)):
        with pytest.raises(ValueError, match="DensifyConfig"):
            pr.DensifyConfig(**bad)


def test_header_rewrite_changes_only_the_count(tmp_path):
    from pixelsplat_b200 import ply_import as pi
    names = f64.gs_properties(2) + ["filter_3D"]
    rec = np.zeros((37, len(names)), np.float32)
    src = f64.write_ply(tmp_path / "in.ply", names, rec, extra_header="comment element vertex 5 in a comment\n")
    data = src.read_bytes()
    layout = pi.parse_header(data)
    head = data[:layout.body_offset]
    for count in (37, 1, 36, 38, 1234567):
        new = pr.rewrite_vertex_count(head, count)
        assert pi.parse_header(new + b"\0" * 4).count == count
        assert new.replace(b"element vertex %d\n" % count, b"") == head.replace(b"element vertex 37\n", b"")
    assert pr.rewrite_vertex_count(head, 37) == head


def test_refine_ply_arguments_default_to_no_densification():
    from pixelsplat_b200.evaluation import __main__ as cli
    base = ["--ply", "p", "--dataset-root", "d", "--index", "i", "--output", "o"]
    assert cli.parse_refine_ply(base).densify is None
    a = cli.parse_refine_ply(base + ["--densify-until", "800"])
    assert a.densify == pr.DensifyConfig(until_step=800)
    a = cli.parse_refine_ply(base + ["--steps", "1000", "--densify-from", "100", "--densify-until", "800",
                                     "--densify-every", "50", "--densify-grad", "1e-3", "--min-opacity", "0.01",
                                     "--opacity-reset-every", "0", "--densify-seed", "7"])
    assert a.densify == pr.DensifyConfig(from_step=100, until_step=800, every=50, grad_threshold=1e-3,
                                         min_opacity=0.01, opacity_reset_every=0, seed=7)
    for bad in (["--densify-until", "-1"], ["--densify-until", "10", "--densify-every", "0"],
                ["--densify-grad", "nan"], ["--min-opacity", "-0.1"]):
        with pytest.raises(SystemExit):
            cli.parse_refine_ply(base + bad)


# ---- ABI


def test_densify_desc_layout_matches_the_header(tmp_path):
    import subprocess
    root = Path(__file__).resolve().parents[1]
    fields = ("n_props", "prune_world", "col_xyz", "col_opacity", "col_scale", "col_rot", "grad_threshold",
              "percent_dense", "min_opacity", "extent")
    src = tmp_path / "probe.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "pixelsplat_b200.h"\n'
                   'int main(void){printf("%zu' + " %zu" * len(fields) + '\\n", sizeof(ps_ply_densify_desc)'
                   + "".join(f", offsetof(ps_ply_densify_desc, {f})" for f in fields) + ');return 0;}\n')
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", str(root / "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    d = _lib.PlyDensifyDesc
    assert got == [ctypes.sizeof(d)] + [getattr(d, f).offset for f in fields]


def _desc(**kw):
    d = _lib.PlyDensifyDesc(n_gaussians=1000, n_props=62, prune_world=0, col_opacity=54, grad_threshold=2e-4,
                            percent_dense=0.01, min_opacity=0.005, extent=1.0)
    d.col_xyz[:] = [0, 1, 2]
    d.col_scale[:] = [55, 56, 57]
    d.col_rot[:] = [58, 59, 60, 61]
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_workspace_is_closed_form():
    for n in (1, 63, 64, 65, 4133, 393_216):
        got = ctypes.c_size_t()
        assert _lib.lib.ps_ply_densify_workspace_bytes(n, ctypes.byref(got)) == 0
        assert got.value == pr.densify_workspace_bytes(n) == (n + 15) // 16 * 16 + 24 * ((n + 63) // 64)
    assert _lib.lib.ps_ply_densify_workspace_bytes(0, ctypes.byref(got)) == 1


def test_densify_entry_points_refuse_bad_arguments_before_launching():
    ws = pr.densify_workspace_bytes(1000)
    before = _lib.lib.ps_launch_count()

    def refused(who, *args):
        rc = getattr(_lib.lib, who)(*args)
        assert rc == 1, rc
        msg = _lib.lib.ps_last_error().decode()
        assert msg.startswith(who + ": "), msg
        return msg

    def count(d, *, records=256, accum=512, cnt=768, wsp=1024, ws_bytes=ws, counts=2048):
        return refused("ps_ply_densify_count", None if d is None else ctypes.byref(d), records, accum, cnt, wsp,
                       ws_bytes, counts, None)

    def apply(d, *, records=256, m=512, v=768, eps=1024, wsp=1280, ws_bytes=ws, counts=1536, out=2048, mo=2304,
              vo=2560):
        return refused("ps_ply_densify_apply", ctypes.byref(d), records, m, v, eps, wsp, ws_bytes, counts, out, mo,
                       vo, None)

    assert "desc is NULL" in count(None)
    assert "n_gaussians 0 < 1" in count(_desc(n_gaussians=0))
    assert "n_props 257 outside [1, 256]" in count(_desc(n_props=257))
    assert "col_rot[3] = 62 outside [0, n_props = 62)" in count(_desc(col_rot=(ctypes.c_int32 * 4)(58, 59, 60, 62)))
    assert "col_opacity[0] = -1 outside" in count(_desc(col_opacity=-1))
    for name in ("grad_threshold", "percent_dense", "min_opacity", "extent"):
        assert f"{name} -1 is negative or not finite" in count(_desc(**{name: -1.0}))
        assert f"{name} nan is negative or not finite" in count(_desc(**{name: math.nan}))
        assert f"{name} inf is negative or not finite" in count(_desc(**{name: math.inf}))
    assert "extent 0 is not positive" in count(_desc(extent=0.0))
    assert "workspace is NULL" in count(_desc(), wsp=None)
    assert "not 16-byte aligned" in count(_desc(), wsp=1028)
    assert f"workspace of {ws - 1} bytes, {ws} needed" in count(_desc(), ws_bytes=ws - 1)
    assert "records is NULL or misaligned" in count(_desc(), records=260)
    assert "accum is NULL or misaligned" in count(_desc(), accum=None)
    assert "count is NULL or misaligned" in count(_desc(), cnt=769)
    assert "counts is NULL or misaligned" in count(_desc(), counts=2052)
    assert "extent -1 is negative" in apply(_desc(extent=-1.0))
    assert f"workspace of 0 bytes" in apply(_desc(), ws_bytes=0)
    for name, bad in (("records", dict(records=264)), ("exp_avg", dict(m=None)), ("exp_avg_sq", dict(v=776)),
                      ("eps", dict(eps=None)), ("counts", dict(counts=1540)), ("records_out", dict(out=2052)),
                      ("exp_avg_out", dict(mo=None)), ("exp_avg_sq_out", dict(vo=2568))):
        assert f"{name} is NULL or misaligned" in apply(_desc(), **bad)
    stats = lambda n, v, *p: refused("ps_ply_densify_stats", n, v, *p, None)
    assert "n_gaussians 0 or n_views 2 < 1" in stats(0, 2, 256, 512, 768, 1024)
    assert "n_views 0 < 1" in stats(10, 0, 256, 512, 768, 1024)
    for i, name in enumerate(("d_means2d", "radii", "accum", "count")):
        ptrs = [256, 512, 768, 1024]
        ptrs[i] = None
        assert f"{name} is NULL or misaligned" in stats(10, 2, *ptrs)
        ptrs[i] = 1026
        assert f"{name} is NULL or misaligned" in stats(10, 2, *ptrs)
    assert _lib.lib.ps_launch_count() == before
