"""CPU tests of the boundary: the C-ABI library loads, exports every symbol include/*.h declares,
its structs agree with the ctypes mirrors, argument validation works without a GPU, and the
product path fails loudly (no fallback) when the library or the device is missing."""
import ctypes
import os
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
HEADER = ROOT / "include" / "pixelsplat_b200.h"


def declared_functions():
    text = HEADER.read_text()
    return sorted(set(re.findall(r"PS_API\s+[\w\s\*]+?\b(ps_\w+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from pixelsplat_b200 import _lib
    names = declared_functions()
    assert len(names) >= 10
    for n in names:
        assert hasattr(_lib.lib, n), f"{n} declared in the header but not exported"
    assert set(_lib.EXPORTS) == set(names)
    assert _lib.lib.ps_version() >= 100


def test_ctypes_structs_match_the_header(tmp_path):
    """Compile a C probe against the header with gcc and compare sizeof/offsetof."""
    from pixelsplat_b200 import _lib
    probe = tmp_path / "probe.c"
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pixelsplat_b200.h"\n'
                     "int main(void){printf(\"%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n\","
                     "sizeof(ps_raster_desc),offsetof(ps_raster_desc,instance_capacity),"
                     "sizeof(ps_raster_inputs),sizeof(ps_raster_state),sizeof(ps_raster_sizes),"
                     "sizeof(ps_raster_layout),sizeof(ps_raster_grads),offsetof(ps_raster_desc,sort_impl),"
                     "sizeof(ps_epipolar_desc),sizeof(ps_epipolar_inputs),sizeof(ps_adapter_desc),"
                     "offsetof(ps_adapter_desc,scale_min),sizeof(ps_adapter_inputs));return 0;}\n")
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", str(HEADER.parent), str(probe), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [ctypes.sizeof(_lib.RasterDesc), _lib.RasterDesc.instance_capacity.offset,
            ctypes.sizeof(_lib.RasterInputs), ctypes.sizeof(_lib.RasterState),
            ctypes.sizeof(_lib.RasterSizes), ctypes.sizeof(_lib.RasterLayout),
            ctypes.sizeof(_lib.RasterGrads), _lib.RasterDesc.sort_impl.offset,
            ctypes.sizeof(_lib.EpipolarDesc), ctypes.sizeof(_lib.EpipolarInputs), ctypes.sizeof(_lib.AdapterDesc),
            _lib.AdapterDesc.scale_min.offset, ctypes.sizeof(_lib.AdapterInputs)]
    assert got == want


def test_sizes_layout_and_validation_without_gpu():
    from pixelsplat_b200 import _lib
    d = _lib.RasterDesc(2, 3, 1000, 25, 4, _lib.PS_SH_3M, _lib.PS_COV_3X3, 70, 50, 0, 0, 12345)
    s, lay = _lib.sizes(d), _lib.layout(d)
    vp, tiles = 2 * 3 * 1000, 4 * 5
    assert lay.depth == 0 and lay.radii >= vp * 4 and lay.keys == 0 and lay.keys_alt >= 12345 * 8
    assert s.binning_bytes >= 2 * 12345 * 8 and s.image_bytes >= 2 * 6 * 70 * 50 * 4
    assert s.backward_bytes >= vp * 40
    offs = [getattr(lay, f) for f, _ in _lib.RasterLayout._fields_[:13]]
    assert offs == sorted(offs) and all(o % 256 == 0 for o in offs)
    assert lay.tile_start - lay.tile_count >= 6 * tiles * 4
    for field, bad in (("n_gaussians", 0), ("sh_degree", 5), ("sh_coeffs", 26), ("sh_layout", 7),
                       ("cov_layout", -1), ("height", 0), ("instance_capacity", 0),
                       ("instance_capacity", 1 << 31)):
        d2 = _lib.RasterDesc(1, 1, 10, 25, 4, 0, 0, 16, 16, 0, 0, 100)
        setattr(d2, field, bad)
        with pytest.raises(ValueError, match="PS_ERR_INVALID_ARGUMENT"):
            _lib.sizes(d2)
    d3 = _lib.RasterDesc(1, 1, 10, 4, 2, 0, 0, 16, 16, 0, 0, 100)    # degree 2 needs 9 coefficients
    with pytest.raises(ValueError, match="needs 9 coefficients"):
        _lib.sizes(d3)
    # NULL pointers are rejected before anything is launched
    d4 = _lib.RasterDesc(1, 1, 10, 25, 4, 0, 0, 16, 16, 0, 0, 100)
    rc = _lib.lib.ps_raster_forward(ctypes.byref(d4), None, None, None, None, None, None)
    assert rc == 1 and b"NULL" in _lib.lib.ps_last_error()


def test_hit_list_option_without_gpu():
    """ps_set_option("composite_hit_lists", 0 | 1 | 2) decides whether the binning state holds the forward's hit
    lists: 2 (automatic) keeps them while 64 bytes x capacity <= 512 MB; other values are rejected."""
    from pixelsplat_b200 import _lib
    small = _lib.RasterDesc(1, 1, 1000, 25, 4, 0, 0, 256, 256, 0, 0, 100_000)
    big = _lib.RasterDesc(1, 1, 1000, 25, 4, 0, 0, 256, 256, 0, 0, (512 << 20) // 64 + 1)
    try:
        for bad in (-1, 3, 4):
            with pytest.raises(ValueError, match="PS_ERR_INVALID_ARGUMENT.*unknown option or bad value: "
                                                 f"composite_hit_lists = {bad}"):
                _lib.set_option("composite_hit_lists", bad)
        binning, hits = {}, {}
        for v in (0, 1, 2):
            _lib.set_option("composite_hit_lists", v)
            binning[v] = {n: _lib.sizes(d).binning_bytes for n, d in (("small", small), ("big", big))}
            hits[v] = {n: _lib.layout(d).block_hits for n, d in (("small", small), ("big", big))}
        assert binning[0]["small"] < binning[1]["small"] == binning[2]["small"]
        assert binning[0]["big"] == binning[2]["big"] < binning[1]["big"]
        assert binning[1]["small"] - binning[0]["small"] >= 100_000 * 64
        assert hits[0] == {"small": 0, "big": 0} and hits[2]["small"] != 0 and hits[2]["big"] == 0
        assert hits[1]["small"] != 0 and hits[1]["big"] != 0
        _lib.set_option("composite_impl", 1)          # the legacy compositor never keeps them
        assert _lib.layout(small).block_hits == 0
    finally:
        _lib.set_option("composite_impl", 2)
        _lib.set_option("composite_hit_lists", 2)
    assert _lib.layout(small).block_hits != 0


def test_no_cpu_fallback():
    """CPU tensors are rejected; a missing library is an ImportError, not a silent fallback."""
    from pixelsplat_b200.rasterizer import rasterize_gaussians
    P = 8
    with pytest.raises(ValueError, match="CUDA tensor"):
        rasterize_gaussians(torch.zeros(1, P, 3), torch.zeros(1, P, 6), torch.zeros(1, P),
                            torch.zeros(1, P, 25, 3), viewmatrix=torch.zeros(1, 16),
                            projmatrix=torch.zeros(1, 16), campos=torch.zeros(1, 3),
                            tanfov=torch.ones(1, 2), background=torch.zeros(1, 3), image_shape=(16, 16),
                            views_per_scene=1, sh_degree=4)
    env = dict(os.environ, PIXELSPLAT_B200_LIB="/nonexistent/libpixelsplat_b200.so")
    r = subprocess.run([sys.executable, "-c", "import pixelsplat_b200.rasterizer"], cwd=str(ROOT), env=env,
                       capture_output=True, text=True)
    assert r.returncode != 0 and "no CPU fallback" in r.stderr


def test_product_never_imports_the_oracle():
    """No file of the product imports, includes, links or loads anything under oracle/."""
    pat = re.compile(r"(^|\s)(import\s+oracle|from\s+oracle)|#include\s*[<\"][^>\"]*oracle|liboracle|oracle/_build|"
                     r"raster_oracle|raster_torch|epipolar_ref")
    for path in (ROOT / "pixelsplat_b200").rglob("*"):
        if path.suffix in (".py", ".cu", ".cuh", ".h") or path.name == "Makefile":
            assert not pat.search(path.read_text()), path
    assert not pat.search((ROOT / "diff_gaussian_rasterization" / "__init__.py").read_text())


def test_synthetic_scenes_are_deterministic():
    from pixelsplat_b200 import synthetic
    a, b = synthetic.scene_re10k_like(seed=3, image_hw=(32, 32)), synthetic.scene_re10k_like(seed=3, image_hw=(32, 32))
    assert torch.equal(a.means, b.means) and torch.equal(a.harmonics, b.harmonics)
    assert a.num_gaussians == 2 * 32 * 32 * 3 and a.harmonics.shape[-2:] == (3, 25)
    assert abs(float(synthetic.scene_re10k_like(seed=0).near[0]) - 0.2933) < 1e-3
    evals = torch.linalg.eigvalsh(a.covariances)
    assert (evals > 0).all()


def test_loss_module_matches_the_reference_formulas():
    """pixelsplat_b200.loss on CPU tensors (pure torch): LossMse == weight * mean(delta^2), compute_psnr clips to
    [0, 1] first, and the from-sums forms give the same numbers (loss_mse.py:30-31, metrics.py:11-19)."""
    from pixelsplat_b200 import loss as L
    g = torch.Generator().manual_seed(0)
    pred = torch.rand(2, 3, 3, 8, 10, generator=g) * 1.5 - 0.25
    tgt = torch.rand(2, 3, 3, 8, 10, generator=g)
    m = L.LossMse(L.LossMseCfgWrapper(L.LossMseCfg(0.5)))
    out = type("O", (), {"color": pred})()
    want = 0.5 * ((pred - tgt) ** 2).mean()
    assert torch.allclose(m(out, {"target": {"image": tgt}}), want) and m.name == "mse"
    sse = ((pred - tgt) ** 2).sum(dim=(2, 3, 4))
    assert torch.allclose(m.from_sse(sse, (8, 10)), want)
    psnr = L.compute_psnr(tgt.flatten(0, 1), pred.flatten(0, 1))
    sse_c = ((pred.clip(0, 1) - tgt.clip(0, 1)) ** 2).sum(dim=(2, 3, 4))
    assert torch.allclose(L.psnr_from_sse(sse_c, (8, 10)).flatten(), psnr, atol=1e-5)


def test_bench_roofline_object_is_built_from_the_profile_file():
    """bench.py's `roofline` (a pure function of the stage times and profiles/kernel_metrics_V1.json): traffic and
    issue_frac come from the profile of the SAME CUDA sources, never from a literal; a stale or missing profile
    yields nulls, not a crash."""
    import json as _json
    import bench
    stage = {"preprocess": 0.032, "count_scan_scatter": 0.030, "tile_sort": 0.030, "composite_fwd": 0.069,
             "grad_zero_fill": 0.019, "composite_bwd": 0.080, "preprocess_bwd": 0.049}
    r = bench.build_roofline(stage, 1, 393216, 399057.0, 125628.0, 65536, standard_workload=True)
    assert r["kernel"] == "composite_bwd" and r["unit"] == "GB/s" and 0 < r["frac"] < 1
    assert r["algorithmic_bytes_per_launch"] == 399057 * (48 + 36) + 65536 * 20
    prof_path = ROOT / "profiles" / "kernel_metrics_V1.json"
    prof = _json.loads(prof_path.read_text()) if prof_path.exists() else None
    if prof is None:        # no profile of this build stored: nothing from it is reported, and the note says why
        assert r["traffic"] is None and r["issue_frac"] is None and "absent" in r["profile"]
    elif prof["csrc_sha"] == bench.csrc_sha():
        kp = prof["k_composite_bwd2"]
        assert r["traffic"] == kp["dram_bytes"] and r["bound"] == "issue"
        assert abs(r["issue_frac"] - kp["warp_inst"] / 0.080e-3 / bench.ISSUE_PEAK) < 1e-12 and 0 < r["issue_frac"] < 1
    else:   # sources changed after the capture: ignored, says so
        assert r["traffic"] is None and r["issue_frac"] is None and "ignored" in r["profile"]
    r2 = bench.build_roofline(stage, 4, 393216, 490518.0, 154705.0, 65536, standard_workload=False)
    assert r2["traffic"] is None and r2["bound"] == "hbm"
    _json.dumps(r), _json.dumps(r2)


def test_launch_list_summary_writes_the_profile_bench_reads(tmp_path):
    """tools/summarize_launches.py --json: kernel names are normalised (`void ps::k_composite_bwd2<4>(...)` ->
    `k_composite_bwd2`), per-launch means are taken, and the CUDA-source hash is the one bench.py computes."""
    import json as _json
    import bench
    rows = ['"ID","Process ID","Process Name","Host Name","Kernel Name","Context","Stream","Block Size","Grid Size",'
            '"Device","CC","Section Name","Metric Name","Metric Unit","Metric Value"']

    def launch(i, name, ns, inst, rd, wr):
        for m, u, v in (("gpu__time_duration.sum", "ns", ns), ("smsp__inst_executed.sum", "inst", inst),
                        ("dram__bytes_read.sum", "byte", rd), ("dram__bytes_write.sum", "byte", wr)):
            rows.append(f'"{i}","1","python","h","{name}","1","7","(128, 1, 1)","(10, 1, 1)","0","10.0","s","{m}","{u}","{v}"')

    launch(0, "void ps::k_composite_bwd2<4>(ps::Dims, ps::Geom)", "70,000", "35,000,000", "36,000,000", "1,000")
    launch(1, "void ps::k_composite_bwd2<4>(ps::Dims, ps::Geom)", "72,000", "35,000,000", "36,000,000", "3,000")
    launch(2, "ps::k_preprocess(ps::Dims, ps::Inputs, ps::Geom, int)", "26,000", "9,000,000", "20,000,000", "4,000,000")
    launch(3, "void at::native::vectorized_elementwise_kernel<4>(int)", "3,000", "100", "0", "0")
    csv_path, out = tmp_path / "launches.csv", tmp_path / "metrics.json"
    csv_path.write_text("==PROF== header line\n" + "\n".join(rows) + "\n")
    subprocess.run([sys.executable, str(ROOT / "tools" / "summarize_launches.py"), str(csv_path), "0", "--json", str(out)],
                   check=True, capture_output=True)
    d = _json.loads(out.read_text())
    assert d["csrc_sha"] == bench.csrc_sha() and set(k for k in d if k.startswith("k_")) == {"k_composite_bwd2", "k_preprocess"}
    kb = d["k_composite_bwd2"]
    assert kb["launches"] == 2 and abs(kb["us"] - 71.0) < 1e-9 and kb["warp_inst"] == 35e6 and kb["dram_bytes"] == 36002000.0
