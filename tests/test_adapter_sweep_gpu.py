"""The fused Gaussian adapter kernels (csrc/gaussian_adapter.cu: k_gaussian_adapter_fwd / _bwd) at the C ABI, against
the float64 restatement tests/adapter_f64.py with its per-entry bars, across the descriptor space the ABI accepts.

  1. Every sh_coeffs (1, 4, 9, 16, 25) x n_samples 1..8 at 3 views x 161 rays: two 128-ray blocks per view, the
     second with one full warp, one warp holding a single ray and two warps past n_rays.
  2. n_rays 1, 31, 32, 33, 127, 128, 129, 255, 257, 1000, 4133 at (sh 25, spp 3) and (sh 4, spp 1), each with 1, 2 and
     14 views.  With sh 4 the gradient rows are an odd 19 floats, so unstage_sh_rows takes its float4 branch where
     view * n_rays is a multiple of 4 and its scalar one elsewhere; both are reached (asserted below).  Plus one call
     at the real per-view ray count, 2 views x 65536 rays (256 x 256), sh 25, spp 3.
  3. Inputs: random SO(3) cameras with origins off the axes; skewed, non-square and generic (non-zero bottom row)
     intrinsics; coordinates in [-0.5, 1.5]; depths from near to far (covariance traces over 1e5 apart); scale ranges
     other than 0.5 / 15; non-square, 1 x N and N x 1 images; scale logits of +-30; and, in calls of their own, zero
     and ~eps-norm raw quaternions (their d_raw is ~1 / eps times the other rays').  The cotangents are normalised per
     Gaussian (d_cov by the float64 trace, d_scales by the mean scale) so that no Gaussian's gradient hides under
     another's.
  4. Optional pointers: NULL scales / rotations leave means, covariances and harmonics bit-identical; NULL d_scales /
     d_rotations give the bits of zero tensors.
  5. Canaries: outputs and gradients in NaN-filled oversized buffers (every in-range entry written, equal to the normal
     call, the tails untouched); inputs in front of tails of NaN and of 3e38 (same bits both ways).
  6. Repeatability: one launch per direction, two runs give the same bits.
  7. The module path: srf = 2, extrinsics, intrinsics and coordinates broadcast over the batch; and with
     materialize_grads off, a training-shaped loss gives the same bits whether or not scales and rotations carry a
     (zero) gradient, at one backward launch.

Measured on an NVIDIA H100 80GB HBM3: see DESIGN.md section 9 "Parity" for the worst ratio of each bar.
"""
import ctypes
import math

import pytest
import torch

from tests import adapter_f64 as af

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

SH = (1, 4, 9, 16, 25)
GRID = [(n_sh, spp) for n_sh in SH for spp in range(1, 9)]
RAYS = (1, 31, 32, 33, 127, 128, 129, 255, 257, 1000, 4133)
RAGGED = [(nv, nr, n_sh, spp) for n_sh, spp in ((25, 3), (4, 1)) for nv in (1, 2, 14) for nr in RAYS]
IMAGES = ((48, 64), (1, 37), (256, 256), (29, 1), (360, 640))
SCALE_RANGES = ((0.5, 15.0), (0.05, 3.0), (1.0, 40.0))
EPS = 1e-8


class Case:
    """One ABI call: float32 device inputs exactly as the kernel reads them, and per-Gaussian normalised cotangents."""

    def __init__(self, nv, nr, ns, n_sh, seed, degenerate=False):
        from pixelsplat_b200 import sh
        from pixelsplat_b200.encoder.gaussian_adapter import quaternion_to_matrix
        g = torch.Generator().manual_seed(seed)
        U = lambda *s: torch.rand(s, generator=g, dtype=torch.float64)
        N = lambda *s: torch.randn(s, generator=g, dtype=torch.float64)
        self.nv, self.nr, self.ns, self.n_sh = nv, nr, ns, n_sh
        self.h, self.w = IMAGES[seed % len(IMAGES)]
        self.smin, self.smax = SCALE_RANGES[seed % len(SCALE_RANGES)]
        q = N(nv, 4)
        E = torch.eye(4, dtype=torch.float64).repeat(nv, 1, 1)
        E[:, :3, :3] = quaternion_to_matrix(q / q.norm(dim=-1, keepdim=True), eps=0.0)
        E[:, :3, 3] = 3.0 * N(nv, 3)
        K = torch.zeros(nv, 3, 3, dtype=torch.float64)
        for v in range(nv):
            fx, fy = 0.6 + 0.8 * float(U(1)), 0.6 + 0.8 * float(U(1))
            kind = (seed + v) % 3
            if kind == 1:                                         # non-square pixels
                fy = 0.35 * fx
            K[v] = torch.tensor([[fx, 0.0, float(U(1))], [0.0, fy, float(U(1))], [0.0, 0.0, 1.0]], dtype=torch.float64)
            if kind != 1:                                         # skew
                K[v, 0, 1] = 0.15 * (float(U(1)) - 0.5)
            if kind == 2:                                         # generic: every entry perturbed
                K[v] += 0.04 * (U(3, 3) - 0.5)
        coords = -0.5 + 2.0 * U(nv, nr, 2)
        near, far = 0.3, 120.0
        depths = 1.0 / (U(nv, nr, ns) * (1 / near - 1 / far) + 1 / far)
        depths.view(-1)[0] = near
        depths.view(-1)[-1] = far
        raw = N(nv, nr, 7 + 3 * n_sh)
        raw[..., :3] *= 3.0
        sat = torch.arange(nr) % 7 == 3
        raw[:, sat, seed % 3] = 30.0
        raw[:, sat, (seed + 1) % 3] = -30.0
        r = torch.arange(nr)
        self.zero_q = (r % 5 == 1) if degenerate else torch.zeros(nr, dtype=torch.bool)
        if degenerate:
            raw[:, self.zero_q, 3:7] = 0.0
            tiny = r % 5 == 3
            qt = N(nv, int(tiny.sum()), 4)
            raw[:, tiny, 3:7] = qt / qt.norm(dim=-1, keepdim=True) * EPS * (0.5 + 1.5 * U(nv, int(tiny.sum()), 1))
        f = lambda t: t.float().contiguous().to(DEV)
        self.E, self.K, self.coords, self.depths, self.raw = f(E), f(K), f(coords), f(depths), f(raw)
        self.D = sh.camera_sh_rotations(self.E, af.sh_degree(n_sh), ("e3nn", "3dgs")[seed % 2]).contiguous()
        self.mask = af.sh_mask(n_sh).float().to(DEV)
        with torch.no_grad():
            fwd = af.forward(*self.ref_args())
        trace = fwd["covariances"].diagonal(dim1=-2, dim2=-1).sum(-1)
        mean_scale = fwd["scales"].mean(-1)
        gd = torch.Generator(device=DEV).manual_seed(seed)
        R = lambda *s: torch.randn(s, generator=gd, device=DEV, dtype=torch.float64)
        self.cot = {k: v.float().contiguous() for k, v in dict(
            d_means=R(nv, nr, ns, 3), d_cov=R(nv, nr, ns, 3, 3) / trace[..., None, None],
            d_harm=R(nv, nr, ns, 3, n_sh), d_scales=R(nv, nr, ns, 3) / mean_scale[..., None],
            d_rot=R(nv, nr, 4)).items()}

    def ref_args(self):
        return (self.E, self.K, self.D, self.mask, self.coords, self.depths, self.raw, (self.h, self.w),
                af.widen(self.smin), af.widen(self.smax), af.widen(EPS))

    def reference(self, cot=None):
        return af.forward_backward(*self.ref_args(), self.cot if cot is None else cot)

    def desc(self):
        from pixelsplat_b200 import _lib
        return _lib.AdapterDesc(self.nv, self.nr, self.ns, self.n_sh, self.h, self.w, self.smin, self.smax, EPS, 0)

    def inputs(self, **override):
        from pixelsplat_b200 import _lib
        t = dict(extrinsics=self.E, intrinsics=self.K, sh_rotation=self.D, sh_mask=self.mask, coordinates=self.coords,
                 depths=self.depths, raw=self.raw)
        t.update(override)
        return _lib.AdapterInputs(*[t[k].data_ptr() for k in ("extrinsics", "intrinsics", "sh_rotation", "sh_mask",
                                                              "coordinates", "depths", "raw")])

    def out_shapes(self):
        nv, nr, ns, n = self.nv, self.nr, self.ns, self.n_sh
        return dict(means=(nv, nr, ns, 3), covariances=(nv, nr, ns, 3, 3), harmonics=(nv, nr, ns, 3, n),
                    scales=(nv, nr, ns, 3), rotations=(nv, nr, 4), d_coordinates=(nv, nr, 2),
                    d_depths=(nv, nr, ns), d_raw=(nv, nr, 7 + 3 * n))


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def kernel_forward(c: Case, outs=None, scales=True, rotations=True, ins=None) -> dict:
    from pixelsplat_b200 import _lib
    shp = c.out_shapes()
    outs = outs if outs is not None else {k: torch.empty(shp[k], device=DEV) for k in af.OUTPUTS}
    desc, inputs = c.desc(), ins if ins is not None else c.inputs()
    rc = _lib.lib.ps_gaussian_adapter_forward(ctypes.byref(desc), ctypes.byref(inputs), _p(outs["means"]),
                                              _p(outs["covariances"]), _p(outs["harmonics"]),
                                              _p(outs["scales"]) if scales else None,
                                              _p(outs["rotations"]) if rotations else None, _stream())
    _lib.check(rc, "ps_gaussian_adapter_forward")
    return outs


def kernel_backward(c: Case, cot=None, outs=None, ins=None) -> dict:
    """cot: the case's cotangents unless given; a None d_scales / d_rot is passed as NULL."""
    from pixelsplat_b200 import _lib
    cot = c.cot if cot is None else cot
    shp = c.out_shapes()
    outs = outs if outs is not None else {k: torch.empty(shp[k], device=DEV) for k in af.GRADIENTS}
    desc, inputs = c.desc(), ins if ins is not None else c.inputs()
    rc = _lib.lib.ps_gaussian_adapter_backward(
        ctypes.byref(desc), ctypes.byref(inputs), _p(cot["d_means"]), _p(cot["d_cov"]), _p(cot["d_harm"]),
        _p(cot.get("d_scales")), _p(cot.get("d_rot")), _p(outs["d_coordinates"]), _p(outs["d_depths"]),
        _p(outs["d_raw"]), _stream())
    _lib.check(rc, "ps_gaussian_adapter_backward")
    return outs


def run(c: Case) -> dict:
    return {**kernel_forward(c), **kernel_backward(c)}


def _check_case(c: Case, tag: str):
    got = run(c)
    ref = c.reference()
    af.check(got, ref, tag)


@pytest.mark.parametrize("n_sh,spp", GRID, ids=[f"sh{n}-spp{s}" for n, s in GRID])
def test_two_blocks_per_view(n_sh, spp):
    seed = GRID.index((n_sh, spp))
    _check_case(Case(3, 161, spp, n_sh, seed), f"sh{n_sh}-spp{spp}")


@pytest.mark.parametrize("nv,nr,n_sh,spp", RAGGED, ids=[f"v{v}-r{r}-sh{n}-spp{s}" for v, r, n, s in RAGGED])
def test_ragged_ray_counts(nv, nr, n_sh, spp):
    seed = 100 + RAGGED.index((nv, nr, n_sh, spp))
    _check_case(Case(nv, nr, spp, n_sh, seed), f"v{nv}-r{nr}-sh{n_sh}-spp{spp}")


def test_ragged_sweep_reaches_both_unstage_branches():
    """unstage_sh_rows copies float4s when the padded row stride equals the row (7 + 3 sh_coeffs odd: sh 4 and 16) and
    the warp's d_raw run starts 16-byte aligned, i.e. (view * n_rays + first ray) * 19 floats is a multiple of 4."""
    vec = scalar = 0
    for nv, nr, n_sh, _ in RAGGED:
        if (7 + 3 * n_sh) % 2 == 1:
            for v in range(nv):
                for ray0 in range(0, nr, 32):
                    if (v * nr + ray0) % 4 == 0:
                        vec += 1
                    else:
                        scalar += 1
    assert vec > 0 and scalar > 0, (vec, scalar)


def test_full_resolution_view():
    _check_case(Case(2, 65536, 3, 25, 7), "v2-r65536-sh25-spp3")


@pytest.mark.parametrize("n_sh", [4, 25])
def test_zero_and_eps_norm_quaternions(n_sh):
    """Every fifth ray has a zero raw quaternion (the kernel's corr = 0 branch: d_raw = d_rot / eps there) and every
    fifth an ~eps-norm one; their quaternion gradients are ~1 / eps times the other rays', so this call's S for those
    components is theirs (the other rays' quaternion gradients are held by every other case)."""
    c = Case(2, 161, 3, n_sh, 51, degenerate=True)
    got = run(c)
    af.check(got, c.reference(), f"degenerate-sh{n_sh}")
    z = c.zero_q.to(DEV)
    assert not got["rotations"][:, z].any()
    want = c.cot["d_rot"][:, z].double() / af.widen(EPS)
    assert float(((got["d_raw"][:, z, 3:7].double() - want).abs() / want.abs()).max()) < 1e-6


@pytest.mark.parametrize("n_sh", [4, 25])
def test_null_optional_pointers(n_sh):
    c = Case(3, 161, 3, n_sh, 11)
    full = kernel_forward(c)
    for scales, rotations in ((False, True), (True, False), (False, False)):
        got = kernel_forward(c, scales=scales, rotations=rotations)
        for k in ("means", "covariances", "harmonics"):
            assert torch.equal(got[k], full[k]), (k, scales, rotations)
    zeros = dict(c.cot, d_scales=torch.zeros_like(c.cot["d_scales"]), d_rot=torch.zeros_like(c.cot["d_rot"]))
    want = kernel_backward(c, zeros)
    for drop in (("d_scales",), ("d_rot",), ("d_scales", "d_rot")):
        cot = {k: (None if k in drop else v) for k, v in zeros.items()}
        got = kernel_backward(c, cot)
        for k in af.GRADIENTS:
            assert torch.equal(got[k].view(torch.int32), want[k].view(torch.int32)), (k, drop)
    # ... and the NULL call is the float64 gradient of the loss without those two terms
    cot = dict(c.cot, d_scales=None, d_rot=None)
    af.check({**full, **kernel_backward(c, cot)}, c.reference(cot), f"null-sh{n_sh}")


def _padded(shape, fill, tail=1024):
    n = math.prod(shape)
    buf = torch.full((n + tail,), fill, device=DEV)
    return buf, buf[:n].view(shape)


@pytest.mark.parametrize("nr,n_sh", [(161, 4), (161, 25), (128, 16), (33, 9)])
def test_every_output_written_once_and_nothing_past_it(nr, n_sh):
    """Outputs and gradients in NaN-filled buffers 1024 floats too long: every in-range entry is written and equals the
    normal call, and the tails keep their NaN bits.  Inputs in front of 1024 floats of NaN, then of 3e38: the kernels
    read nothing past an input's end (the results have the same bits both ways)."""
    c = Case(2, nr, 3, n_sh, 21)
    want = run(c)
    bufs = {k: _padded(tuple(v.shape), float("nan")) for k, v in want.items()}
    kernel_forward(c, outs={k: bufs[k][1] for k in af.OUTPUTS})
    kernel_backward(c, outs={k: bufs[k][1] for k in af.GRADIENTS})
    torch.cuda.synchronize()
    for k, (buf, view) in bufs.items():
        assert torch.equal(view.view(torch.int32), want[k].view(torch.int32)), k
        assert bool(torch.isfinite(view).all()), k
        assert bool(torch.isnan(buf[view.numel():]).all()), (k, "a write past the end")
    runs = []
    for fill in (float("nan"), 3e38):
        held = []

        def tailed(t):
            buf, view = _padded(tuple(t.shape), fill)
            view.copy_(t)
            held.append(buf)
            return view
        ins = c.inputs(**{k: tailed(t) for k, t in dict(extrinsics=c.E, intrinsics=c.K, sh_rotation=c.D,
                                                         sh_mask=c.mask, coordinates=c.coords, depths=c.depths,
                                                         raw=c.raw).items()})
        cot = {k: tailed(t) for k, t in c.cot.items()}
        runs.append({**kernel_forward(c, ins=ins), **kernel_backward(c, cot, ins=ins)})
        torch.cuda.synchronize()
    for k in want:
        assert torch.equal(runs[0][k].view(torch.int32), runs[1][k].view(torch.int32)), k
        assert torch.equal(runs[0][k].view(torch.int32), want[k].view(torch.int32)), k


def test_repeatable_bits_one_launch_per_direction():
    from pixelsplat_b200 import _lib
    c = Case(14, 4133, 3, 25, 31)
    first = run(c)
    torch.cuda.synchronize()
    l0 = _lib.lib.ps_launch_count()
    fwd = kernel_forward(c)
    torch.cuda.synchronize()
    l1 = _lib.lib.ps_launch_count()
    bwd = kernel_backward(c)
    torch.cuda.synchronize()
    assert (l1 - l0, _lib.lib.ps_launch_count() - l1) == (1, 1)
    for k, v in {**fwd, **bwd}.items():
        assert torch.equal(v.view(torch.int32), first[k].view(torch.int32)), k


def _module_call(b=2, v=2, r=37, srf=2, spp=3, seed=41):
    """GaussianAdapter.forward with extrinsics, intrinsics and coordinates broadcast over the batch: the module's
    outputs and leaves, and the same call at the ABI (a Case over b * v views) for the float64 reference."""
    from pixelsplat_b200.encoder.gaussian_adapter import GaussianAdapter, GaussianAdapterCfg
    c = Case(v, r * srf, spp, 25, seed)
    c.smin, c.smax = 0.5, 15.0
    ad = GaussianAdapter(GaussianAdapterCfg(0.5, 15.0, 4)).to(DEV)
    g = torch.Generator().manual_seed(seed)
    leaves = dict(coordinates=c.coords.reshape(1, v, r, srf, 1, 2).clone(),
                  depths=torch.rand(b, v, r, srf, spp, generator=g).mul(20).add(0.5).to(DEV),
                  raw=torch.randn(b, v, r, srf, 1, 82, generator=g).to(DEV))
    leaves = {k: t.requires_grad_(True) for k, t in leaves.items()}
    opac = torch.rand(b, v, r, srf, spp, generator=g).to(DEV)
    out = ad(c.E.reshape(1, v, 1, 1, 1, 4, 4), c.K.reshape(1, v, 1, 1, 1, 3, 3), leaves["coordinates"],
             leaves["depths"], opac, leaves["raw"], (c.h, c.w))
    # the ABI view of the same call: b * v cameras
    abi = Case.__new__(Case)
    abi.__dict__.update(c.__dict__)
    abi.nv = b * v
    from pixelsplat_b200 import sh
    abi.E, abi.K = c.E.repeat(b, 1, 1), c.K.repeat(b, 1, 1)
    abi.D = sh.camera_sh_rotations(abi.E, 4, ad.sh_rotation_convention)         # what the module computes
    abi.coords = c.coords.repeat(b, 1, 1)
    abi.depths = leaves["depths"].detach().reshape(b * v, r * srf, spp).contiguous()
    abi.raw = leaves["raw"].detach().reshape(b * v, r * srf, 82).contiguous()
    return ad, out, leaves, abi


def test_module_path_broadcast_over_the_batch():
    b, v, r, srf, spp = 2, 2, 37, 2, 3
    ad, out, leaves, abi = _module_call(b, v, r, srf, spp)
    lead = (b, v, r, srf, spp)
    with torch.no_grad():
        f = af.forward(*abi.ref_args())
    trace = f["covariances"].diagonal(dim1=-2, dim2=-1).sum(-1).reshape(lead)
    gen = torch.Generator(device=DEV).manual_seed(5)
    R = lambda *s: torch.randn(s, generator=gen, device=DEV)
    cot = dict(means=R(*lead, 3), covariances=R(*lead, 3, 3) / trace[..., None, None].float(),
               harmonics=R(*lead, 3, 25), scales=R(*lead, 3) / f["scales"].mean(-1).reshape(lead).float()[..., None],
               rotations=R(*lead, 4))
    names = list(cot)
    grads = torch.autograd.grad([getattr(out, k) for k in names], list(leaves.values()), [cot[k] for k in names])
    nv, nr = b * v, r * srf
    abi_cot = dict(d_means=cot["means"].reshape(nv, nr, spp, 3), d_cov=cot["covariances"].reshape(nv, nr, spp, 3, 3),
                   d_harm=cot["harmonics"].reshape(nv, nr, spp, 3, 25), d_scales=cot["scales"].reshape(nv, nr, spp, 3),
                   d_rot=cot["rotations"].reshape(nv, nr, spp, 4).sum(2))
    ref = abi.reference(abi_cot)
    got = dict(means=out.means.reshape(nv, nr, spp, 3), covariances=out.covariances.reshape(nv, nr, spp, 3, 3),
               harmonics=out.harmonics.reshape(nv, nr, spp, 3, 25), scales=out.scales.reshape(nv, nr, spp, 3),
               rotations=out.rotations[..., 0, :].reshape(nv, nr, 4),
               d_depths=grads[1].reshape(nv, nr, spp), d_raw=grads[2].reshape(nv, nr, 82))
    assert torch.equal(out.rotations, out.rotations[..., :1, :].expand_as(out.rotations))
    af.check(got, ref, "module", keys=af.OUTPUTS + ("d_depths", "d_raw"))
    # coordinates are shared by the batch: their gradient is the sum of the b cameras', held to the summed bar
    ref_c = dict(ref, d_coordinates=ref["d_coordinates"].reshape(b, v, nr, 2).sum(0),
                 scale=dict(ref["scale"], d_coordinates=ref["scale"]["d_coordinates"].reshape(b, v, nr, 2).sum(0)))
    af.check(dict(d_coordinates=grads[0].reshape(v, nr, 2)), ref_c, "module-coords", keys=("d_coordinates",))


def test_training_loss_passes_null_scale_and_rotation_gradients():
    """Training uses means, covariances, harmonics and opacities; scales and rotations only reach a visualisation
    dump.  With materialize_grads off their cotangents stay None and reach the kernel as NULL: the same bits as the
    same loss plus 0 * (scales.sum() + rotations.sum()), whose zero cotangents the kernel reads, at one launch."""
    from pixelsplat_b200 import _lib
    ws = {}
    results = []
    for extra in (False, True):
        ad, out, leaves, _ = _module_call(seed=43)
        for k in ("means", "covariances", "harmonics", "opacities"):
            if k not in ws:
                ws[k] = torch.randn(getattr(out, k).shape, generator=torch.Generator().manual_seed(len(ws))).to(DEV)
        loss = sum((getattr(out, k) * w).sum() for k, w in ws.items())
        if extra:
            loss = loss + 0.0 * (out.scales.sum() + out.rotations.sum())
        torch.cuda.synchronize()
        l0 = _lib.lib.ps_launch_count()
        grads = torch.autograd.grad(loss, list(leaves.values()))
        torch.cuda.synchronize()
        assert _lib.lib.ps_launch_count() - l0 == 1
        results.append(grads)
    for a, b_ in zip(*results):
        assert torch.equal(a.view(torch.int32), b_.view(torch.int32))
