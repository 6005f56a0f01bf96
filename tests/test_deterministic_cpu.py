"""CPU tests of the deterministic mode's host surface (include/pixelsplat_b200.h ps_set_option "deterministic"): the
option's round trip and its default, and the workspace sizes it implies.  Every test leaves the option and torch's
deterministic flag as it found them."""
import contextlib

import pytest
import torch

align = lambda x: (x + 255) // 256 * 256


@contextlib.contextmanager
def _restored():
    from pixelsplat_b200 import _lib
    flag, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        yield _lib
    finally:
        _lib.set_option("deterministic", 0)
        torch.use_deterministic_algorithms(flag, warn_only=warn_only)


def _desc(depth_mode=0, S=2, V=3, P=1000, H=70, W=50, capacity=12345):
    from pixelsplat_b200 import _lib
    return _lib.RasterDesc(S, V, P, 25, 4, _lib.PS_SH_3M, _lib.PS_COV_3X3, H, W, 0, 0, capacity, 0, depth_mode)


def test_option_round_trip_and_default():
    with _restored() as _lib:
        assert _lib.get_option("deterministic") == 0
        for v in (1, 0, 1):
            _lib.set_option("deterministic", v)
            assert _lib.get_option("deterministic") == v
        for bad in (-1, 2, 7):
            with pytest.raises(ValueError, match="unknown option or bad value: deterministic"):
                _lib.set_option("deterministic", bad)
            assert _lib.get_option("deterministic") == 1
        # the compositor options are independent of it
        assert [_lib.get_option(n) for n in ("composite_impl", "composite_segments", "composite_hit_lists")] == [2, 0, 2]
    assert _lib.get_option("deterministic") == 0


@pytest.mark.parametrize("depth_mode", [0, 1, 4])
@pytest.mark.parametrize("shape", [dict(), dict(S=1, V=1, P=393216, H=256, W=256, capacity=500000)])
def test_sizes_follow_the_documented_formulas(depth_mode, shape):
    """backward_bytes grows by the three record arrays (8 x instance_capacity entries of 8, 16 and 16 bytes),
    image_bytes by the per-task loss partials (S*V*tiles*8 pairs of floats); nothing else moves."""
    with _restored() as _lib:
        d = _desc(depth_mode, **shape)
        S, V, P, H, W, C = d.n_scenes, d.views_per_scene, d.n_gaussians, d.height, d.width, d.instance_capacity
        vp = S * V * P
        tasks = S * V * ((H + 15) // 16) * ((W + 15) // 16) * 8
        off, off_lay = _lib.sizes(d), _lib.layout(d)
        assert off.backward_bytes == align(vp * 8) + 2 * align(vp * 16)
        _lib.set_option("deterministic", 1)
        on, on_lay = _lib.sizes(d), _lib.layout(d)
        assert on.backward_bytes == off.backward_bytes + align(8 * C * 8) + 2 * align(8 * C * 16)
        assert on.image_bytes == off.image_bytes + align(tasks * 8)
        assert (on.geom_bytes, on.binning_bytes) == (off.geom_bytes, off.binning_bytes)
        assert all(getattr(on_lay, f) == getattr(off_lay, f) for f, _ in _lib.RasterLayout._fields_)
        _lib.set_option("deterministic", 0)
        again = _lib.sizes(d)
        assert [getattr(again, f) for f, _ in again._fields_] == [getattr(off, f) for f, _ in off._fields_]


def test_colour_only_sizes_are_todays_with_the_option_off():
    """The colour-only workspace of the option's default is the documented one of before the option existed."""
    with _restored() as _lib:
        S, V, H, W = 2, 3, 70, 50
        px = S * V * H * W
        s = _lib.sizes(_desc(0))
        assert s.image_bytes == 2 * align(px * 4) + align(px * 12) + align(px * 16 * 3)
        assert s.backward_bytes == align(S * V * 1000 * 8) + 2 * align(S * V * 1000 * 16)


def test_legacy_refusal_follows_torch_convention_without_a_gpu():
    """The host-side check runs before anything touches a device: with the legacy compositor selected, torch's flag
    raises RuntimeError, and under warn_only it warns and leaves the library option off."""
    from pixelsplat_b200 import rasterizer
    from tests import util
    with _restored() as _lib, util.composite_variant(1, 1, 0):
        torch.use_deterministic_algorithms(True)
        with pytest.raises(RuntimeError, match="does not have a deterministic implementation"):
            rasterizer._sync_deterministic()
        torch.use_deterministic_algorithms(True, warn_only=True)
        with pytest.warns(UserWarning, match="does not have a deterministic implementation"):
            rasterizer._sync_deterministic()
        assert _lib.get_option("deterministic") == 0
    with _restored() as _lib:
        torch.use_deterministic_algorithms(True)
        rasterizer._sync_deterministic()
        assert _lib.get_option("deterministic") == 1
        torch.use_deterministic_algorithms(False)
        rasterizer._sync_deterministic()
        assert _lib.get_option("deterministic") == 0
