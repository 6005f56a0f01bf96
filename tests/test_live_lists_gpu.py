"""The per-tile live lists the tile sort leaves for the warp-task compositor (ps_common.cuh, kLivePosLimit), pinned
against a NumPy restatement of the compositor's per-block box test.

For every (view, tile) segment of the sorted keys, an entry is live when its cull record's box (x +- ex, y +- ey, float32
arithmetic) meets at least one of the tile's eight 8x4 pixel blocks; the live list holds, in list order, one
(position << 8 | block mask, Gaussian id) record per live entry at the segment's tile_start offset of keys_alt, and
tile_cursor holds the segment's live count.  Checked here bit for bit: positions, ids, masks and counts, on segments
with 0 and 1 entries, a segment longer than any shared-memory sort capacity, the CUB debug sort (sort_impl = 1), a
call whose first attempt overflowed the instance capacity, and a 4-view call."""
import numpy as np
import pytest
import torch

from pixelsplat_b200 import synthetic
from tests import util

pytestmark = pytest.mark.gpu

DEV = util.DEV
TILE = 16


def _u32(buf: np.ndarray, off: int, count: int) -> np.ndarray:
    return buf[off:off + 4 * count].view(np.uint32)


def expected_live(keys: np.ndarray, cull: np.ndarray, x0: int, y0: int):
    """(positions, Gaussian ids, block masks) of the live entries of one sorted segment `keys` (uint64)."""
    g = (keys & np.uint64(0xFFFFFFFF)).astype(np.int64)
    cr = cull[g]
    xl, xh = cr[:, 0] - cr[:, 2], cr[:, 0] + cr[:, 2]          # float32, like the kernels
    yl, yh = cr[:, 1] - cr[:, 3], cr[:, 1] + cr[:, 3]
    mask = np.zeros(g.size, np.uint32)
    for b in range(8):
        bx, by = x0 + (b & 1) * 8, y0 + (b >> 1) * 4
        hit = ((xh >= np.float32(bx)) & (xl <= np.float32(bx + 7)) &
               (yh >= np.float32(by)) & (yl <= np.float32(by + 3)))
        mask |= hit.astype(np.uint32) << np.uint32(b)
    live = mask != 0
    return np.nonzero(live)[0].astype(np.uint32), g[live].astype(np.uint32), mask[live]


def check_live_lists(st) -> dict:
    """Compares every segment's live list in the state `st` (a RasterOutputState) with expected_live.  Returns
    counts of what was seen (segments by length class, entries, live entries)."""
    from pixelsplat_b200 import _lib
    st.verify()
    d = st.desc
    lay = _lib.layout(d)
    vt = d.n_scenes * d.views_per_scene
    gx, gy = (d.width + TILE - 1) // TILE, (d.height + TILE - 1) // TILE
    tiles, P = gx * gy, d.n_gaussians
    n = st.num_instances()
    geom = st.geom.cpu().numpy()
    binning = st.binning.cpu().numpy()
    count = _u32(geom, lay.tile_count, vt * tiles).astype(np.int64)
    start = _u32(geom, lay.tile_start, vt * tiles).astype(np.int64)
    n_live = _u32(geom, lay.tile_cursor, vt * tiles).astype(np.int64)
    cull = geom[lay.cull:lay.cull + 16 * vt * P].view(np.float32).reshape(vt, P, 4)
    keys = binning[lay.keys:lay.keys + 8 * n].view(np.uint64)
    live = binning[lay.keys_alt:lay.keys_alt + 8 * n].view(np.uint32).reshape(n, 2)
    assert count.sum() == n
    seen = dict(empty=0, single=0, longest=0, entries=0, live=0)
    for seg in range(vt * tiles):
        vid, tile = divmod(seg, tiles)
        c, s0 = int(count[seg]), int(start[seg])
        pos, ids, masks = expected_live(keys[s0:s0 + c], cull[vid], (tile % gx) * TILE, (tile // gx) * TILE)
        assert n_live[seg] == pos.size, (seg, int(n_live[seg]), pos.size)
        rec = live[s0:s0 + pos.size]
        assert np.array_equal(rec[:, 0] >> 8, pos), seg
        assert np.array_equal(rec[:, 0] & 0xFF, masks), seg
        assert np.array_equal(rec[:, 1], ids), seg
        seen["empty"] += c == 0
        seen["single"] += c == 1
        seen["longest"] = max(seen["longest"], c)
        seen["entries"] += c
        seen["live"] += pos.size
    return seen


def _one_view(sc, sort_impl=0):
    a = util.view_args(sc)
    _, _, st, _ = util.native(a, (0.0, 0.0, 0.0), *sc.image_shape, sort_impl)
    return st


@pytest.mark.parametrize("sort_impl", [0, 1])
def test_config0(sort_impl):
    """64x64, 1k Gaussians: the native sort and the CUB debug sort leave the same live lists."""
    seen = check_live_lists(_one_view(synthetic.scene_random_frustum(seed=0), sort_impl))
    assert 0 < seen["live"] < seen["entries"]


@pytest.mark.parametrize("sort_impl", [0, 1])
def test_empty_and_single_entry_segments(sort_impl):
    """One Gaussian: every segment has 0 or 1 entries (the sort's n < 2 early exit)."""
    sc = synthetic.scene_random_frustum(seed=10, num_gaussians=1)
    sc.means[0] = torch.tensor([0.0, 0.0, 3.0])
    seen = check_live_lists(_one_view(sc, sort_impl))
    assert seen["empty"] > 0 and seen["single"] > 0 and seen["longest"] == 1 and seen["live"] > 0
    sc = synthetic.scene_random_frustum(seed=9, num_gaussians=64)
    sc.means[:, 2] = -sc.means[:, 2]                      # nothing on screen: no instances at all
    seen = check_live_lists(_one_view(sc, sort_impl))
    assert seen["entries"] == 0


def test_segment_past_the_shared_memory_cap():
    """One 16x16 tile under 30k Gaussians: longer than the largest shared-memory sort (8192), sorted through HBM."""
    sc = synthetic.scene_random_frustum(seed=7, image_hw=(16, 16), num_gaussians=30000, z_range=(2.0, 30.0))
    seen = check_live_lists(_one_view(sc))
    assert seen["longest"] > 8192 and 0 < seen["live"]


def test_capacity_overflow():
    """The first attempt overflows the instance capacity (its sort is skipped); the re-run's lists are whole."""
    from pixelsplat_b200 import rasterizer
    sc = synthetic.scene_random_frustum(seed=11, num_gaussians=3000)
    H, W = sc.image_shape
    rasterizer._capacity_hint[(0, 1, 1, 3000, H, W)] = 16   # far too small
    seen = check_live_lists(_one_view(sc))
    assert rasterizer._capacity_hint[(0, 1, 1, 3000, H, W)] > 16
    assert seen["entries"] > 16


def test_four_views_in_one_call():
    """One scene, 4 target views in one call: per-view cull records and tile offsets."""
    from pixelsplat_b200.rasterizer import rasterize_gaussians
    sc = synthetic.scene_re10k_like(seed=3, image_hw=(64, 64), target_views=4)
    args = [util.view_args(sc, view=v, scale_invariant=False) for v in range(4)]
    cam = lambda k: torch.stack([a[k] for a in args]).to(DEV)
    states = []
    with torch.no_grad():
        rasterize_gaussians(
            args[0]["means"][None].to(DEV), args[0]["cov6"][None].to(DEV), args[0]["opac"][None].to(DEV),
            args[0]["sh"][None].to(DEV), viewmatrix=cam("vm"), projmatrix=cam("pm"), campos=cam("campos"),
            tanfov=torch.tensor([[a["tanfovx"], a["tanfovy"]] for a in args], device=DEV),
            background=torch.zeros(4, 3, device=DEV), image_shape=(64, 64), views_per_scene=4,
            sh_degree=args[0]["sh_degree"], state_out=states)
    seen = check_live_lists(states[0])
    assert 0 < seen["live"] < seen["entries"]
