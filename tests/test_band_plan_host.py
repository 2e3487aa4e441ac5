"""CPU: the band planner of the banded decode of large tiled containers (DESIGN §4.10).

* Bands cover every tile of a plane exactly once, in container order, and their streams (region.rect_streams) are the
  plane's stream columns with their elements moved into band planes.
* The streams rect_streams finds for the rectangles R_s of region updates are stream_columns' columns, cut by tile_grid
  of the rectangle.
* Every band's window is plan_region's window for the same rectangle.
* The NaN dependency check of test_region_plan_host, run on band windows: every planned row stays finite.
* crop=False needs tile=, and the CLI parses `enc --tile`."""
import numpy as np
import pytest
import torch

from tests import util
from tests.test_region_plan_host import _net, _rect_values, _run_chain, _shapes


@pytest.mark.parametrize('cfg,H,W,R,tile', [
    ('cr', 200, 312, 0, (16, 16)), ('cr', 200, 312, 0, (32, 48)), ('cr', 64, 72, 0, (7, 5)),
    ('cr_rgb_shared', 96, 80, 2, (16, 24))])
def test_rect_streams_of_bands_cover_every_tile_once(cfg, H, W, R, tile):
    from l3c_pytorch_b200.codec import stream_layout, tile_grid
    from l3c_pytorch_b200.region import plan_bands, rect_streams
    net = _net(cfg)
    shapes = _shapes(net, H, W, R)
    N = 3
    layout = stream_layout([[s for s in shapes]] * N, tile)
    for idx in range(1, len(shapes)):
        C, h, w = shapes[idx]
        grid = tile_grid(h, w, tile)
        nty = -(-h // tile[0])
        for rows in sorted({1, 2, 3, max(1, nty // 2), nty, nty + 5}):
            bands = plan_bands(shapes, tile, net, idx, rows)
            assert len(bands) == -(-nty // rows)
            assert sum((b.tiles for b in bands), []) == list(range(len(grid)))
            seen = np.zeros((N, C, h * w), np.int64)
            for b in bands:
                y0, x0, y1, x1 = b.rect
                assert x0 == 0 and x1 == w and y0 % tile[0] == 0 and (y1 % tile[0] == 0 or y1 == h)
                cols, n_sym, elem = rect_streams(layout, idx, b)
                e0, e1 = y0 * w, y1 * w
                assert grid[b.tiles[0]][0] == e0
                # the band's columns, channel-major and in tile order, hold the band's symbols of every image
                lo = np.searchsorted(layout[0][0], idx)
                T = len(grid)
                assert (cols == lo + (np.arange(C)[:, None] * T + np.array(b.tiles)[None, :]).reshape(-1)).all()
                assert (layout[0][:, cols] == idx).all()
                full_elem, full_n = layout[1][:, cols], layout[2][:, cols]
                assert (n_sym == full_n).all()
                nc = full_elem // layout[3][idx]
                assert (elem == nc * (e1 - e0) + full_elem - nc * layout[3][idx] - e0).all()
                assert (elem >= 0).all() and (elem + n_sym <= N * C * (e1 - e0)).all()
                for n in range(N):
                    for c in range(C):
                        for col, cnt in zip(full_elem[n], full_n[n]):
                            base = (n * C + c) * layout[3][idx]
                            if base <= col < base + h * w:
                                seen[n, c, col - base:col - base + cnt] += 1
            assert (seen == 1).all()


@pytest.mark.parametrize('H,W,tile,edit', [
    (520, 392, (16, 16), (253, 175, 30, 41)), (520, 392, (16, 24), (0, 0, 520, 392)),
    (520, 392, (64, 64), (47, 61, 34, 50)), (1008, 760, (16, 16), (504, 380, 8, 8)),
    (520, 392, (16, 24), (511, 378, 9, 11))])
def test_rect_streams_of_update_rectangles(H, W, tile, edit):
    from l3c_pytorch_b200.codec import stream_layout, tile_grid
    from l3c_pytorch_b200.region import plan_update, rect_streams, stream_columns
    net = _net('cr')
    shapes = _shapes(net, H, W)
    plan = plan_update(shapes, (0, 0, 0, 0), tile, net, edit)
    layout = stream_layout([shapes], tile)
    for idx, sp in enumerate(plan.scales):
        cols, n_sym, elem = rect_streams(layout, idx, sp)
        lo = np.searchsorted(layout[0][0], idx)
        assert (cols == lo + np.asarray(stream_columns(plan, tile)[idx])).all()
        assert (layout[0][0, cols] == idx).all()
        # the rectangle's own planes, cut by tile_grid in the plane's tile order
        h, w = sp.rect[2] - sp.rect[0], sp.rect[3] - sp.rect[1]
        grid = np.array(tile_grid(h, w, tile), np.int64)
        assert len(grid) == len(sp.tiles)
        for c in range(sp.C):
            part = slice(c * len(grid), (c + 1) * len(grid))
            assert (n_sym[0, part] == grid[:, 1]).all() and (n_sym[0, part] == layout[2][0, cols[part]]).all()
            assert (elem[0, part] == c * h * w + grid[:, 0]).all()
    assert sum(len(rect_streams(layout, idx, sp)[0]) for idx, sp in enumerate(plan.scales)) == plan.streams


@pytest.mark.parametrize('cfg,H,W,R,tile', [
    ('cr', 200, 312, 0, (16, 16)), ('cr', 136, 96, 0, (32, 48)), ('cr_rgb_shared', 96, 80, 2, (16, 24))])
def test_band_windows_are_region_windows(cfg, H, W, R, tile):
    from l3c_pytorch_b200.region import plan_bands, plan_region
    net = _net(cfg)
    shapes = _shapes(net, H, W, R)
    n = len(shapes)
    levels = range(n - 1) if net._rgb else [0]            # regions at level k >= 1 exist for the RGB baselines only
    for level in levels:
        idx = n - 1 - level
        for rows in (1, 2, 3):
            for b in plan_bands(shapes, tile, net, idx, rows):
                y0, _, y1, w = b.rect
                plan = plan_region(shapes, (0, 0, 0, 0), tile, net, (y0, 0, y1 - y0, w), level)
                sp = plan.scales[-1]
                assert (sp.rect, sp.tiles, sp.window, sp.out, sp.fused) == (b.rect, b.tiles, b.window, b.out, b.fused)


@pytest.mark.parametrize('cfg,H,W,R,tile', [
    ('cr', 160, 96, 0, (16, 16)), ('cr_rgb', 160, 64, 0, (16, 24)), ('cr_rgb_shared', 128, 96, 2, (16, 16))])
def test_nan_dependency_check_on_band_windows(cfg, H, W, R, tile):
    """The coarser scales run on their whole planes (as in a banded decode), the banded scale on one band's window of
    them only; NaN outside that window never reaches the band's rows."""
    from l3c_pytorch_b200.region import plan_bands, plan_region

    class _Chain(object):
        def __init__(self, scales):
            self.scales = scales

    net = _net(cfg)
    shapes = _shapes(net, H, W, R)
    whole = plan_region(shapes, (0, 0, 0, 0), tile, net, (0, 0, H, W))
    checked = 0
    for idx in range(1, len(shapes)):
        bands = plan_bands(shapes, tile, net, idx, 2)
        for b in (bands[0], bands[len(bands) // 2], bands[-1]):
            for k, P in _run_chain(net, shapes, _Chain(whole.scales[:idx] + [b])):
                if k == idx:
                    assert torch.isfinite(_rect_values(P, b.rect)).all(), 'NaN reached the rows of band %s' % (b,)
                    checked += 1
    assert checked >= 3 * (len(shapes) - 1)


def test_plan_bands_refusals():
    from l3c_pytorch_b200.region import plan_bands
    net = _net('cr')
    shapes = _shapes(net, 64, 64)
    with pytest.raises(ValueError, match='no decoder network'):
        plan_bands(shapes, (16, 16), net, 0, 1)
    with pytest.raises(ValueError, match='at least one tile row'):
        plan_bands(shapes, (16, 16), net, 3, 0)


def test_crop_false_needs_a_tile():
    from l3c_pytorch_b200 import Bitcoding
    bp = util.blueprint('cr', device='cpu')
    with pytest.raises(ValueError, match='tile='):
        Bitcoding(bp, crop=False)
    assert not Bitcoding(bp, tile=(64, 64), crop=False).crop
    assert Bitcoding(bp).crop and Bitcoding(bp, tile=(64, 64)).crop


def test_plane_limit_refused_on_the_host():
    from l3c_pytorch_b200.codec import MAX_PLANE_PIXELS, check_plane
    check_plane(32768, 32768, 'x')
    assert 32768 * 32768 == MAX_PLANE_PIXELS
    with pytest.raises(ValueError, match='more than'):
        check_plane(32768, 32776, 'x')


def test_cli_tile_flag():
    from l3c_pytorch_b200 import cli
    p = cli.build_parser()
    a = p.parse_args(['enc', 'i.png', 'o.l3c', '--tile', '64,32'])
    assert a.tile == (64, 32)
    assert p.parse_args(['enc', 'i.png', 'o.l3c']).tile is None
    for bad in ('64', '64,32,1', 'a,b', '0,64', '64,65536'):
        with pytest.raises(SystemExit):
            p.parse_args(['enc', 'i.png', 'o.l3c', '--tile', bad])
