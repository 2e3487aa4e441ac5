"""CPU: how a decode_regions call is cut into passes (region.plan_passes, DESIGN §4.8 "Batches") and the padded stream
layout of a ragged region pass (codec.stream_layout(pad_tiles=True))."""
import numpy as np
import pytest

from tests import util


def _shapes(net, H, W, R=0):
    n = net.scales + R + 1
    return [(3 if (s == 0 or net._rgb) else net.config_ms.q.C, H >> s, W >> s) for s in reversed(range(n))]


def _plans(cfg, items, tile=(32, 32)):
    """items: [(H, W, region, level, R)] -> [RegionPlan]"""
    from l3c_pytorch_b200.region import DecoderGeometry, plan_region
    net = util.blueprint(cfg, device='cpu').net
    geo = DecoderGeometry(net)
    return [plan_region(_shapes(net, H, W, R), (0, 0, 0, 0), tile, geo, reg, lev) for (H, W, reg, lev, R) in items]


def test_plans_of_one_level_and_tile_share_one_ragged_pass():
    from l3c_pytorch_b200.region import plan_passes
    plans = _plans('cr', [(256, 320, (100, 100, 20, 30), 0, 0),       # interior
                          (256, 320, (0, 0, 40, 40), 0, 0),           # clipped by the corner
                          (128, 192, (50, 60, 20, 30), 0, 0),         # another image size
                          (256, 320, (101, 99, 20, 30), 0, 0)])       # the first one's shape, elsewhere
    keys = [p.shape_key() for p in plans]
    assert len(set(keys)) >= 3
    assert len({p.pass_key() for p in plans}) == 1
    assert plan_passes(plans, ragged=True) == [([0, 1, 2, 3], True)]
    # without ragged windows: one equal-shape pass per shape_key, in order of first appearance
    grouped = plan_passes(plans, ragged=False)
    assert all(not r for _, r in grouped)
    assert sorted(i for idxs, _ in grouped for i in idxs) == [0, 1, 2, 3]
    assert [idxs[0] for idxs, _ in grouped] == sorted(idxs[0] for idxs, _ in grouped)
    for idxs, _ in grouped:
        assert len({keys[i] for i in idxs}) == 1


def test_single_key_calls_keep_the_equal_shape_pass():
    from l3c_pytorch_b200.region import plan_passes
    one = _plans('cr', [(256, 320, (100, 100, 20, 30), 0, 0)])
    assert plan_passes(one, ragged=True) == [([0], False)]
    same = _plans('cr', [(2048, 2048, (800, 800, 20, 30), 0, 0), (2048, 2048, (1056, 1312, 20, 30), 0, 0)])
    assert same[0].shape_key() == same[1].shape_key()
    assert plan_passes(same, ragged=True) == [([0, 1], False)]
    assert plan_passes(same, ragged=False) == [([0, 1], False)]


def test_levels_and_recursion_depths_are_separate_passes():
    from l3c_pytorch_b200.region import plan_passes
    plans = _plans('cr_rgb_shared', [(128, 96, (10, 10, 20, 20), 0, 0),
                                     (128, 96, (5, 7, 9, 11), 1, 2),
                                     (128, 96, (0, 0, 30, 30), 0, 2),
                                     (96, 64, (40, 30, 12, 5), 0, 0),
                                     (128, 96, (50, 40, 10, 6), 1, 2),
                                     (128, 96, (1, 1, 3, 3), 3, 2)])
    passes = plan_passes(plans, ragged=True)
    assert [idxs for idxs, _ in passes] == [[0, 3], [1, 4], [2], [5]]
    assert [r for _, r in passes] == [True, True, False, False]


def test_regions_of_different_sizes_in_the_same_tiles_have_different_shape_keys():
    """Their rectangles and windows are the same, but the final crop is not: they must not share an equal-shape pass."""
    from l3c_pytorch_b200.region import plan_passes
    plans = _plans('cr', [(256, 320, (100, 100, 20, 20), 0, 0), (256, 320, (100, 100, 5, 4), 0, 0)])
    assert [s.shape_key() for s in plans[0].scales] == [s.shape_key() for s in plans[1].scales]
    assert plans[0].shape_key() != plans[1].shape_key()
    assert plan_passes(plans, ragged=False) == [([0], False), ([1], False)]


def test_tile_sizes_are_separate_passes():
    from l3c_pytorch_b200.region import plan_passes
    a = _plans('cr', [(128, 128, (10, 10, 20, 20), 0, 0)], tile=(32, 32))
    b = _plans('cr', [(128, 128, (10, 10, 40, 20), 0, 0)], tile=(16, 16))
    assert plan_passes(a + b, ragged=True) == [([0], False), ([1], False)]


def test_padded_stream_layout_of_different_tile_counts():
    from l3c_pytorch_b200.codec import stream_layout, tile_grid
    shapes_of = [[(3, 40, 70)], [(3, 20, 30)], [(3, 64, 64)]]
    tile = (32, 32)
    with pytest.raises(ValueError, match='different numbers of tiles'):
        stream_layout(shapes_of, tile)
    si, elem, n_sym, planes = stream_layout(shapes_of, tile, pad_tiles=True)
    T = max(len(tile_grid(h, w, tile)) for [(_, h, w)] in shapes_of)
    assert si.shape == (3, 3 * T) and int(planes[0]) == 64 * 64
    for n, [(C, h, w)] in enumerate(shapes_of):
        grid = tile_grid(h, w, tile)
        for c in range(C):
            row = slice(c * T, (c + 1) * T)
            real = [(elem[n, row][t] - (n * C + c) * planes[0], n_sym[n, row][t]) for t in range(len(grid))]
            assert real == grid
            assert (n_sym[n, row][len(grid):] == 0).all()
            assert (elem[n, row][len(grid):] == (n * C + c) * planes[0]).all()
    # equal tile counts: the same layout with or without padding
    eq = [[(3, 40, 70)], [(3, 64, 70)]]
    for a, b in zip(stream_layout(eq, tile), stream_layout(eq, tile, pad_tiles=True)):
        assert np.array_equal(a, b)


def test_pass_streams_follow_the_padded_layout():
    """region.pass_streams: the planned streams of every channel in stream_columns order, then empty ones up to the
    pass's largest tile count -- column for column the streams stream_layout(pad_tiles=True) lays out."""
    from l3c_pytorch_b200.codec import stream_layout, tile_grid
    from l3c_pytorch_b200.region import pass_streams, stream_columns
    tile = (32, 32)
    plans = _plans('cr', [(256, 320, (100, 100, 20, 30), 0, 0), (256, 320, (0, 0, 40, 40), 0, 0),
                          (128, 192, (30, 60, 90, 30), 0, 0)], tile)
    # stream `col` of scale idx of container n: offset 100000 * idx + 10 * col (from the container's start), col + 1 bytes
    streams_of = [[[(100000 * sp.idx + 10 * col, col + 1) for col in range(sp.C * len(tile_grid(sp.H, sp.W, tile)))]
                   for sp in p.scales] for p in plans]
    starts = np.array([0, 7000000, 9000000], np.int64)
    offs, lens = pass_streams(plans, streams_of, starts)
    rects_of = [[(sp.C, sp.rect[2] - sp.rect[0], sp.rect[3] - sp.rect[1]) for sp in p.scales] for p in plans]
    si, _, n_sym, _ = stream_layout(rects_of, tile, pad_tiles=True)
    assert offs.dtype == lens.dtype == np.int64 and offs.shape == lens.shape == n_sym.shape
    assert ((lens > 0) == (n_sym > 0)).all()                 # empty streams exactly where the layout pads
    assert (offs[lens == 0] == np.broadcast_to(starts[:, None], offs.shape)[lens == 0]).all()
    padded = 0
    for n, p in enumerate(plans):
        for k, (sp, cs) in enumerate(zip(p.scales, stream_columns(p, tile))):
            row = np.flatnonzero(si[n] == k)
            T, Tp = len(sp.tiles), len(row) // sp.C
            assert Tp == max(len(q.scales[k].tiles) for q in plans)
            padded += Tp - T
            for c in range(sp.C):
                real = row[c * Tp:c * Tp + T]
                want = cs[c * T:(c + 1) * T]
                assert (offs[n, real] == starts[n] + 100000 * sp.idx + 10 * np.array(want)).all()
                assert (lens[n, real] == np.array(want) + 1).all()
    assert padded > 0
    # plans of one shape_key: nothing is padded
    same = _plans('cr', [(2048, 2048, (800, 800, 20, 30), 0, 0), (2048, 2048, (1056, 1312, 20, 30), 0, 0)], tile)
    so = [[[(10 * col, col + 1) for col in range(sp.C * len(tile_grid(sp.H, sp.W, tile)))] for sp in p.scales]
          for p in same]
    assert (pass_streams(same, so, np.array([0, 16], np.int64))[1] > 0).all()
