"""CPU: the region planner (DESIGN §4.8).

* Dependency check with NaN: the decoder chain of `cr`, `cr_rgb` and `cr_rgb_shared` (recursive) runs on CPU tensors
  through train._dec_forward / train._prob_clf, the same parameter tree the kernels read, with every input outside
  the planned windows set to NaN.  Every parameter inside a planned rectangle stays finite, and shrinking any window
  edge that is not an image edge by one pixel lets NaN in: the margins are the smallest that work.
* Geometry: tile alignment, regions at every edge, 1x1 and whole-image regions, padding tuples, recursive shapes at
  every level, and every refusal."""
import struct

import numpy as np
import pytest
import torch

from tests import util


def _net(cfg):
    return util.blueprint(cfg, device='cpu').net


def _shapes(net, H, W, R=0):
    """[(C, H, W)] coarse -> fine of a container of an H x W (padded) image."""
    n = net.scales + R + 1
    out = []
    for scale in reversed(range(n)):
        C = 3 if (scale == 0 or net._rgb) else net.config_ms.q.C
        out.append((C, H >> scale, W >> scale))
    return out


def _nan_outside(x, rect):
    y0, x0, y1, x1 = rect
    out = torch.full_like(x, float('nan'))
    out[:, :, y0:y1, x0:x1] = x[:, :, y0:y1, x0:x1]
    return out


def _run_chain(net, shapes, plan, shrink=None):
    """Run the decoder networks of `plan` coarse -> fine on full-size CPU tensors, every input NaN outside its
    window (shrink = (scale position, edge): that window one pixel smaller on that edge).  -> [P per net scale]."""
    from l3c_pytorch_b200 import train
    g = torch.Generator().manual_seed(5)
    Ps, F = [], None
    with torch.no_grad():
        for k, sp in enumerate(plan.scales):
            if sp.window is None:
                continue
            Cb, Hc, Wc = shapes[sp.idx - 1]
            s = min(sp.scale, net.scales - 1)
            win = list(sp.window)
            if shrink is not None and shrink[0] == k:
                e = shrink[1]
                win[e] += 1 if e < 2 else -1
            bn = _nan_outside(torch.rand(1, Cb, Hc, Wc, generator=g) * 2 - 1, win)
            fuse = _nan_outside(F, win) if sp.fused else None
            F = train._dec_forward(net.nets[s].dec, bn, fuse)
            assert F.shape[-2:] == (2 * Hc, 2 * Wc)
            Ps.append((k, train._prob_clf(net.prob_clfs[s], F)))
    return Ps


def _rect_values(P, rect):
    y0, x0, y1, x1 = rect
    return P[:, :, y0:y1, x0:x1]


@pytest.mark.parametrize('cfg,H,W,R,region,tile', [
    ('cr', 320, 288, 0, (150, 140, 10, 12), (16, 16)),
    ('cr_rgb', 320, 256, 0, (170, 100, 6, 20), (16, 24)),
    ('cr_rgb_shared', 256, 320, 2, (120, 150, 16, 16), (16, 16))])
def test_nan_dependency_check(cfg, H, W, R, region, tile):
    from l3c_pytorch_b200.region import plan_region
    net = _net(cfg)
    shapes = _shapes(net, H, W, R)
    plan = plan_region(shapes, (0, 0, 0, 0), tile, net, region)
    assert len(plan.scales) == len(shapes)
    for k, P in _run_chain(net, shapes, plan):
        assert torch.isfinite(_rect_values(P, plan.scales[k].rect)).all(), 'NaN reached the planned rows of %s' % (
            plan.scales[k],)
    # every window edge that is not an image edge is tight
    tested = 0
    for k, sp in enumerate(plan.scales):
        if sp.window is None:
            continue
        Hc, Wc = shapes[sp.idx - 1][1:]
        for e, at_edge in enumerate((sp.window[0] == 0, sp.window[1] == 0, sp.window[2] == Hc, sp.window[3] == Wc)):
            if at_edge:
                continue
            Ps = dict(_run_chain(net, shapes, plan, shrink=(k, e)))
            assert not torch.isfinite(_rect_values(Ps[k], sp.rect)).all(), \
                'window edge %d of %s is wider than needed' % (e, sp)
            tested += 1
    assert tested >= 4


def test_radii_come_from_the_module_tree():
    from l3c_pytorch_b200.region import DecoderGeometry
    g = DecoderGeometry(_net('cr'))
    r = g.radii[0]
    assert (r.head, r.body, r.tail, r.clf) == (0, 2 * 8 + 1, 1, 4)
    assert g.fuses(0) and g.fuses(1) and not g.fuses(2) and not g.fuses(3)
    gs = DecoderGeometry(_net('cr_rgb_shared'))
    assert not gs.fuses(0) and gs.radii_of(3) is gs.radii[0]
    gr = DecoderGeometry(_net('cr_rgb'))
    assert gr.fuses(1) and not gr.fuses(2) and not gr.fuses(4) and gr.radii_of(4) is gr.radii[2]
    # the radii follow the modules, not a table: a wider atrous rate widens the classifier's field
    net = _net('cr_rgb_shared')
    a = net.prob_clfs[0].atrous.atrous[-1]
    old = a.dilation
    a.dilation = (6, 6)
    try:
        assert DecoderGeometry(net).radii[0].clf == 6
    finally:
        a.dilation = old


def _check_aligned(plan, tile):
    th, tw = tile
    for sp in plan.scales:
        y0, x0, y1, x1 = sp.rect
        assert y0 % th == 0 and x0 % tw == 0 and (y1 % th == 0 or y1 == sp.H) and (x1 % tw == 0 or x1 == sp.W)
        assert 0 <= y0 < y1 <= sp.H and 0 <= x0 < x1 <= sp.W
        ntx = -(-sp.W // tw)
        want = sorted(ty * ntx + tx for ty in range(y0 // th, -(-y1 // th)) for tx in range(x0 // tw, -(-x1 // tw)))
        assert sp.tiles == want
        if sp.window is not None:
            wy0, wx0, wy1, wx1 = sp.window
            oy0, ox0, oy1, ox1 = sp.out
            assert (oy1 - oy0, ox1 - ox0) == (y1 - y0, x1 - x0)
            assert 0 <= oy0 and oy1 <= 2 * (wy1 - wy0) and 0 <= ox0 and ox1 <= 2 * (wx1 - wx0)
    # every window lies inside the coarser scale's decoded rectangle
    for fine, coarse in zip(plan.scales[1:], plan.scales[:-1]):
        w, r = fine.window, coarse.rect
        assert r[0] <= w[0] and r[1] <= w[1] and w[2] <= r[2] and w[3] <= r[3]


def test_geometry_edges_corners_and_whole_image():
    from l3c_pytorch_b200.codec import tile_grid
    from l3c_pytorch_b200.region import plan_region
    net = _net('cr')
    H, W = 200, 312
    shapes = _shapes(net, H, W)
    for tile in [(64, 64), (32, 48), (16, 16), (7, 5)]:
        for reg in [(0, 0, 1, 1), (H - 1, W - 1, 1, 1), (0, 100, 9, 30), (H - 9, 100, 9, 30), (60, 0, 20, 9),
                    (60, W - 9, 20, 9), (90, 140, 10, 10), (0, 0, H, W)]:
            plan = plan_region(shapes, (0, 0, 0, 0), tile, net, reg)
            _check_aligned(plan, tile)
            y, x, h, w = reg
            fin = plan.scales[-1].rect
            assert fin[0] <= y and fin[1] <= x and y + h <= fin[2] and x + w <= fin[3]
            assert plan.region == (y, x, y + h, x + w)
            assert plan.symbols == sum(sp.C * (sp.rect[2] - sp.rect[0]) * (sp.rect[3] - sp.rect[1])
                                       for sp in plan.scales)
            assert plan.streams == sum(sp.C * len(sp.tiles) for sp in plan.scales)
        whole = plan_region(shapes, (0, 0, 0, 0), tile, net, (0, 0, H, W))
        for sp in whole.scales:                                          # the whole image plans every tile
            assert sp.tiles == list(range(len(tile_grid(sp.H, sp.W, tile)))) and sp.rect == (0, 0, sp.H, sp.W)
            if sp.window is not None:
                Hc, Wc = shapes[sp.idx - 1][1:]
                assert sp.window == (0, 0, Hc, Wc)
    # an interior region at the finest scale plans fewer symbols than the image has
    small = plan_region(shapes, (0, 0, 0, 0), (16, 16), net, (96, 144, 10, 10))
    assert small.scales[-1].symbols == 3 * 16 * 16 and small.scales[-1].tiles == [6 * 20 + 9]


def test_padding_tuples():
    from l3c_pytorch_b200.region import plan_region
    net = _net('cr')
    shapes = _shapes(net, 64, 72)
    pad = (3, 5, 2, 6)                                                   # left, right, top, bottom
    Hu, Wu = 64 - 8, 72 - 8
    plan = plan_region(shapes, pad, (16, 16), net, (0, 0, 1, 1))
    assert plan.region == (2, 3, 3, 4)
    plan = plan_region(shapes, pad, (16, 16), net, (Hu - 2, Wu - 3, 2, 3))
    assert plan.region == (2 + Hu - 2, 3 + Wu - 3, 2 + Hu, 3 + Wu)
    _check_aligned(plan, (16, 16))
    for bad in [(Hu - 1, 0, 2, 1), (0, Wu, 1, 1), (-1, 0, 1, 1)]:
        with pytest.raises(ValueError, match='outside'):
            plan_region(shapes, pad, (16, 16), net, bad)


@pytest.mark.parametrize('R', [0, 1, 2, 3])
def test_recursive_shapes_every_level(R):
    from l3c_pytorch_b200.region import plan_region
    net = _net('cr_rgb_shared')
    fac = 2 ** (1 + R)
    shapes = _shapes(net, 12 * fac, 10 * fac, R)
    n = len(shapes)
    assert n == R + 2
    for level in range(n):
        _, Hk, Wk = shapes[n - 1 - level]
        sh = 1 if level == 0 else 0            # padding (1, 1, 1, 1) shifts level-0 regions, not thumbnail ones
        Hk, Wk = Hk - 2 * sh, Wk - 2 * sh
        for reg in [(0, 0, 1, 1), (Hk // 2, Wk // 3, 2, 3), (0, 0, Hk, Wk), (Hk - 1, Wk - 1, 1, 1)]:
            plan = plan_region(shapes, (1, 1, 1, 1), (8, 8), net, reg, level)
            assert [sp.scale for sp in plan.scales] == list(reversed(range(level, n)))
            assert plan.scales[0].window is None and all(sp.window is not None for sp in plan.scales[1:])
            assert not any(sp.fused for sp in plan.scales)
            assert plan.region == (reg[0] + sh, reg[1] + sh, reg[0] + reg[2] + sh, reg[1] + reg[3] + sh)
            _check_aligned(plan, (8, 8))
        with pytest.raises(ValueError, match='outside'):
            plan_region(shapes, (1, 1, 1, 1), (8, 8), net, (0, 0, Hk + 1, 1), level)
    with pytest.raises(ValueError, match='does not exist'):
        plan_region(shapes, (0, 0, 0, 0), (8, 8), net, (0, 0, 1, 1), n)


def _container(shapes, tile, pad=(0, 0, 0, 0)):
    """A parseable container with empty streams (the planner never reads a stream)."""
    from l3c_pytorch_b200.codec import ContainerLayout, tile_grid
    layout = ContainerLayout([(n, C, H, W) for n, (C, H, W) in enumerate(shapes)], tile)
    n_streams = sum(C * len(tile_grid(H, W, tile)) for (C, H, W) in shapes)
    total, pieces, _ = layout.header_and_offsets(np.zeros(n_streams, np.int64), pad)
    buf = bytearray(total)
    for o, b in pieces:
        buf[o:o + len(b)] = b
    return bytes(buf)


def test_refusals():
    from l3c_pytorch_b200.codec import BatchCodec
    from l3c_pytorch_b200.region import plan_region
    net = _net('cr')
    shapes = _shapes(net, 64, 64)
    cases = [(None, (0, 0, 1, 1), 0, 'tile='), ((16, 16), (0, 0, 0, 4), 0, 'empty'),
             ((16, 16), (0, 0, 4, -1), 0, 'empty'), ((16, 16), (60, 0, 8, 4), 0, 'outside'),
             ((16, 16), (0, 0, 4, 4), 1, 'not images'), ((16, 16), (0, 0, 4, 4), 4, 'does not exist'),
             ((16, 16), (0, 0, 4, 4), -1, 'does not exist'), ((16, 16), (0, 0, 4, 4), 1.0, 'does not exist'),
             ((16, 16), (0, 0, 4), 0, r'\(y, x, h, w\)')]
    for tile, reg, lev, match in cases:
        with pytest.raises(ValueError, match=match):
            plan_region(shapes, (0, 0, 0, 0), tile, net, reg, lev)
    codec = BatchCodec(util.blueprint('cr', device='cpu'))
    ok = _container(shapes, (16, 16))
    assert len(codec.plan_regions([ok], [(0, 0, 4, 4)])[1]) == 1
    assert struct.unpack_from('<4H', ok) == (0, 0, 0, 0)
    with pytest.raises(ValueError, match='tile='):
        codec.plan_regions([_container(shapes, None)], [(0, 0, 4, 4)])
    rgb = _container(_shapes(_net('cr_rgb_shared'), 64, 64), (16, 16))
    with pytest.raises(ValueError, match='not written by this model'):
        codec.plan_regions([ok, rgb], [(0, 0, 4, 4)] * 2)
    with pytest.raises(ValueError, match='regions for'):
        codec.plan_regions([ok, ok], [(0, 0, 4, 4)])
    with pytest.raises(ValueError, match='levels for'):
        codec.plan_regions([ok], [(0, 0, 4, 4)], [0, 0])
    with pytest.raises(ValueError):
        codec.plan_regions([ok[:40]], [(0, 0, 4, 4)])                    # truncated: as parse_container says


def test_cli_region_flags():
    from l3c_pytorch_b200 import cli
    p = cli.build_parser()
    a = p.parse_args(['dec', 'i.l3c', 'o.png', '--region', '10,20,30,40', '--level', '2'])
    assert a.region == (10, 20, 30, 40) and a.level == 2
    a = p.parse_args(['dec', 'i.l3c', 'o.png'])
    assert a.region is None and a.level == 0
    for bad in ('1,2,3', 'a,b,c,d', '1,2,3,4,5'):
        with pytest.raises(SystemExit):
            p.parse_args(['dec', 'i.l3c', 'o.png', '--region', bad])
