"""CPU: region plans of seek-indexed reference-layout containers (DESIGN §4.13 "Regions").

* The band planner: every scale's decoded range starts on a seek point (or at 0), ends at the last symbol of the rows
  the finer window (the region, at the finest level) reads and covers all of them, and starting one seek point later
  would lose a needed symbol.  The decoder chain of `cr` and `cr_rgb_shared` (test_region_plan_host) with NaN outside
  the planned windows keeps every planned row finite.
* seek.plan_segments over symbol ranges equals a brute-force cut of the streams, with every state index right.
* auto_crop.part_rects equals the geometry of iter_crops for many sizes under a small crop threshold.
* Every refusal (no index, a mismatched one, bad part sets) happens before any GPU work."""
import os

import numpy as np
import pytest
import torch

from tests import util
from tests.test_region_plan_host import _container, _net, _rect_values, _run_chain, _shapes


def _band_checks(plan, shapes, K):
    n = len(shapes)
    for k, sp in enumerate(plan.scales):
        C, H, W = shapes[sp.idx]
        s0, s1 = sp.seg
        if k + 1 < len(plan.scales):
            a, b = plan.scales[k + 1].window[0], plan.scales[k + 1].window[2]       # rows the finer net reads
        else:
            a, b = plan.region[0], plan.region[2]
        assert s0 % K == 0 and s0 <= a * W, (sp, K)                                  # on a seek point, covering row a
        assert s0 + K > a * W                                                        # one point later loses a * W
        assert s1 == b * W                                                           # exact end
        assert sp.rect == (s0 // W, 0, b, W) and sp.tiles == [0]
        assert sp.symbols == C * (s1 - s0) and sp.streams == C
        assert sp.scale == n - 1 - sp.idx
    assert plan.symbols == sum(sp.symbols for sp in plan.scales)


@pytest.mark.parametrize('cfg,H,W,R', [('cr', 200, 312, 0), ('cr_rgb_shared', 96, 160, 2)])
@pytest.mark.parametrize('K', [32, 96, 4096, 1 << 20])
def test_band_plan_geometry(cfg, H, W, R, K):
    from l3c_pytorch_b200.region import _window, geometry_of, plan_region
    net = _net(cfg)
    geo = geometry_of(net)
    shapes = _shapes(net, H, W, R)
    regions = [(0, 0, 1, 1), (H - 1, W - 1, 1, 1), (H // 2, W // 3, 9, 30), (0, 0, H, W), (H // 3, 0, 1, W),
               (H - 64, 0, 64, W), (17, 40, 1, 1)]
    for reg in regions:
        plan = plan_region(shapes, (0, 0, 0, 0), None, geo, reg, every=K)
        assert plan.tile is None and plan.every == K and len(plan.scales) == len(shapes)
        _band_checks(plan, shapes, K)
        for sp in plan.scales:                       # the windows are the tiled planner's for the same rectangles
            if sp.window is not None:
                Hc, Wc = shapes[sp.idx - 1][1:]
                assert (sp.window, sp.out, sp.fused) == _window(geo, sp.scale, sp.rect, sp.H, sp.W, Hc, Wc)[:3]
                assert sp.window[1] == 0 and sp.window[3] == Wc                       # a full-width band
    # the whole image decodes every symbol; a middle band fewer than the container has
    whole = plan_region(shapes, (0, 0, 0, 0), None, geo, (0, 0, H, W), every=K)
    assert whole.symbols == sum(C * h * w for (C, h, w) in shapes)
    mid = plan_region(shapes, (0, 0, 0, 0), None, geo, (H // 2, W // 2, 4, 4), every=K)
    if K <= 4096:
        assert mid.scales[-1].symbols < 3 * H * W


def test_band_plan_levels_and_padding():
    from l3c_pytorch_b200.region import plan_region
    net = _net('cr_rgb_shared')
    shapes = _shapes(net, 48, 40, 1)
    n = len(shapes)
    for level in range(n):
        _, Hk, Wk = shapes[n - 1 - level]
        sh = 1 if level == 0 else 0
        for reg in [(0, 0, 1, 1), (Hk // 2 - sh, 2, 2, 3), (0, 0, Hk - 2 * sh, Wk - 2 * sh)]:
            plan = plan_region(shapes, (1, 1, 1, 1), None, net, reg, level, every=32)
            assert [sp.scale for sp in plan.scales] == list(reversed(range(level, n)))
            _band_checks(plan, shapes, 32)


@pytest.mark.parametrize('cfg,H,W,R,region', [
    ('cr', 320, 288, 0, (150, 140, 10, 12)),
    ('cr_rgb_shared', 256, 320, 2, (120, 150, 16, 16))])
def test_nan_dependency_check(cfg, H, W, R, region):
    """The decoder chain with every input NaN outside its planned window: every row of every planned band stays
    finite, so every symbol the segments decode (and every one the finer windows read) has its exact CDF."""
    from l3c_pytorch_b200.region import plan_region
    net = _net(cfg)
    shapes = _shapes(net, H, W, R)
    for K in (32, 4096):
        plan = plan_region(shapes, (0, 0, 0, 0), None, net, region, every=K)
        for k, P in _run_chain(net, shapes, plan):
            assert torch.isfinite(_rect_values(P, plan.scales[k].rect)).all(), 'NaN reached %s' % (plan.scales[k],)


def test_no_index_is_refused():
    from l3c_pytorch_b200.region import plan_region
    net = _net('cr')
    with pytest.raises(ValueError, match='tile=') as e:
        plan_region(_shapes(net, 64, 64), (0, 0, 0, 0), None, net, (0, 0, 4, 4))
    assert 'seek index' in str(e.value)


# ----------------------------------------------------------------------------------------------
# segment ranges
# ----------------------------------------------------------------------------------------------
def _brute_segments(n_stream, K, start, lo, hi):
    """[(first symbol, n_sym, point index or -1)] of the segments of a stream of n_stream symbols that meet [lo, hi),
    cut at hi: the first one from the seek point at or before lo."""
    out = []
    for j in range(max(1, -(-n_stream // K))):
        a, b = j * K, min((j + 1) * K, n_stream)
        if j >= lo // K and (a < hi or j == lo // K):
            out.append((a, max(0, min(b, hi) - a), j - 1))
    return out


def test_plan_segments_ranges_equal_a_brute_force_cut():
    from l3c_pytorch_b200 import _lib, seek
    rng = np.random.default_rng(7)
    for trial in range(40):
        M = int(rng.integers(1, 9))
        K = int(rng.choice([32, 64, 96, 4096]))
        n_stream = rng.integers(1, 6 * K, M)
        W = rng.integers(1, 40, M)
        lo = np.array([int(rng.integers(0, n)) for n in n_stream], np.int64)
        hi = np.array([int(rng.integers(l + 1, n + 1)) for l, n in zip(lo, n_stream)], np.int64)
        start = np.minimum(lo // K * K, (lo // K * K // W) * W)        # the row of the seek point
        n_desc = hi - start
        addr = np.sort(rng.choice(np.arange(1 << 20, 1 << 21, 8), M, replace=False)).astype(np.int64)
        order = rng.permutation(M)                                     # descriptors in any order
        first = np.concatenate([[0], np.cumsum(seek.point_counts(n_stream, K))[:-1]])
        desc = np.zeros(M, _lib.DEC_STREAM_DTYPE)
        desc['in'] = addr[order]
        desc['n_sym'] = n_desc[order]
        desc['row_pitch'] = 256
        desc['table'] = 10 ** 9 + 10 ** 7 * order
        desc['sym_out'] = 10 ** 6 * order
        state = 1 << 30
        segs = seek.plan_segments(desc, addr, np.full(M, K, np.int64), first, state, start, lo, hi)
        want = []
        for m, i in enumerate(order):
            for a, cnt, pt in _brute_segments(int(n_stream[i]), K, int(start[i]), int(lo[i]), int(hi[i])):
                st = 0 if pt < 0 else state + 4 * seek.STATE_WORDS * (first[i] + pt)
                want.append((int(addr[i]), cnt, int(desc['table'][m]) + 2 * 256 * (a - int(start[i])),
                             int(desc['sym_out'][m]) + a - int(start[i]), st))
        got = list(zip(segs['in'].tolist(), segs['n_sym'].tolist(), segs['table'].tolist(),
                       segs['sym_out'].tolist(), segs['state'].tolist()))
        assert got == want, trial
        # without ranges: the whole streams, as before
        desc['n_sym'] = n_stream[order]
        whole = seek.plan_segments(desc, addr, np.full(M, K, np.int64), first, state)
        assert whole.size == int(np.maximum(1, -(-n_stream // K)).sum())
    with pytest.raises(ValueError, match='outside'):
        seek.plan_segments(desc[:1], addr, np.full(M, 32, np.int64), first, state, np.full(M, 40), np.full(M, 40),
                           np.full(M, 50))


# ----------------------------------------------------------------------------------------------
# parts
# ----------------------------------------------------------------------------------------------
def test_part_rects_equal_iter_crops_geometry(monkeypatch):
    from l3c_pytorch_b200 import auto_crop
    monkeypatch.setenv('AC_NEEDS_CROP_DIM', '20,15')
    rng = np.random.default_rng(3)
    sizes = [(10, 12), (21, 16), (31, 17), (40, 30), (41, 31), (80, 61), (17, 90), (161, 121)] + \
        [tuple(int(v) for v in rng.integers(5, 200, 2)) for _ in range(20)]
    seen = set()
    for H, W in sizes:
        idx = torch.arange(H * W).reshape(1, 1, H, W).expand(1, 3, H, W)
        crops = list(auto_crop.iter_crops(idx))
        want = [(int(c[0, 0, 0, 0]) // W, int(c[0, 0, 0, 0]) % W) + tuple(c.shape[-2:]) for c in crops]
        try:
            rects = auto_crop.part_rects([tuple(c.shape[-2:]) for c in crops])
        except ValueError:
            # an uneven quadrant tree: stitch cannot rebuild the image either
            with pytest.raises(Exception):
                assert torch.equal(auto_crop.stitch(crops), idx)
            continue
        assert rects == want, (H, W)
        assert torch.equal(auto_crop.stitch(crops), idx)
        seen.add(len(crops))
    assert {1, 4, 16} <= seen


def test_part_rects_refusals():
    from l3c_pytorch_b200 import auto_crop
    for bad, match in [([], 'number'), ([(4, 4)] * 3, 'number'), ([(4, 4)] * 9, 'number'), ([(4, 4), (5, 4), (4, 4), (4, 4)], 'row'),
                       ([(4, 4), (4, 4), (4, 5), (4, 4)], 'column')]:
        with pytest.raises(ValueError, match=match):
            auto_crop.part_rects(bad)


# ----------------------------------------------------------------------------------------------
# refusals before any GPU work
# ----------------------------------------------------------------------------------------------
def _fake_index(data, K):
    """A well-formed seek index of `data` (points that parse; the planner never decodes them)."""
    from l3c_pytorch_b200 import seek
    counts = seek.point_counts(seek.stream_symbols(data), K)
    n = int(counts.sum())
    first = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    step = np.arange(n) - np.repeat(first, counts) + 1
    return seek.write_index(data, K, counts, np.zeros(n), np.full(n, 1 << 20), np.zeros(n), 32 + 8 * step)


def test_plan_regions_with_indexes():
    from l3c_pytorch_b200 import seek
    from l3c_pytorch_b200.codec import BatchCodec
    net = _net('cr')
    shapes = _shapes(net, 64, 64)
    codec = BatchCodec(util.blueprint('cr', device='cpu'))
    ref, tiled = _container(shapes, None), _container(shapes, (16, 16))
    sk = _fake_index(ref, 96)
    _, plans = codec.plan_regions([ref, tiled], [(10, 20, 4, 4)] * 2, seeks=[sk, None])
    assert plans[0].tile is None and plans[0].seek.every == 96 and plans[1].tile == (16, 16)
    assert plans[0].pass_key() != plans[1].pass_key()
    assert all(sp.seg is not None for sp in plans[0].scales) and all(sp.seg is None for sp in plans[1].scales)
    with pytest.raises(ValueError, match='tile='):
        codec.plan_regions([ref], [(0, 0, 4, 4)])
    with pytest.raises(ValueError, match='seek indexes for'):
        codec.plan_regions([ref], [(0, 0, 4, 4)], seeks=[sk, sk])
    with pytest.raises(ValueError, match='another container'):
        codec.plan_regions([_container(shapes, None, (0, 0, 0, 2))], [(0, 0, 4, 4)], seeks=[sk])
    with pytest.raises(ValueError, match='reference-layout'):
        codec.plan_regions([tiled], [(0, 0, 4, 4)], seeks=[seek.write_index(tiled, 96, [], [], [], [], [])])


def test_region_file_refusals(tmp_path, monkeypatch):
    from l3c_pytorch_b200 import Bitcoding, engine as E
    net = _net('cr')
    bc = Bitcoding(util.blueprint('cr', device='cpu'))
    monkeypatch.setattr(bc.codec, '_decode_planned', lambda *a, **k: pytest.fail('GPU work after a refusal'))
    shapes = _shapes(net, 64, 64)
    ref = _container(shapes, None)
    p = str(tmp_path / 'a.l3c')
    with open(p, 'wb') as f:
        f.write(ref)
    with pytest.raises(ValueError, match=r'a\.l3c\.seek'):                         # no sidecar: named
        bc.decode_region_file(p, (0, 0, 4, 4))
    with open(p + '.seek', 'wb') as f:
        f.write(_fake_index(_container(shapes, None, (0, 0, 0, 2)), 96))
    with pytest.raises(ValueError, match=r'a\.l3c\.seek.*another container'):     # mismatched: named
        bc.decode_region_file(p, (0, 0, 4, 4))
    # parts: tiled ones, a missing sidecar, level > 0, a region outside the stitched image
    q = str(tmp_path / 'b.l3c')
    for i in range(4):
        with open(q + '.part%d' % i, 'wb') as f:
            f.write(_container(shapes, (16, 16)))
    with pytest.raises(ValueError, match='tiled part'):
        bc.decode_region_file(q, (0, 0, 4, 4))
    for i in range(4):
        with open(q + '.part%d' % i, 'wb') as f:
            f.write(ref)
        if i != 2:
            with open(q + '.part%d.seek' % i, 'wb') as f:
                f.write(_fake_index(ref, 96))
    with pytest.raises(ValueError, match=r'b\.l3c\.part2\.seek'):
        bc.decode_region_file(q, (0, 0, 4, 4))
    with open(q + '.part2.seek', 'wb') as f:
        f.write(_fake_index(ref, 96))
    with pytest.raises(ValueError, match='level'):
        bc.decode_region_file(q + '.part1', (0, 0, 4, 4), level=1)
    with pytest.raises(ValueError, match='outside the 128x128'):
        bc.decode_region_file(q, (100, 100, 40, 4))
    assert E.launch_log(reset=True)[1] == 0
    assert os.path.isfile(q + '.part3.seek')
