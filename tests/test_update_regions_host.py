"""CPU: the host side of batches of region updates (DESIGN §4.12, "Batches of updates").

* The merge rule (region.merge_update_plans): plans conflict when one's edit meets the other's pixel window; merged
  plans are the plan of the bounding rectangle of their edits; the result is a fixpoint, every edit in exactly one plan.
* With the small float64 CPU network of test_update_plan_host: for two plans kept separate, NaN at one edit reaches
  nothing the other plan reads or codes; NaN at both edits changes symbols and CDF parameters only inside the union of
  the plans' R_s.
* Pass planning (region.plan_update_passes): one tile size per pass, windows within the budget.
* Every refusal of update_regions raises with the container and the edit index, on a CPU codec (no GPU work).
* The segments of codec.splice_segments, applied in numpy, give exactly ContainerLayout's bytes of the new container,
  and ContainerLayout.offsets equals header_and_offsets."""
import struct

import numpy as np
import pytest
import torch

from tests import util
from tests.test_update_plan_host import NAN, _dec, _enc, _finite, _net, _shapes


def _bound(rects, pad):
    left, _, top, _ = pad
    ys = [r[0] + top for r in rects]
    xs = [r[1] + left for r in rects]
    return (min(ys), min(xs), max(r[0] + top + r[2] for r in rects), max(r[1] + left + r[3] for r in rects))


def _merged(name, H, W, pad, tile, rects):
    from l3c_pytorch_b200.region import merge_update_plans
    net = _net(name)
    shapes = _shapes(net, H + pad[2] + pad[3], W + pad[0] + pad[1])
    return net, shapes, merge_update_plans(shapes, pad, tile, net, rects)


def _check_fixpoint(plans, rects, pad):
    from l3c_pytorch_b200.region import plans_conflict
    assert sorted(i for _, idxs in plans for i in idxs) == list(range(len(rects)))
    for p, idxs in plans:
        assert idxs == sorted(idxs) and p.edit == _bound([rects[i] for i in idxs], pad)
    for a in range(len(plans)):
        for b in range(a + 1, len(plans)):
            assert not plans_conflict(plans[a][0], plans[b][0])


def test_merge_rule_of_cr():
    pad = (0, 3, 1, 0)
    H, W = 255, 4093
    far = [(10, 50, 20, 30), (200, 3950, 30, 40)]
    _, _, plans = _merged('cr', H, W, pad, (16, 16), far)
    assert [idxs for _, idxs in plans] == [[0], [1]]
    _check_fixpoint(plans, far, pad)
    # an edit inside the first plan's window joins it; the bounding rectangle is planned
    near = far + [(40, 300, 8, 8)]
    _, _, plans = _merged('cr', H, W, pad, (16, 16), near)
    assert [idxs for _, idxs in plans] == [[0, 2], [1]]
    _check_fixpoint(plans, near, pad)
    # overlapping edits and edits whose windows meet: one plan
    over = [(100, 90, 40, 33), (120, 100, 30, 30), (0, 2000, 5, 5), (250, 1900, 5, 5)]
    _, _, plans = _merged('cr', H, W, pad, (16, 24), over)
    assert [idxs for _, idxs in plans] == [[0, 1], [2, 3]]
    _check_fixpoint(plans, over, pad)
    assert _merged('cr', H, W, pad, (16, 16), [])[2] == []


def test_merging_reaches_a_fixpoint():
    """A chain: each edit meets only the window of a neighbour, or only the grown window of a merged plan."""
    from l3c_pytorch_b200.region import plan_update, plans_conflict
    net = _net('cr')
    pad = (0, 0, 0, 0)
    H, W = 256, 8192
    shapes = _shapes(net, H, W)
    p0 = plan_update(shapes, pad, (16, 16), net, (100, 100, 8, 8))
    x1 = p0.window[3] - 4                                              # just inside the first edit's window
    p1 = plan_update(shapes, pad, (16, 16), net, (100, x1, 8, 8))
    x2 = p1.window[3] + 40                                             # outside both single windows
    rects = [(100, 100, 8, 8), (100, x1, 8, 8), (100, x2, 8, 8), (100, 7000, 8, 8)]
    p2 = plan_update(shapes, pad, (16, 16), net, rects[2])
    assert plans_conflict(p0, p1) and not plans_conflict(p1, p2) and not plans_conflict(p0, p2)
    _, _, plans = _merged('cr', H, W, pad, (16, 16), rects)
    _check_fixpoint(plans, rects, pad)
    assert len(plans) in (2, 3) and [0, 1] == plans[0][1][:2]


def _full_run(net, x):
    """Encoder and decoder of every scale on whole planes: -> (q by scale (q[0] the image), F by scale (F[0] the
    image), P by scale (CDF parameters))."""
    S = net.scales
    q, F, inp = [x], [x], x
    for s in range(S):
        inp, qs = _enc(net, s, inp)
        q.append(qs)
        F.append(inp)
    P, D = [None] * S, None
    for s in reversed(range(S)):
        D, P[s] = _dec(net, s, q[s + 1], D if net.fuses(s) else None)
    return q, F, P


def test_separate_plans_are_independent_and_cover_the_combined_edit():
    pad = (2, 3, 1, 2)
    H, W = 93, 1499
    rects = [(40, 30, 12, 20), (20, 1400, 30, 25)]
    net, shapes, plans = _merged('small', H, W, pad, (16, 16), rects)
    assert len(plans) == 2
    _, Hp, Wp = shapes[-1]
    g = torch.Generator().manual_seed(3)
    x = torch.rand(1, 3, Hp, Wp, generator=g, dtype=torch.float64) * 2 - 1
    S = net.scales
    for a, b in ((0, 1), (1, 0)):
        y = x.clone()
        e = plans[b][0].edit
        y[:, :, e[0]:e[2], e[1]:e[3]] = NAN
        q, F, P = _full_run(net, y)
        sc = {sp.scale: sp for sp in plans[a][0].scales}
        assert _finite(y, sc[0].need)                                   # plan a's pixels are the old ones
        for s in range(1, S + 1):
            assert _finite(q[s], sc[s].need) and (s == S or _finite(F[s], sc[s].need))
        for s in range(S):
            assert _finite(P[s], sc[s].rect)
    # both edits NaN: every changed symbol and CDF parameter lies in the union of the plans' R_s
    y = x.clone()
    for p, _ in plans:
        e = p.edit
        y[:, :, e[0]:e[2], e[1]:e[3]] = NAN
    q, _, P = _full_run(net, y)
    for s in range(S + 1):
        planes = [q[s]] + ([P[s]] if s < S else [])
        for t in planes:
            bad = torch.isnan(t).any(1)[0]
            cover = torch.zeros_like(bad)
            for p, _ in plans:
                r = {sp.scale: sp for sp in p.scales}[s].rect
                cover[r[0]:r[2], r[1]:r[3]] = True
            assert bad.any() and not (bad & ~cover).any(), s


def test_pass_planning():
    from l3c_pytorch_b200.region import plan_update, plan_update_passes
    net = _net('cr')
    shapes = _shapes(net, 256, 4096)
    a = [plan_update(shapes, (0, 0, 0, 0), t, net, r) for t, r in
         [((16, 16), (10, 50, 20, 30)), ((64, 64), (10, 50, 20, 30)), ((16, 16), (200, 3950, 30, 40)),
          ((16, 16), (100, 2000, 8, 8))]]
    passes = plan_update_passes(a, 1 << 40)
    assert sorted(sorted(p) for p in passes) == [[0, 2, 3], [1]]
    px = [p.window_pixels for p in a]
    for budget in (max(px), 2 * max(px), 1):
        passes = plan_update_passes(a, budget)
        assert sorted(i for p in passes for i in p) == [0, 1, 2, 3]
        for p in passes:
            assert len({a[i].tile for i in p}) == 1
            hm = max(a[i].window[2] - a[i].window[0] for i in p)
            wm = max(a[i].window[3] - a[i].window[1] for i in p)
            assert len(p) == 1 or len(p) * hm * wm <= budget


def _container(shapes, pad, tile, rng):
    """A container of random stream bytes with the layout of a `cr` container: (bytes, lens)."""
    from l3c_pytorch_b200.codec import ContainerLayout, tile_grid
    layout = ContainerLayout([(i, C, H, W) for i, (C, H, W) in enumerate(shapes)], tile)
    n = sum(C * len(tile_grid(H, W, tile)) for (C, H, W) in shapes)
    lens = rng.integers(1, 60, n)
    total, pieces, offs = layout.header_and_offsets(lens, pad)
    buf = np.zeros(total, np.uint8)
    for o, b in pieces:
        buf[o:o + len(b)] = np.frombuffer(b, np.uint8)
    for o, ln in zip(offs, lens):
        buf[o:o + ln] = rng.integers(0, 256, ln)
    return buf.tobytes(), lens, layout


def test_offsets_and_splice_segments_give_the_layout():
    from l3c_pytorch_b200.codec import parse_container, splice_segments
    rng = np.random.default_rng(0)
    net = _net('cr')
    for (H, W), tile, pad in [((64, 72), (16, 16), (0, 0, 0, 0)), ((120, 200), (16, 24), (1, 2, 3, 4)),
                              ((64, 64), (64, 64), (0, 0, 0, 0))]:
        shapes = _shapes(net, H, W)
        data, lens, layout = _container(shapes, pad, tile, rng)
        total, _, offs = layout.header_and_offsets(lens, pad)
        assert layout.offsets(lens)[0] == total == len(data)
        assert np.array_equal(layout.offsets(lens)[1], offs)
        old_off = np.array([o for (_, _, _, st) in parse_container(data)[1] for (o, _) in st], np.int64)
        assert np.array_equal(old_off, offs)
        for k in (0, 1, 5, lens.size):
            cols = np.sort(rng.choice(lens.size, k, replace=False))
            new = [rng.integers(0, 256, rng.integers(0, 80)).astype(np.uint8) for _ in cols]
            slot_off = np.concatenate([[0], np.cumsum([len(b) + 4 for b in new])]).astype(np.int64)
            slots = np.zeros(int(slot_off[-1]) + 1, np.uint8)
            for o, b in zip(slot_off, new):
                slots[o:o + len(b)] = b
            new_lens = np.array([len(b) for b in new], np.int64)
            all_lens = lens.copy()
            all_lens[cols] = new_lens
            want_total, pieces, want_offs = layout.header_and_offsets(all_lens, pad)
            want = np.zeros(want_total, np.uint8)
            for o, b in pieces:
                want[o:o + len(b)] = np.frombuffer(b, np.uint8)
            src = np.frombuffer(data, np.uint8)
            streams = {c: b for c, b in zip(cols.tolist(), new)}
            for i, (o, ln) in enumerate(zip(want_offs, all_lens)):
                want[o:o + ln] = streams[i] if i in streams else src[offs[i]:offs[i] + lens[i]]
            got_total, new_off = layout.offsets(all_lens)
            seg = splice_segments(np.asarray(offs, np.int64), lens, len(data), new_off, cols, new_lens,
                                  slot_off[:-1], src0=16, dst0=32)
            assert got_total == want_total
            old = np.concatenate([np.zeros(16, np.uint8), src])
            out = np.full(32 + got_total, 0xEE, np.uint8)
            covered = np.zeros(out.size, bool)
            for s, so, d, n in seg.tolist():
                lo = d - 4 * s
                assert not covered[lo:d + n].any()                      # destinations do not overlap
                covered[lo:d + n] = True
                out[d:d + n] = (slots if s else old)[so:so + n]
                if s:
                    out[d - 4:d] = np.frombuffer(struct.pack('<I', n), np.uint8)
            assert covered[32:].all() and not covered[:32].any()
            assert np.array_equal(out[32:], want)
            assert len(seg) <= 2 * k + 1


def _cpu_codec():
    from l3c_pytorch_b200.codec import BatchCodec
    return BatchCodec(util.blueprint('cr', device='cpu'))


def test_refusals_name_container_and_edit():
    from l3c_pytorch_b200.codec import BatchCodec
    rng = np.random.default_rng(1)
    net = _net('cr')
    bc = _cpu_codec()
    data = _container(_shapes(net, 64, 72), (0, 0, 0, 0), (16, 16), rng)[0]
    ref = _container(_shapes(net, 64, 72), (0, 0, 0, 0), None, rng)[0]
    rgb_shapes = [(3, 8, 9), (3, 16, 18), (3, 32, 36), (3, 64, 72)]
    rgb_data = _container(rgb_shapes, (0, 0, 0, 0), (16, 16), rng)[0]
    ok = torch.zeros(3, 4, 4, dtype=torch.uint8)
    good = [((0, 0), ok)]
    cases = [([data, ref], [good, good], r'container 1: .*tiled container'),
             ([data, rgb_data], [[], []], 'container 1 was not written by this model'),
             ([data[:-3]], [good], 'container 0 was not written by this model'),
             ([data, data], [good, good + [((0, 0), torch.zeros(3, 0, 4, dtype=torch.uint8))]],
              'container 1, edit 1: empty'),
             ([data], [good + [((62, 0), ok)]], 'container 0, edit 1: .*outside'),
             ([data], [[((0, -1), ok)]], 'container 0, edit 0: .*outside'),
             ([data], [good * 3 + [((0, 0), torch.zeros(1, 4, 4, dtype=torch.uint8))]],
              'container 0, edit 3: .*3 channels'),
             ([data], [[((0, 0), torch.full((3, 4, 4), 256, dtype=torch.int64))]], 'edit 0: .*0..255'),
             ([data], [[((0, 0), torch.zeros(3, 4, 4, dtype=torch.float32))]], 'edit 0: .*uint8 or int64'),
             ([data], [[((0, 0, 0), ok)]], r'edit 0: pos must be \(y, x\)'),
             ([data], [[((0, 0),)]], r'edit 0: an edit is \(pos, patch\)'),
             ([data], [good, good], '2 edit lists for 1 containers')]
    for ds, eds, match in cases:
        with pytest.raises(ValueError, match=match):
            bc.update_regions(ds, eds)
    rgb = BatchCodec(util.blueprint('cr_rgb_shared', device='cpu'))
    with pytest.raises(ValueError, match='container 0: .*RGB baselines'):
        rgb.update_regions([rgb_data], [[]])
    # nothing refused: the plans of a valid call, empty lists included
    jobs = bc.plan_updates([data, data], [good + [((60, 68), ok)], []])
    assert [len(j.plans) for j in jobs] == [1, 0] and not jobs[0].whole
