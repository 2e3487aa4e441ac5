"""CPU: the planner of region updates (DESIGN §4.12), region.plan_update.

* NaN dependency checks with float64 torch CPU convs on the module weights of an L3C network with the architecture of
  `cr` (three scales, dec.skip) but 8 feature channels and one residual block per body, so that images of a few
  hundred pixels have windows smaller than the image:
  - with the edited pixels NaN, NaN reaches the symbols and CDF parameters of every scale only inside the planned
    rectangle R_s: R_s is a superset of the streams that can change;
  - with every input NaN outside its planned window (each encoder's input window, each decoder's window of the coarser
    symbols and features), everything the plan reads comes out finite: the encoder outputs on `need`, the CDF
    parameters on R_s and the decoder features the finer decoder adds;
  - moving any window edge that is not a plane edge one stride step inward (2 pixels for an encoder window, 1 coarse
    pixel for a decoder window) lets NaN in: the margins are not loose.
* Geometry of `cr`: tile alignment, even encoder-window starts, nesting of the windows, totals, the whole-image edit
  and the refusals."""
import pytest
import torch
import torch.nn.functional as Fn

from tests import util

NAN = float('nan')


def _small_net():
    from l3c_pytorch_b200 import config
    from l3c_pytorch_b200.blueprint import MultiscaleBlueprint
    cfg = config.ms_config('cr')
    cfg.Cf, cfg.enc.num_blocks, cfg.dec.num_blocks = 8, 1, 1
    torch.manual_seed(0)
    bp = MultiscaleBlueprint(cfg, device='cpu')
    bp.set_eval()
    return bp.net


_NET = {}


def _net(name):
    if name not in _NET:
        _NET[name] = _small_net() if name == 'small' else util.blueprint(name, device='cpu').net
    return _NET[name]


def _shapes(net, H, W):
    """[(C, H, W)] coarse -> fine of a container of an H x W (padded) image."""
    return [(3 if s == 0 else net.config_ms.q.C, H >> s, W >> s) for s in reversed(range(net.scales + 1))]


def _conv(m, x):
    return Fn.conv2d(x, m.weight.detach().double(), None if m.bias is None else m.bias.detach().double(), m.stride,
                     m.padding, m.dilation)


def _res_body(body, x):
    blocks = list(body)
    y = x
    for blk in blocks[:-1]:
        y = _conv(blk.body[2], torch.relu(_conv(blk.body[0], y))) + y
    return _conv(blocks[-1], y) + x


def _enc(net, s, x):
    """heads[s] + nets[s].enc on NCHW float64: -> (F_{s+1}, to_q output)."""
    enc = net.nets[s].enc
    head = net.heads[0].head[1].head if s == 0 else net.heads[s].head
    d = _conv(enc.down, _conv(head, x))
    F = _res_body(enc.body, d)
    return F, _conv(enc.to_q[0], F)


def _dec(net, s, bn, fuse):
    """nets[s].dec + prob_clfs[s] on NCHW float64: -> (decoder features, CDF parameters)."""
    dec, clf = net.nets[s].dec, net.prob_clfs[s]
    x = _conv(dec.head, bn)
    if fuse is not None:
        x = x + fuse
    D = Fn.pixel_shuffle(_conv(dec.tail[0], _res_body(dec.body, x)), 2)
    return D, _conv(clf.atrous.lin, torch.cat([_conv(a, D) for a in clf.atrous.atrous], 1))


def _crop(t, r):
    return t[:, :, r[0]:r[2], r[1]:r[3]]


def _nan_outside(t, r):
    out = torch.full_like(t, NAN)
    out[:, :, r[0]:r[2], r[1]:r[3]] = _crop(t, r)
    return out


def _nan_rows_cols(t):
    """Bounding rectangle of the NaN entries of t [1, C, H, W], or None."""
    bad = torch.isnan(t).any(1)[0]
    if not bad.any():
        return None
    ys, xs = torch.nonzero(bad, as_tuple=True)
    return (int(ys.min()), int(xs.min()), int(ys.max()) + 1, int(xs.max()) + 1)


def _inside(a, b):
    return a is None or (b[0] <= a[0] and b[1] <= a[1] and a[2] <= b[2] and a[3] <= b[3])


def _finite(t, r):
    return bool(torch.isfinite(_crop(t, r)).all())


CASES = [  # (unpadded H, W), pad tuple (left, right, top, bottom), edit (y, x, h, w), tile
    ((397, 291), (2, 3, 1, 2), (190, 140, 20, 12), (16, 16)),       # interior, sizes not multiples of 8
    ((397, 291), (2, 3, 1, 2), (0, 100, 9, 30), (16, 24)),          # top edge
    ((397, 291), (2, 3, 1, 2), (200, 285, 30, 6), (16, 16)),        # right edge
    ((397, 291), (2, 3, 1, 2), (390, 0, 7, 8), (16, 24)),           # bottom-left corner
    ((400, 296), (0, 0, 0, 0), (211, 97, 1, 1), (16, 24)),          # one pixel
    ((400, 296), (0, 0, 0, 0), (0, 0, 400, 296), (16, 16)),         # the whole image
]


def _plan(case, name='small'):
    from l3c_pytorch_b200.region import plan_update
    (Hu, Wu), pad, edit, tile = case
    net = _net(name)
    shapes = _shapes(net, Hu + pad[2] + pad[3], Wu + pad[0] + pad[1])
    return net, shapes, plan_update(shapes, pad, tile, net, edit)


def _by_scale(plan):
    return {sp.scale: sp for sp in plan.scales}


@pytest.mark.parametrize('case', CASES)
def test_nan_from_the_edit_stays_inside_the_planned_rectangles(case):
    net, shapes, plan = _plan(case)
    sc = _by_scale(plan)
    S = net.scales
    g = torch.Generator().manual_seed(1)
    _, H, W = shapes[-1]
    x = torch.rand(1, 3, H, W, generator=g, dtype=torch.float64) * 2 - 1
    e = plan.edit
    x[:, :, e[0]:e[2], e[1]:e[3]] = NAN
    q, inp = [x], x
    for s in range(S):
        inp, qs = _enc(net, s, inp)
        q.append(qs)
        assert _nan_rows_cols(qs) is not None
        assert _inside(_nan_rows_cols(qs), sc[s + 1].rect), (s + 1, _nan_rows_cols(qs), sc[s + 1])
    D = None
    for s in reversed(range(S)):
        D, P = _dec(net, s, q[s + 1], D if net.fuses(s) else None)
        bad = _nan_rows_cols(P)
        assert bad is not None and _inside(bad, sc[s].rect), (s, bad, sc[s])


def _window_run(net, shapes, plan, shrink=None):
    """Every stage of the plan on full-size planes, every input NaN outside its window; shrink = (kind, scale, edge):
    that window one stride step smaller on that edge.  -> [(what, ok)] per rectangle the plan reads."""
    sc = _by_scale(plan)
    S = net.scales
    g = torch.Generator().manual_seed(2)
    _, H, W = shapes[-1]
    x = torch.rand(1, 3, H, W, generator=g, dtype=torch.float64) * 2 - 1

    def win(kind, s):
        r = list(sc[s].enc if kind == 'enc' else sc[s].window)
        if shrink is not None and shrink[:2] == (kind, s):
            step = 2 if kind == 'enc' else 1
            r[shrink[2]] += step if shrink[2] < 2 else -step
        return r

    checks = [('image R_0', _finite(x, sc[0].rect))]
    q, inp = [None], _nan_outside(x, win('enc', 0))
    for s in range(S):
        F, qs = _enc(net, s, inp)
        checks.append(('encoder %d' % s, _finite(F, sc[s + 1].need) and _finite(qs, sc[s + 1].need)))
        q.append(qs)
        if s + 1 < S:
            inp = _nan_outside(F, win('enc', s + 1))
    D = None
    for s in reversed(range(S)):
        w = win('dec', s)
        D, P = _dec(net, s, _nan_outside(q[s + 1], w), _nan_outside(D, w) if sc[s].fused else None)
        checks.append(('params %d' % s, _finite(P, sc[s].rect)))
        if s >= 1 and sc[s - 1].fused:
            checks.append(('features %d' % s, _finite(D, sc[s - 1].window)))
    return checks


@pytest.mark.parametrize('case', CASES)
def test_planned_windows_read_nothing_outside_and_are_tight(case):
    net, shapes, plan = _plan(case)
    checks = _window_run(net, shapes, plan)
    assert all(ok for _, ok in checks), checks
    tested = 0
    for sp in plan.scales:
        for kind, r, lim in (('enc', sp.enc, (sp.H, sp.W)), ('dec', sp.window, shapes[sp.idx - 1][1:])):
            if r is None:
                continue
            for e, at_edge in enumerate((r[0] == 0, r[1] == 0, r[2] == lim[0], r[3] == lim[1])):
                if at_edge:
                    continue
                checks = _window_run(net, shapes, plan, shrink=(kind, sp.scale, e))
                assert not all(ok for _, ok in checks), 'edge %d of the %s window of %s is loose' % (e, kind, sp)
                tested += 1
    whole = case[2][2:] == case[0]
    assert tested == 0 if whole else tested >= 4


def _check_geometry(plan, shapes, tile):
    th, tw = tile
    n = len(shapes)
    assert [sp.idx for sp in plan.scales] == list(range(n))
    for sp in plan.scales:
        y0, x0, y1, x1 = sp.rect
        assert y0 % th == 0 and x0 % tw == 0 and (y1 % th == 0 or y1 == sp.H) and (x1 % tw == 0 or x1 == sp.W)
        ntx = -(-sp.W // tw)
        assert sp.tiles == [ty * ntx + tx for ty in range(y0 // th, -(-y1 // th)) for tx in range(x0 // tw, -(-x1 // tw))]
        assert _inside(sp.rect, sp.need)
        if sp.enc is None:
            assert sp.idx == 0 and sp.window is None
            continue
        assert sp.enc[0] % 2 == 0 and sp.enc[1] % 2 == 0 and _inside(sp.enc, sp.need)
        assert _inside(sp.enc, (0, 0, sp.H, sp.W))
        oy0, ox0, oy1, ox1 = sp.out
        wy0, wx0, wy1, wx1 = sp.window
        assert (oy0, ox0) == (y0 - 2 * wy0, x0 - 2 * wx0) and oy1 <= 2 * (wy1 - wy0) and ox1 <= 2 * (wx1 - wx0)
    for fine, coarse in zip(plan.scales[1:], plan.scales[:-1]):
        assert _inside(fine.window, coarse.need)                          # the symbols a decoder window reads
        e = fine.enc                                                      # what the encoder of `fine` produces
        assert _inside((e[0] // 2, e[1] // 2, e[2] // 2, e[3] // 2), (0, 0, coarse.H, coarse.W))
    assert plan.window == plan.scales[-1].need
    assert plan.streams == sum(sp.C * len(sp.tiles) for sp in plan.scales)
    assert plan.window_pixels == (plan.window[2] - plan.window[0]) * (plan.window[3] - plan.window[1])


def test_geometry_of_cr():
    from l3c_pytorch_b200.codec import tile_grid
    from l3c_pytorch_b200.region import plan_update
    net = _net('cr')
    for (H, W), tile in (((1024, 768), (64, 64)), ((520, 776), (16, 24)), ((200, 312), (16, 16))):
        shapes = _shapes(net, H, W)
        total = sum(C * len(tile_grid(h, w, tile)) for (C, h, w) in shapes)
        for edit in [(0, 0, 1, 1), (H - 1, W - 1, 1, 1), (H // 2, W // 2, 30, 40), (0, W // 3, 9, 30),
                     (H // 3, 0, 20, 9), (0, 0, H, W)]:
            plan = plan_update(shapes, (0, 0, 0, 0), tile, net, edit)
            _check_geometry(plan, shapes, tile)
            assert plan.total_streams == total and plan.streams <= total
            assert plan.edit == (edit[0], edit[1], edit[0] + edit[2], edit[1] + edit[3])
        whole = plan_update(shapes, (0, 0, 0, 0), tile, net, (0, 0, H, W))
        assert whole.streams == total and whole.window == (0, 0, H, W)
    # an interior edit of a large image re-encodes a fraction of its streams from a window of its pixels
    shapes = _shapes(net, 3072, 4096)
    plan = plan_update(shapes, (0, 0, 0, 0), (64, 64), net, (1408, 1920, 256, 256))
    assert plan.streams < plan.total_streams // 4 and plan.window_pixels < 3072 * 4096 // 2


def test_padding_tuples_shift_the_edit():
    from l3c_pytorch_b200.region import plan_update
    net = _net('cr')
    shapes = _shapes(net, 64, 72)
    pad = (3, 5, 2, 6)
    Hu, Wu = 64 - 8, 72 - 8
    assert plan_update(shapes, pad, (16, 16), net, (0, 0, 1, 1)).edit == (2, 3, 3, 4)
    assert plan_update(shapes, pad, (16, 16), net, (Hu - 2, Wu - 3, 2, 3)).edit == (Hu, Wu, Hu + 2, Wu + 3)
    for bad in [(Hu - 1, 0, 2, 1), (0, Wu, 1, 1), (-1, 0, 1, 1)]:
        with pytest.raises(ValueError, match='outside'):
            plan_update(shapes, pad, (16, 16), net, bad)


def test_refusals():
    from l3c_pytorch_b200.region import plan_update
    net = _net('cr')
    shapes = _shapes(net, 64, 64)
    for tile, edit, match in [(None, (0, 0, 1, 1), 'tiled container'), ((16, 16), (0, 0, 0, 4), 'empty'),
                              ((16, 16), (0, 0, 4, -1), 'empty'), ((16, 16), (60, 0, 8, 4), 'outside'),
                              ((16, 16), (0, 0, 4), r'\(y, x, h, w\)')]:
        with pytest.raises(ValueError, match=match):
            plan_update(shapes, (0, 0, 0, 0), tile, net, edit)
    with pytest.raises(ValueError, match='model expects'):
        plan_update(shapes[1:], (0, 0, 0, 0), (16, 16), net, (0, 0, 1, 1))
    rgb = _net('cr_rgb_shared')
    with pytest.raises(ValueError, match='RGB baselines'):
        plan_update([(3, 32, 32), (3, 64, 64)], (0, 0, 0, 0), (16, 16), rgb, (0, 0, 1, 1))
