"""Region decode of tiled containers (DESIGN §4.8): which tile streams and decoder windows a crop of the image
depends on.  Pure host code.

Every tile of a tiled container is an independent stream whose symbols depend only on their CDF rows, and a row
depends on the coarser scale only within the bounded receptive field of the decoder network and the probability
classifier.  Every conv kernel computes an output pixel the same way wherever it sits in the tensor, so a decoder
network run on a window of the coarser scale gives, inside the window shrunk by that field, exactly the bits of the
full run.  `plan_region` walks the scales fine to coarse:

  tiles needed at scale s  ->  their P_s rectangle  ->  widened by the classifier's radius (fine grid), halved
  (Upsampler x2), widened by the tail, body and head radii (coarse grid) and clipped to the image: the window of
  bn_{s+1} the decoder of scale s runs on  ->  (with dec.skip) the F_{s+1} region that decoder adds after its
  head  ->  the union, tile-aligned: the tiles needed at scale s+1  ->  ... up to the uniform-prior scale.

At a clipped edge the window edge is the image edge, so the kernels' zero padding is the image's own.  Rectangles
are tile-aligned (their start on a tile boundary, their end on one or at the plane's edge), so `tile_grid` cuts them
into the same tiles, in the same order, as the full plane.

A reference-layout container with a seek index (DESIGN §4.13 "Regions") is planned in full-width bands instead: its
plane is one stream per channel in raster order, so the symbols a scale needs are the rows [a, b) of the finer window
(of the region at the finest level), and its stream decodes them from the seek point at or before the band's first
symbol (ScalePlan.seg).
"""
import numpy as np

from .codec import tile_grid


def _radius(conv):
    """Pixels a same-size conv reads on each side of its output pixel."""
    return conv.dilation[0] * (conv.kernel_size[0] - 1) // 2


class Radii(object):
    """Receptive radii of one scale's decoder (head, body, tail: on the coarse grid) and classifier (fine grid)."""
    __slots__ = ('head', 'body', 'tail', 'clf')

    def __init__(self, dec, clf):
        self.head = _radius(dec.head)
        body = list(dec.body)
        self.body = sum(_radius(m.body[0]) + _radius(m.body[2]) for m in body[:-1]) + _radius(body[-1])
        self.tail = _radius(dec.tail[0])
        self.clf = max(_radius(a) for a in clf.atrous.atrous) + _radius(clf.atrous.lin)


class DecoderGeometry(object):
    """What the planner needs of a MultiscaleNetwork, read from its module tree: the radii of every trained
    scale's decoder and classifier, which scales fuse the coarser decoder's features (dec.skip), and whether the
    scales are images (RGB baselines)."""

    def __init__(self, net):
        self.num_scales = net.scales
        self.rgb = bool(net._rgb)
        self.fuses = net.fuses
        self.radii = [Radii(net.nets[s].dec, net.prob_clfs[s]) for s in range(net.scales)]

    def radii_of(self, scale):
        """Recursive scales (scale >= num_scales) run nets[-1] / prob_clfs[-1]."""
        return self.radii[min(scale, self.num_scales - 1)]


def geometry_of(config):
    return config if isinstance(config, DecoderGeometry) else DecoderGeometry(config)


def _expand(r, m):
    return (r[0] - m, r[1] - m, r[2] + m, r[3] + m)


def _clip(r, H, W):
    return (max(r[0], 0), max(r[1], 0), min(r[2], H), min(r[3], W))


def _union(a, b):
    return (min(a[0], b[0]), min(a[1], b[1]), max(a[2], b[2]), max(a[3], b[3]))


def _area(r):
    return (r[2] - r[0]) * (r[3] - r[1])


def _align(r, H, W, tile):
    th, tw = tile
    return (r[0] // th * th, r[1] // tw * tw, min(-(-r[2] // th) * th, H), min(-(-r[3] // tw) * tw, W))


class ScalePlan(object):
    """One scale of a region plan.  Rectangles are (y0, x0, y1, x1), half-open.
    rect: the tile-aligned symbols decoded, in this scale's coordinates; tiles: their indices in the plane's tile
    grid (tile_grid order).  For a scale with a decoder network: window, the bn_{s+1} rectangle (coarser scale's
    coordinates) its network runs on; out, the rectangle of that network's output (2x the window) that is exact
    and used, i.e. rect relative to 2 * window's origin; fused, whether the coarser decoder's features are added.
    The uniform-prior scale has window = out = None.
    seg: None for a tiled container; for a band of a reference-layout container (every channel one stream, tiles
    [0]) the symbols (s0, s1) of every channel's stream that are decoded: s0 the seek point at or before the band's
    first needed symbol, s1 = b * W.  rect is then (s0 // W, 0, b, W), and its symbols before s0 are not decoded."""
    __slots__ = ('idx', 'scale', 'C', 'H', 'W', 'rect', 'tiles', 'window', 'out', 'fused', 'seg')

    def __init__(self, **kw):
        self.seg = None
        for k, v in kw.items():
            setattr(self, k, v)

    @property
    def streams(self):
        return self.C * len(self.tiles)

    @property
    def symbols(self):
        """symbols handed to the range decoder"""
        return self.C * (_area(self.rect) if self.seg is None else self.seg[1] - self.seg[0])

    @property
    def window_pixels(self):
        return 0 if self.window is None else _area(self.window)

    def shape_key(self):
        r, w = self.rect, self.window
        return (self.C, r[2] - r[0], r[3] - r[1], None if w is None else (w[2] - w[0], w[3] - w[1]), self.out,
                self.fused, len(self.tiles))

    def __repr__(self):
        return 'ScalePlan(scale=%d, rect=%s, tiles=%d, window=%s, out=%s, fused=%s%s)' % (
            self.scale, self.rect, len(self.tiles), self.window, self.out, self.fused,
            '' if self.seg is None else ', seg=%s' % (self.seg,))


class RegionPlan(object):
    """plan_region's result: scales coarse -> fine (the finest is the requested level), the region in that level's
    plane, and the totals.  tile None: bands of a reference-layout container whose seek points lie every `every`
    symbols; `seek`, its parsed index (seek.SeekIndex), is set by BatchCodec.plan_regions."""

    def __init__(self, scales, region, level, tile, n_scales, recursive, every=None):
        self.scales, self.region, self.level, self.tile = scales, region, level, tile
        self.n_scales, self.recursive = n_scales, recursive
        self.every, self.seek = every, None

    @property
    def tiles(self):
        return sum(len(s.tiles) for s in self.scales)

    @property
    def streams(self):
        return sum(s.streams for s in self.scales)

    @property
    def symbols(self):
        return sum(s.symbols for s in self.scales)

    @property
    def window_pixels(self):
        return sum(s.window_pixels for s in self.scales)

    def shape_key(self):
        """Plans with equal keys decode as one batch (BatchCodec.decode_regions): every rectangle has the same size
        and every network output the same used rectangle, wherever the regions lie, and the regions have one size
        (regions of different sizes inside the same tiles plan the same rectangles)."""
        r = self.region
        return (self.tile, self.n_scales, self.level, (r[2] - r[0], r[3] - r[1]),
                tuple(s.shape_key() for s in self.scales))

    def pass_key(self):
        """Plans with equal keys walk the same scales with the same tile size: where ragged windows are supported they
        decode in one pass whatever their shape_key (BatchCodec.decode_regions)."""
        return (self.tile, self.n_scales, self.level)

    def __repr__(self):
        return 'RegionPlan(level=%d, region=%s, tiles=%d, symbols=%d, window_pixels=%d)' % (
            self.level, self.region, self.tiles, self.symbols, self.window_pixels)


def plan_region(shapes, pad_tuple, tile, config, region, level=0, every=None):
    """shapes: [(C, H, W)] of a container's scales, coarse -> fine; pad_tuple: its (left, right, top, bottom);
    tile: its (th, tw), None for the reference layout; config: a MultiscaleNetwork or its DecoderGeometry;
    region = (y, x, h, w): at level 0 in unpadded image coordinates, at level k >= 1 (RGB baselines) in the
    coordinates of the stored scale-k plane; every: the interval K of the seek index of a reference-layout container.
    -> RegionPlan.  A reference-layout plan is one full-width band per scale: rows [a, b) of the finer window (of the
    region at the finest level), and of every channel's stream the symbols [K floor(a W / K), b W) (ScalePlan.seg).
    ValueError for an untiled container without `every`, an empty region or one outside the image, and a level that
    does not exist."""
    geo = geometry_of(config)
    if tile is None and every is None:
        raise ValueError('region decode needs a tiled container (written with Bitcoding(..., tile=(th, tw))) or the '
                         'seek index of a reference-layout one (Bitcoding.seek_index, `idx IN.l3c`): the streams of '
                         'the reference layout are serial')
    if tile is not None:
        tile = (int(tile[0]), int(tile[1]))
    else:
        every = int(every)
    n = len(shapes)
    recursive = n - geo.num_scales - 1
    if recursive < 0:
        raise ValueError('container has %d scales, model expects %d' % (n, geo.num_scales + 1))
    if isinstance(level, bool) or not isinstance(level, (int, np.integer)) or level < 0 or level >= n:
        raise ValueError('level %r does not exist: the container stores levels 0 .. %d' % (level, n - 1))
    level = int(level)
    if level > 0 and not geo.rgb:
        raise ValueError('level %d: only the RGB baselines store images at the coarser scales; the L3C bottlenecks '
                         'are not images' % level)
    if len(region) != 4:
        raise ValueError('region must be (y, x, h, w), got %r' % (region,))
    y, x, h, w = (int(v) for v in region)
    idx_f = n - 1 - level
    _, Hf, Wf = shapes[idx_f]
    if level == 0:
        left, right, top, bottom = (int(v) for v in pad_tuple)
        Hu, Wu, oy, ox = Hf - top - bottom, Wf - left - right, top, left
    else:
        Hu, Wu, oy, ox = Hf, Wf, 0, 0
    if h < 1 or w < 1:
        raise ValueError('empty region %r' % (tuple(region),))
    if y < 0 or x < 0 or y + h > Hu or x + w > Wu:
        raise ValueError('region %r lies outside the %dx%d image' % (tuple(region), Hu, Wu))
    want = (y + oy, x + ox, y + oy + h, x + ox + w)
    region_px = want
    plans = []
    for idx in range(idx_f, -1, -1):
        C, H, W = shapes[idx]
        scale = n - 1 - idx
        seg = None
        if tile is None:
            # a full-width band: the stream decodes from the seek point at or before the band's first symbol, and
            # its rows reach back to that point's row (those rows' CDFs are needed to decode up to the band)
            seg = (want[0] * W // every * every, want[2] * W)
            rect, tiles = (seg[0] // W, 0, want[2], W), [0]
        else:
            rect = _align(want, H, W, tile)
            th, tw = tile
            ntx = -(-W // tw)
            tiles = [ty * ntx + tx for ty in range(rect[0] // th, -(-rect[2] // th))
                     for tx in range(rect[1] // tw, -(-rect[3] // tw))]
        if idx == 0:                                                 # the uniform-prior thumbnail
            plans.append(ScalePlan(idx=idx, scale=scale, C=C, H=H, W=W, rect=rect, tiles=tiles, window=None,
                                   out=None, fused=False, seg=seg))
            break
        Hc, Wc = shapes[idx - 1][1:]
        window, out, fused, want = _window(geo, scale, rect, H, W, Hc, Wc)
        plans.append(ScalePlan(idx=idx, scale=scale, C=C, H=H, W=W, rect=rect, tiles=tiles, window=window, out=out,
                               fused=fused, seg=seg))
    plans.reverse()
    return RegionPlan(plans, region_px, level, tile, n, recursive, every)


def band_tile(plans, idx):
    """The tile the layout kernels (l3c_dmll_build_table_window(s), l3c_reorder_tiles(_images)) are given for scale idx
    of a pass of reference-layout band plans: one row tall and as wide as the pass's widest band.  Tiles that span the
    plane's width put it in raster order whatever their height, and with one row every in-tile product (th * W,
    tw * h) stays at most the band's width."""
    return (1, max(p.scales[idx].W for p in plans))


def _window(geo, scale, rect, H, W, Hc, Wc, features=None):
    """The decoder window of the symbols `rect` of an H x W plane at `scale`, on the Hc x Wc coarser plane: -> (window,
    out, fused, want), `want` being the coarser rectangle the window and (fused) the coarser decoder's features need.
    features: a rectangle of this decoder's own output features that must come out exact as well (the ones a finer
    decoder adds, plan_update)."""
    r = geo.radii_of(scale)
    need_F = _clip(_expand(rect, r.clf), H, W)                   # decoder features the classifier reads
    if features is not None:
        need_F = _union(need_F, features)
    coarse = (need_F[0] // 2, need_F[1] // 2, -(-need_F[2] // 2), -(-need_F[3] // 2))   # Upsampler x2
    window = _clip(_expand(coarse, r.tail + r.body + r.head), Hc, Wc)
    fused = geo.fuses(scale)
    want = window
    if fused:                                                    # F_{s+1}, added after the head
        want = _union(want, _clip(_expand(coarse, r.tail + r.body), Hc, Wc))
    out = (rect[0] - 2 * window[0], rect[1] - 2 * window[1], rect[2] - 2 * window[0], rect[3] - 2 * window[1])
    return window, out, fused, want


def plan_bands(shapes, tile, config, idx, rows):
    """Banded decode of scale `idx` of a tiled container (DESIGN §4.10): its H x W plane cut into horizontal bands of
    `rows` tile rows (the last one partial), each decoded from its own decoder window of the whole coarser scale.
    shapes, tile, config: as in plan_region.  -> [ScalePlan] top to bottom; band b's rect is (y0, 0, y1, W) and its
    tiles are consecutive in container order, so its symbols are the elements [y0 * W, y1 * W) of every channel plane in
    stream order.  Every window and `out` is what plan_region plans for the same rectangle."""
    geo = geometry_of(config)
    n = len(shapes)
    if not 1 <= idx < n:
        raise ValueError('scale index %d has no decoder network (a container of %d scales)' % (idx, n))
    th, tw = (int(tile[0]), int(tile[1]))
    rows = int(rows)
    if rows < 1:
        raise ValueError('a band needs at least one tile row, got %d' % rows)
    C, H, W = shapes[idx]
    Hc, Wc = shapes[idx - 1][1:]
    scale = n - 1 - idx
    ntx, nty = -(-W // tw), -(-H // th)
    bands = []
    for ty0 in range(0, nty, rows):
        ty1 = min(ty0 + rows, nty)
        rect = (ty0 * th, 0, min(ty1 * th, H), W)
        window, out, fused, _ = _window(geo, scale, rect, H, W, Hc, Wc)
        bands.append(ScalePlan(idx=idx, scale=scale, C=C, H=H, W=W, rect=rect,
                               tiles=list(range(ty0 * ntx, ty1 * ntx)), window=window, out=out, fused=fused))
    return bands


def rect_columns(sp, T):
    """Columns of the streams of the tile-aligned rectangle sp (ScalePlan) in the stream list of its scale, which has T
    tiles per channel (a tiled container's order): channel-major, in tile order within a channel."""
    return (np.arange(sp.C)[:, None] * T + np.asarray(sp.tiles, np.int64)[None, :]).reshape(-1)


def stream_columns(plan, tile):
    """Indices, in container order, of the planned streams of every scale: [[column in that scale's stream list]]
    coarse -> fine (rect_columns).  A band plan (tile None) lists every channel's one stream."""
    return [rect_columns(sp, len(tile_grid(sp.H, sp.W, tile))) for sp in plan.scales]


def rect_streams(layout, idx, sp):
    """The streams of the tile-aligned rectangle sp (a ScalePlan: a band, an update's R_s, a whole plane) of scale idx
    of a pass of equal-size images laid out by codec.stream_layout.  -> (cols, n_sym, elem) int64: its columns of the
    pass's [N][streams] arrays (rect_columns), their symbol counts [N][cols] and their first elements in the
    rectangle's own [N][C][h * w] planes in tile order.  tile_grid cuts a tile-aligned rectangle into the plane's tiles,
    in the plane's order, so a stream starts where the rectangle's earlier tiles of its channel end."""
    si, _, n_sym, _ = layout
    lo, hi = np.searchsorted(si[0], [idx, idx + 1])
    cols = lo + rect_columns(sp, (hi - lo) // sp.C)
    n = n_sym[:, cols]
    N = n.shape[0]
    per_c = n.reshape(N, sp.C, -1)
    elem = np.arange(N * sp.C).reshape(N, sp.C, 1) * _area(sp.rect) + np.cumsum(per_c, 2) - per_c
    return cols, n, elem.reshape(N, -1)


def pass_streams(plans, streams_of, starts):
    """Where the streams of one pass of plans lie in the uploaded containers, the counterpart of
    codec.stream_layout(pad_tiles=True): streams_of[n][scale idx] = [(offset, length)] of plan n's container
    (parse_container), starts[n] = where that container begins.  -> (offs, lens) int64 [N][streams]: per scale and
    channel the planned streams in the order of stream_columns, every channel's list padded to the pass's largest tile
    count of that scale with empty streams (the container's start, length 0), which read nothing."""
    T_max = [max(len(p.scales[k].tiles) for p in plans) for k in range(len(plans[0].scales))]
    offs, lens = [], []
    for p, streams, start in zip(plans, streams_of, starts):
        o, ln = [], []
        for k, (sp, cs) in enumerate(zip(p.scales, stream_columns(p, p.tile))):
            T = len(sp.tiles)
            for c in range(sp.C):
                for col in cs[c * T:(c + 1) * T]:
                    o.append(start + streams[sp.idx][col][0])
                    ln.append(streams[sp.idx][col][1])
                o += [start] * (T_max[k] - T)
                ln += [0] * (T_max[k] - T)
        offs.append(o)
        lens.append(ln)
    return np.array(offs, np.int64), np.array(lens, np.int64)


def plan_passes(plans, ragged):
    """How BatchCodec.decode_regions runs a list of plans: -> [(indices into plans, is_ragged)] in order of first
    appearance.  Plans of one shape_key always share a pass of equal shapes.  ragged (the decoder networks can run
    padded batches of windows): plans of one pass_key share one ragged pass, unless their shape_keys are all equal."""
    groups = {}
    for i, p in enumerate(plans):
        groups.setdefault(p.pass_key() if ragged else p.shape_key(), []).append(i)
    return [(idxs, len({plans[i].shape_key() for i in idxs}) > 1) for idxs in groups.values()]


class EncoderGeometry(object):
    """What plan_encoder_bands needs of a MultiscaleNetwork, read from its module tree: per trained scale the radii
    of heads[s] (3x3; the RGB head at scale 0), enc.down (5x5/s2), the encoder body and to_q (1x1).  The RGB
    baselines have no encoder network (their bicubic x0.5 runs whole): radii is empty then."""

    def __init__(self, net):
        self.num_scales = net.scales
        self.rgb = bool(net._rgb)
        self.radii = []
        if self.rgb:
            return
        for s in range(net.scales):
            enc = net.nets[s].enc
            head = net.heads[0].head[1].head if s == 0 else net.heads[s].head
            body = list(enc.body)
            self.radii.append(dict(
                head=_radius(head), down=enc.down.dilation[0] * (enc.down.kernel_size[0] - 1) // 2,
                body=sum(_radius(m.body[0]) + _radius(m.body[2]) for m in body[:-1]) + _radius(body[-1]),
                to_q=_radius(enc.to_q[0])))


class EncoderBand(object):
    """One band of the encoder of a scale: rows = [r0, r1) of the scale-(s+1) planes it writes (S, bottleneck values,
    F); window = [a, b) the rows of the full-width scale-s input (the image or F_s) it runs on, a even; out = r0 - a/2,
    where its rows start in the window's output."""
    __slots__ = ('scale', 'rows', 'window', 'out')

    def __init__(self, scale, rows, window):
        self.scale, self.rows, self.window = scale, rows, window
        self.out = rows[0] - window[0] // 2

    def __repr__(self):
        return 'EncoderBand(scale=%d, rows=%s, window=%s)' % (self.scale, self.rows, self.window)


def encoder_window(geo, scale, r0, r1, H):
    """The rows of the H-row input of scale `scale`'s encoder that its output rows [r0, r1) depend on (DESIGN §4.10):
    widened by the body (and to_q) radius, doubled, widened by the down conv's and the head's radii, clipped to the
    plane and started on an even row (the stride-2 grid of the full run).  -> (a, b)."""
    r = geo.radii[scale]
    m = r['body'] + r['to_q']
    a, b = 2 * (r0 - m) - r['down'] - r['head'], 2 * (r1 + m) + r['down'] + r['head']
    a, b = max(a, 0), min(b, H)
    return a - a % 2, b


def plan_encoder_bands(config, scale, H, rows):
    """Banded encoder of trained scale `scale` (0 .. num_scales - 1) of an L3C network whose input plane has H rows:
    its H / 2 output rows cut into bands of `rows` rows (the last one partial), top to bottom.  config: a
    MultiscaleNetwork or its EncoderGeometry.  -> [EncoderBand]."""
    geo = config if isinstance(config, EncoderGeometry) else EncoderGeometry(config)
    if geo.rgb:
        raise ValueError('the RGB baselines have no encoder network to band (their bicubic x0.5 runs whole)')
    if not 0 <= scale < geo.num_scales:
        raise ValueError('scale %d has no encoder (the network has %d scales)' % (scale, geo.num_scales))
    rows = int(rows)
    if rows < 1:
        raise ValueError('a band needs at least one row, got %d' % rows)
    Ho = H // 2
    return [EncoderBand(scale, (r0, min(r0 + rows, Ho)), encoder_window(geo, scale, r0, min(r0 + rows, Ho), H))
            for r0 in range(0, Ho, rows)]


def encoder_rect(geo, scale, rect, H, W):
    """encoder_window on both axes: the rectangle of the H x W input of scale `scale`'s encoder that its output
    rectangle `rect` (y0, x0, y1, x1) depends on, clipped to the plane and started on an even row and column."""
    a0, a1 = encoder_window(geo, scale, rect[0], rect[2], H)
    b0, b1 = encoder_window(geo, scale, rect[1], rect[3], W)
    return (a0, b0, a1, b1)


def _encoder_reach(geo, scale, r, Ho, Wo):
    """The outputs of scale `scale`'s encoder (an Ho x Wo plane) that the input rectangle r can change: output pixel p
    reads the inputs [2 (p - m) - k, 2 (p + m) + k] (m: body and to_q radius, k: down conv and head radii), on both
    axes.  The inverse of encoder_rect."""
    g = geo.radii[scale]
    m, k = g['body'] + g['to_q'], g['down'] + g['head']

    def axis(e0, e1, n):
        return max(-((k - e0) // 2) - m, 0), min((e1 - 1 + k) // 2 + m + 1, n)
    (y0, y1), (x0, x1) = axis(r[0], r[2], Ho), axis(r[1], r[3], Wo)
    return (y0, x0, y1, x1)


class UpdateScale(ScalePlan):
    """One scale of an update plan (plan_update), in that scale's coordinates.  rect / tiles: the tile-aligned
    rectangle R_s re-encoded and its tiles; window / out / fused: as in ScalePlan, the decoder window that codes rect
    (None at the uniform-prior scale); need: what the walk reads of this scale's encoder outputs (its symbols, values
    and F), at scale 0 the pixel window P_0; enc: the window of this scale's plane its encoder reads (None at the
    uniform-prior scale)."""
    __slots__ = ('need', 'enc')

    def __repr__(self):
        return 'UpdateScale(scale=%d, rect=%s, tiles=%d, window=%s, need=%s, enc=%s)' % (
            self.scale, self.rect, len(self.tiles), self.window, self.need, self.enc)


class UpdatePlan(object):
    """plan_update's result: scales coarse -> fine, the edit in padded image coordinates, the pixel window P_0 and the
    totals: streams re-encoded, streams in the container and the pixels of P_0."""

    def __init__(self, scales, edit, tile, total_streams):
        self.scales, self.edit, self.tile, self.total_streams = scales, edit, tile, total_streams

    @property
    def window(self):
        return self.scales[-1].need

    @property
    def streams(self):
        return sum(s.streams for s in self.scales)

    @property
    def window_pixels(self):
        return _area(self.window)

    def __repr__(self):
        return 'UpdatePlan(edit=%s, window=%s, streams=%d of %d)' % (self.edit, self.window, self.streams,
                                                                    self.total_streams)


def plan_update(shapes, pad_tuple, tile, config, rect):
    """Update of the region rect = (y, x, h, w) (unpadded image coordinates) of a tiled L3C container (DESIGN §4.12).
    shapes, pad_tuple, tile: as in plan_region; config: a MultiscaleNetwork (its DecoderGeometry and EncoderGeometry
    are read from it).  -> UpdatePlan.
    Forward pass, fine to coarse: the edited pixels E_0 change the scale-(s+1) symbols and F where the encoder of scale
    s reads E_s (_encoder_reach), and the scale-s CDFs where the decoder of scale s reads changed symbols of scale s+1
    (head, body and tail radii, x2, the classifier's radius) or, with dec.skip, adds changed coarser decoder features;
    R_s is the tile-aligned bounding rectangle of both (of the symbols alone at the uniform-prior scale).
    Backward pass: fine to coarse the decoder windows that code every R_s (_window; with dec.skip they also give the
    features the finer decoder adds), then coarse to fine the encoder windows that produce every symbol a window or R_s
    reads (encoder_rect), down to the pixel window P_0.
    ValueError for an untiled container, the RGB baselines, a container of the wrong scale count, and an empty
    region or one outside the image."""
    if tile is None:
        raise ValueError('region update needs a tiled container (written with Bitcoding(..., tile=(th, tw))): '
                         'the streams of the reference layout are serial')
    geo = geometry_of(config)
    egeo = config if isinstance(config, EncoderGeometry) else EncoderGeometry(config)
    if geo.rgb:
        raise ValueError('region update is not supported by the RGB baselines: their bicubic encoder has no planned '
                         'windows')
    tile = (int(tile[0]), int(tile[1]))
    n = len(shapes)
    S = geo.num_scales
    if n != S + 1:
        raise ValueError('container has %d scales, model expects %d' % (n, S + 1))
    if len(rect) != 4:
        raise ValueError('region must be (y, x, h, w), got %r' % (rect,))
    y, x, h, w = (int(v) for v in rect)
    left, right, top, bottom = (int(v) for v in pad_tuple)
    _, Hf, Wf = shapes[-1]
    Hu, Wu = Hf - top - bottom, Wf - left - right
    if h < 1 or w < 1:
        raise ValueError('empty region %r' % (tuple(rect),))
    if y < 0 or x < 0 or y + h > Hu or x + w > Wu:
        raise ValueError('region %r lies outside the %dx%d image' % (tuple(rect), Hu, Wu))
    dims = [shapes[n - 1 - s][1:] for s in range(n)]                     # (H, W) by scale, fine -> coarse
    # forward pass: changed symbols E_s, fine -> coarse
    E = [(y + top, x + left, y + top + h, x + left + w)]
    for s in range(S):
        E.append(_encoder_reach(egeo, s, E[s], *dims[s + 1]))
    # changed decoder features G_s (scale-s grid) and CDFs, coarse -> fine
    R, G = [None] * n, [None] * n
    R[S] = _align(E[S], dims[S][0], dims[S][1], tile)
    for s in range(S - 1, -1, -1):
        r = geo.radii_of(s)
        Hc, Wc = dims[s + 1]
        q = _clip(_expand(E[s + 1], r.head + r.body + r.tail), Hc, Wc)
        if geo.fuses(s):
            q = _union(q, _clip(_expand(G[s + 1], r.body + r.tail), Hc, Wc))
        G[s] = (2 * q[0], 2 * q[1], 2 * q[2], 2 * q[3])                 # Upsampler x2
        cdf = _clip(_expand(G[s], r.clf), *dims[s])
        R[s] = _align(_union(E[s], cdf), dims[s][0], dims[s][1], tile)
    # decoder windows, fine -> coarse: R_s and, with dec.skip, the features the finer decoder adds
    win, out, fused, need = [None] * n, [None] * n, [False] * n, [None] * n
    want = None
    for s in range(S):
        win[s], out[s], fused[s], want = _window(geo, s, R[s], dims[s][0], dims[s][1], *dims[s + 1], features=want)
        if not fused[s]:
            want = None
    # encoder windows, coarse -> fine: scale s's encoder produces what scale s + 1 needs
    enc = [None] * n
    need[S] = _union(R[S], win[S - 1])
    for s in range(S - 1, -1, -1):
        enc[s] = encoder_rect(egeo, s, need[s + 1], *dims[s])
        need[s] = _union(enc[s], R[s] if s == 0 else _union(R[s], win[s - 1]))
    scales = []
    for s in range(S, -1, -1):
        H, W = dims[s]
        th, tw = tile
        ntx = -(-W // tw)
        rr = R[s]
        tiles = [ty * ntx + tx for ty in range(rr[0] // th, -(-rr[2] // th)) for tx in range(rr[1] // tw, -(-rr[3] // tw))]
        scales.append(UpdateScale(idx=n - 1 - s, scale=s, C=shapes[n - 1 - s][0], H=H, W=W, rect=rr, tiles=tiles,
                                  window=win[s], out=out[s], fused=fused[s], need=need[s], enc=enc[s]))
    total = sum(C * len(tile_grid(H, W, tile)) for (C, H, W) in shapes)
    return UpdatePlan(scales, E[0], tile, total)


def _meets(a, b):
    return a[0] < b[2] and b[0] < a[2] and a[1] < b[3] and b[1] < a[3]


def plans_conflict(a, b):
    """Whether two update plans of one container must be merged (DESIGN §4.12, "Batches of updates"): the edit E_0 of
    one meets the pixel window P_0 of the other, so the pixels one plan encodes are not the old ones."""
    return _meets(a.edit, b.window) or _meets(b.edit, a.window)


def merge_update_plans(shapes, pad_tuple, tile, config, rects):
    """The update plans of several edits rects = [(y, x, h, w)] of one container (plan_update's arguments otherwise):
    one plan per edit, then any two conflicting plans (plans_conflict) replaced by the plan of the bounding rectangle of
    their edits, until no two conflict.  -> [(UpdatePlan, [indices into rects, ascending])], ordered by their first
    edit.  Plans that stay separate are exact on their own: a plan's streams depend only on the pixels of its P_0, which
    no other plan's edit touches."""
    left, _, top, _ = (int(v) for v in pad_tuple)
    plans = [(plan_update(shapes, pad_tuple, tile, config, r), [i]) for i, r in enumerate(rects)]
    merged = True
    while merged:
        merged = False
        for a in range(len(plans)):
            for b in range(a + 1, len(plans)):
                if plans_conflict(plans[a][0], plans[b][0]):
                    e = _union(plans[a][0].edit, plans[b][0].edit)
                    plan = plan_update(shapes, pad_tuple, tile, config,
                                       (e[0] - top, e[1] - left, e[2] - e[0], e[3] - e[1]))
                    plans[a] = (plan, sorted(plans[a][1] + plans[b][1]))
                    del plans[b]
                    merged = True
                    break
            if merged:
                break
    return plans


def plan_update_passes(plans, budget):
    """How BatchCodec.update_regions groups update plans (of any containers) into passes: -> [[indices into plans]],
    plans of one tile size per pass, grouped by bitcoding.plan_passes over their P_0 shapes so that a pass's padded
    windows hold at most `budget` pixels (a window larger than that is a pass of its own)."""
    from .bitcoding import plan_passes
    by_tile = {}
    for i, p in enumerate(plans):
        by_tile.setdefault(p.tile, []).append(i)
    passes = []
    for idxs in by_tile.values():
        shapes = [(plans[i].window[2] - plans[i].window[0], plans[i].window[3] - plans[i].window[1]) for i in idxs]
        passes += [[idxs[j] for j in grp] for grp in plan_passes(shapes, budget)]
    return passes
