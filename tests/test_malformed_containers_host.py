"""CPU: containers whose headers come from outside -- truncated, extended or crafted -- against every host-side check
that runs before a decode, region decode or region update uploads anything (DESIGN §5, "Malformed containers").

Containers of every layout are built with ContainerLayout.header_and_offsets from the shape lists the models write,
with random stream bytes: compat `cr` at 32 x 32 and 40 x 28 (padded), compat `cr_rgb_shared` at 64 x 64, a recursive
`cr_rgb_shared` container (R = 2), tiled `cr` with tiles 16 x 16 and 16 x 24 on a padded 37 x 53 image, and a whole
tiled container (Bitcoding(crop=False)) of a padded 197 x 130 image in 32 x 32 tiles; and, for the GPU suite, tiled
`cr_rgb_shared` containers at 64 x 64, one of them recursive.  Each is mutated: cut after every
prefix length, extended, its scale headers, tiled tag, length fields, separators and padding tuple rewritten.
* Every malformed mutation is refused with ValueError by each entry point that takes the unmutated container: the
  decode's checks (parse_container, then BatchCodec._check_shapes, as decode_batch runs them before its upload), and
  for tiled containers codec.plan_regions and codec.plan_updates.  Each refusal takes under 50 ms and 1 MB of traced
  Python allocation, whatever the header declares (a 29-byte file declaring 4096^2 tiles of 1 x 1 once took seconds).
* Mutations that are valid by construction -- a boundary moved between two adjacent streams, streams of length 0, a
  padding tuple that leaves pixels on both axes, the prefix of a recursive container that ends at a scale -- are
  accepted by every entry point and parse to exactly what was built.  tests/test_gpu_junk_containers.py decodes them.
"""
import signal
import struct
import time
import tracemalloc

import numpy as np
import pytest
import torch

from tests import util

MAGIC = b'\x46\xE2\x84\x92'
BUDGET_S = 0.05                 # per refusal
BUDGET_BYTES = 1 << 20          # peak traced Python allocation per refusal
HARD_STOP_S = 2.0               # a parse still running then has failed its budget; stop it rather than wait

# kind: (model, padded height, padded width, padding tuple (left, right, top, bottom), tile, recursive scales)
KINDS = {
    'cr_32': ('cr', 32, 32, (0, 0, 0, 0), None, 0),
    'cr_40x28': ('cr', 40, 32, (2, 2, 0, 0), None, 0),
    'rgbs_64': ('cr_rgb_shared', 64, 64, (0, 0, 0, 0), None, 0),
    'rgbs_r2': ('cr_rgb_shared', 64, 64, (0, 0, 0, 0), None, 2),
    'cr_t16': ('cr', 40, 56, (1, 2, 1, 2), (16, 16), 0),
    'cr_t16x24': ('cr', 40, 56, (1, 2, 1, 2), (16, 24), 0),
    'cr_whole': ('cr', 200, 136, (3, 3, 1, 2), (32, 32), 0),
    'rgbs_t16': ('cr_rgb_shared', 64, 64, (0, 0, 0, 0), (16, 16), 0),
    'rgbs_r2_t16': ('cr_rgb_shared', 64, 64, (0, 0, 0, 0), (16, 16), 2),
}


def shapes_of(kind):
    """[(C, H, W)] coarse -> fine, as the kind's model writes them."""
    cfg, H, W, _, _, R = KINDS[kind]
    net = util.blueprint(cfg, device='cpu').net
    return [(3 if (s == 0 or net._rgb) else net.config_ms.q.C, H >> s, W >> s)
            for s in reversed(range(net.scales + R + 1))]


def streams_per_scale(kind):
    from l3c_pytorch_b200.codec import tile_grid
    return [C * len(tile_grid(H, W, KINDS[kind][4])) for (C, H, W) in shapes_of(kind)]


def build(kind, payloads, pad=None):
    """The container of `kind` whose streams hold `payloads` (bytes per stream, container order) -> (data, expected
    parse_container result)."""
    from l3c_pytorch_b200.codec import ContainerLayout
    _, _, _, pad0, tile, _ = KINDS[kind]
    pad = pad0 if pad is None else pad
    shapes = shapes_of(kind)
    lens = [len(p) for p in payloads]
    assert len(lens) == sum(streams_per_scale(kind))
    total, pieces, offs = ContainerLayout([(i,) + s for i, s in enumerate(shapes)], tile).header_and_offsets(lens, pad)
    buf = bytearray(total)
    for o, b in pieces:
        buf[o:o + len(b)] = b
    for o, p in zip(offs, payloads):
        buf[o:o + len(p)] = p
    scales, i = [], 0
    for (C, H, W), n in zip(shapes, streams_per_scale(kind)):
        scales.append((C, H, W, list(zip(offs[i:i + n], lens[i:i + n]))))
        i += n
    return bytes(buf), (tuple(pad), scales)


def random_payloads(kind, seed, max_len=16):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, int(rng.integers(0, max_len + 1)), dtype=np.uint8).tobytes()
            for _ in range(sum(streams_per_scale(kind)))]


_CODECS = {}


def codec(cfg):
    from l3c_pytorch_b200.codec import BatchCodec
    if cfg not in _CODECS:
        _CODECS[cfg] = BatchCodec(util.blueprint(cfg, device='cpu'))
    return _CODECS[cfg]


def entry_points(kind):
    """{name: check(data)} of every host-side entry that takes the unmutated container of `kind`: the checks of a
    decode (parse_container, then _check_shapes), and for tiled containers the planners of decode_regions and (L3C
    only: the RGB baselines refuse updates) update_regions, with one edit and with none."""
    from l3c_pytorch_b200.codec import parse_container
    cfg, _, _, _, tile, _ = KINDS[kind]
    c = codec(cfg)
    eps = {'decode': lambda d: c._check_shapes([s[:3] for s in parse_container(d)[1]])}
    if tile is not None:
        eps['plan_regions'] = lambda d: c.plan_regions([d], [(0, 0, 1, 1)])
        if cfg == 'cr':
            patch = torch.zeros(3, 1, 1, dtype=torch.uint8)
            eps['plan_updates'] = lambda d: c.plan_updates([d], [[((0, 0), patch)]])
            eps['plan_updates_none'] = lambda d: c.plan_updates([d], [[]])
    return eps


class _Overrun(Exception):
    pass


def bounded(fn, data):
    """fn(data) under tracemalloc, stopped after HARD_STOP_S -> (ValueError or _Overrun or None, seconds, peak bytes)."""
    def stop(*_):
        raise _Overrun('still running after %.1f s' % HARD_STOP_S)
    old = signal.signal(signal.SIGALRM, stop)
    tracemalloc.start()
    err = None
    t0 = time.perf_counter()
    try:
        signal.setitimer(signal.ITIMER_REAL, HARD_STOP_S)
        try:
            fn(data)
        finally:
            signal.setitimer(signal.ITIMER_REAL, 0)
    except (ValueError, _Overrun) as e:
        err = e
    finally:
        dt = time.perf_counter() - t0
        peak = tracemalloc.get_traced_memory()[1]
        tracemalloc.stop()
        signal.signal(signal.SIGALRM, old)
    return err, dt, peak


def _layout(kind, data, expect):
    """Byte positions in `data` (expect: its parse): every scale's header, every length field, every separator."""
    heads, fields, seps = [], [], []
    for (_, _, _, st) in expect[1]:
        heads.append(st[0][0] - 9)
        fields += [o - 4 for (o, _) in st]
        seps.append(st[-1][0] + st[-1][1])
    return heads, fields, seps


def tiled_tag_files(kind, data):
    """Files of at most 64 bytes whose tag declares a degenerate or extreme tile over a 65535^2 (and a 4096^2) plane."""
    th, tw = KINDS[kind][4]
    C = data[16]
    out = []
    for tile, (H, W) in [((0, tw), (65535, 65535)), ((th, 0), (65535, 65535)), ((1, 1), (65535, 65535)),
                         ((1, 65535), (65535, 65535)), ((65535, 1), (65535, 65535)), ((1, 1), (4096, 4096))]:
        head = data[:8] + b'L3CT' + struct.pack('<HH', *tile) + struct.pack('<BHH', C, H, W)
        out.append(('tile %s %dx%d' % (tile, H, W), (head + data[21:64])[:64]))
        out.append(('tile %s %dx%d, 29 B' % (tile, H, W), head + data[21:29]))
    return out


def malformed(kind, data, expect):
    """[(class, description, bytes)]: every mutation of `data` that no entry point may accept."""
    _, _, _, pad, tile, R = KINDS[kind]
    heads, fields, seps = _layout(kind, data, expect)
    ends = {s + 4 for s in seps}
    n_model = len(expect[1]) - R                         # the scales of a non-recursive container of this model
    out = []
    for p in range(len(data)):
        # a recursive container cut at a scale boundary is a recursive container of fewer levels (valid_mutations)
        if not (R and p in ends and sum(e <= p for e in ends) >= n_model):
            out.append(('truncation', 'first %d bytes' % p, data[:p]))
    last = data[heads[-1]:]
    for name, tail in [('1 byte', b'\0'), ('4 bytes', b'\xff' * 4), ('5 bytes', struct.pack('<BHH', 3, 8, 8)),
                       ('empty scale', struct.pack('<BHH', 0, 0, 0) + MAGIC), ('copy of the last scale', last)]:
        out.append(('extension', name, data + tail))
    for k, (C, H, W, _) in enumerate(expect[1]):
        for field, vals, at, fmt in [('C', {0, 1, C - 1, C + 1, 255}, 0, '<B'),
                                     ('H', {0, 1, H // 2, 2 * H, H + 1, 65535}, 1, '<H'),
                                     ('W', {0, 1, W // 2, 2 * W, W + 1, 65535}, 3, '<H')]:
            for v in sorted(vals - {(C, H, W)[(0, 1, 3).index(at)]}):
                buf = bytearray(data)
                struct.pack_into(fmt, buf, heads[k] + at, v)
                out.append(('scale header', 'scale %d %s=%d' % (k, field, v), bytes(buf)))
    if tile is not None:
        out += [('tiled tag', name, f) for name, f in tiled_tag_files(kind, data)]
        for i in range(8, 12):
            buf = bytearray(data)
            buf[i] ^= 0xFF
            out.append(('tiled tag', 'tag byte %d flipped' % i, bytes(buf)))
    for i, f in enumerate(fields):
        n, = struct.unpack_from('<I', data, f)
        for v in sorted({n + 1, n - 1, 0, 2 ** 32 - 1, len(data) - f - 4} - {n, -1}):
            buf = bytearray(data)
            struct.pack_into('<I', buf, f, v)
            out.append(('length field', 'stream %d: %d -> %d' % (i, n, v), bytes(buf)))
    for k, s in enumerate(seps):
        buf = bytearray(data)
        buf[s] ^= 0xFF
        out.append(('separator', 'scale %d' % k, bytes(buf)))
    for p in empty_axis_pads(expect):
        out.append(('padding', 'empties an axis: %s' % (p,), struct.pack('<4H', *p) + data[8:]))
    return out


def empty_axis_pads(expect):
    _, H, W, _ = expect[1][-1]
    return [(W, 0, 0, 0), (0, W, 0, 0), (0, 0, H, 0), (0, 0, 0, H), (W // 2, W - W // 2, 0, 0),
            (0, 0, H // 2, H - H // 2), (0, 0, H + 1, 0), (65535,) * 4, (1, 1, 65535, 0)]


def cropping_pads(expect):
    """Padding tuples that leave at least one pixel on both axes, most of them not what the encoder writes."""
    _, H, W, _ = expect[1][-1]
    return [(W - 1, 0, 0, 0), (0, 0, 0, H - 1), (1, 1, 1, 1), (0, W - 1, H - 1, 0), (3, 0, 5, 2)]


def moved_boundaries(kind, payloads):
    """[(description, payloads)]: the bytes of two adjacent streams of one scale re-split at another point (their
    length fields changed by +k and -k)."""
    out, i = [], 0
    for n in streams_per_scale(kind):
        for a in range(i, i + n - 1, max(1, (n - 1) // 3)):
            both = payloads[a] + payloads[a + 1]
            for cut in sorted({0, len(both), len(payloads[a]) + 1, len(payloads[a]) - 1} & set(range(len(both) + 1))):
                if cut != len(payloads[a]):
                    p = list(payloads)
                    p[a], p[a + 1] = both[:cut], both[cut:]
                    out.append(('streams %d|%d split at %d of %d' % (a, a + 1, cut, len(both)), p))
        i += n
    return out


def empty_streams(kind, payloads):
    """[(description, payloads)]: some streams set to length 0."""
    per = streams_per_scale(kind)
    first = np.cumsum([0] + per)
    out = [('every stream', [b''] * len(payloads)),
           ('every other stream', [b'' if i % 2 else p for i, p in enumerate(payloads)])]
    for k in range(len(per)):
        out.append(('scale %d' % k, [b'' if first[k] <= i < first[k + 1] else p for i, p in enumerate(payloads)]))
    return out


def valid_mutations(kind, seed=0):
    """[(class, description, data, expected parse)] of the mutations that are valid by construction."""
    payloads = random_payloads(kind, seed)
    data, expect = build(kind, payloads)
    R = KINDS[kind][5]
    out = []
    for name, p in moved_boundaries(kind, payloads):
        out.append(('moved boundary', name) + build(kind, p))
    for name, p in empty_streams(kind, payloads):
        out.append(('empty streams', name) + build(kind, p))
    for pad in cropping_pads(expect):
        out.append(('padding', 'crops %s' % (pad,)) + build(kind, payloads, pad))
    if R:
        _, _, seps = _layout(kind, data, expect)
        for k in range(len(expect[1]) - R - 1, len(expect[1]) - 1):
            out.append(('recursive prefix', '%d scales' % (k + 1), data[:seps[k] + 4], (expect[0], expect[1][:k + 1])))
    return out


# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', list(KINDS))
def test_malformed_containers_are_refused_everywhere_within_bounds(kind):
    from l3c_pytorch_b200.codec import parse_container
    payloads = random_payloads(kind, 0)
    data, expect = build(kind, payloads)
    assert parse_container(data) == expect
    eps = entry_points(kind)
    for name, check in eps.items():
        err, _, _ = bounded(check, data)
        assert err is None, (name, err)
    bad, per_class, worst = [], {}, (0.0, 0)
    for cls, what, d in malformed(kind, data, expect):
        per_class[cls] = per_class.get(cls, 0) + 1
        for name, check in eps.items():
            err, dt, peak = bounded(check, d)
            worst = (max(worst[0], dt), max(worst[1], peak))
            if not isinstance(err, ValueError) or dt >= BUDGET_S or peak >= BUDGET_BYTES:
                bad.append((cls, what, name, len(d), repr(err), '%.1f ms' % (dt * 1e3), '%d B' % peak))
    print('%s: %d bytes, %s, entry points %s; slowest refusal %.2f ms, largest peak %d B'
          % (kind, len(data), per_class, sorted(eps), worst[0] * 1e3, worst[1]))
    assert not bad, bad[:20]


@pytest.mark.parametrize('kind', list(KINDS))
def test_valid_mutations_parse_to_what_was_built(kind):
    from l3c_pytorch_b200.codec import parse_container
    eps = entry_points(kind)
    muts = valid_mutations(kind)
    assert {m[0] for m in muts} >= {'moved boundary', 'empty streams', 'padding'}
    for cls, what, d, expect in muts:
        assert parse_container(d) == expect, (cls, what)
        for name, check in eps.items():
            check(d)


def test_a_tiny_file_declaring_millions_of_tiles_is_refused_at_once():
    """29 bytes: the padding, a tag of 1 x 1 tiles and a 4096 x 4096 scale header, then 8 bytes; the header declares
    3 * 4096^2 streams whose length fields alone would take 201 MB."""
    from l3c_pytorch_b200.codec import parse_container
    data = struct.pack('<4H', 0, 0, 0, 0) + b'L3CT' + struct.pack('<HH', 1, 1) + struct.pack('<BHH', 3, 4096, 4096) \
        + bytes(8)
    assert len(data) == 29
    err, dt, peak = bounded(parse_container, data)
    print('29-byte 4096^2 file of 1 x 1 tiles: %r after %.3f ms, peak %d B' % (err, dt * 1e3, peak))
    assert isinstance(err, ValueError) and dt < BUDGET_S and peak < BUDGET_BYTES, (err, dt, peak)


def test_padding_that_empties_an_axis_is_refused_by_the_parser():
    from l3c_pytorch_b200.codec import parse_container
    for kind in ('cr_40x28', 'cr_t16'):
        data, expect = build(kind, random_payloads(kind, 1))
        for p in empty_axis_pads(expect):
            with pytest.raises(ValueError, match='padding tuple'):
                parse_container(struct.pack('<4H', *p) + data[8:])
