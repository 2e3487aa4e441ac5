"""GPU: malformed containers and containers whose headers are valid but whose streams are junk, on every decode path.

The containers come from tests/test_malformed_containers_host.py, which shows on the host which mutations are refused
and which are valid by construction.  Only those two kinds are submitted here.
* A. Refusal before any work: one mutation of each refused class, for every container kind, through Bitcoding.decode
  (from a file), decode_batch with and without a decode lane, decode_regions, the banded decode, update_region,
  update_regions and update_regions_begin(...).finish(): each raises ValueError with no launch between a reset of the
  launch log and the raise, and a valid container decodes exactly afterwards.
* B. The oracle on junk: under the sharpened model of test_gpu_peaked_coding every coded CDF row is saturated, so the
  rows do not depend on the implementation.  Compat containers with random, all-0x00, all-0xFF and empty streams,
  moved stream boundaries and streams of another channel swapped in decode to oracle.model.decode_image's image in
  all four precision modes.  Tiled junk containers: every tile's symbols, at every scale, are oracle.ac.decode of that
  tile's bytes on the rows the oracle builds for it (fixed rows for R and the bottlenecks, G's and B's from the R and G
  the oracle decoded at the same pixel).
* C. Paths agree on junk (default-init model; `cr` in all four modes, `cr_rgb_shared` in f16 and f16x2, one container
  recursive): the whole decode of a tiled junk container equals the same call repeated, the call on a lane, the banded
  decode, decode_regions crops (interior, edge, corner, 1 x 1) and the decode beside a valid container of another
  size and of the same size, where the valid container still decodes to its image.  In f16 a compat junk container
  in a ragged batch equals its decode alone.
"""
import struct

import numpy as np
import pytest
import torch

from tests import util
from tests.test_gpu_peaked_coding import family, precision, tile_rects
from tests.test_malformed_containers_host import (KINDS, build, cropping_pads, malformed, moved_boundaries,
                                                  random_payloads, shapes_of, streams_per_scale)

MODES = ['f16', 'f16x2', 'tf32', 'fp32']
V_LEVEL = 12


def _bitcoding(bp, kind):
    from l3c_pytorch_b200 import Bitcoding
    tile = KINDS[kind][4]
    return Bitcoding(bp, tile=tile, crop=not (tile is not None and kind == 'cr_whole'))


def _payloads(data):
    from l3c_pytorch_b200.codec import parse_container
    return [data[o:o + n] for (_, _, _, st) in parse_container(data)[1] for (o, n) in st]


def _swapped(kind, payloads):
    """The streams of channels 0 and 1 of every scale exchanged: valid streams, each on another channel's rows."""
    p, i = list(payloads), 0
    for (C, _, _), n in zip(shapes_of(kind), streams_per_scale(kind)):
        T = n // C
        p[i:i + T], p[i + T:i + 2 * T] = p[i + T:i + 2 * T], p[i:i + T]
        i += n
    return p


def junk_sets(kind, valid_payloads=None):
    """{name: payloads} of junk streams under a valid header of `kind`."""
    rnd = random_payloads(kind, 7, max_len=24)
    lens = [len(p) for p in rnd]
    out = {'random': rnd, 'zeros': [bytes(n) for n in lens], 'ones': [b'\xff' * n for n in lens],
           'empty': [b''] * len(rnd), 'moved': moved_boundaries(kind, rnd)[1][1]}
    if valid_payloads is not None:
        out['swapped'] = _swapped(kind, valid_payloads)
    return out


def _unpadded(kind):
    _, H, W, (left, right, top, bottom), _, _ = KINDS[kind]
    return H - top - bottom, W - left - right


def _valid_image(kind, seed=3):
    return util.make_image(seed, *_unpadded(kind))


# ----------------------------------------------------------------------------------------------
# A. refusal before any work
# ----------------------------------------------------------------------------------------------
def _one_per_class(kind):
    """One mutation of each refused class, and the file cut after its padding (and tag): a container of no scales."""
    data, expect = build(kind, random_payloads(kind, 0))
    picked = {}
    for cls, what, d in malformed(kind, data, expect):
        picked.setdefault(cls, []).append((what, d))
    head = 8 if KINDS[kind][4] is None else 16
    return [(cls, ) + ms[len(ms) // 2] for cls, ms in picked.items()] + [('truncation', 'no scale', data[:head])]


@pytest.mark.gpu
@pytest.mark.parametrize('kind', list(KINDS))
def test_refused_before_any_launch(kind, tmp_path, monkeypatch):
    from l3c_pytorch_b200 import codec, engine as E
    cfg, _, _, _, tile, R = KINDS[kind]
    bc = _bitcoding(util.blueprint(cfg), kind)
    lane = bc.decode_lanes(1, n_lanes=1)[0]
    patch = torch.zeros(3, 1, 1, dtype=torch.uint8)

    def on_lane(fn):
        with torch.cuda.stream(lane.main):
            return fn()

    def banded(d):
        monkeypatch.setattr(codec, 'TILED_BAND_PIXELS', tile[0] * KINDS[kind][2])
        try:
            return bc.decode_batch([d])
        finally:
            monkeypatch.undo()

    calls = {'decode': lambda d: bc.decode(str(tmp_path / 'c.l3c')),
             'decode_batch': lambda d: bc.decode_batch([d]),
             'decode_batch lane': lambda d: on_lane(lambda: bc.decode_batch([d], lane=lane))}
    if tile is not None:
        calls['decode_regions'] = lambda d: bc.decode_regions([d], [(0, 0, 1, 1)])
        calls['banded'] = banded
        if cfg == 'cr':
            calls['update_region'] = lambda d: bc.update_region(d, (0, 0), patch)
            calls['update_regions'] = lambda d: bc.update_regions([d], [[((0, 0), patch)]])
            calls['update_regions_begin'] = lambda d: bc.update_regions_begin([d], [[((0, 0), patch)]]).finish()
    n = 0
    for cls, what, d in _one_per_class(kind):
        with open(str(tmp_path / 'c.l3c'), 'wb') as f:
            f.write(d)
        for name, call in calls.items():
            torch.cuda.synchronize()
            E.launch_log(reset=True)
            with pytest.raises(ValueError):
                call(d)
            assert E.launch_log()[1] == 0, (cls, what, name, E.launch_log()[0])
            n += 1
    torch.cuda.synchronize()
    print('%s: %d refusals, none launched anything' % (kind, n))
    img = _valid_image(kind)
    if R:
        from l3c_pytorch_b200 import Bitcoding
        bc = Bitcoding(util.blueprint(cfg), tile=tile, recursive=R)
    datas, _ = bc.encode_batch(img.unsqueeze(0))
    assert torch.equal(bc.decode_batch(datas)[0][0].cpu(), img.long())


# ----------------------------------------------------------------------------------------------
# B. the oracle on junk, under saturated rows
# ----------------------------------------------------------------------------------------------
_ORACLE = {}


def _oracle_decode(cfg, data):
    from oracle import model as om
    if (cfg, data) not in _ORACLE:
        _, sd = family(cfg, V_LEVEL if cfg == 'cr' else 0)
        _ORACLE[(cfg, data)] = om.decode_image(sd, util.oracle_cfg(cfg), data, 'torch')
    return _ORACLE[(cfg, data)]


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['cr_32', 'cr_40x28', 'rgbs_64'])
@pytest.mark.parametrize('mode', MODES)
def test_compat_junk_decodes_to_the_oracle(mode, kind):
    from l3c_pytorch_b200 import Bitcoding
    from oracle import model as om
    cfg = KINDS[kind][0]
    bp, sd = family(cfg, V_LEVEL if cfg == 'cr' else 0)
    valid = om.encode_image(sd, util.oracle_cfg(cfg), _valid_image(kind), 'torch')
    bc = Bitcoding(bp)
    with precision(mode):
        for name, payloads in junk_sets(kind, _payloads(valid)).items():
            data, _ = build(kind, payloads)
            want = _oracle_decode(cfg, data)
            got = bc.decode_batch([data])[0].cpu()
            assert got.shape == want.shape and torch.equal(got, want), (name, int((got != want).sum()))


def _oracle_tile_symbols(cfg, kind, data):
    """Per scale, coarse -> fine: int64 [C, H, W], every tile oracle.ac.decode of its bytes on the oracle's rows."""
    from l3c_pytorch_b200.codec import parse_container
    from oracle import ac, model as om
    _, sd = family(cfg, V_LEVEL if cfg == 'cr' else 0)
    ocfg = util.oracle_cfg(cfg)
    rgb, other = om.dmlls(ocfg)
    tile = KINDS[kind][4]
    _, scales = parse_container(data)
    n = len(scales)
    _, Hf, Wf, _ = scales[-1]
    with torch.no_grad():
        P = om.forward(sd, ocfg, torch.zeros(1, 3, Hf, Wf)).P          # bias only: the same for every input
    out = []
    for idx, (C, H, W, st) in enumerate(scales):
        scale = n - 1 - idx
        dm = rgb if scale == 0 else other
        rects = tile_rects(H, W, tile)
        S = np.zeros((C, H, W), np.int64)
        dec = torch.zeros(1, C, H, W)
        for c in range(C):
            table = None if idx == 0 else om.cdf_table_torch_formula(dm, P[scale], c, C, dec).reshape(H, W, -1)
            for t, (y0, x0, y1, x1) in enumerate(rects):
                o, ln = st[c * len(rects) + t]
                if table is None:
                    sym = ac.decode(ac.uniform_cdf_row(dm.L), data[o:o + ln], (y1 - y0) * (x1 - x0))
                else:
                    sym = ac.decode(np.ascontiguousarray(table[y0:y1, x0:x1]).reshape(-1, table.shape[-1]),
                                    data[o:o + ln])
                S[c, y0:y1, x0:x1] = sym.reshape(y1 - y0, x1 - x0)
            dec[0, c] = torch.from_numpy(S[c]).float()
        out.append(S)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['cr_t16', 'cr_t16x24'])
@pytest.mark.parametrize('mode', MODES)
def test_tiled_junk_symbols_are_the_oracles(mode, kind, monkeypatch):
    from l3c_pytorch_b200 import Bitcoding, engine as E
    cfg = KINDS[kind][0]
    bp, _ = family(cfg, V_LEVEL)
    bc = Bitcoding(bp, tile=KINDS[kind][4])
    seen, orig = [], E.symbols_to_values

    def record(sym, *a, **kw):
        seen.append(sym.clone())
        return orig(sym, *a, **kw)
    monkeypatch.setattr(E, 'symbols_to_values', record)
    with precision(mode):
        for name in ('random', 'zeros', 'ones'):
            data, _ = build(kind, junk_sets(kind)[name])
            seen.clear()
            S, _ = bc.codec.decode_batch([data])
            got = [s[0].long().cpu().numpy() for s in seen] + [S[0].long().numpy()]
            want = _oracle_tile_symbols(cfg, kind, data)
            assert len(got) == len(want), name
            for idx, (g, w) in enumerate(zip(got, want)):
                assert g.shape == w.shape and np.array_equal(g, w), (name, idx, int((g != w).sum()))


# ----------------------------------------------------------------------------------------------
# C. every path agrees on junk (default-init model)
# ----------------------------------------------------------------------------------------------
def _regions(Hu, Wu):
    return [(Hu // 4, Wu // 5, Hu // 2, Wu // 3), (0, Wu // 3, 5, Wu - Wu // 3), (Hu - 7, 0, 7, 9),
            (Hu - 1, Wu - 1, 1, 1), (0, 0, 1, 1), (Hu // 2, Wu // 2, 1, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize('cfg,mode', [('cr', m) for m in MODES] + [('cr_rgb_shared', 'f16'),
                                                                   ('cr_rgb_shared', 'f16x2')])
def test_paths_agree_on_junk(cfg, mode, monkeypatch):
    from l3c_pytorch_b200 import Bitcoding, codec
    kinds = ['cr_t16', 'cr_t16x24', 'cr_whole'] if cfg == 'cr' else ['rgbs_t16', 'rgbs_r2_t16']
    bp = util.blueprint(cfg)
    with precision(mode):
        for kind in kinds:
            tile, Hu, Wu = KINDS[kind][4], *_unpadded(kind)
            bc = _bitcoding(bp, kind)
            lane = bc.decode_lanes(2, n_lanes=1)[0]
            img = _valid_image(kind)
            other = util.make_image(4, Hu - 8, Wu + 8)
            enc = Bitcoding(bp, tile=tile, crop=kind != 'cr_whole', recursive=KINDS[kind][5])
            valid, _ = enc.encode_batch(img.unsqueeze(0))
            valid_other, _ = enc.encode_batch(other.unsqueeze(0))
            for name, payloads in junk_sets(kind).items():
                data, _ = build(kind, payloads)
                whole = bc.decode_batch([data])[0].cpu()
                assert whole.shape == (1, 3, Hu, Wu), (kind, name)
                assert torch.equal(bc.decode_batch([data])[0].cpu(), whole), (kind, name, 'repeated')
                with torch.cuda.stream(lane.main):
                    got = bc.decode_batch([data], lane=lane)[0]
                torch.cuda.synchronize()
                assert torch.equal(got.cpu(), whole), (kind, name, 'lane')
                monkeypatch.setattr(codec, 'TILED_BAND_PIXELS', tile[0] * KINDS[kind][2])
                assert torch.equal(bc.decode_batch([data])[0].cpu(), whole), (kind, name, 'banded')
                monkeypatch.undo()
                regs = _regions(Hu, Wu)
                for r, (y, x, h, w) in zip(bc.decode_regions([data] * len(regs), regs), regs):
                    assert torch.equal(r.cpu(), whole[:, :, y:y + h, x:x + w]), (kind, name, (y, x, h, w))
                mixed = bc.decode_batch([data, valid_other[0]])
                assert torch.equal(mixed[0].cpu(), whole), (kind, name, 'beside another size')
                assert torch.equal(mixed[1][0].cpu(), other.long()), (kind, name, 'valid beside junk')
                same = bc.decode_batch([valid[0], data])
                assert torch.equal(same[1].cpu(), whole), (kind, name, 'same-shape batch')
                assert torch.equal(same[0][0].cpu(), img.long()), (kind, name, 'valid in a same-shape batch')
        if cfg == 'cr':
            bc = Bitcoding(bp)
            valid, _ = bc.encode_batch(util.make_image(5, 32, 32).unsqueeze(0))
            for name, payloads in junk_sets('cr_40x28').items():
                data, _ = build('cr_40x28', payloads)
                alone = bc.decode_batch([data])[0].cpu()
                both = bc.decode_batch([valid[0], data])                  # ragged in f16, one pass per shape else
                assert torch.equal(both[1].cpu(), alone), name
                assert torch.equal(both[0][0].cpu(), util.make_image(5, 32, 32).long()), name


@pytest.mark.gpu
def test_cropping_pads_are_cropped_as_written():
    """A padding tuple the encoder would not write, but that leaves pixels, crops the decode exactly as written."""
    from l3c_pytorch_b200 import pad as P
    bp = util.blueprint('cr')
    for kind in ('cr_40x28', 'cr_t16'):
        bc = _bitcoding(bp, kind)
        payloads = random_payloads(kind, 11)
        base, expect = build(kind, payloads, (0, 0, 0, 0))
        full = bc.decode_batch([base])[0].cpu()
        for pad in cropping_pads(expect):
            data, _ = build(kind, payloads, pad)
            assert struct.unpack_from('<4H', data) == pad
            assert torch.equal(bc.decode_batch([data])[0].cpu(), P.undo_pad(full, *pad)), (kind, pad)
