"""The codec end to end on sharply peaked mixtures, the regime of a trained model coding a photograph.

`sharpen` turns the seed-0 default-init blueprint into one whose every coded CDF row is saturated: the probability
heads' 1x1 `lin` convs and the `to_q` convs get zero weights and biases that put one component (logit +20) of log-scale
-9 (below the -7 clamp) on a fixed mean -- m_R on R, the coded R on G and the coded G on B (coupling logits +30, -30,
+30), the level v on every bottleneck symbol.  With zero weights a conv returns its bias exactly in every precision
mode, and every mean lies at least 0.5 (RGB) or half a bin (bottlenecks) from the nearest bin edge, i.e. hundreds of
sigmas: every correct implementation gives the same integers, so the containers must equal the oracle's byte for byte.
A sub-pixel equal to its predicted mean codes at the mode (>= 65281 of 2^16 counts), any other value in a 1-count tail.

* Host (oracle only): every entry of every coded row is saturated, the mode and tail intervals are what they should
  be, each image reaches both (or, constant, only the mode), the reference's two CDF formulas give the same bytes, and
  log-scale -9 gives the bytes of -7.  The near-saturated families (weights scaled by eps instead of zeroed) reach
  unsaturated entries and the bound of their size comparison is tight.
* GPU, saturated family, all four precision modes, v = level 0, 12 and 24, 64 x 64, 37 x 53 (padded) and 256 x 256:
  compat containers byte-identical to the oracle's and decoded losslessly (also through the coarse RGB decoder at 1, 2
  and 4 streams per CTA), tiled containers whose every stream is the oracle coder's on the oracle's rows in tile order,
  region decodes, banded decode and encode, region updates, ragged batches, and every stream within its slot.
  Ragged batches run in f16 only: the other modes must refuse them (NotImplementedError).  decode_regions, the banded
  paths and update_region run in every mode (decode_regions shares one ragged pass only in f16 / f16x2).
* GPU, near-saturated families: every path lossless and giving the same bytes, the compat size within a bound derived
  from the oracle's intervals.
* GPU, a planted one-bin shift of the bin edges (encoder and decoder alike) is lossless yet fails the byte comparison.
"""
import contextlib
import functools
import struct

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import util

MODES = ['f16', 'f16x2', 'tf32', 'fp32']
LEVELS = [0, 12, 24]                        # both edges of the bottleneck alphabet and an interior level
SIZES = [(64, 64), (37, 53), (256, 256)]
TILES = [(16, 16), (16, 24), (64, 64)]
IMAGES = ['const', 'patch', 'gradient', 'zeros', 'full', 'noise']
M_R = 128
NEAR = [(0.01, -3.0), (0.05, -1.0)]         # (eps, log-scale) of the near-saturated families
NEAR_IMAGES = ['const', 'patch']
NEAR_LEVEL = 12
LOG2E = 1.4426950408889634
SAT_LO, SAT_HI = -25.0, 40.0                # dmll_math.cuh: a term is exactly pi (u <= -25) or nothing (u >= 40)
MAGIC = b'\x46\xE2\x84\x92'


# ----------------------------------------------------------------------------------------------
# the model and the images
# ----------------------------------------------------------------------------------------------
def sharpen(bp, v_level, m_R, log_scale=-9.0, eps=0.0):
    """Make every mixture of `bp` (in place) one sharp logistic: the probability heads' `lin` and the `to_q` convs get
    their weights multiplied by eps (0: zeroed) and the biases below.  Parameter index p*C*K + c*K + k, p = 0 logits
    (+20 on component 0), 1 means (RGB: m_R on R, 0 on G and B; bottlenecks: v = levels[v_level]), 2 log-scales, 3 RGB
    coupling logits (+30 G<-R, -30 B<-R, +30 B<-G: mu_G = x_R, mu_B = x_G).  `to_q` emits v, so every bottleneck
    symbol of every scale is v_level.  The RGB baselines get the RGB part only."""
    net = bp.net
    mods = dict(net.named_modules())
    K = net.config_ms.prob.K

    def head(name, C, means):
        lin = mods[name]
        b = torch.zeros(4 if C == 3 else 3, C, K)
        b[0, :, 0] = 20.
        b[1] = torch.tensor(means, dtype=torch.float32).reshape(C, 1)
        b[2] = log_scale
        if C == 3:
            b[3, 0], b[3, 1], b[3, 2] = 30., -30., 30.
        assert lin.bias.numel() == b.numel(), (name, lin.bias.shape)
        lin.weight.mul_(eps)
        lin.bias.copy_(b.reshape(-1))

    with torch.no_grad():
        head('prob_clfs.0.atrous.lin', 3, [m_R, 0., 0.])
        if not net._rgb:
            for s in range(net.scales):
                v = float(net.nets[s].enc.levels[v_level])
                q = mods['nets.%d.enc.to_q.0' % s]
                q.weight.mul_(eps)
                q.bias.fill_(v)
                if s + 1 < net.scales:                  # prob_clfs[s + 1] codes the symbols nets[s] emits
                    head('prob_clfs.%d.atrous.lin' % (s + 1), q.out_channels, [v] * q.out_channels)
    return bp


@functools.lru_cache(maxsize=None)
def family(cfg, v_level, log_scale=-9.0, eps=0.0):
    """A fresh seed-0 blueprint (never util.blueprint's cached one), sharpened; -> (blueprint, oracle state dict)."""
    from l3c_pytorch_b200 import config
    from l3c_pytorch_b200.blueprint import MultiscaleBlueprint
    torch.manual_seed(0)
    bp = MultiscaleBlueprint(config.ms_config(cfg), device='cuda:0').set_eval()
    sharpen(bp, v_level, M_R, log_scale, eps)
    return bp, util.cpu_state_dict(bp)


def image(name, H, W):
    """uint8 [3, H, W]: constant 128, the same with a 16 x 16 noise patch, an R = G = B ramp over 0..255, all 0,
    all 255, or noise."""
    img = torch.full((3, H, W), 128, dtype=torch.uint8)
    g = torch.Generator().manual_seed(H * 1000 + W)
    if name == 'patch':
        y, x = H // 3, W // 3
        img[:, y:y + 16, x:x + 16] = torch.randint(0, 256, (3, 16, 16), generator=g).to(torch.uint8)
    elif name == 'gradient':
        img = (torch.arange(H * W) * 255 // (H * W - 1)).reshape(1, H, W).expand(3, H, W).to(torch.uint8).clone()
    elif name == 'zeros':
        img.zero_()
    elif name == 'full':
        img.fill_(255)
    elif name == 'noise':
        img = torch.randint(0, 256, (3, H, W), generator=g).to(torch.uint8)
    else:
        assert name == 'const', name
    return img


# ----------------------------------------------------------------------------------------------
# the oracle's rows, streams and containers
# ----------------------------------------------------------------------------------------------
def oracle_coding(sd, cfg_name, img, params=False):
    """What oracle.model.encode_image codes for img (uint8 [3, H, W]) with the 'torch' CDF formula -> (pad tuple,
    [(C, h, w, [(table, sym, dmll, params)] per channel)] coarse -> fine): the uint16 CDF rows [h*w, L+1] (the
    uniform-prior scale: its one shared row, dmll None), the int16 symbols, and (params) the channel's (pi, mu,
    clamped log-scale) [K, h*w]."""
    from oracle import ac, model as om
    cfg = util.oracle_cfg(cfg_name)
    rgb, other = om.dmlls(cfg)
    H, W = img.shape[1:]
    pt = om.pad_tuple(H, W, 2 ** cfg.num_scales)
    x = img.unsqueeze(0).long()
    if any(pt):
        x = F.pad(x, pt, 'constant')
    xf = x.float()
    out = om.forward(sd, cfg, xf)
    scales = []
    for scale in reversed(range(cfg.num_scales + 1)):
        S = out.S[scale]
        _, C, h, w = S.shape
        syms = [S[0, c].reshape(-1).numpy().astype(np.int16) for c in range(C)]
        dm = rgb if scale == 0 else other
        if scale == cfg.num_scales:
            row = ac.uniform_cdf_row(dm.L)
            scales.append((C, h, w, [(row, s, None, None) for s in syms]))
            continue
        l = out.P[scale]
        bn = xf if scale == 0 else out.bn[scale]
        dec = torch.zeros_like(bn)
        rows = []
        for c in range(C):
            table = om.cdf_table_torch_formula(dm, l, c, C, dec)
            rows.append((table, syms[c], dm, om.channel_params(dm, l, c, C, dec) if params else None))
            dec[:, c] = bn[:, c]
        scales.append((C, h, w, rows))
    return pt, scales


def tile_rects(h, w, tile):
    """(y0, x0, y1, x1) of the streams of an h x w plane: the plane, or its tiles in row-major order."""
    if tile is None:
        return [(0, 0, h, w)]
    th, tw = tile
    return [(y, x, min(y + th, h), min(x + tw, w)) for y in range(0, h, th) for x in range(0, w, tw)]


def oracle_container(coding, tile=None):
    """The container of `coding` (oracle_coding's result): every stream oracle.ac.encode of the oracle's rows and
    symbols restated in that stream's order (the whole plane, or one tile in raster order), laid out as the
    reference's .l3c format (tile None) or the tiled one (`L3CT` + u16 tile_h + u16 tile_w after the padding)."""
    from oracle import ac
    pt, scales = coding
    out = bytearray(struct.pack('<4H', *pt))
    if tile is not None:
        out += b'L3CT' + struct.pack('<HH', *tile)
    for (C, h, w, rows) in scales:
        out += struct.pack('<BHH', C, h, w)
        for table, sym, _, _ in rows:
            t2 = table if table.ndim == 1 else table.reshape(h, w, -1)
            s2 = sym.reshape(h, w)
            for (y0, x0, y1, x1) in tile_rects(h, w, tile):
                t = t2 if table.ndim == 1 else t2[y0:y1, x0:x1].reshape(-1, table.shape[-1])
                b = ac.encode(t, s2[y0:y1, x0:x1].reshape(-1))
                out += struct.pack('<I', len(b)) + b
        out += MAGIC
    return bytes(out)


@functools.lru_cache(maxsize=None)
def expected(cfg, v_level, size, with_tiles=True):
    """{image name: {None: compat container, tile: tiled container}} of the saturated family at `size`."""
    _, sd = family(cfg, v_level)
    res = {}
    for name in IMAGES:
        coding = oracle_coding(sd, cfg, image(name, *size))
        res[name] = {t: oracle_container(coding, t) for t in [None] + (TILES if with_tiles else [])}
    return res


def entry_args(dm, prm):
    """float64 [K, n, L+1]: the argument u = -(t - mu) / sigma * log2(e) of every term of every CDF entry."""
    _, mu, ls = prm
    t = dm.targets().numpy().astype(np.float64)
    inv = np.exp(-ls.astype(np.float64)) * LOG2E
    return -(t[None, None, :] - mu.astype(np.float64)[:, :, None]) * inv[:, :, None]


def saturated(dm, prm):
    """bool [n, L+1]: entries whose every term is saturated (a sum of pi's, the same integer everywhere)."""
    u = entry_args(dm, prm)
    return np.all((u <= SAT_LO) | (u >= SAT_HI), axis=0)


def widths(table, sym=None):
    """Interval widths in counts: of the coded symbols, or (sym None) of every symbol of every row."""
    t = table.astype(np.int64)
    if sym is None:
        return (t[:, 1:] - t[:, :-1]) % 65536
    i, s = np.arange(sym.size), sym.astype(np.int64)
    return (t[i, s + 1] - t[i, s]) % 65536


def size_bound(coding):
    """Bound of |bytes - oracle bytes| for a coder whose CDF entries equal the oracle's where saturated and lie within
    +-1 count elsewhere: the largest code-length change of every coded symbol, summed, plus 2 bytes per stream."""
    bits, n_streams = 0.0, 0
    for (_, _, _, rows) in coding[1]:
        for table, sym, dm, prm in rows:
            if dm is None:                              # the uniform prior: integers, coded identically
                continue
            sat = saturated(dm, prm)
            i, s = np.arange(sym.size), sym.astype(np.int64)
            w = widths(table, sym).astype(np.float64)
            d = (~sat[i, s]).astype(np.float64) + (~sat[i, s + 1])
            lo, hi = np.maximum(w - d, 1.0), w + d
            bits += float(np.maximum(np.log2(w / lo), np.log2(hi / w)).sum())
            n_streams += 1
    return bits / 8 + 2 * n_streams


def slot_caps_hold(datas):
    """Every stream of every container within codec._slot_cap(its symbols); -> the largest length / cap."""
    from l3c_pytorch_b200.codec import _slot_cap, container_tile, parse_container
    worst = 0.0
    for d in datas:
        tile = container_tile(d)
        for (C, H, W, streams) in parse_container(d)[1]:
            n_sym = [(y1 - y0) * (x1 - x0) for (y0, x0, y1, x1) in tile_rects(H, W, tile)] * C
            for (_, n), k in zip(streams, n_sym):
                assert n <= _slot_cap(k), (n, k, _slot_cap(k))
                worst = max(worst, n / _slot_cap(k))
    return worst


@contextlib.contextmanager
def precision(mode):
    from l3c_pytorch_b200 import engine as E
    old = E.get_conv_precision()
    E.set_conv_precision(mode)
    try:
        yield
    finally:
        E.set_conv_precision(old)


def lossless(outs, imgs):
    for o, img in zip(outs, imgs):
        assert o.shape == (1,) + tuple(img.shape) and torch.equal(o[0].cpu(), img.long())


# ----------------------------------------------------------------------------------------------
# host: the regime every case is meant to reach (oracle only)
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('size', [(64, 64), (37, 53)])
@pytest.mark.parametrize('cfg,v', [('cr', 0), ('cr', 12), ('cr', 24), ('cr_rgb_shared', 0)])
def test_saturated_regime(cfg, v, size):
    from oracle import model as om
    _, sd = family(cfg, v)
    _, sd7 = family(cfg, v, -7.0)
    ocfg = util.oracle_cfg(cfg)
    for name in IMAGES:
        img = image(name, *size)
        coding = oracle_coding(sd, cfg, img, params=True)
        n_mode = n_tail = 0
        for (_, _, _, rows) in coding[1]:
            for table, sym, dm, prm in rows:
                if dm is None:
                    continue
                assert np.abs(entry_args(dm, prm)).min() >= SAT_HI, name       # every term of every entry
                w = widths(table)
                mode = w.argmax(1)
                wmode = w[np.arange(w.shape[0]), mode]
                assert wmode.min() >= (65281 if dm.rgb else 65512), name
                w[np.arange(w.shape[0]), mode] = 1
                assert (w == 1).all(), name                                      # every other symbol: a 1-count tail
                at_mode = sym.astype(np.int64) == mode
                ws = widths(table, sym)
                assert (ws[at_mode] == wmode[at_mode]).all() and (ws[~at_mode] == 1).all()
                n_mode += int(at_mode.sum())
                n_tail += int((~at_mode).sum())
        # the zero padding of an odd size codes R in the tail, also around a constant image
        assert n_mode > 0 and (n_tail == 0) == (name == 'const' and not any(coding[0])), (name, n_mode, n_tail)
        torch_bytes = om.encode_image(sd, ocfg, img, 'torch')
        assert oracle_container(coding) == torch_bytes, name                 # the restatement the GPU tests use
        assert om.encode_image(sd, ocfg, img, 'kernel') == torch_bytes, name
        assert om.encode_image(sd7, ocfg, img, 'torch') == torch_bytes, name  # below the clamp = at the clamp
        assert torch.equal(om.decode_image(sd, ocfg, torch_bytes, 'torch')[0], img.long()), name
        print('saturated %s v=%d %dx%d %s: %d B, %d symbols at the mode, %d in the tail'
              % (cfg, v, size[0], size[1], name, len(torch_bytes), n_mode, n_tail))


@pytest.mark.parametrize('eps,log_scale', NEAR)
def test_near_saturated_regime(eps, log_scale):
    """Unsaturated entries are reached, the reference's two formulas differ but stay within the bound, and the bound
    says something (< 10 % of the container)."""
    from oracle import model as om
    _, sd = family('cr', NEAR_LEVEL, log_scale, eps)
    for name in NEAR_IMAGES:
        img = image(name, 64, 64)
        coding = oracle_coding(sd, 'cr', img, params=True)
        unsat = sum(int((~saturated(dm, prm)).sum()) for (_, _, _, rows) in coding[1]
                    for (_, _, dm, prm) in rows if dm is not None)
        assert unsat > 0
        bound = size_bound(coding)
        t = om.encode_image(sd, om.CFG_L3C, img, 'torch')
        k = om.encode_image(sd, om.CFG_L3C, img, 'kernel')
        assert oracle_container(coding) == t
        assert abs(len(k) - len(t)) <= bound and bound < 0.1 * len(t), (len(k), len(t), bound)
        print('near-saturated eps=%g log-scale %g %s: %d B, bound %.1f B (%.2f %%), %d unsaturated entries, '
              'kernel formula %+d B' % (eps, log_scale, name, len(t), bound, 100 * bound / len(t), unsat,
                                        len(k) - len(t)))


# ----------------------------------------------------------------------------------------------
# GPU: the saturated family, byte for byte
# ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('size', SIZES)
@pytest.mark.parametrize('v', LEVELS)
@pytest.mark.parametrize('mode', MODES)
def test_compat_bytes(mode, v, size):
    """3a, 3e, 3f: compat containers equal the oracle's; the oracle's decode losslessly (in f16 also through the coarse
    RGB decoder at 1, 2 and 4 streams per CTA); no stream outgrows its slot."""
    from l3c_pytorch_b200 import Bitcoding, engine as E
    bp, _ = family('cr', v)
    imgs = [image(n, *size) for n in IMAGES]
    want = expected('cr', v, size)
    bc = Bitcoding(bp)
    with precision(mode):
        datas, _ = bc.encode_batch(torch.stack(imgs))
        for name, d in zip(IMAGES, datas):
            assert d == want[name][None], (name, len(d), len(want[name][None]))
        oracle_files = [want[n][None] for n in IMAGES]
        E.launch_log(reset=True)
        lossless(bc.decode_batch(oracle_files), imgs)
        kernels = E.launch_log(reset=True)[0]
        if mode == 'f16':                               # the RGB scale of a compat f16 decode runs on coarse records
            assert any('coarse' in k for k in kernels), kernels
            for spc in (1, 2, 4):
                with E.decoder_streams_per_cta(spc):
                    lossless(bc.decode_batch(oracle_files), imgs)
    worst = slot_caps_hold(datas)
    print('compat %s v=%d %dx%d: %s B, largest stream / slot %.3f'
          % (mode, v, size[0], size[1], [len(d) for d in datas], worst))


@pytest.mark.gpu
@pytest.mark.parametrize('size', SIZES)
@pytest.mark.parametrize('v', LEVELS)
@pytest.mark.parametrize('mode', MODES)
def test_tiled_streams(mode, v, size, monkeypatch):
    """3b, 3f: every stream of a tiled container is the oracle coder's on the oracle's rows in that tile's order, many
    of them 1-3 bytes; lossless, region decodes equal the crops, and the banded decode and encode give the same."""
    from l3c_pytorch_b200 import Bitcoding, codec
    bp, _ = family('cr', v)
    imgs = [image(n, *size) for n in IMAGES]
    want = expected('cr', v, size)
    H, W = size
    Wp = -(-W // 8) * 8
    regions = [(0, 0, H, W), (H // 4, W // 5, H // 2, W // 3), (H - 1, W - 1, 1, 1), (3, W // 2, 17, W - W // 2),
               (H // 3, 0, 16, 16), (H // 2, W // 3, H - H // 2, 5)]
    with precision(mode):
        for tile in TILES:
            bct = Bitcoding(bp, tile=tile)
            datas, _ = bct.encode_batch(torch.stack(imgs))
            for name, d in zip(IMAGES, datas):
                assert d == want[name][tile], (tile, name, len(d), len(want[name][tile]))
            slot_caps_hold(datas)
            lossless(bct.decode_batch(datas), imgs)
            for d, img, (y, x, h, w) in zip(datas, imgs, regions):
                assert torch.equal(bct.decode_region(d, (y, x, h, w))[0].cpu(), img[:, y:y + h, x:x + w].long())
            for got, img, (y, x, h, w) in zip(bct.decode_regions(datas, regions), imgs, regions):
                assert torch.equal(got[0].cpu(), img[:, y:y + h, x:x + w].long()), (tile, (y, x, h, w))
            # bands of one tile row at the finest scale
            monkeypatch.setattr(codec, 'TILED_BAND_PIXELS', len(imgs) * tile[0] * Wp)
            monkeypatch.setattr(codec, 'TILED_ENCODE_BAND_PIXELS', len(imgs) * tile[0] * Wp)
            lossless(bct.decode_batch(datas), imgs)
            assert bct.encode_batch(torch.stack(imgs))[0] == datas, tile
            monkeypatch.undo()
        short = sum(n <= 3 for d in datas for (_, _, _, st) in codec.parse_container(d)[1] for (_, n) in st)
        print('tiled %s v=%d %dx%d: %d streams of 1-3 bytes' % (mode, v, size[0], size[1], short))


@pytest.mark.gpu
@pytest.mark.parametrize('size', SIZES)
@pytest.mark.parametrize('v', LEVELS)
@pytest.mark.parametrize('mode', MODES)
def test_update_region(mode, v, size):
    """3c: a noise patch (its symbols in the tails) gives the oracle's container of the edited image; a patch equal to
    the old pixels gives the container back unchanged."""
    from l3c_pytorch_b200 import Bitcoding
    bp, sd = family('cr', v)
    H, W = size
    tile = (16, 16)
    y, x, h, w = H // 2 - 5, W // 3, 13, 21
    patch = torch.randint(0, 256, (3, h, w), generator=torch.Generator().manual_seed(H + W))
    bct = Bitcoding(bp, tile=tile)
    with precision(mode):
        for name in ('const', 'gradient'):
            img = image(name, H, W)
            data = expected('cr', v, size)[name][tile]
            edited = img.clone()
            edited[:, y:y + h, x:x + w] = patch.to(torch.uint8)
            got = bct.update_region(data, (y, x), patch)
            assert got == oracle_container(oracle_coding(sd, 'cr', edited), tile), name
            assert not bct.codec.update_counts['whole']
            lossless(bct.decode_batch([got]), [edited])
            assert bct.update_region(data, (y, x), img[:, y:y + h, x:x + w]) == data


@pytest.mark.gpu
@pytest.mark.parametrize('v', LEVELS)
@pytest.mark.parametrize('mode', MODES)
def test_ragged_batch(mode, v):
    """3d: in f16 every image of every size in one call, each container the oracle's; the other modes refuse a batch
    of different sizes before coding anything."""
    from l3c_pytorch_b200 import Bitcoding
    bp, _ = family('cr', v)
    bc = Bitcoding(bp)
    imgs = [image(n, *size) for size in SIZES for n in IMAGES]
    with precision(mode):
        if mode != 'f16':
            with pytest.raises(NotImplementedError, match='f16'):
                bc.encode_batch(imgs)
            return
        datas, _ = bc.encode_batch(imgs)
        want = [expected('cr', v, size)[n][None] for size in SIZES for n in IMAGES]
        for k, (d, wd) in enumerate(zip(datas, want)):
            assert d == wd, (k, len(d), len(wd))
        lossless(bc.decode_batch(datas), imgs)


@pytest.mark.gpu
@pytest.mark.parametrize('size', SIZES)
def test_rgb_shared_f16x2(size):
    """3g: the RGB baseline (bench.py's second workload) in f16x2: compat containers equal the oracle's."""
    from l3c_pytorch_b200 import Bitcoding
    bp, _ = family('cr_rgb_shared', 0)
    imgs = [image(n, *size) for n in IMAGES]
    want = expected('cr_rgb_shared', 0, size, with_tiles=False)
    bc = Bitcoding(bp)
    with precision('f16x2'):
        datas, _ = bc.encode_batch(torch.stack(imgs))
        for name, d in zip(IMAGES, datas):
            assert d == want[name][None], (name, len(d), len(want[name][None]))
        lossless(bc.decode_batch(datas), imgs)
    slot_caps_hold(datas)


# ----------------------------------------------------------------------------------------------
# GPU: near-saturated families, a bounded comparison
# ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('eps,log_scale', NEAR)
@pytest.mark.parametrize('mode', MODES)
def test_near_saturated(mode, eps, log_scale, monkeypatch):
    from l3c_pytorch_b200 import Bitcoding, codec
    from oracle import model as om
    bp, sd = family('cr', NEAR_LEVEL, log_scale, eps)
    imgs = [image(n, 64, 64) for n in NEAR_IMAGES]
    other = image('noise', 40, 56)                      # another size: the f16 batch below is ragged
    tile = (16, 24)
    bc, bct = Bitcoding(bp), Bitcoding(bp, tile=tile)
    with precision(mode):
        compat, _ = bc.encode_batch(torch.stack(imgs))
        lossless(bc.decode_batch(compat), imgs)
        if mode == 'f16':
            ragged, _ = bc.encode_batch(imgs + [other])
            assert ragged[:len(imgs)] == compat
            lossless(bc.decode_batch(ragged), imgs + [other])
        tiled, _ = bct.encode_batch(torch.stack(imgs))
        lossless(bct.decode_batch(tiled), imgs)
        for d, img in zip(tiled, imgs):
            assert torch.equal(bct.decode_region(d, (10, 20, 30, 25))[0].cpu(), img[:, 10:40, 20:45].long())
        monkeypatch.setattr(codec, 'TILED_ENCODE_BAND_PIXELS', len(imgs) * tile[0] * 64)
        assert bct.encode_batch(torch.stack(imgs))[0] == tiled
        monkeypatch.undo()
        patch = torch.randint(0, 256, (3, 9, 11), generator=torch.Generator().manual_seed(5))
        for d, img in zip(tiled, imgs):
            edited = img.clone()
            edited[:, 30:39, 7:18] = patch.to(torch.uint8)
            assert bct.update_region(d, (30, 7), patch) == bct.encode_batch(edited.unsqueeze(0))[0][0]
    for name, img, d in zip(NEAR_IMAGES, imgs, compat):
        t = om.encode_image(sd, om.CFG_L3C, img, 'torch')
        bound = size_bound(oracle_coding(sd, 'cr', img, params=True))
        print('near-saturated %s eps=%g log-scale %g %s: %d B, oracle %d B, bound %.1f B'
              % (mode, eps, log_scale, name, len(d), len(t), bound))
        assert bound < 0.1 * len(t)
        assert abs(len(d) - len(t)) <= bound, (name, len(d), len(t), bound)


# ----------------------------------------------------------------------------------------------
# GPU: a planted fault that a lossless round trip cannot see
# ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['f16', 'fp32'])
def test_plant_shifted_bin_edges(mode, monkeypatch):
    """Encoder and decoder both read the bin edges one bin up: the file still decodes, but no longer equals the
    oracle's, and every symbol at the mode now sits in a 1-count tail (about 2 bytes more each)."""
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    bp, _ = family('cr', 12)
    H, W = 64, 64
    img = image('const', H, W)
    want = expected('cr', 12, (H, W))['const'][None]
    bc = Bitcoding(bp)
    with precision(mode):
        assert bc.encode_batch(img.unsqueeze(0))[0][0] == want
        shifted, orig = {}, DiscretizedMixLogisticLoss.targets

        def targets(self, device):
            key = (id(self), str(device))          # kept alive: kernels on other streams read it
            if key not in shifted:
                shifted[key] = orig(self, device) + self.bin_width
            return shifted[key]
        monkeypatch.setattr(DiscretizedMixLogisticLoss, 'targets', targets)
        bad = bc.encode_batch(img.unsqueeze(0))[0][0]
        lossless(bc.decode_batch([bad]), [img])
        torch.cuda.synchronize()
        monkeypatch.undo()
    assert bad != want
    n_mode = 3 * H * W + 5 * (H * W // 4 + H * W // 16)          # every DMLL-coded symbol of the constant image
    grow = len(bad) - len(want)
    assert 1.9 * n_mode <= grow <= 2.1 * n_mode, (grow, n_mode)
