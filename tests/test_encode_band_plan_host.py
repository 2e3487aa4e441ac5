"""CPU: the planner and the routing of the banded encode of large tiled images (DESIGN §4.10).

* Encoder bands cover every output row of every scale exactly once, and every window starts on an even row.
* NaN dependency check of the encoder chain (head, 5x5/s2 down conv, body, to_q) run with torch CPU convs on the module
  weights: with NaN everywhere outside a band's window, the band's rows of F_{s+1} and of the to_q output stay finite,
  and moving a window edge that is not an image edge inward by one stride step lets NaN in.
* encode_banded is true exactly above TILED_ENCODE_BAND_PIXELS, for tiled, equal-size batches without `out`.
* `enc --tile` reads images above Pillow's decompression-bomb limit; without --tile that limit still holds."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from tests import util


def _net(cfg='cr'):
    return util.blueprint(cfg, device='cpu').net


def _conv(m, x):
    return Fn.conv2d(x, m.weight.detach().double(), m.bias.detach().double(), m.stride, m.padding, m.dilation)


def _encoder_chain(net, s, x):
    """heads[s] + nets[s].enc on an NCHW float64 tensor: -> (F_{s+1}, to_q output)."""
    enc = net.nets[s].enc
    head = net.heads[0].head[1].head if s == 0 else net.heads[s].head
    h = _conv(head, x)
    d = _conv(enc.down, h)
    y = d
    body = list(enc.body)
    for blk in body[:-1]:
        y = _conv(blk.body[2], torch.relu(_conv(blk.body[0], y))) + y
    F = _conv(body[-1], y) + d
    return F, _conv(enc.to_q[0], F)


@pytest.mark.parametrize('H,rows', [(200, 7), (200, 100), (128, 1), (96, 200), (64, 13)])
def test_encoder_bands_cover_every_row_once(H, rows):
    from l3c_pytorch_b200.region import EncoderGeometry, plan_encoder_bands
    net = _net()
    geo = EncoderGeometry(net)
    assert geo.radii[0] == dict(head=1, down=2, body=17, to_q=0)
    for s in range(net.scales):
        Hs = H >> s
        bands = plan_encoder_bands(geo, s, Hs, rows)
        seen = np.zeros(Hs // 2, np.int64)
        for b in bands:
            (a, e), (r0, r1) = b.window, b.rows
            assert a % 2 == 0 and 0 <= a < e <= Hs and b.out == r0 - a // 2
            seen[r0:r1] += 1
        assert (seen == 1).all() and len(bands) == -(-(Hs // 2) // rows)


def test_encoder_planner_refusals():
    from l3c_pytorch_b200.region import plan_encoder_bands
    with pytest.raises(ValueError, match='RGB baselines'):
        plan_encoder_bands(_net('cr_rgb_shared'), 0, 64, 4)
    with pytest.raises(ValueError, match='no encoder'):
        plan_encoder_bands(_net(), 3, 64, 4)
    with pytest.raises(ValueError, match='at least one row'):
        plan_encoder_bands(_net(), 0, 64, 0)


@pytest.mark.parametrize('s,H,rows', [(0, 200, 30), (1, 176, 16), (2, 160, 24)])
def test_nan_outside_an_encoder_window_stays_outside_its_rows(s, H, rows):
    from l3c_pytorch_b200.region import EncoderGeometry, plan_encoder_bands
    net = _net()
    geo = EncoderGeometry(net)
    W = 20
    cin = 3 if s == 0 else net.config_ms.Cf
    g = torch.Generator().manual_seed(s)
    x = torch.rand(1, cin, H, W, generator=g, dtype=torch.float64) * 2 - 1
    bands = plan_encoder_bands(geo, s, H, rows)
    assert len(bands) >= 3

    def finite_rows(a, e):
        xin = torch.full_like(x, float('nan'))
        xin[:, :, a:e] = x[:, :, a:e]
        F, q = _encoder_chain(net, s, xin)
        return torch.isfinite(F).all(3).all(1)[0], torch.isfinite(q).all(3).all(1)[0]

    for b in bands:
        (a, e), (r0, r1) = b.window, b.rows
        fF, fq = finite_rows(a, e)
        assert fF[r0:r1].all() and fq[r0:r1].all(), (b, fF.int().tolist())
        # every edge that is not an image edge is minimal: one stride step (2 rows) inward lets NaN in
        if a > 0:
            fF, fq = finite_rows(a + 2, e)
            assert not fF[r0:r1].all(), b
        if e < H:
            fF, fq = finite_rows(a, e - 2)
            assert not fF[r0:r1].all(), b


def test_banding_predicate_follows_the_budget(monkeypatch):
    from l3c_pytorch_b200 import codec
    from l3c_pytorch_b200.codec import BatchCodec
    B = codec.TILED_ENCODE_BAND_PIXELS
    assert B == 32 * 512 * 512
    assert not BatchCodec.encode_banded((16, 3, 512, 512), (64, 64))         # bench.py's tiled batch stays whole
    assert not BatchCodec.encode_banded((32, 3, 512, 512), (64, 64))
    assert BatchCodec.encode_banded((33, 3, 512, 512), (64, 64))
    assert BatchCodec.encode_banded((1, 3, 6000, 8000), (64, 64))
    assert not BatchCodec.encode_banded((1, 3, 6000, 8000), None)              # untiled: serial streams
    assert not BatchCodec.encode_banded((1, 3, 6000, 8000), (64, 64), extents=[(6000, 7936)])
    assert not BatchCodec.encode_banded((1, 3, 6000, 8000), (64, 64), out=object())
    monkeypatch.setattr(codec, 'TILED_ENCODE_BAND_PIXELS', 200 * 136 - 1)
    assert BatchCodec.encode_banded((1, 3, 200, 136), (16, 16))
    monkeypatch.setattr(codec, 'TILED_ENCODE_BAND_PIXELS', 200 * 136)
    assert not BatchCodec.encode_banded((1, 3, 200, 136), (16, 16))


def test_cli_tile_reads_images_above_the_pillow_limit(tmp_path, monkeypatch):
    from PIL import Image
    from l3c_pytorch_b200 import cli, codec
    path = str(tmp_path / 'big.png')
    arr = (np.arange(64 * 48 * 3) % 251).astype(np.uint8).reshape(64, 48, 3)
    Image.fromarray(arr).save(path)
    monkeypatch.setattr(Image, 'MAX_IMAGE_PIXELS', 64 * 48 // 4)      # 4x the limit: Pillow refuses it
    with pytest.raises(Image.DecompressionBombError):
        cli.read_image(path)
    img = cli.read_image(path, codec.MAX_PLANE_PIXELS)
    assert img.shape == (1, 3, 64, 48) and (img[0].permute(1, 2, 0).numpy() == arr).all()
    assert Image.MAX_IMAGE_PIXELS == 64 * 48 // 4                     # restored

    class _Bc(object):
        def __init__(self, tile):
            self.tile = tile

        def encode(self, img, pout):
            return float(img.shape[-1])

    for tile in (None, (16, 16)):
        got = []
        monkeypatch.setattr(cli, 'read_image', lambda p, m=None: got.append(m) or torch.zeros(1, 3, 8, 8))
        cli.encode(_Bc(tile), path, str(tmp_path / 'o.l3c'))
        assert got == [None if tile is None else codec.MAX_PLANE_PIXELS]
