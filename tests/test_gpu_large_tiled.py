"""GPU: whole-image tiled containers and their banded decode (DESIGN §4.10).

* With codec.TILED_BAND_PIXELS patched small (four or more bands at the finest scale, the last one partial), the banded
  decode equals the unbanded one bit for bit and equals the image: `cr` in all four precision modes, `cr_rgb_shared`
  with recursive=2 in f16 and f16x2, one image and a batch of three, with a decode lane and without.
* A 4096 x 3072 image (the classifier's 192-channel buffer is then above 2**31 elements) through `crop=False` encode
  and banded decode of `cr` in f16 and f16x2: lossless, the container equals codec.encode_batch of the same tensor, and a
  512 x 512 decode_region equals the crop of the full decode.
* Peak memory of the banded decode grows with the band, not with the image height.
* `crop=False` writes one file where the reference layout writes parts; the CLI's `enc --tile`, `dec`, `dec --region`.
* A plane beyond codec.MAX_PLANE_PIXELS is refused with ValueError before any kernel runs."""
import contextlib
import os

import numpy as np
import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def _precision(mode):
    from l3c_pytorch_b200 import engine as E
    old = E.get_conv_precision()
    E.set_conv_precision(mode)
    try:
        yield
    finally:
        E.set_conv_precision(old)


def _decode(bc, datas, lane=None):
    if lane is None:
        return bc.codec.decode_batch(datas, to_host=False)[0]
    with torch.cuda.stream(lane.main):
        S = bc.codec.decode_batch(datas, to_host=False, lane=lane)[0]
    torch.cuda.current_stream().wait_stream(lane.main)
    return S


@pytest.mark.parametrize('cfg,mode,R', [('cr', 'f16', 0), ('cr', 'f16x2', 0), ('cr', 'tf32', 0), ('cr', 'fp32', 0),
                                        ('cr_rgb_shared', 'f16', 2), ('cr_rgb_shared', 'f16x2', 2)])
def test_banded_equals_unbanded(cfg, mode, R, monkeypatch):
    from l3c_pytorch_b200 import Bitcoding, codec
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200.region import plan_bands
    bp = util.blueprint(cfg)
    H, W, tile = 200, 136, (16, 16)                     # 13 tile rows at the finest scale, the last one 8 rows high
    imgs = torch.stack([util.make_image(400 + i, H, W) for i in range(3)])
    with _precision(mode):
        bc = Bitcoding(bp, tile=tile, recursive=R)
        datas, _ = bc.encode_batch(imgs)
        lane = bc.decode_lanes(3, 1)[0]
        for batch in ([datas[0]], datas):
            N = len(batch)
            E.launch_log(reset=True)
            whole = _decode(bc, batch)
            torch.cuda.synchronize()
            k_whole = E.launch_log(reset=True)[0]
            # three tile rows per band at the finest scale: 5 bands, the last one partial
            monkeypatch.setattr(codec, 'TILED_BAND_PIXELS', 3 * N * tile[0] * W)
            shapes = [(C, h, w) for (C, h, w, _) in codec.parse_container(batch[0])[1]]
            bands = plan_bands(shapes, tile, bp.net, len(shapes) - 1, 3)
            assert len(bands) >= 4 and bands[-1].rect[2] - bands[-1].rect[0] < 3 * tile[0]
            for ln in (None, lane):
                E.launch_log(reset=True)
                got = _decode(bc, batch, ln)
                torch.cuda.synchronize()
                k_band = E.launch_log(reset=True)[0]
                assert torch.equal(got, whole), (N, ln is not None)
                assert k_band.get('dmll_table_kernel', 0) > k_whole.get('dmll_table_kernel', 0)
            monkeypatch.setattr(codec, 'TILED_BAND_PIXELS', 32 * 512 * 512)
            assert torch.equal(whole.cpu(), imgs[:N])


@pytest.mark.parametrize('mode', ['f16', 'f16x2'])
def test_large_image_whole_container(mode, tmp_path):
    from l3c_pytorch_b200 import Bitcoding, codec
    bp = util.blueprint('cr')
    H, W = 3072, 4096
    assert 192 * H * W > 2 ** 31
    img = util.make_image(410, H, W)
    with _precision(mode):
        bc = Bitcoding(bp, tile=(64, 64), crop=False)
        out = str(tmp_path / 'big.l3c')
        bc.encode(img, out)
        assert not os.path.exists(out + '.part0')
        with open(out, 'rb') as f:
            data = f.read()
        ref, _ = bc.codec.encode_batch(img.unsqueeze(0).cuda(), tile=(64, 64))
        assert data == ref[0]
        assert H * W > codec.TILED_BAND_PIXELS                 # the finest scale decodes in bands
        full = bc.decode(out)
        assert torch.equal(full[0].cpu(), img.long())
        y, x = 1500, 2100
        reg = bc.decode_region(data, (y, x, 512, 512))
        assert torch.equal(reg, full[:, :, y:y + 512, x:x + 512])


def _peak_of_decode(bc, data):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    S = bc.codec.decode_batch([data], to_host=False)[0]
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del S
    return peak


@pytest.mark.parametrize('cfg', ['cr_rgb_shared', 'cr'])
def test_banded_peak_memory_grows_with_the_band(cfg, monkeypatch):
    """Doubling the height with the band fixed adds less than 64 B per added pixel to the decode's peak (what stays
    whole: the symbol planes, the coarser scale's values and, for cr, the coarser decoder's features); an unbanded
    decode takes about 2 KB per pixel (DESIGN §7)."""
    from l3c_pytorch_b200 import Bitcoding, codec
    bp = util.blueprint(cfg)
    W, H = 1024, 768
    monkeypatch.setattr(codec, 'TILED_BAND_PIXELS', 256 * 1024)
    peaks = []
    with _precision('f16'):
        bc = Bitcoding(bp, tile=(64, 64), crop=False)
        for h in (H, 2 * H):
            data = bc.encode_batch([util.make_image(420, h, W)])[0][0]
            _peak_of_decode(bc, data)                    # warm: the allocator's first blocks
            peaks.append(_peak_of_decode(bc, data))
    per_px = (peaks[1] - peaks[0]) / (H * W)
    assert per_px < 64, (peaks, per_px)


def test_crop_false_writes_one_file(tmp_path, monkeypatch):
    from l3c_pytorch_b200 import Bitcoding
    monkeypatch.setenv('AC_NEEDS_CROP_DIM', '64,64')
    bp = util.blueprint('cr')
    img = util.make_image(430, 96, 136)
    with _precision('f16'):
        one = str(tmp_path / 'one.l3c')
        Bitcoding(bp, tile=(32, 32), crop=False).encode(img, one)
        assert os.path.isfile(one) and not os.path.exists(one + '.part0')
        parts = str(tmp_path / 'parts.l3c')
        Bitcoding(bp, tile=(32, 32)).encode(img, parts)
        assert not os.path.exists(parts) and os.path.isfile(parts + '.part0') and os.path.isfile(parts + '.part3')
        bc = Bitcoding(bp)
        assert torch.equal(bc.decode(one)[0].cpu(), img.long())
        assert torch.equal(bc.decode(parts + '.part0')[0].cpu(), img.long())


def test_cli_enc_tile_dec_and_region(tmp_path, monkeypatch):
    from PIL import Image
    from l3c_pytorch_b200 import cli
    monkeypatch.setenv('AC_NEEDS_CROP_DIM', '64,64')
    img = util.make_image(440, 90, 70)
    png = tmp_path / 'x.png'
    Image.fromarray(img.permute(1, 2, 0).numpy()).save(str(png))
    f = tmp_path / 'x.l3c'
    assert cli.main(['--config', 'cr_rgb_shared', 'enc', str(png), str(f), '--tile', '32,32']) == 0
    assert f.is_file() and not (tmp_path / 'x.l3c.part0').exists()
    back = tmp_path / 'back.png'
    assert cli.main(['--config', 'cr_rgb_shared', 'dec', str(f), str(back)]) == 0
    assert np.array_equal(np.array(Image.open(str(back))), img.permute(1, 2, 0).numpy())
    assert cli.main(['--config', 'cr_rgb_shared', 'dec', str(f), str(back), '--region', '10,20,30,40']) == 0
    assert np.array_equal(np.array(Image.open(str(back))), img.permute(1, 2, 0).numpy()[10:40, 20:60])


def test_plane_beyond_the_limit_refused_before_any_kernel():
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200.codec import ContainerLayout, tile_grid
    bp = util.blueprint('cr')
    H, W, tile = 32768, 32776, (4096, 4096)                # one pixel row more than 2**30 pixels
    shapes = [(5, H >> 3, W >> 3), (5, H >> 2, W >> 2), (5, H >> 1, W >> 1), (3, H, W)]
    layout = ContainerLayout([(n, C, h, w) for n, (C, h, w) in enumerate(shapes)], tile)
    total, pieces, _ = layout.header_and_offsets(
        np.zeros(sum(C * len(tile_grid(h, w, tile)) for (C, h, w) in shapes), np.int64), (0, 0, 0, 0))
    buf = bytearray(total)
    for o, b in pieces:
        buf[o:o + len(b)] = b
    bc = Bitcoding(bp, tile=tile, crop=False)
    torch.cuda.synchronize()
    E.launch_log(reset=True)
    with pytest.raises(ValueError, match='more than'):
        bc.codec.decode_batch([bytes(buf)])
    with pytest.raises(ValueError, match='more than'):
        bc.decode_region(bytes(buf), (0, 0, 64, 64))
    big = torch.zeros(1, 3, 1, 1, dtype=torch.uint8, device='cuda').expand(1, 3, H, W)   # no storage of that size
    with pytest.raises(ValueError, match='more than'):
        bc.codec.encode_batch(big, tile=tile)
    assert E.launch_log(reset=True)[1] == 0
