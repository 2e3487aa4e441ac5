"""GPU: region decode of tiled containers (DESIGN §4.8).  A region decoded from only the tiles and decoder windows
it depends on equals, bit for bit, the same crop of the full decode: in every precision for `cr`, in f16x2 and f16
for `cr_rgb_shared` (also every level of a recursive container), for several tile sizes on images that are not
multiples of the tile, with padding, for interior, edge and corner regions.  Also: batches of regions, what is
decoded (launch log and the plan's counts) and a run on 3 SMs."""
import contextlib

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


def _regions(H, W):
    """Interior, edge, corner, 1x1 and whole-image regions of an H x W image."""
    return [(H // 2 - 9, W // 2 - 13, 17, 23),                 # interior
            (0, W // 3, 11, 20), (H - 7, W // 4, 7, 30),     # top and bottom edge
            (H // 3, 0, 25, 6), (H // 4, W - 9, 12, 9),      # left and right edge
            (0, 0, 13, 13), (H - 5, W - 21, 5, 21),          # corners
            (H // 2, W // 2, 1, 1), (0, 0, H, W)]


def _check(bc, data, full, regions):
    for reg in regions:
        y, x, h, w = reg
        got = bc.decode_region(data, reg)
        assert got.dtype == torch.int64 and tuple(got.shape) == (1, 3, h, w) and got.is_cuda
        assert torch.equal(got, full[:, :, y:y + h, x:x + w]), 'region %s differs from the full decode' % (reg,)


@pytest.mark.parametrize('cfg,mode,tile', [
    ('cr', 'f16', (64, 64)), ('cr', 'f16', (32, 48)), ('cr', 'f16', (16, 16)),
    ('cr', 'f16x2', (32, 48)), ('cr', 'tf32', (32, 48)), ('cr', 'fp32', (32, 48)),
    ('cr_rgb_shared', 'f16x2', (32, 48)), ('cr_rgb_shared', 'f16', (16, 16)), ('cr_rgb_shared', 'f16', (64, 64))])
def test_region_equals_crop_of_full_decode(cfg, mode, tile):
    from l3c_pytorch_b200 import Bitcoding
    bp = util.blueprint(cfg)
    H, W = 150, 196                                         # padded to 152 x 200 (cr), not a multiple of any tile
    img = util.make_image(300, H, W)
    with _precision(mode):
        bc = Bitcoding(bp, tile=tile)
        datas, _ = bc.encode_batch([img])
        full = bc.decode_batch(datas)[0]
        assert torch.equal(full[0].cpu(), img.long())
        _check(bc, datas[0], full, _regions(H, W))


@pytest.mark.parametrize('mode', ['f16x2', 'f16'])
def test_recursive_container_every_level(mode):
    from l3c_pytorch_b200 import Bitcoding
    bp = util.blueprint('cr_rgb_shared')
    img = util.make_image(310, 90, 70)                        # padded to 96 x 72 for R = 2
    with _precision(mode):
        bc = Bitcoding(bp, tile=(16, 16), recursive=2)
        datas, _ = bc.encode_batch([img])
        full = bc.decode_batch(datas)[0]
        assert torch.equal(full[0].cpu(), img.long())
        _check(bc, datas[0], full, _regions(90, 70)[:3] + [(89, 69, 1, 1)])
        x, _ = bc._prepare(img, quiet=True)
        thumbs = bp.forward(x, auto_recurse=2).S_u8            # the stored pyramid, fine -> coarse
        assert len(thumbs) == 4
        for k in range(1, 4):
            Hk, Wk = thumbs[k].shape[-2:]
            for reg in [(Hk // 2 - 3, Wk // 2 - 2, 5, 4), (0, 0, Hk, Wk), (Hk - 2, Wk - 3, 2, 3)]:
                y, x0, h, w = reg
                got = bc.decode_region(datas[0], reg, level=k)
                assert torch.equal(got, thumbs[k][:, :, y:y + h, x0:x0 + w].long()), (k, reg)


def test_whole_image_region_and_mixed_batches():
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    with _precision('f16'):
        bc = Bitcoding(bp, tile=(32, 32))
        imgs = [util.make_image(320, 128, 192), util.make_image(321, 128, 192), util.make_image(322, 96, 80)]
        datas = [bc.encode_batch([im])[0][0] for im in imgs]
        fulls = bc.decode_batch(datas)
        for d, f, im in zip(datas, fulls, imgs):
            assert torch.equal(bc.decode_region(d, (0, 0) + tuple(im.shape[1:])), f)
        # a mixed list: plans of equal shape (the same region of the two large images) share one pass, the rest run
        # one after another
        regions = [(40, 70, 20, 30), (50, 100, 20, 30), (10, 10, 30, 30), (0, 0, 128, 192), (40, 70, 20, 30)]
        order = [0, 1, 2, 0, 1]
        _, plans = bc.codec.plan_regions([datas[i] for i in order], regions)
        keys = [p.shape_key() for p in plans]
        assert keys[0] == keys[4] and len(set(keys)) == 4
        many = bc.decode_regions([datas[i] for i in order], regions)
        for i, reg, got in zip(order, regions, many):
            assert torch.equal(got, bc.decode_region(datas[i], reg))
            y, x, h, w = reg
            assert torch.equal(got, fulls[i][:, :, y:y + h, x:x + w])
        # a shared pass launches what one region launches
        torch.cuda.synchronize()
        E.launch_log(reset=True)
        bc.decode_region(datas[0], regions[0])
        one = E.launch_log(reset=True)[1]
        bc.decode_regions([datas[0], datas[1]], [regions[0]] * 2)
        assert E.launch_log(reset=True)[1] == one


def test_interior_region_decodes_only_the_planned_streams():
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200.codec import parse_container
    bp = util.blueprint('cr')
    with _precision('f16'):
        bc = Bitcoding(bp, tile=(32, 32))
        img = util.make_image(330, 256, 320)
        datas, _ = bc.encode_batch([img])
        region = (128, 160, 16, 16)                            # inside one 32 x 32 tile
        _, plans = bc.codec.plan_regions(datas, [region])
        plan = plans[0]
        E.launch_log(reset=True)
        got = bc.decode_region(datas[0], region)
        torch.cuda.synchronize()
        kernels, _ = E.launch_log(reset=True)
        assert torch.equal(got, bc.decode_batch(datas)[0][:, :, 128:144, 160:176])
        counts = bc.codec.region_counts
        assert counts == {'streams': plan.streams, 'symbols': plan.symbols}
        _, scales = parse_container(datas[0])
        assert plan.streams < sum(len(st) for (_, _, _, st) in scales)
        fin = plan.scales[-1]
        assert fin.symbols < 3 * 256 * 320 and len(fin.tiles) == 1
        # one decoder launch per bottleneck scale and per RGB channel, one row build each
        assert kernels.get('dmll_table_kernel', 0) == 3 + 2
        dec = sum(n for k, n in kernels.items() if k.startswith('ac_decode'))
        assert dec == 1 + 3 + 2, kernels
        # symbols for each of the three nets, features for the two fused ones (dec.skip), and the result
        assert kernels.get('crop_rect_kernel', 0) == 3 + 2 + 1


def test_region_on_three_sms():
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    with _precision('f16'):
        bc = Bitcoding(bp, tile=(32, 48))
        img = util.make_image(340, 150, 196)
        datas, _ = bc.encode_batch([img])
        full = bc.decode_batch(datas)[0]
        with E.conv_launch_limits(max_sms=3):
            got = bc.decode_regions(datas * 2, [(60, 70, 30, 40), (0, 150, 20, 46)])
    assert torch.equal(got[0], full[:, :, 60:90, 70:110])
    assert torch.equal(got[1], full[:, :, 0:20, 150:196])


def test_region_refusals_before_any_kernel():
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    img = util.make_image(350, 64, 64)
    with _precision('f16'):
        plain, _ = Bitcoding(bp).encode_batch([img])
        tiled, _ = Bitcoding(bp, tile=(16, 16)).encode_batch([img])
        rgb, _ = Bitcoding(util.blueprint('cr_rgb_shared'), tile=(16, 16)).encode_batch([img])
        torch.cuda.synchronize()
        bc = Bitcoding(bp)
        E.launch_log(reset=True)
        for datas, reg, lev, match in [(plain, (0, 0, 8, 8), 0, 'tile='), (tiled, (0, 0, 0, 8), 0, 'empty'),
                                       (tiled, (60, 0, 8, 8), 0, 'outside'), (tiled, (0, 0, 8, 8), 1, 'not images'),
                                       (tiled, (0, 0, 8, 8), 7, 'does not exist'), (rgb, (0, 0, 8, 8), 0, 'model')]:
            with pytest.raises(ValueError, match=match):
                bc.decode_regions(datas, [reg], [lev])
        with pytest.raises(ValueError, match='model'):
            bc.decode_regions(tiled + rgb, [(0, 0, 8, 8)] * 2)
        assert E.launch_log(reset=True)[1] == 0


def test_cli_region(tmp_path):
    from PIL import Image
    from l3c_pytorch_b200 import Bitcoding, cli
    bp = util.blueprint('cr_rgb_shared')
    img = util.make_image(360, 70, 90)
    png = tmp_path / 'x.png'
    Image.fromarray(img.permute(1, 2, 0).numpy()).save(str(png))
    data, _ = Bitcoding(bp, tile=(32, 32)).encode_batch([img])
    f = tmp_path / 'x.l3c'
    f.write_bytes(data[0])
    out = tmp_path / 'r.png'
    assert cli.main(['--config', 'cr_rgb_shared', 'dec', str(f), str(out), '--region', '10,20,30,40']) == 0
    back = np.array(Image.open(str(out)))
    assert np.array_equal(back, img.permute(1, 2, 0).numpy()[10:40, 20:60])
    (tmp_path / 'y.l3c.part0').write_bytes(data[0])
    assert cli.main(['--config', 'cr_rgb_shared', 'dec', str(tmp_path / 'y.l3c'), str(out), '--region',
                     '0,0,4,4']) == 1
