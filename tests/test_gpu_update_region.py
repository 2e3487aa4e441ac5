"""GPU: region updates of tiled containers (DESIGN §4.12), BatchCodec.update_region / Bitcoding.update_region.

* update_region(encode(img), pos, patch) is byte for byte encode(edited img), and decodes losslessly to it: `cr` in
  f16, f16x2, tf32 and fp32, tiles (16, 16), (16, 24) and (64, 64), edits in the interior, on each edge, in a corner,
  across tile boundaries, 1 x 1 and over the whole image, padded image sizes; a large image whose window lies inside
  it; a patch equal to the old pixels returns the container unchanged; the window path and the whole path (the budget
  monkeypatched) give the same bytes.
* update_counts: the streams the plan re-encodes, fewer than the container's for an interior edit.
* l3c_dmll_intervals_rect equals the whole-plane interval kernel followed by reorder_tiles, restricted to the
  rectangle, full-width rectangles (the bands of a banded encode) included; its refusals.
* Every refusal of update_region raises before any kernel launch; the CLI `upd` round trip."""
import os

import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu

MODES = ['f16', 'f16x2', 'tf32', 'fp32']


@pytest.fixture
def mode():
    from l3c_pytorch_b200 import engine as E
    old = E.get_conv_precision()
    yield E.set_conv_precision
    E.set_conv_precision(old)


def _bc(tile, cfg='cr'):
    from l3c_pytorch_b200.bitcoding import Bitcoding
    return Bitcoding(util.blueprint(cfg, device='cuda:0'), tile=tile, crop=tile is None)


def _image(seed, H, W):
    """A seeded image with smooth structure and noise (uint8 [3, H, W] on the GPU)."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32),
                            indexing='ij')
    base = torch.stack([(yy * 0.37 + xx * 0.11) % 256, (xx * 0.29) % 256, (yy * 0.21 + 60) % 256])
    img = (base + torch.randint(-20, 21, (3, H, W), generator=g)).clamp(0, 255).to(torch.uint8)
    return img.cuda()


def _encode(bc, img):
    return bc.encode_batch([img])[0][0]


def _edits(H, W):
    return {'interior': (H // 2 - 7, W // 2 - 19, 30, 41), 'top': (0, W // 3, 5, 17), 'bottom': (H - 6, 40, 6, 9),
            'left': (H // 3, 0, 12, 3), 'right': (50, W - 4, 7, 4), 'corner': (H - 9, W - 11, 9, 11),
            'tiles': (47, 61, 34, 50), 'pixel': (H // 2, W // 3, 1, 1), 'whole': (0, 0, H, W)}


def _check(bc, data, img, edit, seed):
    y, x, h, w = edit
    patch = torch.randint(0, 256, (3, h, w), generator=torch.Generator().manual_seed(seed), dtype=torch.int64)
    edited = img.clone()
    edited[:, y:y + h, x:x + w] = patch.to(torch.uint8).cuda()
    got = bc.update_region(data, (y, x), patch)
    want = _encode(bc, edited)
    assert got == want, (edit, len(got), len(want))
    dec = bc.decode_batch([got])[0]
    assert torch.equal(dec[0].to(torch.uint8), edited)
    return got


@pytest.mark.parametrize('prec', MODES)
@pytest.mark.parametrize('tile', [(16, 16), (16, 24), (64, 64)])
def test_update_equals_encode_of_the_edited_image(mode, prec, tile):
    mode(prec)
    bc = _bc(tile)
    H, W = 517, 389                                     # padded to 520 x 392
    img = _image(1, H, W)
    data = _encode(bc, img)
    for k, (name, edit) in enumerate(sorted(_edits(H, W).items())):
        _check(bc, data, img, edit, k)
        c = bc.codec.update_counts
        assert not c['whole'] and c['streams'] <= c['total']


@pytest.mark.parametrize('prec', MODES)
def test_update_inside_a_large_image(mode, prec):
    """The window of a small interior edit of a 2600 x 2400 image lies inside the image: every scale's encoder and
    decoder runs on a crop at a non-zero origin."""
    from l3c_pytorch_b200.codec import parse_container
    from l3c_pytorch_b200.region import plan_update
    mode(prec)
    bc = _bc((64, 64))
    H, W = 2600, 2400
    img = _image(2, H, W)
    data = _encode(bc, img)
    edit = (1290, 1170, 20, 33)
    pt, scales = parse_container(data)
    plan = plan_update([s[:3] for s in scales], pt, (64, 64), bc.codec.net, edit)
    P = plan.window
    assert P[0] > 0 and P[1] > 0 and P[2] < H and P[3] < W
    _check(bc, data, img, edit, 7)
    c = bc.codec.update_counts
    assert c['streams'] == plan.streams < c['total'] == plan.total_streams and not c['whole']
    assert c['window_pixels'] == plan.window_pixels < H * W


def test_counts_of_an_interior_edit():
    from l3c_pytorch_b200.codec import parse_container
    from l3c_pytorch_b200.region import plan_update
    bc = _bc((16, 16))
    H, W = 1008, 760
    img = _image(3, H, W)
    data = _encode(bc, img)
    edit = (H // 2, W // 2, 8, 8)
    _check(bc, data, img, edit, 3)
    pt, scales = parse_container(data)
    plan = plan_update([s[:3] for s in scales], pt, (16, 16), bc.codec.net, edit)
    assert bc.codec.update_counts['streams'] == plan.streams < plan.total_streams


def test_unchanged_patch_returns_the_container():
    bc = _bc((16, 24))
    img = _image(4, 301, 255)
    data = _encode(bc, img)
    for (y, x, h, w) in [(100, 90, 40, 33), (0, 0, 301, 255), (300, 254, 1, 1)]:
        assert bc.update_region(data, (y, x), img[:, y:y + h, x:x + w].unsqueeze(0)) == data


def test_whole_path_gives_the_same_bytes(monkeypatch):
    from l3c_pytorch_b200 import codec
    bc = _bc((16, 16))
    H, W = 389, 301
    img = _image(5, H, W)
    data = _encode(bc, img)
    edit = (120, 80, 20, 30)
    window = _check(bc, data, img, edit, 11)
    assert not bc.codec.update_counts['whole']
    wp = bc.codec.update_counts['window_pixels']
    monkeypatch.setattr(codec, 'TILED_ENCODE_BAND_PIXELS', wp - 1)     # the window exceeds the budget: whole path
    whole = _check(bc, data, img, edit, 11)
    assert whole == window and bc.codec.update_counts['whole']
    monkeypatch.setattr(codec, 'TILED_ENCODE_BAND_PIXELS', wp)         # exactly the budget: the window path
    assert _check(bc, data, img, edit, 11) == window and not bc.codec.update_counts['whole']


@pytest.mark.parametrize('rgb', [True, False])
def test_rect_kernel_against_the_whole_plane_kernel(rgb):
    from l3c_pytorch_b200 import engine as E
    dev = torch.device('cuda:0')
    bp = util.blueprint('cr', device='cuda:0')
    dm = bp.losses.loss_dmol_rgb if rgb else bp.losses.loss_dmol_n
    C, K, L = (3 if rgb else 5), 10, dm.L
    Kp = (4 if rgb else 3) * C * K
    N, H, W, tile = 2, 48, 40, (16, 8)
    g = torch.Generator().manual_seed(8)
    l = (torch.randn(N, H + 6, W + 4, Kp, generator=g) * 2).to(dev).contiguous()
    sym = torch.randint(0, L, (N, C, H, W), generator=g, dtype=torch.uint8).to(dev)
    tg = dm.targets(dev)
    oy, ox = 3, 2
    lw = l[:, oy:oy + H, ox:ox + W].contiguous()
    whole = E.dmll_intervals(lw, sym, tg, C, K, L, rgb).view(N, C, H, W)
    for (y0, x0, h, w) in [(16, 8, 16, 16), (0, 0, H, W), (32, 32, 16, 8), (16, 0, 32, 40), (0, 24, 48, 16)]:
        got = E.dmll_intervals_rect(l, oy + y0, ox + x0, sym, (y0, x0, h, w), tg, C, K, L, rgb, tile)
        want = E.reorder_tiles(whole[:, :, y0:y0 + h, x0:x0 + w].contiguous(), h, w, tile, True)
        assert torch.equal(got.view(N, C, -1), want.view(N, C, -1)), (y0, x0, h, w)
        # the same rectangle of a symbol window that sits at (8, 8) of the plane
        win = sym[:, :, 8:, 8:].contiguous()
        if y0 >= 8 and x0 >= 8:
            got = E.dmll_intervals_rect(l, oy + y0, ox + x0, win, (y0 - 8, x0 - 8, h, w), tg, C, K, L, rgb, tile,
                                        origin=(8, 8), plane=(H, W))
            assert torch.equal(got.view(N, C, -1), want.view(N, C, -1))
    E.launch_log(reset=True)
    for kw in [dict(rect=(8, 0, 16, 16)), dict(rect=(0, 4, 16, 8)), dict(rect=(0, 0, 10, 8)),      # not aligned
               dict(rect=(40, 0, 16, 8)), dict(rect=(0, 0, 16, 48)),                              # outside the symbols
               dict(rect=(0, 0, 16, 8), oy=H), dict(rect=(16, 16, 16, 8), origin=(8, 8), plane=(H, W)),
               dict(rect=(0, 0, 16, 8), K=4)]:
        args = dict(oy=0, ox=0, origin=(0, 0), plane=None, K=K)
        args.update(kw)
        with pytest.raises(RuntimeError):
            E.dmll_intervals_rect(l, args['oy'], args['ox'], sym, args['rect'], tg, C, args['K'], L, rgb, tile,
                                  origin=args['origin'], plane=args['plane'])
    lib = E.lib
    iv = torch.empty(N * C * 64, dtype=torch.int32, device=dev)
    assert lib.l3c_dmll_intervals_rect(None, H + 6, W + 4, 0, 0, sym.data_ptr(), H, W, 0, 0, 8, 8, 0, 0, H, W,
                                       tg.data_ptr(), N, C, K, L, int(rgb), 8, 8, iv.data_ptr(), None) != 0
    assert lib.l3c_dmll_intervals_rect(l.data_ptr(), H + 6, W + 4, 0, 0, sym.data_ptr(), H, W, 0, 0, 8, 8, 0, 0, H,
                                       W, tg.data_ptr(), N, 17, K, L, int(rgb), 8, 8, iv.data_ptr(), None) != 0
    assert E.launch_log()[1] == 0


def test_refusals_before_any_launch():
    from l3c_pytorch_b200 import engine as E
    bc = _bc((16, 16))
    img = _image(6, 64, 72)
    data = _encode(bc, img)
    ref = _bc(None)
    ref_data = _encode(ref, img)
    rgb = _bc((16, 16), 'cr_rgb_shared')
    rgb_data = _encode(rgb, img)
    rgb_rec = _bc((16, 16), 'cr_rgb_shared')
    rgb_rec.recursive = 2
    rgb_rec_data = rgb_rec.encode_batch([img])[0][0]
    ok = torch.zeros(3, 4, 4, dtype=torch.uint8)
    cases = [(bc, ref_data, (0, 0), ok, 'tiled container'),
             (bc, rgb_data, (0, 0), ok, 'not written by this model'),
             (rgb, rgb_data, (0, 0), ok, 'RGB baselines'),
             (rgb, rgb_rec_data, (0, 0), ok, 'RGB baselines'),
             (bc, data, (0, 0), torch.zeros(3, 0, 4, dtype=torch.uint8), 'empty'),
             (bc, data, (62, 0), ok, 'outside'),
             (bc, data, (0, -1), ok, 'outside'),
             (bc, data, (0, 0), torch.zeros(1, 4, 4, dtype=torch.uint8), '3 channels'),
             (bc, data, (0, 0), torch.zeros(4, 4, 3, 3, dtype=torch.uint8), '3 channels'),
             (bc, data, (0, 0), torch.full((3, 4, 4), 256, dtype=torch.int64), '0..255'),
             (bc, data, (0, 0), torch.zeros(3, 4, 4, dtype=torch.float32), 'uint8 or int64')]
    torch.cuda.synchronize()
    E.launch_log(reset=True)
    for b, d, pos, patch, match in cases:
        with pytest.raises(ValueError, match=match):
            b.update_region(d, pos, patch)
    assert E.launch_log()[1] == 0


def test_cli_update_round_trip(tmp_path):
    from PIL import Image
    from l3c_pytorch_b200 import cli
    from l3c_pytorch_b200.bitcoding import Bitcoding
    img = _image(9, 131, 97)
    src, patch_p = str(tmp_path / 'img.png'), str(tmp_path / 'patch.png')
    Image.fromarray(img.permute(1, 2, 0).cpu().numpy()).save(src)
    patch = torch.randint(0, 256, (20, 30, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(3))
    Image.fromarray(patch.numpy()).save(patch_p)
    enc, upd = str(tmp_path / 'a.l3c'), str(tmp_path / 'b.l3c')
    assert cli.main(['--config', 'cr', 'enc', src, enc, '--tile', '16,16']) == 0
    assert cli.main(['--config', 'cr', 'upd', enc, patch_p, '40,50', upd]) == 0
    edited = img.clone()
    edited[:, 40:60, 50:80] = patch.permute(2, 0, 1).cuda()
    bc = Bitcoding(cli.load_blueprint('cr'), tile=(16, 16), crop=False)
    with open(upd, 'rb') as f:
        assert f.read() == bc.encode_batch([edited])[0][0]
    assert cli.main(['--config', 'cr', 'upd', enc, patch_p, '40,50', upd]) == 1          # exists, no --overwrite
    assert cli.main(['--config', 'cr', 'upd', enc, patch_p, '40,50', upd, '--overwrite']) == 0
    os.rename(enc, enc + '.part0')
    assert cli.main(['--config', 'cr', 'upd', enc, patch_p, '40,50', upd, '--overwrite']) == 1   # parts refused
    assert cli.main(['--config', 'cr', 'upd', enc + '.part0', patch_p, '0,0', upd, '--overwrite']) == 1
