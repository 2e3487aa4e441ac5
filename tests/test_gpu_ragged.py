"""GPU: ragged batches (DESIGN §4.6) -- images of different sizes in one padded batch.  Every output inside an
image's extent must carry the same bits as the per-image launch, every container must equal the one of the image
coded alone, and the decode must be lossless."""
import numpy as np
import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu

NAN16 = float('nan')


@pytest.fixture
def f16():
    from l3c_pytorch_b200 import engine as E
    old = E.get_conv_precision()
    E.set_conv_precision('f16')
    yield
    E.set_conv_precision(old)


# image smaller than one 8 x 16 output tile, widths that are not multiples of 16
EXT = [(24, 40), (8, 8), (16, 24), (40, 16), (32, 48)]
LIMITS = [(0, 0), (1, 0), (2, 0), (3, 0), (7, 0), (3, 112), (7, 160)]


def _ragged(ext, C, dtype, seed, fill=NAN16, scale=1):
    """NaN-filled padded batch [N,Hb,Wb,C] with random images in the extents, and the images alone"""
    g = torch.Generator().manual_seed(seed)
    Hb, Wb = max(h for h, _ in ext) * scale, max(w for _, w in ext) * scale
    x = torch.full((len(ext), Hb, Wb, C), fill, dtype=dtype)
    alone = []
    for n, (h, w) in enumerate(ext):
        v = (torch.randn(1, h * scale, w * scale, C, generator=g) * 2).to(dtype)
        x[n, :h * scale, :w * scale] = v[0]
        alone.append(v.cuda())
    return x.cuda(), alone


def _band_is_pos_zero(x, ext, halo):
    b = x.view(torch.int16) if x.dtype == torch.float16 else x.view(torch.int32)
    H, W = x.shape[1:3]
    for n, (h, w) in enumerate(ext):
        band = torch.zeros(H, W, dtype=torch.bool, device=x.device)
        band[:min(h + halo, H), :min(w + halo, W)] = True
        band[:h, :w] = False
        if not bool((b[n][band] == 0).all()):
            return False
    return True


def _conv_cases(bp):
    net = bp.net
    return {
        '3x3_d1_relu': (net.nets[0].enc.body[0].body[0], dict(relu=True)),
        '3x3_d2': (net.prob_clfs[0].atrous.atrous[1], {}),
        '3x3_d4': (net.prob_clfs[0].atrous.atrous[2], {}),
        '5x5_s2': (net.nets[0].enc.down, {}),
        'pixel_shuffle': (net.nets[0].dec.tail[0], dict(pixel_shuffle=True)),
    }


@pytest.mark.parametrize('case', ['3x3_d1_relu', '3x3_d2', '3x3_d4', '5x5_s2', 'pixel_shuffle'])
def test_tensor_core_convs_of_a_ragged_batch_equal_per_image_launches(case, f16):
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    conv, kw = _conv_cases(bp)[case]
    x, alone = _ragged(EXT, 64, torch.float16, 7)
    want = [E.conv2d(conv, E.Act(None, a), **kw) for a in alone]
    halo = conv.dilation[0] * (conv.kernel_size[0] // 2)
    f = 0.5 if conv.stride[0] == 2 else (2 if kw.get('pixel_shuffle') else 1)
    for max_sms, kb in LIMITS:
        xr = x.clone()
        with E.conv_launch_limits(max_sms=max_sms, conv_smem_kb=kb), E.ragged_extents(EXT, *x.shape[1:3]):
            got = E.conv2d(conv, E.Act(None, xr), **kw)
        assert _band_is_pos_zero(xr, EXT, halo), (case, max_sms, kb)
        for n, (h, w) in enumerate(EXT):
            ho, wo = int(h * f), int(w * f)
            assert torch.equal(got[n, :ho, :wo], want[n][0]), (case, n, max_sms, kb)


def test_ffma_1x1_with_residual_of_a_ragged_batch(f16):
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    conv = bp.net.nets[0].dec.head                                   # q.C -> Cf, CUDA cores, + residual
    x, alone = _ragged(EXT, 8, torch.float32, 3)
    r, ralone = _ragged(EXT, 64, torch.float32, 4)
    want = [E.conv2d(conv, a, residual=ra) for a, ra in zip(alone, ralone)]
    with E.ragged_extents(EXT, *x.shape[1:3]):
        got = E.conv2d(conv, x, residual=r)
    for n, (h, w) in enumerate(EXT):
        assert torch.equal(got[n, :h, :w], want[n][0]), n


def test_rgb_head_of_a_ragged_batch(f16):
    """im2col taps outside an image's extent are 0 as at its border; the K = 64 GEMM then gives the same bits"""
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    net = bp.net
    args = (net.sub_rgb_mean, net.heads[0].head[0], net.heads[0].head[1].head)
    ext = [(16, 24), (8, 8), (24, 40), (40, 16)]
    Hb, Wb = 40, 40
    g = torch.Generator().manual_seed(5)
    batch = torch.randint(0, 256, (len(ext), 3, Hb, Wb), generator=g, dtype=torch.uint8)   # garbage margins
    alone = [batch[n:n + 1, :, :h, :w].contiguous().cuda() for n, (h, w) in enumerate(ext)]
    want = [E.rgb_head_f16(a, *args).r for a in alone]
    for max_sms, kb in LIMITS:
        with E.conv_launch_limits(max_sms=max_sms, conv_smem_kb=kb), E.ragged_extents(ext, Hb, Wb):
            got = E.rgb_head_f16(batch.cuda(), *args).r
        for n, (h, w) in enumerate(ext):
            assert torch.equal(got[n, :h, :w], want[n][0]), (n, max_sms, kb)


# ---------------------------------------------------------------------------------------------
# model
# ---------------------------------------------------------------------------------------------
SHAPES = [(32, 32), (48, 24), (16, 64), (64, 40), (8, 8)]


def _batch(shapes, seed=0):
    Hb, Wb = max(h for h, _ in shapes), max(w for _, w in shapes)
    imgs = [util.make_image(seed + i, h, w) for i, (h, w) in enumerate(shapes)]
    batch = torch.zeros(len(shapes), 3, Hb, Wb, dtype=torch.uint8)
    for n, im in enumerate(imgs):
        batch[n, :, :im.shape[1], :im.shape[2]] = im
    return imgs, batch.cuda()


def test_ragged_forward_equals_per_image_forwards(f16):
    bp = util.blueprint('cr')
    imgs, batch = _batch(SHAPES)
    out = bp.net(batch, extents=SHAPES)
    outi = bp.net(batch, intervals_of=bp.losses, extents=SHAPES)
    for n, im in enumerate(imgs):
        one = bp.net(im.unsqueeze(0).cuda())
        onei = bp.net(im.unsqueeze(0).cuda(), intervals_of=bp.losses)
        for s in range(4):
            h, w = SHAPES[n][0] >> s, SHAPES[n][1] >> s
            assert torch.equal(out.S_u8[s][n, :, :h, :w], one.S_u8[s][0]), (n, s)
            if s > 0:
                assert torch.equal(out.bn8[s][n, :h, :w], one.bn8[s][0]), (n, s)
            if s < 3:
                assert torch.equal(out.P_nhwc[s][n, :h, :w], one.P_nhwc[s][0]), (n, s)
                C = outi.S_u8[s].shape[1]
                iv = outi.IV[s].view(len(imgs), C, outi.S_u8[s].shape[2], -1)
                assert torch.equal(iv[n, :, :h, :w], onei.IV[s][0].view(C, h, w)), (n, s)
    # decoder side: the get_P_nhwc chain reproduces the ragged forward bit-exactly, also on 3 SMs
    from l3c_pytorch_b200 import engine as E
    for max_sms in (0, 3):
        F_prev = None
        with E.conv_launch_limits(max_sms=max_sms):
            for s in (2, 1, 0):
                l, F_prev = bp.net.get_P_nhwc(s, out.bn8[s + 1], F_prev, extents=SHAPES)
                for n, (h, w) in enumerate(SHAPES):
                    assert torch.equal(l[n, :h >> s, :w >> s], out.P_nhwc[s][n, :h >> s, :w >> s]), (s, n, max_sms)


# ---------------------------------------------------------------------------------------------
# codec
# ---------------------------------------------------------------------------------------------
CODEC_SIZES = [(32, 32), (40, 28), (64, 96), (24, 200), (136, 72), (48, 536)]


def _codec_images():
    g0, g1 = util.golden_npz('l3c_32x32_i0'), util.golden_npz('l3c_40x28_i1')
    imgs = [torch.from_numpy(g0['img']), torch.from_numpy(g1['img'])]
    imgs += [util.make_image(20 + i, h, w) for i, (h, w) in enumerate(CODEC_SIZES[2:])]
    assert [tuple(im.shape[1:]) for im in imgs] == CODEC_SIZES
    return imgs


def test_ragged_encode_matches_per_image_and_decodes_in_one_pass(f16):
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200 import engine as E
    bc = Bitcoding(util.blueprint('cr'))
    imgs = _codec_images()
    want = [bc.encode_batch(im.unsqueeze(0)) for im in imgs]
    E.launch_log(reset=True)
    datas, bpsps = bc.encode_batch(imgs)
    log, _ = E.launch_log(reset=True)
    assert log.get('rgb_im2col_kernel') == 1 and log.get('ac_encode_kernel') == 1, log     # one pass, one launch
    for n in range(len(imgs)):
        assert datas[n] == want[n][0][0], n
        assert bpsps[n] == want[n][1][0], n
    # tuple input, [1,3,H,W] images
    assert bc.encode_batch(tuple(im.unsqueeze(0) for im in imgs))[0] == datas
    # decode: one pass, as many range-decoder launches as the largest image alone
    big = int(np.argmax([h * w for (h, w) in CODEC_SIZES]))
    bc.decode_batch([datas[big]])
    n_alone = E.launch_log(reset=True)[0].get('ac_decode_kernel')
    dec = bc.decode_batch(datas)
    assert E.launch_log(reset=True)[0].get('ac_decode_kernel') == n_alone
    for n, im in enumerate(imgs):
        assert dec[n].shape == (1,) + tuple(im.shape) and torch.equal(dec[n][0].cpu(), im.long()), n
    # a budget that forces several passes gives the same bytes and images
    from l3c_pytorch_b200 import bitcoding
    old = bitcoding.RAGGED_PASS_PIXELS
    bitcoding.RAGGED_PASS_PIXELS = 3 * 136 * 96
    try:
        assert len(bitcoding.plan_passes([(h + (-h) % 8, w + (-w) % 8) for (h, w) in CODEC_SIZES])) > 2
        assert bc.encode_batch(imgs)[0] == datas
        dec2 = bc.decode_batch(datas)
        assert all(torch.equal(a, b) for a, b in zip(dec, dec2))
    finally:
        bitcoding.RAGGED_PASS_PIXELS = old


def test_ragged_encode_on_the_side_stream_beside_a_ragged_decode(f16):
    from l3c_pytorch_b200 import Bitcoding
    bc = Bitcoding(util.blueprint('cr'))
    a = [util.make_image(50 + i, h, w) for i, (h, w) in enumerate([(64, 48), (24, 80), (40, 40)])]
    b = [util.make_image(60 + i, h, w) for i, (h, w) in enumerate([(32, 96), (56, 24), (16, 16), (48, 48)])]
    datas_a, _ = bc.encode_batch(a)
    want_b, _ = bc.encode_batch(b)
    side = bc.side_stream(len(a))
    lane = bc.decode_lanes(len(a), n_lanes=1)[0]
    cur = torch.cuda.current_stream()
    job = bc.encode_batch_begin([im.pin_memory() for im in b], stream=side)
    lane.main.wait_stream(cur)
    with torch.cuda.stream(lane.main):
        dec_a = bc.decode_batch(datas_a, lane=lane)
    assert job.finish()[0] == want_b
    cur.wait_stream(lane.main)
    torch.cuda.synchronize()
    for im, d in zip(a, dec_a):
        assert torch.equal(d[0].cpu(), im.long())


def test_crops_of_different_shapes_share_one_pass(tmp_path, monkeypatch, f16):
    from l3c_pytorch_b200 import Bitcoding, auto_crop
    from l3c_pytorch_b200 import engine as E
    monkeypatch.setenv('AC_NEEDS_CROP_DIM', '40,40')
    bc = Bitcoding(util.blueprint('cr'))
    img = util.make_image(9, 97, 61).unsqueeze(0)
    crops = list(auto_crop.iter_crops(img))
    assert len({(c.shape[2] + (-c.shape[2]) % 8, c.shape[3] + (-c.shape[3]) % 8) for c in crops}) == 2
    p = str(tmp_path / 'x.l3c')
    E.launch_log(reset=True)
    bc.encode(img.long(), p)
    assert E.launch_log(reset=True)[0].get('ac_encode_kernel') == 1
    for i, c in enumerate(crops):
        with open(p + '.part%d' % i, 'rb') as f:
            assert f.read() == bc.encode_batch(c.contiguous())[0][0], i
    dec = bc.decode(p + '.part0')
    assert torch.equal(dec.cpu(), img.long())


def test_unsupported_ragged_combinations_raise():
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200 import engine as E
    ims = [util.make_image(0, 32, 32), util.make_image(1, 16, 48)]
    old = E.get_conv_precision()
    try:
        for prec in ('fp32', 'tf32', 'f16x2'):
            E.set_conv_precision(prec)
            bc = Bitcoding(util.blueprint('cr'))
            with pytest.raises(NotImplementedError, match=prec):
                bc.encode_batch(ims)
            _, batch = _batch([(32, 32), (16, 48)])
            with pytest.raises(NotImplementedError, match=prec):
                bc.codec.encode_batch(batch, extents=[(32, 32), (16, 48)])
            with pytest.raises(NotImplementedError, match=prec):
                bc.blueprint.net(batch, extents=[(32, 32), (16, 48)])
        E.set_conv_precision('f16')
        with pytest.raises(NotImplementedError, match='RGB baselines'):
            Bitcoding(util.blueprint('cr_rgb_shared')).encode_batch(ims)
        with pytest.raises(NotImplementedError, match='tiled'):
            Bitcoding(util.blueprint('cr'), tile=(16, 16)).encode_batch(ims)
        # equally sized lists take the equal-size path everywhere
        E.set_conv_precision('fp32')
        bc = Bitcoding(util.blueprint('cr'))
        same = [util.make_image(2, 32, 32), util.make_image(3, 32, 32)]
        datas, _ = bc.encode_batch(same)
        assert datas == bc.encode_batch(torch.stack(same))[0]
    finally:
        E.set_conv_precision(old)
