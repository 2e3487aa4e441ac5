"""GPU: every conv-stack kernel against a plain PyTorch fp32 CPU reference of the same op
(floating point: rtol 2e-5 / atol 2e-5 for the fp32 FFMA path -- only the accumulation order
differs from MKL-DNN)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import util

pytestmark = pytest.mark.gpu
RTOL, ATOL = 2e-5, 2e-5
FP32 = 0      # _lib.PREC_FP32: these tests pin the CUDA-core path whatever the session default is


def _conv_module(cin, cout, k, stride=1, rate=1, seed=0):
    from l3c_pytorch_b200.network import default_conv
    torch.manual_seed(seed)
    return default_conv(cin, cout, k, rate=rate, stride=stride)


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous().cuda()


@pytest.mark.parametrize('cin,cout,k,stride,rate,H,W', [
    (64, 64, 3, 1, 1, 16, 16), (64, 64, 3, 1, 1, 19, 37), (64, 64, 3, 1, 2, 24, 40), (64, 64, 3, 1, 4, 20, 33),
    (64, 64, 5, 2, 1, 32, 48), (64, 64, 5, 2, 1, 18, 22), (64, 256, 3, 1, 1, 12, 20), (192, 120, 1, 1, 1, 9, 31),
    (192, 150, 1, 1, 1, 16, 16), (64, 64, 3, 1, 1, 8, 16)])
def test_conv_vs_torch(cin, cout, k, stride, rate, H, W):
    from l3c_pytorch_b200 import engine as E
    conv = _conv_module(cin, cout, k, stride, rate)
    x = torch.randn(2, cin, H, W)
    want = conv(x).detach()
    got = E.conv2d(conv.cuda(), _nhwc(x), precision=FP32).cpu().permute(0, 3, 1, 2)
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=RTOL, atol=ATOL)


def test_conv_epilogues():
    from l3c_pytorch_b200 import engine as E
    conv = _conv_module(64, 64, 3)
    x, r = torch.randn(2, 64, 20, 28), torch.randn(2, 64, 20, 28)
    cc = conv.cuda()
    got = E.conv2d(cc, _nhwc(x), relu=True, precision=FP32).cpu().permute(0, 3, 1, 2)
    np.testing.assert_allclose(got.numpy(), F.relu(conv.cpu()(x)).detach().numpy(), rtol=RTOL, atol=ATOL)
    got = E.conv2d(cc.cuda(), _nhwc(x), residual=_nhwc(r), precision=FP32).cpu().permute(0, 3, 1, 2)
    np.testing.assert_allclose(got.numpy(), (conv.cpu()(x) + r).detach().numpy(), rtol=RTOL, atol=ATOL)
    # channel-slice output (atrous concat)
    buf = torch.zeros(2, 20, 28, 192).cuda()
    E.conv2d(conv.cuda(), _nhwc(x), out=buf, out_coff=64, precision=FP32)
    b = buf.cpu()
    assert (b[..., :64] == 0).all() and (b[..., 128:] == 0).all()
    np.testing.assert_allclose(b[..., 64:128].permute(0, 3, 1, 2).numpy(), conv.cpu()(x).detach().numpy(),
                               rtol=RTOL, atol=ATOL)
    # pixel shuffle
    up = _conv_module(64, 256, 3, seed=3)
    want = F.pixel_shuffle(up(x), 2).detach()
    got = E.conv2d(up.cuda(), _nhwc(x), pixel_shuffle=True, precision=FP32).cpu().permute(0, 3, 1, 2)
    assert got.shape == want.shape
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=RTOL, atol=ATOL)


def test_small_channel_convs_and_padding_lanes():
    """RGB head (Cin=3 in a pitch-4 buffer) and decoder head (Cin=5 in a pitch-8 buffer)."""
    from l3c_pytorch_b200 import engine as E
    head = _conv_module(3, 64, 3, seed=1)
    x = torch.randn(1, 3, 17, 23)
    x4 = torch.zeros(1, 17, 23, 4)
    x4[..., :3] = x.permute(0, 2, 3, 1)
    got = E.conv2d(head.cuda(), x4.cuda(), cin=3, precision=FP32).cpu().permute(0, 3, 1, 2)
    np.testing.assert_allclose(got.numpy(), head.cpu()(x).detach().numpy(), rtol=RTOL, atol=ATOL)
    dh = _conv_module(5, 64, 1, seed=2)
    b = torch.randn(2, 5, 9, 11)
    b8 = torch.zeros(2, 9, 11, 8)
    b8[..., :5] = b.permute(0, 2, 3, 1)
    fuse = torch.randn(2, 64, 9, 11)
    got = E.conv2d(dh.cuda(), b8.cuda(), residual=_nhwc(fuse), precision=FP32).cpu().permute(0, 3, 1, 2)
    np.testing.assert_allclose(got.numpy(), (dh.cpu()(b) + fuse).detach().numpy(), rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize('prec', [0, 1])
def test_conv_independent_of_batch_and_position(prec):
    """enc/dec bit-exactness: the same pixel neighbourhood gives the same bits whatever the batch
    size, image size or tile it lands in -- for the CUDA-core and the tensor-core kernel."""
    from l3c_pytorch_b200 import engine as E
    conv = _conv_module(64, 64, 3).cuda()
    x = torch.randn(3, 64, 40, 56)
    full = E.conv2d(conv, _nhwc(x), precision=prec).cpu()
    one = E.conv2d(conv, _nhwc(x[1:2]), precision=prec).cpu()
    assert torch.equal(full[1:2], one)
    crop = E.conv2d(conv, _nhwc(x[:, :, 8:32, 16:48]), precision=prec).cpu()
    assert torch.equal(full[:, 9:31, 17:47], crop[:, 1:-1, 1:-1])


def test_rgb_prep_and_quantize_head():
    from l3c_pytorch_b200 import engine as E
    from oracle import model as om
    bp = util.blueprint('cr')
    sd = util.cpu_state_dict(bp)
    img = torch.stack([util.make_image(i, 24, 40) for i in range(2)])
    _, t = E.rgb_prep(img.cuda(), bp.net.sub_rgb_mean, bp.net.heads[0].head[0])
    want = om._conv(sd, 'heads.0.head.0', om._conv(sd, 'sub_rgb_mean', img.float()))
    np.testing.assert_allclose(t.cpu()[..., :3].permute(0, 3, 1, 2).numpy(), want.numpy(), rtol=1e-6, atol=1e-6)
    assert (t.cpu()[..., 3] == 0).all()
    # to_q + quantiser
    enc = bp.net.nets[0].enc
    Fm = torch.randn(2, 64, 10, 14) * 0.5
    sym, bnq = E.quantize_head(_nhwc(Fm), enc.to_q[0], enc.levels)
    q_in = om._conv(sd, 'nets.0.enc.to_q.0', Fm)
    S, hard = om.quantize(q_in, sd['nets.0.enc.levels'])
    s_got = sym.cpu().long()
    flips = (s_got != S)
    # a flip is only legitimate when q_in sits on a decision boundary to within float noise
    if flips.any():
        lev = sd['nets.0.enc.levels']
        d = (q_in.unsqueeze(-1) - lev).abs().sort(-1)[0]
        assert ((d[..., 1] - d[..., 0])[flips] < 1e-5).all()
    assert flips.float().mean() < 1e-3
    lev = sd['nets.0.enc.levels']
    assert torch.equal(bnq.cpu()[..., :5].permute(0, 3, 1, 2), lev[s_got])     # exactly levels[S]
    assert (bnq.cpu()[..., 5:] == 0).all()
    back = E.symbols_to_values(sym, enc.levels.detach())
    assert torch.equal(back.cpu(), bnq.cpu())                                   # decoder side == encoder side


def test_bicubic_matches_pillow():
    from PIL import Image
    from l3c_pytorch_b200 import engine as E
    for (H, W) in [(64, 64), (50, 38), (256, 256), (33, 17)]:
        img = torch.stack([util.make_image(i, H, W) for i in range(2)])
        # smooth one of them so that the test is not only noise
        img[1] = torch.from_numpy(np.clip(np.cumsum(np.cumsum(img[1].numpy().astype(np.int32) - 127, 1), 2) // 40 + 128,
                                          0, 255).astype(np.uint8))
        got = E.bicubic_half(img.cuda()).cpu()
        for n in range(2):
            pil = Image.fromarray(img[n].permute(1, 2, 0).numpy())
            w, h = pil.size
            want = torch.from_numpy(np.array(pil.resize((int(w * 0.5), int(h * 0.5)), Image.BICUBIC))).permute(2, 0, 1)
            assert torch.equal(got[n], want), (H, W, n, (got[n].int() - want.int()).abs().max())


@pytest.mark.parametrize('cout,rate,H,W,kw', [(64, 1, 16, 16, {}), (64, 2, 24, 40, {}), (64, 4, 19, 37, {}),
                                              (256, 1, 12, 20, dict(pixel_shuffle=True)), (64, 1, 8, 16, dict(relu=True)),
                                              (64, 1, 3, 5, {})])
def test_tcgen05_conv_vs_torch_on_tf32_operands(cout, rate, H, W, kw):
    """The tensor-core kernel (TMA + wgmma, TF32 operands) against a PyTorch fp32 CPU conv
    fed with the SAME TF32-rounded operands: products are exact, only the fp32 accumulation order
    differs -> rtol 1e-4."""
    from l3c_pytorch_b200 import engine as E, _lib
    conv = _conv_module(64, cout, 3, 1, rate)
    x = torch.randn(2, 64, H, W)
    xr = E.round_to_tf32(x)
    wr = E.round_to_tf32(conv.weight.detach())
    want = F.conv2d(xr, wr, conv.bias.detach(), padding=rate, dilation=rate)
    if kw.get('relu'):
        want = F.relu(want)
    if kw.get('pixel_shuffle'):
        want = F.pixel_shuffle(want, 2)
    xa = E.Act(_nhwc(x), _nhwc(xr))
    got = E.conv2d(conv.cuda(), xa, precision=_lib.PREC_TF32, want='act', **kw)
    np.testing.assert_allclose(got.f.cpu().permute(0, 3, 1, 2).numpy(), want.numpy(), rtol=1e-4, atol=1e-4)
    # the twin written by the epilogue is the RN-TF32 image of the fp32 result
    assert torch.equal(got.r.cpu(), E.round_to_tf32(got.f.cpu()))
    r_only = E.conv2d(conv.cuda(), xa, precision=_lib.PREC_TF32, want='round', **kw)
    assert torch.equal(r_only.f.cpu(), got.r.cpu())


@pytest.mark.parametrize('cin,cout,H,W', [(192, 120, 9, 31), (192, 150, 16, 16), (64, 64, 8, 16)])
def test_tcgen05_1x1_conv(cin, cout, H, W):
    """1x1 convs with Cin % 64 == 0 (the 192 -> Kp head of the probability classifier) also run on the
    tensor cores; Cout need not be a multiple of 64 (weight image is zero padded, stores are guarded)."""
    from l3c_pytorch_b200 import engine as E, _lib
    conv = _conv_module(cin, cout, 1)
    x = E.round_to_tf32(torch.randn(2, cin, H, W))
    want = F.conv2d(x, E.round_to_tf32(conv.weight.detach()), conv.bias.detach())
    got = E.conv2d(conv.cuda(), _nhwc(x), precision=_lib.PREC_TF32)
    assert got.shape == (2, H, W, cout)
    np.testing.assert_allclose(got.cpu().permute(0, 3, 1, 2).numpy(), want.numpy(), rtol=1e-4, atol=1e-4)


def _h(x):
    """fp32 -> the FP16 operand image's value (RN, saturating), as fp32"""
    return x.clamp(-65504.0, 65504.0).half().float()


@pytest.mark.parametrize('cout,rate,H,W,kw', [(64, 1, 16, 16, {}), (64, 2, 24, 40, {}), (64, 4, 19, 37, {}),
                                              (256, 1, 12, 20, dict(pixel_shuffle=True)), (64, 1, 8, 16, dict(relu=True)),
                                              (64, 1, 3, 5, {}), (64, 1, 40, 72, dict(residual=True)),
                                              (128, 1, 17, 33, dict(relu=True)), (64, 4, 64, 48, dict(residual=True))])
def test_f16_conv_vs_torch_on_fp16_operands(cout, rate, H, W, kw):
    """conv_f16.cu (TMA + wgmma, FP16 operands) against a PyTorch fp32 CPU conv fed with the SAME
    FP16-rounded operands: products are exact in fp32, only the accumulation order differs -> rtol 1e-4.
    Also: the three output modes ('plain' fp32, 'act' fp32 + FP16 image, 'round' FP16 image only) agree
    bit for bit, the image is the RN-FP16 of the fp32 result, and nothing is written outside the tensor."""
    from l3c_pytorch_b200 import engine as E, _lib
    kw = dict(kw)
    conv = _conv_module(64, cout, 3, 1, rate)
    x = torch.randn(3, 64, H, W)
    x[0, :, 0, 0] = 1e-6                                           # below the FP16 normal range
    want = F.conv2d(_h(x), _h(conv.weight.detach()), conv.bias.detach(), padding=rate, dilation=rate)
    res = None
    if kw.pop('residual', False):
        r = torch.randn(3, cout, H, W)
        want = want + r
        res = _nhwc(r)
    if kw.get('relu'):
        want = F.relu(want)
    if kw.get('pixel_shuffle'):
        want = F.pixel_shuffle(want, 2)
    xa = E.Act(_nhwc(x))                                           # conv2d makes the FP16 operand image
    cc = conv.cuda()
    got = E.conv2d(cc, xa, precision=_lib.PREC_F16, want='act', residual=res, **kw)
    np.testing.assert_allclose(got.f.cpu().permute(0, 3, 1, 2).numpy(), want.numpy(), rtol=1e-4, atol=1e-4)
    assert got.r.dtype == torch.float16 and got.r.shape == got.f.shape
    assert torch.equal(got.r.cpu(), got.f.cpu().clamp(-65504.0, 65504.0).half())
    plain = E.conv2d(cc, xa, precision=_lib.PREC_F16, want='plain', residual=res, **kw)
    assert torch.equal(plain, got.f)
    r_only = E.conv2d(cc, xa, precision=_lib.PREC_F16, want='round', residual=res, **kw)
    assert r_only.f is None and torch.equal(r_only.r, got.r)
    if not kw.get('pixel_shuffle') and res is None:
        # channel-slice output into a wider FP16 buffer (the atrous concat): neighbours untouched
        buf = torch.full((3, H, W, 3 * cout), 7.0, dtype=torch.float16, device='cuda')
        E.conv2d(cc, xa, precision=_lib.PREC_F16, want='round', residual=res, out=buf, out_coff=cout, **kw)
        assert torch.equal(buf[..., cout:2 * cout], got.r)
        assert bool((buf[..., :cout] == 7).all()) and bool((buf[..., 2 * cout:] == 7).all())


def test_f16_call_makes_its_operand_image_whatever_the_process_mode():
    """conv2d(..., precision=f16) on an fp32-only activation reads the FP16 image of it whatever the process-wide
    mode is: the same bits as when the caller passes that image."""
    from l3c_pytorch_b200 import engine as E, _lib
    conv = _conv_module(64, 64, 3).cuda()
    x = _nhwc(torch.randn(2, 64, 20, 28))
    want = E.conv2d(conv, E.Act(x, x.clamp(-65504.0, 65504.0).half()), precision=_lib.PREC_F16)
    old = E.get_conv_precision()
    try:
        for mode in ('tf32', 'fp32', 'f16x2'):
            E.set_conv_precision(mode)
            got = E.conv2d(conv, E.Act(x), precision=_lib.PREC_F16)
            assert torch.equal(got, want), mode
    finally:
        E.set_conv_precision(old)


@pytest.mark.parametrize('cin,cout,H,W', [(192, 120, 9, 31), (192, 150, 16, 16), (64, 64, 8, 16), (192, 120, 64, 64),
                                          (128, 256, 5, 7)])
def test_f16_1x1_conv(cin, cout, H, W):
    """1x1 convs with Cin % 64 == 0 (the 192 -> Kp head) as GEMM tiles of 64 pixels x all output
    channels; pixel counts that are not multiples of 64 and Cout that is not a multiple of 64."""
    from l3c_pytorch_b200 import engine as E, _lib
    conv = _conv_module(cin, cout, 1)
    x = torch.randn(2, cin, H, W)
    want = F.conv2d(_h(x), _h(conv.weight.detach()), conv.bias.detach())
    xa = E.Act(None, _nhwc(x).half())
    got = E.conv2d(conv.cuda(), xa, precision=_lib.PREC_F16)
    assert got.shape == (2, H, W, cout) and got.dtype == torch.float32
    np.testing.assert_allclose(got.cpu().permute(0, 3, 1, 2).numpy(), want.numpy(), rtol=1e-4, atol=1e-4)
    both = E.conv2d(conv.cuda(), xa, precision=_lib.PREC_F16, want='act', relu=True)
    np.testing.assert_allclose(both.f.cpu().permute(0, 3, 1, 2).numpy(), F.relu(want).numpy(), rtol=1e-4, atol=1e-4)
    assert torch.equal(both.r.cpu(), both.f.cpu().half())


def test_f16_conv_independent_of_batch_and_position():
    """enc/dec bit-exactness of the f16 path: a pixel's result does not depend on the batch size, on which
    image of the batch it is in, or on which tile / pipe / CTA computed it."""
    from l3c_pytorch_b200 import engine as E, _lib
    conv = _conv_module(64, 64, 3).cuda()
    x = torch.randn(5, 64, 40, 56)
    xa = E.Act(None, _nhwc(x).half())
    full = E.conv2d(conv, xa, precision=_lib.PREC_F16)
    one = E.conv2d(conv, E.Act(None, xa.r[3:4].contiguous()), precision=_lib.PREC_F16)
    assert torch.equal(full[3:4], one)
    # same content placed elsewhere in a larger image: interior results (2 px away from the seam) identical
    big = torch.zeros(1, 80, 112, 64, dtype=torch.float16, device='cuda')
    big[0, 24:64, 40:96] = xa.r[3]
    moved = E.conv2d(conv, E.Act(None, big), precision=_lib.PREC_F16)
    assert torch.equal(moved[0, 25:63, 41:95], full[3, 1:39, 1:55])


def test_ffma_writes_the_f16_image():
    """CUDA-core layers (Cin = 3 or 5: RGB head, decoder head) also produce the FP16 operand image in f16 mode."""
    from l3c_pytorch_b200 import engine as E, _lib
    conv = _conv_module(5, 64, 1).cuda()
    x = torch.zeros(2, 20, 36, 8, device='cuda')
    x[..., :5] = torch.randn(2, 20, 36, 5, device='cuda')
    fuse = torch.randn(2, 20, 36, 64, device='cuda')
    old = E.get_conv_precision()
    E.set_conv_precision('f16')
    try:
        got = E.conv2d(conv, x, residual=fuse, want='act')
    finally:
        E.set_conv_precision(old)
    want = E.conv2d(conv, x, residual=fuse, precision=FP32)
    assert torch.equal(got.f, want)
    assert torch.equal(got.r, want.clamp(-65504.0, 65504.0).half())


@pytest.mark.parametrize('H,W,kw', [(32, 48, {}), (18, 22, {}), (19, 37, dict(relu=True)), (64, 64, {}), (5, 7, {})])
def test_f16_down_conv_5x5_stride2(H, W, kw):
    """The encoders' 5x5 / stride-2 conv (net.py:101) on the tensor cores: TMA boxes with element strides
    (2, 2) pick the input pixels of one filter tap; odd sizes, image borders (zero padding = TMA out-of-bounds
    fill at negative and past-the-end coordinates)."""
    from l3c_pytorch_b200 import engine as E, _lib
    conv = _conv_module(64, 64, 5, stride=2)
    x = torch.randn(3, 64, H, W)
    want = F.conv2d(_h(x), _h(conv.weight.detach()), conv.bias.detach(), stride=2, padding=2)
    if kw.get('relu'):
        want = F.relu(want)
    xa = E.Act(None, _nhwc(x).half())
    got = E.conv2d(conv.cuda(), xa, precision=_lib.PREC_F16, want='act', **kw)
    assert got.f.shape == (3, want.shape[2], want.shape[3], 64)
    np.testing.assert_allclose(got.f.cpu().permute(0, 3, 1, 2).numpy(), want.numpy(), rtol=1e-4, atol=1e-4)
    assert torch.equal(got.r.cpu(), got.f.cpu().half())
    # batch / position independence (enc/dec bit-exactness is not needed for the encoder-only layer, but
    # encode_batch(imgs[:1]) must give the same bytes as the first image of a bigger batch)
    one = E.conv2d(conv.cuda(), E.Act(None, xa.r[1:2].contiguous()), precision=_lib.PREC_F16, want='plain', **kw)
    assert torch.equal(one, got.f[1:2])


@pytest.mark.parametrize('rgb,C,L,x_min,x_max,H,W', [(True, 3, 256, 0, 255, 24, 40), (False, 5, 25, -1, 1, 16, 16),
                                                     (True, 3, 256, 0, 255, 7, 9)])
def test_fused_lin_dmll_intervals_equal_the_two_step_path(rgb, C, L, x_min, x_max, H, W):
    """The DMLL head fused into the 1x1 conv (l3c_lin_dmll_intervals) must give the SAME integers as the plain
    F16 1x1 conv followed by l3c_dmll_intervals -- that is what the decoder's rows are built from."""
    from l3c_pytorch_b200 import engine as E, _lib
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    K = 10
    Kp = (4 if rgb else 3) * C * K
    conv = _conv_module(192, Kp, 1).cuda()
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        conv.weight.mul_(3.0)
        if rgb:                                          # plausible means for 0..255 data
            conv.bias[C * K:2 * C * K] = torch.rand(C * K, generator=g).cuda() * 255
            conv.weight[C * K:2 * C * K] *= 20
    cat = (torch.randn(2, H, W, 192, generator=g)).half().cuda()
    sym = torch.randint(0, L, (2, C, H, W), generator=g, dtype=torch.uint8).cuda()
    sym[0, :, 0, 0] = L - 1
    sym[0, :, 0, 1] = 0
    dm = DiscretizedMixLogisticLoss(rgb, x_min, x_max, L)
    tg = dm.targets(cat.device)
    l = E.conv2d(conv, E.Act(None, cat), precision=_lib.PREC_F16)
    want = E.dmll_intervals(l, sym, tg, C, K, L, rgb)
    got = E.lin_dmll_intervals(conv, cat, sym, tg, C, K, L, rgb)
    assert got.shape == want.shape
    assert torch.equal(got, want), int((got != want).sum())


@pytest.mark.parametrize('H,W', [(32, 48), (17, 23), (64, 64)])
def test_rgb_head_im2col_gemm(H, W):
    """f16 mode: RGBHead (MeanShift x2 + conv 3 -> 64, 3x3, zero padding of the NORMALISED input) as im2col + a
    K = 64 tensor-core GEMM, against PyTorch on the same FP16-rounded operands."""
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    net = bp.net
    img = torch.stack([util.make_image(i, H, W) for i in range(2)])
    got = E.rgb_head_f16(img.cuda(), net.sub_rgb_mean, net.heads[0].head[0], net.heads[0].head[1].head)
    assert got.f is None and got.r.shape == (2, H, W, 64) and got.r.dtype == torch.float16
    x = img.float()
    m1, m2, hc = net.sub_rgb_mean.cpu(), net.heads[0].head[0].cpu(), net.heads[0].head[1].head.cpu()
    try:
        z = m2(m1(x)).detach()
        want = F.conv2d(_h(z), _h(hc.weight.detach()), hc.bias.detach(), padding=1)
    finally:
        net.cuda()
    np.testing.assert_allclose(got.r.float().cpu().permute(0, 3, 1, 2).numpy(), want.numpy(), rtol=2e-3, atol=2e-3)


# ---------------------------------------------------------------------------------------------
# precision mode 'f16x2': split-FP16 operands (hi + lo / 2^11), three MMAs per K step, two register accumulators
# ---------------------------------------------------------------------------------------------
def _unsplit(img):
    """split image [..., 2C] -> the fp32 value it stands for"""
    C = img.shape[-1] // 2
    return img[..., :C].float() + img[..., C:].float() / 2048.0


@pytest.mark.parametrize('cout,rate,H,W,kw', [(64, 1, 16, 16, {}), (64, 2, 24, 40, {}), (64, 4, 19, 37, {}),
                                              (256, 1, 12, 20, dict(pixel_shuffle=True)), (64, 1, 8, 16, dict(relu=True)),
                                              (64, 1, 3, 5, {}), (64, 1, 40, 72, dict(residual=True)),
                                              (128, 1, 17, 33, dict(relu=True)), (64, 4, 64, 48, dict(residual=True))])
def test_f16x2_conv_vs_torch_fp32(cout, rate, H, W, kw):
    """conv_f16x2.cu against a PyTorch conv in float64 on the UNROUNDED fp32 operands, at the tolerance of the
    CUDA-core fp32 kernel (RTOL / ATOL of test_conv_vs_torch): the split carries 22 significant bits per operand.
    The output modes agree bit for bit, the split image of the output reproduces it to 2^-21, and a channel-slice
    write leaves the neighbours alone."""
    from l3c_pytorch_b200 import engine as E, _lib
    P = _lib.PREC_F16X2
    kw = dict(kw)
    conv = _conv_module(64, cout, 3, 1, rate)
    x = torch.randn(3, 64, H, W)
    x[0, :, 0, 0] = 1e-6
    want = F.conv2d(x.double(), conv.weight.detach().double(), conv.bias.detach().double(), padding=rate, dilation=rate)
    res = None
    if kw.pop('residual', False):
        r = torch.randn(3, cout, H, W)
        want = want + r.double()
        res = _nhwc(r)
    if kw.get('relu'):
        want = F.relu(want)
    if kw.get('pixel_shuffle'):
        want = F.pixel_shuffle(want, 2)
    xf = _nhwc(x)
    xa = E.Act(xf, E.split_f16x2(xf))
    np.testing.assert_allclose(_unsplit(xa.r).cpu().numpy(), xf.cpu().numpy(), rtol=2.0 ** -20, atol=1e-9)
    cc = conv.cuda()
    got = E.conv2d(cc, xa, precision=P, want='act', residual=res, **kw)
    np.testing.assert_allclose(got.f.cpu().permute(0, 3, 1, 2).numpy(), want.float().numpy(), rtol=RTOL, atol=ATOL)
    co = got.f.shape[-1]
    assert got.r.dtype == torch.float16 and got.r.shape[-1] == 2 * co
    np.testing.assert_allclose(_unsplit(got.r).cpu().numpy(), got.f.cpu().numpy(), rtol=2.0 ** -20, atol=1e-9)
    plain = E.conv2d(cc, xa, precision=P, want='plain', residual=res, **kw)
    assert torch.equal(plain, got.f)
    r_only = E.conv2d(cc, xa, precision=P, want='round', residual=res, **kw)
    assert r_only.f is None and torch.equal(r_only.r, got.r)
    if not kw.get('pixel_shuffle') and res is None:
        buf = torch.full((3, H, W, 2 * 3 * cout), 7.0, dtype=torch.float16, device='cuda')
        E.conv2d(cc, xa, precision=P, want='round', out=buf, out_coff=cout, **kw)
        assert torch.equal(buf[..., cout:2 * cout], got.r[..., :cout])
        assert torch.equal(buf[..., 4 * cout:5 * cout], got.r[..., cout:])
        for lo, hi in ((0, cout), (2 * cout, 4 * cout), (5 * cout, 6 * cout)):
            assert bool((buf[..., lo:hi] == 7).all())


@pytest.mark.parametrize('cin,cout,H,W', [(192, 120, 9, 31), (192, 150, 16, 16), (64, 64, 8, 16), (192, 120, 64, 64),
                                          (128, 256, 5, 7)])
def test_f16x2_1x1_conv(cin, cout, H, W):
    from l3c_pytorch_b200 import engine as E, _lib
    conv = _conv_module(cin, cout, 1)
    x = torch.randn(2, cin, H, W)
    want = F.conv2d(x.double(), conv.weight.detach().double(), conv.bias.detach().double()).float()
    xa = E.Act(None, E.split_f16x2(_nhwc(x)))
    got = E.conv2d(conv.cuda(), xa, precision=_lib.PREC_F16X2)
    assert got.shape == (2, H, W, cout) and got.dtype == torch.float32
    np.testing.assert_allclose(got.cpu().permute(0, 3, 1, 2).numpy(), want.numpy(), rtol=RTOL, atol=ATOL)
    got = E.conv2d(conv.cuda(), xa, precision=_lib.PREC_F16X2, relu=True)
    np.testing.assert_allclose(got.cpu().permute(0, 3, 1, 2).numpy(), F.relu(want).numpy(), rtol=RTOL, atol=ATOL)


def test_f16x2_is_much_closer_to_fp32_than_the_fast_modes():
    """what the strict mode is for: error against float64 ~1000x below the f16 / tf32 modes' (same layer, same
    input), within a small factor of the CUDA-core fp32 kernel's"""
    from l3c_pytorch_b200 import engine as E, _lib
    conv = _conv_module(64, 64, 3)
    x = torch.randn(2, 64, 48, 64)
    want = F.conv2d(x.double(), conv.weight.detach().double(), conv.bias.detach().double(), padding=1)
    cc = conv.cuda()
    err = {}
    xf = _nhwc(x)
    for name, p in (('fp32', _lib.PREC_FP32), ('f16', _lib.PREC_F16), ('f16x2', _lib.PREC_F16X2)):
        got = E.conv2d(cc, E.Act(xf, xf.half()) if name == 'f16' else xf, precision=p).cpu().permute(0, 3, 1, 2).double()
        err[name] = float((got - want).abs().max())
    assert err['f16x2'] < err['f16'] / 200, err
    assert err['f16x2'] < 8 * err['fp32'] + 1e-6, err


def test_f16x2_conv_independent_of_batch_and_position():
    from l3c_pytorch_b200 import engine as E, _lib
    P = _lib.PREC_F16X2
    conv = _conv_module(64, 64, 3).cuda()
    x = torch.randn(5, 64, 40, 56)
    r = E.split_f16x2(_nhwc(x))
    full = E.conv2d(conv, E.Act(None, r), precision=P)
    one = E.conv2d(conv, E.Act(None, r[3:4].contiguous()), precision=P)
    assert torch.equal(full[3:4], one)
    big = torch.zeros(1, 80, 112, 128, dtype=torch.float16, device='cuda')
    big[0, 24:64, 40:96] = r[3]
    moved = E.conv2d(conv, E.Act(None, big), precision=P)
    assert torch.equal(moved[0, 25:63, 41:95], full[3, 1:39, 1:55])
