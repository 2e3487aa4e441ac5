"""The tile queue of the persistent tensor-core kernels (tc_conv.cuh TileQueue).

Each pipe of a persistent kernel claims its tiles from a per-launch counter, so which CTA runs a tile depends on
when the CTAs start.  No output bit may depend on it.  Every kernel that walks tiles (conv_f16_kernel<0> and <1>,
conv1x1_tc_kernel in the three precisions, lin_dmll_f16_kernel, conv3x3_tf32_kernel, conv3x3_f16x2_kernel) runs
here on a few SMs, with many tiles per pipe and wrapped stage rings, under the three schedules of
engine.conv_tile_schedule: 0 dynamic, 1 the static stripe, 2 dynamic with odd CTAs starting late.  All three must
give the same bits, into outputs pre-filled with NaN (or two different fills), which shows every tile was claimed
and written.  The counters must be back at zero after each launch and never shared between streams: the same layer
back to back on one stream and on eight streams at once must give the same bits every time."""
import pytest
import torch

gpu = pytest.mark.gpu
SCHEDULES = (0, 1, 2)
LIMITS = [(3, 0), (7, 112)]          # few SMs: many tiles per pipe; 112 KB: one stage per pipe, rings wrap


def _conv(cin, cout, k, stride=1, rate=1, seed=0):
    from l3c_pytorch_b200.network import default_conv
    torch.manual_seed(seed)
    return default_conv(cin, cout, k, rate=rate, stride=stride).cuda()


def _x(N, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(N, H, W, C, generator=g).cuda()


def _nan(shape, dtype=torch.float32):
    return torch.full(shape, float('nan'), dtype=dtype, device='cuda')


def _same_bits_under_every_schedule(name, run):
    """run() -> {output name: tensor pre-filled with NaN before the launch}; every schedule and launch limit must
    give the bits of the default launch, with no NaN left"""
    from l3c_pytorch_b200 import engine as E
    base = run()
    torch.cuda.synchronize()
    for k, v in base.items():
        assert not torch.isnan(v.float()).any(), '%s: %s not fully written by the default launch' % (name, k)
    for m, kb in LIMITS:
        for mode in SCHEDULES:
            with E.conv_launch_limits(max_sms=m, conv_smem_kb=kb), E.conv_tile_schedule(mode):
                got = run()
            torch.cuda.synchronize()
            for k, want in base.items():
                assert not torch.isnan(got[k].float()).any(), \
                    '%s: %s has unwritten elements (schedule %d, max_sms %d, %d KB)' % (name, k, mode, m, kb)
                assert torch.equal(got[k], want), '%s: %s differs under schedule %d, max_sms %d, %d KB: %d elements' % (
                    name, k, mode, m, kb, int((got[k] != want).sum()))


def _conv_outputs(cc, xa, precision, shape, residual=None, relu=False, f16_image=True):
    """one launch writing fp32 into a NaN buffer, and (f16) one writing the FP16 image into a NaN buffer.  f16x2
    takes no output buffer beside a residual, so that case writes a fresh tensor and is held to equal bits only."""
    from l3c_pytorch_b200 import engine as E, _lib
    if precision == _lib.PREC_F16X2 and residual is not None:
        return {'fp32': E.conv2d(cc, xa, precision=precision, relu=relu, residual=residual)}
    out = {'fp32': E.conv2d(cc, xa, precision=precision, relu=relu, residual=residual, out=_nan(shape))}
    if f16_image:
        out['image'] = E.conv2d(cc, xa, precision=precision, relu=relu, residual=residual,
                                out=_nan(shape, torch.float16), want='round').r
    return out


CASES_3X3 = [('f16_d1_residual', 'f16', 1, True), ('f16_d2_relu', 'f16', 2, False),
             ('tf32_d1_residual', 'tf32', 1, True), ('tf32_d2', 'tf32', 2, False),
             ('f16x2_d1_residual', 'f16x2', 1, True), ('f16x2_d2_one_pipe', 'f16x2', 2, False)]


@gpu
@pytest.mark.parametrize('name,prec,rate,res', CASES_3X3, ids=[c[0] for c in CASES_3X3])
def test_3x3_same_bits_under_every_schedule(name, prec, rate, res):
    """conv_f16_kernel<0>, conv3x3_tf32_kernel, conv3x3_f16x2_kernel at 4 x 64 x 128 x 128 (1024 tiles)"""
    from l3c_pytorch_b200 import engine as E, _lib
    N, H, W = 4, 128, 128
    cc = _conv(64, 64, 3, rate=rate, seed=rate)
    xf = _x(N, 64, H, W, 1 + rate)
    r = _x(N, 64, H, W, 7) if res else None
    P = {'f16': _lib.PREC_F16, 'tf32': _lib.PREC_TF32, 'f16x2': _lib.PREC_F16X2}[prec]
    xa = {'f16': lambda: E.Act(xf, xf.half()), 'tf32': lambda: E.Act(xf, E.round_to_tf32(xf)),
          'f16x2': lambda: E.Act(xf, E.split_f16x2(xf))}[prec]()
    _same_bits_under_every_schedule(
        name, lambda: _conv_outputs(cc, xa, P, (N, H, W, 64), residual=r, relu=not res, f16_image=prec == 'f16'))


@gpu
def test_5x5s2_same_bits_under_every_schedule():
    """conv_f16_kernel<1>: 10 units per tile, 4 x 64 x 255 x 253 in -> 128 x 127 out (1024 tiles)"""
    from l3c_pytorch_b200 import engine as E, _lib
    N, H, W = 4, 255, 253
    cc = _conv(64, 64, 5, stride=2, seed=5)
    xa = E.Act(None, _x(N, 64, H, W, 55).half())
    shape = (N, 128, 127, 64)
    _same_bits_under_every_schedule('conv5x5s2_f16', lambda: _conv_outputs(cc, xa, _lib.PREC_F16, shape, relu=True))


CASES_1X1 = [('f16', 192, 120), ('f16', 64, 256), ('tf32', 64, 64), ('f16x2', 128, 256)]


@gpu
@pytest.mark.parametrize('prec,cin,cout', CASES_1X1, ids=['%s_%d_%d' % c for c in CASES_1X1])
def test_1x1_same_bits_under_every_schedule(prec, cin, cout):
    """conv1x1_tc_kernel<KIND, NB> on 2 x 131 x 257 pixels (1052 pixel tiles; f16x2 at 256 outputs: two Cout
    chunks per pixel tile)"""
    from l3c_pytorch_b200 import engine as E, _lib
    N, H, W = 2, 131, 257
    cc = _conv(cin, cout, 1, seed=cin + cout)
    xf = _x(N, cin, H, W, cin * cout)
    if prec == 'f16':
        xa = E.Act(None, xf.half())
    elif prec == 'tf32':
        xa = E.round_to_tf32(xf)
    else:
        xa = E.Act(None, E.split_f16x2(xf))
    P = {'f16': _lib.PREC_F16, 'tf32': _lib.PREC_TF32, 'f16x2': _lib.PREC_F16X2}[prec]
    _same_bits_under_every_schedule(
        'conv1x1_' + prec, lambda: _conv_outputs(cc, xa, P, (N, H, W, cout), relu=cout == 120, f16_image=prec == 'f16'))


@gpu
@pytest.mark.parametrize('rgb', [True, False], ids=['rgb', 'c5'])
def test_lin_dmll_same_bits_under_every_schedule(rgb):
    """lin_dmll_f16_kernel on 2 x 96 x 160 pixels (480 tiles): every interval written (two different fills give
    the same result) and the same under every schedule"""
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200.engine import _ptr, _stream_ptr, check, lib
    C, K, L = (3, 10, 256) if rgb else (5, 10, 25)
    N, H, W, cin = 2, 96, 160, 192
    Kp = (4 if rgb else 3) * C * K
    cc = _conv(cin, Kp, 1, seed=Kp)
    with torch.no_grad():
        cc.weight.mul_(0.3)
    x_h = (_x(N, cin, H, W, 3) * 0.5).half()
    g = torch.Generator().manual_seed(4)
    sym = torch.randint(0, L, (N, C, H * W), generator=g, dtype=torch.uint8).cuda()
    targets = torch.linspace(-1, 1, L + 1).cuda()
    w_h, b = E._packed_obj(cc).get_f16()

    def run():
        out = {}
        for fill in (0, -1):
            iv = torch.full((N, C, H * W), fill, dtype=torch.int32, device='cuda')
            check(lib.l3c_lin_dmll_intervals(_ptr(x_h), _ptr(w_h), _ptr(b), _ptr(sym), _ptr(targets), N, H * W, cin,
                                             C, K, L, int(rgb), _ptr(iv), _stream_ptr()))
            out['fill%d' % fill] = iv
        assert torch.equal(out['fill0'], out['fill-1']), 'lin_dmll: an interval was not written'
        return out
    _same_bits_under_every_schedule('lin_dmll', run)


def _res_layer():
    from l3c_pytorch_b200 import engine as E, _lib
    N, H, W = 4, 64, 96
    cc = _conv(64, 64, 3, seed=9)
    xf = _x(N, 64, H, W, 19)
    xa = E.Act(xf, xf.half())
    r = _x(N, 64, H, W, 29)
    return lambda: E.conv2d(cc, xa, precision=_lib.PREC_F16, residual=r, out=_nan((N, H, W, 64)))


@gpu
@pytest.mark.parametrize('max_sms', [0, 3])
def test_back_to_back_on_one_stream(max_sms):
    """The counters are zero again after every launch: 40 launches of one layer in a row, the same bits each time"""
    from l3c_pytorch_b200 import engine as E
    run = _res_layer()
    base = run()
    with E.conv_launch_limits(max_sms=max_sms):
        outs = [run() for _ in range(40)]
    torch.cuda.synchronize()
    for i, y in enumerate(outs):
        assert torch.equal(y, base), 'launch %d of 40 differs' % i


@gpu
def test_eight_streams_at_once():
    """Launches in flight on eight streams at the same time never share a counter"""
    from l3c_pytorch_b200 import engine as E
    run = _res_layer()
    base = run()
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(8)]
    outs = []
    with E.conv_launch_limits(max_sms=16):
        for rep in range(6):
            for s in streams:
                with torch.cuda.stream(s):
                    outs.append(run())
    torch.cuda.synchronize()
    for i, y in enumerate(outs):
        assert torch.equal(y, base), 'launch %d (stream %d) differs' % (i, i % 8)


@gpu
def test_skewed_schedule_leaves_ctas_without_tiles():
    """Under schedule 2 the even CTAs take every tile of a small layer before the odd ones start: at least one CTA
    runs no tile, exits normally (its resident weights landed), and the bits are those of the default launch"""
    from l3c_pytorch_b200 import engine as E, _lib
    N, H, W = 1, 32, 64                     # 16 tiles
    cc = _conv(64, 64, 3, seed=3)
    xf = _x(N, 64, H, W, 33)
    xa = E.Act(xf, xf.half())
    base = E.conv2d(cc, xa, precision=_lib.PREC_F16, out=_nan((N, H, W, 64)))
    E.conv_idle_ctas(reset=True)
    with E.conv_launch_limits(max_sms=8), E.conv_tile_schedule(2):
        got = E.conv2d(cc, xa, precision=_lib.PREC_F16, out=_nan((N, H, W, 64)))
    idle = E.conv_idle_ctas(reset=True)
    assert idle >= 1, 'no CTA ran without tiles under the skewed schedule'
    assert torch.equal(got, base)
    # the counters are usable again afterwards
    assert torch.equal(E.conv2d(cc, xa, precision=_lib.PREC_F16, out=_nan((N, H, W, 64))), base)


@gpu
def test_schedule_knob_rejects_unknown_modes():
    from l3c_pytorch_b200 import engine as E
    with pytest.raises(RuntimeError, match='l3c_set_conv_tile_schedule'):
        with E.conv_tile_schedule(3):
            pass
