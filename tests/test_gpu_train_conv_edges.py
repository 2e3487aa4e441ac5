"""Edges of the training step's 3x3 / 64-input-channel convolutions (train.FUSED_CONV, DESIGN §4.11) that the
per-layer cases of tests/test_gpu_train_convs.py do not reach, against the same float64 references and budgets:

  A. weight-gradient chunk plans with a short last chunk, chunks across images and >= 3 tiles per chunk;
  B. planes smaller than the dilation (1x1 .. 3x3);
  C. the persistent kernel's other launch conditions (SM caps, stage budget, tile schedules): the same bits;
  D. memory layouts of x and dy (channels_last, channel slices, zero strides, views off a 16-byte boundary);
  E. autograd forms (a layer used twice, frozen inputs or parameters, no_grad, a side stream, double backward) and
     the weight-image cache after optimiser steps;
  F. the TF32 rounding kernel against the host rounding the references use, special values included;
  G. one whole step at a size where every scale has partial tiles, against the cuDNN path.

wgrad_plan() restates the chunk plan of conv_train.cu (wg::plan), so the cases can assert the plan properties they
claim.  The plan, its workspace and the host rounding need no device and run everywhere."""
import math
import struct
from collections import namedtuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import test_gpu_train_convs as tc
from tests import util
from tests.test_gpu_persistent import check_regime, _n_sm, plan as conv_plan

gpu = pytest.mark.gpu
DEV = 'cuda'
LAYERS = [(64, 1), (64, 2), (64, 4), (256, 1)]


# ---------------------------------------------------------------------------------------------
# the weight gradient's chunk plan (conv_train.cu: wg::plan), restated
# ---------------------------------------------------------------------------------------------
WgPlan = namedtuple('WgPlan', 'n_tiles tiles_per_chunk n_chunks last')


def wgrad_plan(N, H, W, cout):
    """8x16-pixel tiles in (image, tile row, tile column) order, split into chunks of tiles_per_chunk tiles, one chunk
    per CTA, about 132 CTAs over the Cout / 64 tiles; last = tiles in the last chunk"""
    n_tiles = N * math.ceil(H / 8) * math.ceil(W / 16)
    tpc = math.ceil(n_tiles / max(1, 132 // (cout // 64)))
    n_chunks = math.ceil(n_tiles / tpc)
    return WgPlan(n_tiles, tpc, n_chunks, n_tiles - (n_chunks - 1) * tpc)


def plan_properties(N, H, W, cout):
    """(short last chunk, a chunk spans two images with partial right and bottom tiles in every image,
    tiles_per_chunk >= 3)"""
    p = wgrad_plan(N, H, W, cout)
    per_image = math.ceil(H / 8) * math.ceil(W / 16)
    spans = any(c * p.tiles_per_chunk // per_image != (min((c + 1) * p.tiles_per_chunk, p.n_tiles) - 1) // per_image
                for c in range(p.n_chunks))
    return p.last < p.tiles_per_chunk, spans and H % 8 != 0 and W % 16 != 0, p.tiles_per_chunk >= 3


def chunk_tiles(N, H, W, cout, chunk):
    """[N, 1, H, W] float64 mask of the output pixels in the tiles of `chunk`"""
    p = wgrad_plan(N, H, W, cout)
    tx, ty = math.ceil(W / 16), math.ceil(H / 8)
    m = torch.zeros(N, 1, H, W, dtype=torch.float64)
    for t in range(chunk * p.tiles_per_chunk, min((chunk + 1) * p.tiles_per_chunk, p.n_tiles)):
        n, r = divmod(t, tx * ty)
        y, x = divmod(r, tx)
        m[n, 0, 8 * y:8 * y + 8, 16 * x:16 * x + 16] = 1
    return m


# ragged shapes per Cout (the plan does not depend on the dilation): 7 x 53 x 45 is 147 tiles in 74 chunks of 2;
# 7 x 61 x 75 is 280 tiles in 94 chunks of 3; 5 x 56 x 16 (Cout 256) is 35 tiles in 18 chunks of 2; 5 x 53 x 29
# (Cout 256) is 70 tiles in 24 chunks of 3.  Each leaves 1 tile in the last chunk.
RAGGED = {64: [(7, 53, 45), (7, 61, 75)], 256: [(5, 56, 16), (5, 53, 29)]}
RAGGED_CASES = [(cout, d) + s for (cout, d) in LAYERS for s in RAGGED[cout]]


def test_wgrad_plan_matches_the_workspace():
    """the restated plan sizes the workspace as l3c_conv3x3_wgrad_workspace does: n_chunks x Cout x (9 x 64 + 1)
    floats"""
    from l3c_pytorch_b200._lib import lib
    shapes = [(N, H, W) for N in (1, 2, 3, 5, 7, 9, 30, 257) for H in (1, 2, 7, 8, 9, 36, 53, 61, 128)
              for W in (1, 3, 15, 16, 17, 44, 45, 75, 128)] + [(65535, 1, 1), (65535, 64, 64), (1, 32768, 32768)]
    for cout in (64, 256):
        for N, H, W in shapes:
            want = wgrad_plan(N, H, W, cout).n_chunks * cout * (9 * 64 + 1) * 4
            assert lib.l3c_conv3x3_wgrad_workspace(N, H, W, cout) == want, (N, H, W, cout)


def test_ragged_cases_cover_every_plan_property():
    print('\n cout  d   N    H    W  tiles  per chunk  chunks  last  short  spans+partial  >=3')
    for cout, d in LAYERS:
        cases = [c[2:] for c in RAGGED_CASES if c[:2] == (cout, d)]
        props = [plan_properties(*s, cout) for s in cases]
        for s, pr in zip(cases, props):
            print('%5d %2d %3d %4d %4d %6d %10d %7d %5d  %5s  %13s  %3s' % ((cout, d) + s + wgrad_plan(*s, cout) + pr))
        for i, name in enumerate(('a short last chunk', 'a chunk across images with partial tiles',
                                  '>= 3 tiles per chunk')):
            assert any(pr[i] for pr in props), (cout, d, name)
    assert wgrad_plan(7, 53, 45, 64) == (147, 2, 74, 1)
    assert wgrad_plan(5, 56, 16, 256) == (35, 2, 18, 1)
    # the step of G: scale 1 of 9 x 72 x 88 is 36 x 44, 135 tiles in 68 chunks of 2
    assert wgrad_plan(9, 36, 44, 64) == (135, 2, 68, 1)


def _check_against_float64(cout, d, N, H, W, seed, limit=None):
    """y, dx, dW and db of one layer against float64 under the budgets B of test_gpu_train_convs: max |err| / B at
    most limit[k] (default 0.5, as there); -> the references"""
    conv = tc._layer(cout, d, seed=seed)
    x, gy = tc._inputs(cout, N, H, W, seed=seed + N * H + W)
    got = dict(zip(('y', 'dx', 'dw', 'db'), tc.run_layer(conv, x, gy)))
    ref, x64, dy64, w64 = tc.references(conv, x, gy)
    r = {k: tc.ratio(got[k], *ref[k]) for k in ref}
    print('cout %d d %d %dx%dx%d  max |err| / B: %s' % (cout, d, N, H, W, ' '.join('%s %.3g' % kv for kv in r.items())))
    for k, v in r.items():
        assert v <= (limit or {}).get(k, 0.5), ((cout, d, N, H, W), k, r)
    return conv, x64, dy64, w64, ref


@gpu
@pytest.mark.parametrize('cout,d,N,H,W', RAGGED_CASES)
def test_ragged_chunk_plans_against_float64(cout, d, N, H, W):
    """A: every tile of a short last chunk is counted once: a float64 dW without the last chunk's pixels, or with
    them twice, is over the budget"""
    _, x64, dy64, w64, ref = _check_against_float64(cout, d, N, H, W, seed=31 * cout + d)
    p = wgrad_plan(N, H, W, cout)
    assert p.last < p.tiles_per_chunk
    mask = chunk_tiles(N, H, W, cout, p.n_chunks - 1).to(dy64.device)
    assert 0 < int(mask.sum()) < 128 * p.tiles_per_chunk
    dw_last = torch.nn.grad.conv2d_weight(x64, w64.shape, dy64 * mask, padding=d, dilation=d)
    for bad in (ref['dw'][0] - dw_last, ref['dw'][0] + dw_last):
        assert tc.ratio(bad, *ref['dw']) > 1


# ---------------------------------------------------------------------------------------------
# B. planes smaller than the dilation
# ---------------------------------------------------------------------------------------------
TINY = [(64, d, N) for d in (1, 2, 4) for N in (1, 5)] + [(256, 1, 1), (256, 1, 5)]


@gpu
@pytest.mark.parametrize('cout,d,N', TINY)
def test_tiny_planes_against_float64(cout, d, N):
    """H, W in {1, 2, 3} (Cout 64) and 1x1, 1x3 (the 64 -> 256 tail, whose gy is twice as large each way).
    dW and db sum K = N H W <= 45 pixels.  With so few terms the errors do not average out, and the worst case is
    reached: db of K = 3 pixels takes 2 fp32 roundings of up to 2^-24 sum |dy| each, 2/3 of its budget.  So dW and db
    are held to their budget B itself here (y and dx, 9 x 64 products each, to 0.5 B as everywhere)."""
    planes = [(H, W) for H in (1, 2, 3) for W in (1, 2, 3)] if cout == 64 else [(1, 1), (1, 3)]
    for H, W in planes:
        _check_against_float64(cout, d, N, H, W, seed=7 * d + N, limit=dict(dw=1.0, db=1.0))


# ---------------------------------------------------------------------------------------------
# C. launch conditions of the persistent forward / data-gradient kernel
# ---------------------------------------------------------------------------------------------
SHAPE_C = (5, 41, 70)           # 150 tiles of 8 x 16, partial right and bottom tiles: CTAs run tiles of two images
CONDITIONS = [('1 SM', dict(max_sms=1), 0), ('3 SMs', dict(max_sms=3), 0), ('17 SMs', dict(max_sms=17), 0),
              ('112 KB', dict(conv_smem_kb=112), 0), ('static stripe', {}, 1), ('skewed start', {}, 2)]


@gpu
@pytest.mark.parametrize('cout,d', [(64, 1), (64, 4), (256, 1)])
def test_launch_conditions_give_the_same_bits(cout, d):
    """C: y and dx under every SM cap, the 112 KB budget and tile schedules 1 and 2 equal the default launch bit for
    bit (the accumulation order is fixed per tile), and so do dW and db, which read none of these knobs.  The TF32
    kernel sizes its ring from the whole of shared memory, not the budget: two stages at d = 1, one when dilated."""
    from l3c_pytorch_b200 import engine as E
    N, H, W = SHAPE_C
    conv = tc._layer(cout, d, seed=41 + d)
    x, gy = tc._inputs(cout, N, H, W, seed=43)
    base = tc.run_layer(conv, x, gy)
    torch.cuda.synchronize()
    for name, limits, schedule in CONDITIONS:
        m, kb = limits.get('max_sms', 0), limits.get('conv_smem_kb', 0)
        # the forward launch (Cout tiles share the SMs) and the data gradient's (Cout / 64 launches of 64 channels)
        for k_cout in (cout, 64):
            p = conv_plan('conv3x3_tf32', _n_sm(m), SHAPE_C, cout=k_cout, dilation=d, conv_smem_kb=kb)
            check_regime(p, m)
            assert p.n_stages == (2 if d == 1 else 1), p
            if m == 17:
                assert p.uneven(), p
        with E.conv_launch_limits(**limits), E.conv_tile_schedule(schedule):
            got = tc.run_layer(conv, x, gy)
            torch.cuda.synchronize()
        for what, u, v in zip(('y', 'dx', 'dw', 'db'), got, base):
            assert torch.equal(u, v), (name, what, int((u != v).sum()))


# ---------------------------------------------------------------------------------------------
# D. layouts
# ---------------------------------------------------------------------------------------------
def _form(t, kind, requires_grad=False):
    """t [N,C,H,W] -> the same values in layout `kind`, a view of a new leaf (which requires grad if asked)"""
    N, C, H, W = t.shape
    if kind in ('nchw', 'channels_last'):
        base = t.clone(memory_format=torch.channels_last if kind == 'channels_last' else torch.contiguous_format)
        view = lambda b: b
    elif kind in ('slice', 'slice_channels_last'):
        base = torch.randn(N, C + 24, H, W, device=t.device)
        if kind == 'slice_channels_last':
            base = base.contiguous(memory_format=torch.channels_last)
        base[:, 8:8 + C] = t
        view = lambda b: b[:, 8:8 + C]
    else:
        # 'offset' / 'offset_channels_last': a contiguous view one float past a 16-byte boundary
        base = torch.empty(t.numel() + 1, device=t.device)
        if kind == 'offset':
            base[1:] = t.flatten()
            view = lambda b: b[1:].view(N, C, H, W)
        else:
            base[1:] = t.permute(0, 2, 3, 1).flatten()
            view = lambda b: b[1:].view(N, H, W, C).permute(0, 3, 1, 2)
    return view(base.requires_grad_(requires_grad))


LAYOUTS = ['nchw', 'channels_last', 'slice', 'slice_channels_last', 'offset', 'offset_channels_last']


def _conv_grads(conv, x, gy):
    """y = the layer's output (Cout channels, no PixelShuffle) and d(y . gy) / (x, W, b) through train._conv"""
    from l3c_pytorch_b200 import train
    old = train.FUSED_CONV
    train.FUSED_CONV = True
    try:
        y = train._conv(conv, x)
        dx, dw, db = torch.autograd.grad(y, (x, conv.weight, conv.bias), gy)
    finally:
        train.FUSED_CONV = old
    return y.detach(), dx, dw, db


@gpu
@pytest.mark.parametrize('cout', [64, 256])
def test_layouts_give_the_same_bits(cout):
    """D: the same values of x and gy in every layout give the same y, dx, dW and db bits.  A channels_last view off
    a 16-byte boundary is copied (train._nhwc), not refused by the kernels' alignment checks."""
    conv = tc._layer(cout, 2 if cout == 64 else 1, seed=51)
    g = torch.Generator().manual_seed(52)
    N, H, W = 2, 13, 21
    x = torch.randn(N, 64, H, W, generator=g).to(DEV)
    gy = torch.randn(N, cout, H, W, generator=g).to(DEV)
    want = None
    for kind in LAYOUTS:
        xf = _form(x, kind, requires_grad=True)
        gyf = _form(gy, kind)
        assert torch.equal(xf, x) and torch.equal(gyf, gy)
        if kind.startswith('offset'):
            assert xf.data_ptr() % 16 == 4 and gyf.data_ptr() % 16 == 4
        if kind == 'offset_channels_last':
            assert xf.is_contiguous(memory_format=torch.channels_last)
        got = _conv_grads(conv, xf, gyf)
        torch.cuda.synchronize()
        if want is None:
            want = got
            continue
        for what, u, v in zip(('y', 'dx', 'dw', 'db'), got, want):
            assert torch.equal(u, v), (kind, what)


@gpu
@pytest.mark.parametrize('cout', [64, 256])
def test_zero_stride_gradients_give_the_same_bits(cout):
    """D: the expanded gradients of y.sum() (every stride 0) and of a row broadcast equal their contiguous copies"""
    conv = tc._layer(cout, 1, seed=53)
    g = torch.Generator().manual_seed(54)
    N, H, W = 2, 13, 21
    x = torch.randn(N, 64, H, W, generator=g).to(DEV).requires_grad_(True)
    row = torch.randn(N, cout, 1, W, generator=g).to(DEV)
    for gy in (torch.ones((), device=DEV).expand(N, cout, H, W), row.expand(N, cout, H, W)):
        assert 0 in gy.stride()
        a = _conv_grads(conv, x, gy)
        b = _conv_grads(conv, x, gy.contiguous())
        torch.cuda.synchronize()
        for what, u, v in zip(('y', 'dx', 'dw', 'db'), a, b):
            assert torch.equal(u, v), (gy.stride(), what)
    # y.sum().backward() itself
    from l3c_pytorch_b200 import train
    old = train.FUSED_CONV
    train.FUSED_CONV = True
    try:
        conv.zero_grad(set_to_none=True)
        x.grad = None
        train._conv(conv, x).sum().backward()
    finally:
        train.FUSED_CONV = old
    want = _conv_grads(conv, x, torch.ones(N, cout, H, W, device=DEV))
    for what, u, v in zip(('dx', 'dw', 'db'), (x.grad, conv.weight.grad, conv.bias.grad), want[1:]):
        assert torch.equal(u, v), what


# ---------------------------------------------------------------------------------------------
# E. autograd forms
# ---------------------------------------------------------------------------------------------
def _output(conv, x):
    """the layer's output as the step uses it (PixelShuffle(2) after the 64 -> 256 tail), FUSED_CONV on"""
    from l3c_pytorch_b200 import train
    old = train.FUSED_CONV
    train.FUSED_CONV = True
    try:
        y = train._conv(conv, x)
    finally:
        train.FUSED_CONV = old
    return F.pixel_shuffle(y, 2) if conv.out_channels == 256 else y


@gpu
@pytest.mark.parametrize('cout,d', [(64, 2), (256, 1)])
def test_a_layer_used_twice_adds_its_gradients(cout, d):
    """one module on two inputs of different shapes in one graph: .grad is the float64 sum of both calls, within
    the sum of their budgets"""
    conv = tc._layer(cout, d, seed=61)
    shapes = [(2, 19, 23), (1, 8, 40)]
    xs, gys, refs = [], [], []
    for i, (N, H, W) in enumerate(shapes):
        x, gy = tc._inputs(cout, N, H, W, seed=62 + i)
        xs.append(x.clone().requires_grad_(True))
        gys.append(gy)
        refs.append(tc.references(conv, x, gy)[0])
    conv.zero_grad(set_to_none=True)
    loss = sum((_output(conv, x) * gy).sum() for x, gy in zip(xs, gys))
    loss.backward()
    for k, got in (('dw', conv.weight.grad), ('db', conv.bias.grad)):
        r = tc.ratio(got, refs[0][k][0] + refs[1][k][0], refs[0][k][1] + refs[1][k][1])
        assert r <= 0.5, (k, r)
    for x, ref in zip(xs, refs):
        assert tc.ratio(x.grad, *ref['dx']) <= 0.5


def _backward_launches(conv, x, gy):
    """-> (y, backward launch log); the log is reset between the forward and the backward"""
    from l3c_pytorch_b200 import engine as E
    y = _output(conv, x)
    torch.cuda.synchronize()
    E.launch_log(reset=True)
    y.backward(gy)
    torch.cuda.synchronize()
    return y.detach(), E.launch_log(reset=True)[0]


@gpu
@pytest.mark.parametrize('cout', [64, 256])
def test_frozen_inputs_skip_their_launches(cout):
    """x without grad: no data-gradient launch, the same dW and db; weight and bias frozen: no weight-gradient
    launch, the same dx"""
    conv = tc._layer(cout, 1, seed=71)
    x, gy = tc._inputs(cout, 2, 19, 23, seed=72)
    y, dx, dw, db = tc.run_layer(conv, x, gy)
    torch.cuda.synchronize()

    conv.zero_grad(set_to_none=True)
    _, log = _backward_launches(conv, x.clone(), gy)
    assert log.get('conv3x3_tf32_kernel', 0) == 0 and log.get('conv3x3_wgrad_kernel', 0) == 1, log
    assert torch.equal(conv.weight.grad, dw) and torch.equal(conv.bias.grad, db)

    conv.zero_grad(set_to_none=True)
    conv.requires_grad_(False)
    try:
        xr = x.clone().requires_grad_(True)
        _, log = _backward_launches(conv, xr, gy)
    finally:
        conv.requires_grad_(True)
    assert log.get('conv3x3_wgrad_kernel', 0) == 0 and log.get('conv3x3_wgrad_finish_kernel', 0) == 0, log
    assert log.get('conv3x3_tf32_kernel', 0) == cout // 64, log
    assert conv.weight.grad is None and conv.bias.grad is None
    assert torch.equal(xr.grad, dx)


@gpu
def test_no_grad_and_side_stream_give_the_same_bits():
    """a forward under torch.no_grad(), and the whole forward and backward on a side stream, equal the default"""
    conv = tc._layer(256, 1, seed=81)
    x, gy = tc._inputs(256, 3, 21, 37, seed=82)
    base = tc.run_layer(conv, x, gy)
    torch.cuda.synchronize()
    with torch.no_grad():
        y = _output(conv, x)
    assert y.grad_fn is None and torch.equal(y, base[0])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = tc.run_layer(conv, x, gy)
    s.synchronize()
    torch.cuda.synchronize()
    for what, u, v in zip(('y', 'dx', 'dw', 'db'), got, base):
        assert torch.equal(u, v), what


@gpu
def test_double_backward_raises():
    """the kernels' gradients carry no graph: differentiating them again raises instead of silently leaving the
    convolution out.  The loss is quadratic in y, so the gradient reaching the layer is itself differentiable (the
    case @once_differentiable guards), and x * x keeps the first derivative differentiable without the layer."""
    conv = tc._layer(64, 1, seed=91)
    x, _ = tc._inputs(64, 1, 9, 17, seed=92)
    x = x.requires_grad_(True)
    loss = (_output(conv, x) ** 2).sum() + (x * x).sum()
    (g,) = torch.autograd.grad(loss, x, create_graph=True)
    assert g.requires_grad
    with pytest.raises(RuntimeError, match='differentiate twice'):
        g.sum().backward()


@gpu
def test_weight_images_after_optimiser_steps(monkeypatch):
    """three RMSprop steps with FUSED_CONV, then a forward and backward: every in-scope layer's cached TF32 image and
    data-gradient image equal, bit for bit, what a fresh PackedConv builds from the current parameters"""
    from l3c_pytorch_b200 import engine as E, train
    monkeypatch.setattr(train, 'FUSED_CONV', True)
    bp = tc._blueprint()
    opt = train.make_optimizer(bp)
    imgs = torch.stack([util.make_image(i, 32, 32) for i in range(2)]).float().to(DEV)
    before = {n: p.detach().clone() for n, p in bp.net.named_parameters()}
    for _ in range(3):
        train.train_step(bp, opt, imgs)
    bp.net.zero_grad()
    train.training_loss(bp, imgs)[0].backward()
    torch.cuda.synchronize()
    layers = [(n, m) for n, m in bp.net.named_modules()
              if isinstance(m, torch.nn.Conv2d) and train.conv3x3_in_scope(m)]
    assert layers
    for n, m in layers:
        assert not torch.equal(m.weight.detach(), before[n + '.weight']), n
        pc = m.__dict__['_l3c_packed']
        fresh = E.PackedConv(m)
        assert pc.w_tc is not None and torch.equal(pc.w_tc, fresh.get_tc()[0]), n
        assert torch.equal(pc.b, fresh.get_tc()[1]), n
        assert pc.w_dgrad is not None and torch.equal(pc.w_dgrad, fresh.get_dgrad()), n


# ---------------------------------------------------------------------------------------------
# F. TF32 rounding
# ---------------------------------------------------------------------------------------------
def _bits(u):
    return struct.unpack('<f', struct.pack('<I', u & 0xFFFFFFFF))[0]


# +-0, the smallest and largest subnormals, subnormal and normal ties (low 13 bits 0x1000) and their neighbours,
# 1 and 1 + 2^-11 (a tie), FLT_MAX (rounds to inf) and the largest value that does not, +-inf, quiet and signalling
# NaNs with low and high payloads (cvt.rna.tf32.f32 keeps the upper 19 bits of an inf or NaN)
SPECIAL = [0x00000000, 0x80000000, 0x00000001, 0x007FFFFF, 0x80000001, 0x807FFFFF, 0x00001000, 0x80001000,
           0x00000FFF, 0x00003000, 0x00801000, 0x80801000, 0x00800FFF, 0x3F800000, 0x3F801000, 0xBF801000,
           0x3F802FFF, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F7FEFFF, 0x7F800000, 0xFF800000,
           0x7FC00000, 0xFFC00000, 0x7FC00001, 0x7FFFFFFF, 0xFFFFFFFF, 0x7FFFF000, 0xFFFFF000, 0x7FC01000,
           0x7F800001, 0x7F800FFF, 0x7F801000, 0x7F802000, 0xFF800001, 0xFFBFFFFF, 0x7FBFE000, 0x7FA00000]


def tf32_rna(u):
    """TF32 image of the fp32 with bits u, from the value: finite x -> the multiple of its TF32 quantum nearest to x,
    ties away from zero (quantum 2^(e - 10) for 2^e <= |x| < 2^(e + 1), 2^-136 for subnormals), inf where that is
    above FLT_MAX; inf and NaN -> the upper 19 bits"""
    if (u >> 23) & 0xFF == 0xFF:
        return u & 0xFFFFE000
    x = _bits(u)
    if x == 0:
        return u
    m, e = math.frexp(abs(x))                               # |x| = m 2^e, 0.5 <= m < 1
    q = math.ldexp(1.0, max(e - 1, -126) - 10)
    r = math.floor(abs(x) / q + 0.5) * q
    out = np.float32(math.copysign(r, x)) if r < 2.0 ** 128 else np.float32(math.copysign(math.inf, x))
    return int(out.view(np.uint32))


def test_host_rounding_of_special_values():
    """engine.round_to_tf32 (the host rounding every float64 reference uses) against the value-level restatement:
    the special values, then random bit patterns (NaNs and infs among them).  A NaN stays NaN unless all of its
    payload lies in the 13 bits TF32 drops, where the instruction, and so the host, give inf."""
    from l3c_pytorch_b200.engine import round_to_tf32
    g = np.random.default_rng(5)
    rand = g.integers(0, 2 ** 32, 200000, dtype=np.uint64)
    rand[:2000] = (rand[:2000] & 0x807FFFFF) | 0x7F800000                # exponent 0xFF: inf and NaN
    for vals in (SPECIAL, [int(v) for v in rand]):
        a = np.array(vals, dtype=np.uint32)
        got = round_to_tf32(torch.from_numpy(a.view(np.float32).copy())).numpy().view(np.uint32)
        want = np.array([tf32_rna(int(v)) for v in a], dtype=np.uint32)
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, ['%08x -> %08x, want %08x' % (a[i], got[i], want[i]) for i in bad[:8]]
        nan = np.isnan(a.view(np.float32))
        keeps = nan & ((a & 0x007FE000) != 0)
        assert np.isnan(got.view(np.float32)[keeps]).all()
        assert np.isinf(got.view(np.float32)[nan & ~keeps]).all()
    assert tf32_rna(0x7F7FFFFF) == 0x7F800000 and tf32_rna(0x3F801000) == 0x3F802000


@gpu
def test_round_tf32_kernel_matches_the_host():
    """engine.round_tf32 (round_tf32_kernel) against engine.round_to_tf32 bit for bit: n = 0 .. 9 (the tail of
    n % 4 elements), a length past the kernel's grid cap of 4 x SMs blocks of 256 float4s with a tail of 3, and the
    special values"""
    from l3c_pytorch_b200 import engine as E
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    g = np.random.default_rng(6)
    special = np.array(SPECIAL, dtype=np.uint32)
    lengths = list(range(10)) + [3 * (4 * sms * 256 * 4) + 3, len(SPECIAL)]
    for n in lengths:
        a = g.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
        if n == len(SPECIAL):
            a = special
        elif n > 1000:
            a[-len(SPECIAL):] = special                      # the specials in the tail and the last float4s
        x = torch.from_numpy(a.view(np.float32).copy())
        got = E.round_tf32(x.to(DEV)).cpu().numpy().view(np.uint32)
        want = E.round_to_tf32(x).numpy().view(np.uint32)
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, (n, ['%08x -> kernel %08x, host %08x' % (a[i], got[i], want[i]) for i in bad[:8]])
        nan = np.isnan(a.view(np.float32))
        assert np.isnan(got.view(np.float32)[nan & ((a & 0x007FE000) != 0)]).all()


# ---------------------------------------------------------------------------------------------
# G. one step at an odd size
# ---------------------------------------------------------------------------------------------
@gpu
def test_step_at_an_odd_size_matches_the_cudnn_path(monkeypatch):
    """one FUSED_CONV step on cr at 9 x 72 x 88 (partial tiles at every scale; scale 1, 36 x 44, leaves one tile in
    the last weight-gradient chunk) against the cuDNN path at test_gpu_train_convs.STEP_TOL"""
    from l3c_pytorch_b200 import engine as E
    seen = []
    real = E.conv3x3_wgrad

    def recording(conv, x, dy):
        seen.append(tuple(dy.shape))
        return real(conv, x, dy)
    monkeypatch.setattr(E, 'conv3x3_wgrad', recording)
    g = torch.Generator(device=DEV).manual_seed(0)
    imgs = (torch.rand(9, 3, 72, 88, device=DEV, generator=g) * 255).round()
    out = {f: tc._step(tc._blueprint(), imgs, f) for f in (False, True)}
    assert (9, 36, 44, 64) in seen, seen
    for N, H, W, cout in seen:
        assert H % 8 or W % 16, (N, H, W)
    p = wgrad_plan(9, 36, 44, 64)
    assert p.tiles_per_chunk == 2 and p.last == 1, p
    (l0, b0, g0, p0), (l1, b1, g1, p1) = out[False], out[True]
    tol = tc.STEP_TOL
    dev = dict(loss=abs(l1 - l0) / l0, bpsp=max(abs(u - v) / abs(v) for u, v in zip(b1, b0)),
               grad=max(float((g1[k].norm() - g0[k].norm()).abs() / (g0[k].norm() + 1e-7)) for k in g0))
    print('9 x 72 x 88: fused vs cuDNN relative deviation %s; weight-gradient shapes %s' % (dev, sorted(set(seen))))
    assert g0.keys() == g1.keys()
    assert dev['loss'] < tol['loss'] and dev['bpsp'] < tol['bpsp'] and dev['grad'] < tol['grad'], dev
    for k in p0:
        same = ((g1[k].sign() == g0[k].sign()) & (g0[k].abs() > 1e-5) & (g1[k].abs() > 1e-5) if k in g0
                else torch.ones_like(p0[k], dtype=torch.bool))
        np.testing.assert_allclose(p1[k][same].cpu().numpy(), p0[k][same].cpu().numpy(), rtol=tol['param_rtol'],
                                   atol=tol['param_atol'], err_msg=k)
