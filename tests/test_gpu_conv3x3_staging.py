"""conv_f16_kernel<0> (the FP16 3x3 convolution) stages ONE halo box per 8x16 output tile: (8 + 2d) rows x 24
pixels x 64 channels, read by all nine taps, with the two 64-row MMA halves being the tile's left and right 8-pixel
columns.  The wgmma descriptors of a tap start inside the 128B-swizzle atom (at pixel dx*d of a box row); a wrong
swizzle phase there reads the right bytes in the wrong order, so it shows up as wrong numbers, not as a fault.

Every case checks the default launch against fp32 PyTorch on the same FP16-rounded operands, on shapes whose W is
not a multiple of 16 and H not a multiple of 8 (partial tiles, zero-filled halo on every side), then requires the
same bits under every grid and stage count (lossless decoding: the decoder's grid differs from the encoder's).
plan() restates the host plan of this kernel (one stage = one tile's halo box, one stage per pipe at any budget)
and every case asserts the regime it claims."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_persistent import (ATOL_OP, GRIDS, RESERVE, RTOL_OP, SMEM_MAX, TH, TW, W_TAP, Plan, _cached,
                                       _ceil, _check_operand_image, _conv_module, _h, _n_sm, _nchw, _nhwc,
                                       _same_bits_in_every_regime, _tdiv, check_regime, smem_cap)

gpu = pytest.mark.gpu


def halo_w(d):
    """width of the halo box: TW + 2d rounded up to whole 8-pixel groups (24 for d = 1..4)"""
    return (TW + 2 * d + 7) // 8 * 8


def plan(n_sm, shape, cout=64, dilation=1, conv_smem_kb=0):
    """conv2d_f16's launch of conv_f16_kernel<0>: plan_ring(conv_smem_cap(), 72 KB + reserve, box bytes, 1) and
    grid_3x3; one ring slot per tile"""
    N, H, W = shape
    cout_pad = _ceil(cout, 64) * 64
    ptiles = N * _ceil(W, TW) * _ceil(H, TH)
    grid = min(max(n_sm // (cout_pad // 64), 1), ptiles)
    a_bytes = (TH + 2 * dilation) * halo_w(dilation) * 128
    fixed = 9 * W_TAP + RESERVE
    n = min(_tdiv(smem_cap(conv_smem_kb) - fixed, 2 * a_bytes), 1)
    if n < 1 and fixed + 2 * a_bytes <= SMEM_MAX:
        n = 1
    return Plan('conv3x3_f16', grid, 2, n, ptiles, 1)


SHAPE = (3, 37, 37)                       # 3 images of 3 x 5 tiles (W % 16 = 5, H % 8 = 5); 45 tiles
BUDGETS = [(2, 112), (2, 227)]            # 112 KB: below one stage per pipe (placed above the budget); 227 KB
REGIMES = GRIDS + BUDGETS
CASES = [
    ('d1', dict(cout=64, dilation=1), {}),
    ('d1_relu_residual', dict(cout=64, dilation=1), dict(relu=True, residual=True)),
    ('d1_slice', dict(cout=64, dilation=1), dict(slice=True)),
    ('d1_c256_shuffle', dict(cout=256, dilation=1), dict(pixel_shuffle=True)),
    ('d2_relu', dict(cout=64, dilation=2), dict(relu=True)),
    ('d2_round', dict(cout=64, dilation=2), dict(round_only=True)),
    ('d2_c256_shuffle_round', dict(cout=256, dilation=2), dict(pixel_shuffle=True, round_only=True)),
    ('d4_residual', dict(cout=64, dilation=4), dict(residual=True)),
    ('d4_slice', dict(cout=64, dilation=4), dict(slice=True)),
    ('d4_c256_shuffle_relu', dict(cout=256, dilation=4), dict(pixel_shuffle=True, relu=True)),
]


def test_staging_plans_cover_both_pipes_and_every_stage_count():
    """Host-side model only (no GPU): on 1-3 SMs every pipe of every CTA runs >= 2 tiles and its ring wraps >= 3
    times, on 7 SMs the pipes are uneven, and at any budget in [112, 227] KB the host code gives these layers
    one stage per pipe."""
    covered = set()
    for _, kw, _ in CASES:
        for m, kb in [(0, 0)] + REGIMES:
            p = plan(m or 132, SHAPE, conv_smem_kb=kb, **kw)
            check_regime(p, m)
            covered.add(p.n_stages)
    possible = set(plan(132, SHAPE, conv_smem_kb=kb, **kw).n_stages for _, kw, _ in CASES for kb in range(112, 228))
    assert covered == possible == {1}, (covered, possible)


@gpu
@pytest.mark.parametrize('case_id,kw,epi', CASES, ids=[c[0] for c in CASES])
def test_f16_3x3_halo_box_every_grid_and_stage_count(case_id, kw, epi):
    """conv_f16_kernel<0> at d = 1, 2, 4: fp32 PyTorch on FP16-rounded operands; same bits for 1, 2, 3, 7 SMs and
    the smallest and largest shared-memory budgets"""
    from l3c_pytorch_b200 import engine as E, _lib
    cout, rate = kw['cout'], kw['dilation']
    N, H, W = SHAPE
    conv = _conv_module(64, cout, 3, 1, rate, seed=3 * cout + rate)
    g = torch.Generator().manual_seed(13 * cout + rate)
    x = torch.randn(N, 64, H, W, generator=g)
    r = torch.randn(N, cout, H, W, generator=g) if epi.get('residual') else None
    relu, ps = bool(epi.get('relu')), bool(epi.get('pixel_shuffle'))

    def reference():
        y = F.conv2d(_h(x), _h(conv.weight.detach()), conv.bias.detach(), padding=rate, dilation=rate)
        if relu:
            y = F.relu(y)
        if r is not None:
            y = y + r
        return F.pixel_shuffle(y, 2) if ps else y
    want = _cached(('conv3x3_f16_halo', case_id), reference)

    cc = conv.cuda()
    xf = _nhwc(x)
    xa = E.Act(xf, xf.clamp(-65504.0, 65504.0).half())
    C = cout // 4 if ps else cout
    conv_kw = dict(relu=relu, pixel_shuffle=ps, residual=_nhwc(r) if r is not None else None,
                   precision=_lib.PREC_F16)
    Ho, Wo = (2 * H, 2 * W) if ps else (H, W)

    def run():
        if epi.get('slice'):
            # channel slices of wider sentinel-filled buffers (the atrous concat): neighbours untouched
            buf_r = torch.full((N, Ho, Wo, 3 * C), 7.0, dtype=torch.float16, device='cuda')
            E.conv2d(cc, xa, want='round', out=buf_r, out_coff=C, **conv_kw)
            buf_f = torch.full((N, Ho, Wo, 3 * C), 7.0, device='cuda')
            E.conv2d(cc, xa, want='plain', out=buf_f, out_coff=C, **conv_kw)
            return {'slice_round': buf_r, 'slice_fp32': buf_f}
        if epi.get('round_only'):
            return {'round': E.conv2d(cc, xa, want='round', **conv_kw).r}
        a = E.conv2d(cc, xa, want='act', **conv_kw)
        return {'fp32': a.f, 'operand': a.r}

    base = run()
    ref_act = E.conv2d(cc, xa, want='act', **conv_kw) if 'fp32' not in base else None
    torch.cuda.synchronize()
    f, op = (base['fp32'], base['operand']) if ref_act is None else (ref_act.f, ref_act.r)
    assert f.shape == (N, Ho, Wo, C)
    np.testing.assert_allclose(_nchw(f).numpy(), want.numpy(), rtol=RTOL_OP, atol=ATOL_OP, err_msg=case_id)
    _check_operand_image('f16', f, op)
    if epi.get('slice'):
        assert torch.equal(base['slice_round'][..., C:2 * C], op) and torch.equal(base['slice_fp32'][..., C:2 * C], f)
        for b in (base['slice_round'], base['slice_fp32']):
            assert bool((b[..., :C] == 7).all()) and bool((b[..., 2 * C:] == 7).all()), case_id
    elif epi.get('round_only'):
        assert torch.equal(base['round'], op), case_id

    def plan_of(m, kb):
        return plan(_n_sm(m), SHAPE, cout=cout, dilation=rate, conv_smem_kb=kb)
    for m, kb in REGIMES:
        check_regime(plan_of(m, kb), m)
    assert [plan_of(m, kb).n_stages for m, kb in BUDGETS] == [1, 1]
    _same_bits_in_every_regime('conv3x3_f16', run, base, REGIMES, plan_of)
