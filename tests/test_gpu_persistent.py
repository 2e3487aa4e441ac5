"""The persistent tensor-core kernels in the regimes production runs them in.

Each CTA of conv_f16_kernel<0> (3x3), conv_f16_kernel<1> (5x5/s2), conv3x3_tf32_kernel, conv3x3_f16x2_kernel,
conv1x1_tc_kernel and lin_dmll_f16_kernel has two pipes -- a TMA producer warp feeding a consumer warpgroup -- that
take alternate tiles of the CTA's sequence and cycle a ring of 1 to 4 shared-memory stages.  At production sizes
every pipe handles tens of tiles, and a decode runs the same layers on fewer SMs than the encode.  Small unit-test
inputs give every CTA one tile.  engine.conv_launch_limits brings the production regime to small inputs: a few SMs
-> many tiles per pipe and rings that wrap across tiles; a smaller shared-memory budget -> fewer stages.

Every case checks the default launch against a plain high-precision CPU reference of the same operation, then
requires the SAME BITS in every output tensor under every other grid and stage count: lossless decoding needs the
decoder's results to equal the encoder's whatever grid each ran with.  plan() restates the host code's choice of
grid, pipes and stages, and every case asserts the regime it claims (every pipe >= 2 tiles, rings wrapped, the
stage count), so that a change of the launch heuristics cannot quietly turn these tests trivial."""
import os
from collections import namedtuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

gpu = pytest.mark.gpu
RTOL, ATOL = 2e-5, 2e-5            # f16x2 against float64 (test_gpu_conv.py)
RTOL_OP, ATOL_OP = 1e-4, 1e-4      # f16 / tf32 against fp32 on the same rounded operands

# ---------------------------------------------------------------------------------------------
# launch plans: the host code (plan_ring, grid_3x3, grid_1x1 in tc_conv.cuh and their callers) restated
# (test infrastructure)
# ---------------------------------------------------------------------------------------------
SMEM_MAX = 227 * 1024
RESERVE = 1024 + 512               # alignment slack + barriers, reserved by every launcher
TH, TW = 8, 16                     # output tile of the 3x3 / 5x5 kernels
W_TAP = 64 * 128                   # one 64 x 64 FP16 weight tap


def _tdiv(a, b):
    """C integer division (truncates toward zero)"""
    return abs(a) // b * (1 if a >= 0 else -1)


def _ceil(a, b):
    return -(-a // b)


def smem_cap(conv_smem_kb=0):
    """conv_smem_cap(): the knob, else L3C_CONV_SMEM_KB, else 227 KB; clamped to [112, 227] KB"""
    kb = conv_smem_kb if conv_smem_kb > 0 else int(os.environ.get('L3C_CONV_SMEM_KB', '227'))
    return min(max(kb, 112), 227) * 1024


class Plan(namedtuple('Plan', 'kernel grid n_pipes n_stages tiles units')):
    """grid: CTAs per Cout tile (gridDim.x); tiles: the tile sequence the CTAs of one Cout tile share;
    units: ring slots one tile takes"""

    def pipe_tiles(self, k):
        """tiles pipe k of each CTA runs: t = blockIdx.x + k * gridDim.x; t += n_pipes * gridDim.x"""
        step = self.n_pipes * self.grid
        return [max(0, _ceil(self.tiles - (b + k * self.grid), step)) for b in range(self.grid)]

    def counts(self):
        return [n for k in range(self.n_pipes) for n in self.pipe_tiles(k)]

    def min_tiles(self):
        """fewest tiles any pipe of any CTA runs"""
        return min(self.counts())

    def wraps(self):
        """most times a ring comes back to stage 0 (stage and phase carried from tile to tile)"""
        return max(n * self.units // self.n_stages for n in self.counts())

    def uneven(self):
        return max(self.counts()) > min(self.counts())


def plan(kernel, n_sm, shape, cin=64, cout=64, dilation=1, conv_smem_kb=0):
    """Launch configuration the host code picks.  shape = (N, H, W) of the input; n_sm = stream_sm_count()."""
    N, H, W = shape
    cap = smem_cap(conv_smem_kb)
    cout_pad = _ceil(cout, 64) * 64
    if kernel in ('conv3x3_f16', 'conv5x5s2_f16', 'conv3x3_tf32', 'conv3x3_f16x2'):
        if kernel == 'conv5x5s2_f16':
            H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1          # the tiles cover the output
        ptiles = N * _ceil(W, TW) * _ceil(H, TH)
        grid = min(max(n_sm // (cout_pad // 64), 1), ptiles)
        a_bytes = (TH + 2 * dilation) * TW * 128
        if kernel == 'conv3x3_f16':
            w_res = 9 * W_TAP
            n = min(_tdiv(cap - RESERVE - w_res, 2 * a_bytes), 3)
            if n < 1 and 2 * a_bytes <= SMEM_MAX - RESERVE - w_res:
                n = 1
            return Plan(kernel, grid, 2, n, ptiles, 3)
        if kernel == 'conv5x5s2_f16':
            return Plan(kernel, grid, 2, 2 if (cap - RESERVE) // (2 * (10 * TW * 128 + 3 * W_TAP)) >= 2 else 1,
                        ptiles, 10)
        room = SMEM_MAX - RESERVE - 2 * 9 * W_TAP             # 144 KB of weights: two K halves / two planes
        if kernel == 'conv3x3_tf32':
            return Plan(kernel, grid, 1 if 2 * a_bytes > room else 2, 1 if 4 * a_bytes > room else 2, ptiles, 6)
        return Plan(kernel, grid, 2 if 4 * a_bytes <= room else 1, 1, ptiles, 3)
    M = N * H * W
    if kernel in ('conv1x1_tf32', 'conv1x1_f16', 'conv1x1_f16x2'):
        kind = ('conv1x1_tf32', 'conv1x1_f16', 'conv1x1_f16x2').index(kernel)
        planes = 2 if kind == 2 else 1
        kunits = cin // 32 if kind == 0 else cin // 64
        w_plane = kunits * cout_pad * 128
        sb = planes * 64 * 128
        n = _tdiv((cap if kind == 1 else SMEM_MAX) - RESERVE - planes * w_plane, 2 * sb)
        if n < 1 and planes * w_plane + 2 * sb <= SMEM_MAX - RESERVE:
            n = 1
        nblk = cout_pad // 64
        nb = (2 if nblk % 2 == 0 else 1) if kind == 2 else nblk
        n_tiles = _ceil(M, 64) * (nblk // nb)                # f16x2: Cout chunks of a pixel tile are tiles
        return Plan(kernel, min(_ceil(n_tiles, 2), n_sm), 2, min(n, 4), n_tiles, kunits)
    if kernel in ('lin_dmll_rgb', 'lin_dmll_c5'):
        npad = 128 if kernel == 'lin_dmll_rgb' else 192
        kchunks = cin // 64
        w_bytes = kchunks * npad * 128
        stg = 2 * 64 * (npad + 1) * 4 + 64
        n = _tdiv(cap - RESERVE - w_bytes - stg, 2 * 64 * 128)
        if n < 1 and w_bytes + stg + 2 * 64 * 128 <= SMEM_MAX - RESERVE:
            n = 1
        n_tiles = _ceil(M, 64)
        return Plan(kernel, min(_ceil(n_tiles, 2), n_sm), 2, min(n, 4), n_tiles, kchunks)
    raise ValueError(kernel)


# ---------------------------------------------------------------------------------------------
# regimes: (max_sms, conv_smem_kb); every one must reproduce the default launch bit for bit
# ---------------------------------------------------------------------------------------------
GRIDS = [(1, 0), (2, 0), (3, 0), (7, 0)]          # odd counts leave CTAs and pipes uneven
BUDGETS = [(2, 112), (2, 160), (2, 227)]          # f16 3x3, d = 1: 1, 2 and 3 stages
ANY_SM = 132                                      # the default grid is never asserted on


def check_regime(p, max_sms):
    """the regime a case claims: with 1-3 SMs every pipe of every CTA runs >= 2 tiles and a ring wraps >= 3
    times; with 7 SMs the pipes get different tile counts"""
    if max_sms in (1, 2, 3):
        assert p.min_tiles() >= 2 and p.wraps() >= 3, p
    elif max_sms == 7:
        assert p.uneven(), p


# cases per kernel: (id, plan() arguments, epilogue)
SHAPE = (3, 21, 37)          # 3 images of 3 x 3 tiles (W % 16 = 5, H % 8 = 5): a pipe's tiles cross images
CASES_F16_3X3 = [
    ('d1', dict(cout=64, dilation=1), {}),
    ('d2_relu', dict(cout=64, dilation=2), dict(relu=True)),
    ('d4_residual', dict(cout=64, dilation=4), dict(residual=True)),
    ('d1_slice', dict(cout=64, dilation=1), dict(slice=True)),
    ('d1_round', dict(cout=64, dilation=1), dict(round_only=True)),
    ('c128_relu', dict(cout=128, dilation=1), dict(relu=True)),
    ('c256_shuffle', dict(cout=256, dilation=1), dict(pixel_shuffle=True)),
]
SHAPE_5X5 = (3, 45, 67)      # odd: 23 x 34 outputs, 3 x 3 tiles per image
CASES_5X5 = [('bias', {}), ('relu', dict(relu=True))]
CASES_TF32 = [('d1', dict(cout=64, dilation=1), {}), ('d2_relu', dict(cout=64, dilation=2), dict(relu=True)),
              ('d4', dict(cout=64, dilation=4), {}), ('c128_residual', dict(cout=128, dilation=1), dict(residual=True))]
CASES_F16X2 = [('d1', dict(cout=64, dilation=1), {}), ('d1_c128_residual', dict(cout=128, dilation=1), dict(residual=True)),
               ('d2', dict(cout=64, dilation=2), {}), ('d4_relu', dict(cout=64, dilation=4), dict(relu=True))]
# 1x1: (precision, Cin, Cout, extra budgets); M = 3 * 21 * 37 = 2331 pixels = 36 tiles of 64 + 27
CASES_1X1 = [
    ('f16', 192, 120, [(2, 112)]),                         # 4 stages, 3 at 112 KB
    ('f16', 192, 256, [(2, 112), (2, 130), (2, 150)]),     # 1, 2, 3 stages; 4 by default
    ('tf32', 192, 120, []),                                # 4 stages
    ('tf32', 192, 256, []),                                # 2 stages (the budget does not apply to tf32 / f16x2)
    ('f16x2', 192, 120, []),                               # 4 stages
    ('f16x2', 128, 256, []),                               # 3 stages; two Cout chunks per pixel tile
    ('f16x2', 192, 192, []),                               # 2 stages; three Cout chunks
    ('f16x2', 192, 256, []),                               # 1 stage
]
CASES_DMLL = [('rgb', True, 3, 256, 0, 255, [(2, 112), (2, 160), (2, 170)]),     # 1, 2, 3 stages; 4 by default
              ('c5', False, 5, 25, -1, 1, [(2, 112), (2, 208)])]                 # 1, 2 stages; 3 by default


def _plans():
    """(kernel, plan, max_sms) of every regime of every case"""
    out = []

    def add(kernel, regimes, **kw):
        for m, kb in [(0, 0)] + regimes:
            out.append((kernel, plan(kernel, m or ANY_SM, conv_smem_kb=kb, **kw), m))
    for _, kw, _ in CASES_F16_3X3:
        add('conv3x3_f16', GRIDS + BUDGETS, shape=SHAPE, **kw)
    for _ in CASES_5X5:
        add('conv5x5s2_f16', GRIDS + BUDGETS, shape=SHAPE_5X5)
    for _, kw, _ in CASES_TF32:
        add('conv3x3_tf32', GRIDS, shape=SHAPE, **kw)
    for _, kw, _ in CASES_F16X2:
        add('conv3x3_f16x2', GRIDS, shape=SHAPE, **kw)
    for prec, cin, cout, extra in CASES_1X1:
        add('conv1x1_' + prec, GRIDS + extra, shape=SHAPE, cin=cin, cout=cout)
    for name, _, _, _, _, _, extra in CASES_DMLL:
        add('lin_dmll_' + name, GRIDS + extra, shape=SHAPE, cin=192)
    return out


def test_launch_plans_cover_both_pipes_and_every_stage_count():
    """Host-side model only (no GPU): over all cases, every kernel runs each of its pipes with >= 2 tiles on every
    CTA, and every stage count the host code can pick for the tested layers (any budget in [112, 227] KB) occurs."""
    plans = _plans()
    for kernel, p, m in plans:
        check_regime(p, m)
    kernels = sorted(set(k for k, _, _ in plans))
    assert len(kernels) == 9, kernels
    for kernel in kernels:
        ps = [p for k, p, m in plans if k == kernel and m in (1, 2, 3)]
        for n_pipes in set(p.n_pipes for k, p, _ in plans if k == kernel):
            assert any(p.n_pipes == n_pipes and p.min_tiles() >= 2 for p in ps), (kernel, n_pipes)
        covered = set(p.n_stages for k, p, _ in plans if k == kernel)
        possible = set(plan(kernel, ANY_SM, shape, conv_smem_kb=kb, **kw).n_stages
                       for shape, kw in _layers(kernel) for kb in range(112, 228))
        assert covered == possible, (kernel, covered, possible)
    # the dilated f16x2 layers run one pipe, the others two
    assert set(p.n_pipes for k, p, _ in plans if k == 'conv3x3_f16x2') == {1, 2}


def _layers(kernel):
    """(shape, plan kwargs) of the layers the cases run on `kernel`"""
    if kernel == 'conv3x3_f16':
        return [(SHAPE, kw) for _, kw, _ in CASES_F16_3X3]
    if kernel == 'conv5x5s2_f16':
        return [(SHAPE_5X5, {})]
    if kernel == 'conv3x3_tf32':
        return [(SHAPE, kw) for _, kw, _ in CASES_TF32]
    if kernel == 'conv3x3_f16x2':
        return [(SHAPE, kw) for _, kw, _ in CASES_F16X2]
    if kernel.startswith('conv1x1_'):
        return [(SHAPE, dict(cin=cin, cout=cout)) for prec, cin, cout, _ in CASES_1X1 if kernel == 'conv1x1_' + prec]
    return [(SHAPE, dict(cin=192))]


# ---------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------
_REF = {}          # CPU references, per case


def _cached(key, fn):
    if key not in _REF:
        _REF[key] = fn()
    return _REF[key]


def _device_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _n_sm(max_sms):
    """what stream_sm_count() returns on an ordinary stream"""
    return min(max_sms, _device_sms()) if max_sms > 0 else _device_sms()


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous().cuda()


def _nchw(y):
    return y.cpu().permute(0, 3, 1, 2)


def _h(x):
    """fp32 -> the FP16 operand image's value (RN, saturating), as fp32"""
    return x.clamp(-65504.0, 65504.0).half().float()


def _conv_module(cin, cout, k, stride=1, rate=1, seed=0):
    from l3c_pytorch_b200.network import default_conv
    torch.manual_seed(seed)
    return default_conv(cin, cout, k, rate=rate, stride=stride)


def _same_bits_in_every_regime(kernel, run, base, regimes, plan_of):
    """run() -> {name: tensor}; each regime's outputs must equal `base` bit for bit"""
    from l3c_pytorch_b200 import engine as E
    for m, kb in regimes:
        p = plan_of(m, kb)
        with E.conv_launch_limits(max_sms=m, conv_smem_kb=kb):
            got = run()
        torch.cuda.synchronize()
        for name, want in base.items():
            assert torch.equal(got[name], want), \
                '%s: %s differs from the default launch under max_sms=%d conv_smem_kb=%d (%s): %d elements' % (
                    kernel, name, m, kb, p, int((got[name] != want).sum()))


# ---------------------------------------------------------------------------------------------
# 3x3 (any dilation) and 5x5/s2 kernels
# ---------------------------------------------------------------------------------------------
def _conv3x3_case(prec_name, case_id, kw, epi, shape=SHAPE, regimes=None):
    """one 3x3 layer in precision `prec_name` (f16 / tf32 / f16x2): default launch vs the CPU reference, then the
    same bits in every regime.  epi: relu / residual / pixel_shuffle / slice / round_only."""
    from l3c_pytorch_b200 import engine as E, _lib
    kernel = {'f16': 'conv3x3_f16', 'tf32': 'conv3x3_tf32', 'f16x2': 'conv3x3_f16x2'}[prec_name]
    P = {'f16': _lib.PREC_F16, 'tf32': _lib.PREC_TF32, 'f16x2': _lib.PREC_F16X2}[prec_name]
    cout, rate = kw['cout'], kw['dilation']
    N, H, W = shape
    conv = _conv_module(64, cout, 3, 1, rate, seed=cout + rate)
    g = torch.Generator().manual_seed(11 * cout + rate)
    x = torch.randn(N, 64, H, W, generator=g)
    r = torch.randn(N, cout, H, W, generator=g) if epi.get('residual') else None
    relu, ps = bool(epi.get('relu')), bool(epi.get('pixel_shuffle'))

    def reference():
        w, b = conv.weight.detach(), conv.bias.detach()
        if prec_name == 'f16':
            y = F.conv2d(_h(x), _h(w), b, padding=rate, dilation=rate)
        elif prec_name == 'tf32':
            y = F.conv2d(E.round_to_tf32(x), E.round_to_tf32(w), b, padding=rate, dilation=rate)
        else:
            y = F.conv2d(x.double(), w.double(), b.double(), padding=rate, dilation=rate)
        if relu:
            y = F.relu(y)
        if r is not None:
            y = y + r.to(y.dtype)
        if ps:
            y = F.pixel_shuffle(y, 2)
        return y.float()
    want = _cached((kernel, case_id, shape), reference)

    cc = conv.cuda()
    xf = _nhwc(x)
    xa = {'f16': lambda: E.Act(xf, xf.clamp(-65504.0, 65504.0).half()),
          'tf32': lambda: E.Act(xf, E.round_to_tf32(xf)),
          'f16x2': lambda: E.Act(xf, E.split_f16x2(xf))}[prec_name]()
    res = _nhwc(r) if r is not None else None
    C = cout // 4 if ps else cout
    conv_kw = dict(relu=relu, pixel_shuffle=ps, residual=res, precision=P)

    def run():
        out = {}
        if epi.get('slice'):
            # channel-slice outputs into wider sentinel-filled buffers (the atrous concat): neighbours untouched
            width = (2 if prec_name == 'f16x2' else 1) * 3 * C
            buf_r = torch.full((N, H, W, width), 7.0, dtype=torch.float16 if prec_name != 'tf32' else torch.float32,
                               device='cuda')
            E.conv2d(cc, xa, want='round', out=buf_r, out_coff=C, **conv_kw)
            buf_f = torch.full((N, H, W, 3 * C), 7.0, device='cuda')
            E.conv2d(cc, xa, want='plain', out=buf_f, out_coff=C, **conv_kw)
            out['slice_round'], out['slice_fp32'] = buf_r, buf_f
        elif epi.get('round_only'):
            out['round'] = E.conv2d(cc, xa, want='round', **conv_kw).r
        else:
            a = E.conv2d(cc, xa, want='act', **conv_kw)
            out['fp32'], out['operand'] = a.f, a.r
        return out

    base = run()
    torch.cuda.synchronize()
    tol = (RTOL, ATOL) if prec_name == 'f16x2' else (RTOL_OP, ATOL_OP)
    if 'fp32' in base:
        got = _nchw(base['fp32'])
        assert got.shape == want.shape
        np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=tol[0], atol=tol[1], err_msg=kernel)
        _check_operand_image(prec_name, base['fp32'], base['operand'])
    else:
        # slice / image-only outputs: equal to the matching part of want='act', which is held to the reference
        ref_act = E.conv2d(cc, xa, want='act', **conv_kw)
        torch.cuda.synchronize()
        np.testing.assert_allclose(_nchw(ref_act.f).numpy(), want.numpy(), rtol=tol[0], atol=tol[1], err_msg=kernel)
        _check_operand_image(prec_name, ref_act.f, ref_act.r)
        if epi.get('slice'):
            wide = 2 if prec_name == 'f16x2' else 1
            b = base['slice_round']
            if wide == 2:
                assert torch.equal(b[..., C:2 * C], ref_act.r[..., :C]) and torch.equal(b[..., 4 * C:5 * C], ref_act.r[..., C:])
                for lo, hi in ((0, C), (2 * C, 4 * C), (5 * C, 6 * C)):
                    assert bool((b[..., lo:hi] == 7).all()), kernel
            else:
                assert torch.equal(b[..., C:2 * C], ref_act.r)
                assert bool((b[..., :C] == 7).all()) and bool((b[..., 2 * C:] == 7).all()), kernel
            bf = base['slice_fp32']
            assert torch.equal(bf[..., C:2 * C], ref_act.f)
            assert bool((bf[..., :C] == 7).all()) and bool((bf[..., 2 * C:] == 7).all()), kernel
        else:
            assert torch.equal(base['round'], ref_act.r), kernel

    if regimes is None:
        regimes = GRIDS + (BUDGETS if prec_name == 'f16' else [])

    def plan_of(m, kb):
        return plan(kernel, _n_sm(m), shape, cout=cout, dilation=rate, conv_smem_kb=kb)
    for m, kb in regimes:
        check_regime(plan_of(m, kb), m)
    if prec_name == 'f16' and rate == 1:
        assert [plan_of(m, kb).n_stages for m, kb in BUDGETS] == [1, 2, 3]
    _same_bits_in_every_regime(kernel, run, base, regimes, plan_of)
    return base, run, plan_of


def _check_operand_image(prec_name, f, r):
    """the operand image an epilogue writes next to the fp32 result is that result's image"""
    from l3c_pytorch_b200 import engine as E
    if prec_name == 'f16':
        assert r.dtype == torch.float16 and torch.equal(r, f.clamp(-65504.0, 65504.0).half())
    elif prec_name == 'tf32':
        assert torch.equal(r, E.round_to_tf32(f))
    else:
        C = r.shape[-1] // 2
        np.testing.assert_allclose((r[..., :C].float() + r[..., C:].float() / 2048.0).cpu().numpy(), f.cpu().numpy(),
                                   rtol=2.0 ** -20, atol=1e-9)


@gpu
@pytest.mark.parametrize('case_id,kw,epi', CASES_F16_3X3, ids=[c[0] for c in CASES_F16_3X3])
def test_f16_3x3_every_grid_and_stage_count(case_id, kw, epi):
    """conv_f16_kernel<0>: fp32 PyTorch on FP16-rounded operands; same bits for 1, 2, 3, 7 SMs and 1, 2, 3 stages"""
    _conv3x3_case('f16', case_id, kw, epi)


@gpu
@pytest.mark.parametrize('case_id,kw,epi', CASES_TF32, ids=[c[0] for c in CASES_TF32])
def test_tf32_3x3_every_grid(case_id, kw, epi):
    """conv3x3_tf32_kernel: fp32 PyTorch on TF32-rounded operands (2 stages at d = 1, 1 stage when dilated)"""
    _conv3x3_case('tf32', case_id, kw, epi)


@gpu
@pytest.mark.parametrize('case_id,kw,epi', CASES_F16X2, ids=[c[0] for c in CASES_F16X2])
def test_f16x2_3x3_every_grid(case_id, kw, epi):
    """conv3x3_f16x2_kernel: float64 PyTorch on the unrounded operands; two pipes at d = 1, one pipe when dilated"""
    _conv3x3_case('f16x2', case_id, kw, epi)


@gpu
@pytest.mark.parametrize('case_id,epi', CASES_5X5, ids=[c[0] for c in CASES_5X5])
def test_f16_5x5s2_every_grid_and_stage_count(case_id, epi):
    """conv_f16_kernel<1> (5x5 / stride 2) on odd H / W: fp32 PyTorch on FP16-rounded operands; same bits for
    1, 2, 3, 7 SMs and 1, 2 stages"""
    from l3c_pytorch_b200 import engine as E, _lib
    N, H, W = SHAPE_5X5
    conv = _conv_module(64, 64, 5, stride=2, seed=5)
    x = torch.randn(N, 64, H, W, generator=torch.Generator().manual_seed(55))
    relu = bool(epi.get('relu'))

    def reference():
        y = F.conv2d(_h(x), _h(conv.weight.detach()), conv.bias.detach(), stride=2, padding=2)
        return F.relu(y) if relu else y
    want = _cached(('conv5x5s2_f16', case_id), reference)
    cc = conv.cuda()
    xa = E.Act(None, _nhwc(x).half())

    def run():
        a = E.conv2d(cc, xa, precision=_lib.PREC_F16, want='act', relu=relu)
        return {'fp32': a.f, 'operand': a.r}
    base = run()
    torch.cuda.synchronize()
    np.testing.assert_allclose(_nchw(base['fp32']).numpy(), want.numpy(), rtol=RTOL_OP, atol=ATOL_OP,
                               err_msg='conv5x5s2_f16')
    _check_operand_image('f16', base['fp32'], base['operand'])

    def plan_of(m, kb):
        return plan('conv5x5s2_f16', _n_sm(m), SHAPE_5X5, conv_smem_kb=kb)
    for m, kb in GRIDS + BUDGETS:
        check_regime(plan_of(m, kb), m)
    assert [plan_of(m, kb).n_stages for m, kb in BUDGETS] == [1, 1, 2]
    _same_bits_in_every_regime('conv5x5s2_f16', run, base, GRIDS + BUDGETS, plan_of)


@gpu
def test_f16_3x3_production_size_at_the_default_grid():
    """conv_f16_kernel<0> at 4 x 64 x 126 x 200 with the whole device: 3-4 tiles per pipe, as in the encoder body
    at the bench workload; the knob-driven grids give the same bits."""
    shape = (4, 126, 200)
    p = plan('conv3x3_f16', _n_sm(0), shape)
    assert p.min_tiles() >= 2 and p.n_stages == 3, p
    _conv3x3_case('f16', 'production', dict(cout=64, dilation=1), dict(relu=True), shape=shape,
                  regimes=[(7, 0), (3, 160)])


@gpu
def test_f16_3x3_on_an_sm_partition_stream():
    """The same layer on a stream confined to an SM group (driver green contexts): the grid is sized to the group,
    with and without the knob, and the bits stay the same.  Skipped where the driver cannot partition."""
    from l3c_pytorch_b200 import engine as E
    dev = torch.device('cuda', torch.cuda.current_device())
    part = E.partition_streams(dev, 24, 3, 4)
    if part is None:
        pytest.skip('driver cannot partition SMs (L3C_EUNSUPPORTED)')
    s_a, _, n_a, _ = part
    base, run, _ = _conv3x3_case('f16', 'd1', dict(cout=64, dilation=1), {}, regimes=[])
    for m in (0, 3):
        p = plan('conv3x3_f16', min(m, n_a) if m else n_a, SHAPE)
        if m:
            check_regime(p, m)
        torch.cuda.synchronize()
        with E.conv_launch_limits(max_sms=m):
            with torch.cuda.stream(s_a[0]):
                got = run()
            s_a[0].synchronize()
        for name, want in base.items():
            assert torch.equal(got[name], want), ('conv3x3_f16 on a partition stream', name, m, p)


# ---------------------------------------------------------------------------------------------
# 1x1 layers: conv1x1_tc_kernel<KIND, NB> in the three precisions
# ---------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('prec,cin,cout,extra', CASES_1X1,
                         ids=['%s_%d_%d' % c[:3] for c in CASES_1X1])
def test_1x1_every_grid_and_stage_count(prec, cin, cout, extra):
    """conv1x1_tc_kernel: tf32 / f16 against fp32 PyTorch on the same rounded operands, f16x2 against float64;
    M = 2331 pixels (not a multiple of 64); same bits for 1, 2, 3, 7 SMs and every stage count"""
    from l3c_pytorch_b200 import engine as E, _lib
    kernel = 'conv1x1_' + prec
    N, H, W = SHAPE
    conv = _conv_module(cin, cout, 1, seed=cin + cout)
    x = torch.randn(N, cin, H, W, generator=torch.Generator().manual_seed(cin * cout))
    relu = cout == 120

    def reference():
        w, b = conv.weight.detach(), conv.bias.detach()
        if prec == 'f16':
            y = F.conv2d(_h(x), _h(w), b)
        elif prec == 'tf32':
            y = F.conv2d(E.round_to_tf32(x), E.round_to_tf32(w), b)
        else:
            y = F.conv2d(x.double(), w.double(), b.double())
        return (F.relu(y) if relu else y).float()
    want = _cached((kernel, cin, cout), reference)
    cc = conv.cuda()
    if prec == 'f16':
        xa = E.Act(None, _nhwc(x).half())
    elif prec == 'tf32':
        xa = _nhwc(E.round_to_tf32(x))
    else:
        xa = E.Act(None, E.split_f16x2(_nhwc(x)))
    P = {'f16': _lib.PREC_F16, 'tf32': _lib.PREC_TF32, 'f16x2': _lib.PREC_F16X2}[prec]

    def run():
        if prec == 'f16':
            a = E.conv2d(cc, xa, precision=P, want='act', relu=relu)
            return {'fp32': a.f, 'operand': a.r}
        return {'fp32': E.conv2d(cc, xa, precision=P, relu=relu)}
    base = run()
    torch.cuda.synchronize()
    assert base['fp32'].shape == (N, H, W, cout)
    tol = (RTOL, ATOL) if prec == 'f16x2' else (RTOL_OP, ATOL_OP)
    np.testing.assert_allclose(_nchw(base['fp32']).numpy(), want.numpy(), rtol=tol[0], atol=tol[1], err_msg=kernel)
    if prec == 'f16':
        _check_operand_image('f16', base['fp32'], base['operand'])

    def plan_of(m, kb):
        return plan(kernel, _n_sm(m), SHAPE, cin=cin, cout=cout, conv_smem_kb=kb)
    for m, kb in GRIDS + extra:
        check_regime(plan_of(m, kb), m)
    _same_bits_in_every_regime(kernel, run, base, GRIDS + extra, plan_of)


# ---------------------------------------------------------------------------------------------
# the DMLL head fused into the 1x1 `lin` conv: lin_dmll_f16_kernel
# ---------------------------------------------------------------------------------------------
def _lin_conv_and_input(rgb, C, N, H, W):
    """A `lin` conv (192 -> Kp) and its input, built so that the parameters look like a trained model's: one
    dominant logit, log-scales from -9 (below the -7 clamp) to -1, the ten means of a pixel close together and
    inside or outside [x_min, x_max].  Input channel 0 moves the means, channel 1 the log-scales; the other 190
    channels are noise that every K chunk of the GEMM carries."""
    K = 10
    Kp = (4 if rgb else 3) * C * K
    conv = _conv_module(192, Kp, 1, seed=7)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(N, 192, H, W, generator=g) * 0.5
    x[:, 0] = torch.rand(N, H, W, generator=g) * 2 - 1
    x[:, 1] = torch.rand(N, H, W, generator=g) * 2 - 1
    k = torch.arange(K, dtype=torch.float32)
    center, spread, step, ls0, ls_step = (128.0, 200.0, 3.0, -4.0, 0.6) if rgb else (0.7, 1.4, 0.01, -5.0, 0.1)
    with torch.no_grad():
        w, b = conv.weight, conv.bias
        w.mul_(0.05)
        w[:, :2] = 0
        for c in range(C):
            lg, mu, ls = c * K, C * K + c * K, 2 * C * K + c * K
            b[lg:lg + K] = torch.where(k == 0, torch.tensor(4.0), torch.tensor(0.0))        # a dominant logit
            b[mu:mu + K] = center + step * k
            w[mu:mu + K, 0, 0, 0] = spread
            b[ls:ls + K] = ls0 + ls_step * (k - 4.5)
            w[ls:ls + K, 1, 0, 0] = 4.0
        if rgb:
            b[3 * C * K:] = torch.randn(3 * K, generator=g)
    return conv, x.half()


def _saturated_group_share(pi, mu, ls, targets, L):
    """share of 32-entry groups of the decoder's CDF rows (whole rows for L <= 32) in which EVERY mixture term of
    every entry is saturated, so that dmll_table_kernel adds up pi's instead of evaluating sigmoids -- numpy float32
    with the kernel's arithmetic: u = (t - mu) * (exp(-max(ls, -7)) * -log2 e), saturated iff u <= -25 or u >= 40"""
    inv_s = (np.exp(-ls.astype(np.float32)) * np.float32(-1.4426950408889634)).astype(np.float32)
    t = np.asarray(targets[:L], np.float32)
    u = (t[None, None, :] - mu[:, :, None]) * inv_s[:, :, None]
    sat = ((u <= -25.0) | (u >= 40.0)).all(axis=0)                            # [pixels][L]
    groups = np.stack([sat[:, g:g + 32].all(axis=1) for g in range(0, L, 32)], axis=1)
    return float(groups.mean())


@gpu
@pytest.mark.parametrize('name,rgb,C,L,x_min,x_max,extra', CASES_DMLL, ids=[c[0] for c in CASES_DMLL])
def test_lin_dmll_every_grid_and_stage_count(name, rgb, C, L, x_min, x_max, extra):
    """lin_dmll_f16_kernel on trained-model-like parameters: (1) bit-identical to the F16 1x1 conv + dmll_intervals,
    (2) the interval bounds are the entries of the rows the decoder builds (dmll_build_table), (3) those rows are
    within one count of the reference kernel's CDF formula; then the same bits for 1, 2, 3, 7 SMs and every stage
    count."""
    from l3c_pytorch_b200 import engine as E, _lib
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    from oracle import model as om
    kernel = 'lin_dmll_' + name
    K = 10
    N, H, W = SHAPE
    HW = H * W
    conv, cat_cpu = _lin_conv_and_input(rgb, C, N, H, W)
    # the parameters: the plain F16 1x1 conv against fp32 PyTorch on the same operands, and the sum of the
    # magnitudes of each output's terms (sum |x w| + |b|): the mean rows add ~200-sized products that cancel, and
    # an fp32 accumulation error is a few ulps of that sum, not of the result
    want_l, mag_l = _cached((kernel, 'l'), lambda: (
        F.conv2d(cat_cpu.float(), _h(conv.weight.detach()), conv.bias.detach()),
        F.conv2d(cat_cpu.float().abs(), _h(conv.weight.detach()).abs(), conv.bias.detach().abs())))
    cc = conv.cuda()
    cat = cat_cpu.permute(0, 2, 3, 1).contiguous().cuda()
    sym_cpu = torch.randint(0, L, (N, C, H, W), generator=torch.Generator().manual_seed(9), dtype=torch.uint8)
    sym_cpu[0, :, 0, 0] = L - 1
    sym_cpu[0, :, 0, 1] = 0
    sym = sym_cpu.cuda()
    dm = DiscretizedMixLogisticLoss(rgb, x_min, x_max, L)
    tg = dm.targets(cat.device)

    def run():
        return {'intervals': E.lin_dmll_intervals(cc, cat, sym, tg, C, K, L, rgb)}
    base = run()
    l = E.conv2d(cc, E.Act(None, cat), precision=_lib.PREC_F16)
    torch.cuda.synchronize()
    err = (_nchw(l) - want_l).abs()
    bound = ATOL_OP + RTOL_OP * want_l.abs() + 2e-6 * mag_l
    assert bool((err <= bound).all()), (kernel, float((err - bound).max()), int((err > bound).sum()))
    # (1) the two-step path
    two_step = E.dmll_intervals(l, sym, tg, C, K, L, rgb)
    assert torch.equal(base['intervals'], two_step), (kernel, int((base['intervals'] != two_step).sum()))
    iv = base['intervals'].cpu().numpy().view(np.uint32).reshape(N, C, HW)
    # (2) the decoder's rows
    pitch = E.table_pitch(L)
    table = torch.zeros(N * C * HW * pitch, dtype=torch.int16, device='cuda')
    for c in (range(C) if rgb else [-1]):
        E.dmll_build_table(l, sym, tg, C, K, L, rgb, c, table)
    tab = table.cpu().numpy().view(np.uint16).reshape(N, C, HW, pitch)[..., :L].astype(np.int64)
    s = sym_cpu.reshape(N, C, HW).numpy().astype(np.int64)
    lo = np.take_along_axis(tab, s[..., None], -1)[..., 0]
    hi = np.where(s == L - 1, 65536, np.take_along_axis(tab, np.minimum(s + 1, L - 1)[..., None], -1)[..., 0])
    assert ((iv & 0xFFFF) == lo).all(), kernel
    assert ((iv >> 16).astype(np.int64) + 1 == hi).all(), kernel
    # (3) the reference kernel's CDF formula (oracle) on the mixture parameters the GPU derives from l.  Those
    # parameters agree with the oracle's to float rounding; the formula is compared on the GPU's own, because with
    # log-scales at the -7 clamp (sigma ~ 1e-3) one ulp of a coupled mean moves an entry on the steep part of a
    # component by many counts.  Also: how often the row builder's saturated shortcut applies.
    from oracle import ac
    odm = om.Dmll(rgb, x_min, x_max, L)
    assert torch.equal(tg.cpu(), odm.targets())
    targets = odm.targets().numpy()
    vals = torch.linspace(x_min, x_max, L)
    x_dec = (sym_cpu.float() if rgb else vals[sym_cpu.long()]).contiguous()
    l_cpu = _nchw(l)
    shares = []
    for c in range(C):
        gp = [t.cpu().numpy().reshape(N, K, HW) for t in E.dmll_channel_params(l, x_dec.cuda(), C, K, rgb, c)]
        for n in range(N):
            dec = torch.zeros(1, C, H, W)
            dec[0, :c] = x_dec[n, :c]
            pi, mu, ls = om.channel_params(odm, l_cpu[n:n + 1], c, C, dec)
            np.testing.assert_allclose(gp[0][n], pi, rtol=1e-5, atol=1e-6, err_msg=kernel)
            np.testing.assert_allclose(gp[1][n], mu, rtol=1e-6, atol=1e-4, err_msg=kernel)   # ulps of 255
            assert np.array_equal(gp[2][n], ls), kernel
            want = ac.mixture_cdf(targets, gp[1][n], gp[2][n], gp[0][n])[:, :L].astype(np.int64)
            d = np.abs(want - tab[n, c])
            assert d.max() <= 1, (kernel, n, c, d.max())
            shares.append(_saturated_group_share(gp[0][n], gp[1][n], gp[2][n], targets, L))
    share = float(np.mean(shares))
    assert 0.1 <= share <= 0.9, (kernel, 'share of fully saturated row groups', share)

    def plan_of(m, kb):
        return plan(kernel, _n_sm(m), SHAPE, cin=192, conv_smem_kb=kb)
    for m, kb in GRIDS + extra:
        check_regime(plan_of(m, kb), m)
    _same_bits_in_every_regime(kernel, run, base, GRIDS + extra, plan_of)
