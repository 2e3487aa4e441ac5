"""The training step's 3x3 / 64-input-channel convolutions on the library's TF32 kernels (train.FUSED_CONV, DESIGN
§4.11): per-layer gradients against float64, determinism, routing (nothing in scope reaches cuDNN) and the whole step
against the cuDNN path and the reference's golden step.

Per-layer budget (as tests/test_gpu_layer_parity.py): the float64 reference is computed from the operands as the
kernels read them (x, dy and the weights rounded to TF32 with RNA), so operand rounding drops out and what remains is
fp32 accumulation on the tensor cores.  Each output element gets B = gamma * sum_i |t_i| over its products t_i:
  * forward and dx (conv3x3_tf32_kernel, wgmma): gamma = K * 2^-23, K = 9 * (channels summed) products, one full fp32
    ulp per product (the tensor cores align a group of products to its largest exponent and truncate); for Cout 256
    the four 64-channel partial sums are added through the residual epilogue: 2^-22 more per add.
  * dW (conv3x3_wgrad_kernel, mma.sync m16n8k8): the sum runs as S sequential steps, the k-steps of 8 pixels of one
    chunk and then the chunks; each step is charged 16 ulps of the running sum of magnitudes, gamma = 2^-23 *
    min(K, 16 S), K = the pixels.
  * db (fp32 sums of the unrounded dy): gamma = K * 2^-24, K = the pixels.
Every output must stay under 0.5 B.  The budget is not vacuous: on every case it rejects a dx or dW computed (on the
host) with one tap shifted, and a dW with one input channel dropped.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import util

pytestmark = pytest.mark.gpu

DEV = 'cuda'
CASES = [(cout, d, N, H, W) for (cout, d) in ((64, 1), (64, 2), (64, 4), (256, 1))
         for (N, H, W) in ((1, 5, 9), (3, 9, 7), (1, 33, 17), (3, 128, 128))]


def rna(t):
    from l3c_pytorch_b200.engine import round_to_tf32
    return round_to_tf32(t.float().contiguous())


def _layer(cout, d, seed):
    g = torch.Generator().manual_seed(seed)
    conv = torch.nn.Conv2d(64, cout, 3, padding=d, dilation=d)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) * 0.05)
        conv.bias.copy_(torch.randn(cout, generator=g) * 0.1)
    return conv.to(DEV)


def _inputs(cout, N, H, W, seed):
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(N, 64, H, W, generator=g)
    gy = torch.randn(N, cout // 4 if cout == 256 else cout, H * (2 if cout == 256 else 1),
                     W * (2 if cout == 256 else 1), generator=g)
    return x.to(DEV), gy.to(DEV)


def run_layer(conv, x, gy):
    """forward and backward through train._conv with FUSED_CONV on (PixelShuffle(2) after the 64 -> 256 tail)"""
    from l3c_pytorch_b200 import train
    old = train.FUSED_CONV
    train.FUSED_CONV = True
    try:
        conv.zero_grad(set_to_none=True)
        xr = x.clone().requires_grad_(True)
        y = train._conv(conv, xr)
        if conv.out_channels == 256:
            y = F.pixel_shuffle(y, 2)
        y.backward(gy)
    finally:
        train.FUSED_CONV = old
    return y.detach(), xr.grad.detach(), conv.weight.grad.detach(), conv.bias.grad.detach()


def chunk_steps(N, H, W, cout):
    """sequential accumulation steps of a dW element (conv_train.cu: wg::plan, 8x16 tiles, 132 CTAs)"""
    tiles = N * math.ceil(H / 8) * math.ceil(W / 16)
    tpc = math.ceil(tiles / max(1, 132 // (cout // 64)))
    return 16 * tpc + math.ceil(tiles / tpc)


def references(conv, x, gy):
    """float64 references and budgets of y, dx, dW, db"""
    d = conv.dilation[0]
    cout = conv.out_channels
    N, _, H, W = x.shape
    w64 = rna(conv.weight.detach()).double()
    x64 = rna(x).double()
    dy = F.pixel_unshuffle(gy, 2) if cout == 256 else gy
    dy64 = rna(dy).double()
    kw = dict(padding=d, dilation=d)
    ref = {}
    y = F.conv2d(x64, w64, conv.bias.detach().double(), **kw)
    ya = F.conv2d(x64.abs(), w64.abs(), None, **kw)
    yb = ya * (9 * 64 * 2.0 ** -23) + y.abs() * 2.0 ** -22           # products, then the bias add
    ref['y'] = (F.pixel_shuffle(y, 2), F.pixel_shuffle(yb, 2)) if cout == 256 else (y, yb)
    dx = torch.nn.grad.conv2d_input(x.shape, w64, dy64, **kw)
    dxa = torch.nn.grad.conv2d_input(x.shape, w64.abs(), dy64.abs(), **kw)
    ref['dx'] = (dx, dxa * (9 * cout * 2.0 ** -23 + (cout // 64 - 1) * 2.0 ** -22))
    dw = torch.nn.grad.conv2d_weight(x64, w64.shape, dy64, **kw)
    dwa = torch.nn.grad.conv2d_weight(x64.abs(), w64.shape, dy64.abs(), **kw)
    K = N * H * W
    ref['dw'] = (dw, dwa * 2.0 ** -23 * min(K, 16 * chunk_steps(N, H, W, cout)))
    dyd = dy.double()
    ref['db'] = (dyd.sum((0, 2, 3)), dyd.abs().sum((0, 2, 3)) * K * 2.0 ** -24)
    return ref, x64, dy64, w64


def ratio(got, want, budget):
    err = (got.double() - want).abs()
    return float((err / budget.clamp_min(1e-300)).max())


@pytest.mark.parametrize('cout,d,N,H,W', CASES)
def test_layer_gradients_against_float64(cout, d, N, H, W):
    conv = _layer(cout, d, seed=cout + d)
    x, gy = _inputs(cout, N, H, W, seed=N * H + W)
    y, dx, dw, db = run_layer(conv, x, gy)
    ref, x64, dy64, w64 = references(conv, x, gy)
    got = dict(y=y, dx=dx, dw=dw, db=db)
    r = {k: ratio(got[k], *ref[k]) for k in ref}
    print('cout %d d %d %dx%dx%d  max |err| / B: %s' % (cout, d, N, H, W, ' '.join('%s %.3g' % kv for kv in r.items())))
    for k, v in r.items():
        assert v <= 0.5, (k, r)
    # non-vacuity: the budget rejects one tap shifted (dx, dW) and one input channel dropped (dW)
    kw = dict(padding=d, dilation=d)
    w_shift = w64.clone()
    w_shift[:, :, 0, 0] = w64[:, :, 0, 1]
    dx_bad = torch.nn.grad.conv2d_input(x.shape, w_shift, dy64, **kw)
    assert ratio(dx_bad, *ref['dx']) > 1
    dw_bad = ref['dw'][0].clone()
    dw_bad[:, :, 0, 0] = ref['dw'][0][:, :, 0, 1]
    assert ratio(dw_bad, *ref['dw']) > 1
    x_drop = x64.clone()
    x_drop[:, 5] = 0
    dw_drop = torch.nn.grad.conv2d_weight(x_drop, w64.shape, dy64, **kw)
    assert ratio(dw_drop, *ref['dw']) > 1


@pytest.mark.parametrize('cout,d', [(64, 1), (64, 4), (256, 1)])
def test_backward_is_deterministic(cout, d):
    conv = _layer(cout, d, seed=7)
    x, gy = _inputs(cout, 3, 128, 128, seed=8)
    a = run_layer(conv, x, gy)
    b = run_layer(conv, x, gy)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_weight_images_follow_the_parameter_version():
    """an optimiser step changes the weights in place: the next backward uses the new flipped image"""
    conv = _layer(64, 1, seed=3)
    x, gy = _inputs(64, 1, 16, 16, seed=4)
    run_layer(conv, x, gy)
    with torch.no_grad():
        conv.weight.mul_(-2.0)
    _, dx, _, _ = run_layer(conv, x, gy)
    want = torch.nn.grad.conv2d_input(x.shape, rna(conv.weight.detach()).double(), rna(gy).double(), padding=1)
    assert ratio(dx, want, want.abs() * 1e-2 + 1e-3) <= 1


def test_non_fp32_raises_type_error():
    from l3c_pytorch_b200 import train
    conv = _layer(64, 1, seed=5)
    old = train.FUSED_CONV
    train.FUSED_CONV = True
    try:
        for dt in (torch.float16, torch.float64):
            with pytest.raises(TypeError):
                train._conv(conv, torch.zeros(1, 64, 8, 8, device=DEV, dtype=dt))
        with pytest.raises(TypeError):
            train._conv(conv.double(), torch.zeros(1, 64, 8, 8, device=DEV))
    finally:
        train.FUSED_CONV = old


def _blueprint():
    from l3c_pytorch_b200 import MultiscaleBlueprint, config
    torch.manual_seed(0)
    bp = MultiscaleBlueprint(config.ms_config('cr'), device=DEV)
    bp.net.float()
    bp.net.train()
    return bp


def test_nothing_in_scope_reaches_cudnn(monkeypatch):
    """FUSED_CONV on: no F.conv2d call carries a 3x3 weight with 64 input channels, every out-of-scope layer of the
    step still calls it, and the library's kernels run; off: no library conv kernel runs"""
    from l3c_pytorch_b200 import engine, train
    bp = _blueprint()
    names = {p.data_ptr(): n for n, p in bp.net.named_parameters()}
    calls = []
    real = F.conv2d

    def counting(x, weight, *a, **k):
        calls.append(names.get(weight.data_ptr(), '?'))
        return real(x, weight, *a, **k)

    monkeypatch.setattr(torch.nn.functional, 'conv2d', counting)
    imgs = torch.stack([util.make_image(i, 32, 32) for i in range(2)]).float().to(DEV)
    seen = {}
    for fused in (False, True):
        monkeypatch.setattr(train, 'FUSED_CONV', fused)
        calls.clear()
        engine.launch_log(reset=True)
        train.train_step(bp, train.make_optimizer(bp), imgs)
        torch.cuda.synchronize()
        seen[fused] = (set(calls), engine.launch_log(reset=True)[0])
    params = dict(bp.net.named_parameters())
    in_scope = {n for n in seen[False][0] if train.conv3x3_in_scope(_module_of(bp.net, n))}
    assert in_scope and all(params[n].shape[1] == 64 and params[n].shape[2:] == (3, 3) for n in in_scope)
    assert seen[True][0] == seen[False][0] - in_scope
    assert not any(params[n].shape[1] == 64 and params[n].shape[2:] == (3, 3) for n in seen[True][0])
    k_on, k_off = seen[True][1], seen[False][1]
    for k in ('conv3x3_tf32_kernel', 'conv3x3_wgrad_kernel', 'conv3x3_wgrad_finish_kernel', 'round_tf32_kernel'):
        assert k_on.get(k, 0) > 0 and k_off.get(k, 0) == 0, (k, k_on, k_off)
    assert k_on['conv3x3_wgrad_kernel'] == len(in_scope)


def _module_of(net, weight_name):
    return net.get_submodule(weight_name.rsplit('.', 1)[0])


def _step(bp, imgs, fused):
    from l3c_pytorch_b200 import train
    old = train.FUSED_CONV
    train.FUSED_CONV = fused
    try:
        opt = train.make_optimizer(bp)
        bp.net.zero_grad()
        loss, bpsps = train.training_loss(bp, imgs)
        loss.backward()
        grads = {k: p.grad.detach().clone() for k, p in bp.net.named_parameters() if p.grad is not None}
        opt.step()
        torch.cuda.synchronize()
    finally:
        train.FUSED_CONV = old
    return float(loss.detach()), bpsps, grads, {k: p.detach().clone() for k, p in bp.net.named_parameters()}


# TF32 against TF32: both paths round the convolutions' operands to 10 mantissa bits, in different places and
# orders (cuDNN's TF32 kernels and ours), so they agree to TF32 precision, not to fp32.  Loss and bpsp relative,
# gradient norms relative per parameter.  RMSprop's first step moves an element by lr g / (0.1 |g| + 1e-8): 10 lr
# sign(g) once |g| >> 1e-7, so where a gradient is near 0 the two paths may move an element by different amounts or
# ways.  Parameters must agree (rtol 1e-3, atol 2e-5) wherever both gradients have the same sign and |g| > 1e-5 (the
# step then varies by < 1 % of 10 lr = 1e-5).
STEP_TOL = dict(loss=2e-3, bpsp=2e-3, grad=3e-2, param_rtol=1e-3, param_atol=2e-5)


@pytest.mark.parametrize('N,S', [(2, 32), (30, 128)])
def test_step_matches_the_cudnn_path(N, S):
    g = torch.Generator(device=DEV).manual_seed(0)
    imgs = (torch.rand(N, 3, S, S, device=DEV, generator=g) * 255).round()
    out = {f: _step(_blueprint(), imgs, f) for f in (False, True)}
    (l0, b0, g0, p0), (l1, b1, g1, p1) = out[False], out[True]
    dev = dict(loss=abs(l1 - l0) / l0, bpsp=max(abs(u - v) / abs(v) for u, v in zip(b1, b0)),
               grad=max(float((g1[k].norm() - g0[k].norm()).abs() / (g0[k].norm() + 1e-7)) for k in g0))
    flips = sum(int((g1[k].sign() != g0[k].sign()).sum()) for k in g0)
    small = sum(int(((g0[k].abs() <= 1e-5) | (g1[k].abs() <= 1e-5)).sum()) for k in g0)
    print('%d x %d^2: fused vs cuDNN relative deviation %s, gradient sign flips %d, |g| <= 1e-5 %d, of %d'
          % (N, S, dev, flips, small, sum(g.numel() for g in g0.values())))
    assert g0.keys() == g1.keys()
    assert dev['loss'] < STEP_TOL['loss'] and dev['bpsp'] < STEP_TOL['bpsp'], dev
    assert dev['grad'] < STEP_TOL['grad'], dev
    for k in p0:
        same = ((g1[k].sign() == g0[k].sign()) & (g0[k].abs() > 1e-5) & (g1[k].abs() > 1e-5) if k in g0
                else torch.ones_like(p0[k], dtype=torch.bool))
        np.testing.assert_allclose(p1[k][same].cpu().numpy(), p0[k][same].cpu().numpy(), rtol=STEP_TOL['param_rtol'],
                                   atol=STEP_TOL['param_atol'], err_msg=k)


def test_step_against_the_reference_golden():
    """tests/golden/train_step.json at test_train_step.py's tolerances (loss 2e-4, grad norms 2e-3, parameters rtol
    1e-3 / atol 2e-5), with the convolutions in TF32 on our kernels"""
    import json
    import os
    with open(os.path.join(os.path.dirname(__file__), 'golden', 'train_step.json')) as f:
        gold = json.load(f)
    imgs = torch.stack([util.make_image(i, 32, 32) for i in range(2)]).float().to(DEV)
    loss, bpsps, grads, params = _step(_blueprint(), imgs, True)
    dev_loss = abs(loss - gold['loss_pc']) / gold['loss_pc']
    grads = {k: float(g.norm()) for k, g in grads.items()}
    dev_grad = max(abs(grads[k] - v) / v for k, v in gold['grad_norms'].items())
    print('fused step vs golden: loss %.3g, bpsp %s, worst grad norm %.3g' % (
        dev_loss, [abs(a - b) / b for a, b in zip(bpsps, gold['nonrecursive_bpsps'])], dev_grad))
    assert dev_loss < 2e-4
    np.testing.assert_allclose(bpsps, gold['nonrecursive_bpsps'], rtol=2e-4)
    for k, want in gold['grad_norms'].items():
        assert abs(grads[k] - want) < 2e-3 * want + 1e-7, (k, grads[k], want)
    for k, want in gold['params_after_step'].items():
        np.testing.assert_allclose(params[k].flatten()[:4].cpu().numpy(), want, rtol=1e-3, atol=2e-5)
