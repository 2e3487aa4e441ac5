"""The closed-form gradients the training kernels evaluate (DESIGN §4.9, dmll.cu dmll_train_grad_kernel and
soft_quantize_kernel), checked in float64 on the CPU against torch.autograd of the torch restatements they replace
(train.dmll_nll, train.soft_quantize_torch).

`dmll_grads` states the gradient of the summed DMLL nats once, in torch operators of any dtype:
* float64, `torch_like=True`: the same arithmetic autograd runs (sigmoid' = s (1 - s), delta = s+ - s-), so it must
  equal autograd to rounding -- this file;
* float64, `stable=True`: the exact values (delta and sigmoid' without cancellation), with the kernel's fp32 branch
  and clamp decisions passed in -- the reference of tests/test_gpu_train_kernels.py;
* float32, `torch_like=True`: the kernel's formula, for the self-test of that file's error budget."""
import math

import numpy as np
import pytest
import torch

from tests.test_gpu_dmll_loss import GRIDS, K, _fam_random, _family

LOG_SCALES_MIN = -7.0


def _softplus_slope(v):
    """d softplus / dv with torch's threshold 20"""
    return torch.where(v > 20, torch.ones_like(v), torch.sigmoid(v))


def dmll_grads(l, x, rgb, half, x_lower, x_upper, g, stable=False, torch_like=False, delta_ok=None):
    """Gradient of sum(train.dmll_nll) for upstream gradient g.  l [N, Kp, H, W], x [N, C, H, W] tensors of one dtype.
    delta_ok (bool like the components [N, C, K, H, W]) overrides the middle branch's clamp decision delta >= 1e-12.
    -> dict: dl [N, Kp, H, W], dx [N, C, H, W] (None for rgb), and the per-component quantities the budget uses."""
    N, C, H, W = x.shape
    P = 4 if rgb else 3
    lr = l.reshape(N, P, C, K, H, W)
    logit, mean, ls_raw = lr[:, 0], lr[:, 1], lr[:, 2]
    ls = torch.clamp(ls_raw, min=LOG_SCALES_MIN)
    x0, x1 = x[:, 0:1], x[:, 1:2] if C > 1 else None
    mu = mean.clone()
    if rgb:
        co = torch.sigmoid(lr[:, 3])
        mu[:, 1] = mean[:, 1] + co[:, 0] * x0
        mu[:, 2] = mean[:, 2] + co[:, 1] * x0 + co[:, 2] * x1
    xr = x[:, :, None]
    inv = torch.exp(-ls)
    cx = xr - mu
    up, um = inv * (cx + half), inv * (cx - half)
    sp, sm = torch.sigmoid(up), torch.sigmoid(um)
    if stable:
        log_delta = torch.log(-torch.expm1(um - up)) + torch.nn.functional.logsigmoid(up) - \
            torch.nn.functional.softplus(um)
        delta = torch.exp(log_delta)
    else:
        delta = sp - sm
        log_delta = torch.log(torch.clamp(delta, min=1e-12))
    ok = (delta >= 1e-12) if delta_ok is None else delta_ok
    hi = (xr > x_upper).expand_as(up)
    lo = (xr < x_lower).expand_as(up)
    sp_t = lambda v: torch.where(v > 20, v, torch.log1p(torch.exp(torch.clamp(v, max=20.))))  # noqa: E731
    lp = torch.where(ok, log_delta, torch.full_like(delta, math.log(np.float32(1e-12)) if l.dtype == torch.float32
                                                   else math.log(1e-12)))
    lp = torch.where(hi, -sp_t(um), lp)
    lp = torch.where(lo, up - sp_t(up), lp)
    logpi = logit - torch.logsumexp(logit, 2, keepdim=True)
    w = lp + logpi
    nll = -torch.logsumexp(w, 2)
    r = torch.exp(w + nll[:, :, None])
    pi = torch.exp(logpi)
    dlogit = g * (pi - r)
    e = -g * r
    if torch_like:
        d_sig = lambda s, v: s * (1 - s)                                                # noqa: E731
        lower = 1 - _softplus_slope(up)
    else:
        d_sig = lambda s, v: s * torch.sigmoid(-v)                                      # noqa: E731
        lower = torch.where(up > 20, torch.zeros_like(up), torch.sigmoid(-up))
    zero = torch.zeros_like(e)
    mid = ok & ~hi & ~lo
    safe = torch.where(mid, delta, torch.ones_like(delta))
    ap = torch.where(lo, e * lower, torch.where(mid, e * d_sig(sp, up) / safe, zero))
    am = torch.where(lo | ~hi, torch.where(mid, -e * d_sig(sm, um) / safe, zero), -e * _softplus_slope(um))
    dmean = -inv * (ap + am)
    dls = torch.where(ls_raw >= LOG_SCALES_MIN, -(up * ap + um * am), zero)
    planes = [dlogit, dmean, dls]
    dx = None
    if rgb:
        dsc = (lambda v: torch.sigmoid(v) * (1 - torch.sigmoid(v))) if torch_like else \
            (lambda v: torch.sigmoid(v) * torch.sigmoid(-v))                            # noqa: E731
        dco = torch.stack([dmean[:, 1] * x0 * dsc(lr[:, 3, 0]), dmean[:, 2] * x0 * dsc(lr[:, 3, 1]),
                           dmean[:, 2] * x1 * dsc(lr[:, 3, 2])], 1)
        planes.append(dco)
    else:
        dx = (inv * (ap + am)).sum(2)
    dl = torch.stack(planes, 1).reshape(l.shape)
    return dict(dl=dl, dx=dx, nll=nll, ap=ap, am=am, up=up, um=um, sp=sp, sm=sm, delta=delta, log_delta=log_delta,
                inv=inv, cx=cx, hi=hi, lo=lo, ok=ok, mid=mid, r=r, pi=pi, w=w, logit=logit, ls_raw=ls_raw, dmean=dmean,
                mean=mean, mu=mu)


def family_nchw(grid, fam, seed=0):
    """a parameter family of tests/test_gpu_dmll_loss.py as one NCHW image of 1 x P pixels: (g, l, x)"""
    if fam == 'random':
        g = GRIDS[grid]
        sym, l, _ = _fam_random(g, np.random.default_rng(77 + seed), 3000)
    else:
        g, sym, l, _ = _family(grid, fam, seed)
    x = g.values[sym.astype(np.int64)]                           # [P, C]
    P = len(x)
    return g, np.ascontiguousarray(l.T).reshape(1, -1, 1, P), np.ascontiguousarray(x.T).reshape(1, g.C, 1, P)


def _dm(g):
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    return DiscretizedMixLogisticLoss(g.rgb, g.x_min, g.x_max, g.L)


HOST_CASES = ([('rgb', f) for f in ('random', 'edge', 'ls_clamp', 'clamp_right', 'clamp_left', 'softplus', 'coupling')]
              + [('bottleneck', f) for f in ('random', 'edge', 'ls_clamp', 'clamp_right', 'clamp_left', 'softplus')])


@pytest.mark.parametrize('grid,fam', HOST_CASES)
def test_dmll_closed_form_equals_autograd(grid, fam):
    from l3c_pytorch_b200 import train
    g, l, x = family_nchw(grid, fam)
    dm = _dm(g)
    gup = 0.37
    lt = torch.from_numpy(l).double().requires_grad_(True)
    xt = torch.from_numpy(x).double().requires_grad_(not g.rgb)
    (train.dmll_nll(dm, xt, lt).sum() * gup).backward()
    d = dmll_grads(lt.detach(), xt.detach(), g.rgb, dm.bin_width / 2, dm.x_lower_bound, dm.x_upper_bound, gup,
                   torch_like=True)
    # every branch the case is about is taken, and the gradient is exactly 0 where the reference's is
    counts = dict(middle=int(d['mid'].sum()), upper=int((d['hi'] & ~d['lo']).sum()), lower=int(d['lo'].sum()),
                  clamped=int((~d['ok'] & ~d['hi'] & ~d['lo']).sum()), ls_clamped=int((d['ls_raw'] < -7).sum()))
    need = {'edge': ('upper', 'lower'), 'softplus': ('upper', 'lower'), 'clamp_right': ('clamped',),
            'ls_clamp': ('ls_clamped',), 'random': ('middle', 'clamped', 'ls_clamped')}.get(fam, ('middle',))
    for k in need:
        assert counts[k] >= 50, (grid, fam, counts)
    want = lt.grad.reshape(d['dl'].shape)
    got = d['dl']
    scale = gup * (1 + d['inv'].max())
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-9, atol=1e-13 * float(scale))
    P = 4 if g.rgb else 3
    lr = want.reshape(1, P, g.C, K, 1, -1)
    assert (lr[:, 2][d['ls_raw'] < -7] == 0).all()
    assert (lr[:, 1][~d['ok'] & ~d['hi'] & ~d['lo']] == 0).all()
    assert (got.reshape(lr.shape)[:, 2][d['ls_raw'] < -7] == 0).all()
    assert (d['ap'][d['hi'] & ~d['lo']] == 0).all() and (d['am'][d['lo']] == 0).all()
    if g.rgb:
        assert float(lr[:, 3].abs().max()) > 0
        assert xt.grad is None
    else:
        np.testing.assert_allclose(d['dx'].numpy(), xt.grad.numpy(), rtol=1e-9, atol=1e-13 * float(scale))


def soft_quantize_grad64(q, levels, sigma, g):
    """2 sigma Var_phi(levels) in centred form, phi = softmax_l(-sigma (q - c_l)^2), times g"""
    d = (q[..., None] - levels) ** 2
    phi = torch.softmax(-sigma * d, -1)
    cbar = (phi * levels).sum(-1, keepdim=True)
    return g * 2 * sigma * (phi * (levels - cbar) ** 2).sum(-1)


def test_soft_quantizer_gradient_is_two_sigma_variance():
    from l3c_pytorch_b200 import train
    rng = np.random.default_rng(5)
    levels = torch.linspace(-1, 1, 25, dtype=torch.float64)
    q = torch.from_numpy(np.concatenate([rng.uniform(-1.3, 1.3, 4000), rng.normal(0, 0.05, 1000),
                                         levels.numpy() + rng.normal(0, 1e-3, 25), [-5.0, 5.0, 1 / 24]]))
    q = q.reshape(1, 1, 1, -1).requires_grad_(True)
    g = torch.from_numpy(rng.normal(0, 1, q.shape))
    for sigma in (2.0, 0.5, 40.0):
        q.grad = None
        x_soft, x_hard, sym = train.soft_quantize_torch(q, levels, sigma)
        x_soft.backward(g)
        got = soft_quantize_grad64(q.detach(), levels, sigma, g)
        np.testing.assert_allclose(got.numpy(), q.grad.numpy(), rtol=1e-9, atol=1e-14)
        assert float(got.abs().max()) > 0.1
