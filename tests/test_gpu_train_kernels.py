"""The training kernels (DESIGN §4.9: l3c_dmll_nll_train, l3c_soft_quantize) and the training step that runs on them.

* DMLL gradients, element by element and for every Kp plane, against `dmll_grads` (tests/test_train_kernels_host.py)
  in float64 without cancellation, given the kernel's fp32 branch and clamp decisions.  Every element carries a
  first-order fp32 budget (`grad_budget`) that follows the cancellation of delta = sigmoid(u+) - sigmoid(u-); a CPU
  self-test holds the budget against a float32 evaluation of the same formula and checks that it is not vacuous.
  The parameter families are those of tests/test_gpu_dmll_loss.py, as NCHW batches of N = 2 and HW % 128 != 0.
* The quantiser: symbols bit-equal to torch.min on CUDA (ties included), values exact, dq within budget.
* The whole step: the fused and the torch-loss paths on the same weights and batch, and the fused step against the
  unmodified reference's step (tests/golden/train_step.json).
* Determinism, launches per scale, peak memory against the torch path, and the refusals."""
import json
import os

import numpy as np
import pytest
import torch

from tests.test_gpu_dmll_loss import FAMILY_CASES, K, U, nll64, quantiser_inputs, _cr_levels
from tests.test_train_kernels_host import dmll_grads, family_nchw, _dm, soft_quantize_grad64

F32 = np.float32
GUP = 0.731                       # an upstream gradient != 1
TINY = 2.0 ** -110                # absolute floor of the budget: intermediates below fp32's normal range


# ---------------------------------------------------------------------------------------------
# the budget
# ---------------------------------------------------------------------------------------------
def _bounds(dm):
    return dm.bin_width / 2, float(F32(dm.x_lower_bound)), float(F32(dm.x_upper_bound))


def reference(g, l, x, dm, gup):
    """-> (d64: dmll_grads in float64, exact, with the fp32 decisions; d32: the same formula in float32)"""
    half, lo_b, hi_b = _bounds(dm)
    l32, x32 = torch.from_numpy(l).float(), torch.from_numpy(x).float()
    d32 = dmll_grads(l32, x32, g.rgb, F32(half), F32(lo_b), F32(hi_b), F32(gup), torch_like=True)
    d64 = dmll_grads(l32.double(), x32.double(), g.rgb, half, lo_b, hi_b, gup, stable=True, delta_ok=d32['ok'])
    return d64, d32


def grad_budget(d, rgb):
    """First-order fp32 error of every gradient element, from the float64 quantities d (dmll_grads, stable) -> dict
    dl, dx like d['dl'], d['dx'], and the natural scale of every element (the sum of the magnitudes it is made of).

    u = inv (x - mu +- half) is off by eta = inv (2u|x - mu| + eps_mu) + 3u|u| (eps_mu: the rounding of a coupled
    mean).  delta = s+ - s- is off by a relative z = (4u (s+ + s-) + eta (s+' + s-')) / delta, so 1 / delta by at most
    a factor q = delta / max(delta (1 - z), 1e-12) (an element the kernel did not clamp has delta32 >= 1e-12).  lp is
    off by eps = log q + 8u (1 + |lp|) (edge branches: 8u (1 + |lp| + |u|) + eta), w_k by eps_k + 2u (|logit| + |lse|),
    nats by sum_k r_k eps_w + 16u (1 + |nll|), so r_k by a relative rho_k = expm1(eps_w + eps_nll + 4u (1 + |w|)) and
    pi by 4u (1 + |logit| + |lse|).  a+- = e sigmoid'(u)/delta (or e times a sigmoid on an edge) is off by
    (1 + rho)(1 + eta + 2u / sigmoid(-u) + 4u) q - 1 (sigmoid' and sigmoid move by at most eta per unit of u; the
    kernel forms sigmoid' as s (1 - s) and the lower slope as 1 - s, as torch does, and 1 - s is off by u absolutely,
    2u / sigmoid(-u) relatively; likewise sigmoid'(coeff)).  dmean, dlogscale, dx and
    dcoeff add the relative errors of the products they are made of and 4u per operation, doubled.  Underflow: every a+-
    may lose TINY / delta (middle branch) or TINY, every element TINY."""
    ap, am, up, um = d['ap'], d['am'], d['up'], d['um']
    sp, sm, inv, r, pi, w, nll = d['sp'], d['sm'], d['inv'], d['r'], d['pi'], d['w'], d['nll']
    eps_mu = torch.zeros_like(up)
    if rgb:
        eps_mu = 4 * U * (d['mean'].abs() + (d['mu'] - d['mean']).abs())
        eps_mu[:, 0] = 0                                     # R: the mean is a parameter, not a rounded sum
    eta_of = lambda v: inv * (2 * U * d['cx'].abs() + eps_mu) + 3 * U * v.abs()      # noqa: E731
    eta_p, eta_m = eta_of(up), eta_of(um)
    dsig_p, dsig_m = sp * torch.sigmoid(-up), sm * torch.sigmoid(-um)
    delta = d['delta'].clamp(min=1e-300)
    z = (4 * U * (sp + sm) + eta_p * dsig_p + eta_m * dsig_m) / delta
    # delta32 lies in [max(delta (1 - z), 1e-12), delta (1 + z)]: 1 / delta32 is off by at most a relative q - 1
    q_up = delta / torch.maximum(delta * (1 - z).clamp(min=0), torch.full_like(delta, 1e-12))
    q = 1 + torch.maximum(q_up - 1, z / (1 + z))
    q = torch.where(d['mid'], q, torch.ones_like(q))
    lp = w - (d['logit'] - torch.logsumexp(d['logit'], 2, keepdim=True))
    edge = d['hi'] | d['lo']
    arg = torch.where(d['lo'], up, um)
    eps_lp = torch.where(edge, 8 * U * (1 + lp.abs() + arg.abs()) + torch.where(d['lo'], eta_p, eta_m),
                         torch.log(q) + 8 * U * (1 + lp.abs()))
    lse = torch.logsumexp(d['logit'], 2, keepdim=True)
    eps_w = eps_lp + 2 * U * (d['logit'].abs() + lse.abs())
    eps_nll = (r * eps_w).sum(2, keepdim=True) + 16 * U * (1 + nll.abs()[:, :, None])
    rho = torch.expm1(eps_w + eps_nll + 4 * U * (1 + w.abs()))
    pi_rel = 4 * U * (1 + d['logit'].abs() + lse.abs())
    dlogit_b = abs(GUP) * (r * rho + pi * pi_rel) + 2 * U * abs(GUP) * (pi + r)
    dlogit_s = abs(GUP) * (pi + r)
    # 1 - s is off by u absolutely: sigmoid' = s (1 - s) and 1 - s by a relative 2u / sigmoid(-u)
    om_p, om_m = 2 * U / torch.sigmoid(-up).clamp(min=1e-300), 2 * U / torch.sigmoid(-um).clamp(min=1e-300)
    rel_p = (1 + rho) * (1 + eta_p + om_p + 4 * U) * q - 1 + 4 * U
    rel_m = (1 + rho) * (1 + eta_m + om_m + 4 * U) * q - 1 + 4 * U
    ea_p, ea_m = ap.abs() * rel_p, am.abs() * rel_m
    inv_rel = 2 * U * (1 + d['ls_raw'].clamp(min=-7).abs())
    mean_s = inv * (ap.abs() + am.abs())
    # a product that underflows fp32 on the way (r, a sigmoid's tail) loses < TINY, which 1 / delta, inv and u can grow
    tiny_a = TINY * torch.where(d['mid'], 1 / delta.clamp(min=1e-12), torch.ones_like(delta))
    ea_p, ea_m = ea_p + tiny_a, ea_m + tiny_a
    mean_b = inv * (ea_p + ea_m) + mean_s * (inv_rel + 4 * U)
    ls_s = (1 + up.abs()) * ap.abs() + (1 + um.abs()) * am.abs()
    ls_b = up.abs() * ea_p + um.abs() * ea_m + ap.abs() * eta_p + am.abs() * eta_m + 4 * U * ls_s
    ls_b = torch.where(d['ls_raw'] >= -7, ls_b, torch.zeros_like(ls_b))
    planes_b, planes_s = [dlogit_b, mean_b, ls_b], [dlogit_s, mean_s, ls_s]
    out = {}
    if rgb:
        N, C, _, H, W = ap.shape
        l = d['dl'].reshape(N, 4, C, K, H, W)
        x = d['x']
        co_raw = d['co_raw']
        dsc = torch.sigmoid(co_raw) * torch.sigmoid(-co_raw)
        srcs = [(1, x[:, 0:1]), (2, x[:, 0:1]), (2, x[:, 1:2])]
        cb, cs = [], []
        for j, (c, xv) in enumerate(srcs):
            f = xv.abs() * dsc[:, j]
            om = 2 * U / torch.sigmoid(-co_raw[:, j]).clamp(min=1e-300)
            cb.append(f * mean_b[:, c] + l[:, 3, j].abs() * (8 * U + om) + 255 * TINY)
            cs.append(f * mean_s[:, c])
        planes_b.append(torch.stack(cb, 1))
        planes_s.append(torch.stack(cs, 1))
    else:
        out['dx'] = 2 * (mean_b.sum(2) + 2 * K * U * mean_s.sum(2)) + TINY
        out['dx_scale'] = mean_s.sum(2)
    shape = d['dl'].shape
    out['dl'] = 2 * torch.stack(planes_b, 1).reshape(shape) + TINY
    out['dl_scale'] = torch.stack(planes_s, 1).reshape(shape)
    return out


def _with_inputs(d, l, x, g):
    d['x'] = torch.from_numpy(x).double()
    if g.rgb:
        N, C, H, W = x.shape
        d['co_raw'] = torch.from_numpy(l).double().reshape(N, 4, C, K, H, W)[:, 3]
    return d


def _assert_within(got, want, budget, what):
    err = (got - want).abs()
    ok = err <= budget
    if not bool(ok.all()):
        i = int(torch.argmax(torch.where(ok, torch.zeros_like(err), err / budget.clamp(min=1e-300))))
        raise AssertionError('%s: %d of %d elements outside their budget; worst flat index %d: got %r, float64 %r, '
                             'budget %.3g' % (what, int((~ok).sum()), ok.numel(), i, float(got.flatten()[i]),
                                              float(want.flatten()[i]), float(budget.flatten()[i])))
    return float((err / budget.clamp(min=1e-300)).max())


def _batch(grid, fam):
    """the family as N = 2 images of HW pixels, HW % 128 != 0"""
    g, l, x = family_nchw(grid, fam)
    P = l.shape[-1] - l.shape[-1] % 2
    if (P // 2) % 128 == 0:
        P -= 2
    HW = P // 2
    l = np.ascontiguousarray(l[..., :P].reshape(l.shape[1], 2, HW).transpose(1, 0, 2)).reshape(2, -1, 1, HW)
    x = np.ascontiguousarray(x[..., :P].reshape(g.C, 2, HW).transpose(1, 0, 2)).reshape(2, g.C, 1, HW)
    return g, l, x


BUDGET_CASES = FAMILY_CASES + [('rgb', 'random'), ('bottleneck', 'random')]


def test_grad_budget_covers_the_fp32_formula_and_is_not_vacuous():
    """The budget against the float32 evaluation of the kernel's formula on every family: every element inside its
    budget; on the well-conditioned components of well-conditioned sub-pixels (posterior-weighted conditioning of
    delta below 4 and no component's above 1e3, the component's own below 10, |u+-| <= 5 there and <= 30 for every
    component of the sub-pixel, logits within +-20, no coupled mean) the budget of the
    logit, mean and log-scale gradients stays below 1e-4 of the element's natural scale, so it cannot hide a real
    error."""
    n_el, n_well, worst = 0, 0, 0.0
    for grid, fam in BUDGET_CASES:
        g, l, x = _batch(grid, fam)
        d64, d32 = reference(g, l, x, _dm(g), GUP)
        b = grad_budget(_with_inputs(d64, l, x, g), g.rgb)
        worst = max(worst, _assert_within(d32['dl'].double(), d64['dl'], b['dl'], '%s/%s dl emulated' % (grid, fam)))
        if not g.rgb:
            worst = max(worst, _assert_within(d32['dx'].double(), d64['dx'], b['dx'], '%s/%s dx' % (grid, fam)))
        n_el += d64['dl'].numel()
        sa, sb = d64['sp'], d64['sm']
        cond = (sa + sb + d64['inv'] * d64['cx'].abs() * (sa * (1 - sa) + sb * (1 - sb))) / d64['delta'].clamp(min=1e-12)
        cond = torch.where(d64['hi'] | d64['lo'], torch.zeros_like(cond), cond)
        well = (((d64['r'] * cond).sum(2) < 4) & (cond.amax(2) < 1e3) & (d64['logit'].abs().amax(2) <= 20)
                & (torch.maximum(d64['up'].abs(), d64['um'].abs()).amax(2) <= 30))
        if g.rgb:
            well &= torch.zeros_like(well).index_fill_(1, torch.tensor([0]), True)        # R: no coupled mean
        well = well[:, :, None] & (cond < 10) & (d64['up'].abs() <= 5) & (d64['um'].abs() <= 5)
        N, C, H, W = x.shape
        P = 4 if g.rgb else 3
        rel = (b['dl'] / (b['dl_scale'] + 1e-30)).reshape(N, P, C, K, H, W)[:, :3]
        for i in range(3):
            assert bool((rel[:, i][well] < 1e-4).all()), (grid, fam, i, float(rel[:, i][well].max()))
        n_well += int(well.sum())
    print('\ngradient budget self-test: %d elements, largest error / budget %.3f, %d well-conditioned sub-pixels'
          % (n_el, worst, n_well))
    assert n_well >= 10000


# ---------------------------------------------------------------------------------------------
# GPU: the DMLL loss and its gradient per element
# ---------------------------------------------------------------------------------------------
def _kernel(g, l, x, gup):
    from l3c_pytorch_b200 import engine as E
    dm = _dm(g)
    half, lo_b, hi_b = dm.bin_width / 2, dm.x_lower_bound, dm.x_upper_bound
    lt, xt = torch.from_numpy(l).cuda(), torch.from_numpy(x).cuda()
    nll = E.dmll_nll_train(lt, xt, K, g.rgb, half, lo_b, hi_b)
    dl, dx = E.dmll_nll_train(lt, xt, K, g.rgb, half, lo_b, hi_b, grad=torch.tensor(gup, device='cuda'),
                              want_dx=not g.rgb)
    return nll.cpu(), dl.cpu().double(), None if dx is None else dx.cpu().double()


@pytest.mark.gpu
@pytest.mark.parametrize('grid,fam', FAMILY_CASES)
def test_dmll_gradients_within_budget_of_float64(grid, fam):
    g, l, x = _batch(grid, fam)
    d64, d32 = reference(g, l, x, _dm(g), GUP)
    b = grad_budget(_with_inputs(d64, l, x, g), g.rgb)
    nll, dl, dx = _kernel(g, l, x, GUP)
    worst = _assert_within(dl, d64['dl'], b['dl'], '%s/%s dl' % (grid, fam))
    if not g.rgb:
        worst = max(worst, _assert_within(dx, d64['dx'], b['dx'], '%s/%s dx' % (grid, fam)))
    print('%s/%s: largest error / budget %.3f' % (grid, fam, worst))
    # exactly 0 where the reference's gradient is 0
    N, C, _, HW = x.shape
    P = 4 if g.rgb else 3
    lr = dl.reshape(N, P, C, K, 1, HW)
    assert bool((lr[:, 2][d64['ls_raw'] < -7] == 0).all())
    clamped = ~d64['ok'] & ~d64['hi'] & ~d64['lo']
    assert bool((lr[:, 1][clamped] == 0).all()) and bool((lr[:, 2][clamped] == 0).all())
    # the forward: per-image nats against nll64 within the summed per-sub-pixel budget
    for n in range(N):
        ln = l[n].reshape(l.shape[1], HW).T
        xn = x[n].reshape(C, HW).T
        d = nll64(ln, xn, g)
        assert abs(float(nll[n]) - float(d['nll'].sum())) <= float(d['budget'].sum()) + 1e-9 * abs(float(nll[n]))


@pytest.mark.gpu
def test_gradients_are_deterministic_and_take_one_launch_per_pass():
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200 import train
    for grid in ('rgb', 'bottleneck'):
        g, l, x = _batch(grid, 'random')
        dm = _dm(g)
        lt = torch.from_numpy(l).cuda().requires_grad_(True)
        xt = torch.from_numpy(x).cuda().requires_grad_(not g.rgb)
        runs = []
        for _ in range(2):
            lt.grad = xt.grad = None
            E.launch_log(reset=True)
            loss = train.dmll_nll_sum(dm, xt, lt)
            fwd, n_fwd = E.launch_log(reset=True)
            (loss * GUP).backward()
            bwd, n_bwd = E.launch_log(reset=True)
            assert fwd == {'dmll_train_nll_kernel': 1, 'nll_finish_kernel': 1} and n_fwd == 2, fwd
            assert bwd == {'dmll_train_grad_kernel': 1} and n_bwd == 1, bwd
            runs.append((loss.detach().clone(), lt.grad.clone(), None if g.rgb else xt.grad.clone()))
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
        if not g.rgb:
            assert torch.equal(runs[0][2], runs[1][2])
    q = torch.randn(3, 5, 33, 17, device='cuda', requires_grad=True)
    levels = torch.linspace(-1, 1, 25, device='cuda')
    E.launch_log(reset=True)
    v, _, _ = train.soft_quantize(q, levels, 2.0)
    assert E.launch_log(reset=True)[0] == {'soft_quantize_kernel': 1}
    v.sum().backward()
    assert E.launch_log(reset=True)[0] == {'soft_quantize_kernel': 1}


# ---------------------------------------------------------------------------------------------
# GPU: the quantiser
# ---------------------------------------------------------------------------------------------
def _sq_budget(q, levels, sigma, g):
    d = (q[..., None] - levels) ** 2
    phi = torch.softmax(-sigma * d, -1)
    cbar = (phi * levels).sum(-1, keepdim=True)
    L = levels.numel()
    dcbar = (L + 2) * U * (phi * levels.abs()).sum(-1, keepdim=True)
    dev = (levels - cbar).abs()
    t = phi * (dev ** 2 * (6 * U * (1 + sigma * d) + L * U) + 2 * dev * dcbar)
    val = soft_quantize_grad64(q, levels, sigma, g)
    return 2 * (2 * sigma * g.abs() * t.sum(-1) + val.abs() * (L + 4) * U)


@pytest.mark.gpu
def test_soft_quantizer_symbols_values_and_gradient():
    from l3c_pytorch_b200 import engine as E
    ties, others = quantiser_inputs()
    lv = _cr_levels()
    finite = others[np.isfinite(others) & (np.abs(others) < 1e18)]
    rng = np.random.default_rng(9)
    vals = np.concatenate([np.concatenate(ties), finite, rng.uniform(-1.2, 1.2, 20000).astype(F32),
                           np.array([np.inf, -np.inf, 3.4e38, -3.4e38], F32)])
    q = torch.from_numpy(rng.permutation(vals).astype(F32)).reshape(2, 1, 1, -1).cuda()
    levels = torch.from_numpy(lv).cuda()
    sym, val = E.soft_quantize(q.contiguous(), levels, 2.0)
    want = torch.min(torch.pow(q.unsqueeze(-1) - levels, 2), -1)[1]            # torch.min on CUDA
    assert sym.dtype == torch.int64 and torch.equal(sym, want)
    assert torch.equal(val, levels[want])
    n_ties = sum(len(t) for t in ties)
    assert n_ties >= 6
    fin = torch.isfinite(q) & (q.abs() < 10)
    gq = torch.from_numpy(rng.normal(0, 1, q.shape).astype(F32)).cuda()
    for sigma in (2.0, 0.5, 40.0):
        dq = E.soft_quantize(q.contiguous(), levels, sigma, grad=gq).double()
        q64, lv64, g64 = q.double()[fin], levels.double(), gq.double()[fin]
        want = soft_quantize_grad64(q64, lv64, sigma, g64)
        budget = _sq_budget(q64, lv64, sigma, g64)
        assert bool(((dq[fin] - want).abs() <= budget).all()), (sigma, float(((dq[fin] - want).abs() / budget).max()))


# ---------------------------------------------------------------------------------------------
# GPU: the whole step
# ---------------------------------------------------------------------------------------------
@pytest.fixture
def strict_fp32():
    """TF32 and non-deterministic cuDNN off for this test only"""
    saved = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic,
             torch.backends.cudnn.benchmark)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic,
     torch.backends.cudnn.benchmark) = saved


def _step(fused, imgs):
    from l3c_pytorch_b200 import MultiscaleBlueprint, config, train
    torch.manual_seed(0)
    bp = MultiscaleBlueprint(config.ms_config('cr'), device='cuda:0')
    bp.net.float()
    bp.net.train()
    opt = train.make_optimizer(bp)
    saved = train.FUSED_LOSS
    train.FUSED_LOSS = fused
    try:
        bp.net.zero_grad()
        loss, bpsps = train.training_loss(bp, imgs)
        loss.backward()
        grads = {k: p.grad.detach().clone() for k, p in bp.net.named_parameters() if p.grad is not None}
        opt.step()
    finally:
        train.FUSED_LOSS = saved
    params = {k: p.detach().clone() for k, p in bp.net.named_parameters()}
    return float(loss), bpsps, grads, params, opt.defaults


@pytest.mark.gpu
def test_fused_step_equals_the_torch_loss_step_and_the_reference(strict_fp32):
    """The fused and the torch-loss step: loss and bpsp to 1e-5 relative; the gradient of all parameters to 1e-5 of its
    norm and of every tensor to 1e-4 of the tensor's norm (measured on an H100: 7e-7 and 2e-6); after one RMSprop step,
    every parameter whose gradient is not small (|g| > 1e-3 max |g| of its tensor, so the step's sign is settled) to
    1e-6.  The fused step also meets the reference's golden step at test_train_step.py's tolerances."""
    from tests import util
    imgs = torch.stack([util.make_image(i, 32, 32) for i in range(2)]).float().cuda()
    lf, bf, gf, pf, _ = _step(True, imgs)
    lt, bt, gt, pt, od = _step(False, imgs)
    assert abs(lf - lt) <= 1e-5 * abs(lt)
    np.testing.assert_allclose(bf, bt, rtol=1e-5)
    assert gf.keys() == gt.keys() and len(gf) > 50
    rel = {k: float((gf[k] - gt[k]).norm()) / max(float(gt[k].norm()), 1e-30) for k in gt}
    total = float(torch.sqrt(sum(((gf[k] - gt[k]) ** 2).sum() for k in gt)))
    total_t = float(torch.sqrt(sum((v ** 2).sum() for v in gt.values())))
    worst = sorted(rel.items(), key=lambda kv: -kv[1])[:3]
    print('fused vs torch loss: gradient difference %.2e of the total norm; worst tensors %s'
          % (total / total_t, ', '.join('%s %.2e' % kv for kv in worst)))
    assert total <= 1e-5 * total_t
    for k in gt:
        assert rel[k] <= 1e-4, (k, rel[k])
        settled = gt[k].abs() > 1e-3 * gt[k].abs().max()
        assert float((pf[k] - pt[k])[settled].abs().max()) <= 1e-6, k
    with open(os.path.join(os.path.dirname(__file__), 'golden', 'train_step.json')) as f:
        gold = json.load(f)
    assert abs(lf - gold['loss_pc']) < 2e-4 * gold['loss_pc']
    np.testing.assert_allclose(bf, gold['nonrecursive_bpsps'], rtol=2e-4)
    for k, want in gold['grad_norms'].items():
        got = float(gf[k].norm())
        assert abs(got - want) < 2e-3 * want + 1e-7, (k, got, want)
    total = float(torch.sqrt(sum((v ** 2).sum() for v in gf.values())))
    assert abs(total - gold['total_grad_norm']) < 2e-3 * gold['total_grad_norm']
    for k, want in gold['params_after_step'].items():
        np.testing.assert_allclose(pf[k].flatten()[:4].cpu().numpy(), want, rtol=1e-3, atol=2e-5)


def loss_inputs(N=30, S=128, seed=0):
    """the loss subgraph of a cr step at N x 3 x S x S: leaf predictions of the three scales, the to_q outputs of
    the three quantisers and the image"""
    gen = torch.Generator(device='cuda').manual_seed(seed)
    img = (torch.rand(N, 3, S, S, device='cuda', generator=gen) * 255).round()
    preds = [(torch.randn(N, 120, S, S, device='cuda', generator=gen)),
             torch.randn(N, 150, S // 2, S // 2, device='cuda', generator=gen),
             torch.randn(N, 150, S // 4, S // 4, device='cuda', generator=gen)]
    qs = [torch.randn(N, 5, S // 2 ** (i + 1), S // 2 ** (i + 1), device='cuda', generator=gen) * 0.6
          for i in range(3)]
    return img, [p.requires_grad_(True) for p in preds], [q.requires_grad_(True) for q in qs]


def loss_pass(img, preds, qs):
    """the three DMLL terms and the three quantisers, forward and backward, as training_loss runs them"""
    from l3c_pytorch_b200 import config, train
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    cfg = config.ms_config('cr')
    levels = torch.linspace(-1, 1, 25, device='cuda')
    bns = [train.soft_quantize(q, levels, cfg.q.sigma)[0] for q in qs]
    rgb, bn = DiscretizedMixLogisticLoss(True), DiscretizedMixLogisticLoss(False, -1, 1, 25)
    total = train.dmll_nll_sum(rgb, img, preds[0])
    for s in (1, 2):
        total = total + train.dmll_nll_sum(bn, bns[s - 1], preds[s])
    (total / (np.log(2.) * img.numel()) + 0 * bns[2].sum()).backward()
    return total


@pytest.mark.gpu
def test_fused_loss_peak_memory_is_below_the_torch_path():
    from l3c_pytorch_b200 import train
    img, preds, qs = loss_inputs()
    peaks = {}
    for fused in (True, False):
        train.FUSED_LOSS = fused
        try:
            for t in preds + qs:
                t.grad = None
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            loss_pass(img, preds, qs)
            torch.cuda.synchronize()
            peaks[fused] = torch.cuda.max_memory_allocated() - base
        finally:
            train.FUSED_LOSS = True
    print('loss forward + backward at 30 x 128^2: peak %.0f MB fused, %.0f MB torch'
          % (peaks[True] / 2 ** 20, peaks[False] / 2 ** 20))
    assert peaks[True] < peaks[False]


# ---------------------------------------------------------------------------------------------
# refusals and the CPU path
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals_and_the_cpu_path():
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200 import train
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    rgb, bn = DiscretizedMixLogisticLoss(True), DiscretizedMixLogisticLoss(False, -1, 1, 25)
    img = torch.rand(2, 3, 9, 7, device='cuda') * 255
    l = torch.randn(2, 120, 9, 7, device='cuda')
    with pytest.raises(ValueError, match='require'):
        train.dmll_nll_sum(rgb, img.clone().requires_grad_(True), l)
    with pytest.raises(ValueError, match='Kp'):
        train.dmll_nll_sum(rgb, img, l[:, :90])
    with pytest.raises(ValueError, match='Kp'):
        train.dmll_nll_sum(bn, torch.zeros(2, 5, 9, 7, device='cuda'), torch.randn(2, 140, 9, 7, device='cuda'))
    with pytest.raises(TypeError, match='fp32'):
        train.dmll_nll_sum(rgb, img.half(), l.half())
    with pytest.raises(TypeError, match='fp32'):
        train.dmll_nll_sum(rgb, img.double(), l.double())
    with pytest.raises(TypeError, match='fp32'):
        train.soft_quantize(torch.zeros(1, 5, 4, 4, device='cuda', dtype=torch.float16),
                            torch.linspace(-1, 1, 25, device='cuda'), 2.0)
    with pytest.raises(ValueError, match='devices'):
        train.dmll_nll_sum(rgb, img.cpu(), l)
    # CPU tensors: the torch restatement, no kernel
    E.launch_log(reset=True)
    lc, xc = l.cpu(), img.round().cpu()
    assert torch.equal(train.dmll_nll_sum(rgb, xc, lc), train.dmll_nll(rgb, xc, lc).sum())
    q = torch.randn(1, 5, 4, 4)
    lev = torch.linspace(-1, 1, 25)
    a, b = train.soft_quantize(q, lev, 2.0), train.soft_quantize_torch(q, lev, 2.0)
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    assert E.launch_log(reset=True)[1] == 0
