"""The DMLL head's loss, sampling and quantiser kernels, sub-pixel by sub-pixel, against float64 restatements of the
reference (criterion/logistic_mixture.py:146-207, 277-323, 334-345; modules/quantizer.py:72-83).

* `nll64` is the reference's NLL in float64 on the kernel's fp32 inputs, with its clamps and edge branches as written.
  The fp32 formula is ill-conditioned wherever sigma(plus) - sigma(min) cancels (the reference shares that), so every
  sub-pixel carries its own error budget derived from the conditioning (`_nll_budget`).  A CPU self-test checks the
  budget against a numpy-float32 emulation of the kernel's formula and checks that it is not vacuous.
* Parameter families that are built to reach one regime each (edge bins, the -7 log-scale clamp, the 1e-12 clamp of
  cdf_delta, the softplus threshold, extreme logits, saturated R/G coupling) go through l3c_dmll_nll with the
  per-sub-pixel map; every family asserts how many sub-pixels it puts into its regime.
* The reduction (CTA partials, tails of HW % 128, the finish kernel, ragged extents) against float64 sums, and the
  bpsp accounting of get_loss / get_loss_per_image against nll64 of the network's own parameters.
* The quantiser on exact fp32 ties, values beyond both ends and non-finite values, against torch.min of the reference,
  with no allowance for flips.
* Sampling at the limits of u, of the log-scales and of the coefficients, with every clamp taken and exact Gumbel
  ties, against a float64 restatement with a propagated budget."""
import math

import numpy as np
import pytest
import torch

U = 2.0 ** -24                  # unit roundoff of fp32
K = 10
F32 = np.float32
LOG_CLAMP = math.log(float(F32(1e-12)))    # the reference clamps an fp32 cdf_delta at 1e-12 (as fp32)


# ---------------------------------------------------------------------------------------------
# value grids
# ---------------------------------------------------------------------------------------------
class Grid:
    """The symbol grid of one DMLL: RGB (0..255, L = 256, R/G coupling) or the bottleneck (linspace(-1, 1, 25),
    C = 5, no coupling).  `values` are the kernel's symbol values (DiscretizedMixLogisticLoss.values)."""

    def __init__(self, rgb, C, x_min, x_max, L):
        self.rgb, self.C, self.x_min, self.x_max, self.L = rgb, C, x_min, x_max, L
        self.P = 4 if rgb else 3
        self.bw = (x_max - x_min) / (L - 1)
        self.values = torch.linspace(x_min, x_max, L, dtype=torch.float32).numpy()
        self.name = 'rgb' if rgb else 'bottleneck'


RGB = Grid(True, 3, 0, 255, 256)
BN = Grid(False, 5, -1, 1, 25)
GRIDS = {'rgb': RGB, 'bottleneck': BN}


def _sig64(v):
    return np.exp(-np.logaddexp(0.0, -v))


def _softplus64(v):
    """torch.nn.functional.softplus (threshold 20), in float64"""
    return np.where(v > 20, v, np.logaddexp(0.0, np.minimum(v, 20.0)))


def _lse(v, axis=-1):
    m = v.max(axis, keepdims=True)
    return (m + np.log(np.exp(v - m).sum(axis, keepdims=True))).squeeze(axis)


# ---------------------------------------------------------------------------------------------
# NLL: float64 restatement, error budget, fp32 emulation of the kernel
# ---------------------------------------------------------------------------------------------
def nll64(l, x, g):
    """logistic_mixture.py:146-207 in float64 on fp32 inputs.  l [P, Kp] fp32 parameters of P pixels (the kernel's
    NHWC layout: plane, channel, component), x [P, C] fp32 values of the symbols.  -> dict of float64 arrays:
    nll [P, C], budget [P, C] (_nll_budget) and the per-component quantities [P, C, K] the families check."""
    P, C = x.shape
    lp = l.astype(np.float64).reshape(P, g.P, C, K)
    x64 = x.astype(np.float64)
    logit, mean, ls_raw = lp[:, 0], lp[:, 1], lp[:, 2]
    ls = np.maximum(ls_raw, -7.0)
    mu = mean.copy()
    eps_mu = np.zeros_like(mean)          # rounding of the coupled fp32 mean (absolute)
    if g.rgb:
        co = _sig64(lp[:, 3])             # [P, 3, K]: lambda_gr, lambda_br, lambda_bg
        t_gr = co[:, 0] * x64[:, 0:1]
        t_br, t_bg = co[:, 1] * x64[:, 0:1], co[:, 2] * x64[:, 1:2]
        mu[:, 1] += t_gr
        mu[:, 2] += t_br + t_bg
        eps_mu[:, 1] = 4 * U * (np.abs(mean[:, 1]) + t_gr)
        eps_mu[:, 2] = 4 * U * (np.abs(mean[:, 2]) + t_br + t_bg)
    half = (g.x_max - g.x_min) / (g.L - 1) / 2
    inv = np.exp(-ls)
    cx = x64[:, :, None] - mu
    a, b = inv * (cx + half), inv * (cx - half)          # plus_in, min_in
    sp_a, sp_b = np.logaddexp(0.0, a), np.logaddexp(0.0, b)
    with np.errstate(divide='ignore'):
        log_delta = np.log(-np.expm1(b - a)) + (a - sp_a) - sp_b     # log(sigma(a) - sigma(b)), stably
    out_a = np.maximum(log_delta, LOG_CLAMP)
    x32 = x.astype(F32)[:, :, None]
    hi = np.broadcast_to(x32 > F32(g.x_max) - F32(0.001), a.shape)
    lo = np.broadcast_to(x32 < F32(g.x_min) + F32(0.001), a.shape)
    lp_k = np.where(hi, -_softplus64(b), out_a)
    lp_k = np.where(lo, a - _softplus64(a), lp_k)
    lse_logit = _lse(logit)
    w = lp_k + (logit - lse_logit[..., None])
    nll = -_lse(w)
    r = np.exp(w + nll[..., None])                        # posterior weight of every component
    d = dict(nll=nll, a=a, b=b, lp=lp_k, log_delta=log_delta, lo=lo, hi=hi, ls_raw=ls_raw, inv=inv, cx=cx,
             eps_mu=eps_mu, r=r, logit=logit, lse_logit=lse_logit)
    d['budget'] = _nll_budget(d)
    return d


def _nll_budget(d):
    """Error budget of one sub-pixel of the fp32 NLL (kernel or reference) against nll64.
    Per component k, with delta_k = sigma(a_k) - sigma(b_k) in float64, the fp32 difference of the two sigmoids is off
    by a relative z_k = 4u (sigma(a_k) + sigma(b_k)) / max(delta_k, 1e-12) -- plus the absolute error of the
    arguments moved through the sigmoids' slopes, inv_k t_k (sigma'(a_k) + sigma'(b_k)) / max(delta_k, 1e-12), where
    t_k = 2u |x - mu_k| + eps_mu_k is the rounding of x - mu (which cx +- half can cancel) and, where the mean is
    coupled to R / G, of the fp32 mean -- and log max(delta_k, 1e-12) by 8u (1 + |log max(delta_k, 1e-12)|) from the
    relative rounding of the arguments.  To first order that is e_k = z_k + 8u (1 + |log max(delta_k, 1e-12)|); here z_k enters as log(1 + z_k) upwards
    and -log(1 - z_k) downwards, and neither side passes the clamp at 1e-12 or log 1 = 0.  On an edge branch the
    component's value is log sigma(a) or -softplus(b), well-conditioned: e_k = 8u (1 + |lp_k| + |arg_k| s_k) +
    inv_k t_k s_k, s_k = sigma(-a_k) or sigma(b_k) its slope.  The mixture moves by at most log sum_k r_k exp(+-e_k),
    r_k the posterior weight softmax_k(lp_k + log pi_k) -- to first order sum_k r_k e_k -- and the fp32 log-softmax
    of the logits and log-sum-exp of the mixture add 2u sum_k r_k (|logit_k| + |lse(logit)|) + 16u (1 + |nll|)."""
    a, b = d['a'], d['b']
    sa, sb = _sig64(a), _sig64(b)
    dmax = np.maximum(np.exp(d['log_delta']), 1e-12)
    shift = d['inv'] * (2 * U * np.abs(d['cx']) + d['eps_mu'])
    z = (4 * U * (sa + sb) + shift * (sa * (1 - sa) + sb * (1 - sb))) / dmax
    arg_err = 8 * U * (1 + np.abs(np.log(dmax)))
    down = np.minimum(-np.log1p(-np.minimum(z, 1 - 1e-16)), np.log(dmax) - LOG_CLAMP) + arg_err
    up = np.minimum(np.log1p(z), -np.log(dmax)) + arg_err
    arg = np.where(d['lo'], a, b)
    slope = np.where(d['lo'], 1 - sa, sb)             # |d lp / d arg| on the edge branch
    e_edge = 8 * U * (1 + np.abs(d['lp']) + np.abs(arg) * slope) + shift * slope
    edge = d['lo'] | d['hi']
    up, down = np.where(edge, e_edge, up), np.where(edge, e_edge, down)
    r = d['r']
    b_up = np.log1p((r * np.expm1(up)).sum(-1))
    b_down = -np.log1p((r * np.expm1(-down)).sum(-1))
    e_pi = 2 * U * (r * (np.abs(d['logit']) + np.abs(d['lse_logit'])[..., None])).sum(-1)
    return np.maximum(b_up, b_down) + e_pi + 16 * U * (1 + np.abs(d['nll']))


def _sig32(v):
    return F32(1) / (F32(1) + np.exp(-v))


def _softplus32(v):
    return np.where(v > F32(20), v, np.log1p(np.exp(v)))


def nll32_emulated(l, x, g):
    """The kernel's formula (dmll.cu, dmll_nll_kernel) in numpy float32: -> (nll [P, C], cdf_delta [P, C, K])."""
    P, C = x.shape
    lp = l.astype(F32).reshape(P, g.P, C, K)
    half = F32((g.x_max - g.x_min) / (g.L - 1) / 2.0)
    hi_t, lo_t = F32(g.x_max) - F32(0.001), F32(g.x_min) + F32(0.001)
    out = np.empty((P, C), F32)
    delta = np.empty((P, C, K), F32)
    with np.errstate(over='ignore', under='ignore', divide='ignore', invalid='ignore'):
        for c in range(C):
            xc = x[:, c]
            logit, mean, logs = lp[:, 0, c], lp[:, 1, c], lp[:, 2, c]
            lmax = logit.max(1)
            lsum = np.zeros(P, F32)
            for k in range(K):
                lsum = lsum + np.exp(logit[:, k] - lmax)
            lse = lmax + np.log(lsum)
            w = np.empty((P, K), F32)
            for k in range(K):
                mu = mean[:, k]
                if g.rgb and c == 1:
                    mu = mu + _sig32(lp[:, 3, 0, k]) * x[:, 0]
                if g.rgb and c == 2:
                    mu = mu + (_sig32(lp[:, 3, 1, k]) * x[:, 0] + _sig32(lp[:, 3, 2, k]) * x[:, 1])
                inv = np.exp(-np.maximum(logs[:, k], F32(-7)))
                cx = xc - mu
                pin, mn = inv * (cx + half), inv * (cx - half)
                delta[:, c, k] = _sig32(pin) - _sig32(mn)
                v = np.log(np.maximum(delta[:, c, k], F32(1e-12)))
                v = np.where(xc > hi_t, -_softplus32(mn), v)
                v = np.where(xc < lo_t, pin - _softplus32(pin), v)
                w[:, k] = v + (logit[:, k] - lse)
            wmax = w.max(1)
            s = np.zeros(P, F32)
            for k in range(K):
                s = s + np.exp(w[:, k] - wmax)
            out[:, c] = -(wmax + np.log(s))
    return out, delta


# ---------------------------------------------------------------------------------------------
# parameter families
# ---------------------------------------------------------------------------------------------
def _pack(g, logit, mu_eff, ls, co, sym):
    """l [P, Kp] fp32 from the per-component logits, EFFECTIVE means (after the R / G coupling), log-scales
    [P, C, K] and coefficient logits [P, 3, K]; the raw means are what gives mu_eff with the coded R / G values."""
    x = g.values[sym].astype(np.float64)
    mean = mu_eff.copy()
    if g.rgb:
        s = _sig64(co.astype(F32).astype(np.float64))
        mean[:, 1] -= s[:, 0] * x[:, 0:1]
        mean[:, 2] -= s[:, 1] * x[:, 0:1] + s[:, 2] * x[:, 1:2]
        planes = [logit, mean, ls, co]
    else:
        planes = [logit, mean, ls]
    return np.stack(planes, 1).reshape(len(sym), -1).astype(F32)


def _interior(g, rng, shape):
    return rng.integers(1, g.L - 1, shape)


def _base(g, rng, P):
    """random-init-like components around the coded value: the families overwrite what they are about"""
    C = g.C
    sym = rng.integers(0, g.L, (P, C))
    x = g.values[sym].astype(np.float64)
    logit = rng.normal(0, 2, (P, C, K))
    mu = x[..., None] + rng.choice([-1, 1], (P, C, K)) * g.bw * np.exp(rng.uniform(-4, 5, (P, C, K)))
    ls = rng.uniform(-8, 4, (P, C, K))
    co = rng.normal(0, 3, (P, 3, K))
    return sym, logit, mu, ls, co


def _fam_random(g, rng, P):
    sym, logit, mu, ls, co = _base(g, rng, P)
    return sym, _pack(g, logit, mu, ls, co, sym), {}


def _fam_edge(g, rng, P):
    """x exactly at x_min and x_max and one bin inside each, components within a few bins of x"""
    sym, logit, mu, ls, co = _base(g, rng, P)
    sym = rng.choice([0, 1, g.L - 2, g.L - 1], (P, g.C))
    x = g.values[sym].astype(np.float64)
    mu = x[..., None] + g.bw * rng.normal(0, 1.5, mu.shape)
    ls = math.log(g.bw) + rng.uniform(-3, 1.5, ls.shape)
    return sym, _pack(g, logit, mu, ls, co, sym), {}


def _dominant(rng, P, C, hi=8.0, others=None):
    """one dominant component per sub-pixel: (index [P, C], logits [P, C, K])"""
    k0 = rng.integers(0, K, (P, C))
    logit = rng.normal(0, 1, (P, C, K)) if others is None else np.full((P, C, K), others)
    np.put_along_axis(logit, k0[..., None], hi, axis=2)
    return k0, logit


def _set(arr, k0, v):
    np.put_along_axis(arr, k0[..., None], np.asarray(v)[..., None], axis=2)


def _fam_ls_clamp(g, rng, P):
    """the dominant component's log-scale below -7, exactly -7, or large (sigma >> the range); the two small
    classes put the bin edge within a few clamped sigmas of the mean"""
    sym, _, mu, ls, co = _base(g, rng, P)
    sym = _interior(g, rng, (P, g.C))
    x = g.values[sym].astype(np.float64)
    k0, logit = _dominant(rng, P, g.C)
    cls = rng.integers(0, 3, (P, g.C))
    l0 = np.where(cls == 0, rng.uniform(-12, -7.05, cls.shape), np.where(cls == 1, -7.0, rng.uniform(3, 6, cls.shape)))
    off = rng.choice([-1, 1], cls.shape) * (g.bw / 2 + rng.uniform(0.3, 3, cls.shape) * math.exp(-7))
    off = np.where(cls == 2, rng.normal(0, 3, cls.shape) * g.bw, off)
    _set(ls, k0, l0)
    _set(mu, k0, x + off)
    return sym, _pack(g, logit, mu, ls, co, sym), dict(k0=k0, cls=cls)


def _fam_tail(g, rng, P, right):
    """1..3 components (logits in [-2, 2]) far in one tail of x, the others at logit -80.  Right tail
    (x >= mu + half + 18 sigma): both fp32 sigmoids round to 1, cdf_delta is 0 and the clamp decides.  Left tail
    (x <= mu - half - 18 sigma, sigma <= one bin): no cancellation, delta >= 1e-11."""
    sym, _, mu, ls, co = _base(g, rng, P)
    C = g.C
    sym = _interior(g, rng, (P, C))
    x = g.values[sym].astype(np.float64)
    logit = np.full((P, C, K), -80.0)
    n_s = rng.integers(1, 4, (P, C))
    sel = np.argsort(rng.random((P, C, K)), axis=2) < n_s[..., None]        # the chosen components
    logit = np.where(sel, rng.uniform(-2, 2, logit.shape), logit)
    if right:
        lsk = rng.uniform(-7, math.log(g.bw) + 1, ls.shape)
        t = rng.uniform(18, 40, ls.shape)
        mu_t = x[..., None] - g.bw / 2 - t * np.exp(lsk)
    else:
        lsk = rng.uniform(max(-7.0, math.log(g.bw) - 1.5), math.log(g.bw), ls.shape)
        t = rng.uniform(18, 24, ls.shape)
        mu_t = x[..., None] + g.bw / 2 + t * np.exp(lsk)
    ls = np.where(sel, lsk, ls)
    mu = np.where(sel, mu_t, mu)
    return sym, _pack(g, logit, mu, ls, co, sym), dict(sel=sel)


def _fam_softplus(g, rng, P):
    """x on an edge bin, the dominant component's softplus argument (min_in at x_max, plus_in at x_min) in
    [19, 21]: both sides of the threshold 20"""
    sym, _, mu, ls, co = _base(g, rng, P)
    sym = rng.choice([0, g.L - 1], (P, g.C))
    x = g.values[sym].astype(np.float64)
    k0, logit = _dominant(rng, P, g.C, hi=0.0, others=-40.0)
    s = np.exp(rng.uniform(-5, 0, k0.shape)) * g.bw
    t = rng.uniform(19, 21, k0.shape)
    # x_max: min_in = (x - mu - half) / s = t;  x_min: plus_in = (x - mu + half) / s = t
    _set(mu, k0, np.where(sym == g.L - 1, x - g.bw / 2 - t * s, x + g.bw / 2 - t * s))
    _set(ls, k0, np.log(s))
    return sym, _pack(g, logit, mu, ls, co, sym), dict(k0=k0)


def _fam_logits(g, rng, P):
    """logits spread over 100 (pi underflows in fp32) or all ten equal"""
    sym, logit, mu, ls, co = _base(g, rng, P)
    spread = rng.random((P, g.C)) < 0.5
    wide = rng.uniform(-50, 50, logit.shape)
    ends = np.argsort(rng.random((P, g.C, K)), axis=2)
    np.put_along_axis(wide, ends[..., :1], 50.0, axis=2)
    np.put_along_axis(wide, ends[..., 1:2], -50.0, axis=2)
    equal = np.broadcast_to(np.where(rng.random((P, g.C, 1)) < 0.3, 0.0, rng.uniform(-30, 30, (P, g.C, 1))),
                            logit.shape)
    logit = np.where(spread[..., None], wide, equal)
    return sym, _pack(g, logit, mu, ls, co, sym), dict(spread=spread)


def _fam_coupling(g, rng, P):
    """RGB: coefficient logits at -30, 0 and +30, a different one per plane, R / G coded at 0 or 255 (mostly
    different), narrow components around the coupled means"""
    assert g.rgb
    sym, logit, mu, ls, co = _base(g, rng, P)
    choice = rng.permuted(np.broadcast_to(np.array([-30.0, 0.0, 30.0])[:, None], (P, 3, K)).copy(), axis=1)
    co = choice
    rg = rng.choice([0, 255], (P, 2))
    rg[:, 1] = np.where(rng.random(P) < 0.75, 255 - rg[:, 0], rg[:, 1])
    sym[:, :2] = np.where(rng.random((P, 1)) < 0.8, rg, sym[:, :2])
    sym[:, 2] = _interior(g, rng, P)
    x = g.values[sym].astype(np.float64)
    mu = x[..., None] + g.bw * rng.normal(0, 2, mu.shape)
    ls = rng.uniform(-3, 1, ls.shape)
    return sym, _pack(g, logit, mu, ls, co, sym), dict(co=co)


def _fam_mix(g, rng, P):
    """trained-like mixtures (peaked, broad, mixed) of the coarse-row tests"""
    from tests.test_gpu_coarse_rows import _params
    ls_, syms = [], []
    for kind in ('peaked', 'broad', 'mixed'):
        l, sym = _params(kind, rng)              # [N, H, W, Kp], [N, C, HW]
        ls_.append(l.reshape(-1, l.shape[-1]))
        syms.append(sym.transpose(0, 2, 1).reshape(-1, sym.shape[1]))
    return np.concatenate(syms).astype(np.int64), np.concatenate(ls_), {}


FAMILIES = {
    'edge': _fam_edge, 'ls_clamp': _fam_ls_clamp, 'clamp_right': lambda g, r, P: _fam_tail(g, r, P, True),
    'clamp_left': lambda g, r, P: _fam_tail(g, r, P, False), 'softplus': _fam_softplus, 'logits': _fam_logits,
    'coupling': _fam_coupling, 'mix': _fam_mix, 'random': _fam_random}
FAMILY_CASES = ([('rgb', f) for f in FAMILIES if f != 'random'] +
                [('bottleneck', f) for f in FAMILIES if f not in ('coupling', 'mix', 'random')])
FAMILY_PIXELS = 3000


def _family(grid, fam, seed=0):
    g = GRIDS[grid]
    rng = np.random.default_rng(1000 + 17 * seed + sorted(FAMILIES).index(fam) + (50 if g.rgb else 0))
    sym, l, info = FAMILIES[fam](g, rng, FAMILY_PIXELS)
    return g, sym.astype(np.uint8), l, info


def _regimes(g, fam, sym, l, info):
    """-> {regime: number of sub-pixels in it, required minimum}; also the reference's clamp values"""
    x = g.values[sym]
    d = nll64(l, x, g)
    _, delta32 = nll32_emulated(l, x, g)
    out = {}
    if fam == 'edge':
        out['x at x_min'] = (int((sym == 0).sum()), 300)
        out['x at x_max'] = (int((sym == g.L - 1).sum()), 300)
        out['x one bin inside'] = (int(((sym == 1) | (sym == g.L - 2)).sum()), 600)
        out['edge branch taken'] = (int(d['lo'][..., 0].sum() + d['hi'][..., 0].sum()), 600)
    elif fam == 'ls_clamp':
        ls0 = np.take_along_axis(d['ls_raw'], info['k0'][..., None], 2)[..., 0]
        out['log-scale < -7'] = (int((ls0 < -7).sum()), 500)
        out['log-scale == -7'] = (int((ls0 == -7).sum()), 500)
        out['log-scale > 3'] = (int((ls0 > 3).sum()), 500)
    elif fam == 'clamp_right':
        clamped = np.where(info['sel'], delta32 == 0, True).all(-1)
        out['every chosen component clamped in fp32'] = (int(clamped.sum()), clamped.size)
    elif fam == 'clamp_left':
        sel = info['sel']
        tail = np.where(sel, (d['a'] <= -18) & (delta32 > F32(1e-12)) & (d['log_delta'] > LOG_CLAMP), True).all(-1)
        out['every chosen component in the left tail, unclamped'] = (int(tail.sum()), tail.size)
    elif fam == 'softplus':
        k0 = info['k0'][..., None]
        arg = np.where(sym == 0, np.take_along_axis(d['a'], k0, 2)[..., 0], np.take_along_axis(d['b'], k0, 2)[..., 0])
        out['softplus argument in (19, 20]'] = (int(((arg > 19) & (arg <= 20)).sum()), 500)
        out['softplus argument in (20, 21)'] = (int(((arg > 20) & (arg < 21)).sum()), 500)
    elif fam == 'logits':
        spread = d['logit'].max(-1) - d['logit'].min(-1)
        out['logits spread >= 100'] = (int((spread >= 100).sum()), 1000)
        out['ten equal logits'] = (int((spread == 0).sum()), 1000)
    elif fam == 'coupling':
        co = info['co']
        distinct = (co[:, 0] != co[:, 1]) & (co[:, 1] != co[:, 2]) & (co[:, 0] != co[:, 2])
        out['three different coefficient planes'] = (int(distinct.all(-1).sum()), co.shape[0])
        for v in (-30.0, 0.0, 30.0):
            out['coefficient logit %g' % v] = (int((co == v).sum()), 5000)
        out['R at 0 or 255'] = (int(np.isin(sym[:, 0], (0, 255)).sum()), 1500)
        out['G at 0 or 255'] = (int(np.isin(sym[:, 1], (0, 255)).sum()), 1500)
        out['R != G'] = (int((sym[:, 0] != sym[:, 1]).sum()), 1500)
    elif fam == 'mix':
        out['sub-pixels'] = (d['nll'].size, 3 * 960 * 3)
    return out, d


def _assert_within(got, d, what):
    got = np.asarray(got, np.float64)
    err = np.abs(got - d['nll'])
    ok = err <= d['budget']
    if not ok.all():
        i = np.unravel_index(np.argmax(np.where(ok, 0, err / d['budget'])), got.shape)
        raise AssertionError('%s: %d of %d sub-pixels outside their budget; worst at %s: got %r, nll64 %r, budget %.3g'
                             % (what, int((~ok).sum()), ok.size, i, float(got[i]), float(d['nll'][i]),
                                float(d['budget'][i])))
    return float((err / d['budget']).max())


# ---------------------------------------------------------------------------------------------
# CPU: the references and the budget
# ---------------------------------------------------------------------------------------------
def test_nll64_restates_the_reference_formula():
    """where nothing cancels, nll64 equals the naive float64 formula of the reference; on the edge bins it takes
    the edge branches, and a clamped component contributes log(1e-12)"""
    g = RGB
    rng = np.random.default_rng(3)
    sym, l, _ = _fam_random(g, rng, 2000)
    x = g.values[sym]
    d = nll64(l, x, g)
    lp = l.astype(np.float64).reshape(len(x), 4, 3, K)
    mu = lp[:, 1].copy()
    co = 1 / (1 + np.exp(-lp[:, 3]))
    mu[:, 1] += co[:, 0] * x[:, 0:1]
    mu[:, 2] += co[:, 1] * x[:, 0:1] + co[:, 2] * x[:, 1:2]
    inv = np.exp(-np.maximum(lp[:, 2], -7))
    cx = x[..., None] - mu
    with np.errstate(over='ignore', divide='ignore'):
        a, b = inv * (cx + 0.5), inv * (cx - 0.5)
        delta = 1 / (1 + np.exp(-a)) - 1 / (1 + np.exp(-b))
        naive = np.log(np.maximum(delta, 1e-12))
    edge = (x[..., None] > 254.999) | (x[..., None] < 0.001)
    naive = np.where(x[..., None] > 254.999, -np.logaddexp(0, b), naive)
    naive = np.where(x[..., None] < 0.001, a - np.logaddexp(0, a), naive)
    well = (delta > 1e-3) | edge | (delta < 1e-13)          # no cancellation, an edge branch, or the clamp
    assert well.mean() > 0.5 and (delta < 1e-13).sum() > 1000 and edge.sum() > 20
    np.testing.assert_allclose(d['lp'][well], naive[well], rtol=1e-9, atol=3e-9)   # softplus threshold: e^-20
    assert (d['lp'][~edge & (delta < 1e-13)] == LOG_CLAMP).all()
    logpi = lp[:, 0] - _lse(lp[:, 0])[..., None]
    all_well = well.all(-1)
    assert all_well.sum() > 100
    np.testing.assert_allclose(d['nll'][all_well], -_lse(naive + logpi)[all_well], rtol=1e-9, atol=3e-9)


def test_nll_budget_covers_the_fp32_formula_and_is_not_vacuous():
    """The budget against a numpy-float32 emulation of the kernel's formula: >= 10^5 random sub-pixels with
    log-scales in [-8, 4] and means up to e^5 bins from x on both grids, and every family.  Every sub-pixel stays
    inside its budget; on the well-conditioned ones (no cancellation, no coupling, logits within +-20) the budget stays below
    1e-5 (1 + |nll|), so it cannot hide a real error."""
    worst, n_sub, well_worst, n_well, n_random, edge_err = 0.0, 0, 0.0, 0, 0, 0.0
    cases = [(grid, 'random', s) for grid in GRIDS for s in range(4)] + [(g, f, 0) for g, f in FAMILY_CASES]
    for grid, fam, seed in cases:
        g = GRIDS[grid]
        rng = np.random.default_rng(500 + seed + (50 if g.rgb else 0))
        if fam == 'random':
            sym, l, _ = _fam_random(g, rng, 20000 if g.rgb else 12000)
        else:
            g, sym, l, _ = _family(grid, fam)
        x = g.values[sym]
        d = nll64(l, x, g)
        got, _ = nll32_emulated(l, x, g)
        worst = max(worst, _assert_within(got, d, '%s/%s emulated' % (grid, fam)))
        n_sub += got.size
        err = np.abs(got - d['nll'])
        # condition number of log delta in the sigmoids and in x - mu, weighted by the posterior
        sa, sb = _sig64(d['a']), _sig64(d['b'])
        cond = (sa + sb + d['inv'] * np.abs(d['cx']) * (sa * (1 - sa) + sb * (1 - sb))) / np.maximum(
            np.exp(d['log_delta']), 1e-12)
        well = (((d['r'] * np.where(d['lo'] | d['hi'], 0, cond)).sum(-1) < 4) & (d['eps_mu'].max(-1) == 0)
                & (np.abs(d['logit']).max(-1) <= 20))
        edge = (d['lo'] | d['hi']).any(-1)
        rel = d['budget'] / (1 + np.abs(d['nll']))
        assert (rel[well] < 1e-5).all(), (grid, fam, float(rel[well].max()))
        if well.any():
            well_worst = max(well_worst, float((err / (1 + np.abs(d['nll'])))[well].max()))
        if fam == 'random':
            n_well += int(well.sum())
            n_random += got.size
        if edge.any():
            edge_err = max(edge_err, float(err[edge].max()))
    print('\nbudget self-test: %d sub-pixels, largest error / budget %.3f; %d of %d random ones well-conditioned, '
          'largest relative error there %.2e; largest error on the edge bins %.2e nats'
          % (n_sub, worst, n_well, n_random, well_worst, edge_err))
    assert n_random >= 10 ** 5 and n_well >= n_random // 10


@pytest.mark.parametrize('grid,fam', FAMILY_CASES)
def test_families_reach_their_regimes(grid, fam):
    g, sym, l, info = _family(grid, fam)
    reg, d = _regimes(g, fam, sym, l, info)
    assert reg
    for name, (n, need) in reg.items():
        assert n >= need, '%s/%s: %d sub-pixels in regime %r, need %d' % (grid, fam, n, name, need)
    assert np.isfinite(d['nll']).all() and np.isfinite(d['budget']).all()
    if fam == 'clamp_right':
        # the fp32 reference prices these sub-pixels at the clamp, float64 partly does not
        want = _clamp_value(d, info['sel'])
        assert (np.abs(want - d['nll']) > 1.0).sum() > 100
        assert (want > -LOG_CLAMP - 1e-9).all()
    if fam == 'clamp_left':
        rel = d['budget'] / (1 + np.abs(d['nll']))
        assert (rel[:, 0] < 1e-5).all(), float(rel[:, 0].max())


def _clamp_value(d, sel):
    """the fp32 reference's value on a clamp_right sub-pixel: every chosen component gives log(1e-12f), the others
    are negligible -> -log(1e-12f) - log(sum of the chosen pi)"""
    logpi = d['logit'] - _lse(d['logit'])[..., None]
    return -LOG_CLAMP - _lse(np.where(sel, logpi, -np.inf))


# ---------------------------------------------------------------------------------------------
# GPU: NLL per sub-pixel
# ---------------------------------------------------------------------------------------------
def _dm(g):
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    return DiscretizedMixLogisticLoss(g.rgb, g.x_min, g.x_max, g.L)


def _kernel_nll(g, l, sym, N=1):
    """l [N * HW, Kp], sym [N * HW, C] -> (out [N] float64, map [N * HW, C])"""
    dm = _dm(g)
    HW = len(sym) // N
    l_dev = torch.from_numpy(l.reshape(N, 1, HW, -1)).cuda()
    s_dev = torch.from_numpy(np.ascontiguousarray(sym.reshape(N, HW, g.C).transpose(0, 2, 1)).reshape(N, g.C, 1, HW))
    out, m = dm.nll_sum(s_dev.cuda(), l_dev, want_map=True)
    m = m.cpu().numpy().reshape(N, g.C, HW).transpose(0, 2, 1).reshape(N * HW, g.C)
    return out.cpu().numpy(), m


@pytest.mark.gpu
@pytest.mark.parametrize('grid,fam', FAMILY_CASES)
def test_nll_map_within_budget_of_float64(grid, fam):
    g, sym, l, info = _family(grid, fam)
    reg, d = _regimes(g, fam, sym, l, info)
    for name, (n, need) in reg.items():
        assert n >= need, (grid, fam, name, n, need)
    out, m = _kernel_nll(g, l, sym)
    worst = _assert_within(m, d, '%s/%s' % (grid, fam))
    print('%s/%s: largest error / budget %.3f' % (grid, fam, worst))
    if fam == 'clamp_right':
        want = _clamp_value(d, info['sel'])
        err = np.abs(m - want)
        assert (err <= 1e-5 * np.abs(want)).all(), ('the clamp value of the fp32 reference', float(err.max()))
    if fam == 'clamp_left':
        # no cancellation in this tail: the kernel follows the float64 value, not a clamp
        rel = np.abs(m - d['nll']) / (1 + np.abs(d['nll']))
        assert (rel[:, 0] < 1e-5).all(), float(rel[:, 0].max())
    assert abs(float(out[0]) - float(m.astype(np.float64).sum())) <= 1e-12 * abs(float(out[0]))


# ---------------------------------------------------------------------------------------------
# GPU: reduction
# ---------------------------------------------------------------------------------------------
def _shape_case(g, HW, N, seed):
    """N different images of HW pixels, every pixel drawn from one of the families"""
    rng = np.random.default_rng(seed)
    fams = [f for f in ('random', 'edge', 'ls_clamp', 'logits', 'softplus', 'coupling') if g.rgb or f != 'coupling']
    P = N * HW
    pick = rng.integers(0, len(fams), P)
    sym = np.zeros((P, g.C), np.int64)
    l = np.zeros((P, g.P * g.C * K), F32)
    for i, f in enumerate(fams):
        idx = np.nonzero(pick == i)[0]
        if len(idx):
            s, lf, _ = FAMILIES[f](g, rng, len(idx))
            sym[idx], l[idx] = s, lf
    return sym.astype(np.uint8), l


def _nll64_chunked(l, x, g, chunk=1 << 15):
    nll, bud = [], []
    for i in range(0, len(x), chunk):
        d = nll64(l[i:i + chunk], x[i:i + chunk], g)
        nll.append(d['nll'])
        bud.append(d['budget'])
    return dict(nll=np.concatenate(nll), budget=np.concatenate(bud))


@pytest.mark.gpu
@pytest.mark.parametrize('grid', ['rgb', 'bottleneck'])
@pytest.mark.parametrize('N', [1, 3])
@pytest.mark.parametrize('HW', [1, 127, 128, 129, 300 * 517])
def test_nll_sums_every_pixel_once(grid, N, HW):
    """out[n] is the float64 sum of the kernel's own map (the CTA partials, the tail of HW % 128 and the finish
    kernel) and lies within the summed budget of the float64 truth"""
    g = GRIDS[grid]
    sym, l = _shape_case(g, HW, N, seed=HW * 7 + N + (1 if g.rgb else 2))
    d = _nll64_chunked(l, g.values[sym], g)
    out, m = _kernel_nll(g, l, sym, N)
    _assert_within(m, d, '%s HW=%d N=%d' % (grid, HW, N))
    per = m.astype(np.float64).reshape(N, HW, g.C)
    truth = d['nll'].reshape(N, HW, g.C).sum((1, 2))
    budget = d['budget'].reshape(N, HW, g.C).sum((1, 2))
    for n in range(N):
        own = per[n].sum()
        assert abs(out[n] - own) <= 1e-12 * abs(own), (n, float(out[n]), own)
        assert abs(out[n] - truth[n]) <= budget[n], (n, float(out[n]), truth[n], budget[n])
    if N > 1:
        assert len(set(out.tolist())) == N             # the images differ


RAGGED_HW = (37, 41)
RAGGED_EXT = [(37, 1), (1, 41), (23, 17), (37, 41), (5, 29)]


@pytest.mark.gpu
@pytest.mark.parametrize('grid', ['rgb', 'bottleneck'])
def test_ragged_nll_equals_per_image_calls_and_float64(grid):
    g = GRIDS[grid]
    H, W = RAGGED_HW
    N = len(RAGGED_EXT)
    dm = _dm(g)
    rng = np.random.default_rng(91 if g.rgb else 92)
    l = np.full((N, H, W, g.P * g.C * K), np.nan, F32)
    sym = np.full((N, g.C, H, W), 255, np.uint8)
    truth, budget = [], []
    for n, (h, w) in enumerate(RAGGED_EXT):
        s, lf = _shape_case(g, h * w, 1, seed=int(rng.integers(1 << 30)))
        l[n, :h, :w] = lf.reshape(h, w, -1)
        sym[n, :, :h, :w] = s.T.reshape(g.C, h, w)
        d = nll64(lf, g.values[s], g)
        truth.append(d['nll'].sum())
        budget.append(d['budget'].sum())
    l_dev, s_dev = torch.from_numpy(l).cuda(), torch.from_numpy(sym).cuda()
    got = dm.nll_sum(s_dev, l_dev, extents=RAGGED_EXT).cpu()
    for n, (h, w) in enumerate(RAGGED_EXT):
        one = dm.nll_sum(s_dev[n:n + 1, :, :h, :w].contiguous(), l_dev[n:n + 1, :h, :w].contiguous()).cpu()
        assert torch.equal(got[n:n + 1], one), (n, float(got[n]), float(one[0]))
        assert abs(float(got[n]) - truth[n]) <= budget[n], (n, float(got[n]), truth[n], budget[n])


# ---------------------------------------------------------------------------------------------
# GPU: the bpsp accounting
# ---------------------------------------------------------------------------------------------
def _scale_nll64(dm, P_nhwc, S_u8, exts=None):
    """per image: (float64 nats, budget) of one scale's parameters and symbols, over each image's extent"""
    g = Grid(dm.rgb_scale, S_u8.shape[1], dm.x_min, dm.x_max, dm.L)
    l, S = P_nhwc.cpu().numpy(), S_u8.cpu().numpy()
    N, C, H, W = S.shape
    out = []
    for n in range(N):
        h, w = exts[n] if exts is not None else (H, W)
        lf = l[n, :h, :w].reshape(h * w, -1)
        sym = S[n, :, :h, :w].reshape(C, h * w).T
        d = nll64(lf, g.values[sym], g)
        out.append((d['nll'].sum(), d['budget'].sum()))
    return np.array(out)


@pytest.mark.gpu
@pytest.mark.parametrize('cfg', ['cr', 'cr_rgb_shared'])
def test_bpsp_accounting_against_float64(cfg):
    """every entry of get_loss(out).nonrecursive_bpsps and get_loss_per_image, recomputed in float64 from the
    network's own parameters and symbols (within the summed budget: at random init the RGB scale has many sub-pixels
    in the fp32 clamp region, so that budget is wide), and exactly, to 1e-12, from the float64 sums of the kernel's
    own per-sub-pixel maps; the final scale costs C h w ln L"""
    from tests import util
    bp = util.blueprint(cfg)
    imgs = torch.stack([util.make_image(60 + i, 64, 48) for i in range(2)]).cuda()
    out = bp.forward(imgs)
    dms = [bp.losses.loss_dmol_rgb] + [bp.losses.loss_dmol_n] * (len(out.P_nhwc) - 1)
    per_scale = [_scale_nll64(dm, out.P_nhwc[s], out.S_u8[s]) for s, dm in enumerate(dms)]
    maps = [dm.nll_sum(out.S_u8[s], out.P_nhwc[s], want_map=True)[1].double().cpu().numpy()
            for s, dm in enumerate(dms)]
    own = [m.reshape(m.shape[0], -1).sum(1) for m in maps]
    N, C, h, w = out.S_u8[-1].shape
    uniform = C * h * w * math.log(bp.losses.loss_dmol_n.L)
    nsub = imgs.numel()
    for n_sub in (None, nsub - 3 * 7 * 48):
        conv = math.log(2.0) * (n_sub or nsub)
        got = bp.get_loss(out, num_subpixels_before_pad=n_sub).nonrecursive_bpsps
        assert len(got) == len(per_scale) + 1
        for s, ps in enumerate(per_scale):
            want, tol = ps[:, 0].sum() / conv, ps[:, 1].sum() / conv
            assert abs(got[s] - want) <= tol, (cfg, s, got[s], want, tol)
            assert abs(got[s] - own[s].sum() / conv) <= 1e-12 * got[s], (cfg, s, got[s], own[s].sum() / conv)
            print('%s scale %d: %.6f bpsp, float64 %.6f, budget %.2e relative' % (cfg, s, got[s], want, tol / want))
        assert abs(got[-1] - N * uniform / conv) <= 1e-14 * got[-1], (got[-1], N * uniform / conv)
    per_img = bp.get_loss_per_image(out)
    conv = math.log(2.0) * nsub / N
    for n in range(N):
        want = (sum(ps[n, 0] for ps in per_scale) + uniform) / conv
        tol = sum(ps[n, 1] for ps in per_scale) / conv
        assert abs(per_img[n] - want) <= tol, (n, per_img[n], want, tol)
        exact = (sum(o[n] for o in own) + uniform) / conv
        assert abs(per_img[n] - exact) <= 1e-12 * exact, (n, per_img[n], exact)


@pytest.mark.gpu
def test_ragged_bpsp_accounting_against_float64():
    from l3c_pytorch_b200 import engine as E
    from tests import util
    shapes = [(32, 32), (48, 24), (16, 40)]
    Hb, Wb = 48, 40
    batch = torch.zeros(len(shapes), 3, Hb, Wb, dtype=torch.uint8)
    for n, (h, w) in enumerate(shapes):
        batch[n, :, :h, :w] = util.make_image(70 + n, h, w)
    bp = util.blueprint('cr')
    old = E.get_conv_precision()
    E.set_conv_precision('f16')
    try:
        out = bp.forward(batch.cuda(), extents=shapes)
    finally:
        E.set_conv_precision(old)
    dms = [bp.losses.loss_dmol_rgb] + [bp.losses.loss_dmol_n] * (len(out.P_nhwc) - 1)
    per_scale = [_scale_nll64(dm, out.P_nhwc[s], out.S_u8[s], out.extents_at(s)) for s, dm in enumerate(dms)]
    own = []             # float64 sums of the kernel's map of every image alone, over its extent
    for s, dm in enumerate(dms):
        own.append([float(dm.nll_sum(out.S_u8[s][n:n + 1, :, :h, :w].contiguous(), out.P_nhwc[s][n:n + 1, :h, :w]
                                     .contiguous(), want_map=True)[1].double().sum())
                    for n, (h, w) in enumerate(out.extents_at(s))])
    C_last = out.S_u8[-1].shape[1]
    explicit = [3 * (h - 5) * w for (h, w) in shapes]
    for counts in (None, explicit):
        got = bp.get_loss_per_image(out, num_subpixels_before_pad=counts)
        for n, (h, w) in enumerate(shapes):
            hl, wl = out.extents_at(-1)[n]
            uniform = C_last * hl * wl * math.log(bp.losses.loss_dmol_n.L)
            conv = math.log(2.0) * (counts[n] if counts else 3 * h * w)
            want = (sum(ps[n, 0] for ps in per_scale) + uniform) / conv
            tol = sum(ps[n, 1] for ps in per_scale) / conv
            assert abs(got[n] - want) <= tol, (n, got[n], want, tol)
            exact = (sum(o[n] for o in own) + uniform) / conv
            assert abs(got[n] - exact) <= 1e-12 * exact, (n, got[n], exact)


# ---------------------------------------------------------------------------------------------
# quantiser
# ---------------------------------------------------------------------------------------------
def _cr_levels():
    return torch.linspace(-1, 1, 25).numpy()      # nn.Parameter(torch.linspace(lo, hi, L)) of the cr config


def _f32_neighbours(m, n):
    out, lo, hi = [F32(m)], F32(m), F32(m)
    for _ in range(n):
        lo, hi = np.nextafter(lo, F32(-np.inf)), np.nextafter(hi, F32(np.inf))
        out += [lo, hi]
    return np.array(out, F32)


def quantiser_inputs():
    """(ties, others): fp32 values x with (x - l_i)^2 == (x - l_{i+1})^2 in fp32, and their neighbours 1 ulp
    either side, the two values bracketing every decision boundary, values beyond both ends, and non-finite ones"""
    lv = _cr_levels()
    ties, near = [], []
    for i in range(len(lv) - 1):
        c = _f32_neighbours((float(lv[i]) + float(lv[i + 1])) / 2, 200)
        d0, d1 = (c - lv[i]) * (c - lv[i]), (c - lv[i + 1]) * (c - lv[i + 1])
        t = c[d0 == d1]
        ties.append(t)
        for v in t:
            near += [np.nextafter(v, F32(-np.inf)), np.nextafter(v, F32(np.inf))]
        below = c[d0 < d1].max()
        near += [below, np.nextafter(below, F32(np.inf))]
    ends = [-1.0, 1.0, -1.0000001, 1.0000001, -1.5, 1.5, -7.0, 7.0, -1e19, 1e19, -2e19, 2e19, -1e30, 1e30,
            -3.4e38, 3.4e38, 0.0, -0.0, 1e-45, -1e-45]
    others = np.concatenate([np.array(near, F32), np.array(ends, F32)])
    return ties, others


def _reference_symbols(x, lv):
    """modules/quantizer.py:72-83 on the CPU in fp32: torch.min of the squared distances (the first minimum)"""
    xt = torch.from_numpy(np.asarray(x, F32))
    return torch.min(torch.pow(xt.unsqueeze(-1) - torch.from_numpy(lv), 2), -1)[1].numpy()


def test_quantiser_ties_exist_and_the_reference_takes_the_first():
    ties, others = quantiser_inputs()
    lv = _cr_levels()
    found = [i for i, t in enumerate(ties) if len(t)]
    assert len(found) >= 6, found             # a tie needs a representable midpoint
    all_ties = np.concatenate(ties)
    sym = _reference_symbols(all_ties, lv)
    lower = np.concatenate([np.full(len(t), i) for i, t in enumerate(ties)])
    assert np.array_equal(sym, lower)                         # the tie goes to the lower level
    x = np.array([np.inf, -np.inf, np.nan, 1e30, -1e30], F32)
    assert np.array_equal(_reference_symbols(x, lv), np.zeros(5))   # all distances inf / NaN: index 0


def _to_q(Cf, C):
    conv = torch.nn.Conv2d(Cf, C, 1)
    with torch.no_grad():
        conv.weight.zero_()
        conv.bias.zero_()
        for c in range(C):
            conv.weight[c, c, 0, 0] = 1.0
    return conv.cuda()


@pytest.mark.gpu
def test_quantiser_on_ties_ends_and_non_finite_values():
    from l3c_pytorch_b200 import engine as E
    from tests import util
    levels = util.blueprint('cr').net.nets[0].enc.levels.detach()
    lv = _cr_levels()
    assert np.array_equal(levels.cpu().numpy(), lv)
    ties, others = quantiser_inputs()
    vals = np.concatenate([np.concatenate(ties), others, np.array([0.3, -0.7], F32)])
    rng = np.random.default_rng(5)
    # C = 5 of Cf = 8 channels, one-hot weights: q = f exactly; every channel sees every value
    C, Cf = 5, 8
    P = len(vals)
    f = np.zeros((2, 1, P, Cf), F32)
    for n in range(2):
        for c in range(C):
            f[n, 0, :, c] = rng.permutation(vals)
    cases = [(f, C, Cf)]
    # non-finite values: one channel (a 0 weight times inf would turn the others into NaN)
    nf = np.array([np.inf, -np.inf, np.nan, -np.nan, 1e30, -3.4e38, 0.04166666, -0.04166666], F32)
    f1 = np.zeros((1, 1, len(nf), 4), F32)
    f1[0, 0, :, 0] = nf
    cases.append((f1, 1, 4))
    for fx, C_, Cf_ in cases:
        sym, bnq = E.quantize_head(torch.from_numpy(fx).cuda(), _to_q(Cf_, C_), levels)
        sym, bnq = sym.cpu().numpy(), bnq.cpu().numpy()
        N_, _, P_, _ = fx.shape
        want = _reference_symbols(fx[..., :C_].transpose(0, 3, 1, 2), lv)        # [N, C, 1, P]
        bad = np.argwhere(sym != want)
        assert bad.size == 0, ('C=%d: %d symbols differ from torch.min, first at %s: x=%r got %d want %d'
                               % (C_, len(bad), bad[0], fx[tuple(bad[0][[0, 2, 3, 1]])], sym[tuple(bad[0])],
                                  want[tuple(bad[0])]))
        assert np.array_equal(bnq[..., :C_], lv[sym].transpose(0, 2, 3, 1))      # levels[sym], bit for bit
        assert (bnq[..., C_:] == 0).all()
        back = E.symbols_to_values(torch.from_numpy(sym).cuda(), levels).cpu().numpy()
        assert np.array_equal(back, bnq)


@pytest.mark.gpu
def test_symbols_to_values_with_the_rgb_shift():
    from l3c_pytorch_b200 import engine as E
    from tests import util
    bp = util.blueprint('cr_rgb_shared')
    values, shift = bp.net.nets[0].enc._consts(torch.device('cuda'))
    rng = np.random.default_rng(8)
    sym = rng.integers(0, 256, (2, 3, 7, 19)).astype(np.uint8)
    sym[0, :, 0, :2] = [[0, 255]] * 3
    s_dev = torch.from_numpy(sym).cuda()
    for sh in (None, shift):
        got = E.symbols_to_values(s_dev, values, sh).cpu()
        want = values.cpu()[torch.from_numpy(sym).long()]
        if sh is not None:
            want = want - sh.cpu().view(1, 3, 1, 1)
        assert torch.equal(got[..., :3], want.permute(0, 2, 3, 1))
        assert (got[..., 3:] == 0).all()


# ---------------------------------------------------------------------------------------------
# sampling
# ---------------------------------------------------------------------------------------------
U_LO, U_HI = F32(1e-5), F32(1 - 1e-5)


def sample64(l, u_sel, u_x, g):
    """logistic_mixture.py:277-323 in float64 on the same uniforms.  l [P, Kp], u_sel [P, C, K], u_x [P, C] ->
    dict: x [P, C], budget [P, C], sel [P, C], ambiguous [P] (top two Gumbel scores within their fp32 error),
    pre [P, C] (values before the clamps)"""
    P, C = u_x.shape
    lp = l.astype(np.float64).reshape(P, g.P, C, K)
    us = u_sel.astype(np.float64)
    gum = np.log(-np.log(us))
    score = lp[:, 0] - gum
    err = 8 * U * (1 + np.abs(lp[:, 0]) + np.abs(gum) + np.abs(score))
    sel = np.argmax(score, -1)
    top = np.take_along_axis(score, sel[..., None], -1)[..., 0]
    rest = np.where(np.arange(K) == sel[..., None], -np.inf, score).max(-1)
    gap = top - rest
    amb = ((gap > 0) & (gap <= 2 * err.max(-1))).any(-1)
    mean = np.take_along_axis(lp[:, 1], sel[..., None], -1)[..., 0]
    ls = np.maximum(np.take_along_axis(lp[:, 2], sel[..., None], -1)[..., 0], -7.0)
    ux = u_x.astype(np.float64)
    lu, l1u = np.log(ux), np.log1p(-ux)
    raw = mean + np.exp(ls) * (lu - l1u)
    bud = 8 * U * (np.abs(mean) + np.exp(ls) * (np.abs(lu) + np.abs(l1u)))
    pre = raw.copy()
    x = raw.copy()
    if g.rgb:
        co = _sig64(lp[:, 3])
        c_gr = np.take_along_axis(co[:, 0], sel[:, 1:2], -1)[:, 0]
        c_br = np.take_along_axis(co[:, 1], sel[:, 2:3], -1)[:, 0]
        c_bg = np.take_along_axis(co[:, 2], sel[:, 2:3], -1)[:, 0]
        x[:, 0] = np.clip(raw[:, 0], 0, 255)
        pre[:, 1] = raw[:, 1] + c_gr * x[:, 0]
        x[:, 1] = np.clip(pre[:, 1], 0, 255)
        pre[:, 2] = raw[:, 2] + c_br * x[:, 0] + c_bg * x[:, 1]
        x[:, 2] = np.clip(pre[:, 2], 0, 255)
        e0 = bud[:, 0]
        e1 = bud[:, 1] + c_gr * e0 + 8 * U * (c_gr * x[:, 0] + np.abs(pre[:, 1]))
        e2 = bud[:, 2] + c_br * e0 + c_bg * e1 + 8 * U * (c_br * x[:, 0] + c_bg * x[:, 1] + np.abs(pre[:, 2]))
        bud = np.stack([e0, e1, e2], 1)
    return dict(x=x, budget=bud, sel=sel, ambiguous=amb, pre=pre, ls=np.take_along_axis(lp[:, 2], sel[..., None],
                                                                                         -1)[..., 0])


def sample32_emulated(l, u_sel, u_x, g):
    """dmll_sample_kernel in numpy float32"""
    P, C = u_x.shape
    lp = l.astype(F32).reshape(P, g.P, C, K)
    with np.errstate(over='ignore'):
        v = lp[:, 0] - np.log(-np.log(u_sel))
        sel = np.argmax(v, -1)                      # the first maximum, as the kernel's strict >
        mean = np.take_along_axis(lp[:, 1], sel[..., None], -1)[..., 0]
        ls = np.maximum(np.take_along_axis(lp[:, 2], sel[..., None], -1)[..., 0], F32(-7))
        x = mean + np.exp(ls) * (np.log(u_x) - np.log(F32(1) - u_x))
        if g.rgb:
            co = _sig32(lp[:, 3])
            c_gr = np.take_along_axis(co[:, 0], sel[:, 1:2], -1)[:, 0]
            c_br = np.take_along_axis(co[:, 1], sel[:, 2:3], -1)[:, 0]
            c_bg = np.take_along_axis(co[:, 2], sel[:, 2:3], -1)[:, 0]
            x0 = np.clip(x[:, 0], F32(0), F32(255))
            x1 = np.clip(x[:, 1] + c_gr * x0, F32(0), F32(255))
            x2 = np.clip(x[:, 2] + c_br * x0 + c_bg * x1, F32(0), F32(255))
            x = np.stack([x0, x1, x2], 1)
    return x.astype(F32), sel


def _uniforms(rng, shape):
    u = rng.uniform(1e-5, 1 - 1e-5, shape).astype(F32)
    r = rng.random(shape)
    return np.where(r < 0.1, U_LO, np.where(r < 0.2, U_HI, u)).astype(F32)


def sample_case(kind, P=4096, seed=0):
    """(g, l, u_sel, u_x): 'edges' (RGB: u at its limits, log-scales from below the clamp to 5, coefficients at
    +-30, means that drive every channel past 0 and 255), 'ties' (RGB: exact Gumbel ties of all ten or of two
    components) and 'bottleneck' (C = 5, nothing clamped)"""
    rng = np.random.default_rng(300 + seed + ('edges', 'ties', 'bottleneck').index(kind))
    g = BN if kind == 'bottleneck' else RGB
    C = g.C
    logit = rng.normal(0, 2, (P, C, K))
    ls = rng.uniform(-10, 5, (P, C, K))
    co = np.where(rng.random((P, 3, K)) < 0.5, rng.choice([-30.0, 30.0], (P, 3, K)), rng.normal(0, 3, (P, 3, K)))
    u_sel, u_x = _uniforms(rng, (P, C, K)), _uniforms(rng, (P, C))
    if kind == 'bottleneck':
        mean = rng.uniform(-3, 3, (P, C, K))
        ls = rng.uniform(-10, 1, (P, C, K))
    elif kind == 'edges':
        mean = rng.uniform(-150, 400, (P, C, K))
    else:
        mean = np.broadcast_to(20.0 * np.arange(K) + 15.0, (P, C, K)).copy()
        ls = rng.uniform(-9, -1, (P, C, K))
        all_ten = rng.random((P, C)) < 0.5
        same = rng.uniform(-3, 3, (P, C, 1))
        u_same = np.where(rng.random((P, C, 1)) < 0.2, U_LO, rng.uniform(1e-5, 1 - 1e-5, (P, C, 1))).astype(F32)
        # two components tied above the others
        pair = np.sort(np.argsort(rng.random((P, C, K)), -1)[..., :2], -1)
        two = np.full((P, C, K), -12.0)
        np.put_along_axis(two, pair, same, -1)
        logit = np.where(all_ten[..., None], same, two)
        u_pair = np.full((P, C, K), F32(0.5))
        np.put_along_axis(u_pair, pair, u_same, -1)
        u_sel = np.where(all_ten[..., None], u_same, u_pair).astype(F32)
    planes = [logit, mean, ls] + ([co] if g.rgb else [])
    l = np.stack(planes, 1).reshape(P, -1).astype(F32)
    return g, l, u_sel, u_x


def _sample_regimes(kind, g, l, u_sel, u_x, d):
    out = {'u_x == 1e-5': ((u_x == U_LO).sum(), 200), 'u_x == 1 - 1e-5': ((u_x == U_HI).sum(), 200)}
    if kind != 'ties':
        out['u_sel == 1e-5'] = ((u_sel == U_LO).sum(), 2000)
        out['u_sel == 1 - 1e-5'] = ((u_sel == U_HI).sum(), 2000)
        out['selected log-scale < -7'] = ((d['ls'] < -7).sum(), 500)
        out['selected log-scale > %g' % (0 if g is BN else 4)] = ((d['ls'] > (0 if g is BN else 4)).sum(), 100)
    if kind == 'edges':
        for c in range(3):
            m = 1.0 + d['budget'][:, c]
            out['channel %d below 0' % c] = ((d['pre'][:, c] < -m).sum(), 200)
            out['channel %d above 255' % c] = ((d['pre'][:, c] > 255 + m).sum(), 200)
        co = l.reshape(len(l), 4, 3, K)[:, 3]
        out['coefficient logit +-30'] = ((np.abs(co) == 30).sum(), 10000)
    if kind == 'bottleneck':
        out['|x| > 1, not clamped'] = ((np.abs(d['x']) > 1.5).sum(), 1000)
    if kind == 'ties':
        lp = l.reshape(len(l), g.P, g.C, K)
        score = lp[:, 0].astype(np.float64) - np.log(-np.log(u_sel.astype(np.float64)))
        top = score.max(-1, keepdims=True)
        n_top = (score == top).sum(-1)
        out['all ten tied'] = ((n_top == K).sum(), 3000)
        out['two tied on top'] = ((n_top == 2).sum(), 3000)
    return {k: (int(v), need) for k, (v, need) in out.items()}


def _assert_sample(got, d, what):
    ok_pix = ~d['ambiguous']
    assert ok_pix.mean() > 0.98, (what, float(ok_pix.mean()))
    err = np.abs(got.astype(np.float64) - d['x'])
    bad = (~(err <= d['budget'])) & ok_pix[:, None]
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError('%s: %d samples outside their budget; first at %s: got %r, float64 %r (sel %s), budget '
                             '%.3g' % (what, int(bad.sum()), i, float(got[i]), float(d['x'][i]), d['sel'][i[0]],
                                       float(d['budget'][i])))


@pytest.mark.parametrize('kind', ['edges', 'ties', 'bottleneck'])
def test_sample_budget_covers_the_fp32_formula(kind):
    g, l, u_sel, u_x = sample_case(kind)
    d = sample64(l, u_sel, u_x, g)
    for name, (n, need) in _sample_regimes(kind, g, l, u_sel, u_x, d).items():
        assert n >= need, (kind, name, n, need)
    got, sel = sample32_emulated(l, u_sel, u_x, g)
    assert np.array_equal(sel[~d['ambiguous']], d['sel'][~d['ambiguous']])
    _assert_sample(got, d, kind + ' emulated')
    if kind == 'ties':
        first = np.argmax(l.reshape(len(l), 4, 3, K)[:, 0] - np.log(-np.log(u_sel)), -1)
        assert np.array_equal(d['sel'], first)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['edges', 'ties', 'bottleneck'])
def test_sampling_kernel_against_float64(kind):
    from l3c_pytorch_b200 import engine as E
    g, l, u_sel, u_x = sample_case(kind)
    d = sample64(l, u_sel, u_x, g)
    for name, (n, need) in _sample_regimes(kind, g, l, u_sel, u_x, d).items():
        assert n >= need, (kind, name, n, need)
    P, C = u_x.shape
    got = E.dmll_sample(torch.from_numpy(l.reshape(1, 1, P, -1)).cuda(),
                        torch.from_numpy(np.ascontiguousarray(u_sel.transpose(1, 2, 0)).reshape(1, C, K, 1, P)).cuda(),
                        torch.from_numpy(np.ascontiguousarray(u_x.T).reshape(1, C, 1, P)).cuda(), C, K, g.rgb)
    got = got.cpu().numpy().reshape(C, P).T
    _assert_sample(got, d, kind)
    if g.rgb:
        assert got.min() >= 0 and got.max() <= 255
