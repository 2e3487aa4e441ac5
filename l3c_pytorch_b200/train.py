"""Training step of L3C (SURVEY.md section 8 row f4): PyTorch autograd over the SAME parameter tree
(`MultiscaleNetwork`'s nn.Conv2d containers), so that what it trains loads into the sm_90a coding path unchanged.
The convolutions and their backward are torch's (cuDNN on the GPU).  The two per-pixel losses are the library's
kernels on CUDA tensors (DESIGN §4.9): the DMLL negative log-likelihood of every scale and the soft quantiser, each
forward and backward in one pass over its inputs, without torch's per-element autograd graph.  CPU tensors, and CUDA
tensors with FUSED_LOSS = False, take the torch restatements `dmll_nll` and `soft_quantize_torch`, which stay the
reference the kernels are tested against.  `tools/bench_train.py` measures both paths.

Reference (under /root/reference/src):
  train/multiscale_trainer.py:173-226   train_step: zero_grad, forward, get_loss, backward, optim.step
  modules/quantizer.py:62-90            soft/hard quantiser (straight-through: hard values, soft gradient)
  modules/net.py:136-148,173-184        encoder / decoder forward (training: the decoder is fed `bn`, the soft one)
  modules/multiscale_network.py:262-306 _forward_with_scales
  criterion/logistic_mixture.py:146-246 discretised-logistic-mixture NLL (+ RGB mean coupling)
  blueprints/multiscale_blueprint.py:64-95  bpsp conversion, loss_pc = sum of the per-scale costs without the
                                            uniform-prior final scale
Works on CPU tensors as well as CUDA ones.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import engine as E
from .dmll import non_shared_get_K

_LOG_SCALES_MIN = -7.
_K = 10                       # the mixture size the kernels are built for (dmll.cu check_common)

# CUDA tensors: True runs the DMLL loss and the soft quantiser as the library's kernels, False as the torch
# restatements below (for comparisons on the GPU: tests/test_gpu_train_kernels.py, tools/bench_train.py)
FUSED_LOSS = True


def _require_f32(what, *ts):
    for t in ts:
        if t.dtype != torch.float32:
            raise TypeError('%s: the training kernels take fp32 tensors, got %s' % (what, t.dtype))
        if not t.is_cuda:
            raise ValueError('%s: mixed devices (%s); the kernels need every tensor on the GPU' % (what, t.device))


class _SoftQuantizeFn(torch.autograd.Function):
    """(q, levels, sigma) -> (hard values levels[sym] with the soft quantiser's gradient, sym int64)."""

    @staticmethod
    def forward(ctx, q, levels, sigma):
        q, levels = q.contiguous(), levels.detach().contiguous()
        sym, val = E.soft_quantize(q, levels, sigma)
        ctx.save_for_backward(q, levels)
        ctx.sigma = sigma
        ctx.mark_non_differentiable(sym)
        return val, sym

    @staticmethod
    def backward(ctx, g_val, g_sym):
        q, levels = ctx.saved_tensors
        return E.soft_quantize(q, levels, ctx.sigma, grad=g_val.contiguous()), None, None


def soft_quantize(x, levels, sigma):
    """quantizer.py:62-90 -> (x_soft with hard data and soft gradient, x_hard, symbols).  CUDA: the soft quantiser
    kernels (x_hard shares x_soft's data, as in the torch path); CPU: soft_quantize_torch."""
    if not (FUSED_LOSS and x.is_cuda):
        return soft_quantize_torch(x, levels, sigma)
    _require_f32('soft_quantize', x, levels)
    x_soft, sym = _SoftQuantizeFn.apply(x, levels, float(sigma))
    return x_soft, x_soft.detach(), sym


def soft_quantize_torch(x, levels, sigma):
    """quantizer.py:62-90 -> (x_soft with hard data and soft gradient, x_hard, symbols), in torch operators."""
    N, C, H, W = x.shape
    xv = x.view(N, C, H * W, 1)
    d = torch.pow(xv - levels, 2)
    phi_soft = F.softmax(-sigma * d, dim=-1)
    x_soft = torch.sum(levels * phi_soft, dim=-1).view(N, C, H, W)
    _, sym = torch.min(d.detach(), dim=-1)
    sym = sym.view(N, C, H, W)
    x_hard = levels[sym]
    x_soft.data = x_hard                      # assign data, keep gradient
    return x_soft, x_hard, sym


def _res_body(body, x):
    """Sequential of ResBlocks + final conv with the outer skip (net.py:144,181; edsr.py:83-86)."""
    y = x
    for m in list(body)[:-1]:
        y = m.body[2](F.relu(m.body[0](y))) + y
    return body[-1](y) + x


def _enc_forward(enc, x):
    """EDSRLikeEnc.forward in training mode (net.py:136-148): -> (bn soft, bn_q, S, F)."""
    x = enc.down(x)
    x = _res_body(enc.body, x)
    feat = x
    q = enc.to_q[0](x)
    bn, bn_q, sym = soft_quantize(q, enc.levels, enc.q.sigma)
    return bn, bn_q, sym, feat


def _dec_forward(dec, bn, fuse):
    x = dec.head(bn)
    if fuse is not None:
        x = x + fuse
    x = _res_body(dec.body, x)
    return F.pixel_shuffle(dec.tail[0](x), 2)


def _prob_clf(clf, x):
    a = clf.atrous
    return a.lin(torch.cat([c(x) for c in a.atrous], dim=1))


def dmll_nll(dm, x, l):
    """DiscretizedMixLogisticLoss.forward (logistic_mixture.py:146-207): x NCHW targets on the value grid (may carry
    gradient), l NKpHW -> NCHW negative log-likelihood in nats."""
    N, C, H, W = x.shape
    K = non_shared_get_K(l.shape[1], C)
    lr = l.reshape(N, dm._num_params, C, K, H, W)
    logit_pis, means = lr[:, 0], lr[:, 1]
    log_scales = torch.clamp(lr[:, 2], min=_LOG_SCALES_MIN)
    xr = x.reshape(N, C, 1, H, W)
    if dm.use_coeffs:
        assert C == 3
        co = torch.sigmoid(lr[:, 3])
        means = torch.stack((means[:, 0],
                             means[:, 1] + co[:, 0] * xr[:, 0],
                             means[:, 2] + co[:, 1] * xr[:, 0] + co[:, 2] * xr[:, 1]), dim=1)
    centered = xr - means
    inv_stdv = torch.exp(-log_scales)
    plus_in = inv_stdv * (centered + dm.bin_width / 2)
    min_in = inv_stdv * (centered - dm.bin_width / 2)
    cdf_delta = torch.sigmoid(plus_in) - torch.sigmoid(min_in)
    log_cdf_plus = plus_in - F.softplus(plus_in)
    log_one_minus_cdf_min = -F.softplus(min_in)
    out_a = torch.log(torch.clamp(cdf_delta, min=1e-12))
    cond_b = (xr > dm.x_upper_bound).float()
    out_b = cond_b * log_one_minus_cdf_min + (1. - cond_b) * out_a
    cond_c = (xr < dm.x_lower_bound).float()
    log_probs = cond_c * log_cdf_plus + (1. - cond_c) * out_b
    weighted = log_probs + F.log_softmax(logit_pis, dim=2)
    return -torch.logsumexp(weighted, dim=2)


class _DmllNllFn(torch.autograd.Function):
    """(l, x, dm) -> the summed nats of dmll_nll as a 0-dim fp32 tensor; saves only l and x."""

    @staticmethod
    def forward(ctx, l, x, dm):
        l, x = l.contiguous(), x.contiguous()
        ctx.save_for_backward(l, x)
        ctx.dm = dm
        nll = E.dmll_nll_train(l, x, _K, dm.use_coeffs, dm.bin_width / 2, dm.x_lower_bound, dm.x_upper_bound)
        return nll.sum().float()

    @staticmethod
    def backward(ctx, g):
        l, x = ctx.saved_tensors
        dm = ctx.dm
        dl, dx = E.dmll_nll_train(l, x, _K, dm.use_coeffs, dm.bin_width / 2, dm.x_lower_bound, dm.x_upper_bound,
                                  grad=g.float().contiguous(), want_dx=ctx.needs_input_grad[1])
        return dl, dx, None


def dmll_nll_sum(dm, x, l):
    """dmll_nll(dm, x, l).sum(): the total nats of one scale as a 0-dim fp32 tensor, with its gradient to l and, at a
    bottleneck scale, to x.  CUDA: the training kernels (the per-image sums in float64, then their total); CPU: the
    torch restatement.  An RGB target (dm.use_coeffs) must not require grad: the image is a leaf."""
    if not (FUSED_LOSS and l.is_cuda):
        return dmll_nll(dm, x, l).sum()
    _require_f32('dmll_nll_sum', l, x)
    if x.dim() != 4 or l.dim() != 4 or l.shape[0] != x.shape[0] or l.shape[2:] != x.shape[2:]:
        raise ValueError('dmll_nll_sum: l %s and x %s are not NKpHW / NCHW of one batch'
                         % (tuple(l.shape), tuple(x.shape)))
    C = x.shape[1]
    if l.shape[1] != dm._num_params * C * _K:
        raise ValueError('dmll_nll_sum: l has %d channels; the kernels take Kp = %d x C x K = %d (C = %d, K = %d)'
                         % (l.shape[1], dm._num_params, dm._num_params * C * _K, C, _K))
    if dm.use_coeffs and (C != 3 or x.requires_grad):
        raise ValueError('dmll_nll_sum: an RGB scale needs C = 3 targets that do not require grad (got C = %d, '
                         'requires_grad = %s)' % (C, x.requires_grad))
    return _DmllNllFn.apply(l, x, dm)


def forward_train(net, x):
    """MultiscaleNetwork.forward in training mode (multiscale_network.py:226-306) for the L3C configurations:
    x NCHW float in [0, 255] -> (targets, predictions) per scale fine -> coarse, plus the symbols of every scale.
    targets[0] is the image, targets[i >= 1] the SOFT bottleneck of scale i (gradient flows through it)."""
    if net._rgb:
        raise NotImplementedError('the training step is built for the L3C configurations (learned bottlenecks)')
    syms = [x.round().long()]
    h = net.sub_rgb_mean(x)
    inp = h
    encs = []
    for s in range(net.scales):
        head = net.heads[s]
        inp = head.head[1].head(head.head[0](inp)) if s == 0 else head.head(inp)
        bn, bn_q, sym, feat = _enc_forward(net.nets[s].enc, inp)
        encs.append((bn, bn_q))
        syms.append(sym)
        inp = feat                                   # enc.feed_F
    dec_f = [None] * net.scales
    prev = None
    for s in reversed(range(net.scales)):
        fuse = prev if (net._fuse_feat and s != net.scales - 1) else None
        prev = _dec_forward(net.nets[s].dec, encs[s][0], fuse)          # training: the decoder sees the soft bn
        dec_f[s] = prev
    preds = [_prob_clf(net.prob_clfs[s], dec_f[s]) for s in range(net.scales)]
    targets = [x] + [encs[s][0] for s in range(net.scales - 1)]
    return targets, preds, syms


def training_loss(blueprint, x):
    """-> (loss_pc, [bpsp per scale incl. the uniform-prior final scale]) as multiscale_blueprint.py:64-95."""
    net, losses = blueprint.net, blueprint.losses
    targets, preds, syms = forward_train(net, x)
    costs = []
    for i, (t, p) in enumerate(zip(targets, preds)):
        dm = losses.loss_dmol_rgb if i == 0 else losses.loss_dmol_n
        costs.append(dmll_nll_sum(dm, t, p))
    num_subpixels = int(np.prod(x.shape))
    conversion = np.log(2.) * num_subpixels
    costs_bpsp = [c / conversion for c in costs]
    final = int(np.prod(syms[-1].shape)) * np.log(net.config_ms.q.L) / conversion
    return sum(costs_bpsp), [float(c.detach()) for c in costs_bpsp] + [float(final)]


def make_optimizer(blueprint):
    """multiscale_trainer.py:72-80: optimiser class and initial learning rate from the model config."""
    cfg = blueprint.net.config_ms
    cls = {'RMSprop': torch.optim.RMSprop, 'Adam': torch.optim.Adam, 'SGD': torch.optim.SGD}[cfg.optim]
    return cls(blueprint.net.parameters(), cfg.lr.initial, weight_decay=cfg.weight_decay)


def train_step(blueprint, optimizer, img_batch):
    """One optimisation step on an NCHW float batch in [0, 255] (multiscale_trainer.py:173-200).
    -> (loss_pc as float, bpsp per scale)."""
    blueprint.net.zero_grad()
    loss_pc, bpsps = training_loss(blueprint, img_batch)
    loss_pc.backward()
    optimizer.step()
    return float(loss_pc.detach()), bpsps
