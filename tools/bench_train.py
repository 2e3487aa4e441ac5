"""Training step and training loss, torch-loss path against the fused loss kernels (DESIGN §4.9, §7).

    python tools/bench_train.py [--arm loss|conv] [--batch 30] [--crop 128] [--reps 5] [--iters 10]

cr.cf with its seed-0 initial weights, seeded crops of batch x 3 x crop x crop, RMSprop (make_optimizer).  For each
rep the two paths (train.FUSED_LOSS False / True) run alternately, each timed with CUDA events over `iters` calls
after a warm-up:
  step: the whole train_step (forward, loss, backward, optimiser step);
  loss: the loss alone -- the three DMLL terms and the three soft quantisers, forward and backward, on leaf inputs
        shaped like the step's.
Peak memory is torch.cuda.max_memory_allocated over one call, above what was allocated before it with every
gradient freed.  Prints the card and its power limit, then one JSON line.  Nothing is written.

--arm conv: the 3x3 / 64-input-channel convolutions (train.FUSED_CONV, DESIGN §4.11) instead of the loss.
  macs:  the in-scope share of the forward's multiply-adds, from the shapes every nn.Conv2d of forward_train sees;
  step:  train_step with FUSED_CONV False (cuDNN) and True, alternating, and the peak memory of each;
  copies: aten::copy_ calls and their device time in one step of each path (torch.profiler, a run of its own);
  layer: per in-scope layer shape (Cout, dilation, plane), the backward alone -- dx, dW and db of one layer from a
         retained graph -- through cuDNN (NCHW input, as the cuDNN step runs it) and through _Conv3x3Fn."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from l3c_pytorch_b200 import MultiscaleBlueprint, config, train            # noqa: E402


def gpu_info():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else 'unknown'


def time_calls(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def peak_of(fn, clear):
    clear()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=30)
    ap.add_argument('--crop', type=int, default=128)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--arm', choices=('loss', 'conv'), default='loss')
    a = ap.parse_args()
    if a.arm == 'conv':
        return conv_arm(a)
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    bp = MultiscaleBlueprint(config.ms_config('cr'), device=dev)
    bp.net.float()
    bp.net.train()
    opt = train.make_optimizer(bp)
    gen = torch.Generator(device=dev).manual_seed(0)
    imgs = (torch.rand(a.batch, 3, a.crop, a.crop, device=dev, generator=gen) * 255).round()

    # leaf inputs of the loss, shaped like the step's: predictions of the three scales and the to_q outputs
    S, N = a.crop, a.batch
    preds = [torch.randn(N, 120, S, S, device=dev, generator=gen).requires_grad_(True)] + \
            [torch.randn(N, 150, S >> s, S >> s, device=dev, generator=gen).requires_grad_(True) for s in (1, 2)]
    qs = [(0.6 * torch.randn(N, 5, S >> s, S >> s, device=dev, generator=gen)).requires_grad_(True) for s in (1, 2, 3)]
    levels = bp.net.nets[0].enc.levels.detach()
    sigma = bp.net.config_ms.q.sigma
    dm_rgb, dm_bn = bp.losses.loss_dmol_rgb, bp.losses.loss_dmol_n

    def clear():
        bp.net.zero_grad(set_to_none=True)
        for t in preds + qs:
            t.grad = None

    def step():
        train.train_step(bp, opt, imgs)

    def loss():
        for t in preds + qs:
            t.grad = None
        bns = [train.soft_quantize(q, levels, sigma)[0] for q in qs]
        total = train.dmll_nll_sum(dm_rgb, imgs, preds[0])
        for s in (1, 2):
            total = total + train.dmll_nll_sum(dm_bn, bns[s - 1], preds[s])
        (total / (np.log(2.) * imgs.numel()) + 0 * bns[2].sum()).backward()

    res = {'step_ms': {'torch': [], 'fused': []}, 'loss_ms': {'torch': [], 'fused': []}}
    peaks = {}
    paths = (('torch', False), ('fused', True))
    for fused_name, fused in paths:
        train.FUSED_LOSS = fused
        for _ in range(a.warmup):
            step()
            loss()
        peaks[fused_name] = {'step_MB': peak_of(step, clear) / 2 ** 20, 'loss_MB': peak_of(loss, clear) / 2 ** 20}
    for _ in range(a.reps):
        for name, fused in paths:
            train.FUSED_LOSS = fused
            res['step_ms'][name].append(time_calls(step, a.iters))
            res['loss_ms'][name].append(time_calls(loss, a.iters))
    train.FUSED_LOSS = True
    card = gpu_info()
    print('card: %s' % card)
    print('torch version %s, batch %d x 3 x %d^2, TF32 conv %s' % (torch.__version__, N, S,
                                                                torch.backends.cudnn.allow_tf32))
    for k in ('step_ms', 'loss_ms'):
        for name, _ in paths:
            v = res[k][name]
            print('%s %-6s median %.2f ms  (%s)' % (k, name, float(np.median(v)), ' '.join('%.2f' % t for t in v)))
    for name, _ in paths:
        print('peak %-6s step %.0f MB, loss %.0f MB' % (name, peaks[name]['step_MB'], peaks[name]['loss_MB']))
    print(json.dumps({'card': card, 'batch': N, 'crop': S,
                      'step_ms': {n: float(np.median(v)) for n, v in res['step_ms'].items()},
                      'loss_ms': {n: float(np.median(v)) for n, v in res['loss_ms'].items()},
                      'peak_MB': peaks}))


def conv_shapes(bp, imgs):
    """-> (in-scope MACs, all MACs, {(Cout, dilation, H, W): layers}) of one forward_train, from the output shapes"""
    macs = {'in': 0, 'all': 0}
    shapes = {}

    def hook(m, inp, out):
        n = m.kernel_size[0] * m.kernel_size[1] * (m.in_channels // m.groups) * out.numel()
        macs['all'] += n
        if train.conv3x3_in_scope(m):
            macs['in'] += n
            key = (m.out_channels, m.dilation[0], out.shape[2], out.shape[3])
            shapes[key] = shapes.get(key, 0) + 1

    hs = [m.register_forward_hook(hook) for m in bp.net.modules() if isinstance(m, torch.nn.Conv2d)]
    train.FUSED_CONV = False
    with torch.no_grad():
        train.forward_train(bp.net, imgs)
    for h in hs:
        h.remove()
    return macs['in'], macs['all'], shapes


def copies_of(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if e.key == 'aten::copy_':
            return e.count, e.device_time_total / 1e3
    return 0, 0.0


def layer_backward_ms(cout, d, N, H, W, fused, iters, dev):
    g = torch.Generator(device=dev).manual_seed(1)
    conv = torch.nn.Conv2d(64, cout, 3, padding=d, dilation=d).to(dev)
    x = torch.randn(N, 64, H, W, device=dev, generator=g)
    if fused:
        x = x.contiguous(memory_format=torch.channels_last)
    x.requires_grad_(True)
    train.FUSED_CONV = fused
    y = train._conv(conv, x)
    gy = torch.randn(y.shape, device=dev, generator=g)
    if fused:
        gy = gy.contiguous(memory_format=torch.channels_last)
    params = [x, conv.weight, conv.bias]
    run = lambda: torch.autograd.grad(y, params, gy, retain_graph=True)      # noqa: E731
    for _ in range(3):
        run()
    return time_calls(run, iters)


def conv_arm(a):
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    bp = MultiscaleBlueprint(config.ms_config('cr'), device=dev)
    bp.net.float()
    bp.net.train()
    opt = train.make_optimizer(bp)
    gen = torch.Generator(device=dev).manual_seed(0)
    imgs = (torch.rand(a.batch, 3, a.crop, a.crop, device=dev, generator=gen) * 255).round()
    N, S = a.batch, a.crop
    mac_in, mac_all, shapes = conv_shapes(bp, imgs)

    def clear():
        bp.net.zero_grad(set_to_none=True)

    def step():
        train.train_step(bp, opt, imgs)

    paths = (('cudnn', False), ('fused', True))
    res = {n: [] for n, _ in paths}
    peaks, copies = {}, {}
    for name, fused in paths:
        train.FUSED_CONV = fused
        for _ in range(a.warmup):
            step()
        peaks[name] = peak_of(step, clear) / 2 ** 20
        copies[name] = copies_of(step)
    for _ in range(a.reps):
        for name, fused in paths:
            train.FUSED_CONV = fused
            res[name].append(time_calls(step, a.iters))
    layers = {}
    for (cout, d, H, W), count in sorted(shapes.items()):
        layers['%d d%d %dx%d' % (cout, d, H, W)] = {
            'layers': count, **{name: layer_backward_ms(cout, d, N, H, W, fused, a.iters, dev) for name, fused in paths}}
    train.FUSED_CONV = False
    card = gpu_info()
    print('card: %s' % card)
    print('torch version %s, batch %d x 3 x %d^2, cuDNN TF32 %s' % (torch.__version__, N, S,
                                                                  torch.backends.cudnn.allow_tf32))
    print('in-scope share of the forward multiply-adds: %.1f %% (%.3g of %.3g GMAC)'
          % (100.0 * mac_in / mac_all, mac_in / 1e9, mac_all / 1e9))
    for name, _ in paths:
        v = res[name]
        print('step_ms %-6s median %.2f ms  (%s)  peak %.0f MB, aten::copy_ %d calls %.2f ms'
              % (name, float(np.median(v)), ' '.join('%.2f' % t for t in v), peaks[name], *copies[name]))
    for k, v in layers.items():
        print('layer backward %-16s x%-2d cudnn %.3f ms  fused %.3f ms' % (k, v['layers'], v['cudnn'], v['fused']))
    print(json.dumps({'card': card, 'batch': N, 'crop': S, 'mac_share': mac_in / mac_all,
                      'step_ms': {n: float(np.median(v)) for n, v in res.items()}, 'peak_MB': peaks,
                      'copies': copies, 'layer_backward_ms': layers}))


if __name__ == '__main__':
    main()
