"""Training step and training loss, torch-loss path against the fused loss kernels (DESIGN §4.9, §7).

    python tools/bench_train.py [--batch 30] [--crop 128] [--reps 5] [--iters 10]

cr.cf with its seed-0 initial weights, seeded crops of batch x 3 x crop x crop, RMSprop (make_optimizer).  For each
rep the two paths (train.FUSED_LOSS False / True) run alternately, each timed with CUDA events over `iters` calls
after a warm-up:
  step: the whole train_step (forward, loss, backward, optimiser step);
  loss: the loss alone -- the three DMLL terms and the three soft quantisers, forward and backward, on leaf inputs
        shaped like the step's.
Peak memory is torch.cuda.max_memory_allocated over one call, above what was allocated before it with every
gradient freed.  Prints the card and its power limit, then one JSON line.  Nothing is written."""
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
    a = ap.parse_args()
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


if __name__ == '__main__':
    main()
