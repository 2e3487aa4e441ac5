#!/usr/bin/env python
"""bench_seek.py -- decode reference-layout containers serially and from seek indexes (DESIGN §4.13), one GPU.

  python tools/bench_seek.py [--steps K] [--warmup W] [--sizes 1,16] [--every 4096,16384] [--size S]

Workload: `cr` with seed-0 default-init weights, f16, reference layout, batches of N uint8 noise images of S x S
(default 512; N = 1 and 16).  Per batch size the arms alternate inside every step, each timed with CUDA events around
one synchronised call: serial decode_batch, decode_batch(seeks=) at every K, encode_batch and encode_batch(seek=K) at
the first K.  Every decode is checked lossless and the containers with and without seek identical.  Prints the median
ms per arm, the index bytes per image and their share of the container, and one JSON line with the card's name and
power limit, read in the same call."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def make_images(n, s):
    import torch
    out = []
    for i in range(n):
        g = torch.Generator().manual_seed(1000 + i)
        out.append((torch.rand(3, s, s, generator=g) * 255).round().to(torch.uint8))
    return torch.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--sizes', default='1,16')
    ap.add_argument('--every', default='4096,16384')
    ap.add_argument('--size', type=int, default=512)
    args = ap.parse_args()

    import numpy as np
    import torch
    import l3c_pytorch_b200 as l3c
    from l3c_pytorch_b200 import config
    assert torch.cuda.is_available(), 'bench_seek.py needs a GPU; there is no CPU fallback'
    torch.cuda.set_device(0)
    dev = torch.device('cuda', 0)
    l3c.set_conv_precision('f16')
    torch.manual_seed(0)
    bp = l3c.MultiscaleBlueprint(config.ms_config('cr'), device=dev).set_eval()
    bc = l3c.Bitcoding(bp)
    Ks = [int(k) for k in args.every.split(',')]

    def timed(fn):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b), out

    results = []
    for N in [int(n) for n in args.sizes.split(',')]:
        imgs = make_images(N, args.size).to(dev)
        want = [im.unsqueeze(0).long() for im in imgs]
        datas, _ = bc.encode_batch(imgs)
        seeks = {K: bc.encode_batch(imgs, seek=K)[2] for K in Ks}
        arms = {'decode serial': lambda: bc.decode_batch(datas)}
        for K in Ks:
            arms['decode seek K=%d' % K] = (lambda K: lambda: bc.decode_batch(datas, seeks=seeks[K]))(K)
        arms['encode'] = lambda: bc.encode_batch(imgs)
        arms['encode seek K=%d' % Ks[0]] = lambda: bc.encode_batch(imgs, seek=Ks[0])
        ms = {k: [] for k in arms}
        for step in range(args.warmup + args.steps):
            for name, fn in arms.items():
                t, out = timed(fn)
                if name.startswith('decode'):
                    assert all(torch.equal(a, b.to(a.device)) for a, b in zip(out, want)), name
                else:
                    assert out[0] == datas, name
                if step >= args.warmup:
                    ms[name].append(t)
        cont = float(np.mean([len(d) for d in datas]))
        row = {'N': N, 'size': args.size, 'container_bytes_per_image': cont,
               'ms': {k: float(np.median(v)) for k, v in ms.items()},
               'index': {K: {'bytes_per_image': float(np.mean([len(s) for s in seeks[K]])),
                             'share': float(np.mean([len(s) for s in seeks[K]])) / cont,
                             'bpsp': float(np.mean([len(s) for s in seeks[K]])) * 8 / (3 * args.size ** 2)}
                         for K in Ks}}
        results.append(row)
        for k, v in row['ms'].items():
            print('N=%d %-20s %9.2f ms' % (N, k, v))
        for K, v in row['index'].items():
            print('N=%d index K=%d: %.0f B per image, %.4f %% of the container, %.4f bpsp'
                  % (N, K, v['bytes_per_image'], 100 * v['share'], v['bpsp']))
    try:
        power = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = None
    print(json.dumps({'bench': 'seek', 'config': 'cr', 'precision': 'f16', 'results': results, 'lossless': True,
                      'gpu': torch.cuda.get_device_name(0), 'power_limit': power}))


if __name__ == '__main__':
    main()
