#!/usr/bin/env python
"""bench_theory.py -- theoretical bpsp (the harness's default mode) of images of DIFFERENT sizes, one GPU.

  python tools/bench_theory.py [--steps K] [--warmup W] [--images N] [--batch B]

Workload: N (default 32) uint8 noise images of seeded sizes, H and W uniform in [256, 768] (mostly not multiples
of 8, so most are padded), L3C cr.cf with seed-0 default-init weights, precision f16.  Two arms run alternating in
one process, every step runs each once:
  ragged      harness.ragged_theory_bpsps: every image padded on its own, planned into ragged passes of at most B
              (default 16) images, forward(extents=) + get_loss_per_image per pass
  per_image   one forward + get_loss_per_image per image (what the harness does for a test set whose images all
              differ in size when ragged passes are unavailable)
Images/s and Mpixels/s count unpadded pixels; the host-side reads of the test set are not part of either arm.
The per-image bpsp of both arms must be identical (asserted).  Prints one JSON line with the card name and its
power limit.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = 'images/s theoretical bpsp (harness default mode), images of different sizes'


def make_image(i, h, w):
    import torch
    g = torch.Generator().manual_seed(1000 + i)
    return (torch.rand(3, h, w, generator=g) * 255).round().to(torch.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--images', type=int, default=32)
    ap.add_argument('--batch', type=int, default=16)
    ap.add_argument('--min-side', type=int, default=256)
    ap.add_argument('--max-side', type=int, default=768)
    args = ap.parse_args()

    import numpy as np
    import torch
    import l3c_pytorch_b200 as l3c
    from l3c_pytorch_b200 import config, engine as E
    from l3c_pytorch_b200.bitcoding import plan_passes
    from l3c_pytorch_b200.harness import ragged_theory_bpsps
    assert torch.cuda.is_available(), 'bench_theory.py needs a GPU; there is no CPU fallback'
    torch.cuda.set_device(0)
    dev = torch.device('cuda', 0)
    E.set_conv_precision('f16')
    torch.manual_seed(0)
    bp = l3c.MultiscaleBlueprint(config.ms_config('cr'), device=dev).set_eval()
    assert bp.net.ragged_unsupported() is None
    rng = np.random.default_rng(0)
    sizes = [(int(rng.integers(args.min_side, args.max_side + 1)), int(rng.integers(args.min_side, args.max_side + 1)))
             for _ in range(args.images)]
    imgs = [make_image(i, h, w) for i, (h, w) in enumerate(sizes)]
    px = sum(h * w for (h, w) in sizes)
    fac = 2 ** bp.net.config_ms.num_scales
    padded = [(h + (-h) % fac, w + (-w) % fac) for (h, w) in sizes]

    def ragged():
        return ragged_theory_bpsps(bp, imgs, fac, args.batch)

    def per_image():
        out = []
        for im in imgs:
            batch, _ = bp.unpack_batch_pad(im.unsqueeze(0), fac=fac)
            out.append(float(bp.get_loss_per_image(bp.forward(batch), num_subpixels_before_pad=im.numel())[0]))
        return out

    arms = {'ragged': ragged, 'per_image': per_image}
    ms = {k: [] for k in arms}
    last = {}
    with torch.no_grad():
        for step in range(args.warmup + args.steps):
            for name, fn in arms.items():               # alternating: every step runs every arm once
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                last[name] = fn()                       # ends in a device -> host copy of the costs
                b.record()
                torch.cuda.synchronize()
                if step >= args.warmup:
                    ms[name].append(a.elapsed_time(b))
    assert last['ragged'] == last['per_image'], 'per-image bpsp of the two arms differ'
    ips = {k: len(imgs) * len(v) / (sum(v) / 1e3) for k, v in ms.items()}
    mpx = {k: px * len(v) / (sum(v) / 1e3) / 1e6 for k, v in ms.items()}
    try:
        power = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                               capture_output=True, text=True, timeout=30).stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    line = {
        'metric': METRIC, 'value': ips['ragged'], 'unit': 'images/s', 'n_gpus': 1, 'steps': args.steps,
        'warmup': args.warmup, 'higher_is_better': True, 'dtype': 'f16', 'data': 'synthetic',
        'config': {'workload': 'L3C cr.cf, %d uint8 noise images of seeded sizes (H, W uniform in [%d, %d])'
                               % (args.images, args.min_side, args.max_side),
                   'sizes': sizes, 'unpadded_pixels_per_step': px, 'batch': args.batch,
                   'passes': len(plan_passes(padded, max_images=args.batch))},
        'mpixels_per_s': mpx['ragged'],
        'per_image': {'value': ips['per_image'], 'mpixels_per_s': mpx['per_image'], 'unit': 'images/s',
                      'api': 'one MultiscaleBlueprint.forward + get_loss_per_image per image'},
        'median_ms_per_step': {k: float(np.median(v)) for k, v in ms.items()},
        'speedup': ips['ragged'] / ips['per_image'],
        'mean_bpsp': float(np.mean(last['ragged'])), 'bpsp_equal_per_image': True,
        'gpu': torch.cuda.get_device_name(0), 'power_limit': power,
    }
    print(json.dumps(line))
    return 0


if __name__ == '__main__':
    sys.exit(main())
