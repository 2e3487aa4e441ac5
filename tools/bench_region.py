#!/usr/bin/env python
"""bench_region.py -- region decode of tiled containers (DESIGN §4.8) against the full decode, one GPU.

  python tools/bench_region.py [--images 8] [--height 1024] [--width 1536] [--region 256] [--tile 64] [--mode f16]
                               [--iters 5]

Workload: N (default 8) uint8 noise images of H x W (default 1024 x 1536), `cr.cf` with seed-0 default-init weights,
coded as tiled containers (default 64 x 64 tiles).  One call of `decode_regions` (a region x region crop at the
centre of every image, default 256 x 256) alternates with one call of `decode_batch` on the same containers; each
call is timed with a host clock around work that ends in a device synchronise, after one warm-up call of each.  The
first region call is checked against the crop of the full decode.  Prints one JSON line: ms per call (median, min,
max), symbols handed to the range decoder and decoder-window pixels of both, with the card name and its power
limit."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=8)
    ap.add_argument('--height', type=int, default=1024)
    ap.add_argument('--width', type=int, default=1536)
    ap.add_argument('--region', type=int, default=256)
    ap.add_argument('--tile', type=int, default=64)
    ap.add_argument('--mode', default='f16')
    ap.add_argument('--iters', type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import torch
    import l3c_pytorch_b200 as l3c
    from l3c_pytorch_b200 import config, engine as E
    assert torch.cuda.is_available(), 'bench_region.py needs a GPU; there is no CPU fallback'
    torch.cuda.set_device(0)
    dev = torch.device('cuda', 0)
    torch.manual_seed(0)
    bp = l3c.MultiscaleBlueprint(config.ms_config('cr'), device=dev).set_eval()
    E.set_conv_precision(args.mode)
    bc = l3c.Bitcoding(bp, tile=(args.tile, args.tile))
    N, H, W, R = args.images, args.height, args.width, args.region
    imgs = []
    for i in range(N):
        g = torch.Generator().manual_seed(1000 + i)
        imgs.append((torch.rand(3, H, W, generator=g) * 255).round().to(torch.uint8))
    datas, _ = bc.encode_batch(torch.stack(imgs).to(dev))
    regions = [((H - R) // 2, (W - R) // 2, R, R)] * N

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    # warm-up, and the check: every region equals the crop of the full decode
    _, full = timed(lambda: bc.decode_batch(datas))
    _, regs = timed(lambda: bc.decode_regions(datas, regions))
    y, x = regions[0][:2]
    for f, r in zip(full, regs):
        assert torch.equal(r, f[:, :, y:y + R, x:x + R]), 'region differs from the full decode'
    del full, regs
    counts = dict(bc.codec.region_counts)
    _, plans = bc.codec.plan_regions(datas, regions)
    ms_reg, ms_full = [], []
    for _ in range(args.iters):
        ms_reg.append(timed(lambda: bc.decode_regions(datas, regions))[0])
        ms_full.append(timed(lambda: bc.decode_batch(datas))[0])
    from l3c_pytorch_b200.codec import parse_container
    _, scales = parse_container(datas[0])
    full_symbols = N * sum(C * h * w for (C, h, w, _) in scales)
    full_window = N * sum(h * w for (_, h, w, _) in scales[:-1])          # every net runs on the whole coarser plane
    E.set_conv_precision('fp32')
    try:
        power = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                               capture_output=True, text=True, timeout=30).stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None

    def stats(v):
        return {'median': float(np.median(v)), 'min': float(np.min(v)), 'max': float(np.max(v))}

    line = {'metric': 'ms per call: decode_regions vs decode_batch of tiled containers',
            'config': {'workload': 'cr.cf seed-0 weights, %d x 3x%dx%d uint8 noise, tile %dx%d, %dx%d centre region'
                                   % (N, H, W, args.tile, args.tile, R, R), 'mode': args.mode, 'iters': args.iters},
            'region': {'ms': stats(ms_reg), 'symbols': counts['symbols'], 'streams': counts['streams'],
                       'window_pixels': int(sum(p.window_pixels for p in plans))},
            'full': {'ms': stats(ms_full), 'symbols': full_symbols,
                     'streams': N * sum(len(st) for (_, _, _, st) in scales), 'window_pixels': full_window},
            'speedup_median': float(np.median(ms_full) / np.median(ms_reg)),
            'gpu': torch.cuda.get_device_name(0), 'power_limit': power}
    print(json.dumps(line))
    return 0


if __name__ == '__main__':
    sys.exit(main())
