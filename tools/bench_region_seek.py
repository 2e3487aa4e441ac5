#!/usr/bin/env python
"""bench_region_seek.py -- region decodes of seek-indexed reference-layout containers (DESIGN §4.13 "Regions") against
the whole indexed decode they replace, one GPU.

  python tools/bench_region_seek.py [--steps K] [--warmup W] [--every 4096] [--requests 1,16]

Workload: `cr` with seed-0 default-init weights, f16, uint8 noise images in the reference layout with a seek index every
K symbols: a 2000 x 1500 image (one container, at the reference's crop threshold) and a 4000 x 3000 image (stored as 4
parts of 2000 x 1500, as the reference stores it).  Arms per image, alternated inside every step and each timed with
CUDA events around one synchronised call:
  * whole: decode_batch of every container (every part) from its index;
  * 256^2, 1024^2, strip64 (64 rows, full width): N requests in one decode_regions call, at N = 1 and 16, every
    region inside one container (part), at seeded positions;
  * 1024^2 across parts (4000 x 3000 only): one decode_region_file call on a region that meets all 4 parts.
Every result is checked against the crop of the whole decode, and every arm runs in the warm-up steps first.  Prints
the median ms, the symbols the range decoders decoded, the decoder-window pixels and the peak memory of every arm, and
one JSON line with the card's name and power limit, read in the same call.  Files go to a temporary directory."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--every', type=int, default=4096)
    ap.add_argument('--requests', default='1,16')
    args = ap.parse_args()

    import numpy as np
    import torch
    import l3c_pytorch_b200 as l3c
    from l3c_pytorch_b200 import auto_crop, config, part_suffix_helper, seek as _seek
    from l3c_pytorch_b200.codec import parse_container
    assert torch.cuda.is_available(), 'bench_region_seek.py needs a GPU; there is no CPU fallback'
    torch.cuda.set_device(0)
    dev = torch.device('cuda', 0)
    l3c.set_conv_precision('f16')
    torch.manual_seed(0)
    bp = l3c.MultiscaleBlueprint(config.ms_config('cr'), device=dev).set_eval()
    bc = l3c.Bitcoding(bp)
    K = args.every
    reqs = [int(n) for n in args.requests.split(',')]
    tmp = tempfile.mkdtemp(prefix='l3c_bench_region_seek_')

    def timed(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b), out, torch.cuda.max_memory_allocated()

    results = []
    for H, W in [(1500, 2000), (3000, 4000)]:
        g = torch.Generator().manual_seed(H)
        img = (torch.rand(1, 3, H, W, generator=g) * 255).round().to(torch.uint8)
        pout = os.path.join(tmp, '%dx%d.l3c' % (W, H))
        bc.encode(img.long(), pout, seek=K)
        paths = [pout] if os.path.isfile(pout) else part_suffix_helper.existing_parts(pout)
        datas = [open(p, 'rb').read() for p in paths]
        seeks = [open(p + '.seek', 'rb').read() for p in paths]
        shapes = []
        for d in datas:
            (left, right, top, bottom), scales = parse_container(d)
            shapes.append((scales[-1][1] - top - bottom, scales[-1][2] - left - right))
        rects = auto_crop.part_rects(shapes)
        want = img.to(dev).long()

        def whole():
            parts = bc.decode_batch(datas, seeks=seeks)
            return auto_crop.stitch(parts) if len(parts) > 1 else parts[0]

        rng = np.random.default_rng(H)
        arms, expect, arm_items = {'whole': whole}, {'whole': [(0, 0, H, W)]}, {}
        for name, (h, w) in [('256^2', (256, 256)), ('1024^2', (1024, 1024)), ('strip64', (64, None))]:
            for N in reqs:
                items = []
                for _ in range(N):
                    i = int(rng.integers(len(rects)))
                    py, px, ph, pw = rects[i]
                    ww = pw if w is None else w
                    y, x = int(rng.integers(0, ph - h + 1)), int(rng.integers(0, pw - ww + 1))
                    items.append((i, (y, x, h, ww), (py + y, px + x, h, ww)))
                key = '%s x%d' % (name, N)
                arms[key] = (lambda items: lambda: bc.decode_regions(
                    [datas[i] for i, _, _ in items], [r for _, r, _ in items], seeks=[seeks[i] for i, _, _ in items]))(
                    items)
                expect[key] = [r for _, _, r in items]
                arm_items[key] = items
        if len(paths) > 1:
            reg = (H // 2 - 512, W // 2 - 512, 1024, 1024)
            arms['1024^2 across parts'] = lambda: [bc.decode_region_file(pout, reg)]
            expect['1024^2 across parts'] = [reg]
        in_file = int(sum(int(_seek.stream_symbols(d).sum()) for d in datas))
        windows = {'whole': 0}                     # decoder-window pixels the plans of every region arm run on
        for key, regs in expect.items():
            if key == 'whole':
                continue
            if key == '1024^2 across parts':
                y, x, h, w = regs[0]
                cut = [(i, (max(y, r[0]) - r[0], max(x, r[1]) - r[1], min(y + h, r[0] + r[2]) - max(y, r[0]),
                            min(x + w, r[1] + r[3]) - max(x, r[1]))) for i, r in enumerate(rects)]
            else:
                cut = [(i, r) for i, r, _ in arm_items[key]]
            _, plans = bc.codec.plan_regions([datas[i] for i, _ in cut], [r for _, r in cut],
                                             seeks=[seeks[i] for i, _ in cut])
            windows[key] = sum(p.window_pixels for p in plans)
        ms = {k: [] for k in arms}
        stats = {}
        for step in range(args.warmup + args.steps):
            for name, fn in arms.items():
                t, out, peak = timed(fn)
                out = [out] if torch.is_tensor(out) else out
                for got, (y, x, h, w) in zip(out, expect[name]):
                    assert torch.equal(got, want[:, :, y:y + h, x:x + w]), name
                if step >= args.warmup:
                    ms[name].append(t)
                stats[name] = {'symbols': bc.codec.region_counts['symbols'] if name != 'whole' else in_file,
                               'window_pixels': windows[name], 'peak_bytes': peak}
        row = {'image': '%dx%d' % (W, H), 'parts': len(paths), 'every': K,
               'symbols_in_file': in_file,
               'arms': {k: {'ms': float(np.median(v)), **stats[k]} for k, v in ms.items()}}
        results.append(row)
        for k, v in row['arms'].items():
            print('%s %-22s %9.2f ms  %11d symbols  %10d window px  peak %7.0f MB' % (
                row['image'], k, v['ms'], v['symbols'], v['window_pixels'], v['peak_bytes'] / 2 ** 20))
    shutil.rmtree(tmp, ignore_errors=True)
    try:
        power = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = None
    print(json.dumps({'bench': 'region_seek', 'config': 'cr', 'precision': 'f16', 'results': results,
                      'checked': True, 'gpu': torch.cuda.get_device_name(0), 'power_limit': power}))


if __name__ == '__main__':
    main()
