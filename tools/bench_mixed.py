#!/usr/bin/env python
"""bench_mixed.py -- round trip of images of DIFFERENT sizes (ragged batches, DESIGN §4.6), one GPU.

  python tools/bench_mixed.py [--steps K] [--warmup W] [--images N] [--dump-outputs DIR]

Workload: N (default 16) uint8 noise images of seeded sizes, H and W uniform in [256, 768] (mostly not multiples
of 8), L3C cr.cf with seed-0 default-init weights, precision f16.  Four arms run alternating in one process,
every step runs each once:
  ragged          Bitcoding.encode_batch(list) -> decode_batch, images resident in HBM (one pass per
                  bitcoding.plan_passes group: one network pass and one range-coder launch each)
  ragged_e2e      the same from pinned host images, decoded images copied back to the host
  per_image       one encode_batch / decode_batch per image (the path without ragged batches)
  per_image_e2e   the same from / to the host
Mpixels/s counts unpadded pixels.  Every container of every arm must equal the per-image one and every round
trip must be lossless (asserted).  Prints one JSON line with the card name and its power limit.
`--dump-outputs DIR` writes the container sizes and the decoded images of the last ragged step as DIR/*.npy.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = 'Mpixels/s encode+decode (lossless round-trip), images of different sizes'


def make_image(i, h, w):
    import torch
    g = torch.Generator().manual_seed(1000 + i)
    return (torch.rand(3, h, w, generator=g) * 255).round().to(torch.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--images', type=int, default=16)
    ap.add_argument('--min-side', type=int, default=256)
    ap.add_argument('--max-side', type=int, default=768)
    ap.add_argument('--dump-outputs', metavar='DIR', default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    import l3c_pytorch_b200 as l3c
    from l3c_pytorch_b200 import config, engine as E
    from l3c_pytorch_b200.bitcoding import plan_passes
    assert torch.cuda.is_available(), 'bench_mixed.py needs a GPU; there is no CPU fallback'
    torch.cuda.set_device(0)
    dev = torch.device('cuda', 0)
    E.set_conv_precision('f16')
    torch.manual_seed(0)
    bp = l3c.MultiscaleBlueprint(config.ms_config('cr'), device=dev).set_eval()
    bc = l3c.Bitcoding(bp)
    rng = np.random.default_rng(0)
    sizes = [(int(rng.integers(args.min_side, args.max_side + 1)), int(rng.integers(args.min_side, args.max_side + 1)))
             for _ in range(args.images)]
    imgs = [make_image(i, h, w) for i, (h, w) in enumerate(sizes)]
    host = [im.pin_memory() for im in imgs]
    dev_imgs = [im.to(dev) for im in imgs]
    px = sum(h * w for (h, w) in sizes)
    fac = 2 ** bp.net.config_ms.num_scales
    padded = [(h + (-h) % fac, w + (-w) % fac) for (h, w) in sizes]

    def ragged():
        datas, _ = bc.encode_batch(dev_imgs)
        return datas, bc.decode_batch(datas)

    def ragged_e2e():
        datas, _ = bc.encode_batch_begin(host).finish()
        return datas, [d.cpu() for d in bc.decode_batch(datas)]

    def per_image():
        datas = [bc.encode_batch(im.unsqueeze(0))[0][0] for im in dev_imgs]
        return datas, [bc.decode_batch([d])[0] for d in datas]

    def per_image_e2e():
        datas = [bc.encode_batch(im.unsqueeze(0))[0][0] for im in host]
        return datas, [bc.decode_batch([d])[0].cpu() for d in datas]

    arms = {'ragged': ragged, 'ragged_e2e': ragged_e2e, 'per_image': per_image, 'per_image_e2e': per_image_e2e}
    ms = {k: [] for k in arms}
    last = {}
    for step in range(args.warmup + args.steps):
        for name, fn in arms.items():                   # alternating: every step runs every arm once
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            last[name] = fn()
            b.record()
            torch.cuda.synchronize()
            if step >= args.warmup:
                ms[name].append(a.elapsed_time(b))
    for name, (datas, dec) in last.items():
        assert datas == last['per_image'][0], '%s: containers differ from the per-image encodes' % name
        for im, d in zip(imgs, dec):
            assert torch.equal(d[0].cpu(), im.long()), '%s: round trip is not lossless' % name
    datas, dec = last['ragged']
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, 'container_sizes.npy'), np.asarray([len(d) for d in datas], np.float64))
        for i, d in enumerate(dec):
            np.save(os.path.join(args.dump_outputs, 'decoded_%02d.npy' % i), d[0].cpu().numpy().astype(np.float32))
    mpx = {k: px * len(v) / (sum(v) / 1e3) / 1e6 for k, v in ms.items()}
    try:
        power = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                               capture_output=True, text=True, timeout=30).stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    line = {
        'metric': METRIC, 'value': mpx['ragged'], 'unit': 'Mpixels/s', 'n_gpus': 1, 'steps': args.steps,
        'warmup': args.warmup, 'higher_is_better': True, 'dtype': 'f16', 'data': 'synthetic',
        'config': {'workload': 'L3C cr.cf, %d uint8 noise images of seeded sizes (H, W uniform in [%d, %d])'
                               % (args.images, args.min_side, args.max_side),
                   'sizes': sizes, 'unpadded_pixels_per_step': px, 'passes': len(plan_passes(padded))},
        'e2e': {'value': mpx['ragged_e2e'], 'unit': 'Mpixels/s',
                'api': 'Bitcoding.encode_batch_begin(list of pinned images).finish() -> decode_batch -> host'},
        'per_image': {'value': mpx['per_image'], 'e2e_value': mpx['per_image_e2e'], 'unit': 'Mpixels/s',
                      'api': 'one Bitcoding.encode_batch / decode_batch per image'},
        'median_ms_per_step': {k: float(np.median(v)) for k, v in ms.items()},
        'speedup': mpx['ragged'] / mpx['per_image'], 'speedup_e2e': mpx['ragged_e2e'] / mpx['per_image_e2e'],
        'bpsp': sum(len(d) for d in datas) * 8 / sum(3 * h * w for (h, w) in padded),
        'containers_equal_per_image': True, 'lossless': True,
        'gpu': torch.cuda.get_device_name(0), 'power_limit': power,
    }
    print(json.dumps(line))
    return 0


if __name__ == '__main__':
    sys.exit(main())
