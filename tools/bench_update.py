#!/usr/bin/env python
"""bench_update.py -- region updates of large tiled containers (DESIGN §4.12) against re-encoding the image, one GPU.

  python tools/bench_update.py [--sizes 4096x3072,8000x6000] [--patch 256] [--tile 64] [--mode f16] [--runs 3]

Workload: one seeded uint8 noise image per size (about 12.6 and 48 Mpx), `cr.cf` with seed-0 default-init weights,
tiles of --tile, its container written once.  Per size and per place of a --patch x --patch patch (the centre and
the top-left corner), three arms, alternated --runs times after one warm-up of each:
  * update: Bitcoding.update_region of the container;
  * dec+enc: decode_batch of the container, paste, encode_batch of the whole edited image -- what a caller who holds
    only the container does without update_region;
  * enc: encode_batch of the edited image alone -- a caller who holds the pixels.
Every figure is a host clock around work that ends in a device synchronise; peak device memory is
torch.cuda.max_memory_allocated above what was allocated before the call.  The update's bytes are checked against the
encode's.  Prints one JSON line per size and place with the streams re-encoded, the window pixels, the card name and
its power limit."""
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
    ap.add_argument('--sizes', default='4096x3072,8000x6000', help='WxH,WxH,...')
    ap.add_argument('--patch', type=int, default=256)
    ap.add_argument('--tile', type=int, default=64)
    ap.add_argument('--mode', default='f16')
    ap.add_argument('--runs', type=int, default=3)
    args = ap.parse_args()

    import numpy as np
    import torch
    import l3c_pytorch_b200 as l3c
    from l3c_pytorch_b200 import config, engine as E
    assert torch.cuda.is_available(), 'bench_update.py needs a GPU; there is no CPU fallback'
    torch.cuda.set_device(0)
    dev = torch.device('cuda', 0)
    torch.manual_seed(0)
    bp = l3c.MultiscaleBlueprint(config.ms_config('cr'), device=dev).set_eval()
    E.set_conv_precision(args.mode)
    tile = (args.tile, args.tile)
    bc = l3c.Bitcoding(bp, tile=tile, crop=False)
    try:
        power = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                               capture_output=True, text=True, timeout=30).stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    card = torch.cuda.get_device_name(0)

    def measured(fn):
        """-> (ms, peak MB above the memory allocated before the call, result)."""
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        res = fn()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        return ms, (torch.cuda.max_memory_allocated() - base) / 2 ** 20, res

    p = args.patch
    for k, size in enumerate(args.sizes.split(',')):
        W, H = (int(v) for v in size.lower().split('x'))
        g = torch.Generator().manual_seed(k)
        img = torch.randint(0, 256, (3, H, W), generator=g, dtype=torch.uint8).to(dev)
        data = bc.encode_batch(img.unsqueeze(0))[0][0]
        patch = torch.randint(0, 256, (3, p, p), generator=g, dtype=torch.uint8).to(dev)
        for place, (y, x) in (('centre', ((H - p) // 2, (W - p) // 2)), ('corner', (0, 0))):
            edited = img.clone()
            edited[:, y:y + p, x:x + p] = patch

            def update():
                return bc.update_region(data, (y, x), patch)

            def dec_enc():
                dec = bc.decode_batch([data])[0].to(torch.uint8)
                dec[:, :, y:y + p, x:x + p] = patch
                return bc.encode_batch(dec)[0][0]

            def enc():
                return bc.encode_batch(edited.unsqueeze(0))[0][0]

            arms = {'update': update, 'dec+enc': dec_enc, 'enc': enc}
            times = {a: [] for a in arms}
            peak = {}
            outs = {}
            for r in range(args.runs + 1):                         # run 0: warm-up of every arm
                for a, fn in arms.items():
                    ms, mb, res = measured(fn)
                    outs[a] = res
                    if r:
                        times[a].append(ms)
                        peak[a] = max(peak.get(a, 0.0), mb)
            assert outs['update'] == outs['enc'] == outs['dec+enc'], 'update bytes differ from the encode'
            c = bc.codec.update_counts
            print(json.dumps(dict(
                size='%dx%d' % (W, H), mpx=round(W * H / 1e6, 1), patch=p, place=place, mode=args.mode, tile=tile,
                streams=c['streams'], streams_total=c['total'], window_pixels=c['window_pixels'], whole=c['whole'],
                ms={a: [round(t, 1) for t in v] for a, v in times.items()},
                median_ms={a: round(float(np.median(v)), 1) for a, v in times.items()},
                peak_mb={a: round(v) for a, v in peak.items()}, bytes=len(outs['update']),
                card=card, power_limit=power)), flush=True)


if __name__ == '__main__':
    main()
