#!/usr/bin/env python
"""bench_update.py -- region updates of large tiled containers (DESIGN §4.12) against re-encoding the image, one GPU.

  python tools/bench_update.py [--sizes 4096x3072,8000x6000] [--patch 256] [--tile 64] [--mode f16] [--runs 3]
  python tools/bench_update.py --edits K [--containers M] [--sizes 4096x3072] [--patch 256] ...

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
its power limit.

With --edits K (batches of updates, DESIGN §4.12): M = --containers containers of the first size (seeded images), K
patches each at seeded places (anywhere, or with --cluster S inside an S x S square at the centre), three arms
alternated the same way:
  * updates: one Bitcoding.update_regions call for every container and edit;
  * sequential: K update_region calls per container, one after another;
  * dec+enc: per container decode_batch, paste the K patches, encode_batch.
The bytes of the three arms are checked equal.  One JSON line with the plans after merging, the streams re-encoded and
the host stage split of the last update_regions call (BatchCodec.updates_stage_ms: parse, upload, GPU, splice)."""
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
    ap.add_argument('--edits', type=int, default=0, help='K > 0: the batched-update arm, K edits per container')
    ap.add_argument('--containers', type=int, default=1, help='M containers in the batched-update arm')
    ap.add_argument('--cluster', type=int, default=0,
                    help='S > 0: the K patches of a container lie in an S x S square at the image centre (edits close '
                         'together, whose merged window stays within the budget); 0: anywhere in the image')
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
    if args.edits > 0:
        W, H = (int(v) for v in args.sizes.split(',')[0].lower().split('x'))
        g = torch.Generator().manual_seed(100)
        imgs = [torch.randint(0, 256, (3, H, W), generator=g, dtype=torch.uint8).to(dev)
                for _ in range(args.containers)]
        datas = [bc.encode_batch(img.unsqueeze(0))[0][0] for img in imgs]
        if args.cluster > 0:
            S = min(args.cluster, H, W)
            y0, x0, ry, rx = (H - S) // 2, (W - S) // 2, max(S - p, 0) + 1, max(S - p, 0) + 1
        else:
            y0, x0, ry, rx = 0, 0, H - p + 1, W - p + 1
        edits = [[((y0 + int(torch.randint(0, ry, (1,), generator=g)), x0 + int(torch.randint(0, rx, (1,),
                                                                                                  generator=g))),
                   torch.randint(0, 256, (3, p, p), generator=g, dtype=torch.uint8).to(dev))
                  for _ in range(args.edits)] for _ in datas]

        def updates():
            return bc.update_regions(datas, edits)

        def sequential():
            outs = []
            for data, ed in zip(datas, edits):
                for pos, patch in ed:
                    data = bc.update_region(data, pos, patch)
                outs.append(data)
            return outs

        def dec_enc():
            outs = []
            for data, ed in zip(datas, edits):
                dec = bc.decode_batch([data])[0].to(torch.uint8)
                for (y, x), patch in ed:
                    dec[:, :, y:y + p, x:x + p] = patch
                outs.append(bc.encode_batch(dec)[0][0])
            return outs

        arms = {'updates': updates, 'sequential': sequential, 'dec+enc': dec_enc}
        times, peak, outs = {a: [] for a in arms}, {}, {}
        for r in range(args.runs + 1):                             # run 0: warm-up of every arm
            for a, fn in arms.items():
                ms, mb, res = measured(fn)
                outs[a] = res
                if r:
                    times[a].append(ms)
                    peak[a] = max(peak.get(a, 0.0), mb)
                if a == 'updates':
                    stages = dict(bc.codec.updates_stage_ms)
        assert outs['updates'] == outs['sequential'] == outs['dec+enc'], 'batched update bytes differ'
        c = bc.codec.updates_counts
        print(json.dumps(dict(
            size='%dx%d' % (W, H), mpx=round(W * H / 1e6, 1), patch=p, edits=args.edits, containers=args.containers,
            cluster=args.cluster,
            mode=args.mode, tile=tile, plans=[x['plans'] for x in c], streams=sum(x['streams'] for x in c),
            streams_total=sum(x['total'] for x in c), whole=[x['whole'] for x in c],
            ms={a: [round(t, 1) for t in v] for a, v in times.items()},
            median_ms={a: round(float(np.median(v)), 1) for a, v in times.items()},
            stage_ms={k: round(v, 1) for k, v in stages.items()},
            peak_mb={a: round(v) for a, v in peak.items()}, card=card, power_limit=power)), flush=True)
        return
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
