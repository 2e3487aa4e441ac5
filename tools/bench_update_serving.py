#!/usr/bin/env python
"""bench_update_serving.py -- region updates served beside region decodes (DESIGN §4.12, "Serving updates"), one GPU.

  python tools/bench_update_serving.py [--size 4096x3072] [--containers 2] [--regions 16] [--region 256]
                                       [--edits 2] [--patch 128] [--tile 64] [--mode f16] [--rounds 8] [--runs 3]

Workload: --containers seeded uint8 noise images of --size, `cr.cf` with seed-0 default-init weights, tiled containers
of --tile written once.  A round is one decode_regions call of --regions seeded --region x --region crops spread over
the containers, and one update_regions call of --edits seeded --patch x --patch patches per container.  Two arms of
--rounds rounds each, alternated --runs times after one warm-up of each:
  * serial: per round the region decode on decode lane 0, then the update on lane 1, each waited for before the next;
  * overlapped: per round the region decode is queued on lane 0 and update_regions_begin on lane 1, then the update's
    finish() and, at the end of the arm, lane 0 are waited for.
Every time is a host clock around work that ends in a device synchronise.  The regions and the update bytes of the
two arms are checked equal.  Prints one JSON line: region Mpx/s and updates/s (update calls per second) of each arm,
the card name and its power limit."""
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
    ap.add_argument('--size', default='4096x3072', help='WxH')
    ap.add_argument('--containers', type=int, default=2)
    ap.add_argument('--regions', type=int, default=16)
    ap.add_argument('--region', type=int, default=256)
    ap.add_argument('--edits', type=int, default=2)
    ap.add_argument('--patch', type=int, default=128)
    ap.add_argument('--tile', type=int, default=64)
    ap.add_argument('--mode', default='f16')
    ap.add_argument('--rounds', type=int, default=8)
    ap.add_argument('--runs', type=int, default=3)
    args = ap.parse_args()

    import numpy as np
    import torch
    import l3c_pytorch_b200 as l3c
    from l3c_pytorch_b200 import config, engine as E
    assert torch.cuda.is_available(), 'bench_update_serving.py needs a GPU; there is no CPU fallback'
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

    W, H = (int(v) for v in args.size.lower().split('x'))
    g = torch.Generator().manual_seed(300)
    imgs = [torch.randint(0, 256, (3, H, W), generator=g, dtype=torch.uint8).to(dev) for _ in range(args.containers)]
    datas = [bc.encode_batch(img.unsqueeze(0))[0][0] for img in imgs]
    r, p = min(args.region, H, W), min(args.patch, H, W)

    def place(size):
        return int(torch.randint(0, H - size + 1, (1,), generator=g)), int(torch.randint(0, W - size + 1, (1,),
                                                                                         generator=g))

    rounds = []
    for _ in range(args.rounds):
        which = [i % len(datas) for i in range(args.regions)]
        regions = [place(r) + (r, r) for _ in which]
        edits = [[(place(p), torch.randint(0, 256, (3, p, p), generator=g, dtype=torch.uint8).to(dev))
                  for _ in range(args.edits)] for _ in datas]
        rounds.append(([datas[i] for i in which], regions, edits))
    lanes = bc.decode_lanes(max(args.regions, args.containers), n_lanes=2)
    cur = torch.cuda.current_stream()

    def serial():
        regs, outs = [], []
        for ds, regions, edits in rounds:
            with torch.cuda.stream(lanes[0].main):
                regs.append(bc.decode_regions(ds, regions, lane=lanes[0]))
            lanes[0].main.synchronize()
            with torch.cuda.stream(lanes[1].main):
                outs.append(bc.update_regions_begin(datas, edits, lane=lanes[1]).finish())
        return regs, outs

    def overlapped():
        regs, outs = [], []
        for ds, regions, edits in rounds:
            with torch.cuda.stream(lanes[0].main):
                regs.append(bc.decode_regions(ds, regions, lane=lanes[0]))
            with torch.cuda.stream(lanes[1].main):
                job = bc.update_regions_begin(datas, edits, lane=lanes[1])
            outs.append(job.finish())
        lanes[0].main.synchronize()
        return regs, outs

    arms = {'serial': serial, 'overlapped': overlapped}
    times, res = {a: [] for a in arms}, {}
    for run in range(args.runs + 1):                               # run 0: warm-up of every arm
        for a, fn in arms.items():
            torch.cuda.synchronize()
            for ln in lanes:
                ln.main.wait_stream(cur)
            t0 = time.perf_counter()
            res[a] = fn()
            torch.cuda.synchronize()
            if run:
                times[a].append(time.perf_counter() - t0)
    for x, y in zip(res['serial'][0], res['overlapped'][0]):
        assert all(torch.equal(u, v) for u, v in zip(x, y)), 'regions differ between the arms'
    assert res['serial'][1] == res['overlapped'][1], 'update bytes differ between the arms'
    mpx = args.rounds * args.regions * r * r / 1e6
    med = {a: float(np.median(v)) for a, v in times.items()}
    print(json.dumps(dict(
        size='%dx%d' % (W, H), containers=args.containers, regions=args.regions, region=r, edits=args.edits, patch=p,
        mode=args.mode, tile=tile, rounds=args.rounds,
        s={a: [round(t, 3) for t in v] for a, v in times.items()},
        region_mpx_s={a: round(mpx / t, 1) for a, t in med.items()},
        updates_s={a: round(args.rounds / t, 2) for a, t in med.items()},
        overlap_gain=round(med['serial'] / med['overlapped'], 3), card=card, power_limit=power)), flush=True)


if __name__ == '__main__':
    main()
