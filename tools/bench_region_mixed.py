#!/usr/bin/env python
"""bench_region_mixed.py -- a serving-like list of region requests of different shapes (DESIGN §4.8 "Batches"), one GPU.

  python tools/bench_region_mixed.py [--mode f16] [--regions 32] [--tile 64] [--iters 5]

Workload: 8 uint8 noise images, four of 1024 x 1536 and four of 1280 x 1920 (seeded), `cr.cf` with seed-0 default-init
weights, coded as tiled containers (default 64 x 64 tiles), and 32 seeded regions of 32 to 512 px a side over them:
a third in the interior, a third touching one image edge, a third in a corner.  Nearly every region has its own
RegionPlan.shape_key, which is what a viewer or tile server sees.

  1. grouped vs one pass: the same decode_regions call with codec.REGION_RAGGED_PASS = False (one pass per shape_key,
     one after another) and True (one ragged pass), alternating, each timed with a host clock around work that ends in
     a device synchronise, after one warm-up call of each.
  2. beside other work: the one-pass call on decode lane 0 while an encode_batch_begin of four images runs on the side
     stream and a decode_batch of four containers runs on lane 1; the wall time of the three together against the
     three run one after another on the current stream.

Every region result is checked against the crop of the full decode, and the lane results against the sequential
ones.  Prints one JSON line with the card name and its power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _regions(sizes, which, n, seed):
    """n regions of 32..512 px a side: interior, touching one edge, in a corner (in turn)."""
    import numpy as np
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        H, W = sizes[which[i]]
        h, w = (int(v) for v in rng.integers(32, 513, 2))
        kind = i % 3
        if kind == 0:
            y, x = int(rng.integers(1, H - h)), int(rng.integers(1, W - w))
        elif kind == 1:
            y, x = [(0, int(rng.integers(1, W - w))), (H - h, int(rng.integers(1, W - w))),
                    (int(rng.integers(1, H - h)), 0), (int(rng.integers(1, H - h)), W - w)][int(rng.integers(4))]
        else:
            y, x = (0 if rng.integers(2) else H - h), (0 if rng.integers(2) else W - w)
        out.append((y, x, h, w))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--regions', type=int, default=32)
    ap.add_argument('--tile', type=int, default=64)
    ap.add_argument('--mode', default='f16')
    ap.add_argument('--iters', type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import torch
    import l3c_pytorch_b200 as l3c
    from l3c_pytorch_b200 import codec, config, engine as E
    assert torch.cuda.is_available(), 'bench_region_mixed.py needs a GPU; there is no CPU fallback'
    torch.cuda.set_device(0)
    dev = torch.device('cuda', 0)
    torch.manual_seed(0)
    bp = l3c.MultiscaleBlueprint(config.ms_config('cr'), device=dev).set_eval()
    E.set_conv_precision(args.mode)
    bc = l3c.Bitcoding(bp, tile=(args.tile, args.tile))
    sizes = [(1024, 1536)] * 4 + [(1280, 1920)] * 4
    imgs = []
    for i, (H, W) in enumerate(sizes):
        g = torch.Generator().manual_seed(1000 + i)
        imgs.append((torch.rand(3, H, W, generator=g) * 255).round().to(torch.uint8))
    datas = bc.encode_batch(torch.stack(imgs[:4]).to(dev))[0] + bc.encode_batch(torch.stack(imgs[4:]).to(dev))[0]
    which = [int(v) for v in np.random.default_rng(7).integers(0, len(sizes), args.regions)]
    regions = _regions(sizes, which, args.regions, 8)
    ds = [datas[k] for k in which]
    _, plans = bc.codec.plan_regions(ds, regions)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    def regions_call(one_pass):
        codec.REGION_RAGGED_PASS = one_pass
        try:
            return bc.decode_regions(ds, regions)
        finally:
            codec.REGION_RAGGED_PASS = True

    # warm-up, and the check: every region of both ways equals the crop of the full decode
    fulls = bc.decode_batch(datas)
    for one_pass in (False, True):
        got = timed(lambda: regions_call(one_pass))[1]
        for k, (y, x, h, w), r in zip(which, regions, got):
            assert torch.equal(r, fulls[k][:, :, y:y + h, x:x + w]), 'region differs from the full decode'
    counts = dict(bc.codec.region_counts)
    del got
    ms = {False: [], True: []}
    for _ in range(args.iters):
        for one_pass in (False, True):
            ms[one_pass].append(timed(lambda: regions_call(one_pass))[0])

    # 2. beside an encode on the side stream and a decode on a second lane
    enc_batch = torch.stack(imgs[:4]).pin_memory()
    dec_datas = datas[:4]
    want_enc = bc.encode_batch(enc_batch)[0]
    want_dec = fulls[:4]
    lanes = bc.decode_lanes(4, n_lanes=2)
    side = bc.side_stream(4, n_lanes=2)

    def together():
        cur = torch.cuda.current_stream()
        job = bc.encode_batch_begin(enc_batch, stream=side)
        for ln in lanes:
            ln.main.wait_stream(cur)
        with torch.cuda.stream(lanes[0].main):
            reg = bc.decode_regions(ds, regions, lane=lanes[0])
        with torch.cuda.stream(lanes[1].main):
            dec = bc.decode_batch(dec_datas, lane=lanes[1])
        enc = job.finish()[0]
        for ln in lanes:
            cur.wait_stream(ln.main)
        return reg, dec, enc

    def sequential():
        return bc.decode_regions(ds, regions), bc.decode_batch(dec_datas), bc.encode_batch(enc_batch)[0]

    ms_tog, ms_seq = [], []
    for it in range(args.iters + 1):
        t_tog, (reg, dec, enc) = timed(together)
        assert enc == want_enc, 'side-stream encode differs'
        assert all(torch.equal(a, b) for a, b in zip(dec, want_dec)), 'lane decode differs'
        for k, (y, x, h, w), r in zip(which, regions, reg):
            assert torch.equal(r, fulls[k][:, :, y:y + h, x:x + w]), 'lane region differs from the full decode'
        t_seq = timed(sequential)[0]
        if it:                                                                   # the first round warms up
            ms_tog.append(t_tog)
            ms_seq.append(t_seq)
    E.set_conv_precision('fp32')
    try:
        power = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                               capture_output=True, text=True, timeout=30).stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None

    def stats(v):
        return {'median': float(np.median(v)), 'min': float(np.min(v)), 'max': float(np.max(v))}

    line = {'metric': 'ms per decode_regions call: per-shape groups vs one ragged pass; and beside other work',
            'config': {'workload': 'cr.cf seed-0 weights, 4 x 1024x1536 + 4 x 1280x1920 uint8 noise, tile %dx%d, '
                                   '%d regions of 32-512 px (interior / edge / corner)'
                                   % (args.tile, args.tile, args.regions),
                       'mode': args.mode, 'iters': args.iters},
            'shape_keys': len({p.shape_key() for p in plans}), 'symbols': counts['symbols'],
            'streams': counts['streams'],
            'grouped': stats(ms[False]), 'one_pass': stats(ms[True]),
            'speedup_median': float(np.median(ms[False]) / np.median(ms[True])),
            'beside_other_work': {'together': stats(ms_tog), 'sequential': stats(ms_seq),
                                  'work': 'decode_regions on lane 0 + decode_batch of 4 x 1024x1536 on lane 1 + '
                                          'encode_batch_begin of 4 x 1024x1536 on the side stream'},
            'gpu': torch.cuda.get_device_name(0), 'power_limit': power}
    print(json.dumps(line))
    return 0


if __name__ == '__main__':
    sys.exit(main())
