#!/usr/bin/env python
"""bench_recursive.py -- round trip of RECURSIVE containers of the RGB-shared baseline (DESIGN §4.7), one GPU.

  python tools/bench_recursive.py [--steps K] [--warmup W] [--images N] [--size S] [--depths 0,3] [--modes f16,f16x2]

Workload: N (default 16) uint8 noise images of S x S (default 512), cr_rgb_shared.cf with seed-0 default-init
weights.  For every precision mode and every recursion depth R the round trip runs device-resident and pipelined as
bench.py runs it (two encodes queued ahead on the encode streams, the decode of batch s on a decode lane beside
the encodes of batches s+1, s+2), K steps timed with CUDA events around the whole loop.  Beside it, one encode and one
decode are timed on their own (synchronised), so that the growth of the decode's serial range-coder chain with R
shows.  Every round trip is checked lossless.  Prints one JSON line with the card name and its power limit.
At default-init weights recursion makes the files LARGER (the bpsp gain needs a trained checkpoint)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def make_images(first, n, h, w):
    import torch
    out = []
    for i in range(n):
        g = torch.Generator().manual_seed(1000 + first + i)
        out.append((torch.rand(3, h, w, generator=g) * 255).round().to(torch.uint8))
    return torch.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=6)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--images', type=int, default=16)
    ap.add_argument('--size', type=int, default=512)
    ap.add_argument('--depths', default='0,3')
    ap.add_argument('--modes', default='f16,f16x2')
    args = ap.parse_args()

    import numpy as np
    import torch
    import l3c_pytorch_b200 as l3c
    from l3c_pytorch_b200 import config, engine as E
    assert torch.cuda.is_available(), 'bench_recursive.py needs a GPU; there is no CPU fallback'
    torch.cuda.set_device(0)
    dev = torch.device('cuda', 0)
    torch.manual_seed(0)
    bp = l3c.MultiscaleBlueprint(config.ms_config('cr_rgb_shared'), device=dev).set_eval()
    codec = l3c.Bitcoding(bp).codec
    N, S = args.images, args.size
    sets = [make_images(s * N, N, S, S).to(dev) for s in range(2)]
    px_step = N * S * S
    lanes, _, enc_streams = codec.lanes(dev, 3 * N, 1)

    def shapes_of(info):
        return [(C, h, w) for (_, C, h, w) in info['shapes']]

    def pipelined(R, steps):
        """bench.py's resident pipeline: -> (ms, last decoded batch, its containers' sizes)"""
        cur = torch.cuda.current_stream()
        for st in enc_streams + [ln.main for ln in lanes]:
            st.wait_stream(cur)
        jobs = {}

        def begin(i):
            if i < steps:
                with torch.cuda.stream(enc_streams[i % len(enc_streams)]):
                    jobs[i] = codec.encode_begin(sets[i % 2], recursive=R)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(cur)
        for i in range(len(enc_streams)):
            begin(i)
        out = None
        for s in range(steps):
            blob, info = jobs.pop(s).finish(to_host=False)
            begin(s + len(enc_streams))
            ln = lanes[0]
            with torch.cuda.stream(ln.main):
                ln.main.wait_event(info['ready'])
                blob.record_stream(ln.main)
                out = (codec.decode_device(blob, info['stream_offsets'], info['lens'], shapes_of(info), lane=ln),
                       info['sizes'], s % 2)
        for st in enc_streams + [ln.main for ln in lanes]:
            cur.wait_stream(st)
        b.record(cur)
        torch.cuda.synchronize()
        return a.elapsed_time(b), out

    def timed(fn):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        r = fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b), r

    results = {}
    for mode in args.modes.split(','):
        E.set_conv_precision(mode)
        for R in (int(r) for r in args.depths.split(',')):
            pipelined(R, args.warmup)
            ms, (dec, sizes, k) = pipelined(R, args.steps)
            assert torch.equal(dec, sets[k]), '%s R=%d: round trip is not lossless' % (mode, R)
            enc_ms, (blob, info) = timed(lambda: codec.encode_batch(sets[0], to_host=False, recursive=R))
            codec.stage_events = []
            dec_ms, back = timed(lambda: codec.decode_device(blob, info['stream_offsets'], info['lens'],
                                                             shapes_of(info)))
            stages = codec.stage_ms()
            assert torch.equal(back, sets[0])
            results['%s_R%d' % (mode, R)] = {
                'value': px_step * args.steps / (ms / 1e3) / 1e6, 'unit': 'Mpixels/s', 'ms_per_step': ms / args.steps,
                'encode_ms': enc_ms, 'decode_ms': dec_ms, 'decode_stage_ms': stages,
                'bpsp': float(np.sum(sizes)) * 8 / (px_step * 3), 'scales': len(info['shapes'])}
    E.set_conv_precision('fp32')
    try:
        power = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                               capture_output=True, text=True, timeout=30).stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    line = {'metric': 'Mpixels/s encode+decode (lossless round-trip), RGB-shared, recursive containers',
            'n_gpus': 1, 'steps': args.steps, 'warmup': args.warmup, 'data': 'synthetic',
            'config': {'workload': 'cr_rgb_shared.cf seed-0 weights, %d x 3x%dx%d uint8 noise, resident, pipelined'
                                   % (N, S, S)},
            'results': results, 'lossless': True, 'gpu': torch.cuda.get_device_name(0), 'power_limit': power}
    print(json.dumps(line))
    return 0


if __name__ == '__main__':
    sys.exit(main())
