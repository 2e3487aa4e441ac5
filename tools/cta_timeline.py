#!/usr/bin/env python
"""When the CTAs of the persistent tensor-core convolutions run inside a bench-shaped step: per launch, from the
records a library built with L3C_CTA_TRACE writes (`python -m l3c_pytorch_b200.build --cta-trace`; this tool
builds it if it is missing and loads it instead of the default library).

    python tools/cta_timeline.py [--workload l3c] [--steps 4] [--schedule 0|1|2] [--json out.json]

The steps are pipelined as in bench.py and tools/step_profile.py.  Per launch, from the CTAs' first and last
%globaltimer readings:
  span         first CTA start -> last CTA exit
  fill         summed CTA lifetimes / (span x CTAs): how much of the grid's SM-time inside its span the CTAs
               actually held; 1 - fill is lost to CTAs that started late or left early
  start spread last CTA start - first CTA start
  tail         share of the span after the median CTA left
Printed per kernel (launch-log name), summed over the launches of the timed steps.  --schedule runs the steps
under engine.conv_tile_schedule (0 dynamic, 1 static stripe).  The GPU name and power limit come first."""
import argparse
import collections
import json
import os
import sys

os.environ['L3C_CTA_TRACE'] = '1'           # before the package is imported: load libl3c_b200_trace.so
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import bench  # noqa: E402
from step_profile import gpu_identity  # noqa: E402

REC_DTYPE = [('t_start', '<u8'), ('t_end', '<u8'), ('smid', '<u4'), ('tiles', '<u4'), ('launch', '<u4'),
             ('cta', '<u4')]                 # l3c_cta_record_t


def launch_stats(recs):
    import numpy as np
    t0, t1 = recs['t_start'].astype(np.int64), recs['t_end'].astype(np.int64)
    span = int(t1.max() - t0.min())
    busy = int((t1 - t0).sum())
    return dict(ctas=len(recs), span=span, busy=busy, spread=int(t0.max() - t0.min()),
                tail=float(t1.max() - np.median(t1)) / span if span else 0.0, tiles=int(recs['tiles'].sum()),
                idle_ctas=int((recs['tiles'] == 0).sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='l3c', choices=['l3c', 'rgb_shared'])
    ap.add_argument('--steps', type=int, default=4)
    ap.add_argument('--lanes', type=int, default=None)
    ap.add_argument('--schedule', type=int, default=0)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()

    import ctypes
    import numpy as np
    import torch
    import l3c_pytorch_b200 as l3c
    from l3c_pytorch_b200 import config, engine as E
    from l3c_pytorch_b200._lib import check, lib

    assert torch.cuda.is_available(), 'cta_timeline.py needs a GPU'
    wl = bench.WORKLOADS[args.workload]
    n_lanes = args.lanes or wl.get('lanes', 4)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    ident = gpu_identity()
    print('GPU (name, power limit, max SM clock): %s' % ident, flush=True)
    E.set_conv_precision(wl['precision'])
    torch.manual_seed(0)
    bp = l3c.MultiscaleBlueprint(config.ms_config(wl['cfg']), device=dev).set_eval()
    codec = l3c.Bitcoding(bp).codec
    n_img, H, W = wl['n_img'], wl['H'], wl['W']
    dev_sets = [bench.make_images(s * n_img, n_img, H, W).to(dev) for s in range(2)]
    lanes = codec.lanes(dev, 3 * n_img, n_lanes)[0]
    enc_streams = codec.encode_streams(dev, 3 * n_img, n_lanes)
    depth = len(enc_streams)

    def run(steps):
        """`steps` round trips, pipelined as bench.py's run_resident does it"""
        cur = torch.cuda.current_stream()
        for s in list(enc_streams) + [ln.main for ln in lanes]:
            s.wait_stream(cur)
        jobs = {}

        def begin(i):
            if i < steps:
                with torch.cuda.stream(enc_streams[i % depth]):
                    jobs[i] = codec.encode_begin(dev_sets[i % 2])

        for i in range(depth):
            begin(i)
        S = None
        for s in range(steps):
            blob, info = jobs.pop(s).finish(to_host=False)
            begin(s + depth)
            ln = lanes[s % n_lanes]
            with torch.cuda.stream(ln.main):
                ln.main.wait_event(info['ready'])
                blob.record_stream(ln.main)
                S = codec.decode_device(blob, info['stream_offsets'], info['lens'],
                                        [(C, h, w) for (_, C, h, w) in info['shapes']], lane=ln)
        for s in list(enc_streams) + [ln.main for ln in lanes]:
            cur.wait_stream(s)
        return S

    cap = 1 << 21
    rec_buf = torch.zeros(cap * 4, dtype=torch.int64, device=dev)
    with E.conv_tile_schedule(args.schedule):
        run(max(n_lanes + 1, args.steps))                       # warm-up, not recorded
        torch.cuda.synchronize()
        check(lib.l3c_cta_trace_register(ctypes.c_void_p(rec_buf.data_ptr()), cap))
        S = run(args.steps)
        torch.cuda.synchronize()
        n = ctypes.c_int64(0)
        text = ctypes.create_string_buffer(1 << 24)
        check(lib.l3c_cta_trace_launches(text, len(text), ctypes.byref(n)))
        check(lib.l3c_cta_trace_register(None, 0))
    assert torch.equal(S, dev_sets[(args.steps - 1) % 2]), 'round trip is not lossless'
    recs = np.frombuffer(rec_buf[:n.value * 4].cpu().numpy().tobytes(), dtype=REC_DTYPE)
    launches = [ln.split() for ln in text.value.decode().splitlines()]
    assert (recs['t_end'] > 0).all(), 'a CTA did not record its exit'

    per = collections.defaultdict(list)
    for idx, name, gx, gy, first, _ in launches:
        first, nc = int(first), int(gx) * int(gy)
        per[name].append(launch_stats(recs[first:first + nc]))
    rows = []
    for name, ls in per.items():
        sm_time = sum(l['span'] * l['ctas'] for l in ls)
        rows.append(dict(name=name, launches=len(ls), span_ms_per_step=sum(l['span'] for l in ls) / 1e6 / args.steps,
                         sm_ms_per_step=sm_time / 1e6 / args.steps,
                         fill=sum(l['busy'] for l in ls) / sm_time if sm_time else 1.0,
                         spread_us=float(np.mean([l['spread'] for l in ls])) / 1e3,
                         tail=float(np.mean([l['tail'] for l in ls])),
                         idle_ctas=sum(l['idle_ctas'] for l in ls), ctas=sum(l['ctas'] for l in ls)))
    rows.sort(key=lambda r: -r['sm_ms_per_step'])
    print('workload %s, schedule %d, %d lanes, %d pipelined steps, %d launches, %d CTAs recorded'
          % (args.workload, args.schedule, n_lanes, args.steps, len(launches), len(recs)))
    print('%-24s %8s %11s %13s %6s %11s %6s %9s' % ('kernel', 'launches', 'span ms/st', 'span*CTAs ms', 'fill',
                                                     'spread us', 'tail', 'idle CTAs'))
    for r in rows:
        print('%-24s %8d %11.2f %13.1f %6.3f %11.1f %6.3f %5d/%d' % (
            r['name'][:24], r['launches'], r['span_ms_per_step'], r['sm_ms_per_step'], r['fill'], r['spread_us'],
            r['tail'], r['idle_ctas'], r['ctas']))
    tot = sum(r['sm_ms_per_step'] for r in rows)
    lost = sum(r['sm_ms_per_step'] * (1 - r['fill']) for r in rows)
    print('all persistent conv launches: %.1f SM-ms per step inside their spans, %.1f %% of it lost to late starts '
          'and idle tails' % (tot, 100 * lost / tot if tot else 0.0))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(gpu=ident, workload=args.workload, schedule=args.schedule, steps=args.steps, rows=rows,
                           lost_share=lost / tot if tot else 0.0), f, indent=1)
    return 0


if __name__ == '__main__':
    sys.exit(main())
