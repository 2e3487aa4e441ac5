#!/usr/bin/env python
"""Where the GPU time of a bench-shaped step goes: per-kernel totals of warmed, pipelined round trips of the
bench.py workload under torch.profiler (CUDA activities), grouped by the name the kernel has in the library's
launch log.

    python tools/step_profile.py [--workload l3c] [--steps 4] [--lanes 4] [--json out.json]

The steps run exactly as bench.py pipelines them (encodes of the next batches on the encode streams beside the
decodes of earlier ones, `--lanes` decodes in flight).  Kernel times of concurrent streams overlap, so the
shares are of the summed kernel time, not of the wall time; the wall time per step of the same steps without
the profiler is printed beside them.  The GPU name and power limit are part of every number and are printed
first.
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload table, seeded images, CUDA_DEVICE_MAX_CONNECTIONS as the bench sets it)

# kernels whose launch-log name is not their function name (one template, several launch names)
LAUNCH_NAMES = [
    ('conv_f16_kernel<0>', 'conv3x3_f16_kernel'),
    ('conv_f16_kernel<1>', 'conv5x5s2_f16_kernel'),
    ('conv1x1_tc_kernel<0,', 'conv1x1_tf32_kernel'),
    ('conv1x1_tc_kernel<1,', 'conv1x1_f16_kernel'),
    ('conv1x1_tc_kernel<2,', 'conv1x1_f16x2_kernel'),
    ('ac_decode32_kernel', 'ac_decode_kernel'),
]
CONV_KERNELS = ('conv3x3_f16_kernel', 'conv5x5s2_f16_kernel', 'conv1x1_f16_kernel', 'lin_dmll_f16_kernel',
                'conv3x3_tf32_kernel', 'conv1x1_tf32_kernel', 'conv3x3_f16x2_kernel', 'conv1x1_f16x2_kernel',
                'conv_ffma_kernel')


def launch_name(kernel):
    """CUDA kernel name as the profiler reports it -> launch-log name (torch's own kernels: 'torch: <name>')"""
    k = re.sub(r'\s+', '', re.sub(r'^void\s+', '', kernel).replace('(anonymous namespace)', ''))
    for pat, name in LAUNCH_NAMES:
        if pat in k:
            return name
    base = re.sub(r'[<(].*', '', k).rsplit('::', 1)[-1]      # drop the template, the arguments, the namespaces
    return base if k.startswith('l3c::') else 'torch: ' + base[:60]


def gpu_identity():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else 'nvidia-smi printed nothing'
    except (OSError, subprocess.TimeoutExpired):
        return 'nvidia-smi unavailable'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='l3c', choices=['l3c', 'rgb_shared'])
    ap.add_argument('--precision', default=None)
    ap.add_argument('--steps', type=int, default=4, help='pipelined round trips under the profiler')
    ap.add_argument('--lanes', type=int, default=None)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import l3c_pytorch_b200 as l3c
    from l3c_pytorch_b200 import config, engine as E

    assert torch.cuda.is_available(), 'step_profile.py needs a GPU'
    wl = bench.WORKLOADS[args.workload]
    precision = args.precision or wl['precision']
    n_lanes = args.lanes or wl.get('lanes', 4)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    ident = gpu_identity()
    print('GPU (name, power limit, max SM clock): %s' % ident, flush=True)
    E.set_conv_precision(precision)
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
                es = enc_streams[i % depth]
                with torch.cuda.stream(es):
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

    # warm-up: every lane and encode stream (allocator pools, modules), then one timed run without the profiler
    run(max(n_lanes + 1, args.steps))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    S = run(args.steps)
    e1.record()
    torch.cuda.synchronize()
    wall_ms = e0.elapsed_time(e1) / args.steps
    assert torch.equal(S, dev_sets[(args.steps - 1) % 2]), 'round trip is not lossless'

    E.launch_log(reset=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(args.steps)
        torch.cuda.synchronize()
    logged, logged_total = E.launch_log(reset=True)

    tot, cnt = collections.Counter(), collections.Counter()
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name
        if name.startswith('Memcpy') or name.startswith('Memset'):
            key = 'copy: ' + name.split()[0]
        else:
            key = launch_name(name)
        tot[key] += ev.time_range.elapsed_us() / 1e3
        cnt[key] += 1
    T = sum(tot.values())
    conv = sum(v for k, v in tot.items() if k in CONV_KERNELS)
    rows = [dict(name=k, launches=cnt[k], launch_log=logged.get(k), ms_per_step=v / args.steps, share=v / T)
            for k, v in sorted(tot.items(), key=lambda kv: -kv[1])]
    print('workload %s (%s), %d lanes, %d pipelined steps; wall %.2f ms per step without the profiler'
          % (args.workload, precision, n_lanes, args.steps, wall_ms))
    print('%-40s %9s %9s %12s %7s' % ('kernel (launch-log name)', 'launches', 'log', 'ms per step', 'share'))
    for r in rows:
        if r['share'] < 0.0005:
            continue
        print('%-40s %9d %9s %12.3f %6.1f%%' % (r['name'][:40], r['launches'], r['launch_log'] if r['launch_log']
                                                 is not None else '-', r['ms_per_step'], 100 * r['share']))
    print('summed kernel time %.2f ms per step; conv kernels %.2f ms per step = %.1f %% of it; %d launches in the '
          'launch log' % (T / args.steps, conv / args.steps, 100 * conv / T, logged_total))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(gpu=ident, workload=args.workload, precision=precision, lanes=n_lanes, steps=args.steps,
                           wall_ms_per_step=wall_ms, kernel_ms_per_step=T / args.steps,
                           conv_ms_per_step=conv / args.steps, kernels=rows), f, indent=1)
    return 0


if __name__ == '__main__':
    sys.exit(main())
