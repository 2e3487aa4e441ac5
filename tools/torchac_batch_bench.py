"""Batched torchac calls against a loop of one-stream calls and the reference's CPU coder.

    python tools/torchac_batch_bench.py [--reps 3] [--quick]

Arms, per case (B streams of peaked tables from the test stream factory at alphabet L, CPU tensors as the drop-in
API takes them):
  batched      encode_cdf_batch / decode_cdf_batch on the CPU tables
  batched_dev  the same on tables and symbols already on the GPU
  loop         encode_cdf / decode_cdf, one call per stream
  ref_cpu      the compiled reference's encode_cdf / decode_cdf (oracle/_ref), one CPU thread -- when present
Each time is a whole call (host-to-device copies, kernels, device-to-host copies) between CUDA events closed by a
synchronise, after one warm-up call; the median of --reps.  Reported per case: ns per symbol per stream
(time / symbols of one stream) and aggregate Msymbols/s (all symbols / time).  One JSON line per case, then the
GPU's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from l3c_pytorch_b200 import torchac  # noqa: E402
from tests.test_gpu_coder_launches import make_stream  # noqa: E402

ROW_CAP = 128 << 20          # table bytes per stream
CASE_CAP = 2 << 30           # table bytes per case
N_MAX = 4096


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'unknown'
    return dict(gpu=name, power_limit_and_max_sm_clock=q)


def timed(fn, reps):
    fn()
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) * 1e-3)
    return statistics.median(out)


def wall(fn, reps):
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        out.append(time.perf_counter() - t0)
    return statistics.median(out)


def streams(Ls, B, seed):
    """B peaked streams at the alphabets Ls (cycled); 4 distinct tables per alphabet, reused"""
    rng = np.random.default_rng(seed)
    row = 2 * (max(Ls) + 1)
    n = int(min(N_MAX, ROW_CAP // row, CASE_CAP // (B * row)))
    made = {}
    out = []
    for i in range(B):
        L = Ls[i % len(Ls)]
        k = (L, (i // len(Ls)) % 4)
        if k not in made:
            s = make_stream(rng, 'peaked', n, L)
            made[k] = (torch.from_numpy(s.cdf.view(np.int16)).reshape(1, 1, n, L + 1), torch.from_numpy(s.sym))
        out.append(made[k])
    return n, out


def run_case(Ls, B, reps, ref):
    n, ss = streams(Ls, B, 1000 + B + sum(Ls))
    cdfs = [c for c, _ in ss]
    syms = [s for _, s in ss]
    res = dict(L=Ls[0] if len(Ls) == 1 else 'mixed:' + '/'.join(map(str, Ls)), B=B, n_sym=n)
    datas = torchac.encode_cdf_batch(cdfs, syms)
    back = torchac.decode_cdf_batch(cdfs, datas)
    ok = all(torch.equal(b, s) for b, s in zip(back, syms))
    ok = ok and all(torchac.encode_cdf(cdfs[i], syms[i]) == datas[i] for i in {0, B - 1})
    res['bits_per_sym'] = 8.0 * sum(map(len, datas)) / (B * n)
    dcdfs = [c.cuda() for c in cdfs]
    dsyms = [s.cuda() for s in syms]
    arms = {
        'batched': (lambda: torchac.encode_cdf_batch(cdfs, syms), lambda: torchac.decode_cdf_batch(cdfs, datas)),
        'batched_dev': (lambda: torchac.encode_cdf_batch(dcdfs, dsyms),
                        lambda: torchac.decode_cdf_batch(dcdfs, datas)),
        'loop': (lambda: [torchac.encode_cdf(c, s) for c, s in zip(cdfs, syms)],
                 lambda: [torchac.decode_cdf(c, d) for c, d in zip(cdfs, datas)]),
    }
    for name, (enc, dec) in arms.items():
        for what, fn in (('enc', enc), ('dec', dec)):
            t = timed(fn, reps)
            res['%s_%s_ns_per_sym' % (name, what)] = t * 1e9 / n
            res['%s_%s_msym_s' % (name, what)] = B * n / t * 1e-6
    if ref is not None:
        threads = torch.get_num_threads()
        torch.set_num_threads(1)
        ok = ok and ref.encode_cdf(cdfs[0], syms[0]) == datas[0]
        for what, fn in (('enc', lambda: [ref.encode_cdf(c, s) for c, s in zip(cdfs, syms)]),
                         ('dec', lambda: [ref.decode_cdf(c, d) for c, d in zip(cdfs, datas)])):
            t = wall(fn, max(1, reps // 2))
            res['ref_cpu_%s_ns_per_sym' % what] = t * 1e9 / n
            res['ref_cpu_%s_msym_s' % what] = B * n / t * 1e-6
        torch.set_num_threads(threads)
    res['ok'] = bool(ok)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--quick', action='store_true', help='B in {1, 48}, L in {25, 1024}')
    ap.add_argument('--no-ref', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('torchac_batch_bench needs a GPU')
    ref = None
    if not a.no_ref:
        try:
            from oracle import build_ref
            ref = build_ref.load()
        except Exception as e:          # the reference is optional: its arm is then "not measured"
            print(json.dumps(dict(ref_cpu='not measured: %s' % e)), flush=True)
    Bs, Ls = ((1, 48), (25, 1024)) if a.quick else ((1, 16, 48, 256), (25, 256, 1024, 32768))
    cases = [((L,), B) for L in Ls for B in Bs] + [((25, 256, 1024, 32768), 48)]
    for Lc, B in cases:
        print(json.dumps(run_case(list(Lc), B, a.reps, ref)), flush=True)
    print(json.dumps(gpu_info()), flush=True)


if __name__ == '__main__':
    main()
