#!/usr/bin/env python
"""bench_large.py -- large images as one tiled container (DESIGN §4.10) against the reference's crop parts, one GPU.

  python tools/bench_large.py [--sizes 4096x3072,6000x4000,8000x6000,16384x16384] [--tile 64] [--mode f16]
                              [--runs 2] [--no-unbanded] [--no-parts]

Workload: one uint8 noise image per size (default about 12, 24 and 48 Mpx), `cr.cf` with seed-0 default-init weights.
Per size, three ways to store it, run alternated `--runs` times after one warm-up of each:
  * whole: one tiled container (tiles of --tile), its encode and decode banded;
  * unbanded: the same container encoded and decoded with banding switched off (codec.TILED_ENCODE_BAND_PIXELS,
    codec.TILED_BAND_PIXELS), where that fits on the card;
  * parts: the image cut by auto_crop into the reference's crops (2000 x 1500 px at most), each a tiled container.
Every figure is a host clock around work that ends in a device synchronise; peak device memory is
torch.cuda.max_memory_allocated above what was allocated before the call.  Every decode is checked lossless.  Also a
512 x 512 decode_region from the whole container.  Prints one JSON line per size with the card name and its power
limit; "oom" marks a call the card could not hold."""
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
    ap.add_argument('--sizes', default='4096x3072,6000x4000,8000x6000', help='WxH,WxH,...')
    ap.add_argument('--tile', type=int, default=64)
    ap.add_argument('--mode', default='f16')
    ap.add_argument('--runs', type=int, default=2)
    ap.add_argument('--no-unbanded', action='store_true')
    ap.add_argument('--no-parts', action='store_true')
    args = ap.parse_args()

    import numpy as np
    import torch
    import l3c_pytorch_b200 as l3c
    from l3c_pytorch_b200 import auto_crop, codec, config, engine as E
    assert torch.cuda.is_available(), 'bench_large.py needs a GPU; there is no CPU fallback'
    torch.cuda.set_device(0)
    dev = torch.device('cuda', 0)
    torch.manual_seed(0)
    bp = l3c.MultiscaleBlueprint(config.ms_config('cr'), device=dev).set_eval()
    E.set_conv_precision(args.mode)
    tile = (args.tile, args.tile)
    bc = l3c.Bitcoding(bp, tile=tile, crop=False)
    budget, enc_budget = codec.TILED_BAND_PIXELS, codec.TILED_ENCODE_BAND_PIXELS
    try:
        power = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                               capture_output=True, text=True, timeout=30).stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None

    def measured(fn):
        """-> (ms, peak MB, result) or ('oom', 'oom', None)."""
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        try:
            out = fn()
            torch.cuda.synchronize()
        except torch.cuda.OutOfMemoryError:
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            return 'oom', 'oom', None
        ms = (time.perf_counter() - t0) * 1e3
        return ms, (torch.cuda.max_memory_allocated() - base) / 2 ** 20, out

    for spec in args.sizes.split(','):
        W, H = (int(v) for v in spec.lower().split('x'))
        g = torch.Generator().manual_seed(1000)
        img = (torch.rand(3, H, W, generator=g) * 255).round().to(torch.uint8)
        x = img.unsqueeze(0).to(dev)
        crops = [c[0] for c in auto_crop.iter_crops(x)]

        def enc_whole(band=True):
            codec.TILED_ENCODE_BAND_PIXELS = enc_budget if band else 1 << 62
            try:
                return bc.codec.encode_batch(x, tile=tile)[0]
            finally:
                codec.TILED_ENCODE_BAND_PIXELS = enc_budget

        def dec_whole(datas, band):
            codec.TILED_BAND_PIXELS = budget if band else 1 << 62
            try:
                return bc.codec.decode_batch(datas, to_host=False)[0]          # uint8 [1, 3, H, W]
            finally:
                codec.TILED_BAND_PIXELS = budget

        def enc_parts():
            return bc.encode_batch(list(crops))[0]

        def lossless(name, out):
            got = auto_crop.stitch(out)[0] if name == 'parts' else out[0]
            return torch.equal(got, x[0].to(got.dtype))

        variants = {'whole': (enc_whole, lambda d: dec_whole(d, True))}
        if not args.no_parts:
            variants['parts'] = (enc_parts, bc.decode_batch)
        if not args.no_unbanded:
            variants['unbanded'] = (lambda: enc_whole(False), lambda d: dec_whole(d, False))
        res = {k: {'enc_ms': [], 'enc_peak_mb': [], 'dec_ms': [], 'dec_peak_mb': []} for k in variants}
        datas_of = {}
        for run in range(args.runs + 1):                  # run 0 warms every shape up and checks the result
            for name, (enc, dcd) in variants.items():
                ms_e, mb_e, datas = measured(enc)
                if datas is None:
                    datas = datas_of.get(name)
                else:
                    datas_of[name] = datas
                ms_d, mb_d, out = ('oom', 'oom', None) if datas is None else measured(lambda: dcd(datas))
                if run == 0:
                    assert out is None or lossless(name, out), '%s: decode is not lossless' % name
                    del out
                    continue
                del out
                res[name]['enc_ms'].append(ms_e)
                res[name]['enc_peak_mb'].append(mb_e)
                res[name]['dec_ms'].append(ms_d)
                res[name]['dec_peak_mb'].append(mb_d)
        region = None
        if datas_of.get('whole'):
            d = datas_of['whole'][0]
            reg = ((H - 512) // 2, (W - 512) // 2, 512, 512)
            bc.decode_region(d, reg)
            region = [measured(lambda: bc.decode_region(d, reg))[:2] for _ in range(max(args.runs, 3))]
        line = {'metric': 'large image: one tiled container (banded encode and decode) vs unbanded vs crop parts',
                'config': {'workload': 'cr.cf seed-0 weights, one 3x%dx%d uint8 noise image (%.1f Mpx), tile %dx%d'
                                       % (H, W, H * W / 1e6, tile[0], tile[1]), 'mode': args.mode, 'runs': args.runs,
                           'band_pixels': budget, 'encode_band_pixels': enc_budget, 'parts': len(crops)},
                'bytes': {k: (sum(len(v) for v in datas_of[k]) if datas_of.get(k) else None) for k in variants},
                'results': res, 'region_512': {'ms_and_peak_mb': region},
                'gpu': torch.cuda.get_device_name(0), 'power_limit': power}
        print(json.dumps(line), flush=True)
        del x, crops, datas_of
        torch.cuda.empty_cache()
    return 0


if __name__ == '__main__':
    sys.exit(main())
