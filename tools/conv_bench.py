"""Micro-benchmark of the conv kernels by layer type and precision mode (CUDA events, L2-cold inputs by
size: every tensor is far larger than the 50 MB L2 at the default shape).

    python tools/conv_bench.py [--n 16] [--hw 256] [--modes f16,tf32] [--reps 20] [--cases pair,down]

Layer types (the shapes an L3C round trip is made of):
  res1   first conv of a ResBlock: 3x3 64->64 + ReLU, output feeds only the next tensor-core conv ('round')
  res2   second conv: 3x3 64->64 + fp32 residual, fp32 output + operand image ('act')
  pair   res1 followed by res2 (one ResBlock)
  plain  3x3 64->64, fp32 output only
  tail   3x3 64->256 + PixelShuffle(2), 'act' (decoder features of scales 1, 2) / 'round' (scale 0)
  atr4   3x3 dilation 4 into a slice of the 192-channel concat buffer ('round')
  lin    1x1 192->120 on the concat buffer (the DMLL parameters); lin_fused: the same conv with the DMLL head in
         its epilogue (coding intervals out, encode side; tf32: the two-step path for comparison)
  down   5x5 stride 2 on the operand image: f16 runs the tensor-core kernel (conv5x5s2_f16_kernel), tf32 and
         f16x2 the CUDA-core kernel on the fp32 input; its FLOPs and bytes are per INPUT pixel (four per output
         pixel)
Prints ms per launch, TFLOP/s, and algorithmic HBM bytes per launch / GB/s (what the layer must move, per
DESIGN.md 4.1).
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=16)
    ap.add_argument('--hw', type=int, default=256)
    ap.add_argument('--modes', default='f16,tf32')
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--cases', default=None, help='comma-separated subset of the layer types (default: all)')
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    import l3c_pytorch_b200 as l3c
    from l3c_pytorch_b200 import config, engine as E
    from l3c_pytorch_b200.network import default_conv
    dev = torch.device('cuda', 0)
    torch.manual_seed(0)
    N, H = args.n, args.hw
    px = N * H * H
    c33 = default_conv(64, 64, 3).to(dev)
    c33b = default_conv(64, 64, 3).to(dev)
    ctail = default_conv(64, 256, 3).to(dev)
    catr = default_conv(64, 64, 3, rate=4).to(dev)
    clin = default_conv(192, 120, 1).to(dev)
    cdown = default_conv(64, 64, 5, stride=2).to(dev)
    results = {}
    for mode in args.modes.split(','):
        E.set_conv_precision(mode)
        op_b = 2 if mode == 'f16' else 4                  # bytes per operand-image element
        x = torch.randn(N, H, H, 64, device=dev)
        xa = E.as_operand(x)
        res = torch.randn(N, H, H, 64, device=dev)
        cat_dtype = torch.float16 if mode in ('f16', 'f16x2') else torch.float32
        cat = torch.randn(N, H, H, 384 if mode == 'f16x2' else 192, device=dev).to(cat_dtype)
        cat_act = E.Act(None, cat) if mode in ('f16', 'f16x2') else E.Act(cat, cat)
        mid = {}
        sym = torch.randint(0, 256, (N, 3, H, H), dtype=torch.uint8, device=dev)
        tgt = torch.linspace(-0.5, 255.5, 257, device=dev)

        def res1():
            mid['r'] = E.conv2d(c33, xa, relu=True, want='round')

        def res2():
            E.conv2d(c33b, mid['r'], residual=res, want='act')

        def pair():
            res1()
            res2()

        cases = {
            'res1': (res1, 2 * 9 * 64 * 64, 64 * op_b + 64 * op_b),
            'res2': (res2, 2 * 9 * 64 * 64, 64 * op_b + 256 + 256 + 64 * op_b),
            'pair': (pair, 4 * 9 * 64 * 64, 64 * op_b * 4 + 512),
            'plain': (lambda: E.conv2d(c33, xa), 2 * 9 * 64 * 64, 64 * op_b + 256),
            'tail_act': (lambda: E.conv2d(ctail, xa, pixel_shuffle=True, want='act'), 2 * 9 * 64 * 256,
                         64 * op_b + 1024 + 256 * op_b),
            'tail_round': (lambda: E.conv2d(ctail, xa, pixel_shuffle=True, want='round'), 2 * 9 * 64 * 256,
                           64 * op_b + 256 * op_b),
            'atr4': (lambda: E.conv2d(catr, xa, out=cat, out_coff=64, want='round'), 2 * 9 * 64 * 64, 64 * op_b * 2),
            'lin': (lambda: E.conv2d(clin, cat_act), 2 * 192 * 120, 192 * op_b + 480),
            'lin_fused': ((lambda: E.lin_dmll_intervals(clin, cat, sym, tgt, 3, 10, 256, True)) if mode == 'f16'
                          else (lambda: E.dmll_intervals(E.conv2d(clin, cat_act), sym, tgt, 3, 10, 256, True)),
                          2 * 192 * 120, 192 * op_b + 3 + 12),
            # f16 reads the FP16 operand image, the CUDA-core kernel of the other modes the fp32 input
            'down': (lambda: E.conv2d(cdown, xa, want='act'), 2 * 25 * 64 * 64 / 4.0,
                     (64 * op_b if mode == 'f16' else 256) + (256 + 64 * op_b) / 4.0),
        }
        for name, (fn, flop_px, bytes_px) in cases.items():
            if args.cases and name not in args.cases.split(','):
                continue
            try:
                for _ in range(3):
                    fn()
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.reps):
                    fn()
                b.record()
                torch.cuda.synchronize()
                ms = a.elapsed_time(b) / args.reps
                r = dict(ms=ms, tflops=flop_px * px / ms / 1e9, alg_MB=bytes_px * px / 1e6,
                         alg_GBps=bytes_px * px / ms / 1e6)
            except Exception as ex:                        # keep going: one broken case must not hide the others
                r = dict(error=str(ex)[:200])
            results['%s/%s' % (mode, name)] = r
            print('%-5s %-10s %s' % (mode, name, ' '.join('%s=%.4g' % kv if not isinstance(kv[1], str) else '%s=%s' % kv
                                                         for kv in r.items())), flush=True)
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(dict(n=N, hw=H, results=results), f, indent=1)


if __name__ == '__main__':
    main()
