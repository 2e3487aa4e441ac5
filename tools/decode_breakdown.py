"""Bring-up helper: CUDA-event breakdown of decode_device phases (monkeypatches the codec)."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import l3c_pytorch_b200 as l3c
from l3c_pytorch_b200 import config, engine as E, codec as C

E.set_conv_precision('tf32')
torch.manual_seed(0)
bp = l3c.MultiscaleBlueprint(config.ms_config('cr')).set_eval()
codec = l3c.BatchCodec(bp)
N = 16
imgs = torch.stack([(torch.rand(3, 512, 512, generator=torch.Generator().manual_seed(1000 + i)) * 255).round().to(torch.uint8) for i in range(N)]).cuda()
marks = []
def mark(name):
    e = torch.cuda.Event(enable_timing=True); e.record(); marks.append((name, e))
orig_getP = bp.net.get_P_nhwc
def getP(scale, bn8, F, **kw):
    mark('getP%d_begin' % scale); r = orig_getP(scale, bn8, F, **kw); mark('getP%d_end' % scale); return r
bp.net.get_P_nhwc = getP
orig_tab = E.dmll_build_table
orig_dec = E.ac_decode_streams
orig_rgb = codec._decode_rgb_pipelined
def rgb(*a, **k):
    mark('rgb_begin'); r = orig_rgb(*a, **k); mark('rgb_end'); return r
codec._decode_rgb_pipelined = rgb
for it in range(3):
    blob, info = codec.encode_batch(imgs, to_host=False)
    shapes = [(C_, H, W) for (_, C_, H, W) in info['shapes']]
    torch.cuda.synchronize(); marks.clear(); mark('start')
    S = codec.decode_device(blob, info['stream_offsets'], info['lens'], shapes)
    mark('end'); torch.cuda.synchronize()
t0 = marks[0][1]
print(json.dumps({n: round(t0.elapsed_time(e), 2) for n, e in marks}))
for nch in ((64,) if '--quick' in sys.argv else (32, 64, 96, 128)):
    codec._decode_rgb_pipelined = lambda *a, **k: orig_rgb(*a, n_chunks=nch, **k)
    best = 1e9
    for it in range(2):
        torch.cuda.synchronize(); a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record(); S = codec.decode_device(blob, info['stream_offsets'], info['lens'], shapes); b.record(); torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b))
    print('n_chunks', nch, 'decode_ms', round(best, 2), bool((S == imgs).all()))
