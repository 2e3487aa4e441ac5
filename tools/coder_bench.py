"""Micro-benchmark of the range-coder kernels alone: ns per symbol per stream."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from l3c_pytorch_b200 import engine as E, _lib

def run(L, n_streams, n_sym, peaked, rare=False, own_tables=False, uniform=False, ref_cpu=False):
    dev = torch.device('cuda')
    rng = np.random.default_rng(0)
    pitch = E.table_pitch(L)
    # one random table shared by all streams (content is irrelevant for timing, sizes are not)
    w = rng.integers(1, 40, size=(n_sym, L)).astype(np.float64)
    if peaked:
        w[np.arange(n_sym), rng.integers(0, L, n_sym)] *= (2000 if not rare else 3e7)
    w = w / w.sum(1, keepdims=True) * (65536 - L - 40)
    c = np.floor(np.cumsum(w, 1)).astype(np.int64) + np.arange(1, L + 1)
    cdf = np.concatenate([np.zeros((n_sym, 1), np.int64), c[:, :-1]], 1)          # [n_sym, L]
    hi_all = np.concatenate([cdf[:, 1:], np.full((n_sym, 1), 65536)], 1)
    sym = np.array([rng.choice(L, p=(wi / wi.sum())) for wi in w[:2000]])
    sym = np.resize(sym, n_sym).astype(np.int64)
    if rare:      # symbols drawn uniformly under a peaked model: ~15 bits each (random-init L3C on noise)
        sym = rng.integers(0, L, n_sym).astype(np.int64)
    if uniform:       # the uniform-prior scale: ONE row (l3c_uniform_cdf_row) shared by every symbol, row pitch 0
        row = E.uniform_cdf_row(L).astype(np.int64)
        row[L] = 65536
        cdf = np.repeat(row[None, :L], n_sym, 0); hi_all = np.repeat(row[None, 1:], n_sym, 0)
        sym = rng.integers(0, L, n_sym).astype(np.int64)
    lo = cdf[np.arange(n_sym), sym]; hi = hi_all[np.arange(n_sym), sym]
    iv = torch.from_numpy((lo | ((hi - 1) << 16)).astype(np.uint32).view(np.int32)).to(dev)
    tab = np.zeros((n_sym, pitch), np.uint16); tab[:, :L] = cdf
    tab_dev = torch.from_numpy(tab.view(np.int16)).to(dev)
    cap = ((n_sym * 17 + 7) // 8 + 64 + 3) & ~3
    slots = torch.zeros(n_streams * cap, dtype=torch.uint8, device=dev)
    desc = np.zeros(n_streams, dtype=_lib.ENC_STREAM_DTYPE)
    desc['intervals'] = iv.data_ptr(); desc['n_sym'] = n_sym; desc['out_cap'] = cap
    desc['out'] = slots.data_ptr() + cap * np.arange(n_streams)
    def timed(fn, reps=3):
        best = 1e9
        for _ in range(reps):
            torch.cuda.synchronize(); a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record(); torch.cuda.synchronize(); best = min(best, a.elapsed_time(b))
        return best
    ddev = E._desc_to_device(desc, dev)
    lens = torch.empty(n_streams, dtype=torch.int32, device=dev)
    t_enc = timed(lambda: E.check(E.lib.l3c_ac_encode_streams(E._ptr(ddev), n_streams, E._ptr(lens), E._stream_ptr())))
    nbytes = int(lens[0])
    esz = 2 if L > 256 else 1         # the decoder writes uint16 symbols above 256
    out = torch.zeros(n_streams * n_sym * esz, dtype=torch.uint8, device=dev)
    dd = np.zeros(n_streams, dtype=_lib.DEC_STREAM_DTYPE)
    if own_tables:      # every stream streams its own rows from HBM (as in the real pipeline)
        big = tab_dev.repeat(n_streams, 1)
        dd['table'] = big.data_ptr() + np.arange(n_streams, dtype=np.int64) * (n_sym * pitch * 2)
    else:
        dd['table'] = tab_dev.data_ptr()
    dd['in'] = slots.data_ptr() + cap * np.arange(n_streams)
    dd['sym_out'] = out.data_ptr() + esz * n_sym * np.arange(n_streams); dd['row_pitch'] = 0 if (uniform and not own_tables) else pitch
    dd['n_sym'] = n_sym; dd['in_len'] = nbytes
    dddev = E._desc_to_device(dd, dev)
    t_dec = timed(lambda: E.check(E.lib.l3c_ac_decode_streams(E._ptr(dddev), n_streams, L, 0, n_sym, E._stream_ptr())))
    got = out.cpu().numpy().view(np.uint16 if esz == 2 else np.uint8).reshape(n_streams, n_sym)
    ok = bool((got == sym[None, :]).all())
    extra = {}
    if ref_cpu:       # the compiled reference's decode_cdf of stream 0, one CPU thread
        import time
        from oracle import build_ref
        ref = build_ref.load()
        if ref is not None:
            torch.set_num_threads(1)
            t_cdf = torch.from_numpy(np.concatenate([tab[:, :L], np.zeros((n_sym, 1), np.uint16)], 1).view(np.int16))
            data = slots[:nbytes].cpu().numpy().tobytes()
            t0 = time.perf_counter()
            back = ref.decode_cdf(t_cdf.reshape(1, 1, n_sym, L + 1), data)
            extra = dict(ref_cpu_ns_per_sym=(time.perf_counter() - t0) * 1e9 / n_sym,
                         ref_ok=bool((back.numpy().astype(np.int64) == sym).all()))
    print(json.dumps(dict(L=L, streams=n_streams, n_sym=n_sym, peaked=peaked, rare=rare, own_tables=own_tables, uniform=uniform, bits_per_sym=nbytes * 8 / n_sym,
                          enc_ns_per_sym=t_enc * 1e6 / n_sym, dec_ns_per_sym=t_dec * 1e6 / n_sym, ok=ok, **extra)))

def run_coarse(n_streams, kind, H=128, W=128):
    """The coarse RGB decoder alone (l3c_ac_decode_streams_coarse): n_streams planes of H x W sub-pixels, records
    from l3c_dmll_build_coarse, streams encoded on dmll_table_kernel's full rows.  kind 'bench': sigma ~ 1 bin and
    uniform symbols, as on the noise images of bench.py (most symbols land in linear brackets); 'peaked': one
    dominant component per sub-pixel, symbols at its mode (trained-like: the brackets are evaluated)."""
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    dev = torch.device('cuda')
    C, K, L, HW = 3, 10, 256, H * W
    N = -(-n_streams // C)
    rng = np.random.default_rng(0)
    shp = (N, HW, C, K)
    logit, mean = rng.normal(0, 1, shp), rng.uniform(0, 255, shp)
    if kind == 'bench':
        logs, coef = rng.normal(0, 0.5, shp), rng.normal(0, 1, shp)
        sym = rng.integers(0, 256, (N, C, HW))
    else:
        dom = rng.integers(0, K, (N, HW, C))
        np.put_along_axis(logit, dom[..., None], 8.0, axis=3)
        logs, coef = rng.uniform(-1, 1, shp), np.full(shp, -30.0)            # no channel coupling
        mu = np.take_along_axis(mean, dom[..., None], axis=3)[..., 0]         # [N, HW, C]
        sym = np.clip(np.rint(mu + rng.normal(0, 1, mu.shape)), 0, 255).transpose(0, 2, 1)
    sym = sym.astype(np.uint8)
    l = torch.from_numpy(np.stack([logit, mean, logs, coef], 2).reshape(N, H, W, 4 * C * K).astype(np.float32)).to(dev)
    sym_dev = torch.from_numpy(sym.reshape(N, C, H, W)).to(dev)
    tg = DiscretizedMixLogisticLoss(True, 0, 255, L).targets(dev)
    S = N * C
    rows = torch.zeros(S * HW * L, dtype=torch.int16, device=dev)
    rec = torch.zeros(S * HW * E.COARSE_PITCH, dtype=torch.int16, device=dev)
    for c in range(C):
        E.dmll_build_table(l, sym_dev, tg, C, K, L, True, c, rows)
        E.dmll_build_coarse(l, sym_dev, tg, K, L, c, rec)
    r = rows.view(S, HW, L).to(torch.int64) & 0xFFFF
    s = torch.from_numpy(sym.reshape(S, HW).astype(np.int64)).to(dev)
    lo = r.gather(2, s[..., None])[..., 0]
    hi = torch.where(s < L - 1, r.gather(2, (s + 1).clamp(max=L - 1)[..., None])[..., 0], torch.full_like(s, 65536))
    iv = lo | ((hi - 1) << 16)
    iv = torch.where(iv >= 2 ** 31, iv - 2 ** 32, iv).to(torch.int32).contiguous()
    del rows, r
    # the fraction of symbols whose bracket is linear (mixture_linear() on the records' parameters)
    par = rec.view(S, HW, E.COARSE_PITCH)[..., :64].contiguous().view(torch.float32)       # [S, HW, 32]
    t = tg[:256]
    u0 = (t[0::8][None, None, :, None] - par[..., None, 10:20]) * par[..., None, 20:30]
    u1 = (t[7::8][None, None, :, None] - par[..., None, 10:20]) * par[..., None, 20:30]
    lin = ((u0 <= -25.0) | (u1 >= 40.0)).all(-1)                                            # [S, HW, 32]
    frac_lin = float(lin[:n_streams].gather(2, (s[:n_streams] >> 3)[..., None]).float().mean())
    cap = ((HW * 17 + 7) // 8 + 64 + 3) & ~3
    slots = torch.zeros(S * cap, dtype=torch.uint8, device=dev)
    desc = np.zeros(S, dtype=_lib.ENC_STREAM_DTYPE)
    desc['intervals'] = iv.data_ptr() + 4 * HW * np.arange(S); desc['n_sym'] = HW; desc['out_cap'] = cap
    desc['out'] = slots.data_ptr() + cap * np.arange(S)
    _, lens = E.ac_encode_streams(desc, dev)
    out = torch.zeros(S * HW, dtype=torch.uint8, device=dev)
    dd = np.zeros(S, dtype=_lib.DEC_STREAM_DTYPE)
    dd['table'] = rec.data_ptr() + 2 * E.COARSE_PITCH * HW * np.arange(S); dd['row_pitch'] = E.COARSE_PITCH
    dd['in'] = slots.data_ptr() + cap * np.arange(S); dd['in_len'] = lens.cpu().numpy()
    dd['sym_out'] = out.data_ptr() + HW * np.arange(S); dd['n_sym'] = HW
    ddev = E._desc_to_device(dd, dev)
    times = []
    for _ in range(4):
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); a.record()
        E.ac_decode_streams_coarse(dd, dev, tg, 0, HW, desc_dev=ddev, n=n_streams)
        b.record(); torch.cuda.synchronize(); times.append(a.elapsed_time(b))
    got = out.view(S, HW)[:n_streams].cpu().numpy()
    ok = bool((got == sym.reshape(S, HW)[:n_streams]).all())
    print(json.dumps(dict(coarse=kind, streams=n_streams, n_sym=HW, bits_per_sym=float(lens[:n_streams].float().mean()) * 8 / HW,
                          linear_fraction=frac_lin, dec_ns_per_sym=min(times[1:]) * 1e6 / HW, ok=ok)))


def run_encoder(n_streams, kind, n_sym=262144, reps=5):
    """The encoder alone at the size of an RGB plane of bench.py (512 x 512 symbols per stream), every stream its own
    intervals (one pattern rotated per stream).  kind 'bench': symbols drawn from flat random rows of 256 entries
    (~8 bits per symbol, as on bench.py's noise images); 'peaked': one dominant entry per row, 80 % of the symbols on
    it (~1-2 bits per symbol, trained-like).  Reports the median of `reps` launches after one warm-up launch."""
    dev = torch.device('cuda')
    rng = np.random.default_rng(1)
    L, n_rows = 256, 8192
    w = rng.integers(1, 40, size=(n_rows, L)).astype(np.float64)
    p = rng.integers(0, L, n_rows)
    if kind == 'peaked':
        w[np.arange(n_rows), p] *= 2000
    w = w / w.sum(1, keepdims=True) * (65536 - L)
    c = np.floor(np.cumsum(w, 1)).astype(np.int64) + np.arange(1, L + 1)
    c[:, -1] = 65536
    cdf = np.concatenate([np.zeros((n_rows, 1), np.int64), c], 1)
    sym = rng.integers(0, L, n_rows)
    if kind == 'peaked':
        sym = np.where(rng.random(n_rows) < 0.8, p, sym)
    r = np.arange(n_rows)
    iv1 = torch.from_numpy((cdf[r, sym] | ((cdf[r, sym + 1] - 1) << 16)).astype(np.uint32).view(np.int32))
    base = iv1.repeat(n_sym // n_rows + 1)[:n_sym].to(dev)
    iv = torch.stack([torch.roll(base, 977 * i) for i in range(n_streams)])
    cap = ((n_sym * 17 + 7) // 8 + 64 + 3) & ~3
    slots = torch.zeros(n_streams * cap, dtype=torch.uint8, device=dev)
    desc = np.zeros(n_streams, dtype=_lib.ENC_STREAM_DTYPE)
    desc['intervals'] = iv.data_ptr() + 4 * n_sym * np.arange(n_streams); desc['n_sym'] = n_sym; desc['out_cap'] = cap
    desc['out'] = slots.data_ptr() + cap * np.arange(n_streams)
    ddev = E._desc_to_device(desc, dev)
    lens = torch.empty(n_streams, dtype=torch.int32, device=dev)
    times = []
    for _ in range(reps + 1):
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); a.record()
        E.check(E.lib.l3c_ac_encode_streams(E._ptr(ddev), n_streams, E._ptr(lens), E._stream_ptr()))
        b.record(); torch.cuda.synchronize(); times.append(a.elapsed_time(b))
    t = float(np.median(times[1:]))
    # a digest of every stream's bytes, to compare builds
    ln = lens.cpu().numpy().astype(np.int64)
    h = slots.view(n_streams, cap).to(torch.int64)
    mask = torch.arange(cap, device=dev)[None, :] < torch.from_numpy(ln).to(dev)[:, None]
    digest = int(((h * mask) * torch.arange(1, cap + 1, device=dev)[None, :]).sum()) & 0xFFFFFFFFFFFF
    print(json.dumps(dict(encoder=kind, streams=n_streams, n_sym=n_sym, bits_per_sym=float(ln.mean()) * 8 / n_sym,
                          enc_ms=t, enc_ns_per_sym=t * 1e6 / n_sym, digest=digest)))


if __name__ == '__main__':
    only = int(sys.argv[sys.argv.index('--only') + 1]) if '--only' in sys.argv else None
    if '--encoder' in sys.argv:       # the encoder alone: 1, 48 and 288 streams of an RGB plane of bench.py
        import subprocess
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True).stdout.strip()
        print(json.dumps(dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q)))
        for kind in ('bench', 'peaked'):
            for ns in (1, 48, 288):
                run_encoder(ns, kind)
        sys.exit(0)
    if '--coarse' in sys.argv:        # the coarse RGB decoder (f16 mode, L = 256), 1 and 48 streams
        import subprocess
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True).stdout.strip()
        print(json.dumps(dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q)))
        for kind in ('bench', 'peaked'):
            for ns in (1, 48):
                run_coarse(ns, kind)
        sys.exit(0)
    if '--wide' in sys.argv:          # alphabets above 256 (drop-in torchac range), against the reference on the CPU
        import subprocess
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True).stdout.strip()
        print(json.dumps(dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q)))
        for L in (257, 1024, 4096, 32768):
            n = min(16384, (128 << 20) // (2 * E.table_pitch(L)))      # <= 128 MB of rows per stream
            for ns in (1, 48):
                run(L, ns, n, True, own_tables=ns > 1, ref_cpu=ns == 1)
        sys.exit(0)
    if '--custom' in sys.argv:        # --custom L,streams,n_sym,peaked,rare,own_tables,uniform  (0/1 flags)
        v = [int(x) for x in sys.argv[sys.argv.index('--custom') + 1].split(',')]
        run(v[0], v[1], v[2], bool(v[3]), bool(v[4]), bool(v[5]), bool(v[6]))
        sys.exit(0)
    for ci, (L, ns, n, pk, rare, own, uni) in enumerate([(256, 48, 65536, True, False, False, False), (256, 48, 65536, True, True, False, False),
                                      (25, 80, 65536, True, True, False, False), (256, 48, 65536, True, True, True, False),
                                      (25, 80, 65536, True, True, True, False), (256, 96, 16384, False, False, False, True),
                                      (25, 80, 4096, False, False, False, True)]):
        if only is None or only == ci:
            run(L, ns, n, pk, rare, own, uni)
