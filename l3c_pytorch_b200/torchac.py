"""Drop-in for the reference's `torchac` module (/root/reference/src/torchac/torchac.py:87-166):
same four functions, same argument meaning, same exceptions -- backed by libl3c_b200.so instead of
the pybind modules torchac_backend_{cpu,gpu}.

Differences by design: there is no CPU backend (CPU_SUPPORTED is False; `encode_cdf`/`decode_cdf`
still take CPU tensors, as in the reference, but the coding runs on the GPU), and no CDF table is
materialised for `encode_logistic_mixture`.

Beyond the reference: `encode_cdf_batch`, `decode_cdf_batch`, `encode_logistic_mixture_batch` and
`decode_logistic_mixture_batch` code a list of streams in one call, with the results of the one-stream functions.
"""
import ctypes

import numpy as np
import torch

from . import _lib, engine as E
from ._lib import lib, check

CUDA_SUPPORTED = _lib.cuda_supported()
CPU_SUPPORTED = False


def _np_ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _require_backend():
    if not _lib.cuda_supported():
        raise ValueError('torchac (l3c_pytorch_b200) needs an sm_90 GPU; there is no CPU backend.')


def _check_cdf(cdf):
    if cdf.dim() != 4 or cdf.shape[0] != 1:
        raise RuntimeError('Invalid size for cdf! Expected 1HWLp')        # torchac.cpp:135
    if cdf.dtype != torch.int16:
        raise RuntimeError('cdf must be int16')
    return np.ascontiguousarray(cdf.numpy()).view(np.uint16).reshape(-1, cdf.shape[-1])


def encode_cdf(cdf, sym):
    """cdf: 1HWLp int16 on CPU; sym: int16 on CPU -> bytes."""
    if cdf.is_cuda or sym.is_cuda:
        raise ValueError('CDF and symbols must be on CPU for `encode_cdf`')
    _require_backend()
    table = _check_cdf(cdf)
    s = np.ascontiguousarray(sym.numpy().astype(np.int16, copy=False)).reshape(-1)
    if s.size != table.shape[0]:
        raise RuntimeError('sym has %d entries, cdf describes %d symbols' % (s.size, table.shape[0]))
    cap = s.size * 3 + 64
    out = np.empty(cap, np.uint8)
    n = ctypes.c_size_t(0)
    check(lib.l3c_encode_cdf(_np_ptr(table), table.shape[0], table.shape[1], _np_ptr(s), _np_ptr(out), cap,
                             ctypes.byref(n)))
    return out[:n.value].tobytes()


def decode_cdf(cdf, input_string):
    """cdf: 1HWLp int16 on CPU -> int16 tensor [H*W] on CPU."""
    if cdf.is_cuda:
        raise ValueError('CDF must be on CPU for `decode_cdf`')
    _require_backend()
    table = _check_cdf(cdf)
    buf = np.frombuffer(bytes(input_string), np.uint8)
    out = np.empty(table.shape[0], np.int16)
    check(lib.l3c_decode_cdf(_np_ptr(table), table.shape[0], table.shape[1],
                             _np_ptr(buf) if buf.size else None, buf.size, _np_ptr(out)))
    return torch.from_numpy(out)


def _check_mixture(targets, means, log_scales, logit_probs_softmax):
    if not (targets.is_cuda == means.is_cuda == log_scales.is_cuda == logit_probs_softmax.is_cuda):
        raise ValueError('targets, means, log_scales, logit_probs_softmax must all be on the same device! Got '
                         f'{targets.device}, {means.device}, {log_scales.device}, {logit_probs_softmax.device}.')
    if not targets.is_cuda:
        raise ValueError('Got CPU tensor, but l3c_pytorch_b200 has no CPU backend; move the tensors to the GPU.')
    if means.dim() != 4 or means.shape[0] != 1:
        raise RuntimeError('Invalid size for means! Expected 1KHW')           # torchac.cpp:239
    if means.shape != log_scales.shape or means.shape != logit_probs_softmax.shape:
        raise RuntimeError('Invalid size for log_scales/logit_probs_softmax! Expected 1KHW')
    ts = [t.float().contiguous() for t in (targets, means, log_scales, logit_probs_softmax)]
    return ts, means.shape[1], means.shape[2] * means.shape[3], targets.shape[0]


def encode_logistic_mixture(targets, means, log_scales, logit_probs_softmax, sym):
    """targets [Lp], means/log_scales/logit_probs_softmax 1KHW (CUDA); sym int16 on CPU -> bytes."""
    (t, m, ls, pi), K, n_sym, Lp = _check_mixture(targets, means, log_scales, logit_probs_softmax)
    if sym.is_cuda:
        raise ValueError('sym must be on CPU!')
    s = np.ascontiguousarray(sym.numpy().astype(np.int16, copy=False)).reshape(-1)
    if s.size != n_sym:
        raise RuntimeError('sym has %d entries, parameters describe %d symbols' % (s.size, n_sym))
    cap = n_sym * 3 + 64
    out = np.empty(cap, np.uint8)
    n = ctypes.c_size_t(0)
    torch.cuda.current_stream().synchronize()       # inputs may have been produced on another stream
    check(lib.l3c_encode_logistic_mixture(t.data_ptr(), m.data_ptr(), ls.data_ptr(), pi.data_ptr(), K, n_sym, Lp,
                                          _np_ptr(s), _np_ptr(out), cap, ctypes.byref(n)))
    return out[:n.value].tobytes()


def decode_logistic_mixture(targets, means, log_scales, logit_probs_softmax, input_string):
    (t, m, ls, pi), K, n_sym, Lp = _check_mixture(targets, means, log_scales, logit_probs_softmax)
    buf = np.frombuffer(bytes(input_string), np.uint8)
    out = np.empty(n_sym, np.int16)
    torch.cuda.current_stream().synchronize()
    check(lib.l3c_decode_logistic_mixture(t.data_ptr(), m.data_ptr(), ls.data_ptr(), pi.data_ptr(), K, n_sym, Lp,
                                          _np_ptr(buf) if buf.size else None, buf.size, _np_ptr(out)))
    return torch.from_numpy(out)


# ----------------------------------------------------------------------------------------------
# Batched calls: many streams per call (include/l3c_b200.h sections B and F; DESIGN §4.4)
# ----------------------------------------------------------------------------------------------
# Device scratch of one batched call, in bytes.  A decode builds the rows its decoders read chunk by chunk, and the
# rows of one chunk, summed over its streams, stay under this; an encode codes its streams in groups whose intervals
# (4 B per symbol) and output slots (17 bits per symbol) stay under it.  A stream whose encode scratch alone exceeds
# it is a group of its own.  1 GiB holds 16384 rows of L = 32768 (341 symbols of each of 48 such streams per chunk).
BATCH_SCRATCH_BYTES = 1 << 30
# symbols per stream a decode group is sized for: streams whose rows for this many symbols exceed the scratch
# together are decoded one group after the other
MIN_CHUNK_SYMBOLS = 64
# side streams the decoder launches of different alphabets run on (per device); more alphabets share them
MAX_SIDE_STREAMS = 8
PACK_MAX_STREAMS = 65535            # l3c_pack_streams: streams per launch (grid.y)

_SIDE = {}


def row_bytes(L):
    """bytes of one decoder row for alphabet(s) L (numpy-friendly)"""
    L = np.asarray(L, np.int64)
    return 2 * np.where(L <= 32, 32, np.where(L <= 256, 256, (L + 7) // 8 * 8))


SLOT_CAP_MAX = (1 << 32) - 4        # the encoder's out_cap is a uint32 multiple of 4


def slot_caps(n_sym):
    """encoder slot bytes of streams of n_sym symbols: 17 bits per symbol (every symbol on a 1-count interval) and the
    terminator, clamped to SLOT_CAP_MAX (from about 2.02e9 symbols on; such a stream must code below 16 bits per
    symbol, else _pack_offsets refuses it)"""
    n = np.asarray(n_sym, np.int64)
    return np.minimum(((n * 17 + 7) // 8 + 64 + 3) & ~3, SLOT_CAP_MAX)


def enc_scratch_bytes(n_sym):
    """encode scratch of streams of n_sym symbols: 4 B of intervals per symbol and the coder's output slot"""
    return 4 * np.asarray(n_sym, np.int64) + slot_caps(n_sym)


def _pack_offsets(len_words, caps, streams):
    """The encoder's output lengths of the streams `streams` (uint32, as the int32 words of the device buffer) ->
    (lengths int64, pack offsets int64 [len + 1]).  RuntimeError, before anything is packed, when a stream did not fit
    its slot: the coder then wrote only its first caps bytes."""
    lens = np.asarray(len_words).view(np.uint32).astype(np.int64)
    over = np.flatnonzero(lens > caps)
    if over.size:
        k = int(over[0])
        raise RuntimeError('stream %d: range coder output of %d bytes exceeded its slot of %d bytes (rows not strictly '
                           'increasing?)' % (int(streams[k]), int(lens[k]), int(caps[k])))
    return lens, np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)


def plan_decode(n_sym, L, cap=None):
    """The decoder launches of a batched decode: -> [(streams, first, count)], in launch order.  `streams` are the
    indices (sorted by L, then index) of the streams that still have symbols at `first`; each of them decodes
    symbols [first, first + count) clipped to its length, and the rows of those symbols, summed over the streams,
    stay under `cap` bytes (default BATCH_SCRATCH_BYTES).  Streams are grouped by L, and split into groups that are
    decoded one after the other when their rows for MIN_CHUNK_SYMBOLS symbols each would exceed the cap together."""
    cap = BATCH_SCRATCH_BYTES if cap is None else int(cap)
    n = np.asarray(n_sym, np.int64).reshape(-1)
    Ls = np.asarray(L, np.int64).reshape(-1)
    if n.size == 0:
        return []
    rb = row_bytes(Ls)
    if int(rb.max()) > cap:
        raise ValueError('batched decode: a scratch of %d bytes cannot hold one row of L=%d (%d bytes)'
                         % (cap, int(Ls[rb.argmax()]), int(rb.max())))
    groups, cur, need = [], [], 0
    for j in np.lexsort((np.arange(n.size), Ls)):
        want = int(rb[j]) * min(int(n[j]), MIN_CHUNK_SYMBOLS)
        if cur and need + want > cap:
            groups.append(np.array(cur, np.int64))
            cur, need = [], 0
        cur.append(int(j))
        need += want
    groups.append(np.array(cur, np.int64))
    chunks = []
    for g in groups:
        first, n_max = 0, int(n[g].max())
        while first < n_max:
            act = g[n[g] > first]
            rem, b = n[act] - first, rb[act]
            count = int(rem.max())
            if int((rem * b).sum()) > cap:           # the largest count whose rows fit (1 always does)
                lo, hi = 1, count
                while lo < hi:
                    mid = (lo + hi + 1) // 2
                    if int((np.minimum(rem, mid) * b).sum()) <= cap:
                        lo = mid
                    else:
                        hi = mid - 1
                count = lo
            chunks.append((act, first, count))
            first += count
    return chunks


def plan_encode(n_sym, cap=None):
    """Streams coded together by a batched encode: -> [index arrays] in input order, each group's encode scratch
    (enc_scratch_bytes) under `cap` (default BATCH_SCRATCH_BYTES); a stream above it alone is a group of its own."""
    cap = BATCH_SCRATCH_BYTES if cap is None else int(cap)
    need = enc_scratch_bytes(n_sym).reshape(-1)
    groups, start, acc = [], 0, 0
    for j in range(need.size):
        if j > start and acc + int(need[j]) > cap:
            groups.append(np.arange(start, j))
            start, acc = j, 0
        acc += int(need[j])
    if need.size:
        groups.append(np.arange(start, need.size))
    return groups


def _side_streams(dev, k):
    pool = _SIDE.setdefault(dev.index, [])
    while len(pool) < min(k, MAX_SIDE_STREAMS):
        pool.append(torch.cuda.Stream(device=dev))
    return pool


def _streams(*seqs):
    """the argument sequences as lists of one length -> (lists, number of streams)"""
    seqs = [list(q) for q in seqs]
    if len({len(q) for q in seqs}) != 1:
        raise ValueError('every argument needs one entry per stream; got %s entries'
                         % ' / '.join(str(len(q)) for q in seqs))
    return seqs, len(seqs[0])


def _one_device(tensors, what):
    devs = {t.device for t in tensors}
    if len(devs) != 1:
        raise ValueError('%s must all be on one device; got %s' % (what, ', '.join(sorted(map(str, devs)))))
    return devs.pop()


def _check_lp_nsym(i, n_sym, Lp):
    if not 2 <= Lp <= 32769:
        raise RuntimeError('stream %d: Lp=%d not in [2,32769]' % (i, Lp))
    if not 1 <= n_sym < (1 << 31):
        raise RuntimeError('stream %d: n_sym=%d not in [1, 2^31)' % (i, n_sym))


def _table_sources(cdfs):
    """Checks the tables (one-stream errors, with the stream index) -> (device, src descriptors, n_sym, Lp, keep).
    CPU tables are concatenated in pinned memory and copied to the device once."""
    dev = _one_device(cdfs, 'CDF tables')
    n = np.zeros(len(cdfs), np.int64)
    Lp = np.zeros(len(cdfs), np.int64)
    for i, cdf in enumerate(cdfs):
        if cdf.dim() != 4 or cdf.shape[0] != 1:
            raise RuntimeError('stream %d: Invalid size for cdf! Expected 1HWLp' % i)
        if cdf.dtype != torch.int16:
            raise RuntimeError('stream %d: cdf must be int16' % i)
        n[i], Lp[i] = cdf.shape[1] * cdf.shape[2], cdf.shape[3]
        _check_lp_nsym(i, int(n[i]), int(Lp[i]))
    _require_backend()
    src = np.zeros(len(cdfs), dtype=_lib.CODE_SRC_DTYPE)
    src['n_sym'], src['Lp'] = n, Lp
    if dev.type == 'cpu':
        dev = torch.device('cuda', torch.cuda.current_device())
        off = np.concatenate([[0], np.cumsum(n * Lp)])
        host = torch.empty(int(off[-1]), dtype=torch.int16, pin_memory=True)
        torch.cat([c.reshape(-1) for c in cdfs], out=host)          # torch's CPU threads share the copy
        tab = host.to(dev, non_blocking=True)
        src['table'] = tab.data_ptr() + 2 * off[:-1]
        return dev, src, n, Lp, [tab], True
    keep = [c.contiguous() for c in cdfs]
    src['table'] = [t.data_ptr() for t in keep]
    return dev, src, n, Lp, keep, False


def _mixture_sources(targets, means, log_scales, logit_probs_softmax):
    m = len(targets)
    src = np.zeros(m, dtype=_lib.CODE_SRC_DTYPE)
    keep = []
    for i in range(m):
        try:
            (t, mu, ls, pi), K, n_sym, Lp = _check_mixture(targets[i], means[i], log_scales[i], logit_probs_softmax[i])
        except (ValueError, RuntimeError) as e:
            raise type(e)('stream %d: %s' % (i, e)) from None
        _check_lp_nsym(i, n_sym, Lp)
        keep += [t, mu, ls, pi]
        src[i] = (0, t.data_ptr(), mu.data_ptr(), ls.data_ptr(), pi.data_ptr(), 0, n_sym, Lp, K)
    dev = _one_device(keep, 'mixture parameters')
    _require_backend()
    return dev, src, src['n_sym'].astype(np.int64), src['Lp'].astype(np.int64), keep


def _symbols(syms, n, Lp, dev, src, keep, allowed):
    """Symbols into the descriptors: CPU symbols are checked here and copied to the device once; CUDA symbols are
    used in place (the interval kernel checks them).  -> the CUDA symbol tensors, or None for CPU symbols."""
    if len(syms) != len(n):
        raise ValueError('%d symbol tensors for %d streams' % (len(syms), len(n)))
    sdev = _one_device(syms, 'symbols')
    if sdev not in allowed:
        raise ValueError('symbols on %s, stream sources on %s' % (sdev, ' / '.join(map(str, allowed))))
    for i, s in enumerate(syms):
        if s.numel() != n[i]:
            raise RuntimeError('stream %d: sym has %d entries, the stream describes %d symbols' % (i, s.numel(), n[i]))
    if sdev.type == 'cpu':
        off = np.concatenate([[0], np.cumsum(n)])
        host = torch.empty(int(off[-1]), dtype=torch.int16, pin_memory=True)
        hv = host.numpy()
        for i, s in enumerate(syms):
            v = s.numpy().astype(np.int16, copy=False).reshape(-1)
            bad = np.flatnonzero((v < 0) | (v > Lp[i] - 2))
            if bad.size:
                raise RuntimeError('stream %d: symbol %d at position %d outside [0,%d]'
                                   % (i, int(v[bad[0]]), int(bad[0]), int(Lp[i]) - 2))
            hv[off[i]:off[i + 1]] = v
        sym_dev = host.to(dev, non_blocking=True)
        keep.append(sym_dev)
        src['sym'] = sym_dev.data_ptr() + 2 * off[:-1]
        return None
    flat = [s.reshape(-1).to(torch.int16).contiguous() for s in syms]
    keep += flat
    src['sym'] = [s.data_ptr() for s in flat]
    return flat


def _encode_group(dev, src, n, Lp, cuda_syms, g):
    """one interval launch, one encoder launch and one pack for the streams g -> [bytes]"""
    ng = len(g)
    ng_src = np.ascontiguousarray(src[g])
    sym_off = np.concatenate([[0], np.cumsum(n[g])]).astype(np.int64)
    total = int(sym_off[-1])
    caps = slot_caps(n[g])
    slot_off = np.concatenate([[0], np.cumsum(caps)])
    src_dev = E._desc_to_device(ng_src, dev)
    off_dev = E._to_device_async(sym_off, dev)
    iv = torch.empty(total, dtype=torch.int32, device=dev)
    bad_lens = torch.empty(2 * ng, dtype=torch.int32, device=dev)
    check(lib.l3c_batch_intervals(E._ptr(src_dev), E._ptr(off_dev), ng, total, E._ptr(iv), E._ptr(bad_lens),
                                  E._stream_ptr()))
    slots = torch.empty(int(slot_off[-1]), dtype=torch.uint8, device=dev)
    desc = np.zeros(ng, dtype=_lib.ENC_STREAM_DTYPE)
    desc['intervals'] = iv.data_ptr() + 4 * sym_off[:-1]
    desc['out'] = slots.data_ptr() + slot_off[:-1]
    desc['n_sym'] = n[g]
    desc['out_cap'] = caps
    desc_dev = E._desc_to_device(desc, dev)
    lens_ptr = ctypes.c_void_p(bad_lens.data_ptr() + 4 * ng)
    check(lib.l3c_ac_encode_streams(E._ptr(desc_dev), ng, lens_ptr, E._stream_ptr()))
    E.LAUNCHES['n'] += 2
    host = torch.empty(2 * ng, dtype=torch.int32, pin_memory=True)
    host.copy_(bad_lens, non_blocking=True)
    torch.cuda.current_stream().synchronize()
    bad = host.numpy()[:ng].astype(np.int64)
    for k in np.flatnonzero(bad >= 0):
        i = int(g[k])
        sym = int(cuda_syms[i][int(bad[k])].item()) if cuda_syms is not None else None
        raise RuntimeError('stream %d: symbol %s at position %d outside [0,%d]' % (i, sym, int(bad[k]), int(Lp[i]) - 2))
    lens, dst = _pack_offsets(host.numpy()[ng:], caps, g)
    blob = torch.empty(int(dst[-1]) + 16, dtype=torch.uint8, device=dev)
    dst_dev = E._to_device_async(dst[:-1], dev)
    esz = np.dtype(_lib.ENC_STREAM_DTYPE).itemsize
    for a in range(0, ng, PACK_MAX_STREAMS):
        b = min(ng, a + PACK_MAX_STREAMS)
        check(lib.l3c_pack_streams(ctypes.c_void_p(desc_dev.data_ptr() + esz * a),
                                   ctypes.c_void_p(bad_lens.data_ptr() + 4 * (ng + a)),
                                   ctypes.c_void_p(dst_dev.data_ptr() + 8 * a), b - a, E._ptr(blob), E._stream_ptr()))
        E.LAUNCHES['n'] += 1
    out = torch.empty(blob.shape, dtype=torch.uint8, pin_memory=True)
    out.copy_(blob, non_blocking=True)
    torch.cuda.current_stream().synchronize()
    buf = out.numpy()
    return [buf[dst[k]:dst[k + 1]].tobytes() for k in range(ng)]


def _encode_batch(dev, src, n, Lp, syms, keep, allowed):
    with torch.cuda.device(dev):
        cuda_syms = _symbols(syms, n, Lp, dev, src, keep, allowed)
        res = []
        for g in plan_encode(n):
            res += _encode_group(dev, src, n, Lp, cuda_syms, g)
        return res


def _decode_batch(dev, src, n, Lp, strings, to_cpu):
    """the chunks of plan_decode: per chunk one row launch on the current stream, then one decoder launch per
    alphabet, each alphabet on its own side stream; the next chunk's rows wait for every decoder of this one"""
    m = len(n)
    if len(strings) != m:
        raise ValueError('%d input strings for %d streams' % (len(strings), m))
    L = Lp - 1
    bufs = [bytes(s) for s in strings]
    in_len = np.array([len(b) for b in bufs], np.int64)
    if (in_len >= (1 << 32)).any():
        raise RuntimeError('stream %d: input of %d bytes' % (int(in_len.argmax()), int(in_len.max())))
    in_off = np.concatenate([[0], np.cumsum(in_len)])
    wide = L > 256
    out_off = np.zeros(m, np.int64)                   # in the uint8 buffer (narrow) or the int16 one (wide)
    for mask in (~wide, wide):
        out_off[mask] = np.concatenate([[0], np.cumsum(n[mask])[:-1]]) if mask.any() else []
    n8, n16 = int(n[~wide].sum()), int(n[wide].sum())
    chunks = plan_decode(n, L)
    with torch.cuda.device(dev):
        cur = torch.cuda.current_stream()
        host_in = torch.zeros(int(in_off[-1]) + 8, dtype=torch.uint8, pin_memory=True)
        hv = host_in.numpy()
        for i, b in enumerate(bufs):
            hv[in_off[i]:in_off[i + 1]] = np.frombuffer(b, np.uint8)
        blob = host_in.to(dev, non_blocking=True)
        out8 = torch.empty(max(n8, 1), dtype=torch.uint8, device=dev)
        out16 = torch.empty(max(n16, 1), dtype=torch.int16, device=dev)
        state = torch.empty(_lib.DEC_STATE_WORDS * m, dtype=torch.int32, device=dev)
        rows = torch.empty(max(int((np.minimum(n[s] - f, c) * row_bytes(L[s])).sum()) for s, f, c in chunks) // 2,
                           dtype=torch.int16, device=dev)
        alphabets = sorted(set(L.tolist()), key=lambda x: (x > 256, x))     # narrow first: the wide launch waits
        side = _side_streams(dev, len(alphabets))
        side_of = {a: side[k % len(side)] for k, a in enumerate(alphabets)}
        pitch = row_bytes(L) // 2
        ssz, dsz = np.dtype(_lib.CODE_SRC_DTYPE).itemsize, np.dtype(_lib.DEC_STREAM_DTYPE).itemsize
        keep, done = [], []
        for (act, first, count) in chunks:
            k = act.size
            r = np.minimum(n[act] - first, count)
            row_off = np.concatenate([[0], np.cumsum(r * pitch[act])]).astype(np.int64)
            dd = np.zeros(k, dtype=_lib.DEC_STREAM_DTYPE)
            dd['table'] = rows.data_ptr() + 2 * (row_off[:-1] - first * pitch[act])
            dd['in'] = blob.data_ptr() + in_off[act]
            dd['sym_out'] = np.where(wide[act], out16.data_ptr() + 2 * out_off[act], out8.data_ptr() + out_off[act])
            dd['state'] = state.data_ptr() + 4 * _lib.DEC_STATE_WORDS * act
            dd['row_pitch'] = pitch[act]
            dd['n_sym'] = n[act]
            dd['in_len'] = in_len[act]
            packed = np.concatenate([np.ascontiguousarray(src[act]).view(np.uint8), row_off.view(np.uint8),
                                     dd.view(np.uint8)])
            for ev in done:                              # the rows buffer is free once every decoder has read it
                cur.wait_event(ev)
            done = []
            meta = E._to_device_async(packed, dev)
            keep.append(meta)
            p = meta.data_ptr()
            check(lib.l3c_batch_rows(ctypes.c_void_p(p), ctypes.c_void_p(p + ssz * k), k, int(row_off[-1]), first,
                                     E._ptr(rows), E._stream_ptr()))
            E.LAUNCHES['n'] += 1
            built = torch.cuda.Event()
            built.record(cur)
            d0 = p + ssz * k + 8 * (k + 1)
            La = L[act]
            for a in alphabets:
                sel = np.flatnonzero(La == a)
                if not sel.size:
                    continue
                s = side_of[a]
                s.wait_event(built)
                check(lib.l3c_ac_decode_streams(ctypes.c_void_p(d0 + dsz * int(sel[0])), int(sel.size), int(a), first,
                                                count, ctypes.c_void_p(s.cuda_stream)))
                E.LAUNCHES['n'] += 1
                ev = torch.cuda.Event()
                ev.record(s)
                done.append(ev)
        for ev in done:
            cur.wait_event(ev)
        if to_cpu:
            h8 = torch.empty(out8.shape, dtype=torch.uint8, pin_memory=True)
            h16 = torch.empty(out16.shape, dtype=torch.int16, pin_memory=True)
            h8.copy_(out8, non_blocking=True)
            h16.copy_(out16, non_blocking=True)
            cur.synchronize()
            a8, a16 = h8.numpy().astype(np.int16), h16.numpy()
            return [torch.from_numpy((a16 if wide[i] else a8)[out_off[i]:out_off[i] + n[i]].copy()) for i in range(m)]
        w8 = out8.to(torch.int16)
        return [(out16 if wide[i] else w8)[out_off[i]:out_off[i] + n[i]] for i in range(m)]


def encode_cdf_batch(cdfs, syms):
    """encode_cdf for many streams in one call: cdfs[i] 1HWLp int16, syms[i] int16, all on the CPU or all on one
    GPU -> [bytes], result i equal to encode_cdf(cdfs[i], syms[i])."""
    (cdfs, syms), m = _streams(cdfs, syms)
    if m == 0:
        return []
    dev, src, n, Lp, keep, on_cpu = _table_sources(cdfs)
    return _encode_batch(dev, src, n, Lp, syms, keep, (torch.device('cpu'),) if on_cpu else (dev,))


def decode_cdf_batch(cdfs, strings):
    """decode_cdf for many streams in one call -> [int16 tensor [H*W]] on the device of the tables, result i equal
    to decode_cdf(cdfs[i], strings[i])."""
    (cdfs, strings), m = _streams(cdfs, strings)
    if m == 0:
        return []
    dev, src, n, Lp, keep, on_cpu = _table_sources(cdfs)
    return _decode_batch(dev, src, n, Lp, strings, on_cpu)


def encode_logistic_mixture_batch(targets, means, log_scales, logit_probs_softmax, syms):
    """encode_logistic_mixture for many streams in one call (parameters on one GPU, symbols on the CPU or that GPU;
    every stream its own Lp and K) -> [bytes], result i equal to encode_logistic_mixture on entry i."""
    (targets, means, log_scales, logit_probs_softmax, syms), m = _streams(targets, means, log_scales,
                                                                         logit_probs_softmax, syms)
    if m == 0:
        return []
    dev, src, n, Lp, keep = _mixture_sources(targets, means, log_scales, logit_probs_softmax)
    return _encode_batch(dev, src, n, Lp, syms, keep, (torch.device('cpu'), dev))


def decode_logistic_mixture_batch(targets, means, log_scales, logit_probs_softmax, strings):
    """decode_logistic_mixture for many streams in one call -> [int16 tensor [H*W]] on the parameters' GPU.  The
    rows are built chunk by chunk under BATCH_SCRATCH_BYTES, so memory stays bounded at any Lp."""
    (targets, means, log_scales, logit_probs_softmax, strings), m = _streams(targets, means, log_scales,
                                                                             logit_probs_softmax, strings)
    if m == 0:
        return []
    dev, src, n, Lp, keep = _mixture_sources(targets, means, log_scales, logit_probs_softmax)
    return _decode_batch(dev, src, n, Lp, strings, False)
