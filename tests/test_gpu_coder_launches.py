"""Every launch path of the range coder against the CPU oracle (oracle.ac, bit-exact by construction).

The decoder kernel is chosen by the alphabet (range_coder.cu, l3c_ac_decode_streams): L <= 32 runs
ac_decode32_kernel, 33..255 ac_decode_kernel<8,false>, 256 v3::ac_decode256_kernel<SPC> with SPC streams per CTA
(engine.decoder_streams_per_cta).  Here every one of them decodes many ragged streams per launch, in place from odd
byte offsets of one blob, resumed from saved state under several chunk schedules, with corrupt and truncated
streams beside valid ones in the same launches.  After every launch the saved coder state of every stream is
compared with the oracle's state at that symbol, so a wrong resume shows up at the chunk where it happens.  The
channel-pipelined RGB decode (l3c_decode_rgb_pipelined) is checked on its own against a sequential R -> G -> B decode.

The stream factory is checked on the CPU (test_stream_factory_round_trips_on_the_oracle): a failure in a GPU test
belongs to the kernel, not to the generated tables."""
import types

import numpy as np
import pytest
import torch

from oracle import ac

ALPHABETS = (2, 3, 25, 32, 33, 100, 255, 256)
LENGTHS = (1, 2, 7, 8, 9, 31, 32, 33, 63, 64, 65, 1501, 5003)
KINDS = ('flat', 'peaked', 'tail', 'straddle', 'uniform', 'mix')
# (kind, n_sym) added to the LENGTHS x KINDS grid: a second uniform stream, and streams that code only the
# midpoint-straddling symbol, so (L >= 3) they owe 7-9 more bits per symbol up to the terminator
EXTRA = (('uniform', 1501), ('straddle-run', 5003), ('straddle-run', 65))
HALF = 32768

# (L, streams per CTA of the L = 256 decoder): every decoder kernel of the library
DECODE_CASES = [(L, 0) for L in ALPHABETS if L != 256] + [(256, 1), (256, 2), (256, 4)]


def decoder_kernel(L, spc):
    """the kernel l3c_ac_decode_streams launches for alphabet L under decoder_streams_per_cta(spc)"""
    if L <= 32:
        return 'ac_decode32_kernel'
    if L < 256:
        return 'ac_decode_kernel<8,false>'
    return 'v3::ac_decode256_kernel<%d>' % (spc or 1)


# ----------------------------------------------------------------------------------------------
# stream factory: CDF rows [n, L+1] (the last entry is never read) and symbols, one kind per call
# ----------------------------------------------------------------------------------------------
def _rows_random(rng, n, L, peaked):
    """random rows (test_gpu_coder._random_table); peaked: one entry 500x heavier, 80 % of the symbols on it"""
    w = rng.integers(1, 4000 if peaked else 40, size=(n, L)).astype(np.float64)
    p = rng.integers(0, L, n)
    if peaked:
        w[np.arange(n), p] *= 500
    w = w / w.sum(1, keepdims=True) * (65536 - L - 41)
    c = np.floor(np.cumsum(w, 1)).astype(np.int64) + np.arange(1, L + 1)
    rows = np.zeros((n, L + 1), np.int64)
    rows[:, 0] = rng.integers(0, 30, n)
    rows[:, 1:L] = c[:, :-1] + rows[:, :1]
    sym = rng.integers(0, L, n)
    if peaked:
        sym = np.where(rng.random(n) < 0.8, p, sym)
    return rows, sym


def _rows_tail(rng, n, L):
    """one wide interval at a random entry p, every other interval 1 count wide; the symbols sit on 1-count
    intervals only: entry 0, entry L-1 (interval [65535, 65536)), the middle one or a random one"""
    p = rng.integers(0, L, n)[:, None]
    j = np.arange(L)[None]
    rows = np.zeros((n, L + 1), np.int64)
    rows[:, :L] = np.where(j <= p, j, 65536 - L + j)
    sym = np.choose(rng.integers(0, 4, n), [np.zeros(n, np.int64), np.full(n, L - 1), np.full(n, L // 2),
                                            rng.integers(0, L, n)])
    p = p[:, 0]
    return rows, np.where(sym == p, (p + 1) % L, sym)


def _rows_straddle(rng, n, L, release=True):
    """_underflow_case (test_gpu_coder) for any L >= 3: symbol m's interval [32768 - a, 32768 + a), a a power of two
    in 32..256, is centred on the midpoint.  From the full interval [0, 2^32) coding it decides no bit and owes
    log2(2^15 / a) = 7..9 underflow bits, after which the coder is back at [0, 2^32) exactly (low + high = 2^32 - 1
    is kept by every step) -- so the owed bits grow without bound, past 32 and across the encoder's 32-symbol
    batches, until another symbol releases them (release=False: only at the terminator).  Releases start at symbol
    40.  For L >= 5 the rows also hold the dyadic intervals [0, 2^14) (symbol 0) and [3 * 2^14, 2^16) (symbol
    L-1), and releases use only those: two decided bits bring the coder back to [0, 2^32), so the next run builds
    up again.  (L = 3, 4: a release is any symbol; the runs after it are short.)  L = 2 has no middle symbol: its
    one boundary sits at 32768 +- 3."""
    rows = np.zeros((n, L + 1), np.int64)
    if L == 2:
        rows[:, 1] = HALF + rng.integers(-3, 4, n)
        return rows, rng.integers(0, 2, n)
    m = (rng.integers(2, L - 2, n) if L >= 5 else rng.integers(1, L - 1, n))[:, None]
    a = 1 << rng.integers(5, 9, (n, 1))
    j = np.arange(L)[None]
    below = np.where(j == 0, 0, np.where(j == m, HALF - a, 2 ** 14 + (j - 1) * (2 ** 14 - a) // np.maximum(m - 1, 1)))
    above = HALF + a + (j - m - 1) * (2 ** 14 - a) // np.maximum(L - m - 2, 1)                 # j = L-1: 3 * 2^14
    rows[:, :L] = np.where(j <= m, below, above)
    sym = m[:, 0].copy()
    if release:
        rel = rng.random(n) < 1 / 37
        rel[:40] = False
        k = int(rel.sum())
        sym[rel] = np.where(rng.random(k) < 0.5, 0, L - 1) if L >= 5 else rng.integers(0, L, k)
    return rows, sym


def owed_bits(s, L):
    """underflow bits the oracle encoder (ac_oracle.c:69-95) owes after each symbol of stream s; the last entry is
    what it owes at the terminator"""
    M, H, Q = 0xFFFFFFFF, 1 << 31, 1 << 30
    low, high, pending = 0, M, 0
    out = np.zeros(s.n, np.int64)
    for i, sy in enumerate(s.sym.tolist()):
        span = high - low + 1
        c_lo, c_hi = int(s.cdf[i, sy]), 65536 if sy == L - 1 else int(s.cdf[i, sy + 1])
        high = (low - 1 + ((span * c_hi) >> 16)) & M
        low = (low + ((span * c_lo) >> 16)) & M
        while True:
            if high < H or low >= H:                  # a decided bit releases the owed ones
                pending = 0
                low, high = (low << 1) & M, ((high << 1) | 1) & M
            elif low >= Q and high < 3 * Q:           # underflow: one more bit owed
                pending += 1
                low, high = (low << 1) & 0x7FFFFFFF, ((high << 1) | 0x80000001) & M
            else:
                break
        out[i] = pending
    return out


def _rows_uniform(rng, n, L):
    """the uniform prior: for L a power of two every symbol takes exactly 2^-log2(L) of the interval and the span
    stays 2^32 (the FULL2 copy of the L = 256 decoder's loop); otherwise the reference's rounded row"""
    if L & (L - 1) == 0:
        row = np.arange(L + 1, dtype=np.int64) * (65536 // L)
    else:
        row = ac.uniform_cdf_row(L).astype(np.int64)
    row[L] = 0
    return np.tile(row, (n, 1)), rng.integers(0, L, n)


def _rows_mix(rng, n, L):
    """up to five kinds one after the other in one stream; no switch on a multiple of 8 (inside a group)"""
    cand = np.array([i for i in range(1, n) if i % 8])
    cuts = np.sort(rng.choice(cand, min(4, cand.size), replace=False)) if cand.size else []
    bounds = [0] + [int(c) for c in cuts] + [n]
    kinds = rng.permutation(['flat', 'peaked', 'tail', 'straddle', 'uniform'])
    parts = [_rows(kinds[i], rng, b - a, L) for i, (a, b) in enumerate(zip(bounds[:-1], bounds[1:]))]
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def _rows(kind, rng, n, L):
    if kind in ('flat', 'peaked'):
        return _rows_random(rng, n, L, kind == 'peaked')
    if kind == 'tail':
        return _rows_tail(rng, n, L)
    if kind in ('straddle', 'straddle-run'):
        return _rows_straddle(rng, n, L, release=(kind == 'straddle'))
    if kind == 'uniform':
        return _rows_uniform(rng, n, L)
    return _rows_mix(rng, n, L)


def make_stream(rng, kind, n, L):
    rows, sym = _rows(kind, rng, n, L)
    assert rows.shape == (n, L + 1) and sym.shape == (n,)
    assert rows.min() >= 0 and rows.max() <= 65535
    return types.SimpleNamespace(kind=kind, n=n, cdf=rows.astype(np.uint16), sym=sym.astype(np.int16))


_STREAMS = {}


def streams_for(L):
    """the streams of alphabet L, in launch order (cached).  Positions 0-3 are one CTA of the SPC = 4 decoder: a
    uniform (FULL2 at L = 256) stream, a peaked one, the one JUNK[0] replaces with junk and a 1-symbol one."""
    if L not in _STREAMS:
        rng = np.random.default_rng(7000 + L)
        specs = [(k, n) for n in LENGTHS for k in KINDS] + list(EXTRA)
        ss = [make_stream(rng, k, n, L) for (k, n) in specs]
        for s in ss:
            s.want = ac.encode(s.cdf, s.sym)
        order = [int(i) for i in rng.permutation(len(ss))]
        first = [specs.index(('uniform', 5003)), specs.index(('peaked', 5003)), specs.index(('flat', 1501)),
                 specs.index(('tail', 1))]
        order = first + [i for i in order if i not in first]
        _STREAMS[L] = [ss[i] for i in order]
    return _STREAMS[L]


# corrupt input, by launch position: junk of the stream's own length, and in_len cut to (fraction of) the length
JUNK = (2, 11, 29)
TRUNCATE = {6: 0.0, 19: 0.33, 37: -1, 45: 1, 52: 0.9}


def _intervals(s, L):
    lo = s.cdf[np.arange(s.n), s.sym].astype(np.int64)
    hi = np.where(s.sym == L - 1, 65536, s.cdf[np.arange(s.n), np.minimum(s.sym + 1, L)].astype(np.int64))
    return (lo | ((hi - 1) << 16)).astype(np.uint32)


def test_stream_factory_round_trips_on_the_oracle():
    """Every generated row is strictly increasing over its L used entries, every symbol has a non-empty interval,
    the kinds are what they claim, and every stream round-trips through the CPU oracle."""
    for L in ALPHABETS:
        ss = streams_for(L)
        max_owed = 0
        assert len(ss) == len(LENGTHS) * len(KINDS) + len(EXTRA)
        assert [(s.kind, s.n) for s in ss[:4]] == [('uniform', 5003), ('peaked', 5003), ('flat', 1501), ('tail', 1)]
        for s in ss:
            used = s.cdf[:, :L].astype(np.int64)
            assert (np.diff(used, axis=1) > 0).all(), (L, s.kind, s.n)
            assert ((0 <= s.sym) & (s.sym < L)).all()
            iv = _intervals(s, L).astype(np.int64)
            width = (iv >> 16) + 1 - (iv & 0xFFFF)
            assert (width >= 1).all()
            if s.kind == 'tail':
                assert (width == 1).all()
            if s.kind == 'straddle-run' and L > 2:
                assert ((iv & 0xFFFF) < HALF).all() and ((iv >> 16) >= HALF).all() and (width <= 512).all()
            if s.kind.startswith('straddle') and L > 2:
                # the encoder carries more than 31 owed bits across its first 32-symbol batch boundary (its
                # sequential sink, range_coder.cu emit_serial, then emits them); a run owes them at the terminator
                owed = owed_bits(s, L)
                if s.n >= 64:
                    assert owed[31] > 31, (L, s.kind, s.n, owed[31])
                if s.kind == 'straddle-run' and s.n >= 33:
                    assert owed[-1] > 31 and (np.diff(owed) > 0).all(), (L, s.n, owed[-1])
                max_owed = max(max_owed, int(owed.max()))
        if L > 2:
            print('L=%d: straddling streams owe up to %d underflow bits' % (L, max_owed))
            assert max_owed > 4000
            if s.kind == 'uniform' and L == 256:
                assert (s.cdf[:, :L] == np.arange(L) * 256).all()
            assert (ac.decode(s.cdf, s.want) == s.sym).all(), (L, s.kind, s.n)
        # corrupt positions lie in every launch (the smallest launch has len(ss) - 3 streams) on long streams
        assert max(JUNK + tuple(TRUNCATE)) < len(ss) - 3
    # bookkeeping, not evidence: decoder_kernel() restates the library's dispatch rule, so this only says that
    # DECODE_CASES names an alphabet / SPC for each of the five decoder kernels.  The launch log does not name the
    # variant; that the knob really switches the L = 256 kernel is shown by breaking one variant (e.g. its grid)
    # and watching test_chunked_ragged_decode_matches_oracle fail for that SPC only.
    assert {decoder_kernel(L, spc) for (L, spc) in DECODE_CASES} == {
        'ac_decode32_kernel', 'ac_decode_kernel<8,false>', 'v3::ac_decode256_kernel<1>',
        'v3::ac_decode256_kernel<2>', 'v3::ac_decode256_kernel<4>'}


def test_decoder_streams_per_cta_knob_rejects_other_values():
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200._lib import lib
    for bad in (-1, 3, 5, 8, 64):
        with pytest.raises(RuntimeError, match='streams_per_cta'):
            with E.decoder_streams_per_cta(bad):
                pass
    for spc in (0, 1, 2, 4):
        assert lib.l3c_set_decoder_streams_per_cta(spc) == 0
    assert lib.l3c_set_decoder_streams_per_cta(0) == 0


# ----------------------------------------------------------------------------------------------
# GPU: batched encode, pack at odd offsets
# ----------------------------------------------------------------------------------------------
def _encode_and_pack(ss, L, dev):
    """all streams in one l3c_ac_encode_streams launch (slots of codec._slot_cap bytes), gathered by
    l3c_pack_streams into one blob at odd, varied offsets -> (lens, dst offsets, blob, slot caps)"""
    from l3c_pytorch_b200 import _lib, codec, engine as E
    n = np.array([s.n for s in ss], np.int64)
    iv_dev = torch.from_numpy(np.concatenate([_intervals(s, L) for s in ss]).view(np.int32)).to(dev)
    caps = np.array([codec._slot_cap(int(k)) for k in n], np.int64)
    slots = torch.full((int(caps.sum()),), 0x5A, dtype=torch.uint8, device=dev)
    desc = np.zeros(len(ss), dtype=_lib.ENC_STREAM_DTYPE)
    desc['intervals'] = iv_dev.data_ptr() + 4 * np.concatenate([[0], np.cumsum(n)[:-1]])
    desc['out'] = slots.data_ptr() + np.concatenate([[0], np.cumsum(caps)[:-1]])
    desc['n_sym'] = n
    desc['out_cap'] = caps
    desc_dev, lens_dev = E.ac_encode_streams(desc, dev)
    lens = lens_dev.cpu().numpy().astype(np.int64)
    gaps = 1 + np.arange(len(ss)) % 4
    dst = np.concatenate([[3], 3 + np.cumsum(lens[:-1] + gaps[:-1])]).astype(np.int64)
    blob = torch.zeros(int(dst[-1] + lens[-1] + 16), dtype=torch.uint8, device=dev)
    E.pack_streams(desc_dev, lens_dev, dst, len(ss), blob)
    torch.cuda.synchronize()
    del iv_dev, slots
    return lens, dst, blob, caps


@pytest.mark.gpu
@pytest.mark.parametrize('L', ALPHABETS)
def test_batched_encode_matches_oracle_within_the_slot_bound(L):
    """One encode launch for all streams of an alphabet: the bytes equal the oracle's for every stream, and no
    stream exceeds its slot (17 bits per symbol + 64 B, codec._slot_cap) -- the tail streams code every symbol
    on a 1-count interval, the worst case the bound is for."""
    dev = torch.device('cuda')
    ss = streams_for(L)
    lens, dst, blob, caps = _encode_and_pack(ss, L, dev)
    hb = blob.cpu().numpy()
    for i, s in enumerate(ss):
        got = hb[dst[i]:dst[i] + lens[i]].tobytes()
        assert got == s.want, (L, i, s.kind, s.n)
    assert (lens <= caps).all(), [(s.kind, s.n) for s, ln, c in zip(ss, lens, caps) if ln > c]
    tail = [8.0 * ln / s.n for s, ln in zip(ss, lens) if s.kind == 'tail' and s.n >= 1000]
    print('L=%d: tail streams (every symbol on a 1-count interval) take at most %.4f bits/symbol (slot: 17 + 512/n)'
          % (L, max(tail)))
    assert max(tail) < 17.0


# ----------------------------------------------------------------------------------------------
# GPU: batched, chunked, ragged, in-place decode with corrupt streams in the same launches
# ----------------------------------------------------------------------------------------------
def _schedules(rng, n_max):
    """chunk schedules [(first, count)] covering [0, n_max)"""
    cand = rng.choice(np.arange(1, n_max), 60, replace=False)
    cuts = np.sort(cand[cand % 4 != 0][:16])
    bounds = [0] + [int(c) for c in cuts] + [n_max]
    return [('one launch', [(0, n_max)]),
            ('1, 1, 3, rest', [(0, 1), (1, 1), (2, 3), (5, n_max - 5)]),
            ('random cuts', [(a, b - a) for a, b in zip(bounds[:-1], bounds[1:])]),
            ('count past every end', [(0, 13), (13, 2 ** 32 - 1)]),
            ('first beyond the short streams', [(0, 9), (9, 57), (66, 1437), (1503, 3001), (4504, 600)])]


def _check_decode_launches(L, spc):
    from l3c_pytorch_b200 import _lib, engine as E
    dev = torch.device('cuda')
    rng = np.random.default_rng(100 + L + spc)
    ss = streams_for(L)
    n_all = len(ss)
    n = np.array([s.n for s in ss], np.int64)
    lens, dst, blob, _ = _encode_and_pack(ss, L, dev)
    # corrupt in place: junk of the stream's own length, truncation through a smaller in_len (never more bytes
    # than lie behind `in`: the packed stream itself, then the rest of the blob)
    in_len = lens.copy()
    for i in JUNK:
        blob[int(dst[i]):int(dst[i] + lens[i])] = torch.from_numpy(rng.integers(0, 256, int(lens[i]), np.uint8))
    for i, f in TRUNCATE.items():
        in_len[i] = lens[i] - 1 if f == -1 else (f if f == 1 else int(lens[i] * f))
    hb = blob.cpu().numpy()
    want_sym, trace = [], []
    for i, s in enumerate(ss):
        passed = hb[dst[i]:dst[i] + in_len[i]].tobytes()
        sym, tr = ac.decode_trace(s.cdf, passed)
        if i not in JUNK and i not in TRUNCATE:
            assert (sym == s.sym).all(), (L, i)
        want_sym.append(sym.astype(np.uint8))
        trace.append(tr)
    # rows at the library's pitch; outputs at offsets +0..+3 from a 4-byte boundary, each followed by guard bytes
    pitch = E.table_pitch(L)
    tab = np.zeros((int(n.sum()), pitch), np.uint16)
    tab[:, :L] = np.concatenate([s.cdf[:, :L] for s in ss])
    tab_dev = torch.from_numpy(tab.view(np.int16)).to(dev)
    row0 = np.concatenate([[0], np.cumsum(n)[:-1]])
    slot = (n + 8 + 3) // 4 * 4 + 4
    out0 = np.concatenate([[0], np.cumsum(slot)[:-1]]) + np.arange(n_all) % 4
    out = torch.empty(int(slot.sum()), dtype=torch.uint8, device=dev)
    state = torch.empty(4 * n_all, dtype=torch.int32, device=dev)
    dd = np.zeros(n_all, dtype=_lib.DEC_STREAM_DTYPE)
    dd['table'] = tab_dev.data_ptr() + 2 * pitch * row0
    dd['in'] = blob.data_ptr() + dst
    dd['sym_out'] = out.data_ptr() + out0
    dd['state'] = state.data_ptr() + 16 * np.arange(n_all)
    dd['row_pitch'] = pitch
    dd['n_sym'] = n
    dd['in_len'] = in_len
    desc_dev = E._desc_to_device(dd, dev)
    name = decoder_kernel(L, spc)
    with E.decoder_streams_per_cta(spc):
        for k, (sched_name, sched) in enumerate(_schedules(rng, int(n.max()))):
            r = 1 + k % 3
            n_use = n_all - (n_all - r) % 4      # n_use % 4 == r: partial last CTA (SPC 2: when r is odd)
            out.fill_(0xA5)
            state.fill_(-1)
            for (first, count) in sched:
                E.ac_decode_streams(dd, dev, L, first, count, desc_dev=desc_dev, n=n_use)
                st = state.cpu().numpy().view(np.uint32).reshape(n_all, 4)
                for i in range(n_use):
                    if first >= n[i]:
                        continue
                    last = min(first + count, int(n[i]))
                    want = trace[i][min(last, int(n[i]) - 1)]
                    assert (st[i] == want).all(), (
                        '%s, schedule "%s", launch (%d, %d), stream %d (%s, n=%d, in_len=%d/%d): saved state %s, '
                        'oracle %s' % (name, sched_name, first, count, i, ss[i].kind, n[i], in_len[i], lens[i],
                                       st[i].tolist(), want.tolist()))
            got = out.cpu().numpy()
            for i in range(n_all):
                o = int(out0[i])
                seg, guard = got[o:o + int(n[i])], got[o + int(n[i]):o + int(n[i]) + 8]
                if i >= n_use:
                    assert (seg == 0xA5).all(), (name, sched_name, 'stream outside the launch was written', i)
                    continue
                bad = np.flatnonzero(seg != want_sym[i])
                assert bad.size == 0, ('%s, schedule "%s", stream %d (%s, n=%d, in_len=%d/%d): %d wrong symbols, '
                                       'first at %d' % (name, sched_name, i, ss[i].kind, n[i], in_len[i], lens[i],
                                                        bad.size, bad[:1]))
                assert (guard == 0xA5).all(), (name, sched_name, 'write past the end of stream', i)
    del tab_dev, blob


@pytest.mark.gpu
@pytest.mark.parametrize('L,spc', DECODE_CASES)
def test_chunked_ragged_decode_matches_oracle(L, spc):
    """All streams of one alphabet (lengths 1 .. 5003, ragged in one descriptor array) decoded in place from odd
    byte offsets under five chunk schedules -- one launch; counts 1, 1, 3, rest; random cuts that are not
    multiples of 4; a count past every stream's end; chunks that start beyond the shorter streams -- with
    3 junk and 5 truncated streams (in_len 0, 1, a third, 90 %, all but one byte) beside the valid ones.  Each
    schedule launches a stream count with n % 4 = 1, 2 or 3.  Every stream decodes to the oracle's symbols for the
    bytes it was given, its saved state equals the oracle's after every launch, and nothing is written past a
    stream's symbols or for streams beyond the launch's count."""
    _check_decode_launches(L, spc)


# ----------------------------------------------------------------------------------------------
# GPU: the channel-pipelined RGB decode on its own
# ----------------------------------------------------------------------------------------------
RGB = {}
RGB_HW = (12, 20)                    # 240 pixels: chunk size 1 is 720 decoder launches
RGB_K = 10


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def _rgb_case(dev):
    """mixture parameters l [N, H, W, 4*3*K] shaped like a trained model's (one dominant logit, log-scales down to
    and below the -7 clamp, means inside and outside [0, 255], random coupling coefficients), symbols mostly at the
    dominant component's mode, some anywhere (mostly 1-count tail intervals), some 0 and 255; images of HW, HW-37,
    9 and 1 pixels in compact planes of HW; encoded on the GPU and checked against the oracle on the rows the
    decoder builds."""
    if 'case' in RGB:
        return RGB['case']
    from l3c_pytorch_b200 import _lib, codec, engine as E
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    rng = np.random.default_rng(31)
    H, W = RGB_HW
    HW, C, K, L = H * W, 3, RGB_K, 256
    ns = np.array([HW, HW - 37, 9, 1], np.int64)
    N = len(ns)
    shp = (N, HW, C, K)
    dom = rng.integers(0, K, (N, HW, C))

    def at_dom(a, v):
        np.put_along_axis(a, dom[..., None], v[..., None], axis=3)

    logit = rng.normal(0, 1, shp)
    at_dom(logit, rng.uniform(4, 12, dom.shape))
    mean = rng.uniform(-60, 315, shp)
    at_dom(mean, rng.uniform(-20, 275, dom.shape))
    logs = rng.uniform(-9, 1.5, shp)
    at_dom(logs, rng.uniform(-9.5, -2, dom.shape))
    coef = rng.normal(0, 2, shp)
    l = np.stack([logit, mean, logs, coef], axis=2).reshape(N, H, W, 4 * C * K).astype(np.float32)
    mu = np.take_along_axis(mean, dom[..., None], axis=3)[..., 0]            # dominant component's mean
    sym = np.zeros((N, C, HW), np.int64)
    for c in range(C):
        m = mu[:, :, c].copy()
        if c == 1:
            m += _sigmoid(np.take_along_axis(coef[:, :, 0], dom[:, :, 1:2], axis=2)[..., 0]) * sym[:, 0]
        elif c == 2:
            m += (_sigmoid(np.take_along_axis(coef[:, :, 1], dom[:, :, 2:3], axis=2)[..., 0]) * sym[:, 0] +
                  _sigmoid(np.take_along_axis(coef[:, :, 2], dom[:, :, 2:3], axis=2)[..., 0]) * sym[:, 1])
        s = np.clip(np.rint(m + rng.normal(0, 0.4, m.shape)), 0, 255)
        u = rng.random(m.shape)
        s = np.where(u < 0.12, rng.integers(0, 256, m.shape), s)
        s = np.where((u >= 0.12) & (u < 0.15), 0, s)
        s = np.where((u >= 0.15) & (u < 0.18), 255, s)
        sym[:, c] = s
    l_dev = torch.from_numpy(l).to(dev)
    sym_u8 = sym.astype(np.uint8)
    sym_dev = torch.from_numpy(sym_u8.reshape(N, C, H, W)).to(dev)
    tg = DiscretizedMixLogisticLoss(True, 0, 255, L).targets(dev)
    iv = E.dmll_intervals(l_dev, sym_dev, tg, C, K, L, True)
    # encode the first ns[n] symbols of every plane in one launch, pack at odd offsets
    desc = np.zeros((N, C), dtype=_lib.ENC_STREAM_DTYPE)
    caps = np.array([codec._slot_cap(int(k)) for k in ns], np.int64)
    slots = torch.zeros(int(C * caps.sum()), dtype=torch.uint8, device=dev)
    cap_nc = np.repeat(caps, C).reshape(N, C)
    desc['intervals'] = iv.data_ptr() + 4 * HW * (np.arange(N)[:, None] * C + np.arange(C)[None])
    desc['out'] = slots.data_ptr() + np.concatenate([[0], np.cumsum(cap_nc.reshape(-1))[:-1]]).reshape(N, C)
    desc['n_sym'] = ns[:, None]
    desc['out_cap'] = cap_nc
    desc = desc.reshape(-1)
    desc_dev, lens_dev = E.ac_encode_streams(desc, dev)
    lens = lens_dev.cpu().numpy().astype(np.int64)
    dst = np.concatenate([[5], 5 + np.cumsum(lens[:-1] + 3)]).astype(np.int64)
    blob = torch.zeros(int(dst[-1] + lens[-1] + 16), dtype=torch.uint8, device=dev)
    E.pack_streams(desc_dev, lens_dev, dst, N * C, blob)
    # the rows the decoder will use, built from the true symbols: the encoded bytes are the oracle's on them
    table = torch.zeros(N * C * HW * L, dtype=torch.int16, device=dev)
    for c in range(C):
        E.dmll_build_table(l_dev, sym_dev, tg, C, K, L, True, c, table)
    rows = table.cpu().numpy().view(np.uint16).reshape(N, C, HW, L)
    hb = blob.cpu().numpy()
    ones = 0
    for nn in range(N):
        for c in range(C):
            j = nn * C + c
            k = int(ns[nn])
            r = np.concatenate([rows[nn, c, :k], np.zeros((k, 1), np.uint16)], 1)
            assert hb[dst[j]:dst[j] + lens[j]].tobytes() == ac.encode(r, sym[nn, c, :k]), (nn, c)
            s = sym[nn, c, :k]
            hi = np.where(s == L - 1, 65536, r[np.arange(k), np.minimum(s + 1, L - 1)].astype(np.int64))
            ones += int((hi - r[np.arange(k), s] <= 2).sum())
    RGB['case'] = types.SimpleNamespace(l=l_dev, tg=tg, sym=sym_u8, ns=ns, lens=lens, dst=dst, blob=blob, N=N,
                                        H=H, W=W, C=C, K=K, L=L, tail_frac=ones / float(C * ns.sum()))
    return RGB['case']


def _rgb_descs(cs, dev, S, table, state):
    from l3c_pytorch_b200 import _lib
    N, C, HW = cs.N, cs.C, cs.H * cs.W
    d = np.zeros((N, C), dtype=_lib.DEC_STREAM_DTYPE)
    plane = np.arange(N)[:, None] * C + np.arange(C)[None]
    d['in'] = cs.blob.data_ptr() + cs.dst.reshape(N, C)
    d['in_len'] = cs.lens.reshape(N, C)
    d['n_sym'] = cs.ns[:, None]
    d['sym_out'] = S.data_ptr() + HW * plane
    d['table'] = table.data_ptr() + 2 * cs.L * HW * plane
    d['row_pitch'] = cs.L
    d['state'] = 0 if state is None else state.data_ptr() + 16 * plane
    return d


def _rgb_sequential(cs, dev):
    """the reference order: rows of channel c built after channel c-1 is fully decoded, one launch per channel
    (default streams per CTA, no saved state)"""
    from l3c_pytorch_b200 import engine as E
    S = torch.zeros(cs.N, cs.C, cs.H, cs.W, dtype=torch.uint8, device=dev)
    table = torch.zeros(cs.N * cs.C * cs.H * cs.W * cs.L, dtype=torch.int16, device=dev)
    d = _rgb_descs(cs, dev, S, table, None)
    for c in range(cs.C):
        E.dmll_build_table(cs.l, S, cs.tg, cs.C, cs.K, cs.L, True, c, table)
        E.ac_decode_streams(np.ascontiguousarray(d[:, c]), dev, cs.L)
    return S.cpu().numpy().reshape(cs.N, cs.C, -1)


def _rgb_pipelined(cs, dev, chunk, bld, dec):
    from l3c_pytorch_b200 import engine as E
    S = torch.zeros(cs.N, cs.C, cs.H, cs.W, dtype=torch.uint8, device=dev)
    table = torch.zeros(cs.N * cs.C * cs.H * cs.W * cs.L, dtype=torch.int16, device=dev)
    state = torch.full((cs.N * cs.C * 4,), -1, dtype=torch.int32, device=dev)
    d = _rgb_descs(cs, dev, S, table, state)
    descs = [E._desc_to_device(np.ascontiguousarray(d[:, c]), dev) for c in range(cs.C)]
    E.decode_rgb_pipelined(cs.l, S, cs.tg, cs.K, cs.L, table, descs, chunk, torch.cuda.current_stream(), bld, dec)
    torch.cuda.synchronize()
    return S.cpu().numpy().reshape(cs.N, cs.C, -1)


@pytest.mark.gpu
@pytest.mark.parametrize('spc', [1, 2, 4])
def test_pipelined_rgb_decode_matches_sequential_decode(spc):
    """l3c_decode_rgb_pipelined with chunks of 1, 5, 8, 13, 64, HW-1, HW and 3 HW pixels (chunks that split the
    decoder's 8-symbol groups, a single chunk, a chunk larger than the plane) on ragged images (HW, HW-37, 9 and 1
    pixels in compact planes), on plain torch streams and on a BatchCodec decode lane (SM partitions where the
    driver offers them), under every streams-per-CTA variant: the decoded planes equal the coded symbols and a
    sequential R -> G -> B decode."""
    from l3c_pytorch_b200 import codec, engine as E
    dev = torch.device('cuda')
    cs = _rgb_case(dev)
    HW = cs.H * cs.W
    print('RGB case: %.1f %% of the coded sub-pixels sit on intervals of at most 2 counts' % (100 * cs.tail_frac))
    assert cs.tail_frac > 0.05
    seq = _rgb_sequential(cs, dev)
    for nn in range(cs.N):
        k = int(cs.ns[nn])
        assert (seq[nn, :, :k] == cs.sym[nn, :, :k]).all(), nn
    plain = ([torch.cuda.Stream(device=dev) for _ in range(3)], [torch.cuda.Stream(device=dev) for _ in range(3)])
    lane = codec.BatchCodec(types.SimpleNamespace(net=None)).lanes(dev, cs.N * cs.C, 1)[0][0]
    print('decode lane on SM partitions: %s' % lane.partitioned)
    runs = [(chunk, 'torch streams', plain) for chunk in (1, 5, 8, 13, 64, HW - 1, HW, 3 * HW)]
    runs += [(chunk, 'decode lane (partitioned: %s)' % lane.partitioned, (lane.bld, lane.dec)) for chunk in (13, HW)]
    with E.decoder_streams_per_cta(spc):
        for chunk, where, (bld, dec) in runs:
            got = _rgb_pipelined(cs, dev, chunk, bld, dec)
            for nn in range(cs.N):
                k = int(cs.ns[nn])
                bad = np.flatnonzero((got[nn, :, :k] != seq[nn, :, :k]).reshape(-1))
                assert bad.size == 0, ('SPC %d, chunk %d, %s, image %d (%d px): %d wrong sub-pixels, first at '
                                       'channel %d pixel %d' % (spc, chunk, where, nn, k, bad.size, bad[0] // k,
                                                                bad[0] % k))
