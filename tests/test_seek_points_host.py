"""CPU: the seek points of the C oracle's decoder at C speed, and the streams the seek kernels are tested on
(DESIGN §4.13).

* oracle_points() derives every point of a stream from the oracle's decoder trace: low, high and bits are the trace's,
  flip is bit 31 of value ^ window, the window being the 32 code bits ending at `bits` (seek.code_windows).  It equals
  the restated reference decoder (test_seek_host.record_points) on the whole test_gpu_coder_launches stream grid,
  streams of K - 1 .. 2K + 1 symbols, and junk and truncated streams, at every alphabet.
* At every symbol of every one of those streams value ^ window is 0 or 2^31, the claim a one-bit flag rests on.
* The coverage inventory: per alphabet and K the points after an underflow shift (flip), the points whose window
  crosses the end of the stream's bytes or lies wholly past it, and the points with span 2^32 (low 0, high 2^32 - 1).
  Each is asserted non-zero at every alphabet and K (must_cover), so the GPU tests (test_gpu_seek_launches.py) that
  run these streams keep meeting every kind of point."""
import types

import numpy as np
import pytest

from oracle import ac
from l3c_pytorch_b200 import seek
from tests.test_gpu_coder_launches import ALPHABETS, EXTRA, KINDS, LENGTHS, make_stream

M32 = 0xFFFFFFFF
FLIP = 1 << 31
EVERY = (32, 64, 96, 4096)
# lengths K - 1, K, K + 1, 2K and 2K + 1 at K = 32 and 96 beside the grid's: segments and point counts at their edges
EDGE_LENGTHS = tuple(sorted({m * K + d for K in (32, 96) for (m, d) in ((1, -1), (1, 0), (1, 1), (2, 0), (2, 1))}
                            - set(LENGTHS)))
COVERAGE = ('flip', 'crosses end', 'past end', 'span 2^32')


def code_windows(data, bits):
    """the 32 code bits ending at each of `bits` (int64) of the stream bytes `data`, zero past their end"""
    buf = np.frombuffer(bytes(data) + b'\0', np.uint8)        # never empty: code_windows indexes the blob
    return seek.code_windows(buf, 0, len(data), np.asarray(bits, np.int64))


def oracle_points(cdf, data, every, trace=None):
    """int64 [points][4] (low, high, flip, bits) of the decoder reading the bytes `data` under the rows `cdf` [n, L+1],
    before symbols every, 2 every, ... < n: low, high and bits from the oracle's trace (decode_trace, or `trace`),
    flip = (window ^ value) & 2^31"""
    if trace is None:
        _, trace = ac.decode_trace(cdf, data)
    t = trace[every::every].astype(np.int64)
    flip = (code_windows(data, t[:, 3]) ^ t[:, 2]) & FLIP
    return np.stack([t[:, 0], t[:, 1], flip, t[:, 3]], 1)


def encoder_words(pts):
    """points (oracle_points) -> uint32 [points][4] as l3c_ac_encode_streams_seek writes them: low, high, bits low
    word, bits high word | flip"""
    pts = np.asarray(pts, np.int64).reshape(-1, 4)
    return np.stack([pts[:, 0], pts[:, 1], pts[:, 3] & M32, (pts[:, 3] >> 32) | pts[:, 2]], 1).astype(np.uint32)


def classify(pts, n_bytes):
    """bool masks per COVERAGE kind of the points pts of a stream of n_bytes bytes"""
    pts = np.asarray(pts, np.int64).reshape(-1, 4)
    end = 8 * np.asarray(n_bytes, np.int64)
    return {'flip': pts[:, 2] != 0,
            'crosses end': (pts[:, 3] - 32 < end) & (pts[:, 3] > end),
            'past end': pts[:, 3] - 32 >= end,
            'span 2^32': (pts[:, 0] == 0) & (pts[:, 1] == M32)}


def must_cover(L, every):
    """the COVERAGE kinds seek_streams(L) holds at every alphabet and K of EVERY: flips come from the straddle-run
    streams (L >= 3) and the flat and peaked ones; span 2^32 from the uniform streams where L is a power of two and
    from the straddling ones (coding the middle symbol returns to [0, 2^32)); the window positions from the cut and
    truncated copies"""
    return set(COVERAGE)


def _stream(s, data, note):
    sym, trace = ac.decode_trace(s.cdf, data)
    return types.SimpleNamespace(kind=s.kind, n=s.n, cdf=s.cdf, sym=s.sym, data=data, want=sym.astype(np.uint8),
                                 trace=trace, note=note)


_SEEK_STREAMS = {}


def seek_streams(L):
    """The streams of alphabet L the seek kernels run (cached): KINDS x (LENGTHS + EDGE_LENGTHS) + EXTRA, coded by the
    oracle, then corrupt copies -- junk of the stream's own length; truncated to a third, 90 %, all but one byte, one
    byte and nothing; and per K of EVERY a copy of a 5003-symbol stream cut inside the window of one of its points.
    Each has .data (the bytes a decoder is given), .want and .trace (the oracle's decode of those bytes)."""
    if L in _SEEK_STREAMS:
        return _SEEK_STREAMS[L]
    rng = np.random.default_rng(8100 + L)
    specs = [(k, n) for n in LENGTHS + EDGE_LENGTHS for k in KINDS] + list(EXTRA)
    valid = {}
    out = []
    for k, n in specs:
        s = make_stream(rng, k, n, L)
        st = _stream(s, ac.encode(s.cdf, s.sym), 'valid')
        assert (st.want == s.sym).all(), (L, k, n)
        valid.setdefault((k, n), st)
        out.append(st)
    for k, n in (('peaked', 5003), ('uniform', 1501), ('mix', 65), ('straddle-run', 5003)):
        s = valid[(k, n)]
        out.append(_stream(s, rng.integers(0, 256, len(s.data), np.uint8).tobytes(), 'junk'))
    for (k, n), f in ((('flat', 5003), 0.33), (('straddle', 1501), 0.9), (('peaked', 5003), -1), (('mix', 5003), 1),
                      (('tail', 1501), 0)):
        s = valid[(k, n)]
        cut = len(s.data) - 1 if f == -1 else f if f in (0, 1) else int(len(s.data) * f)
        out.append(_stream(s, s.data[:cut], 'truncated to %d of %d bytes' % (cut, len(s.data))))
    s = valid[('flat', 5003)]
    for K in EVERY:
        bits = s.trace[K::K, 3].astype(np.int64)
        for j, b in enumerate(bits):
            cut = int(b - 12) // 8
            t = _stream(s, s.data[:cut], 'cut inside the window of point %d at K=%d' % (j, K))
            if classify(oracle_points(t.cdf, t.data, K, t.trace), cut)['crosses end'].any():
                out.append(t)
                break
        else:
            raise AssertionError('L=%d K=%d: no cut of the flat stream puts a point\'s window across its end' % (L, K))
    _SEEK_STREAMS[L] = out
    return out


_POINTS = {}


def stream_points(L, every):
    """oracle_points of every seek_streams(L) stream at `every`, on the bytes it is given (cached)"""
    if (L, every) not in _POINTS:
        _POINTS[(L, every)] = [oracle_points(s.cdf, s.data, every, s.trace) for s in seek_streams(L)]
    return _POINTS[(L, every)]


def coverage(pts, n_bytes):
    """COVERAGE counts over the point sets pts (one per stream) of streams of n_bytes bytes"""
    got = dict.fromkeys(COVERAGE, 0)
    for p, nb in zip(pts, n_bytes):
        for name, m in classify(p, nb).items():
            got[name] += int(m.sum())
    return got


# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('L', ALPHABETS)
def test_oracle_points_equal_the_restated_decoder(L):
    from tests.test_seek_host import record_points
    ss = seek_streams(L)
    for i, s in enumerate(ss):
        pts, sym = record_points(s.cdf, s.data, L, 32)
        assert np.array_equal(sym.astype(np.uint8), s.want), (L, i, s.kind, s.n, s.note)
        pts = np.array(pts, np.int64).reshape(-1, 4)
        for K in EVERY:
            got = oracle_points(s.cdf, s.data, K, s.trace)
            assert got.shape == (seek.point_counts([s.n], K)[0], 4)
            want = pts[K // 32 - 1::K // 32]
            assert np.array_equal(got, want), (L, K, i, s.kind, s.n, s.note)
        w = encoder_words(pts)
        assert np.array_equal(w[:, 2].astype(np.int64) | (w[:, 3].astype(np.int64) & 0x7FFFFFFF) << 32, pts[:, 3])
        assert np.array_equal(w[:, 3].astype(np.int64) & FLIP, pts[:, 2])


@pytest.mark.parametrize('L', ALPHABETS)
def test_value_is_the_window_up_to_bit_31_at_every_symbol(L):
    """DESIGN §4.13: value - window is 0 or 2^31 for any input, junk included -- at every symbol, not only at points"""
    n_sym = n_flip = 0
    for s in seek_streams(L):
        t = s.trace.astype(np.int64)
        x = code_windows(s.data, t[:, 3]) ^ t[:, 2]
        bad = np.flatnonzero(x & 0x7FFFFFFF)
        assert bad.size == 0, (L, s.kind, s.n, s.note, 'symbol %d: value %#x' % (bad[0], t[bad[0], 2]))
        n_sym += s.n
        n_flip += int((x != 0).sum())
    print('L=%d: %d symbols, the value is the window with bit 31 flipped at %d' % (L, n_sym, n_flip))
    if L >= 3:
        assert n_flip > 0


@pytest.mark.parametrize('L', ALPHABETS)
def test_coverage_inventory(L):
    ss = seek_streams(L)
    n_bytes = [len(s.data) for s in ss]
    for K in EVERY:
        got = coverage(stream_points(L, K), n_bytes)
        n_pts = int(sum(p.shape[0] for p in stream_points(L, K)))
        print('L=%d K=%d: %d points; %s' % (L, K, n_pts, ', '.join('%s %d' % kv for kv in got.items())))
        for name in must_cover(L, K):
            assert got[name] > 0, (L, K, name, got)
    # an exact uniform prior keeps the coder at [0, 2^32): every point of a valid uniform stream has span 2^32, and
    # every point of a straddle-run stream (only the middle symbol, which decides no bit) follows an underflow shift
    for s, p in zip(ss, stream_points(L, 32)):
        if s.note != 'valid' or not p.shape[0]:
            continue
        if s.kind == 'uniform' and L & (L - 1) == 0:
            assert classify(p, len(s.data))['span 2^32'].all(), (L, s.n)
        if s.kind == 'straddle-run' and L >= 3:
            assert classify(p, len(s.data))['flip'].all(), (L, s.n)
