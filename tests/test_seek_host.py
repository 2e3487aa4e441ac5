"""CPU: seek indexes (DESIGN §4.13).  A restatement of the reference decoder loop (torchac.cpp:325-373) records the
seek points of streams from the C oracle; they agree with the oracle's own decoder trace, and the sidecar writer and
parser round-trip them.  The segment planner's descriptors for equal-size, ragged and recursive layouts, and every
refusal of the parser."""
import struct
import zlib

import numpy as np
import pytest

from oracle import ac
from l3c_pytorch_b200 import _lib, seek
from l3c_pytorch_b200.codec import MAGIC, TILED_MAGIC, stream_layout
from tests.test_gpu_coder_launches import make_stream

M32 = 0xFFFFFFFF
M64 = (1 << 64) - 1


def record_points(cdf, data, L, every):
    """torchac.cpp:325-373 restated in Python: the decoder's (low, high, flip, bits) before symbols every, 2 every,
    ... < n, where flip is 2^31 when the last renormalisation shift was an underflow shift (then the code value is the
    last 32 code bits with bit 31 flipped), and the decoded symbols."""
    buf = bytes(data)
    n = cdf.shape[0]
    pos = [0]

    def bit():
        p = pos[0]
        pos[0] += 1
        return (buf[p >> 3] >> (7 - (p & 7))) & 1 if (p >> 3) < len(buf) else 0

    low, high, value, flip = 0, M32, 0, 0
    for _ in range(32):
        value = ((value << 1) | bit()) & M32
    pts, out = [], np.zeros(n, np.int64)
    for i in range(n):
        if i and i % every == 0:
            pts.append((low, high, flip, 32 + pos[0] - 32))
        span = high - low + 1
        # in uint64 as the reference computes it: on junk input the value can lie below low, and the difference wraps
        count = (((value - low + 1) * 65536 - 1) & M64) // span & 0xFFFF
        row = [int(v) for v in cdf[i, :L]]
        sym = max(m for m in range(L) if row[m] <= count) if row[0] <= count else 0
        out[i] = sym
        if i == n - 1:
            break
        c_lo, c_hi = row[sym], 65536 if sym == L - 1 else row[sym + 1]
        high = (low - 1 + ((span * c_hi) >> 16)) & M32
        low = (low + ((span * c_lo) >> 16)) & M32
        while True:
            if low >= 0x80000000 or high < 0x80000000:
                low, high = (low << 1) & M32, ((high << 1) | 1) & M32
                value = ((value << 1) | bit()) & M32
                flip = 0
            elif low >= 0x40000000 and high < 0xC0000000:
                low, high = (low << 1) & 0x7FFFFFFF, ((high << 1) | 0x80000001) & M32
                value = (((value - 0x40000000) << 1) | bit()) & M32
                flip = 0x80000000
            else:
                break
    return pts, out


def container(streams):
    """a reference-layout container holding each (n_sym, bytes) as the one stream of a 1 x 1 x n_sym scale"""
    parts = [struct.pack('<4H', 0, 0, 0, 0)]
    for n, b in streams:
        parts += [struct.pack('<BHH', 1, 1, n), struct.pack('<I', len(b)), b, MAGIC]
    return b''.join(parts)


def window(buf, bits):
    p, w = bits - 32, 0
    for k in range(32):
        q = p + k
        w = (w << 1) | (((buf[q >> 3] >> (7 - (q & 7))) & 1) if (q >> 3) < len(buf) else 0)
    return w


STREAMS = [('flat', 700, 5), ('peaked', 1501, 40), ('straddle-run', 999, 25), ('uniform', 640, 256),
           ('tail', 1, 9), ('flat', 64, 256)]


@pytest.fixture(scope='module')
def coded():
    rng = np.random.default_rng(11)
    out = []
    for kind, n, L in STREAMS:
        s = make_stream(rng, kind, n, L)
        out.append((s, ac.encode(s.cdf, s.sym), L))
    return out


@pytest.mark.parametrize('every', [32, 96, 4096])
def test_restated_points_match_oracle_trace_and_round_trip(coded, every):
    streams, all_pts = [], []
    for s, data, L in coded:
        pts, sym = record_points(s.cdf, data, L, every)
        assert np.array_equal(sym, s.sym.astype(np.int64)), s.kind
        _, trace = ac.decode_trace(s.cdf, data)
        assert len(pts) == seek.point_counts([s.n], every)[0]
        for k, (low, high, flip, bits) in enumerate(pts):
            j = (k + 1) * every
            t = [int(v) for v in trace[j]]
            assert (low, high, bits) == (t[0], t[1], t[3]), (s.kind, j)
            assert window(data, bits) ^ flip == t[2], (s.kind, j)          # the value is not stored
        streams.append((s.n, data))
        all_pts.append(pts)
    cont = container(streams)
    counts = [len(p) for p in all_pts]
    flat = [p for ps in all_pts for p in ps]
    cols = [np.array([p[i] for p in flat], np.int64) for i in range(4)]
    idx = seek.write_index(cont, every, counts, *cols)
    assert len(idx) == 28 + 4 * len(streams) + 12 * len(flat) + 4
    parsed = seek.parse_index(idx, cont)
    assert parsed.every == every and list(parsed.counts) == counts
    for a, b in zip((parsed.low, parsed.high, parsed.flip, parsed.bits), cols):
        assert np.array_equal(a, b)
    w = parsed.state_words()
    assert np.array_equal(w[:, 3].astype(np.int64) | (w[:, 4].astype(np.int64) << 32), cols[3])


# ----------------------------------------------------------------------------------------------
# segment planner
# ----------------------------------------------------------------------------------------------
def _descs(shapes_of, pitch, base=1 << 20):
    """decoder descriptors of every stream of a batch laid out by stream_layout (one fake blob, tables, planes)"""
    si, elem, n_sym, _ = stream_layout(shapes_of)
    N, P = n_sym.shape
    desc = np.zeros(N * P, _lib.DEC_STREAM_DTYPE)
    offs = (np.arange(N * P, dtype=np.int64) * 4096 + base).reshape(N, P)
    desc['in'] = offs.reshape(-1)
    desc['in_len'] = 100
    desc['n_sym'] = n_sym.reshape(-1)
    desc['sym_out'] = (1 << 40) + elem.reshape(-1)
    desc['table'] = (1 << 41) + 2 * pitch * elem.reshape(-1)
    desc['row_pitch'] = pitch
    return desc, offs, n_sym


LAYOUTS = {
    'equal': [[(5, 8, 8), (5, 16, 16), (3, 32, 32)]] * 2,
    'ragged': [[(5, 8, 8), (5, 16, 16), (3, 32, 32)], [(5, 4, 6), (5, 8, 12), (3, 16, 24)]],
    'recursive': [[(3, 2, 2), (3, 4, 4), (3, 8, 8), (3, 16, 16), (3, 32, 32)]] * 2,
}


@pytest.mark.parametrize('layout', sorted(LAYOUTS))
@pytest.mark.parametrize('every', [32, 96, 4096])
def test_plan_segments(layout, every):
    shapes_of = LAYOUTS[layout]
    pitch = 256
    desc, offs, n_sym = _descs(shapes_of, pitch)
    N, P = n_sym.shape
    counts = seek.point_counts(n_sym.reshape(-1), every)
    # image 1 has no index: its streams are one segment each
    every_s = np.full(N * P, every, np.int64)
    every_s[P:] = 1 << 40
    first = np.cumsum(counts) - counts
    state_ptr = 1 << 44
    order = np.random.default_rng(3).permutation(desc.size)            # any subset, any order
    segs = seek.plan_segments(desc[order], offs.reshape(-1), every_s, first, state_ptr)
    want = []
    for i in order:
        n, K = int(desc['n_sym'][i]), int(every_s[i])
        for j, s0 in enumerate(range(0, n, K)):
            want.append((int(desc['in'][i]), int(desc['table'][i]) + 2 * pitch * s0, int(desc['sym_out'][i]) + s0,
                         min(K, n - s0), 0 if j == 0 else state_ptr + 4 * seek.STATE_WORDS * (first[i] + j - 1)))
    got = list(zip(*(segs[f].astype(np.int64).tolist() for f in ('in', 'table', 'sym_out', 'n_sym', 'state'))))
    assert got == want
    assert (segs['in_len'] == 100).all() and (segs['row_pitch'] == pitch).all()
    # every symbol of every stream exactly once
    assert segs['n_sym'].astype(np.int64).sum() == desc['n_sym'].astype(np.int64).sum()


def test_plan_segments_shared_row_and_unknown_stream():
    desc, offs, n_sym = _descs(LAYOUTS['equal'], 0)
    segs = seek.plan_segments(desc, offs.reshape(-1), np.full(desc.size, 32, np.int64),
                              np.zeros(desc.size, np.int64), 0)
    assert (segs['table'] == desc['table'][0]).all()                      # one shared row: never offset
    with pytest.raises(ValueError):
        seek.plan_segments(desc, offs.reshape(-1)[1:], np.full(desc.size, 32, np.int64),
                           np.zeros(desc.size, np.int64), 0)


# ----------------------------------------------------------------------------------------------
# parser refusals
# ----------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def indexed(coded):
    every = 96
    streams, flat, counts = [], [], []
    for s, data, L in coded:
        pts, _ = record_points(s.cdf, data, L, every)
        streams.append((s.n, data))
        flat += pts
        counts.append(len(pts))
    cont = container(streams)
    cols = [np.array([p[i] for p in flat], np.int64) for i in range(4)]
    return cont, every, counts, cols


def _recrc(b):
    b = bytearray(b)
    b[-4:] = struct.pack('<I', zlib.crc32(bytes(b[:-4])) & M32)
    return bytes(b)


def _point_word(counts, k, w):
    """byte offset of word w of point k (all streams' points in order)"""
    per, acc = [], 28
    for c in counts:
        acc += 4
        per += [acc + 12 * i for i in range(c)]
        acc += 12 * c
    return per[k] + 4 * w


def _mutations(cont, every, counts, cols):
    good = seek.write_index(cont, every, counts, *cols)
    low_pt = _point_word(counts, 0, 0)
    yield 'magic', b'XXXX' + good[4:], cont
    yield 'version', _recrc(good[:4] + struct.pack('<I', 2) + good[8:]), cont
    yield 'crc', good[:-1] + bytes([good[-1] ^ 1]), cont
    yield 'container length', good, cont + b'\0'
    yield 'container crc', good, cont[:-5] + bytes([cont[-5] ^ 1]) + cont[-4:]
    for K in (16, 48, 1 << 25):
        yield 'every %d' % K, _recrc(good[:8] + struct.pack('<I', K) + good[12:]), cont
    yield 'count', _recrc(good[:28] + struct.pack('<I', counts[0] + 1) + good[32:]), cont
    b = bytearray(good)
    b[low_pt:low_pt + 4] = struct.pack('<I', struct.unpack_from('<I', good, low_pt)[0] | 0x80000000)
    yield 'low bit 31', _recrc(bytes(b)), cont
    b = bytearray(good)
    b[low_pt + 4:low_pt + 8] = b[low_pt:low_pt + 4]
    yield 'high <= low', _recrc(bytes(b)), cont
    b = bytearray(good)
    b[low_pt + 8:low_pt + 12] = struct.pack('<I', 64 * every + 1)
    yield 'advance', _recrc(bytes(b)), cont
    tiled = cont[:8] + TILED_MAGIC + struct.pack('<HH', 8, 8) + cont[8:]
    yield 'tiled', _recrc(good[:12] + struct.pack('<QI', len(tiled), zlib.crc32(tiled) & M32) + good[24:]), tiled
    yield 'short', good[:20], cont


def test_parser_refusals(indexed):
    cont, every, counts, cols = indexed
    seek.parse_index(seek.write_index(cont, every, counts, *cols), cont)     # the unmutated index parses
    names = []
    for name, idx, data in _mutations(cont, every, counts, cols):
        with pytest.raises(ValueError):
            seek.parse_index(idx, data)
        names.append(name)
    assert len(names) == 14


def test_check_every():
    for K in (32, 64, 4096, 1 << 24):
        assert seek.check_every(K) == K
    for K in (0, 31, 33, 1 << 25, 4096.0, True, None):
        with pytest.raises(ValueError):
            seek.check_every(K)
