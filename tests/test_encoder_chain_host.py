"""CPU: the range encoder's coding recurrence (range_coder.cu, encode_records) as a pure-Python model, against the
r-recurrence it replaced (kernel_models.coder_records, which test_host_logic pins to the oracle's bytes).

The kernel carries (low before its shift, s, and the next symbol's products (width - 1) * c + c pre-shifted by 16)
from one symbol to the next, shifts the products once by s = k + u and leaves bit 31 of the shifted low uncleared;
the r-recurrence carries (low, r = high - low) and forms span * c = r * c + c after both renormalisation shifts.  Both must give the same interval bounds mod 2^32,
the same records (low, k, u) per symbol and the same final low (the terminator bit) -- on streams of valid intervals
and at the edges: a stream's first symbol (span 2^32), c_hi = 65536 (where hi16 wraps to 0), c_lo = 0, the whole
range [0, 65536) (a width of 2^32), 1-count intervals, and on the step itself every shift s from 0 to 32."""
import numpy as np
import pytest

from tests.kernel_models import M32, coder_records as encode_r, shl as shl_c

M64 = (1 << 64) - 1


def shl64_hi(x, n):
    """PTX shf.l.clamp.b32 on the words of a 64-bit x: ((x << min(n, 32)) mod 2^64) >> 32"""
    return ((x << min(n, 32)) & M64) >> 32


def clz_nz(x):
    """PTX bfind.shiftamt.u32: clz for x != 0, 0xFFFFFFFF for 0"""
    return 32 - x.bit_length() if x else M32


def renorm(low, high):
    """the kernel's k and u: low ^ high is never 0 (the width is at least 2^14), and d & low == low & ~high"""
    d = low ^ high
    k = clz_nz(d)
    u = clz_nz(~shl_c(((d & low) << 1) & M32, k) & M32)
    return k, u


def encode_split(iv):
    """the kernel's recurrence: one shift by s, the next products formed from width before s is known, low's bit 31
    cleared only in the records and the terminator"""
    rec = []
    lowp, s = 0, 32                         # span 2^32 = 1 << 32
    c_lo, c_hi = iv[0] if iv else (0, 1)
    xl, xh = c_lo << 16, c_hi << 16
    for j in range(len(iv)):
        c_lo1, c_hi1 = iv[j + 1] if j + 1 < len(iv) else (0, 1)
        lo16, hi16 = shl64_hi(xl, s), shl64_hi(xh, s)
        lowm = shl_c(lowp, s)                   # bit 31 not cleared: it only flips bit 31 of low and high
        low = (lowm + lo16) & M32
        high = (lowm + hi16 - 1) & M32
        wm1 = (hi16 - lo16 - 1) & M32
        xl = ((wm1 * c_lo1 + c_lo1) << 16) & M64
        xh = ((wm1 * c_hi1 + c_hi1) << 16) & M64
        k, u = renorm(low, high)
        rec.append((low ^ (lowm & 0x80000000), k, u))
        lowp, s = low, k + u
    return rec, shl_c(lowp, s) & 0x7FFFFFFF


def _intervals(rng, n, L, peaked):
    """(c_lo, c_hi) of random symbols under random rows of L entries, every entry at least 1 count"""
    w = rng.integers(1, 40, size=(n, L)).astype(np.float64)
    if peaked:
        w[np.arange(n), rng.integers(0, L, n)] *= 3e4
    w = w / w.sum(1, keepdims=True) * (65536 - L)
    c = np.floor(np.cumsum(w, 1)).astype(np.int64) + np.arange(1, L + 1)
    c[:, -1] = 65536
    cdf = np.concatenate([np.zeros((n, 1), np.int64), c], 1)
    sym = rng.integers(0, L, n)
    return [(int(cdf[i, sym[i]]), int(cdf[i, sym[i] + 1])) for i in range(n)]


EDGE_STREAMS = {
    'whole range': [(0, 65536)] * 5,
    'whole range, then a symbol': [(0, 65536), (0, 65536), (17, 40000)],
    'c_hi = 65536': [(65535, 65536), (0, 65536), (1, 65536), (40000, 65536)] * 8,
    'c_lo = 0': [(0, 1), (0, 2), (0, 32768), (0, 65535)] * 8,
    'one count': [(v, v + 1) for v in (0, 1, 32767, 32768, 65534, 65535, 12345, 1)] * 8,
    'straddle the midpoint': [(32767, 32769)] * 64 + [(0, 1)],
    'alternate halves': [(0, 32768), (32768, 65536)] * 40,
}


@pytest.mark.parametrize('name', sorted(EDGE_STREAMS))
def test_split_recurrence_equals_r_recurrence_at_the_edges(name):
    iv = EDGE_STREAMS[name]
    assert encode_split(iv) == encode_r(iv)


@pytest.mark.parametrize('L,peaked,seed', [(2, False, 0), (3, True, 1), (25, True, 2), (256, False, 3),
                                           (256, True, 4), (4096, True, 5)])
def test_split_recurrence_equals_r_recurrence_on_random_streams(L, peaked, seed):
    rng = np.random.default_rng(seed)
    for n in (1, 2, 31, 33, 3001):
        iv = _intervals(rng, n, L, peaked)
        assert encode_split(iv) == encode_r(iv), (L, peaked, n)


def test_the_edges_reach_the_shifts_of_valid_streams():
    """a valid stream's span stays above 2^30, so a symbol of c counts leaves a width of at least c * 2^14 and s <= 18;
    the edge streams take s = 0, 1, 15 and 16.  Shifts up to 32 are checked on the step itself below"""
    seen = set()
    for iv in EDGE_STREAMS.values():
        seen |= {k + u for _, k, u in encode_split(iv)[0]}
    assert {0, 1, 15, 16} <= seen and max(seen) <= 18, sorted(seen)


@pytest.mark.parametrize('s', [0, 1, 15, 16, 17, 30, 31, 32])
def test_one_shift_of_the_products_equals_the_span_products(s):
    """hi32((((width - 1) * c + c) << 16) << s) == (((width << s) - 1) * c + c) >> 16 mod 2^32 for every width the
    renormalisation leaves at most 2^32 wide (width 0 stands for 2^32), c in [0, 65536]"""
    rng = np.random.default_rng(s)
    cs = [0, 1, 2, 32767, 32768, 65535, 65536] + [int(v) for v in rng.integers(0, 65537, 40)]
    top = 1 << (32 - s)                     # width << s <= 2^32
    ws = {1, top, max(top - 1, 1), top // 2 + 1} | {int(v) for v in rng.integers(1, top + 1, 40)}
    for w in ws:
        w32 = w & M32
        r = (shl_c(w32, s) - 1) & M32
        for c in cs:
            want = ((r * c + c) >> 16) & M32
            x = ((((w32 - 1) & M32) * c + c) << 16) & M64
            assert shl64_hi(x, s) == want, (w, s, c)
