"""Pins ac_oracle.c against the reference's own torchac.cpp (oracle/_ref, built by build_ref.py) for alphabets of
257 to 32768 symbols (Lp 258 .. 32769), which pin_oracle.py does not reach: random flat and peaked tables, long
underflow runs, junk and truncated input, and a uniform-row known answer at L = 1024.

As in pin_oracle.py, `--record` stores the sha256 of every reference output (and the KAT's bytes as hex) in
tests/golden/pin_oracle_wide.json where oracle/_ref is available; without it the same seeded cases are checked
against that file.  Every case keeps n_sym * Lp < 2^31, so the reference's own `int` row offset is valid.

row_search() gives the oracle's row search (ac_oracle.c row_search, the reference's torchac.cpp:276-296) for any
count, without a new export: a one-symbol stream whose first 32 code bits are count << 16 starts the decoder at
low = 0, high = 2^32 - 1, where its count ((value + 1) * 2^16 - 1) / 2^32 is exactly `count`.
TEST INFRASTRUCTURE ONLY."""
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ac, build_ref  # noqa: E402
from oracle.pin_oracle import _Live, _Stored  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden',
                      'pin_oracle_wide.json')
KAT_L = 1024
KAT_SYM = [0, 1023, 512, 1, 1022, 77, 640, 333, 0, 0, 1023, 999]


def row_search(row, counts):
    """the symbol the oracle's decoder picks in `row` (uint16 [Lp], strictly increasing over entries 0..L-1) for each
    count in `counts` (0..65535) -> int64 array"""
    row = ac._as_cdf(row).reshape(-1)
    counts = np.asarray(counts, np.int64).reshape(-1)
    assert ((0 <= counts) & (counts < 65536)).all()
    code = (counts.astype('>u4') << 16).astype('>u4')            # big-endian 32-bit code values
    buf = np.ascontiguousarray(code).view(np.uint8)
    out = np.empty(1, np.int16)
    f = ac.lib().oracle_ac_decode
    rp, bp, op, Lp = row.ctypes.data, buf.ctypes.data, out.ctypes.data, row.size
    res = np.empty(counts.size, np.int64)
    for i in range(counts.size):
        f(rp, 0, 1, Lp, ctypes.c_void_p(bp + 4 * i), 4, op)
        res[i] = out[0]
    return res


def random_rows(rng, n, L, peaked):
    """strictly increasing rows [n, L+1] with >= 1 count per symbol, first entry 0..29; peaked: one entry 500x
    heavier and 80 % of the symbols on it"""
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
    assert (np.diff(rows[:, :L], axis=1) > 0).all() and rows.max() <= 65535
    return rows.astype(np.uint16), sym.astype(np.int16)


def straddle_rows(rng, n, L):
    """symbol m = L/2 has [32768 - a, 32768 + a), a = 32..256, centred on the midpoint: coding it owes 7-9
    underflow bits and leaves the coder at the full interval, so owed bits pile up; 1 symbol in 37 (from symbol 40
    on) is 0 or L-1 and releases them"""
    m = L // 2
    a = 1 << rng.integers(5, 9, (n, 1))
    j = np.arange(L)[None]
    below = (j * (32768 - a)) // m
    above = 32768 + a + (j - m - 1) * (32768 - a - 1) // (L - m - 1)
    rows = np.zeros((n, L + 1), np.int64)
    rows[:, :L] = np.where(j <= m, below, above)
    sym = np.full(n, m)
    rel = rng.random(n) < 1 / 37
    rel[:40] = False
    sym[rel] = np.where(rng.random(int(rel.sum())) < 0.5, 0, L - 1)
    assert (np.diff(rows[:, :L], axis=1) > 0).all() and rows.max() <= 65535
    return rows.astype(np.uint16), sym.astype(np.int16)


def kat_row():
    """uniform row at L = 1024: entry m is 64 m, the dead last entry 0"""
    row = np.arange(KAT_L + 1, dtype=np.int64) * (65536 // KAT_L)
    row[KAT_L] = 0
    return row.astype(np.uint16)


def main(record=False):
    ref = build_ref.load()
    if ref is None:
        if not os.path.isfile(GOLDEN):
            print('reference backend and %s unavailable; nothing pinned' % GOLDEN)
            return 1
        chk = _Stored(GOLDEN)
        enc_ok = lambda got, t_cdf, sym: chk.encode(got)              # noqa: E731
        dec_ok = lambda got, t_cdf, data: chk.decode(got)             # noqa: E731
    else:
        chk = _Live(ref)
        enc_ok, dec_ok = chk.encode, chk.decode
    rng = np.random.default_rng(11)
    n_cases = 0

    def check(cdf, sym, what):
        n_sym, Lp = cdf.shape
        assert n_sym * Lp < 2 ** 31, what
        t_cdf = torch.from_numpy(cdf.view(np.int16).copy()).reshape(1, 1, n_sym, Lp)
        got = ac.encode(cdf, sym)
        assert enc_ok(got, t_cdf, sym), what
        dec = ac.decode(cdf, got)
        assert dec_ok(dec, t_cdf, got) and (dec == sym).all(), what
        # junk of half the length, and the stream cut in half: the decoder zero-fills, and must agree
        junk = bytes(rng.integers(0, 256, size=max(1, len(got) // 2)).astype(np.uint8))
        assert dec_ok(ac.decode(cdf, junk), t_cdf, junk), what + ('junk',)
        cut = got[:len(got) // 2]
        assert dec_ok(ac.decode(cdf, cut), t_cdf, cut), what + ('truncated',)

    for Lp, n_sym in [(258, 2000), (259, 777), (513, 1500), (1025, 1000), (4097, 300), (32769, 40)]:
        for peaked in (False, True):
            cdf, sym = random_rows(rng, n_sym, Lp - 1, peaked)
            check(cdf, sym, (Lp, n_sym, peaked))
            n_cases += 1
    n_under = 0
    for Lp, n_sym in [(1025, 3000), (4097, 500)]:
        cdf, sym = straddle_rows(rng, n_sym, Lp - 1)
        check(cdf, sym, ('underflow', Lp, n_sym))
        n_under += 1
    n_cases += n_under
    # KAT: uniform row at L = 1024, every symbol exactly 10 bits
    row = kat_row()
    kat = ac.encode(row, np.array(KAT_SYM, np.int16)).hex()
    assert (ac.decode(row, bytes.fromhex(kat), len(KAT_SYM)) == KAT_SYM).all()
    if ref is not None:
        t_row = torch.from_numpy(np.tile(row, (len(KAT_SYM), 1)).view(np.int16).copy()).reshape(1, 1, len(KAT_SYM), -1)
        assert ref.encode_cdf(t_row, torch.tensor(KAT_SYM, dtype=torch.int16)).hex() == kat
    if ref is None:
        assert chk.i == len(chk.calls)
        with open(GOLDEN) as f:
            assert json.load(f)['kat_uniform_1024'] == kat
    elif record:
        with open(GOLDEN, 'w') as f:
            json.dump({'source': 'reference torchac.cpp compiled by oracle/build_ref.py; sha256 of its encode '
                                 'bytes / decoded int16 symbols, in call order of pin_oracle_wide.main',
                       'kat_uniform_1024': kat, 'calls': chk.calls}, f, indent=0)
    print('pinned: %d random cases at Lp 258..32769 (incl. %d long-underflow ones) + uniform KAT at L = %d '
          'byte-identical to %s' % (n_cases, n_under, KAT_L, 'oracle/_ref' if ref is not None
                                    else 'the recorded reference outputs'))
    return 0


if __name__ == '__main__':
    sys.exit(main(record='--record' in sys.argv))
