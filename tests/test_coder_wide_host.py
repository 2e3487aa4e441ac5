"""CPU: the two-level row search of the wide range decoder (range_coder.cu, wide::ac_decode_wide_kernel, alphabets of
257 to 32768 symbols) as a numpy model, against the oracle's binary search for every count; and the C oracle pinned
against the reference's compiled coder at those alphabets (oracle/pin_oracle_wide.py)."""
import numpy as np
import pytest

from oracle import pin_oracle_wide

COUNTS = np.arange(65536, dtype=np.int64)


def wide_search(row, L, counts):
    """the symbol the wide decoder picks for each count, computed as the kernel does: `passes` is exact_step's
    compare, cdf[m] <= count.
      level 1: 256 packed heads (cdf[j*s] << 16) | j, s = ceil(L/256), 0 for buckets past the row; head 0 always
               passes (floor 0); the largest passing head gives the bucket j;
      level 2: entries m = j*s + t, t < s, m < L propose (cdf[m] << 16) | (cdf[m+1] - 1), 2^16 above entry L-1,
               0 past the bucket; entry j*s always passes; the symbol is j*s + (proposals up to the largest passing
               one) - 1.
    Returns (symbol, lower bound, upper bound - 1) per count."""
    c = np.asarray(row, np.int64)[:L]
    s = -(-L // 256)
    j = np.arange(256)
    valid1 = j * s < L
    head_cdf = np.where(valid1, c[np.minimum(j * s, L - 1)], 0)
    head = np.where(valid1, (head_cdf << 16) | j, 0)
    t = np.arange(128)
    out = []
    for blk in np.array_split(counts, 16):
        cnt = blk[:, None]
        pass1 = head_cdf[None] <= cnt
        pass1[:, 0] = True
        m0 = (np.where(pass1, head[None], 0).max(1) & 0xFFFF) * s
        m = m0[:, None] + t[None]
        valid2 = (t[None] < s) & (m < L)
        mc = np.minimum(m, L - 1)
        hi = np.where(mc + 1 == L, 65536, c[np.minimum(mc + 1, L - 1)])
        prop = np.where(valid2, (c[mc] << 16) | ((hi - 1) & 0xFFFF), 0)
        pass2 = c[mc] <= cnt
        pass2[:, 0] = True
        top = np.where(pass2, prop, 0).max(1)
        sym = m0 + (valid2 & (prop <= top[:, None])).sum(1) - 1
        out.append(np.stack([sym, top >> 16, top & 0xFFFF], 1))
    return np.concatenate(out)


def _check_row(row, L, what):
    row = np.asarray(row, np.int64)
    assert (np.diff(row[:L]) > 0).all() and row.min() >= 0 and row[:L].max() <= 65535, what
    got = wide_search(row, L, COUNTS)
    want = pin_oracle_wide.row_search(np.concatenate([row[:L], [0]]).astype(np.uint16), COUNTS)
    bad = np.flatnonzero(got[:, 0] != want)
    assert bad.size == 0, (what, 'count', int(bad[0]), 'model', int(got[bad[0], 0]), 'oracle', int(want[bad[0]]))
    # the winning proposal carries the symbol's interval
    sym = got[:, 0]
    hi = np.where(sym == L - 1, 65536, row[np.minimum(sym + 1, L - 1)])
    assert (got[:, 1] == row[sym]).all() and (got[:, 2] == hi - 1).all(), what


def _weighted_row(L, heavy, lead, weight):
    """cumulative row of 1-count intervals with entry `heavy` (a list) `weight` counts wide, starting at `lead`"""
    w = np.ones(L, np.int64)
    w[np.asarray(heavy)] = weight
    row = lead + np.concatenate([[0], np.cumsum(w)[:-1]])
    assert row[-1] + w[-1] <= 65536
    return row


@pytest.mark.parametrize('L', [257, 300, 1024, 4097, 32768])
def test_search_model_matches_oracle_on_random_rows(L):
    rng = np.random.default_rng(L)
    for peaked in (False, True):
        rows, _ = pin_oracle_wide.random_rows(rng, 2, L, peaked)
        for r in rows:
            _check_row(r, L, (L, peaked))


@pytest.mark.parametrize('L', [257, 300, 1024, 4097, 32768])
def test_search_model_matches_oracle_at_bucket_boundaries(L):
    """mass on entries j*s-1, j*s, j*s+1 (bucket edges), on entry 0 and on entry L-1, with cdf[0] = 0 and > 0"""
    s = -(-L // 256)
    rng = np.random.default_rng(50 + L)
    room = 65536 - L
    js = [1, int(rng.integers(2, (L - 2) // s)), (L - 2) // s]
    for j in js:
        for e in (j * s - 1, j * s, j * s + 1):
            if 0 < e < L:
                _check_row(_weighted_row(L, [e], 0, room // 2), L, (L, 'entry', e))
    _check_row(_weighted_row(L, [0], 0, room - 100), L, (L, 'entry 0'))
    _check_row(_weighted_row(L, [L - 1], 0, room - 100), L, (L, 'entry L-1'))
    _check_row(_weighted_row(L, [0, L - 1], 0, room // 3), L, (L, 'entries 0 and L-1'))
    # every bucket edge heavy at once
    edges = [e for j in range(1, -(-L // s)) for e in (j * s - 1, j * s) if e < L]
    _check_row(_weighted_row(L, edges, 0, 1 + (room - 50) // len(edges)), L, (L, 'all edges'))


@pytest.mark.parametrize('L', [257, 1024, 32768])
def test_search_model_matches_oracle_when_the_row_starts_above_0(L):
    """cdf[0] > 0: counts below it take the floor, symbol 0"""
    room = 65536 - L
    for lead in (1, 777, room - 1):
        _check_row(_weighted_row(L, [L // 2], lead, 1 + (room - lead) // 2), L, (L, 'lead', lead))
    _check_row(_weighted_row(L, [0], 65536 - L - 1, 1), L, (L, 'all at the top'))


def test_wide_oracle_pinned_against_compiled_reference():
    """the C oracle against the reference's torchac.cpp at Lp 258 .. 32769: live where oracle/_ref is built,
    otherwise against the reference outputs recorded in tests/golden/pin_oracle_wide.json"""
    assert pin_oracle_wide.main() == 0


def test_wide_oracle_pinned_against_the_recorded_outputs(monkeypatch):
    """the same cases against the recorded outputs alone, as on a machine without the reference"""
    from oracle import build_ref
    monkeypatch.setattr(build_ref, 'load', lambda: None)
    assert pin_oracle_wide.main() == 0


def test_table_pitch_for_wide_alphabets():
    from l3c_pytorch_b200 import engine as E
    assert [E.table_pitch(L) for L in (1, 25, 32, 33, 255, 256)] == [32, 32, 32, 256, 256, 256]
    assert [E.table_pitch(L) for L in (257, 263, 264, 265, 1024, 32767, 32768)] == [
        264, 264, 264, 272, 1024, 32768, 32768]
