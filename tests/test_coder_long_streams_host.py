"""CPU: closed forms of the range coder on uniform rows at L = 2^k, pinned against the C oracle (oracle.ac), that let
the GPU tests of streams past 2^32 bits and 2^31 bytes (test_gpu_coder_long_streams.py) know every byte, symbol and
coder state of such a stream without running the oracle on it; and the 32-bit position arithmetic the decoders used
before, restated, at the positions those tests reach.

On a uniform row at L = 2^k (cdf[m] = m 2^(16-k)) every symbol narrows the full interval [0, 2^32) to one of 2^k
equal parts, emits exactly its k bits MSB first and leaves the coder in its initial state: low = 0, high = 2^32 - 1,
no underflow bits owed.  So
  * a stream of j such symbols is their k-bit concatenation followed by the terminator, the two bits 01 (a decided
    0 and the one bit owed at termination, ac_oracle.c), zero-padded to a byte;
  * the decoder reaches symbol j in the state low = 0, high = 2^32 - 1, value = the 32 code bits from bit k j on
    (zero past the end), after 32 + k j bits;
  * j uniform symbols followed by any tail coded at the same L is the prefix's k j bits followed by
    oracle.encode(tail), when k j is a multiple of 8, and the decoder's states over the tail are those of
    oracle.decode_trace(tail) with k j more bits read.
The tails are those of test_gpu_coder_launches (flat, peaked, 1-count, straddle, straddle-run with more than 31
owed bits, uniform) and, above 256 symbols, a straddling row built for wide alphabets."""
import numpy as np
import pytest

from oracle import ac
from tests.test_gpu_coder_launches import HALF, make_stream, owed_bits

KS = tuple(range(1, 9)) + (15,)
TAIL_KINDS = ('flat', 'peaked', 'tail', 'straddle', 'straddle-run', 'uniform')
M32 = 0xFFFFFFFF


def uniform_row(L):
    """the row [L + 1] of the uniform prior at L = 2^k: cdf[m] = m 2^16 / L (the last entry is never read)"""
    assert L & (L - 1) == 0 and 2 <= L <= 32768
    row = np.arange(L + 1, dtype=np.int64) * (65536 // L)
    row[L] = 0
    return row.astype(np.uint16)


def pack_bits(values, k):
    """the k-bit MSB-first concatenation of values -> (bytes zero-padded, number of bits)"""
    v = np.asarray(values, np.int64)
    bits = ((v[:, None] >> np.arange(k - 1, -1, -1)[None]) & 1).reshape(-1).astype(np.uint8)
    return np.packbits(bits).tobytes(), bits.size


def uniform_stream(sym, k):
    """the closed form of the oracle's bytes for symbols on the uniform row at L = 2^k: the k-bit concatenation, the
    terminator bits 01, zero padding"""
    bits = ((np.asarray(sym, np.int64)[:, None] >> np.arange(k - 1, -1, -1)[None]) & 1).reshape(-1)
    return np.packbits(np.concatenate([bits, [0, 1]]).astype(np.uint8)).tobytes()


def uniform_trace(data, k, j):
    """the closed form of the decoder state at symbol j of a uniform stream: (low, high, value, bits read)"""
    buf = np.frombuffer(bytes(data) + bytes(8), np.uint8)
    b = k * j
    win = int.from_bytes(buf[b // 8:b // 8 + 5].tobytes(), 'big')          # 40 bits from byte b // 8
    return np.array([0, M32, (win >> (8 - b % 8)) & M32, 32 + b], np.uint32)


def _straddle_wide(rng, n, L, release):
    """straddling rows for L > 256 (make_stream's hold 2^14-count ranges, too narrow for so many entries): symbol m =
    L / 2 takes [32768 - a, 32768 + a), a = 2^5..2^8, the entries below and above it are spread evenly, so coding m
    from the full interval decides no bit and owes 7..9; releases are other symbols, from symbol 40 on"""
    m = L // 2
    a = 1 << rng.integers(5, 9, (n, 1))
    j = np.arange(L)[None]
    below = (j * (HALF - a)) // m
    above = HALF + a + ((j - m - 1) * (HALF - a)) // (L - m - 1)
    rows = np.zeros((n, L + 1), np.int64)
    rows[:, :L] = np.where(j <= m, below, above)
    rows[:, m] = (HALF - a)[:, 0]
    sym = np.full(n, m, np.int64)
    if release:
        rel = rng.random(n) < 1 / 37
        rel[:40] = False
        sym[rel] = rng.integers(0, L, int(rel.sum()))
        sym[rel & (sym == m)] = 0
    return rows, sym


def tail_stream(rng, kind, n, L):
    """a tail of the given kind at alphabet L (test_gpu_coder_launches.make_stream, straddling rows of their own above
    L = 256), with its oracle bytes in .want"""
    if kind.startswith('straddle') and L > 256:
        rows, sym = _straddle_wide(rng, n, L, kind == 'straddle')
        import types
        s = types.SimpleNamespace(kind=kind, n=n, cdf=rows.astype(np.uint16), sym=sym.astype(np.int16))
    else:
        s = make_stream(rng, kind, n, L)
    used = s.cdf[:, :L].astype(np.int64)
    assert (np.diff(used, axis=1) > 0).all(), (kind, L)
    s.want = ac.encode(s.cdf, s.sym)
    return s


# ----------------------------------------------------------------------------------------------
# the closed forms against the oracle
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('k', KS)
def test_uniform_stream_bytes_and_states_are_the_closed_form(k):
    L = 1 << k
    rng = np.random.default_rng(k)
    row = uniform_row(L)
    for n in (1, 2, 3, 7, 8, 9, 31, 33, 64, 257):
        sym = rng.integers(0, L, n)
        sym[:min(n, 2)] = (0, L - 1)[:min(n, 2)]
        rows = np.tile(row, (n, 1))
        data = ac.encode(rows, sym)
        assert data == uniform_stream(sym, k), (k, n)
        assert len(data) == (k * n + 2 + 7) // 8
        got, trace = ac.decode_trace(rows, data)
        assert (got == sym).all()
        want = np.stack([uniform_trace(data, k, j) for j in range(n)])
        assert (trace == want).all(), (k, n, np.argwhere(trace != want)[:1])
    # the terminator alone: a stream of one symbol 0 at k = 8 is 00 40
    if k == 8:
        assert ac.encode(np.tile(row, (1, 1)), [0]) == b'\x00\x40'


@pytest.mark.parametrize('k', KS)
def test_uniform_prefix_then_any_tail_is_prefix_bits_then_the_tail(k):
    """j uniform symbols, then a tail of each kind at the same L: the oracle's bytes are the prefix's bits followed by
    oracle.encode(tail) whenever k j is a multiple of 8, and its decoder states over the tail are the tail's own,
    k j bits further on"""
    L = 1 << k
    rng = np.random.default_rng(100 + k)
    row = uniform_row(L)
    kinds = [kd for kd in TAIL_KINDS if not (L == 2 and kd == 'straddle-run')]
    max_owed = 0
    for kind in kinds:
        for n_tail in (1, 9, 40, 301):
            tail = tail_stream(rng, kind, n_tail, L)
            if kind.startswith('straddle') and L > 2 and n_tail >= 64:
                max_owed = max(max_owed, int(owed_bits(tail, L).max()))
            for j in sorted({8 // np.gcd(k, 8), 2 * 8 // np.gcd(k, 8), 40}):
                if (k * j) % 8:
                    continue
                pre = rng.integers(0, L, j)
                rows = np.concatenate([np.tile(row, (j, 1)), tail.cdf])
                sym = np.concatenate([pre, tail.sym])
                data = ac.encode(rows, sym)
                head, nb = pack_bits(pre, k)
                assert nb == k * j and data == head + tail.want, (k, kind, n_tail, j)
                got, trace = ac.decode_trace(rows, data)
                assert (got == sym).all()
                _, tt = ac.decode_trace(tail.cdf, tail.want)
                shifted = tt.astype(np.int64)
                shifted[:, 3] += k * j
                assert (trace[j:].astype(np.int64) == shifted).all(), (k, kind, n_tail, j)
                assert (trace[:j] == np.stack([uniform_trace(data, k, i) for i in range(j)])).all()
    if L > 2:
        assert max_owed > 31, (k, max_owed)           # straddle-run tails owe more than a word of bits


# ----------------------------------------------------------------------------------------------
# the decoders' bit positions: the 32-bit arithmetic they used before, restated, against the word they must read
# ----------------------------------------------------------------------------------------------
def _s32(x):
    x &= M32
    return x - (1 << 32) if x >> 31 else x


def old_seek_word(bits, mis):
    """range_coder.cu before: open_stream seeks to state[3] + bit0 (32 bits) and takes word p >> 5"""
    return (((bits & M32) + 8 * mis) & M32) >> 5


def old_word_read(i, mis, in_len):
    """range_coder.cu before: load_raw(i) reads word i iff (int)end_byte - (int)(4u * i) > 0"""
    return _s32(mis + in_len) - _s32(4 * i) > 0


def old_window_moves(pos, n, wbase):
    """range_coder.cu before: skip(n) moves the window iff ((pos + n) >> 5) != wbase, pos a 32-bit bit count"""
    return (((pos + n) & M32) >> 5) != wbase


def seek_word(bits, mis):
    """the word holding code bit `bits` of a stream whose first byte lies mis bytes past a word boundary"""
    return (bits + 8 * mis) >> 5


def word_read(i, mis, in_len):
    """word i (from the word boundary below the stream) holds at least one byte of the stream"""
    return 4 * i < mis + in_len


def new_seek_word(state3, state4, mis):
    """range_coder.cu now: the 64-bit position in state words 3 and 4, wbase = p >> 5 as a 32-bit word index"""
    return ((((state4 << 32) | state3) + 8 * mis) >> 5) & M32


def new_word_read(i, mis, in_len):
    """range_coder.cu now: i < wend = ceil((mis + in_len) / 4), in 64 bits"""
    return i < ((mis + in_len + 3) >> 2)


def new_window_moves(pos, n):
    """range_coder.cu now: the window moves iff bit 5 of the (wrapping) bit counter flips"""
    return bool((pos ^ ((pos + n) & M32)) & 32)


# the positions test_gpu_coder_long_streams resumes at or crosses, as (code bits read, in_len)
BIT_BOUNDARY, BYTE_BOUNDARY, BYTE_END = 1 << 32, 1 << 31, (1 << 32) - 1


def test_the_old_32_bit_positions_read_the_wrong_words_past_the_boundaries():
    for mis in range(4):
        # below 2^32 bits both agree; at and past it the old seek lands 2^27 words early (the stream's start)
        for bits in (BIT_BOUNDARY - 64, BIT_BOUNDARY - 33):
            assert old_seek_word(bits, mis) == seek_word(bits, mis) == new_seek_word(bits & M32, bits >> 32, mis)
        for bits in (BIT_BOUNDARY, BIT_BOUNDARY + 8 * 5 + 32, 8 * BYTE_BOUNDARY + 32, 8 * (BYTE_END - 40)):
            want = seek_word(bits, mis)
            assert old_seek_word(bits, mis) != want and old_seek_word(bits, mis) < want - (1 << 26)
            assert new_seek_word(bits & M32, bits >> 32, mis) == want
        # a stream that ends at or past byte 2^31 (from the word boundary): its words below byte 2^31 read as zero
        # before, as themselves now
        for in_len in (BYTE_BOUNDARY - mis, BYTE_BOUNDARY + 7, BYTE_END):
            for i in (1, 2, (1 << 28) + 3, (1 << 29) - 1):
                assert word_read(i, mis, in_len) and new_word_read(i, mis, in_len)
                assert not old_word_read(i, mis, in_len), (mis, in_len, i)
            for i in ((mis + in_len + 3) // 4, (mis + in_len + 3) // 4 + 1):
                assert not word_read(i, mis, in_len) and not new_word_read(i, mis, in_len)
        for in_len in (BYTE_BOUNDARY - 4 - mis, 1000):
            for i in (0, (mis + in_len - 1) // 4, (mis + in_len + 3) // 4):
                assert old_word_read(i, mis, in_len) == word_read(i, mis, in_len) == new_word_read(i, mis, in_len)
    # past 2^32 bits the old bit counter has wrapped and no longer matches the window: it moves on every refill
    wbase = BIT_BOUNDARY // 32 + 3
    pos = (32 * wbase + 5) & M32
    assert all(old_window_moves(pos, n, wbase) for n in (0, 1, 8, 26))
    assert [new_window_moves(pos, n) for n in (0, 1, 8, 26, 27, 32)] == [False] * 4 + [True] * 2
    # and the state it saved kept only the low word of the position
    bits = 8 * BYTE_BOUNDARY + 32
    assert (bits & M32) == 32 and new_seek_word(bits & M32, bits >> 32, 0) == bits >> 5


# ----------------------------------------------------------------------------------------------
# the drop-in encoder's slot sizes and output lengths
# ----------------------------------------------------------------------------------------------
def test_slot_caps_fit_the_coders_uint32_and_lengths_read_as_uint32():
    from l3c_pytorch_b200 import codec, torchac
    n = np.array([1, 1000, 2 ** 30, 2_021_161_000, 2_021_161_100, 2 ** 31 - 1], np.int64)
    old = ((n * 17 + 7) // 8 + 64 + 3) & ~3
    caps = torchac.slot_caps(n)
    assert (caps <= torchac.SLOT_CAP_MAX).all() and (caps % 4 == 0).all()
    assert (caps == np.minimum(old, (1 << 32) - 4)).all()
    assert old[-1] >= 1 << 32 and (old[-1] & M32) < old[-1] // 2          # what a uint32 out_cap kept before
    assert (caps[:3] == codec._slot_cap(n[:3])).all()
    # lengths above 2^31 arrive as negative int32 words
    lens = np.array([5, 2 ** 31 + 3, 2 ** 32 - 5, 7], np.int64)
    words = lens.astype(np.uint32).view(np.int32)
    assert (words[1:3] < 0).all()
    caps = np.array([8, 2 ** 31 + 4, (1 << 32) - 4, 8], np.int64)
    got, dst = torchac._pack_offsets(words, caps, np.arange(4))
    assert (got == lens).all() and (dst == np.concatenate([[0], np.cumsum(lens)])).all() and (np.diff(dst) >= 0).all()
    assert (codec._host_lens(words) == lens).all()
    with pytest.raises(RuntimeError, match=r'stream 11: range coder output of 2147483651 bytes exceeded its slot of '
                                           r'2147483648 bytes'):
        torchac._pack_offsets(words, caps - np.array([0, 4, 0, 0]), np.arange(10, 14))
    with pytest.raises(RuntimeError, match='stream 2: range coder output of 4294967295 bytes'):
        torchac._pack_offsets(np.array([-1], np.int32), np.array([(1 << 32) - 4]), np.array([2]))
