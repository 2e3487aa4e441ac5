"""GPU: the range decoders and the encoder on streams past 2^32 bits (512 MiB), past 2^31 bytes and up to 2^32 - 1
bytes, against the oracle's closed forms (test_coder_long_streams_host.py).

* Resumed decodes.  A resumed decode reads nothing before its saved position, so a stream whose oracle-coded tail
  lies at byte P needs only the tail in memory: `in` points P bytes before it, in_len = P + the tail's length, and the
  decoder resumes from the tail's initial state (low 0, high 2^32 - 1, its first 32 code bits) at bit 8 P + 32.  Every
  decoder family runs such tails of every kind, at offsets +0..+3 of `in` from a word boundary, crossing 2^32 bits and
  2^31 bytes inside a launch, resumed past them, and ending at byte 2^32 - 1, under chunk schedules of 1, 13 and the
  whole tail; after every launch the saved state equals the oracle's trace of the tail, 8 P bits further on, and
  after each schedule the symbols equal the tail's with the guard bytes behind them intact.
* A decode from symbol 0 of a uniform stream longer than 512 MiB, built on the GPU from the closed form (L = 256),
  and a round trip of more than 2^29 symbols through the drop-in's batched mixture calls, whose decode resumes its
  chunks past 2^32 bits.  (The same decode at L = 32768 takes about 1.1 us per symbol of its one stream, 316 s on an
  H100 80GB HBM3 at 700 W for 2.9e8 symbols, too long for the suite; the wide decoder meets the boundaries in the
  resumed decodes.)
* The encoder writing one stream of more than 2^31 bytes (15 bits per symbol: intervals of width 2), into a slot that
  holds it and into one that does not, and the drop-in's host path (lengths read as uint32, slot check, pack
  offsets) and pack on it.

Each test prints its peak device memory; it is skipped, with the reason, where the device has too little free."""
import time
import types

import numpy as np
import pytest
import torch

from oracle import ac
from tests.test_coder_long_streams_host import M32, tail_stream, uniform_row

gpu = pytest.mark.gpu
CANARY = 0xA5
GUARD = 64
# the symbol index every resumed tail starts at: any index will do, as nothing before it is read; its rows' address
# table - 2 pitch J stays a valid (positive) address at the widest pitch
J = 2 ** 30 + 3
N_TAIL = 301
KINDS = ('flat', 'peaked', 'tail', 'straddle', 'straddle-run', 'uniform')
CHUNK = 1 << 26                    # bytes per step of the on-device builders and comparisons
# the saved state of a stream of 2^28 bytes or more: low, high, value, code bits read (low word, high word)
STATE_WORDS = 5
PAST_END = 0x80000000              # bit 31 of word 0: a shorter stream's position is 2^32 bits or more


@pytest.fixture
def big_memory():
    """-> need(bytes): skips the test unless that much device memory is free.  Prints the test's peak device memory
    and its time."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()

    def need(nbytes):
        free = torch.cuda.mem_get_info()[0]
        if free < nbytes:
            pytest.skip('needs %.1f GB of free device memory, %.1f GB are free' % (nbytes / 1e9, free / 1e9))

    yield need
    torch.cuda.synchronize()
    print('peak device memory: %.2f GiB, %.1f s' % (torch.cuda.max_memory_allocated() / 2 ** 30,
                                                     time.perf_counter() - t0))
    torch.cuda.empty_cache()


def _engine():
    from l3c_pytorch_b200 import _lib, engine as E
    return _lib, E


# ----------------------------------------------------------------------------------------------
# resumed decodes at the boundaries
# ----------------------------------------------------------------------------------------------
def _positions(nbytes, final_bits):
    """byte offsets P of a tail of nbytes whose decoder has read final_bits when its last symbol is reached ->
    [(name, P)]: crossing 2^32 bits and 2^31 bytes inside a launch (resumed below, ending past), resumed past each,
    and ending at byte 2^32 - 1"""
    c = min(12, final_bits // 8)
    assert c >= 5, (nbytes, final_bits)                   # 8 (B - c) + 32 < 8 B <= 8 (B - c) + final_bits
    out = []
    for name, B in (('2^32 bits', 1 << 29), ('2^31 bytes', 1 << 31)):
        out += [(name + ', crossed', B - c), (name + ', resumed past', B + 5)]
    return out + [('in_len 2^32 - 1', (1 << 32) - 1 - nbytes)]


def _check_resumed(name, tails, esz, launch, dev):
    """tails: [SimpleNamespace(label, n, want bytes, sym, trace, table = device address of its row for symbol 0,
    pitch = its row pitch)];
    launch(desc_dev, n_streams, first, count).  One stream per (tail, position, offset of `in`), all in each launch."""
    _lib, E = _engine()
    items = []
    for t in tails:
        for pos_name, P in _positions(len(t.want), int(t.trace[-1, 3])):
            for mis in range(4):
                items.append((t, pos_name, P, mis))
    m = len(items)
    # the tails at word offsets of one blob, each placed so that `in` = its address - P lies mis bytes past a word
    base = np.cumsum([0] + [len(t.want) // 4 * 4 + 16 for (t, _, _, _) in items])[:-1]
    blob = torch.zeros(int(base[-1]) + len(items[-1][0].want) + 32, dtype=torch.uint8, device=dev)
    bp = blob.data_ptr()
    off = np.array([b + (mis + P - bp) % 4 for b, (_, _, P, mis) in zip(base, items)], np.int64)
    hb = np.zeros(blob.numel(), np.uint8)
    for o, (t, _, _, _) in zip(off, items):
        hb[o:o + len(t.want)] = np.frombuffer(t.want, np.uint8)
    blob.copy_(torch.from_numpy(hb))
    # outputs at +0..+3 (even for uint16 symbols), followed by guard bytes
    slot = np.array([t.n * esz + GUARD + 8 for (t, _, _, _) in items], np.int64)
    out0 = np.concatenate([[0], np.cumsum(slot)[:-1]]) + (np.arange(m) % 4) * esz
    out = torch.empty(int(slot.sum()), dtype=torch.uint8, device=dev)
    state = torch.empty(STATE_WORDS * m, dtype=torch.int32, device=dev)
    dd = np.zeros(m, dtype=_lib.DEC_STREAM_DTYPE)
    P = np.array([P for (_, _, P, _) in items], np.int64)
    dd['in'] = (bp + off - P).astype(np.uint64)
    assert ((dd['in'].astype(np.int64) & 3) == np.array([mis for (_, _, _, mis) in items])).all()
    dd['in_len'] = P + np.array([len(t.want) for (t, _, _, _) in items])
    dd['table'] = [t.table for (t, _, _, _) in items]
    dd['row_pitch'] = [t.pitch for (t, _, _, _) in items]
    dd['sym_out'] = (out.data_ptr() + out0 - J * esz).astype(np.uint64)
    dd['state'] = state.data_ptr() + 4 * STATE_WORDS * np.arange(m)
    dd['n_sym'] = [J + t.n for (t, _, _, _) in items]
    desc_dev = E._desc_to_device(dd, dev)
    start = 8 * P + 32                                          # the resumed bit position
    end = 8 * P + np.array([int(t.trace[-1, 3]) for (t, _, _, _) in items], np.int64)
    crossed = np.array(['crossed' in pn for (_, pn, _, _) in items])
    big_bits = np.array([pn.startswith('2^32 bits') for (_, pn, _, _) in items])
    big_bytes = ~big_bits
    # the boundaries are reached: crossed inside a launch, resumed at or past them, in_len at or past 2^31 bytes
    assert ((start < 2 ** 32) & (end >= 2 ** 32))[crossed & big_bits].all()
    assert ((start < 2 ** 34) & (end >= 2 ** 34))[crossed & ~big_bits].all()
    assert (start[~crossed & big_bits] >= 2 ** 32).all() and (start[~crossed & ~big_bits] >= 2 ** 34).all()
    assert (dd['in_len'][big_bytes].astype(np.int64) >= 2 ** 31).all() and dd['in_len'].max() == M32
    n_max = max(t.n for t in tails)
    schedules = [('whole tail', [(0, n_max)]), ('1, 13, rest', [(0, 1), (1, 13), (14, n_max)]),
                 ('13 at a time', [(f, 13) for f in range(0, n_max, 13)])]
    init = np.zeros((m, STATE_WORDS), np.uint32)
    init[:, 1] = M32
    init[:, 2] = [t.trace[0, 2] for (t, _, _, _) in items]
    init[:, 3], init[:, 4] = start & M32, start >> 32
    for sched_name, sched in schedules:
        out.fill_(CANARY)
        state.copy_(torch.from_numpy(init.reshape(-1).view(np.int32)))
        for first, count in sched:
            launch(desc_dev, m, J + first, count)
            st = state.cpu().numpy().view(np.uint32).reshape(m, STATE_WORDS).astype(np.int64)
            for i, (t, pn, P_i, mis) in enumerate(items):
                if first >= t.n:
                    continue
                tr = t.trace[min(first + count, t.n - 1)].astype(np.int64)
                want = [tr[0], tr[1], tr[2], 8 * P_i + tr[3]]
                got = [st[i, 0], st[i, 1], st[i, 2], st[i, 3] | (st[i, 4] << 32)]
                assert got == want, ('%s, %s, schedule "%s", launch (J + %d, %d), %s (P = %d), in at +%d: saved '
                                     'state %s, oracle %s' % (name, t.label, sched_name, first, count, pn, P_i, mis,
                                                              got, want))
        got = out.cpu().numpy()
        for i, (t, pn, P_i, mis) in enumerate(items):
            o = int(out0[i])
            seg = got[o:o + t.n * esz].view(np.uint16 if esz == 2 else np.uint8)
            bad = np.flatnonzero(seg != t.sym)
            assert bad.size == 0, ('%s, %s, schedule "%s", %s, in at +%d: %d wrong symbols, first at %d'
                                   % (name, t.label, sched_name, pn, mis, bad.size, bad[0]))
            assert (got[o + t.n * esz:o + t.n * esz + GUARD] == CANARY).all(), (name, t.label, pn, 'guard')
            assert (got[o - (o % 4):o] == CANARY).all(), (name, t.label, pn, 'written before the symbols')
    print('%s: %d streams per launch, in_len up to %d, resumed at bits %d .. %d' % (name, m, int(dd['in_len'].max()),
                                                                                  int(start.min()), int(start.max())))


def _row_tails(L, dev):
    """one tail of every kind at alphabet L, its rows at the library's pitch on the device -> (tails, keep)"""
    _lib, E = _engine()
    rng = np.random.default_rng(4000 + L)
    pitch = E.table_pitch(L)
    tails, keep = [], []
    for kind in KINDS:
        s = tail_stream(rng, kind, N_TAIL, L)
        sym, trace = ac.decode_trace(s.cdf, s.want)
        assert (sym == s.sym).all()
        tab = np.zeros((s.n, pitch), np.uint16)
        tab[:, :L] = s.cdf[:, :L]
        tab_dev = torch.from_numpy(tab.view(np.int16)).to(dev)
        keep.append(tab_dev)
        tails.append(types.SimpleNamespace(label=kind, n=s.n, want=s.want, sym=s.sym.astype(np.int64), trace=trace,
                                           table=tab_dev.data_ptr() - 2 * pitch * J, pitch=pitch))
        assert tails[-1].table > 0
    return tails, keep


@gpu
@pytest.mark.parametrize('L,spc', [(2, 0), (32, 0), (33, 1), (33, 2), (33, 4), (255, 1), (255, 2), (255, 4),
                                   (256, 1), (256, 2), (256, 4), (257, 0), (32768, 0)])
def test_resumed_decode_past_2_to_the_32_bits_and_2_to_the_31_bytes(L, spc):
    """ac_decode32 (L = 2, 32), v3 (33, 255 at SPC 1, 2, 4), v3 FULLROW (256, its uniform tail in span-2^32 groups)
    and the wide decoder (257, 32768), each on tails of every kind"""
    _lib, E = _engine()
    dev = torch.device('cuda')
    tails, keep = _row_tails(L, dev)

    def launch(desc_dev, m, first, count):
        E.check(E.lib.l3c_ac_decode_streams(E._ptr(desc_dev), m, L, first, count, E._stream_ptr()))

    with E.decoder_streams_per_cta(spc):
        _check_resumed('L=%d SPC=%d' % (L, spc), tails, 2 if L > 256 else 1, launch, dev)
    del keep


@gpu
@pytest.mark.parametrize('kind', ('peaked', 'broad', 'mixed'))
def test_resumed_coarse_rgb_decode_past_2_to_the_32_bits_and_2_to_the_31_bytes(kind):
    """the coarse RGB decoder on the three channels' oracle streams of a whole plane (test_gpu_coarse_rows), resumed
    from their records at the same positions"""
    from tests import test_gpu_coarse_rows as cr
    _lib, E = _engine()
    dev = torch.device('cuda')
    cs = cr._case(kind)
    tails = []
    for c in range(cr.C):
        full = np.concatenate([cs['rows'][0, c, :cr.HW], np.zeros((cr.HW, 1), np.uint16)], 1)
        data = cs['streams'][0][c]
        sym, trace = ac.decode_trace(full, data)
        assert (sym == cs['sym'][0, c]).all()
        tails.append(types.SimpleNamespace(label='%s channel %d' % (kind, c), n=cr.HW, want=data,
                                           sym=sym.astype(np.int64), trace=trace,
                                           table=cs['rec'].data_ptr() + 2 * E.COARSE_PITCH * (cr.HW * c - J),
                                           pitch=E.COARSE_PITCH))

    def launch(desc_dev, m, first, count):
        E.check(E.lib.l3c_ac_decode_streams_coarse(E._ptr(desc_dev), m, E._ptr(cs['tg']), first, count,
                                                   E._stream_ptr()))

    _check_resumed('coarse ' + kind, tails, 1, launch, dev)


@gpu
@pytest.mark.parametrize('L', (32, 256, 1024))
def test_short_stream_read_past_2_to_the_32_bits_stays_past_its_end(L):
    """A stream below 2^28 bytes keeps 4 state words.  Its decoder, resumed far past the stream's end just below 2^32
    bits, reads zeros (symbol 0 of the uniform row, k bits each) across 2^32 bits; the saved position wraps to a
    value inside the stream, with bit 31 of word 0 set, and the next launches still read zeros, not the stream's
    bytes.  The 5th word is never written.  (ac_decode32, v3 FULLROW and the wide decoder.)"""
    _lib, E = _engine()
    dev = torch.device('cuda')
    k = L.bit_length() - 1
    first0, n = 5, 40
    pitch = E.table_pitch(L)
    tab = np.zeros((first0 + n, pitch), np.uint16)
    tab[:, :L] = uniform_row(L)[:L]
    tab_dev = torch.from_numpy(tab.view(np.int16)).to(dev)
    junk = torch.from_numpy(np.random.default_rng(L).integers(1, 256, 200, np.uint8)).to(dev)
    in_len = 100
    esz = 2 if L > 256 else 1
    out = torch.full(((first0 + n) * esz + GUARD,), CANARY, dtype=torch.uint8, device=dev)
    state = torch.full((8,), -1, dtype=torch.int32, device=dev)
    bits0 = (1 << 32) - 5 * k                            # 5 symbols below 2^32 bits, far past the 100-byte stream
    init = np.array([0, M32, 0, bits0, 0x12345678], np.uint32)
    state[:5] = torch.from_numpy(init.view(np.int32))
    dd = np.zeros(1, dtype=_lib.DEC_STREAM_DTYPE)
    dd['table'], dd['row_pitch'] = tab_dev.data_ptr(), pitch
    dd['in'], dd['in_len'] = junk.data_ptr(), in_len
    dd['sym_out'], dd['n_sym'] = out.data_ptr(), first0 + n
    dd['state'] = state.data_ptr()
    desc_dev = E._desc_to_device(dd, dev)
    for first, count in ((first0, 8), (first0 + 8, 1), (first0 + 9, 13), (first0 + 22, n)):
        E.ac_decode_streams(dd, dev, L, first, count, desc_dev=desc_dev, n=1)
        st = state.cpu().numpy().view(np.uint32).astype(np.int64)
        bits = bits0 + k * (min(first + count, first0 + n - 1) - first0)
        assert bits >= 1 << 32 and (bits & M32) < 8 * in_len
        assert st[:4].tolist() == [PAST_END, M32, 0, bits & M32], (L, first, count, st.tolist())
        assert st[4] == 0x12345678 and (st[5:] == M32).all()
    got = out.cpu().numpy()
    assert (got[first0 * esz:(first0 + n) * esz] == 0).all(), (L, got[first0 * esz:(first0 + n) * esz])
    assert (got[:first0 * esz] == CANARY).all() and (got[(first0 + n) * esz:] == CANARY).all()


# ----------------------------------------------------------------------------------------------
# decodes from symbol 0 and round trips longer than 512 MiB
# ----------------------------------------------------------------------------------------------
def _pack_k(s, k, b0, b1):
    """bytes [b0, b1) of the closed-form stream of the symbols s (device, values < 2^k, 7 <= k <= 15): their k-bit
    MSB-first concatenation, the terminator bits 01, zero padding"""
    n = s.numel()
    bit = 8 * torch.arange(b0, b1, device=s.device, dtype=torch.int64)
    i = bit // k
    r = bit - i * k

    def ext(idx):
        v = s[idx.clamp(max=n - 1)].to(torch.int64) & ((1 << k) - 1)
        return torch.where(idx < n, v, torch.where(idx == n, torch.full_like(v, 1 << (k - 2)), torch.zeros_like(v)))

    v = (ext(i) << k) | ext(i + 1)
    return ((v >> (2 * k - 8 - r)) & 0xFF).to(torch.uint8)


def _stream_bytes(n, k):
    return (k * n + 2 + 7) // 8


def _assert_equal_chunked(a, b, what):
    for x in range(0, a.numel(), CHUNK):
        assert torch.equal(a[x:x + CHUNK], b[x:x + CHUNK]), (what, 'chunk at', x)


@gpu
@pytest.mark.parametrize('k', (8,))
def test_decode_from_symbol_0_of_a_uniform_stream_longer_than_512_mib(k, big_memory):
    """one l3c_ac_decode_streams launch over a whole uniform stream (shared row, pitch 0) of more than 2^32 bits, at
    L = 256 (v3 FULLROW, span-2^32 groups): the closed form's symbols and final state"""
    _lib, E = _engine()
    dev = torch.device('cuda')
    L = 1 << k
    n = (1 << 32) // k + (1 << 20)
    nb = _stream_bytes(n, k)
    assert 8 * nb > 2 ** 32
    esz = 2 if L > 256 else 1
    big_memory(n * (2 + esz) + nb + (1 << 30))
    g = torch.Generator(device=dev).manual_seed(k)
    s = torch.randint(0, L, (n,), generator=g, device=dev, dtype=torch.int32).to(torch.int16)
    data = torch.zeros(nb + 16, dtype=torch.uint8, device=dev)
    for b0 in range(0, nb, CHUNK):
        data[b0:min(nb, b0 + CHUNK)] = _pack_k(s, k, b0, min(nb, b0 + CHUNK))
    row = torch.from_numpy(np.resize(uniform_row(L)[:L], E.table_pitch(L)).view(np.int16).copy()).to(dev)
    out = torch.full((n * esz + GUARD,), CANARY, dtype=torch.uint8, device=dev)
    state = torch.zeros(STATE_WORDS, dtype=torch.int32, device=dev)
    dd = np.zeros(1, dtype=_lib.DEC_STREAM_DTYPE)
    dd['table'], dd['row_pitch'] = row.data_ptr(), 0
    dd['in'], dd['in_len'] = data.data_ptr(), nb
    dd['sym_out'], dd['n_sym'] = out.data_ptr(), n
    dd['state'] = state.data_ptr()
    t0 = time.perf_counter()
    E.ac_decode_streams(dd, dev, L, 0, n)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print('L=%d: %d symbols, %d bytes (%.3f x 2^32 bits) decoded in %.2f s (%.1f ns/symbol)'
          % (L, n, nb, 8 * nb / 2 ** 32, dt, dt * 1e9 / n))
    got = out[:n * esz].view(torch.int16 if esz == 2 else torch.uint8)
    _assert_equal_chunked(got, s if esz == 2 else s.to(torch.uint8), 'L=%d symbols' % L)
    assert bool((out[n * esz:] == CANARY).all()), 'guard'
    # the state at the final symbol: value = the 32 code bits from bit k (n - 1), after 32 + k (n - 1) bits
    bits = k * (n - 1)
    tail = data[bits // 8:bits // 8 + 8].cpu().numpy()
    value = (int.from_bytes(tail[:5].tobytes(), 'big') >> (8 - bits % 8)) & M32
    st = state.cpu().numpy().view(np.uint32).astype(np.int64)
    assert st[:3].tolist() == [0, M32, value] and (st[3] | (st[4] << 32)) == 32 + bits, (st.tolist(), value, bits)


@gpu
def test_mixture_round_trip_of_more_than_2_to_the_29_symbols(big_memory):
    """encode_logistic_mixture_batch and decode_logistic_mixture_batch of one broad K = 1 mixture at Lp = 257 over
    uniformly drawn symbols (about 9 bits each): the stream is longer than 512 MiB and plan_decode's chunks resume
    past 2^32 bits; the decoded symbols are the encoded ones"""
    from l3c_pytorch_b200 import torchac
    dev = torch.device('cuda')
    n = (1 << 29) + (1 << 16)
    big_memory(3 * 4 * n + 4 * n + 3 * n + 2 * n + (3 << 30))
    t = torch.linspace(-1.0, 1.0, 257, device=dev)
    mu = torch.zeros((1, 1, 1, n), device=dev)
    ls = torch.zeros((1, 1, 1, n), device=dev)
    pi = torch.ones((1, 1, 1, n), device=dev)
    g = torch.Generator(device=dev).manual_seed(5)
    sym = torch.randint(0, 256, (n,), generator=g, device=dev, dtype=torch.int16)
    t0 = time.perf_counter()
    data = torchac.encode_logistic_mixture_batch([t], [mu], [ls], [pi], [sym])[0]
    t1 = time.perf_counter()
    assert 8 * len(data) > 2 ** 32, len(data)
    back = torchac.decode_logistic_mixture_batch([t], [mu], [ls], [pi], [data])[0]
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    chunks = torchac.plan_decode(np.array([n], np.int64), np.array([256], np.int64))
    print('%d symbols, %d bytes (%.3f x 2^32 bits), %d decoder launches; encode %.1f s, decode %.1f s'
          % (n, len(data), 8 * len(data) / 2 ** 32, len(chunks), t1 - t0, t2 - t1))
    assert len(chunks) > 1
    _assert_equal_chunked(back, sym, 'mixture round trip')


# ----------------------------------------------------------------------------------------------
# the encoder and the drop-in's host path past 2^31 bytes
# ----------------------------------------------------------------------------------------------
@gpu
def test_encoder_writes_a_stream_of_more_than_2_to_the_31_bytes(big_memory):
    """intervals [2m, 2m + 2) for random 15-bit m: every symbol codes exactly m's 15 bits.  A stream of more than 2^31
    bytes: out_len, the bytes, the guard bytes behind the slot; the same stream into a slot of 2^31 bytes: the slot
    holds its first 2^31 bytes, nothing is written behind it and out_len still reports the whole length; the drop-in's
    host path reads that length as uint32, accepts the first slot and refuses the second before anything is packed,
    and the pack at its offsets returns the stream"""
    from l3c_pytorch_b200 import torchac
    _lib, E = _engine()
    dev = torch.device('cuda')
    n = 1_150_000_000
    nb = _stream_bytes(n, 15)
    assert nb > 2 ** 31
    cap = int(torchac.slot_caps(np.array([n]))[0])
    big_memory(4 * n + 2 * n + 2 * (cap + GUARD) + (1 << 30))
    g = torch.Generator(device=dev).manual_seed(15)
    m = torch.randint(0, 1 << 15, (n,), generator=g, device=dev, dtype=torch.int16)
    iv = torch.empty(n, dtype=torch.int32, device=dev)
    for a in range(0, n, CHUNK):
        x = m[a:a + CHUNK].to(torch.int64)
        w = 2 * x + ((2 * x + 1) << 16)
        iv[a:a + CHUNK] = torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)
    slot = torch.full((cap + GUARD,), CANARY, dtype=torch.uint8, device=dev)

    def encode(out_cap):
        desc = np.zeros(1, dtype=_lib.ENC_STREAM_DTYPE)
        desc['intervals'], desc['out'], desc['n_sym'], desc['out_cap'] = iv.data_ptr(), slot.data_ptr(), n, out_cap
        t0 = time.perf_counter()
        desc_dev, lens_dev = E.ac_encode_streams(desc, dev)
        torch.cuda.synchronize()
        print('out_cap %d: %d symbols encoded in %.2f s' % (out_cap, n, time.perf_counter() - t0))
        words = lens_dev.cpu().numpy()
        assert words[0] < 0                                  # an int32 read would see a negative length
        assert int(words.view(np.uint32)[0]) == nb, (out_cap, int(words.view(np.uint32)[0]), nb)
        assert bool((slot[out_cap:out_cap + GUARD] == CANARY).all()), (out_cap, 'written past out_cap')
        for b0 in range(0, min(nb, out_cap), CHUNK):
            b1 = min(nb, out_cap, b0 + CHUNK)
            assert torch.equal(slot[b0:b1], _pack_k(m, 15, b0, b1)), (out_cap, 'bytes at', b0)
        return desc_dev, lens_dev, words

    # the whole stream, then the drop-in's host path on it: uint32 lengths, the slot check, the pack offsets, the pack
    desc_dev, lens_dev, words = encode(cap)
    lens, dst = torchac._pack_offsets(words, np.array([cap]), np.array([0]))
    assert lens.tolist() == [nb] and dst.tolist() == [0, nb]
    blob = torch.full((int(dst[-1]) + 16,), CANARY, dtype=torch.uint8, device=dev)
    E.pack_streams(desc_dev, lens_dev, dst[:-1], 1, blob)
    torch.cuda.synchronize()
    for b0 in range(0, nb, CHUNK):
        b1 = min(nb, b0 + CHUNK)
        assert torch.equal(blob[b0:b1], _pack_k(m, 15, b0, b1)), ('packed bytes at', b0)
    assert bool((blob[nb:] == CANARY).all())
    del blob
    # the same stream into a slot of 2^31 bytes: truncated there, its full length reported, refused before the pack
    slot[1 << 31:(1 << 31) + GUARD] = CANARY
    _, _, words_small = encode(1 << 31)
    with pytest.raises(RuntimeError, match='stream 0: range coder output of %d bytes exceeded its slot of %d bytes'
                       % (nb, 1 << 31)):
        torchac._pack_offsets(words_small, np.array([1 << 31]), np.array([0]))
