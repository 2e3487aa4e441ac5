"""GPU: every launch shape of the seek-index coders (DESIGN §4.13) against the C oracle.

* The recording encoder (l3c_ac_encode_streams_seek, ac_encode_seek_kernel<SPC>) at every alphabet and 1, 2 and 4
  streams per CTA, K = 32, 64, 96 and 4096, on the test_gpu_coder_launches stream grid and streams of K - 1 .. 2K + 1
  symbols: the bytes are the oracle's, every point equals oracle_points word for word, the sentinel rows around each
  stream's points (and the one a stream without points is given) are untouched, and the points round-trip through the
  sidecar writer and parser.
* The segment decoders (l3c_ac_decode_segments: ac_decode32_kernel<SEG>, v3::ac_decode_kernel<FULLROW, SPC, SEG> at
  SPC 1, 2 and 4) at K = 32, 64, 96 and one K above every length, on the same streams plus junk and truncated ones,
  planned by seek.plan_segments from the oracle's points: whole streams and random band cuts (start / lo / hi), in a
  shuffled order that mixes head and point segments of different lengths in one CTA, with zero-length segments and
  segment counts of every residue mod 4.  Every segment writes the oracle's symbols to its own output at +0..+3 from a
  word boundary, and nothing after them.  The points launched are counted per kind (test_seek_points_host.COVERAGE).
* The coarse segment decoder (l3c_ac_decode_segments_coarse) the same way on RGB planes of 23 points per stream at
  K = 32, from dmll_build_coarse records of peaked, broad and mixed mixtures.
* One stream past 2^32 code bits from the recording encoder through the sidecar to the segment decoder.
* The C entry points refuse bad arguments before they launch anything."""
import struct
import time

import numpy as np
import pytest
import torch

from oracle import ac
from tests.test_gpu_coder_launches import ALPHABETS, DECODE_CASES, _intervals, make_stream
from tests.test_seek_points_host import (COVERAGE, M32, classify, encoder_words, must_cover, oracle_points,
                                         seek_streams, stream_points)

pytestmark = pytest.mark.gpu

SENTINEL = 0x5EC0DE5A                  # the rows around each stream's points
UNWRITTEN = 0xA5A5A5A5                 # a point row before the launch (bit 31 of low set: no point has it)
GUARD = 8
CANARY = 0xA5


@pytest.fixture
def timed():
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print('wall time %.1f s' % (time.perf_counter() - t0))


def _container(streams):
    """a reference-layout container holding each (H, W, bytes) as the one stream of a 1 x H x W scale"""
    from l3c_pytorch_b200.codec import MAGIC
    parts = [struct.pack('<4H', 0, 0, 0, 0)]
    for h, w, b in streams:
        parts += [struct.pack('<BHH', 1, h, w), struct.pack('<I', len(b)), b, MAGIC]
    return b''.join(parts)


def _unpack_words(w):
    """encoder point words -> (low, high, flip, bits) int64"""
    w = w.astype(np.int64).reshape(-1, 4)
    return w[:, 0], w[:, 1], w[:, 3] & 0x80000000, w[:, 2] | ((w[:, 3] & 0x7FFFFFFF) << 32)


def _round_trip_index(ss, every, words, counts):
    from l3c_pytorch_b200 import seek
    cont = _container([(1, s.n, s.data) for s in ss])
    cols = _unpack_words(words)
    parsed = seek.parse_index(seek.write_index(cont, every, counts, *cols), cont)
    assert list(parsed.counts) == list(counts)
    for a, b in zip((parsed.low, parsed.high, parsed.flip, parsed.bits), cols):
        assert np.array_equal(a, b)


# ----------------------------------------------------------------------------------------------
# the recording encoder
# ----------------------------------------------------------------------------------------------
def _point_rows(counts):
    """rows of a points buffer: a sentinel row, then per stream its points and a sentinel row; a stream without
    points is given the sentinel row before it -> (first row per stream, row count, bool mask of sentinel rows)"""
    off = np.zeros(len(counts), np.int64)
    sent = [0]
    cur = 1
    for i, c in enumerate(counts):
        off[i] = cur if c else cur - 1
        if c:
            cur += int(c)
            sent.append(cur)
            cur += 1
    mask = np.zeros(cur, bool)
    mask[sent] = True
    return off, cur, mask


@pytest.mark.parametrize('spc', [1, 2, 4])
@pytest.mark.parametrize('L', ALPHABETS)
def test_recording_encoder_matches_oracle_points(L, spc, timed):
    from l3c_pytorch_b200 import _lib, codec, engine as E, seek
    dev = torch.device('cuda')
    ss = [s for s in seek_streams(L) if s.note == 'valid']
    idx = [i for i, s in enumerate(seek_streams(L)) if s.note == 'valid']
    n = np.array([s.n for s in ss], np.int64)
    iv = torch.from_numpy(np.concatenate([_intervals(s, L) for s in ss]).view(np.int32)).to(dev)
    caps = np.array([codec._slot_cap(int(k)) for k in n], np.int64)
    slots = torch.full((int(caps.sum()),), 0x5A, dtype=torch.uint8, device=dev)
    desc = np.zeros(len(ss), _lib.ENC_STREAM_DTYPE)
    desc['intervals'] = iv.data_ptr() + 4 * (np.cumsum(n) - n)
    desc['out'] = slots.data_ptr() + np.cumsum(caps) - caps
    desc['n_sym'], desc['out_cap'] = n, caps
    for every in (32, 64, 96, 4096):
        counts = seek.point_counts(n, every)
        off, _, sent = _point_rows(counts)
        init = np.where(sent[:, None], SENTINEL, UNWRITTEN).astype(np.uint32) * np.ones((1, 4), np.uint32)
        pts = torch.from_numpy(init.view(np.int32)).to(dev)
        with E.encoder_streams_per_cta(spc):
            _, lens, _ = E.ac_encode_streams_seek(desc, dev, every, pts, off)
        lens = lens.cpu().numpy().astype(np.int64)
        host = slots.cpu().numpy()
        words = pts.cpu().numpy().view(np.uint32)
        assert (words[sent] == SENTINEL).all(), (L, spc, every, 'sentinel rows written: %s'
                                                 % np.flatnonzero((words[sent] != SENTINEL).any(1)))
        for i, s in enumerate(ss):
            o = int(desc['out'][i] - slots.data_ptr())
            assert lens[i] == len(s.data) and host[o:o + lens[i]].tobytes() == s.data, (L, spc, every, s.kind, s.n)
            want = encoder_words(stream_points(L, every)[idx[i]])
            got = words[off[i]:off[i] + counts[i]]
            bad = np.flatnonzero((got != want).any(1))
            assert bad.size == 0, ('L=%d SPC %d K=%d stream %s n=%d: point %d is %s, oracle %s'
                                   % (L, spc, every, s.kind, s.n, bad[0], got[bad[0]].tolist(),
                                      want[bad[0]].tolist()))
        _round_trip_index(ss, every, words[~sent], counts)
        launched = [stream_points(L, every)[i] for i in idx]
        cov = {k: sum(int(classify(p, len(s.data))[k].sum()) for p, s in zip(launched, ss)) for k in COVERAGE}
        print('L=%d SPC %d K=%d: %d points recorded; %s' % (L, spc, every, int(counts.sum()),
                                                            ', '.join('%s %d' % kv for kv in cov.items())))
        # valid streams only: a window wholly past the end needs a truncated stream, and at K = 4096 no point of a
        # valid stream lies within 32 bits of its end
        for k in ('flip', 'span 2^32') + (('crosses end',) if every < 4096 else ()):
            assert cov[k] > 0, (L, spc, every, k)


# ----------------------------------------------------------------------------------------------
# the segment decoders
# ----------------------------------------------------------------------------------------------
class Streams(object):
    """streams on the device for segment launches: their bytes at odd, varied offsets of one blob, and per stream
    the address of its first row in `table` (row_pitch entries per symbol)"""

    def __init__(self, datas, n_sym, rows_addr, pitch, dev):
        self.datas, self.n = datas, np.asarray(n_sym, np.int64)
        lens = np.array([len(d) for d in datas], np.int64)
        gaps = 1 + np.arange(len(datas)) % 4
        self.dst = np.concatenate([[3], 3 + np.cumsum(lens[:-1] + gaps[:-1])]).astype(np.int64)
        blob = np.zeros(int(self.dst[-1] + lens[-1] + 16), np.uint8)
        for d, o in zip(datas, self.dst):
            blob[o:o + len(d)] = np.frombuffer(d, np.uint8)
        self.blob = torch.from_numpy(blob).to(dev)
        self.lens, self.rows_addr, self.pitch = lens, np.asarray(rows_addr, np.int64), pitch

    def descs(self, start):
        """decoder descriptors of every stream from symbol `start` on (sym_out: symbol index in the stream, rebased
        per segment by _launch)"""
        from l3c_pytorch_b200 import _lib
        d = np.zeros(len(self.datas), _lib.DEC_STREAM_DTYPE)
        d['in'] = self.blob.data_ptr() + self.dst
        d['in_len'] = self.lens
        d['n_sym'] = self.n - start
        d['table'] = self.rows_addr + 2 * self.pitch * start
        d['sym_out'] = start
        d['row_pitch'] = self.pitch
        return d


def _plan(st, pts, every, start=None, lo=None, hi=None):
    """seek.plan_segments over all streams of `st` from the oracle's points pts (one int64 [p][4] per stream) ->
    (segments, stream of each segment, first symbol of each segment, the state table that must stay alive)"""
    from l3c_pytorch_b200 import seek
    dev = st.blob.device
    counts = np.array([p.shape[0] for p in pts], np.int64)
    allp = np.concatenate(pts + [np.zeros((0, 4), np.int64)])
    index = seek.SeekIndex(every, counts, allp[:, 0], allp[:, 1], allp[:, 2], allp[:, 3])
    states = torch.from_numpy(np.concatenate([index.state_words().reshape(-1), np.zeros(8, np.uint32)])
                              .view(np.int32)).to(dev)
    s0 = np.zeros(len(pts), np.int64) if start is None else start
    desc = st.descs(s0)
    addr = desc['in'].astype(np.int64)
    order = np.argsort(addr)
    rank = np.empty_like(order)
    rank[order] = np.arange(order.size)
    kw = {} if start is None else dict(start=s0[order], lo=lo[order], hi=hi[order])
    segs = seek.plan_segments(desc, addr[order], np.full(len(pts), every, np.int64), index.first[order],
                              states.data_ptr(), **kw)
    sid = np.searchsorted(addr[order], segs['in'].astype(np.int64))
    sid = order[sid]
    at = segs['sym_out'].astype(np.int64)          # descs() put the stream's symbol index in sym_out
    return segs, sid, at, states, allp


def _launch(L, segs, sid, at, want, dev, spc, targets=None, rng=None, residue=0):
    """one l3c_ac_decode_segments(_coarse) launch of `segs` in a random order, padded with zero-length segments to a
    count = residue (mod 4), each segment writing to its own output at +0..+3 with GUARD canary bytes behind it;
    checks every segment's symbols against want[stream][first symbol ...] -> the launched order of (segment index or
    -1 for padding)"""
    from l3c_pytorch_b200 import engine as E
    pad = (residue - segs.size) % 4
    if pad:
        # zero-length copies of real segments: with a point and at the head
        extra = segs[rng.integers(0, segs.size, pad)].copy()
        extra['n_sym'] = 0
        extra['state'][::2] = 0
        segs = np.concatenate([segs, extra])
        sid = np.concatenate([sid, np.full(pad, -1)])
        at = np.concatenate([at, np.zeros(pad, np.int64)])
    perm = rng.permutation(segs.size)
    segs, sid, at = segs[perm], sid[perm], at[perm]
    nn = segs['n_sym'].astype(np.int64)
    slot = (nn + GUARD + 3) // 4 * 4 + 4
    out0 = np.cumsum(slot) - slot + np.arange(segs.size) % 4
    out = torch.full((int(slot.sum()),), CANARY, dtype=torch.uint8, device=dev)
    segs['sym_out'] = out.data_ptr() + out0
    with E.decoder_streams_per_cta(spc):
        E.ac_decode_segments(segs, dev, L, targets=targets)
        got = out.cpu().numpy()
    for k in range(segs.size):
        o, m = int(out0[k]), int(nn[k])
        if sid[k] >= 0:
            w = want[sid[k]][at[k]:at[k] + m]
            bad = np.flatnonzero(got[o:o + m] != w)
            assert bad.size == 0, ('segment %d (stream %d, symbols %d..%d, %s): %d wrong symbols, first at +%d'
                                   % (k, sid[k], at[k], at[k] + m, 'head' if segs['state'][k] == 0 else 'point',
                                      bad.size, bad[0]))
        assert (got[o + m:o + m + GUARD] == CANARY).all(), ('segment %d (stream %d, %d symbols) wrote past its end'
                                                            % (k, sid[k], m))
    return segs, sid


def _cta_mixes(segs, spc):
    """whether some CTA of the launch holds a head segment and a point segment of another length"""
    g = max(spc, 1)
    n = segs.size // g * g
    st = (segs['state'][:n] != 0).reshape(-1, g)
    ln = segs['n_sym'][:n].astype(np.int64).reshape(-1, g)
    for a, b in zip(st, ln):
        if a.any() and (~a).any() and len(set(b[a]) | set(b[~a])) > 1:
            return True
    return False


def _bands(rng, n, every):
    """random band cuts per stream: lo <= hi in [0, n], start at or before the point at or before lo; a few zero-length
    bands on a point"""
    lo = (rng.random(n.size) * (n + 1)).astype(np.int64)
    hi = lo + (rng.random(n.size) * (n - lo + 1)).astype(np.int64)
    z = rng.random(n.size) < 0.05
    lo[z] = hi[z] = lo[z] // every * every
    start = ((lo // every * every) * rng.random(n.size)).astype(np.int64)
    start[::3] = lo[::3] // every * every                               # some starting on their first point
    return start, lo, hi


def _check_segments(L, spc, st, pts_of, want, every, dev, rng, targets=None, assert_cover=True, tag=''):
    """whole streams and band cuts at `every`; -> coverage counts of the point segments launched"""
    from l3c_pytorch_b200 import seek
    pts = pts_of(every)
    residue = int(rng.integers(1, 4))
    # whole streams
    segs, sid, at, states, allp = _plan(st, pts, every)
    assert int(segs['n_sym'].astype(np.int64).sum()) == int(st.n.sum())
    lsegs, lsid = _launch(L, segs, sid, at, want, dev, spc, targets, rng, residue)
    assert lsegs.size % 4 == residue
    # the points the launch started segments from
    k = np.flatnonzero((lsegs['state'] != 0) & (lsid >= 0))
    g = (lsegs['state'][k].astype(np.int64) - states.data_ptr()) // (4 * seek.STATE_WORDS)
    assert g.size == allp.shape[0] and np.array_equal(np.sort(g), np.arange(g.size))
    cov = {name: int(m.sum()) for name, m in classify(allp[g], st.lens[lsid[k]]).items()}
    heads_and_points = _cta_mixes(lsegs, spc)
    # band cuts
    start, lo, hi = _bands(rng, st.n, every)
    segs, sid, at, states, _ = _plan(st, pts, every, start, lo, hi)
    nb = segs['n_sym'].astype(np.int64)
    cut = int(((at + nb < st.n[sid]) & (nb % 8 != 0)).sum())            # segments ending short of their stream
    after_start = int(((lo // every * every > start) & (hi > lo)).sum())
    zero = int((nb == 0).sum())
    _launch(L, segs, sid, at, want, dev, spc, targets, rng, (residue + 1) % 4)
    print('%sK=%d: %d points launched, %s; band cuts: %d segments end short of their stream at n_sym %% 8 != 0, %d '
          'bands start at a point after their descriptor\'s start, %d zero-length; heads and point segments share '
          'a CTA: %s' % (tag, every, sum(p.shape[0] for p in pts), ', '.join('%s %d' % kv for kv in cov.items()),
                         cut, after_start, zero, heads_and_points))
    assert cut > 0
    if any(p.shape[0] for p in pts):
        assert after_start > 0
    if assert_cover and any(p.shape[0] for p in pts):
        for name in must_cover(L, every):
            assert cov[name] > 0, (tag, every, name, cov)
        if spc >= 2:
            assert heads_and_points
    return cov


@pytest.mark.parametrize('L,spc', DECODE_CASES)
def test_segment_decoders_match_oracle(L, spc, timed):
    from l3c_pytorch_b200 import engine as E
    dev = torch.device('cuda')
    rng = np.random.default_rng(300 + L + spc)
    ss = seek_streams(L)
    n = np.array([s.n for s in ss], np.int64)
    pitch = E.table_pitch(L)
    tab = np.zeros((int(n.sum()), pitch), np.uint16)
    tab[:, :L] = np.concatenate([s.cdf[:, :L] for s in ss])
    tab_dev = torch.from_numpy(tab.view(np.int16)).to(dev)
    st = Streams([s.data for s in ss], n, tab_dev.data_ptr() + 2 * pitch * (np.cumsum(n) - n), pitch, dev)
    want = [s.want for s in ss]
    big = (int(n.max()) // 32 + 1) * 32
    for every in (32, 64, 96, big):
        _check_segments(L, spc, st, lambda K: stream_points(L, K), want, every, dev, rng,
                        tag='L=%d SPC %d ' % (L, spc))


# ----------------------------------------------------------------------------------------------
# the coarse segment decoder
# ----------------------------------------------------------------------------------------------
CH, CW = 24, 32                          # 768 pixels: 23 points per stream at K = 32
CNS = np.array([CH * CW, CH * CW - 37, 9, 1], np.int64)


def _coarse_case(kind, dev):
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    from tests.test_gpu_coarse_rows import C, K, KINDS, L, _params
    N, HW = CNS.size, CH * CW
    rng = np.random.default_rng(70 + KINDS.index(kind))
    l, sym = _params(kind, rng, N, CH, CW)
    l_dev = torch.from_numpy(l).to(dev)
    sym_dev = torch.from_numpy(sym.reshape(N, C, CH, CW)).to(dev)
    tg = DiscretizedMixLogisticLoss(True, 0, 255, L).targets(dev)
    table = torch.zeros(N * C * HW * L, dtype=torch.int16, device=dev)
    rec = torch.zeros(N * C * HW * E.COARSE_PITCH, dtype=torch.int16, device=dev)
    for c in range(C):
        E.dmll_build_table(l_dev, sym_dev, tg, C, K, L, True, c, table)
        E.dmll_build_coarse(l_dev, sym_dev, tg, K, L, c, rec)
    rows = table.cpu().numpy().view(np.uint16).reshape(N, C, HW, L)
    items = []                         # (plane, full rows, bytes given to the decoder)
    for nn in range(N):
        for c in range(C):
            full = np.concatenate([rows[nn, c, :CNS[nn]], np.zeros((CNS[nn], 1), np.uint16)], 1)
            data = ac.encode(full, sym[nn, c, :CNS[nn]])
            items.append((nn * C + c, full, data))
    # junk of a stream's own length and of 40 bytes, truncations to a half, 3 bytes and nothing
    items += [(0, items[0][1], rng.integers(0, 256, len(items[0][2]), np.uint8).tobytes()),
              (5, items[5][1], rng.integers(0, 256, 40, np.uint8).tobytes()),
              (1, items[1][1], items[1][2][:len(items[1][2]) // 2]), (3, items[3][1], items[3][2][:3]),
              (2, items[2][1], b'')]
    traces = [ac.decode_trace(full, data) for _, full, data in items]
    for i in range(N * C):
        nn, c = divmod(items[i][0], C)
        assert (traces[i][0] == sym[nn, c, :CNS[nn]]).all(), (kind, nn, c)
    return items, traces, tg, rec


@pytest.mark.parametrize('spc', [1, 2, 4])
@pytest.mark.parametrize('kind', ['peaked', 'broad', 'mixed'])
def test_coarse_segment_decoder_matches_oracle(kind, spc, timed):
    from l3c_pytorch_b200 import engine as E
    dev = torch.device('cuda')
    items, traces, tg, rec = _coarse_case(kind, dev)
    HW = CH * CW
    n = np.array([full.shape[0] for _, full, _ in items], np.int64)
    plane = np.array([p for p, _, _ in items], np.int64)
    st = Streams([d for _, _, d in items], n, rec.data_ptr() + 2 * E.COARSE_PITCH * HW * plane, E.COARSE_PITCH, dev)
    want = [t[0].astype(np.uint8) for t in traces]
    rng = np.random.default_rng(400 + spc)

    def pts_of(K):
        return [oracle_points(full, data, K, t[1]) for (_, full, data), t in zip(items, traces)]

    assert min(p.shape[0] for p in pts_of(32)[:3]) >= 20
    for every in (32, 96):
        _check_segments(256, spc, st, pts_of, want, every, dev, rng, targets=tg, assert_cover=False,
                        tag='coarse %s SPC %d ' % (kind, spc))


# ----------------------------------------------------------------------------------------------
# past 2^32 code bits, encoder to decoder
# ----------------------------------------------------------------------------------------------
def test_recording_encoder_past_2_32_bits_to_segments(timed):
    """Under the uniform L = 256 prior every symbol is its byte, 8 code bits, and leaves the coder at (0, 2^32 - 1):
    n random symbols code to their bytes followed by the terminator 0x40, and the point before symbol j is
    (0, 2^32 - 1, no flip, 32 + 8 j).  n = 2^29 + 2^22 + 5000 at K = 2^20 puts five points past 2^32 bits."""
    from l3c_pytorch_b200 import _lib, engine as E, seek
    dev = torch.device('cuda')
    n, every = (1 << 29) + (1 << 22) + 5000, 1 << 20
    hgt, wid = 9752, 55483                      # n = 9752 x 55483: one 1 x H x W scale of the container
    assert hgt * wid == n
    chunk = 1 << 24
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < 7 * n + (1 << 28):
        pytest.skip('needs %.1f GB of free device memory, %.1f GB are free' % ((7 * n + (1 << 28)) / 1e9, free / 1e9))
    g = torch.Generator(device=dev).manual_seed(6)
    src = torch.randint(0, 256, (n,), dtype=torch.uint8, device=dev, generator=g)
    iv = torch.empty(n, dtype=torch.int32, device=dev)
    for a in range(0, n, chunk):                 # interval [256 s, 256 s + 256): lo | (hi - 1) << 16, as uint32
        s = src[a:a + chunk].long() << 8
        w = s | ((s + 255) << 16)
        iv[a:a + chunk] = (w - ((w >> 31) << 32)).int()
    cap = (n + 64 + 3) // 4 * 4
    out = torch.zeros(cap, dtype=torch.uint8, device=dev)
    desc = np.zeros(1, _lib.ENC_STREAM_DTYPE)
    desc['intervals'], desc['out'], desc['n_sym'], desc['out_cap'] = iv.data_ptr(), out.data_ptr(), n, cap
    c = int(seek.point_counts([n], every)[0])
    pts = torch.full((c + 2, 4), SENTINEL, dtype=torch.int32, device=dev)
    _, lens, _ = E.ac_encode_streams_seek(desc, dev, every, pts, [1])
    torch.cuda.synchronize()
    del iv
    torch.cuda.empty_cache()
    assert int(lens.item()) & M32 == n + 1
    assert all(torch.equal(out[a:min(a + chunk, n)], src[a:a + chunk]) for a in range(0, n, chunk))
    assert int(out[n]) == 0x40
    words = pts.cpu().numpy().view(np.uint32)
    assert (words[[0, -1]] == SENTINEL).all()
    j = every * np.arange(1, c + 1, dtype=np.int64)
    closed = np.stack([np.zeros(c, np.int64), np.full(c, M32), np.zeros(c, np.int64), 32 + 8 * j], 1)
    assert np.array_equal(words[1:-1], encoder_words(closed))
    assert int((closed[:, 3] > (1 << 32)).sum()) == 5
    # the sidecar: 64-bit positions from 32-bit advances
    cont = _container([(hgt, wid, out[:n + 1].cpu().numpy().tobytes())])
    parsed = seek.parse_index(seek.write_index(cont, every, [c], *_unpack_words(words[1:-1])), cont)
    assert np.array_equal(parsed.bits, closed[:, 3]) and not parsed.flip.any()
    del cont
    states = torch.from_numpy(parsed.state_words().reshape(-1).view(np.int32).copy()).to(dev)
    row = torch.from_numpy(E.uniform_cdf_row(256).astype(np.uint16).view(np.int16)[:256].copy()).to(dev)
    dec = torch.full((n,), CANARY, dtype=torch.uint8, device=dev)
    dd = np.zeros(1, _lib.DEC_STREAM_DTYPE)
    dd['in'], dd['in_len'], dd['n_sym'] = out.data_ptr(), n + 1, n
    dd['table'], dd['row_pitch'], dd['sym_out'] = row.data_ptr(), 0, dec.data_ptr()
    segs = seek.plan_segments(dd, np.array([out.data_ptr()], np.int64), [every], [0], states.data_ptr())
    assert segs.size == c + 1
    E.ac_decode_segments(segs, dev, 256)
    bad = [a for a in range(0, n, chunk) if not torch.equal(dec[a:a + chunk], src[a:a + chunk])]
    assert not bad, 'symbols differ in the chunks at %s' % bad
    print('peak device memory: %.2f GiB' % (torch.cuda.max_memory_allocated() / 2 ** 30))


# ----------------------------------------------------------------------------------------------
# C ABI refusals
# ----------------------------------------------------------------------------------------------
def test_c_entry_points_refuse_bad_arguments_before_launching():
    from l3c_pytorch_b200 import _lib, codec, engine as E
    from l3c_pytorch_b200._lib import lib
    dev = torch.device('cuda')
    sp = E._stream_ptr()
    L, nsym = 100, 200
    s = make_stream(np.random.default_rng(5), 'flat', nsym, L)
    cdf, sym, rows = s.cdf, s.sym, s.cdf[:, :L]
    data = ac.encode(cdf, sym)
    iv = torch.from_numpy(_intervals(s, L).view(np.int32)).to(dev)
    cap = codec._slot_cap(nsym)
    enc_out = torch.full((cap,), CANARY, dtype=torch.uint8, device=dev)
    lens = torch.full((1,), -1, dtype=torch.int32, device=dev)
    pts = torch.full((8, 4), SENTINEL, dtype=torch.int32, device=dev)
    desc = np.zeros(1, _lib.ENC_STREAM_DTYPE)
    desc['intervals'], desc['out'], desc['n_sym'], desc['out_cap'] = iv.data_ptr(), enc_out.data_ptr(), nsym, cap
    desc_dev = E._desc_to_device(desc, dev)
    ptrs = E._to_device_async(np.array([pts.data_ptr()], np.int64), dev)
    refusals = []

    def refused(name, rc):
        assert rc != 0, name
        refusals.append((name, lib.l3c_last_error().decode()))

    for every in (0, 16, 48):
        refused('encode every=%d' % every, lib.l3c_ac_encode_streams_seek(desc_dev.data_ptr(), 1, lens.data_ptr(),
                                                                          every, ptrs.data_ptr(), sp))
    refused('encode n_streams=-1', lib.l3c_ac_encode_streams_seek(desc_dev.data_ptr(), -1, lens.data_ptr(), 32,
                                                                  ptrs.data_ptr(), sp))
    for what, args in (('descriptors', (None, 1, lens.data_ptr(), 32, ptrs.data_ptr(), sp)),
                       ('lengths', (desc_dev.data_ptr(), 1, None, 32, ptrs.data_ptr(), sp)),
                       ('points', (desc_dev.data_ptr(), 1, lens.data_ptr(), 32, None, sp))):
        refused('encode null %s' % what, lib.l3c_ac_encode_streams_seek(*args))
    # decoders: a valid one-segment launch of the stream, refused for each bad argument
    blob = torch.from_numpy(np.frombuffer(data, np.uint8).copy()).to(dev)
    pitch = E.table_pitch(L)
    tab = np.zeros((nsym, pitch), np.uint16)
    tab[:, :L] = rows
    tab_dev = torch.from_numpy(tab.view(np.int16)).to(dev)
    dec_out = torch.full((nsym + GUARD,), CANARY, dtype=torch.uint8, device=dev)
    seg = np.zeros(1, _lib.DEC_STREAM_DTYPE)
    seg['in'], seg['in_len'], seg['n_sym'] = blob.data_ptr(), len(data), nsym
    seg['table'], seg['row_pitch'], seg['sym_out'] = tab_dev.data_ptr(), pitch, dec_out.data_ptr()
    seg_dev = E._desc_to_device(seg, dev)
    tg = torch.zeros(256, dtype=torch.float32, device=dev)
    for bad_L in (0, 257):
        refused('segments L=%d' % bad_L, lib.l3c_ac_decode_segments(seg_dev.data_ptr(), 1, bad_L, sp))
    refused('segments n_segs=-1', lib.l3c_ac_decode_segments(seg_dev.data_ptr(), -1, L, sp))
    refused('segments null descriptors', lib.l3c_ac_decode_segments(None, 1, L, sp))
    refused('coarse n_segs=-1', lib.l3c_ac_decode_segments_coarse(seg_dev.data_ptr(), -1, tg.data_ptr(), sp))
    refused('coarse null descriptors', lib.l3c_ac_decode_segments_coarse(None, 1, tg.data_ptr(), sp))
    refused('coarse null targets', lib.l3c_ac_decode_segments_coarse(seg_dev.data_ptr(), 1, None, sp))
    torch.cuda.synchronize()
    for name, msg in refusals:
        print('%s: %s' % (name, msg))
        assert ('l3c_ac_encode_streams_seek' if name.startswith('encode') else
                'l3c_ac_decode_segments_coarse' if name.startswith('coarse') else 'l3c_ac_decode_segments') in msg
    # nothing ran: every output as it was
    assert int(lens.item()) == -1
    assert (enc_out.cpu().numpy() == CANARY).all() and (pts.cpu().numpy().view(np.uint32) == SENTINEL).all()
    assert (dec_out.cpu().numpy() == CANARY).all()
    # and the same arguments with the bad one corrected do run
    check = _lib.check
    check(lib.l3c_ac_encode_streams_seek(desc_dev.data_ptr(), 1, lens.data_ptr(), 32, ptrs.data_ptr(), sp))
    check(lib.l3c_ac_decode_segments(seg_dev.data_ptr(), 1, L, sp))
    torch.cuda.synchronize()
    assert int(lens.item()) == len(data) and enc_out[:len(data)].cpu().numpy().tobytes() == data
    got = dec_out.cpu().numpy()
    assert (got[:nsym] == sym).all() and (got[nsym:] == CANARY).all()
    want = encoder_words(oracle_points(cdf, data, 32))
    assert np.array_equal(pts.cpu().numpy().view(np.uint32)[:want.shape[0]], want)
