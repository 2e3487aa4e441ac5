"""Seek indexes of reference-layout containers (DESIGN §4.13): the range coder's state every K symbols of every
stream, kept in a sidecar file, so that each stream splits into segments of K symbols that decode in parallel.

A seek point of a stream is the decoder's state before one of its symbols j = K, 2K, ... < n_sym:
  low, high    the coder interval (torchac.cpp:316-317, after the renormalisation of symbol j - 1);
  bits         the code bits the decoder has read: 32 + the sum of the renormalisation shifts of the symbols before j;
  flip         whether the last of those shifts was an "underflow" shift (torchac.cpp:350-362): it subtracts 2^30 from
               the code value before shifting, so the value is then the last 32 code bits read with bit 31 flipped,
               and otherwise those bits.  The index therefore does not store the value.

Sidecar bytes, little-endian:
  magic b'L3SK', u32 version (1), u32 K, u64 container length, u32 CRC32 of the container, u32 number of streams;
  per stream in container order: u32 point count (ceil(n_sym / K) - 1), then per point u32 low, u32 high and u32
  `advance` = (bits - bits of the previous point, or - 32 for the first) | flip << 31;
  u32 CRC32 of every byte before it.
Positions only move forward: an advance is unsigned, and one of more than 64 K bits (more than any K symbols read)
is refused.

The planner (plan_segments) turns decoder descriptors (l3c_dec_stream_t) into segment descriptors for
l3c_ac_decode_segments, vectorised over every stream of a scale, whatever the layout (equal-size, ragged or
recursive batches): descriptors are matched to their streams by the device address of their bytes."""
import struct
import zlib

import numpy as np

MAGIC = b'L3SK'
VERSION = 1
DEFAULT_EVERY = 4096
MAX_EVERY = 1 << 24
_HEAD = struct.Struct('<4sIIQII')
# words per point on the device: low, high, flip (0 or 2^31), bits low word, bits high word (l3c_ac_decode_segments)
STATE_WORDS = 5


def check_every(every):
    """K as an int; ValueError unless it is a multiple of 32 in [32, 2^24]."""
    if isinstance(every, bool) or not isinstance(every, (int, np.integer)) or every < 32 or every > MAX_EVERY \
            or every % 32:
        raise ValueError('seek interval %r must be a multiple of 32 in [32, 2^24]' % (every,))
    return int(every)


def point_counts(n_sym, every):
    """seek points of streams of n_sym symbols (int64 array) at interval `every`"""
    n = np.asarray(n_sym, np.int64)
    return np.maximum(0, -(-n // every) - 1)


def stream_symbols(data):
    """-> int64 [streams] symbols of every stream of a reference-layout container, in container order.  ValueError for
    a malformed or tiled container."""
    from .codec import container_tile, parse_container
    if container_tile(data) is not None:
        raise ValueError('seek indexes are for reference-layout containers; a tiled container\'s tiles already '
                         'decode in parallel')
    _, scales = parse_container(data)
    return np.array([H * W for (C, H, W, st) in scales for _ in st], np.int64)


class SeekIndex(object):
    """A parsed index: every (K), and per stream of the container its points as int64 arrays low, high, flip
    (0 or 2^31) and bits (absolute), concatenated in container order; first[i] is stream i's first point."""
    __slots__ = ('every', 'counts', 'first', 'low', 'high', 'flip', 'bits')

    def __init__(self, every, counts, low, high, flip, bits):
        self.every = int(every)
        self.counts = np.asarray(counts, np.int64)
        self.first = np.concatenate([[0], np.cumsum(self.counts)[:-1]]).astype(np.int64) if self.counts.size else \
            np.zeros(0, np.int64)
        self.low, self.high = np.asarray(low, np.int64), np.asarray(high, np.int64)
        self.flip, self.bits = np.asarray(flip, np.int64), np.asarray(bits, np.int64)

    def state_words(self):
        """uint32 [points][STATE_WORDS] as l3c_ac_decode_segments reads them"""
        w = np.zeros((self.low.size, STATE_WORDS), np.uint32)
        w[:, 0], w[:, 1], w[:, 2] = self.low, self.high, self.flip
        w[:, 3], w[:, 4] = self.bits & 0xFFFFFFFF, self.bits >> 32
        return w


def write_index(data, every, counts, low, high, flip, bits):
    """sidecar bytes of container `data` (see the module doc); the points as SeekIndex holds them"""
    every = check_every(every)
    counts = np.asarray(counts, np.int64)
    low, high = np.asarray(low, np.int64), np.asarray(high, np.int64)
    flip, bits = np.asarray(flip, np.int64), np.asarray(bits, np.int64)
    first = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64) if counts.size else counts
    prev = np.empty_like(bits)
    if bits.size:
        prev[1:] = bits[:-1]
        prev[first[counts > 0]] = 32
    adv = (bits - prev) | (flip & 0x80000000)
    rows = np.zeros((bits.size, 3), np.uint32)
    rows[:, 0], rows[:, 1], rows[:, 2] = low, high, adv & 0xFFFFFFFF
    parts = [_HEAD.pack(MAGIC, VERSION, every, len(data), zlib.crc32(data) & 0xFFFFFFFF, counts.size)]
    for i in range(counts.size):
        parts.append(struct.pack('<I', int(counts[i])))
        parts.append(rows[first[i]:first[i] + counts[i]].tobytes())
    out = b''.join(parts)
    return out + struct.pack('<I', zlib.crc32(out) & 0xFFFFFFFF)


def parse_index(idx, data):
    """-> SeekIndex of sidecar bytes `idx` for container `data`.  ValueError, before anything is sized from it, for a
    bad magic, version or CRC, a container whose length or CRC32 differs from the recorded ones, a tiled container, a
    K that is not a multiple of 32 in [32, 2^24], a point count other than ceil(n_sym / K) - 1 for a stream, a low
    with bit 31 set, a high not above its low, and an advance of more than 64 K bits."""
    idx = bytes(idx)
    if len(idx) < _HEAD.size + 4:
        raise ValueError('seek index too short')
    magic, version, every, clen, ccrc, n_streams = _HEAD.unpack_from(idx, 0)
    if magic != MAGIC:
        raise ValueError('not a seek index (bad magic)')
    if version != VERSION:
        raise ValueError('seek index version %d not supported' % version)
    if zlib.crc32(idx[:-4]) & 0xFFFFFFFF != struct.unpack_from('<I', idx, len(idx) - 4)[0]:
        raise ValueError('seek index CRC mismatch')
    if clen != len(data) or ccrc != zlib.crc32(data) & 0xFFFFFFFF:
        raise ValueError('seek index belongs to another container (length or CRC32 differs)')
    check_every(every)
    n_sym = stream_symbols(data)
    if n_streams != n_sym.size:
        raise ValueError('seek index lists %d streams, the container has %d' % (n_streams, n_sym.size))
    want = point_counts(n_sym, every)
    if len(idx) != _HEAD.size + 4 * n_sym.size + 12 * int(want.sum()) + 4:
        raise ValueError('seek index size does not match K=%d and the container\'s streams' % every)
    pos, rows = _HEAD.size, []
    for i in range(n_sym.size):
        cnt, = struct.unpack_from('<I', idx, pos)
        if cnt != want[i]:
            raise ValueError('stream %d: %d seek points, K=%d and %d symbols need %d' % (i, cnt, every, n_sym[i],
                                                                                     want[i]))
        pos += 4
        rows.append(np.frombuffer(idx, np.uint32, 3 * cnt, pos).reshape(cnt, 3))
        pos += 12 * cnt
    r = np.concatenate(rows).astype(np.int64) if rows else np.zeros((0, 3), np.int64)
    low, high, adv = r[:, 0], r[:, 1], r[:, 2]
    if (low >> 31).any():
        raise ValueError('seek point with bit 31 of low set')
    if (high <= low).any():
        raise ValueError('seek point whose high is not above its low')
    step = adv & 0x7FFFFFFF
    if (step > 64 * every).any():
        raise ValueError('seek point more than 64 K bits past the previous one')
    first = np.concatenate([[0], np.cumsum(want)[:-1]]).astype(np.int64)
    # absolute positions: per stream 32 + the running sum of its advances
    cs = np.cumsum(step)
    base = np.repeat(cs[first[want > 0]] - step[first[want > 0]], want[want > 0]) if step.size else step
    bits = 32 + cs - base
    return SeekIndex(every, want, low, high, adv & 0x80000000, bits)


def code_windows(blob_host, offs, lens, bits):
    """The 32 code bits ending at `bits` of the streams at byte offsets offs (length lens) of the uint8 array
    blob_host, zero past a stream's end (torchac.cpp:109-112), as int64 -- vectorised over points."""
    p = np.asarray(bits, np.int64) - 32
    byte = p >> 3
    acc = np.zeros(p.shape, np.int64)
    for k in range(5):
        i = byte + k
        ok = i < lens
        acc = (acc << 8) | np.where(ok, blob_host[np.where(ok, offs + i, 0)], 0).astype(np.int64)
    return (acc >> (8 - (p & 7))) & 0xFFFFFFFF


def plan_segments(desc, in_addr, every, first_point, state_ptr, start=None, lo=None, hi=None):
    """Segment descriptors (DEC_STREAM_DTYPE) of the decoder descriptors `desc` [M]: every stream cut into segments of
    its `every` symbols, segment s > 0 starting from seek point first_point + s - 1 of the batch's device state table
    at state_ptr (STATE_WORDS uint32 per point), segment 0 at the stream head.  in_addr: int64 sorted device addresses
    of the bytes of every stream of the batch; every / first_point: int64 per stream, in in_addr's order (a stream
    without an index has every >= its n_sym: one segment).
    start / lo / hi (int64 per stream, in in_addr's order; None: 0, 0 and start + n_sym): a descriptor's table and
    sym_out hold the stream's symbols from `start` on, and only [lo, hi) of them are needed (a band of a region decode,
    DESIGN §4.13 "Regions").  Then only the segments that meet [lo, hi) are emitted: the first one from the seek point
    at or before lo (which must not lie before `start`), the last one cut at hi.  Vectorised: no loop per segment."""
    addr = desc['in'].astype(np.int64)
    k = np.minimum(np.searchsorted(in_addr, addr), max(in_addr.size - 1, 0))
    if desc.size and (in_addr.size == 0 or (in_addr[k] != addr).any()):
        raise ValueError('a decoder descriptor reads no stream of the batch')
    K = np.asarray(every, np.int64)[k]
    n = desc['n_sym'].astype(np.int64)
    base = np.zeros_like(n) if start is None else np.asarray(start, np.int64)[k]
    a = base if lo is None else np.asarray(lo, np.int64)[k]
    b = base + n if hi is None else np.asarray(hi, np.int64)[k]
    j0 = a // K
    if (j0 * K < base).any() or (b > base + n).any():
        raise ValueError('a segment range reaches outside its descriptor\'s symbols')
    nseg = np.maximum(1, -(-b // K) - j0)
    sid = np.repeat(np.arange(desc.size), nseg)
    j = j0[sid] + np.arange(sid.size) - np.repeat(np.cumsum(nseg) - nseg, nseg)
    at = j * K[sid]                                      # the segment's first symbol, in stream coordinates
    rel = at - base[sid]                                 # ... and in the descriptor's
    segs = desc[sid].copy()
    segs['n_sym'] = np.maximum(0, np.minimum(K[sid], b[sid] - at))
    pitch = desc['row_pitch'].astype(np.int64)[sid]
    segs['table'] = desc['table'].astype(np.int64)[sid] + 2 * rel * pitch
    segs['sym_out'] = desc['sym_out'].astype(np.int64)[sid] + rel
    pt = np.asarray(first_point, np.int64)[k][sid] + j - 1
    segs['state'] = np.where(j == 0, 0, state_ptr + 4 * STATE_WORDS * pt)
    return segs
