"""Batched, device-resident encode/decode of `.l3c` containers -- the H100-first core that the
reference-shaped `Bitcoding` class (bitcoding.py) drives.

What the reference does one image, one scale, one channel at a time with a GPU->CPU round trip per
channel (src/bitcoding/bitcoding.py:85-123,163-294, coders.py:38-90) is done here
for a whole batch of images -- equally sized, or of any mix of sizes (a ragged batch, DESIGN §4.6: f16, learned
bottlenecks, the reference layout) -- with
  * ONE network pass,
  * one interval kernel per scale (no CDF table on the encode side),
  * ONE range-coder launch covering every stream of every image (N * 18 warps for L3C),
  * ONE gather kernel + ONE device->host copy producing the byte-exact container layout
    (bitcoding.py:326-363: 4 x u16 padding | per scale: u8 C, u16 H, u16 W | per channel: u32 len +
    stream | 4-byte magic).
Decoding uploads the concatenated containers once and decodes every stream in place.

Equal-size, tiled and ragged batches share one encode and one decode path: `stream_layout` says where every
stream's intervals (encode) or symbols and CDF rows (decode) sit in the `[N][C][plane]` tensor of its scale, and
only the step between those stream planes and the raster planes of the networks differs (a view, l3c_reorder_tiles
or l3c_ragged_pack).  Every decode -- full (`decode_device`) or of regions of tiled containers (`decode_region_pass`,
DESIGN §4.8) -- is one coarse-to-fine walk, `BatchCodec._decode_scales`, told its geometry by the caller; a large
scale of a tiled pass is decoded in bands of tile rows (DESIGN §4.10).  The encodes on windows -- a large tiled batch in
bands (DESIGN §4.10) and a region update (DESIGN §4.12) -- share two walks told their rectangles by the caller:
`BatchCodec._encode_windows`, the encoders fine to coarse, and `BatchCodec._code_rects`, the intervals of tile-aligned
rectangles coarse to fine, whose streams `region.rect_streams` finds and `_enc_descs` gives slots and descriptors.
"""
import functools
import os
import struct
import time

import numpy as np
import torch

from . import _lib
from . import engine as E
from . import seek as _seek
from .dmll import non_shared_get_K

MAGIC = b'\x46\xE2\x84\x92'          # bitcoding.py:36


def _on_device(fn):
    """Run a codec entry point with the blueprint's GPU as the current CUDA device: the kernels of the
    shared library launch on whatever device is current, and `current_stream()` is per device -- a
    Blueprint(device='cuda:1') must not depend on the caller having called torch.cuda.set_device(1)."""
    @functools.wraps(fn)
    def wrapped(self, *a, **kw):
        dev = self.codec.blueprint.device if isinstance(self, (EncodeJob, UpdateJob)) else self.blueprint.device
        if dev.type != 'cuda':
            return fn(self, *a, **kw)
        with torch.cuda.device(dev):
            return fn(self, *a, **kw)
    return wrapped


def _under_injection_tool():
    """True when a CUDA injection tool (Nsight Compute / Systems) is attached to this process: either it
    announced itself through the environment or its injection libraries are mapped.  Nsight Compute cannot
    profile kernels launched into green-context streams (it loses the process at the first one:
    "Failed to prepare kernel for profiling"), so the SM partitions are switched off under it -- same
    kernels, same bytes, ordinary streams; L3C_SM_PARTITION=1 forces them on."""
    if any(k in os.environ for k in ('CUDA_INJECTION64_PATH', 'CUDA_INJECTION32_PATH', 'NVTX_INJECTION64_PATH')):
        return True
    try:
        with open('/proc/self/maps') as f:
            for line in f:
                low = line.lower()
                if 'nsight' in low or 'injection' in low:
                    return True
    except OSError:
        pass
    return False


def _slot_cap(n_sym):
    """worst case: every symbol has probability 2^-16 -> 17 bits, plus termination."""
    return ((n_sym * 17 + 7) // 8 + 64 + 3) & ~3


def _enc_descs(ptrs, n_sym, dev):
    """Range-coder descriptors of the streams whose intervals start at the device addresses ptrs and hold n_sym symbols
    (int64 arrays of one shape), each given a slot of _slot_cap(n_sym) bytes in one new slot buffer.
    -> (caps, slots, desc): caps of ptrs' shape, desc flat in the arrays' order."""
    caps = _slot_cap(n_sym)
    slot_off = np.concatenate([[0], np.cumsum(caps)])
    slots = torch.empty(int(slot_off[-1]), dtype=torch.uint8, device=dev)
    desc = np.zeros(caps.size, dtype=_lib.ENC_STREAM_DTYPE)
    desc['intervals'] = ptrs.reshape(-1)
    desc['n_sym'] = n_sym.reshape(-1)
    desc['out_cap'] = caps.reshape(-1)
    desc['out'] = slots.data_ptr() + slot_off[:-1]
    return caps, slots, desc


def _host_lens(words):
    """the range coder's uint32 output lengths, as the int32 words a device tensor holds them -> int64"""
    return np.asarray(words).view(np.uint32).astype(np.int64)


def _check_lens(lens, caps):
    if (lens > caps).any():
        raise RuntimeError('range coder output exceeded its slot (corrupt CDF?)')


def _crop(src, at, r, nhwc):
    """Rectangle r (y0, x0, y1, x1) of every image of the plane src whose element (0, 0) sits at `at`, as a new tensor
    (l3c_crop_rect).  nhwc: src is NHWC [N, H, W, C]; otherwise planes [N, P, H, W]."""
    org = np.tile(np.array([r[0] - at[0], r[1] - at[1]], np.int32), (src.shape[0], 1))
    return E.crop_rect(src, E._to_device_async(org, src.device), r[2] - r[0], r[3] - r[1], nhwc=nhwc)


def _put(dst, D, K, src, at, nhwc):
    """Rectangle K (y0, x0, y1, x1) of the plane src, whose element (0, 0) sits at `at`, to its place in the destination
    plane of rectangle D: dst, allocated at the first piece written into it (dst None).  A first piece that is all of D
    becomes the destination itself, without a copy.  nhwc as in _crop.  -> the destination."""
    y, x = (1, 2) if nhwc else (2, 3)
    h, w = D[2] - D[0], D[3] - D[1]
    if dst is None:
        if tuple(K) == tuple(D) and tuple(at) == tuple(D[:2]) and (src.shape[y], src.shape[x]) == (h, w):
            return src.contiguous()
        shape = list(src.shape)
        shape[y], shape[x] = h, w
        dst = torch.empty(shape, dtype=src.dtype, device=src.device)

    def part(t, o):
        idx = [slice(None)] * t.dim()
        idx[y], idx[x] = slice(K[0] - o[0], K[2] - o[0]), slice(K[1] - o[1], K[3] - o[1])
        return t[tuple(idx)]
    part(dst, D).copy_(part(src, at))
    return dst


# BatchCodec.decode_regions: False runs every group of equal RegionPlan.shape_key on its own, also where one ragged pass
# per pass key would do (to compare the two)
REGION_RAGGED_PASS = True

# Largest N * H * W of one scale of an equal-size tiled pass that decode_device decodes whole; a larger scale is decoded
# in bands of tile rows of about this many pixels (DESIGN §4.10).  The rows, mixture parameters and classifier
# features of a whole-plane decode take about 2.1 KB per pixel (DESIGN §7), so a band of 8 Mpx keeps them near 20 GB.
TILED_BAND_PIXELS = 32 * 512 * 512

# Largest N * H * W of the image batch of an equal-size tiled encode that encode_begin runs whole; a larger one is
# encoded in bands (DESIGN §4.10): the encoder fine to coarse in bands of output rows, then the coding coarse to fine in
# the bands of tile rows of the banded decode, each band at most about this many pixels.  The whole-image encode takes
# about 750 B per pixel (DESIGN §7); the budget keeps bench.py's 16 x 512^2 tiled batch on that path.
TILED_ENCODE_BAND_PIXELS = 32 * 512 * 512

# Largest plane (H * W of one scale of one image) the kernels index: they take a plane's pixel count and the pixel
# index of a thread as 32-bit ints, so a plane is kept well below 2**31 pixels (DESIGN §4.10, "Index width").
MAX_PLANE_PIXELS = 2 ** 30


def check_plane(H, W, what):
    """ValueError, before any GPU work, for a plane the kernels cannot index (MAX_PLANE_PIXELS)."""
    if int(H) * int(W) > MAX_PLANE_PIXELS:
        raise ValueError('%s: a %dx%d plane has more than %d pixels, the most the kernels index'
                         % (what, H, W, MAX_PLANE_PIXELS))


TILED_MAGIC = b'L3CT'                # tiled containers: this tag + u16 tile_h + u16 tile_w follow the padding tuple


def tile_grid(H, W, tile):
    """[(offset, n_sym)] of the streams of one H x W symbol plane in stream order: the whole plane (compat
    format) or its tiles of tile = (th, tw) in row-major tile order (tile-major symbol order, dmll.cu)."""
    if tile is None:
        return [(0, H * W)]
    th, tw = tile
    out, off = [], 0
    for ty in range(-(-H // th)):
        h = min(th, H - ty * th)
        for tx in range(-(-W // tw)):
            w = min(tw, W - tx * tw)
            out.append((off, h * w))
            off += h * w
    return out


def stream_layout(shapes_of, tile=None, pad_tiles=False):
    """Where every stream of a batch lives (DESIGN §4.6 "Stream order").  shapes_of: [image][(C, h, w)] coarse ->
    fine.  Scale si has the plane length plane[si] = max_n h_n * w_n (H * W when the images are equal), and stream
    (n, si, c, t) covers the elements [(n*C + c) * plane[si] + off_t, ... + n_t) of that scale's [N][C][plane]
    tensor, (off_t, n_t) = tile_grid(h_n, w_n, tile)[t].
    pad_tiles: images whose planes have different tile counts (a ragged pass of region rectangles, DESIGN §4.8) get
    their per-channel stream lists padded to the largest count with empty streams (off 0, n_sym 0); otherwise such a
    batch is refused.
    -> (scale, elem, n_sym, plane): the scale index, first element and symbol count of every stream, int64
    [N][streams per image] in container order (image, scale, channel[, tile]), and plane int64 [scales]."""
    N = len(shapes_of)
    dims = np.array(shapes_of, np.int64).reshape(N, -1, 3)                 # [N][scale][C, h, w]
    if (dims[:, :, 0] != dims[:1, :, 0]).any():
        raise ValueError('images with different channel counts in one batch')
    plane = (dims[:, :, 1] * dims[:, :, 2]).max(0)
    img = np.arange(N)[:, None, None]
    grids, si, elem, n_sym = {}, [], [], []
    for k in range(dims.shape[1]):
        C = int(dims[0, k, 0])
        ext = list(map(tuple, dims[:, k, 1:].tolist()))
        distinct = set(ext)
        for e in distinct - grids.keys():
            grids[e] = np.array(tile_grid(e[0], e[1], tile), np.int64).T      # [offset, n_sym][tile]
        if len({grids[e].shape for e in distinct}) > 1:
            if not pad_tiles:
                raise ValueError('images with different numbers of tiles in one batch')
            T = max(grids[e].shape[1] for e in distinct)
            g = np.stack([np.pad(grids[e], ((0, 0), (0, T - grids[e].shape[1]))) for e in ext], 1)
        else:
            g = grids[ext[0]][:, None] if len(distinct) == 1 else np.stack([grids[e] for e in ext], 1)
        off, cnt = g[:, :, None, :]                                          # [N or 1][1][tiles] each
        shape = (N, C, off.shape[-1])
        si.append(np.full(shape, k))
        elem.append((img * C + np.arange(C)[None, :, None]) * plane[k] + off)
        n_sym.append(np.broadcast_to(cnt, shape))
    return tuple(np.concatenate([x.reshape(N, -1) for x in xs], 1) for xs in (si, elem, n_sym)) + (plane,)


class ContainerLayout(object):
    """Byte layout of one container given its per-stream lengths (scale order coarse -> fine).
    tile = None: the reference's `.l3c` layout (bitcoding.py:326-363), one stream per channel and scale.
    tile = (th, tw): the throughput layout -- every channel plane is cut into tiles that are coded as
    independent streams (thousands per batch instead of 18 per image); NOT readable by the reference and a few
    bytes per tile larger (4-byte length + termination), reported by bench.py as `tiled`."""

    def __init__(self, shapes, tile=None):
        self.shapes = shapes            # [(scale, C, H, W)] coarse -> fine
        self.tile = tile

    def header_and_offsets(self, lens, pad_tuple):
        """lens: stream byte counts in container order.  Returns (total size, [(offset, bytes)]
        header pieces, [stream offsets])."""
        pieces = [(0, struct.pack('<4H', *pad_tuple))]
        pos = 8
        if self.tile is not None:
            pieces.append((pos, TILED_MAGIC + struct.pack('<HH', *self.tile)))
            pos += 8
        offs = []
        i = 0
        for (_, C, H, W) in self.shapes:
            pieces.append((pos, struct.pack('<BHH', C, H, W)))
            pos += 5
            for _ in range(C * len(tile_grid(H, W, self.tile))):
                n = int(lens[i])
                pieces.append((pos, struct.pack('<I', n)))
                pos += 4
                offs.append(pos)
                pos += n
                i += 1
            pieces.append((pos, MAGIC))
            pos += 4
        return pos, pieces, offs

    def offsets(self, lens):
        """header_and_offsets' total size and stream offsets, without a loop over the streams: lens int64 [streams] in
        container order -> (total size, int64 [streams]).  Every stream's bytes follow its 4-byte length; a scale's
        streams follow its 5-byte header, and its 4-byte magic follows them."""
        th, tw = self.tile if self.tile is not None else (1 << 30, 1 << 30)
        per_scale = [C * -(-H // th) * -(-W // tw) for (_, C, H, W) in self.shapes]
        scale_of = np.repeat(np.arange(len(per_scale), dtype=np.int64), per_scale)
        lens = np.asarray(lens, np.int64)
        head = 8 if self.tile is None else 16
        offs = head + 9 * scale_of + 5 + np.cumsum(lens + 4) - lens
        return head + 9 * len(per_scale) + int((lens + 4).sum()), offs


def splice_segments(old_off, old_len, total_old, new_off, cols, lens, slot_off, src0=0, dst0=0):
    """The segments of l3c_splice_streams that turn one container into its update: old_off / old_len int64 [streams]
    where its streams lie in the old container of total_old bytes, new_off the offsets of the new layout
    (ContainerLayout.offsets), cols the ascending columns of the re-encoded streams, lens their new lengths and
    slot_off where their bytes lie in the slot buffer.  The old container sits at src0 of the source buffer, the new
    one at dst0 of the output.  -> int64 [segments][4] (src, src_off, dst_off, bytes): src 0 a run of unchanged streams
    with everything between them (their headers, scale headers and magics), from the end of the previous re-encoded
    stream to the length field of the next; src 1 a re-encoded stream, whose length field the kernel writes.  Runs of
    no bytes are left out."""
    cols = np.asarray(cols, np.int64)
    lens = np.asarray(lens, np.int64)
    a = np.concatenate([[0], old_off[cols] + old_len[cols]])           # run starts in the old container
    b = np.concatenate([old_off[cols] - 4, [total_old]])               # and ends
    d = np.concatenate([[0], new_off[cols] + lens])                    # their places in the new one
    seg = np.zeros((2 * cols.size + 1, 4), np.int64)
    seg[0::2] = np.stack([np.zeros_like(a), src0 + a, dst0 + d, b - a], 1)
    seg[1::2] = np.stack([np.ones_like(cols), np.asarray(slot_off, np.int64), dst0 + new_off[cols], lens], 1)
    return seg[(seg[:, 0] == 1) | (seg[:, 3] > 0)]


def update_layout_inputs(containers, caps):
    """The inputs of l3c_update_layout for the containers of an update call, from what the host knows before the new
    stream lengths exist.  containers: per container (scales, tile, old_base, old_bytes, cols, src): parse_container's
    scales and the tile size, where the old container lies in the uploaded buffer and its size, the ascending columns of
    its re-encoded streams and each one's index into the call's new lengths and caps (int64).  Each new container is
    given an upper bound of its size, old_bytes + sum(caps[src] - old length), rounded up to 16, and they follow one
    another in the output in input order.  -> (containers UPDATE_CONTAINER_DTYPE, streams UPDATE_STREAM_DTYPE, int64
    output offset of every container, output bytes)."""
    conts = np.zeros(len(containers), _lib.UPDATE_CONTAINER_DTYPE)
    streams, starts = [], np.zeros(len(containers), np.int64)
    pos = first = seg = 0
    for k, (scales, tile, base, nbytes, cols, src) in enumerate(containers):
        old = np.concatenate([np.asarray(st, np.int64).reshape(-1, 2) for (_, _, _, st) in scales])
        fixed_total, fixed_off = ContainerLayout([(i, C, H, W) for i, (C, H, W, _) in enumerate(scales)],
                                                 tile).offsets(np.zeros(len(old), np.int64))
        d = np.zeros(len(old), _lib.UPDATE_STREAM_DTYPE)
        d['fixed_off'], d['old_off'], d['old_len'], d['src'] = fixed_off, old[:, 0], old[:, 1], -1
        d['src'][cols] = src
        cap = (nbytes + int((np.asarray(caps, np.int64)[src] - old[cols, 1]).sum()) + 15) & ~15
        conts[k] = (first, len(old), fixed_total, base, nbytes, pos, cap, seg, len(cols))
        streams.append(d)
        starts[k] = pos
        pos, first, seg = pos + cap, first + len(old), seg + 2 * len(cols) + 1
    return conts, np.concatenate(streams) if streams else np.zeros(0, _lib.UPDATE_STREAM_DTYPE), starts, pos


def container_tile(data):
    """tile size (th, tw) of a tiled container, None for the reference layout."""
    if len(data) >= 16 and bytes(data[8:12]) == TILED_MAGIC:
        return struct.unpack_from('<HH', data, 12)
    return None


def _walk_streams(data, pos, n, out):
    """Read n streams (u32 length, then its bytes) from pos: -> the position after them, their (offset, length)
    appended to `out` unless it is None.  ValueError where the file ends first."""
    for _ in range(n):
        if pos + 4 > len(data):
            raise ValueError('truncated stream length')
        ln, = struct.unpack_from('<I', data, pos)
        pos += 4
        if pos + ln > len(data):
            raise ValueError('stream runs past the end of the file')
        if out is not None:
            out.append((pos, ln))
        pos += ln
    return pos


def parse_container(data):
    """-> (pad_tuple, [(C, H, W, [(offset, length), ...])] coarse -> fine); tiled containers (container_tile)
    list C * tiles streams per scale.  Raises ValueError on a malformed file (the reference asserts on the
    magic, bitcoding.py:154) and on a padding tuple that leaves no pixel of the finest scale on an axis.
    The work is bounded by the file's size, whatever its headers declare: a scale whose streams' length fields and
    separator cannot fit in the bytes left is refused before anything is built per stream."""
    if len(data) < 8:
        raise ValueError('container too short')
    pad_tuple = struct.unpack_from('<4H', data, 0)
    pos = 8
    tile = container_tile(data)
    if tile is not None:
        if tile[0] < 1 or tile[1] < 1:
            raise ValueError('tiled container with an empty tile size')
        pos = 16
    scales = []
    while pos < len(data):
        if pos + 5 > len(data):
            raise ValueError('truncated scale header')
        C, H, W = struct.unpack_from('<BHH', data, pos)
        pos += 5
        n = C * (1 if tile is None else -(-H // tile[0]) * -(-W // tile[1]))
        if 4 * n + 4 > len(data) - pos:
            # the walk fails within (len(data) - pos) / 4 fields; it only names where, as for a truncated file
            _walk_streams(data, pos, n, None)
            raise ValueError('scale separator missing: not a valid .l3c file')
        streams = []
        pos = _walk_streams(data, pos, n, streams)
        if data[pos:pos + 4] != MAGIC:
            raise ValueError('scale separator missing: not a valid .l3c file')
        pos += 4
        scales.append((C, H, W, streams))
    if scales:
        left, right, top, bottom = pad_tuple
        _, H, W, _ = scales[-1]
        if left + right >= W or top + bottom >= H:
            raise ValueError('padding tuple %r leaves no pixel of the %dx%d image' % (pad_tuple, H, W))
    return pad_tuple, scales


def _upload(datas, dev):
    """One upload of every container: -> (device blob, readable 16 bytes past every container; start of each)."""
    starts = np.zeros(len(datas), np.int64)
    pos = 0
    for n, dta in enumerate(datas):
        starts[n] = pos
        pos += (len(dta) + 15) & ~15
    host = torch.zeros(pos + 16, dtype=torch.uint8, pin_memory=True)
    hb = host.numpy()
    for n, dta in enumerate(datas):
        hb[starts[n]:starts[n] + len(dta)] = np.frombuffer(dta, np.uint8)
    return host.to(dev, non_blocking=True), starts


class DecodeLane(object):
    """Streams of one decode in flight (BatchCodec.lanes)."""
    __slots__ = ('main', 'dec', 'bld', 'partitioned')


class EncodeJob:
    """An encode in flight (BatchCodec.encode_begin): the range coder is queued on the current stream and the
    stream lengths are on their way to pinned memory.  finish() waits for them, lays the containers out, gathers
    the streams into one blob on the job's stream and (to_host) brings the bytes back: same results as
    encode_batch.  shapes: [(scale, C, H, W)] of the batch tensors; shapes_of / pads: the container shapes
    [(scale, C, h_n, w_n)] and the padding tuple of every image; caps: slot bytes [N][streams per image]."""

    seek = None        # (K, point counts per stream, device points int32 [points][4]): encode_begin(seek=K)

    def __init__(self, codec, shapes, shapes_of, pads, tile, out, caps, desc_dev, lens_dev, keep):
        self.codec, self.shapes, self.shapes_of, self.pads, self.tile, self.out = codec, shapes, shapes_of, pads, tile, out
        self.caps, self.desc_dev, self.lens_dev = caps, desc_dev, lens_dev
        self.keep = keep                                       # alive until finish()
        self.lens_host = torch.empty(lens_dev.shape, dtype=lens_dev.dtype, pin_memory=True)
        self.lens_host.copy_(lens_dev, non_blocking=True)
        self.stream = torch.cuda.current_stream()
        self.coded = torch.cuda.Event()
        self.coded.record(self.stream)

    @_on_device
    def finish(self, to_host=True):
        N, per_img = self.caps.shape
        self.coded.synchronize()                                                   # sync #1 (tiny)
        lens = _host_lens(self.lens_host.numpy()).reshape(N, per_img)
        _check_lens(lens, self.caps)
        with torch.cuda.stream(self.stream):
            # ---- container layout + gather + single D2H
            sizes, pieces_all, dst = [], [], np.zeros((N, per_img), np.int64)
            pos = 0
            starts = []
            for n in range(N):
                layout = ContainerLayout(self.shapes_of[n], self.tile)
                total, pieces, offs = layout.header_and_offsets(lens[n], self.pads[n])
                starts.append(pos)
                dst[n] = pos + np.asarray(offs, np.int64)
                pieces_all.append(pieces)
                sizes.append(total)
                pos += (total + 15) & ~15
            # seek points (encode_begin(seek=K)) ride behind the containers: one copy to the host for both
            n_pt = 0 if self.seek is None else self.seek[2].shape[0]
            blob = torch.empty(pos + 16 + 16 * n_pt, dtype=torch.uint8, device=self.lens_dev.device)
            E.pack_streams(self.desc_dev, self.lens_dev, dst.reshape(-1), N * per_img, blob)
            info = dict(sizes=sizes, starts=starts, lens=lens, shapes=self.shapes, shapes_of=self.shapes_of,
                        out=self.out, stream_offsets=dst, tile=self.tile)
            if n_pt:
                blob[pos + 16:].view(torch.int32).view(n_pt, 4).copy_(self.seek[2])
            if self.seek is not None:
                info['seek_points'] = blob[pos + 16:].view(torch.int32).view(n_pt, 4)
            if not to_host:
                self.packed = torch.cuda.Event()
                self.packed.record(self.stream)
                info['ready'] = self.packed          # consumers on another stream wait for this event
                self.keep = None
                return blob, info
            host = torch.empty(blob.shape, dtype=torch.uint8, pin_memory=True)
            host.copy_(blob, non_blocking=True)
            self.stream.synchronize()                                              # sync #2
        self.keep = None
        buf = host.numpy()
        datas = []
        for n in range(N):
            s0 = starts[n]
            for (o, b) in pieces_all[n]:
                buf[s0 + o:s0 + o + len(b)] = np.frombuffer(b, np.uint8)
            datas.append(buf[s0:s0 + sizes[n]].tobytes())
        if self.seek is not None:
            info['seeks'] = self._seek_indexes(datas, buf[pos + 16:].view(np.uint32).reshape(-1, 4), per_img)
        return datas, info

    def _seek_indexes(self, datas, words, per_img):
        """the sidecar bytes of every container from the recorded points (l3c_ac_encode_streams_seek's layout)"""
        every, counts, _ = self.seek
        words = words.astype(np.int64)
        first = np.cumsum(counts) - counts
        out = []
        for n, dta in enumerate(datas):
            cnt = counts[n * per_img:(n + 1) * per_img]
            a = int(first[n * per_img]) if cnt.size else 0
            w = words[a:a + int(cnt.sum())]
            out.append(_seek.write_index(dta, every, cnt, w[:, 0], w[:, 1], w[:, 3] & 0x80000000,
                                         w[:, 2] | ((w[:, 3] & 0x7FFFFFFF) << 32)))
        return out


class _UpdateJob(object):
    """One container of an update_regions call (BatchCodec.plan_updates): its bytes, parse_container's result, tile
    size, the edits as (y, x, h, w) rectangles and their patches (uint8 [1, 3, h, w] on the device) in list order, the
    merged plans (region.merge_update_plans) and whether it takes the whole path."""
    __slots__ = ('data', 'pad_tuple', 'parsed', 'tile', 'rects', 'patches', 'plans', 'whole')

    def __init__(self, data, pad_tuple, parsed, tile, rects, patches, plans, whole):
        self.data, self.pad_tuple, self.parsed, self.tile = data, pad_tuple, parsed, tile
        self.rects, self.patches, self.plans, self.whole = rects, patches, plans, whole


def _host_counts(job):
    """updates_counts of a container whose edit list is empty or that takes the whole path (_UpdateJob)."""
    total = job.plans[0][0].total_streams if job.plans else sum(len(st) for (_, _, _, st) in job.parsed)
    if not job.plans:
        return {'streams': 0, 'total': total, 'window_pixels': 0, 'whole': False, 'plans': 0}
    _, H, W = job.parsed[-1][:3]
    return {'streams': total, 'total': total, 'window_pixels': H * W, 'whole': True, 'plans': len(job.plans)}


class _WindowWork(object):
    """What BatchCodec._enqueue_windows queued for the window path of an update call."""
    __slots__ = ('blob', 'starts', 'upload_ms', 't_enqueue', 'keep', 'caps', 'slot_off', 'slots', 'lens_dev', 'cols',
                 'sl', 'counts')


class UpdateJob(object):
    """An update_regions call in flight (BatchCodec.update_regions_begin).  counts: one dict per container, with the
    keys of BatchCodec.updates_counts.  finish() -> the new container bytes in input order, as update_regions returns
    them.  It is the only place that waits for the GPU: one small copy of the window path's sizes and error flag,
    then its bytes, and the whole-path containers' EncodeJob.finish()."""

    def __init__(self, codec, outs, counts, whole, window):
        self.codec, self.counts = codec, counts
        self._outs = outs                  # containers done on the host (empty edit lists), None elsewhere
        self._whole = whole                # [(i, EncodeJob)]
        self._window = window              # None or (input indices, output starts, out, info_host, ready, stream, keep)

    @_on_device
    def finish(self):
        if self._outs is None:
            raise RuntimeError('UpdateJob.finish() was called before')
        outs, self._outs = self._outs, None
        if self._window is not None:
            idx, starts, out, info_host, ready, stream, _ = self._window
            ready.synchronize()
            info = info_host.numpy().astype(np.int64)
            sizes, flag = info[:-1], int(info[-1])
            if flag & 1:
                raise RuntimeError('range coder output exceeded its slot (corrupt CDF?)')
            if flag:
                raise RuntimeError('region update: a splice segment fell outside its buffer (flag %d)' % flag)
            end = int((starts + sizes).max())
            host = torch.empty(end, dtype=torch.uint8, pin_memory=True)
            with torch.cuda.stream(stream):
                host.copy_(out[:end], non_blocking=True)
                stream.synchronize()
            buf = host.numpy()
            for i, s0, n in zip(idx, starts, sizes):
                outs[i] = buf[s0:s0 + n].tobytes()
            self._window = None
        for i, job in self._whole:
            outs[i] = job.finish()[0][0]
        self._whole = []
        return outs


class _SegmentDecode(object):
    """decode_device's stream hook for seek-indexed images (DESIGN §4.13): the seek points of the batch uploaded once,
    and per call one l3c_ac_decode_segments launch of every segment of the descriptors' streams.  blob / offs as in
    decode_device; seeks: seek.SeekIndex or None per image.
    A region pass (decode_region_pass) gives the first P streams of every container (those of the scales its plans
    walk) and ranges = (start, lo, hi) int64 [N][P]: the stream symbol a descriptor's table and symbols start at and
    the symbols [lo, hi) to decode (seek.plan_segments)."""

    def __init__(self, blob, offs, seeks, ranges=None):
        N, P = offs.shape
        self.dev = blob.device
        addr = blob.data_ptr() + offs.reshape(-1)
        every = np.full(N * P, 1 << 40, np.int64)            # no index: one segment per stream
        first = np.zeros(N * P, np.int64)
        words, base = [], 0
        for n, sk in enumerate(seeks):
            if sk is None:
                continue
            if sk.counts.size != P and (ranges is None or sk.counts.size < P):
                raise ValueError('seek index %d lists %d streams, the container has %d' % (n, sk.counts.size, P))
            every[n * P:(n + 1) * P] = sk.every
            first[n * P:(n + 1) * P] = base + sk.first[:P]
            words.append(sk.state_words())
            base += sk.low.size
        order = np.argsort(addr, kind='stable')
        self.addr, self.every, self.first = addr[order], every[order], first[order]
        self.ranges = (None,) * 3 if ranges is None else tuple(np.asarray(r, np.int64).reshape(-1)[order]
                                                               for r in ranges)
        w = np.concatenate(words) if words else np.zeros((0, _seek.STATE_WORDS), np.uint32)
        self.states = E._to_device_async(np.concatenate([w.reshape(-1), [0]]).astype(np.uint32).view(np.int32),
                                         self.dev)

    def decode(self, dmll, desc, coarse):
        segs = _seek.plan_segments(desc, self.addr, self.every, self.first, self.states.data_ptr(), *self.ranges)
        E.ac_decode_segments(segs, self.dev, dmll.L, dmll.targets(self.dev) if coarse else None)


class _StateRecorder(object):
    """decode_device's stream hook for BatchCodec.seek_index: decodes the descriptors' streams serially in launches of
    `every` symbols and copies their saved states (l3c_dec_stream_t.state) into `points` after each launch, where the
    stream has symbols left.  n_sym int64 [N][P]: symbols of every stream, in offs' order."""

    def __init__(self, blob, offs, n_sym, every):
        self.dev, self.every = blob.device, every
        self.counts = _seek.point_counts(n_sym.reshape(-1), every)
        self.first = np.concatenate([[0], np.cumsum(self.counts)[:-1]]).astype(np.int64)
        addr = blob.data_ptr() + offs.reshape(-1)
        self.order = np.argsort(addr, kind='stable')
        self.addr = addr[self.order]
        self.points = torch.zeros(int(self.counts.sum()), _lib.DEC_STATE_WORDS, dtype=torch.int32, device=self.dev)

    def decode(self, dmll, desc, coarse):
        M, K = desc.size, self.every
        k = self.order[np.searchsorted(self.addr, desc['in'].astype(np.int64))]
        state = torch.zeros(M, _lib.DEC_STATE_WORDS, dtype=torch.int32, device=self.dev)
        desc = desc.copy()
        desc['state'] = state.data_ptr() + 4 * _lib.DEC_STATE_WORDS * np.arange(M)
        desc_dev = E._desc_to_device(desc, self.dev)
        n = desc['n_sym'].astype(np.int64)
        tg = dmll.targets(self.dev) if coarse else None
        for first in range(0, int(n.max()) if M else 0, K):
            if coarse:
                E.ac_decode_streams_coarse(None, self.dev, tg, first, K, desc_dev, M)
            else:
                E.ac_decode_streams(None, self.dev, dmll.L, first, K, desc_dev, M)
            sel = np.nonzero(n > first + K)[0]
            if sel.size:
                rows = self.first[k[sel]] + first // K
                self.points.index_copy_(0, E._to_device_async(rows, self.dev),
                                        state.index_select(0, E._to_device_async(sel.astype(np.int64), self.dev)))


class BatchCodec(object):
    def __init__(self, blueprint):
        self.blueprint = blueprint
        self.net = blueprint.net
        self._const = {}
        self._lane_cache = {}
        self._geo = None
        # streams and symbols the last decode_regions call handed to the range decoder (decode_region_pass)
        self.region_counts = {'streams': 0, 'symbols': 0}
        # what the last update_region call did: streams re-encoded, streams in the container, pixels of the window it
        # encoded and whether it took the whole-image path
        self.update_counts = {'streams': 0, 'total': 0, 'window_pixels': 0, 'whole': False}
        # one dict per container of the last update_regions call: update_counts' keys and `plans`, the plans after merging
        self.updates_counts = []
        # host clock of its stages in ms (tools/bench_update.py): parse and plan, upload, GPU (up to the new stream
        # lengths on the host), splice (layout, splice launch, copy to the host) and whole-path containers
        self.updates_stage_ms = {}

    # ------------------------------------------------------------------------------------------
    def iter_scale_dmll(self, recursive=0):
        """coarse -> fine: (scale, dmll, uniform) -- bitcoding.py:163-169.  recursive = R: a recursive container
        (DESIGN §4.7) with R more scales num_scales .. num_scales + R - 1 between the trained ones and the
        uniform-prior thumbnail (scale num_scales + R)."""
        losses = self.blueprint.losses
        n = self.net.scales + recursive
        for scale in reversed(range(n + 1)):
            yield (scale, losses.loss_dmol_rgb if scale == 0 else losses.loss_dmol_n, scale == n)

    def check_recursive(self, recursive):
        """-> R as an int: the number of extra applications of the last trained scale (a recursive container,
        DESIGN §4.7).  ValueError unless it is a non-negative int, and for R > 0 on a model that is not an RGB
        baseline: the learned bottlenecks of L3C are not images that its last scale could code again."""
        if isinstance(recursive, bool) or not isinstance(recursive, (int, np.integer)) or recursive < 0:
            raise ValueError('recursive must be a non-negative int, got %r' % (recursive,))
        if recursive and not self.net._rgb:
            raise ValueError('recursive=%d: only the RGB baselines code recursively (their scales are bicubic '
                             'thumbnails); the L3C bottlenecks cannot be coded by the last scale again' % recursive)
        return int(recursive)

    def _uniform(self, L, device):
        key = ('uniform', L, str(device))
        if key not in self._const:
            row = E.uniform_cdf_row(L).astype(np.int64)
            hi = np.concatenate([row[1:L], [65536]])
            lut = np.zeros(256, np.int64)
            lut[:L] = row[:L] | ((hi - 1) << 16)
            lut_dev = torch.from_numpy(lut.astype(np.uint32).view(np.int32).copy()).to(device)
            pitch = E.table_pitch(L)
            trow = np.zeros(pitch, np.uint16)
            trow[:L] = row[:L]
            row_dev = torch.from_numpy(trow.view(np.int16).copy()).to(device)
            self._const[key] = (lut_dev, row_dev)
        return self._const[key]

    def _rgb_shift(self, device):
        """RGB baselines feed `S - 255*rgb_mean` to the decoder nets (net.py:77-80; SURVEY finding 2)."""
        if not self.net._rgb:
            return None
        return self.net.nets[0].enc._consts(device)[1]

    # ------------------------------------------------------------------------------------------
    def encode_batch(self, imgs_u8, pad_tuple=(0, 0, 0, 0), out=None, to_host=True, tile=None, extents=None,
                     recursive=0, seek=None):
        """imgs_u8: uint8 [N,3,H,W] on the GPU, H and W multiples of 2**num_scales.  pad_tuple: the padding
        tuple written into every container, or a list of one per image.
        Returns a list of N container byte strings (or, with to_host=False, the device blob,
        per-image sizes and offsets, leaving the bytes in HBM).  `out`: a precomputed network Out.
        tile = (th, tw): tiled containers (ContainerLayout).
        extents = [(h_n, w_n)]: a ragged batch (encode_begin).
        recursive = R: recursive containers (encode_begin).
        seek = K: also seek indexes (encode_begin); info['seeks'] holds them."""
        return self.encode_begin(imgs_u8, pad_tuple, out, tile, extents, recursive, seek).finish(to_host)

    def ragged_unsupported(self, tile=None):
        """Why this codec cannot code a ragged batch (a message naming it), or None when it can."""
        why = self.net.ragged_unsupported()
        if why is None and tile is not None:
            why = 'ragged batches are not supported with tiled containers (tile=%s)' % (tuple(tile),)
        return why

    def _ragged_extents(self, extents, N, H, W, tile):
        """Validated [(h_n, w_n)] of a ragged batch of N images in an H x W tensor, or None when every image fills
        the tensor (then the call is the equal-size one, with the same kernel arguments)."""
        if extents is None:
            return None
        ext = [(int(h), int(w)) for (h, w) in extents]
        fac = 2 ** self.net.config_ms.num_scales
        if len(ext) != N:
            raise ValueError('%d extents for a batch of %d images' % (len(ext), N))
        for (h, w) in ext:
            if not (1 <= h <= H and 1 <= w <= W) or h % fac or w % fac:
                raise ValueError('extent %dx%d must lie in the %dx%d batch and be a multiple of %d'
                                 % (h, w, H, W, fac))
        if all(e == (H, W) for e in ext):
            return None
        why = self.ragged_unsupported(tile)
        if why is not None:
            raise NotImplementedError(why)
        return ext

    @_on_device
    def encode_begin(self, imgs_u8, pad_tuple=(0, 0, 0, 0), out=None, tile=None, extents=None, recursive=0,
                     seek=None):
        """First half of encode_batch: enqueues the whole GPU side of an encode (networks, intervals,
        the range-coder launch, the copy of the stream lengths to pinned memory) on the CURRENT stream
        and returns without waiting.  EncodeJob.finish() completes it.  Lets a caller overlap the
        encode of one batch with other work, e.g. the latency-bound decode of the previous batch.

        pad_tuple: one padding tuple for every container, or a list of one per image.
        extents = [(h_n, w_n)]: a ragged batch (DESIGN §4.6): image n is the top-left h_n x w_n of imgs_u8[n]
        (zero elsewhere; multiples of 2**num_scales), and every container is byte-identical to the one of that
        image encoded on its own -- one network pass and one range-coder launch for the batch.  f16, learned
        bottlenecks, reference layout only.  Extents that all equal the tensor are the equal-size call.
        recursive = R > 0 (RGB baselines, DESIGN §4.7): the last trained scale codes its own thumbnails R more
        times (forward(auto_recurse=R)); H and W must be multiples of 2**(num_scales + R); every stream of the
        batch is still coded in one range-coder launch.  `out`, if given, must come from forward(auto_recurse=R).
        seek = K (reference layout only, DESIGN §4.13): the range coder also records every stream's state every K
        symbols (l3c_ac_encode_streams_seek; the containers are the same bytes) and finish() returns a seek index per
        container in info['seeks'].  ValueError with tile= and for a K that is not a multiple of 32 in [32, 2^24]."""
        assert imgs_u8.dtype == torch.uint8 and imgs_u8.dim() == 4 and imgs_u8.shape[1] == 3
        if seek is not None:
            if tile is not None:
                raise ValueError('seek indexes are for the reference layout; tiled containers (tile=%s) decode their '
                                 'tiles in parallel already' % (tuple(tile),))
            seek = _seek.check_every(seek)
        recursive = self.check_recursive(recursive)
        dev = imgs_u8.device
        N, _, Hb, Wb = imgs_u8.shape
        check_plane(Hb, Wb, 'encode')
        if recursive:
            fac = 2 ** (self.net.scales + recursive)
            if Hb % fac or Wb % fac:
                raise ValueError('recursive=%d needs H and W divisible by %d, got %dx%d' % (recursive, fac, Hb, Wb))
        ext = self._ragged_extents(extents, N, Hb, Wb, tile)
        if len(pad_tuple) and isinstance(pad_tuple[0], (tuple, list)):
            pads = [tuple(int(v) for v in p) for p in pad_tuple]
            if len(pads) != N:
                raise ValueError('%d padding tuples for a batch of %d images' % (len(pads), N))
        else:
            pads = [tuple(int(v) for v in pad_tuple)] * N
        if tile is not None:
            tile = (int(tile[0]), int(tile[1]))
        if self.encode_banded(imgs_u8.shape, tile, ext, out):
            return self._encode_banded(imgs_u8, pads, tile, recursive)
        if out is None:
            # f16 mode: DMLL head fused into the convs
            out = self.net(imgs_u8, recursive, intervals_of=self.blueprint.losses, extents=ext)
        elif recursive and len(out.S_u8) != self.net.scales + recursive + 1:
            raise ValueError('the network output has %d scales, recursive=%d needs %d'
                             % (len(out.S_u8), recursive, self.net.scales + recursive + 1))

        # ---- per-symbol intervals, scale by scale (coarse -> fine = container order), as stream planes
        shapes, shapes_of, ivs = [], [[] for _ in range(N)], []
        for (scale, C, H, W), iv in self._scale_intervals(out, dev, recursive):
            f = Hb // H
            es = [(H, W)] * N if ext is None else [(h // f, w // f) for (h, w) in ext]
            if ext is not None:
                iv = E.ragged_pack(iv, C, H, W, E._to_device_async(np.asarray(es, np.int32), dev),
                                   max(h * w for (h, w) in es), True)
            elif tile is not None:
                # intervals are produced in raster order; the streams of a tiled container read them tile by tile
                iv = E.reorder_tiles(iv, H, W, tile, True)
            shapes.append((scale, C, H, W))
            ivs.append(iv)
            for sh, (h, w) in zip(shapes_of, es):
                sh.append((scale, C, h, w))

        # ---- one range-coder launch for all streams, each with its own slot
        si, elem, n_sym, _ = stream_layout([[s[1:] for s in sh] for sh in shapes_of], tile)
        bases = np.array([iv.data_ptr() for iv in ivs], np.int64)
        caps, slots, desc = _enc_descs(bases[si] + elem * 4, n_sym, dev)
        if seek is None:
            desc_dev, lens_dev = E.ac_encode_streams(desc, dev)
            return EncodeJob(self, shapes, shapes_of, pads, tile, out, caps, desc_dev, lens_dev, (imgs_u8, ivs, slots))
        counts = _seek.point_counts(desc['n_sym'], seek)
        points = torch.empty(max(1, int(counts.sum())), 4, dtype=torch.int32, device=dev)
        desc_dev, lens_dev, ptrs = E.ac_encode_streams_seek(desc, dev, seek, points,
                                                            np.cumsum(counts) - counts)
        job = EncodeJob(self, shapes, shapes_of, pads, tile, out, caps, desc_dev, lens_dev,
                        (imgs_u8, ivs, slots, ptrs))
        job.seek = (seek, counts, points[:int(counts.sum())])
        return job

    @staticmethod
    def encode_banded(shape, tile, extents=None, out=None):
        """Whether encode_begin encodes a batch of this shape (N, 3, H, W) in bands (DESIGN §4.10): a tiled,
        equal-size batch (extents None) without a precomputed `out` whose image planes exceed
        TILED_ENCODE_BAND_PIXELS (the image is the largest scale)."""
        N, _, H, W = (int(v) for v in shape)
        return tile is not None and extents is None and out is None and N * H * W > TILED_ENCODE_BAND_PIXELS

    def _encode_banded(self, imgs, pads, tile, recursive):
        """encode_begin of a large tiled batch in bands (DESIGN §4.10), same containers as the whole-image encode.
        Encoder phase (_encode_windows): every scale's encoder runs band by band on its window of the whole input
        (region.plan_encoder_bands), each band writing its rows of the whole planes.  Coding phase (_code_rects): the
        uniform-prior scale whole, then the bands of tile rows of the banded decode (region.plan_bands); the intervals
        of every piece go to one scratch buffer and one range-coder launch codes the piece's streams.  All launches
        share one slot buffer and one descriptor array, in launch order; the lengths are put back in container order
        for EncodeJob."""
        from .region import EncoderGeometry, ScalePlan, plan_bands, plan_encoder_bands, rect_streams
        dev, net = imgs.device, self.net
        N, _, Hb, Wb = imgs.shape
        budget = TILED_ENCODE_BAND_PIXELS
        if net._rgb:
            enc = [((0, 0), imgs, None)]
            for s in list(range(net.scales)) + [-1] * recursive:        # the bicubic x0.5 runs whole
                eo = net.nets[s].enc(enc[-1][1])
                enc.append(((0, 0), eo.S, eo.bn_q))
        else:
            geo, walk = EncoderGeometry(net), []
            for s in range(net.scales):
                H, W = Hb >> s, Wb >> s
                bands = plan_encoder_bands(geo, s, H, max(1, budget // (2 * N * W)))
                walk.append(((0, 0, H // 2, W // 2),
                             [((b.window[0], 0, b.window[1], W), (b.rows[0], 0, b.rows[1], W // 2)) for b in bands]))
            enc = self._encode_windows(imgs, (0, 0), walk)

        # ---- coding phase: the pieces of every scale, their streams and the descriptors in launch order
        scales = list(self.iter_scale_dmll(recursive))
        shapes = [(scale,) + tuple(enc[scale][1].shape[1:]) for (scale, _, _) in scales]
        layout = stream_layout([[sh[1:] for sh in shapes]] * N, tile)
        rects = []
        for idx, ((scale, C, H, W), (_, _, uniform)) in enumerate(zip(shapes, scales)):
            if uniform:
                whole = ScalePlan(idx=idx, scale=scale, C=C, H=H, W=W, rect=(0, 0, H, W),
                                  tiles=list(range(len(tile_grid(H, W, tile)))), window=None, out=None, fused=False)
                rects.append((None, [(whole, None)]))
            else:
                bands = plan_bands([sh[1:] for sh in shapes], tile, self._geometry(), idx,
                                   max(1, budget // (N * tile[0] * W)))
                rects.append(((0, 0, H, W), [(b, b.rect) for b in bands]))
        streams = [rect_streams(layout, idx, sp) for idx, (_, pieces) in enumerate(rects) for sp, _ in pieces]
        # the intervals of every piece go to one scratch buffer: a piece's range coder reads it before the next piece's
        # interval kernel writes it (one stream)
        scratch = torch.empty(max(int(n.sum()) for _, n, _ in streams), dtype=torch.int32, device=dev)
        ptrs = np.zeros_like(layout[2])
        for cols, _, elem in streams:
            ptrs[:, cols] = scratch.data_ptr() + elem * 4
        caps, slots, desc = _enc_descs(ptrs, layout[2], dev)
        groups = [(np.arange(N)[:, None] * caps.shape[1] + cols[None, :]).reshape(-1) for cols, _, _ in streams]
        order = np.concatenate(groups)
        desc_l = E._desc_to_device(desc[order], dev)
        desc_c = E._desc_to_device(desc, dev)
        lens_l = torch.empty(order.size, dtype=torch.int32, device=dev)
        first = 0
        for _, group in zip(self._code_rects(rects, enc, tile, scratch, fuse=True), groups):
            E.ac_encode_slice(desc_l, lens_l, first, group.size)
            first += group.size
        inv = np.empty_like(order)
        inv[order] = np.arange(order.size)
        lens_c = lens_l[E._to_device_async(inv, dev)]
        return EncodeJob(self, shapes, [list(shapes) for _ in range(N)], pads, tile, None, caps, desc_c, lens_c,
                         (imgs, enc, scratch, slots, desc_l, lens_l))

    def _encode_windows(self, img, at, walk):
        """The encoder of every trained scale of an L3C network, fine to coarse, on windows of its input (the banded
        encode and region updates, DESIGN §4.10 and §4.12).  img: the pixels uint8 [N][3][h][w], whose element (0, 0)
        sits at `at` of the image plane.  walk: per trained scale s, (D, [(A, K)]): the rectangle D (y0, x0, y1, x1) of
        the scale-(s+1) planes produced and the pieces written into it (_put), each the input rectangle A of scale s
        (even origin) the head and encoder run on and the rectangle K of their output that goes to D.
        -> [(origin, symbols [N][C][h][w], bottleneck values NHWC)] by scale: scale 0 the pixels (values None), every
        other scale its D."""
        net = self.net
        out = [(at, img, None)]
        x = img                               # scale-s input: the image, then the operand heads[s] reads of F_s
        for s, (D, pieces) in enumerate(walk):
            S = bq = F = None
            for A, K in pieces:
                inp = _crop(x, at, A, nhwc=s > 0)
                if s == 0:
                    inp = net._rgb_head_input(inp)
                    hd = inp if isinstance(inp, E.Act) else net.heads[0](inp)
                else:
                    hd = net.heads[s](self._operand_act(inp))
                eo = net.nets[s].enc(hd)
                o = (A[0] // 2, A[1] // 2)
                S = _put(S, D, K, eo.S, o, nhwc=False)
                bq = _put(bq, D, K, eo.bn_q, o, nhwc=True)
                if s + 1 < net.scales:                  # F_{s+1} feeds heads[s + 1]: keep what that conv reads
                    F = _put(F, D, K, eo.F.r if E.tensor_core_mode() else eo.F.f, o, nhwc=True)
                del eo, hd, inp
            out.append((D[:2], S, bq))
            x, at = F, D[:2]
        return out

    def _code_rects(self, rects, enc, tile, out=None, fuse=False):
        """The coding phase of an encode on windows (the banded encode and region updates, DESIGN §4.10 and §4.12),
        coarse to fine.  rects: per scale walked (iter_scale_dmll), (D, [(sp, K)]): the tile-aligned rectangles sp
        (region.ScalePlan) coded and, where the next finer scale adds this scale's decoder features, the rectangle D
        they are assembled in and the rectangle K of each piece's that goes there (_band_window).  enc: by scale, as
        _encode_windows returns.  Per rectangle the decoder network runs on its window of the coarser scale and the
        intervals of its symbols go, in its own tile order, to `out` (an int32 buffer every rectangle reuses; None: a
        new tensor each).  fuse: in f16 a band's intervals come from the classifier's 1x1 conv fused with the interval
        kernel, where that kernel is built (lin_dmll_intervals_band).
        Yields (idx, sp, intervals int32 [N][C][h * w]) once a rectangle's intervals are queued."""
        net, K = self.net, self.net.config_ms.prob.K
        F = None                              # (origin, features) the next finer decoder adds
        for idx, ((scale, dmll, uniform), (D, pieces)) in enumerate(
                zip(self.iter_scale_dmll(len(rects) - 1 - net.scales), rects)):
            o, S, _ = enc[scale]
            dev, dst = S.device, None
            for sp, Kr in pieces:
                r, C = sp.rect, sp.C
                h, w = r[2] - r[0], r[3] - r[1]
                ivb = None if out is None else out[:S.shape[0] * C * h * w]
                if uniform:
                    sym = S if r == (0, 0, sp.H, sp.W) else _crop(S, o, r, nhwc=False)
                    iv = E.reorder_tiles(E.lut_intervals(sym, self._uniform(dmll.L, dev)[0]), h, w, tile, True, out=ivb)
                    yield idx, sp, iv
                    continue
                bn8, keep = (enc[scale + 1][0], enc[scale + 1][2]), (D, Kr, dst)
                if fuse and E.f16_mode() and net.prob_clfs[min(scale, net.scales - 1)].atrous.lin.in_channels % 64 == 0 \
                        and C == (3 if dmll.rgb_scale else 5):
                    iv, dst = self._band_window(sp, bn8, F, keep, fused=(S, dmll, (sp.out[0], r[0], h, tile, ivb)))
                else:
                    l, dst = self._band_window(sp, bn8, F, keep)
                    iv = E.dmll_intervals_rect(l, sp.out[0], sp.out[1], S, (r[0] - o[0], r[1] - o[1], h, w),
                                               dmll.targets(dev), C, K, dmll.L, dmll.rgb_scale, tile, origin=o,
                                               plane=(sp.H, sp.W), out=ivb)
                    del l
                yield idx, sp, iv
            F = None if dst is None else (D[:2], dst)

    @staticmethod
    def _operand_act(op):
        """The engine.Act through which a conv reads the cropped operand `op` of an activation (fp32 in fp32, the TF32
        twin in tf32, the FP16 or split image in f16 / f16x2): what the conv reads of the whole activation."""
        if not E.tensor_core_mode():
            return E.Act(op)
        if E.f16_mode() or E.f16x2_mode():
            return E.Act(None, op)
        return E.Act(op, op)

    def _band_window(self, sp, bn8, F, keep, fused=None):
        """The decoder network of one tile-aligned rectangle sp (region.ScalePlan: a band of region.plan_bands, an
        update's R_s) run on its window sp.window of the coarser scale, for the banded decode and _code_rects.
        bn8 = (origin, symbol values NHWC) and F = (origin, decoder features NHWC or their engine.Act) are planes of the
        coarser scale whose element (0, 0) sits at origin; the window is cut out of both (of F where dec.skip adds them).
        keep = (D, K, dst): where the next finer scale adds this decoder's features, their rectangle K goes to the
        destination dst of rectangle D (_put).  fused: get_P_nhwc's.
        -> (get_P_nhwc's first result, the destination, or None where the finer scale adds no features)."""
        win = _crop(bn8[1], bn8[0], sp.window, nhwc=True)
        Fw = None
        if self.net.fuses(sp.scale):
            Fw = _crop(F[1] if torch.is_tensor(F[1]) else F[1].f, F[0], sp.window, nhwc=True)
        l, Fo = self.net.get_P_nhwc(sp.scale, win, Fw, fused=fused)
        if sp.scale < 1 or not self.net.fuses(sp.scale - 1):
            return l, None
        D, K, dst = keep
        return l, _put(dst, D, K, Fo.f, (2 * sp.window[0], 2 * sp.window[1]), nhwc=True)

    def _scale_intervals(self, out, dev, recursive=0):
        """Coding intervals of every scale, coarse -> fine: [(shape (scale, C, H, W), int32 [N][C][H*W])]."""
        K = self.net.config_ms.prob.K
        res = []
        for scale, dmll, uniform in self.iter_scale_dmll(recursive):
            S = out.S_u8[scale]
            _, C, H, W = S.shape
            if uniform:
                iv = E.lut_intervals(S, self._uniform(dmll.L, dev)[0])
            elif out.IV is not None and out.IV[scale] is not None:
                iv = out.IV[scale]                                           # produced by the fused head
            else:
                l = out.P_nhwc[scale]
                assert non_shared_get_K(l.shape[-1], C) == K
                iv = E.dmll_intervals(l, S, dmll.targets(dev), C, K, dmll.L, dmll.rgb_scale)
            res.append(((scale, C, H, W), iv))
        return res

    # ------------------------------------------------------------------------------------------
    @_on_device
    def decode_batch(self, datas, to_host=True, lane=None, seeks=None):
        """datas: list of container byte strings of equally shaped images -- or, where ragged batches are supported
        (ragged_unsupported), of any mix of shapes: image n then is the top-left H_n x W_n of the result (the
        finest scale of its container), zero elsewhere.
        seeks: one seek index (sidecar bytes, seek.parse_index) or None per container: containers with one decode
        every stream as parallel segments (decode_device), the others serially; the same result either way.
        Returns (uint8 [N,3,H,W] incl. padding, pad_tuple list)."""
        dev = self.blueprint.device
        N = len(datas)
        if seeks is not None:
            if len(seeks) != N:
                raise ValueError('%d seek indexes for %d containers' % (len(seeks), N))
            seeks = [None if sk is None else _seek.parse_index(sk, dta) for sk, dta in zip(seeks, datas)]
        parsed = [parse_container(d) for d in datas]
        tile = container_tile(datas[0])
        shapes_of = [[(C, H, W) for (C, H, W, _) in p[1]] for p in parsed]
        if any(container_tile(dta) != tile for dta in datas) or \
                (any(sh != shapes_of[0] for sh in shapes_of) and self.ragged_unsupported(tile) is not None):
            raise ValueError('decode_batch needs containers of identical shape')
        if any(len(sh) != len(shapes_of[0]) for sh in shapes_of):
            raise ValueError('decode_batch: containers with different numbers of scales')
        for sh in {tuple(sh): sh for sh in shapes_of}.values():
            self._check_shapes(sh)                  # before the upload: nothing is sized from a header it refuses
        blob, starts = _upload(datas, dev)
        offs = np.array([[starts[n] + o for (_, _, _, st) in parsed[n][1] for (o, _) in st] for n in range(N)],
                        np.int64)
        lens = np.array([[ln for (_, _, _, st) in parsed[n][1] for (_, ln) in st] for n in range(N)], np.int64)
        S = self.decode_device(blob, offs, lens, shapes_of, lane=lane, tile=tile, seeks=seeks)
        pads = [p[0] for p in parsed]
        if to_host:
            return S.cpu(), pads
        return S, pads

    @_on_device
    def seek_index(self, datas, every=_seek.DEFAULT_EVERY, lane=None):
        """Seek indexes (sidecar bytes, DESIGN §4.13) of reference-layout containers, e.g. ones the reference or an
        earlier encode wrote: one serial decode of the batch (containers as decode_batch takes them) in launches of
        `every` symbols, the decoders' saved states copied aside on the device after each.  The same bytes as
        encode_begin(..., seek=every) writes for the same containers.  ValueError for a tiled container or an
        interval that is not a multiple of 32 in [32, 2^24]."""
        every = _seek.check_every(every)
        n_sym = [_seek.stream_symbols(dta) for dta in datas]
        dev = self.blueprint.device
        N = len(datas)
        parsed = [parse_container(d) for d in datas]
        shapes_of = [[(C, H, W) for (C, H, W, _) in p[1]] for p in parsed]
        if any(sh != shapes_of[0] for sh in shapes_of) and self.ragged_unsupported() is not None:
            raise ValueError('seek_index needs containers of identical shape')
        if any(len(sh) != len(shapes_of[0]) for sh in shapes_of):
            raise ValueError('seek_index: containers with different numbers of scales')
        for sh in {tuple(sh): sh for sh in shapes_of}.values():
            self._check_shapes(sh)
        blob, starts = _upload(datas, dev)
        offs = np.array([[starts[n] + o for (_, _, _, st) in parsed[n][1] for (o, _) in st] for n in range(N)],
                        np.int64)
        lens = np.array([[ln for (_, _, _, st) in parsed[n][1] for (_, ln) in st] for n in range(N)], np.int64)
        rec = _StateRecorder(blob, offs, np.stack(n_sym), every)
        self.decode_device(blob, offs, lens, shapes_of, lane=lane, _streams=rec.decode)
        words = rec.points.cpu().numpy().view(np.uint32).astype(np.int64)
        # the saved state (l3c_dec_stream_t.state) -> (low, high, flip, bits)
        pt_stream = np.repeat(np.arange(N * offs.shape[1]), rec.counts)
        pt_len = lens.reshape(-1)[pt_stream]
        long_ = pt_len >= (1 << 28)
        past = (words[:, 0] >> 31) & 1
        bits = words[:, 3] | (np.where(long_, words[:, 4], past) << 32)
        low = words[:, 0] & 0x7FFFFFFF
        host = np.zeros(int(starts[-1]) + len(datas[-1]) if N else 0, np.uint8)
        for n, dta in enumerate(datas):
            host[starts[n]:starts[n] + len(dta)] = np.frombuffer(dta, np.uint8)
        flip = (words[:, 2] ^ _seek.code_windows(host, offs.reshape(-1)[pt_stream], pt_len, bits)) & 0x80000000
        out, P = [], offs.shape[1]
        for n in range(N):
            cnt = rec.counts[n * P:(n + 1) * P]
            a, b = rec.first[n * P], rec.first[n * P] + cnt.sum()
            out.append(_seek.write_index(datas[n], every, cnt, low[a:b], words[a:b, 1], flip[a:b], bits[a:b]))
        return out

    def _decode_rgb_pipelined(self, l, S, tg, C, K, L, table, d, dev, n_chunks=None, lane=None, coarse=False):
        """RGB scale: channel c's means depend on the decoded channels < c at the same pixel
        (logistic_mixture.py:262-272), so the reference codes R, G, B strictly one after the other.
        Here the three serial decoders run concurrently, staggered by one chunk of pixels: as soon as
        chunk j of channel c-1 is decoded, the CDF rows of chunk j of channel c are built (on the SM
        group the decoders do not own, _rgb_streams) and channel c's warps continue -- coder state is
        carried across launches.  Serial depth drops from 3*HW to (1 + 2/n_chunks)*HW symbols (whole
        decode at 16x512^2 with 32 / 64 / 128 chunks: 120.5 / 118.7 / 117.7 ms when measured).
        coarse: `table` and the descriptors hold coarse records (E.COARSE_PITCH) instead of full rows."""
        N, HW = S.shape[0], S.shape[2] * S.shape[3]
        if n_chunks is None:
            n_chunks = int(os.environ.get('L3C_RGB_CHUNKS', 64))
        csz = max(2048, -(-HW // n_chunks))
        csz = -(-csz // 64) * 64
        state = torch.zeros(N * C * _lib.DEC_STATE_WORDS, dtype=torch.int32, device=dev)
        d['state'][:] = state.data_ptr() + 4 * _lib.DEC_STATE_WORDS * (np.arange(N)[:, None] * C + np.arange(C)[None, :])
        descs = [E._desc_to_device(np.ascontiguousarray(d[:, c]), dev) for c in range(C)]
        cur = torch.cuda.current_stream()
        if lane is None:
            lane = self.lanes(dev, N * C, 1)[0][0]
        # the chunk loop itself (2 x 3 x n_chunks launches + as many event records / waits) runs inside the library
        E.decode_rgb_pipelined(l, S, tg, K, L, table, descs, csz, cur, lane.bld, lane.dec, coarse=coarse)

    def encode_stream(self, dev, n_decoders, n_lanes=1):
        """A stream for encodes that run beside decodes (EncodeJob pipelining): confined to the SM group of
        the row builders, so that its persistent conv kernels never sit on the decoders' SMs."""
        return self.lanes(dev, n_decoders, n_lanes)[1]

    def lanes(self, dev, n_decoders, n_lanes=1):
        """-> ([DecodeLane] * n_lanes, encode stream).  A DecodeLane is the set of streams ONE decode in flight
        uses: `main` (decoder networks, CDF rows of the bottleneck scales), `bld[3]` (CDF-row builders of the
        R, G, B channels), `dec[3]` (the range decoders).  The `dec` streams of all lanes own a group of SMs
        (driver green contexts, l3c_partition_streams) sized for `L3C_DEC_WARPS_PER_SM` decoder-kernel warps
        per SM (default 4 for one lane = one latency-bound warp per SM sub-partition, 8 for two or three lanes,
        16 from four lanes on; a
        decoder warp that shares its scheduler with throughput-bound warps runs ~1.5x slower); everything else -- including the encode
        stream, which has the lowest priority -- runs on the remaining SMs.  Several lanes = several batches
        being decoded side by side: the decode of ONE batch is bound by the serial chain of its range coder
        and keeps only ~1/6 of the GPU busy.  L3C_SM_PARTITION=0, a driver without green contexts or an
        attached profiler give ordinary streams (slower, same bytes)."""
        key = (str(dev), n_decoders, n_lanes)
        cache = self._lane_cache
        if key not in cache:
            part = None
            # encode streams: an encode is a throughput phase (the networks) followed by a latency-bound one (the
            # range encoders, a coding warp and an emitter warp per stream); encodes on the same stream run one
            # after the other
            n_enc = max(1, int(os.environ.get('L3C_ENC_STREAMS', 2)))
            want_part = os.environ.get('L3C_SM_PARTITION', '1') != '0'
            if want_part and _under_injection_tool() and 'L3C_SM_PARTITION' not in os.environ:
                # Nsight Compute cannot profile kernels launched into green-context streams (it lost the
                # process at the first one): under a CUDA injection tool use ordinary streams
                import sys
                print('l3c_pytorch_b200: profiler injection detected, SM partitions off '
                      '(set L3C_SM_PARTITION=1 to force them)', file=sys.stderr)
                want_part = False
            if want_part:
                n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
                # one lane: 4 warps per SM (lowest latency); several lanes: 8, from four lanes on 16 (measured at
                # 16 x 512^2: 3 lanes on 36 / 48 / 72 SMs -> 86 / 69 / 63 Mpx/s, 4 lanes on 32 / 48 SMs -> 89 / 80: what
                # the decoders' group takes is lost to the throughput work; 4 lanes with the coarse RGB decoder, 12 vs
                # 16 warps = 32 vs 24 SMs: 69.2 - 71.6 vs 72.8 - 74.3 Mpx/s, DESIGN §7)
                wps = int(os.environ.get('L3C_DEC_WARPS_PER_SM', 4 if n_lanes == 1 else (8 if n_lanes <= 3 else 16)))
                # every stream = decoder warp + helper warp (measured at 16 x 512^2, one lane, 4 warps per SM:
                # 48 / 24 / 16 SMs -> decode 95 / 86 / 93 ms)
                want = -(-(2 * n_decoders * n_lanes) // (8 * wps)) * 8
                want = min(max(8, want), (n_sm // 16) * 8)
                want = int(os.environ.get('L3C_DEC_SMS', want))           # bring-up knob
                part = E.partition_streams2(dev, want, 3 * n_lanes, 4 * n_lanes, n_enc)
            lanes = []
            for i in range(n_lanes):
                ln = DecodeLane()
                if part is not None:
                    a, b = part[0], part[1]
                    ln.dec = a[3 * i:3 * i + 3]
                    ln.main = b[4 * i]
                    ln.bld = b[4 * i + 1:4 * i + 4]
                    ln.partitioned = True
                else:
                    ln.dec = [torch.cuda.Stream(device=dev, priority=-1) for _ in range(3)]
                    ln.bld = [torch.cuda.Stream(device=dev, priority=-1) for _ in range(3)]
                    ln.main = torch.cuda.Stream(device=dev, priority=-1)
                    ln.partitioned = False
                lanes.append(ln)
            # two encode streams (default priority): the range-encoder launch of one batch is latency-bound (~11 ms
            # for an RGB plane of 512 x 512, DESIGN §7) and overlaps the convs of the next batch when they alternate
            encs = part[2] if part is not None else [torch.cuda.Stream(device=dev) for _ in range(n_enc)]
            cache[key] = (lanes, encs[0], encs)
        return cache[key]

    def encode_streams(self, dev, n_decoders, n_lanes=1):
        """The two default-priority streams for encodes that run beside decodes (alternate between them)."""
        return self.lanes(dev, n_decoders, n_lanes)[2]

    def _on_decoder_stream(self, lane, fn):
        """Run the launches of `fn` on the lane's first decoder stream (the decoders' SM group), ordered
        after what the current stream has queued and before what it queues next."""
        if lane is None or not lane.partitioned:
            return fn()
        cur = torch.cuda.current_stream()
        ev = torch.cuda.Event()
        ev.record(cur)
        with torch.cuda.stream(lane.dec[0]):
            lane.dec[0].wait_event(ev)
            out = fn()
            done = torch.cuda.Event()
            done.record(lane.dec[0])
        cur.wait_event(done)
        return out

    def _stream_descs(self, blob, offs, lens, n_sym, elem, Sp, table, pitch):
        """Range-decoder descriptors of the streams of one scale, or of one band of it (offs / lens / n_sym / elem int64
        [N][C * T], channel-major): every stream reads its bytes in place in `blob`, writes its symbols to its elements
        of the stream planes Sp [N][C][plane] and finds its CDF rows at the same elements of `table` (int16, `pitch`
        entries per symbol; pitch 0: the one row of a uniform prior).  -> (desc [N * C * T], its [N][C][T] view)."""
        N, C = Sp.shape[:2]
        T = n_sym.shape[1] // C
        desc = np.zeros(N * C * T, dtype=_lib.DEC_STREAM_DTYPE)
        d = desc.reshape(N, C, T)
        d['in'][:] = (blob.data_ptr() + offs).reshape(N, C, T)
        d['in_len'][:] = lens.reshape(N, C, T)
        d['n_sym'][:] = n_sym.reshape(N, C, T)
        d['sym_out'][:] = (Sp.data_ptr() + elem).reshape(N, C, T)
        d['table'][:] = (table.data_ptr() + elem * (pitch * 2)).reshape(N, C, T)
        d['row_pitch'][:] = pitch
        return desc, d

    def _decode_scales(self, blob, offs, lens, layout, channels, recursive, lane, network, rows, raster,
                       symbols=lambda idx, S: S, features=lambda idx, F: F,
                       row_pitch=lambda dmll: E.table_pitch(dmll.L), bands=lambda idx: None, streams=None,
                       zero=False):
        """The coarse-to-fine walk of every decode: full decodes of equal-size, tiled and ragged batches
        (decode_device) and region passes (decode_region_pass).  blob: the uploaded containers; offs / lens int64
        [N][streams per image] in the order of the stream_layout `layout`, where every stream reads its bytes in place;
        channels: C of every scale walked, coarse -> fine (a region at level k stops early); recursive: as in
        iter_scale_dmll; lane: as in decode_device.  -> the raster planes of the last scale.
        Every scale decodes into stream planes Sp [N][C][plane], where its CDF rows are built too, and then goes back
        to the raster planes the network of the next scale reads:
          * the uniform-prior scale is one range-decoder launch on the lane's decoder stream;
          * any other scale runs its decoder network, checks the output against the container, lays out the row
            table and runs the channel steps: on an RGB scale channel c's means depend on the decoded channels < c
            of the same pixel, so R, G, B go one after the other -- the rows of c, then one launch decoding every
            stream of c -- while a bottleneck scale builds all rows and decodes every stream in one launch;
          * the symbols become raster planes, and the next scale gets their values and this scale's features.
        What differs between the passes is geometry, asked of the caller's hooks with the scale's index idx:
          network(idx, scale, bn8, F) -> (l, F, (H, W)): get_P_nhwc on the coarser scale's values bn8 and features F,
            and the height and width its output l must have;
          row_pitch(dmll) -> entries per row of the table (full rows unless the caller's `rows` reads coarse records);
          rows(idx, dmll, l, Sp, table, d, steps): code the scale -- steps(build) runs the channel steps above with
            build(c) building the rows of channel c (of every channel for c = -1) -- or decode it some other way
            from the [N][C][T] descriptors d;
          raster(idx, Sp) -> S [N][C][H][W]; symbols(idx, S), features(idx, F) -> what of them the next network reads
            (all of it by default);
          streams(dmll, desc, coarse) -> None: decodes the streams of the descriptors desc in place of one
            l3c_ac_decode_streams launch (seek-indexed decodes, DESIGN §4.13); coarse: the tables hold coarse records;
          zero: the stream planes start zeroed (a region pass over bands leaves the symbols before a seek point
            undecoded);
          bands(idx) -> None, or the bands (region.plan_bands) the scale is decoded in (DESIGN §4.10): then per band
            network(..., band) runs on the band's window of the whole coarser scale, rows(..., band) builds the band's
            rows into a table of the band's own stream planes, the band's streams decode into those planes and their
            symbols are copied to their elements of Sp; the F the walk hands on is what network returned for the last
            band."""
        dev = blob.device
        N = offs.shape[0]
        K = self.net.config_ms.prob.K
        bn8, F, S = None, None, None
        self._mark('start')
        for idx, ((scale, dmll, uniform), C) in enumerate(zip(self.iter_scale_dmll(recursive), channels)):
            Sp = (torch.zeros if zero else torch.empty)(N, C, int(layout[3][idx]), dtype=torch.uint8,
                                                        device=dev)                        # symbols in stream order

            def decode(dsc):
                if streams is not None:
                    coarse = not uniform and row_pitch(dmll) == E.COARSE_PITCH
                    return self._on_decoder_stream(lane, lambda: streams(dmll, dsc, coarse))
                self._on_decoder_stream(lane, lambda: E.ac_decode_streams(dsc, dev, dmll.L))

            def steps(build):
                if dmll.rgb_scale:
                    for c in range(C):
                        build(c)
                        decode(np.ascontiguousarray(d[:, c, :]).reshape(-1))
                else:
                    build(-1)
                    decode(desc)

            def run_net(F_in, *band):
                l, F_out, want = network(idx, scale, bn8, F_in, *band)
                if tuple(l.shape[1:3]) != want or non_shared_get_K(l.shape[-1], C) != K:
                    raise ValueError('container scale %d (%dx%dx%d) does not match the model output %s'
                                     % (scale, C, want[0], want[1], tuple(l.shape)))
                return l, F_out

            band_list = None if uniform else bands(idx)
            cols = slice(*np.searchsorted(layout[0][0], [idx, idx + 1]))          # the scale's streams
            if uniform:
                table, pitch = self._uniform(dmll.L, dev)[1], 0
                desc, d = self._stream_descs(blob, offs[:, cols], lens[:, cols], layout[2][:, cols], layout[1][:, cols],
                                             Sp, table, pitch)
                decode(desc)
            elif band_list is None:
                l, F = run_net(F)
                self._mark(('rnet%d' if scale >= self.net.scales else 'net%d') % scale)
                pitch = row_pitch(dmll)
                table = torch.empty(Sp.numel() * pitch, dtype=torch.int16, device=dev)
                desc, d = self._stream_descs(blob, offs[:, cols], lens[:, cols], layout[2][:, cols], layout[1][:, cols],
                                             Sp, table, pitch)
                rows(idx, dmll, l, Sp, table, d, steps)
            else:
                # banded (DESIGN §4.10): per band its network window, its rows and its streams; only one band's
                # parameters and rows are alive at a time, and its symbols go to their elements of Sp
                from .region import rect_streams
                pitch, F_in = row_pitch(dmll), F
                for band in band_list:
                    l, F = run_net(F_in, band)
                    b_cols, n_sym, elem = rect_streams(layout, idx, band)
                    e0, e1 = band.rect[0] * band.W, band.rect[2] * band.W
                    Sb = torch.empty(N, C, e1 - e0, dtype=torch.uint8, device=dev)
                    table = torch.empty(Sb.numel() * pitch, dtype=torch.int16, device=dev)
                    desc, d = self._stream_descs(blob, offs[:, b_cols], lens[:, b_cols], n_sym, elem, Sb, table, pitch)
                    rows(idx, dmll, l, Sb, table, d, steps, band)
                    Sp[:, :, e0:e1].copy_(Sb)
                    del l, table
                self._mark(('rnet%d' if scale >= self.net.scales else 'net%d') % scale)
            S = raster(idx, Sp)
            self._mark('uniform' if uniform else ('rgb' if dmll.rgb_scale and scale == 0 else
                                                  ('R%d' if scale >= self.net.scales else 'S%d') % scale))
            if idx + 1 < len(channels):
                bn8 = E.symbols_to_values(symbols(idx, S), self._symbol_values(scale, dmll, dev),
                                          self._rgb_shift(dev))
                F = features(idx, F)
        return S

    @_on_device
    def decode_device(self, blob, offs, lens, shapes, lane=None, tile=None, seeks=None, _streams=None):
        """Decode streams that already sit in HBM: `blob` uint8 device buffer (readable 4 bytes past
        every stream), offs/lens int64 [N][streams per image] in container order (coarse -> fine,
        channel-major), shapes [(C,H,W)] coarse -> fine.  Returns uint8 [N,3,H,W] on the device.
        `lane` (self.lanes()): the stream set of this decode when several decodes are in flight; the caller
        has made `lane.main` the current stream.  Without it the range decoders of the bottleneck scales run
        on the current stream and the RGB scale on lane 0 of a one-lane partition.
        `tile` = (th, tw): the streams are the tiles of a tiled container (ContainerLayout): thousands of short
        streams, so the three RGB channels are simply decoded one after the other, all tiles at once.
        shapes may also be one list per image: a ragged batch (DESIGN §4.6) when they differ; image n then is the
        top-left H_n x W_n of the result, zero elsewhere.
        The scales are walked by _decode_scales; between stream and raster planes lies a view, l3c_reorder_tiles
        (tiled) or l3c_ragged_pack (ragged).
        seeks: one seek.SeekIndex (or None) per image (reference layout only, DESIGN §4.13): every stream of an image
        with an index decodes as segments from its seek points, one l3c_ac_decode_segments launch per bottleneck or
        uniform scale and per RGB channel, whose rows are built whole first.  Images without one decode serially."""
        dev = blob.device
        N = offs.shape[0]
        # _streams: _StateRecorder.decode (seek_index)
        if seeks is not None and any(sk is not None for sk in seeks):
            if tile is not None:
                raise ValueError('seek indexes are for reference-layout containers, not tiled ones')
            _streams = _SegmentDecode(blob, offs, seeks).decode
        if shapes and isinstance(shapes[0][0], (tuple, list)):
            shapes_of = [[tuple(int(v) for v in s) for s in sh] for sh in shapes]
            if len(shapes_of) != N:
                raise ValueError('%d shape lists for %d images' % (len(shapes_of), N))
        else:
            shapes_of = [[tuple(int(v) for v in s) for s in shapes]] * N
        ragged = any(sh != shapes_of[0] for sh in shapes_of)
        if ragged:
            why = self.ragged_unsupported(tile)
            if why is not None:
                raise NotImplementedError(why)
        # every distinct shape list once; R (recursive scales) is what the scale count says beyond the model's own
        Rs = {self._check_shapes(sh) for sh in {tuple(sh): sh for sh in shapes_of}.values()}
        if len(Rs) != 1:
            raise ValueError('containers with different numbers of scales in one batch')
        if tile is not None:
            tile = (int(tile[0]), int(tile[1]))
        fin = [sh[-1][1:] for sh in shapes_of] if ragged else None      # extents at the finest scale
        K = self.net.config_ms.prob.K
        # per scale: H, W of the batch's raster planes and (ragged) every image's extent on the device, uploaded once
        dims = [tuple(max(sh[idx][k] for sh in shapes_of) for k in (1, 2)) for idx in range(len(shapes_of[0]))]
        ext_dev = functools.lru_cache(None)(
            lambda idx: E._to_device_async(np.array([sh[idx][1:] for sh in shapes_of], np.int32), dev))

        def coarse(dmll):
            # the RGB scale of an equal-size batch in f16 mode decodes from coarse records (parameters + every 8th
            # CDF entry, 192 instead of 512 B per sub-pixel; the decoder evaluates the bracketed entries itself);
            # tiled and ragged batches, the bottleneck scales, L < 256 and the other precision modes build full rows
            return dmll.rgb_scale and tile is None and not ragged and dmll.L == 256 and K == 10 and E.f16_mode()

        def bands(idx):
            # an equal-size tiled pass whose plane at this scale exceeds the budget: bands of whole tile rows
            H, W = dims[idx]
            if tile is None or ragged or N * H * W <= TILED_BAND_PIXELS:
                return None
            from .region import plan_bands
            return plan_bands(shapes_of[0], tile, self._geometry(), idx, max(1, TILED_BAND_PIXELS // (N * tile[0] * W)))

        whole_F = [None]                  # the features of the scale being banded, assembled band by band

        def network(idx, scale, bn8, F, band=None):
            if band is not None:
                # the features of the next finer scale are assembled in one whole plane, band by band
                keep = ((0, 0) + dims[idx], band.rect, whole_F[0] if band.rect[0] else None)
                l, whole_F[0] = self._band_window(band, ((0, 0), bn8), ((0, 0), F), keep)
                return l, whole_F[0], (2 * (band.window[2] - band.window[0]), 2 * bn8.shape[2])
            if ragged:
                ext_dev(idx)                      # queued ahead of the network: the rows and the raster step read it
            l, F = self.net.get_P_nhwc(scale, bn8, F if self.net.fuses(scale) else None, extents=fin)
            return l, F, dims[idx]

        def rows(idx, dmll, l, Sp, table, d, steps, band=None):
            C, plane, (H, W) = Sp.shape[1], Sp.shape[2], dims[idx]
            tg = dmll.targets(dev)
            if band is not None:
                (oy, ox), h = band.out[:2], band.rect[2] - band.rect[0]
                return steps(lambda c: E.dmll_build_table_window(l, oy, ox, Sp, tg, C, K, dmll.L, c >= 0, c, table, h,
                                                                 W, tile))
            if tile is not None:
                # every tile of every image at once (N*T streams per launch)
                return steps(lambda c: E.dmll_build_table_tiled(l, Sp, tg, C, K, dmll.L, c >= 0, c, table, tile))
            # per-pixel kernels from here on: the stream planes are an N x 1 x plane "image" each
            if ragged:
                l = E.ragged_pack(l, 1, H, W, ext_dev(idx), plane, True)
            l = l.view(N, 1, plane, l.shape[-1])
            Sv = Sp.view(N, C, 1, plane)
            if dmll.rgb_scale and _streams is not None:
                # every channel's rows whole, then all its segments in one launch (steps)
                if coarse(dmll):
                    steps(lambda c: E.dmll_build_coarse(l, Sv, tg, K, dmll.L, c, table))
                else:
                    steps(lambda c: E.dmll_build_table(l, Sv, tg, C, K, dmll.L, True, c, table))
            elif dmll.rgb_scale:
                self._decode_rgb_pipelined(l, Sv, tg, C, K, dmll.L, table, d.reshape(N, C), dev, lane=lane,
                                           coarse=coarse(dmll))
            else:
                steps(lambda c: E.dmll_build_table(l, Sv, tg, C, K, dmll.L, False, -1, table))

        def raster(idx, Sp):
            C, (H, W) = Sp.shape[1], dims[idx]
            if ragged:
                return E.ragged_pack(Sp, C, H, W, ext_dev(idx), Sp.shape[2], False)    # zero-padded [N][C][H][W]
            if tile is not None:
                return E.reorder_tiles(Sp, H, W, tile, False).view(N, C, H, W)
            return Sp.view(N, C, H, W)

        return self._decode_scales(
            blob, offs, lens, stream_layout(shapes_of, tile), [s[0] for s in shapes_of[0]], Rs.pop(), lane,
            network, rows, raster, row_pitch=lambda dmll: E.COARSE_PITCH if coarse(dmll) else E.table_pitch(dmll.L),
            bands=bands, streams=_streams)

    def _geometry(self):
        """region.DecoderGeometry of this codec's network, built once."""
        if self._geo is None:
            from .region import DecoderGeometry
            self._geo = DecoderGeometry(self.net)
        return self._geo

    # ------------------------------------------------------------------------------------------
    def plan_regions(self, datas, regions, levels=None, seeks=None):
        """Parse, validate and plan (region.plan_region) every (container, region, level) of a decode_regions call,
        before any GPU work: -> ([(pad_tuple, scales)] parsed, [RegionPlan]).  seeks: None, or one seek index
        (sidecar bytes) or None per container; every index is parsed (seek.parse_index) first, and a reference-layout
        container with one is planned in bands (RegionPlan.seek holds its SeekIndex).  ValueError for a
        reference-layout container without an index, a malformed or mismatched index, a container this model cannot
        have written, an empty region or one outside the image, and a level that does not exist."""
        from .region import DecoderGeometry, plan_region
        if len(regions) != len(datas):
            raise ValueError('%d regions for %d containers' % (len(regions), len(datas)))
        levels = [0] * len(datas) if levels is None else list(levels)
        if len(levels) != len(datas):
            raise ValueError('%d levels for %d containers' % (len(levels), len(datas)))
        seeks = [None] * len(datas) if seeks is None else list(seeks)
        if len(seeks) != len(datas):
            raise ValueError('%d seek indexes for %d containers' % (len(seeks), len(datas)))
        indexes = []
        for i, (sk, dta) in enumerate(zip(seeks, datas)):
            try:
                indexes.append(None if sk is None else _seek.parse_index(sk, dta))
            except ValueError as err:
                raise ValueError('seek index %d: %s' % (i, err))
        geo = DecoderGeometry(self.net)
        parsed, plans = [], []
        for i, (dta, reg, lev, sk) in enumerate(zip(datas, regions, levels, indexes)):
            pt, scales = parse_container(dta)
            tile = container_tile(dta)
            if tile is None and sk is None:
                raise ValueError('container %d: region decode needs a tiled container (written with '
                                 'Bitcoding(..., tile=(th, tw))) or the seek index of a reference-layout one '
                                 '(Bitcoding.seek_index, `idx IN.l3c`); the streams of the reference layout are serial'
                                 % i)
            shapes = [(C, H, W) for (C, H, W, _) in scales]
            try:
                self._check_shapes(shapes)
            except ValueError as err:
                raise ValueError('container %d was not written by this model: %s' % (i, err))
            parsed.append((pt, scales))
            plan = plan_region(shapes, pt, tile, geo, reg, lev, every=None if sk is None else sk.every)
            plan.seek = sk
            plans.append(plan)
        return parsed, plans

    @_on_device
    def decode_regions(self, datas, regions, levels=None, lane=None, seeks=None):
        """Decode one region of each container (DESIGN §4.8): -> [uint8 [1, C, h, w] on the device] in input order,
        each equal to the same crop of the full decode (at level k >= 1, of the stored scale-k plane).  Only the tile
        streams and decoder windows the region depends on are decoded.  In f16 and f16x2, pairs whose plans walk
        the same scales with the same tile size (RegionPlan.pass_key) share one ragged pass: one network pass per scale
        on a padded batch of their windows and one range-decoder launch per channel step; pairs of equal
        RegionPlan.shape_key share an equal-shape pass, and in tf32 / fp32 the groups of equal shape_key run one after
        another (region.plan_passes, decode_region_pass; REGION_RAGGED_PASS = False forces that grouping everywhere).
        regions: (y, x, h, w) each; levels: None (all 0) or one int each.
        seeks: None, or one seek index (sidecar bytes) or None per container: a reference-layout container needs one
        and decodes full-width bands, each channel's stream from the seek point before its band (DESIGN §4.13
        "Regions"); its passes never include tiled containers.
        lane: as in decode_batch -- the caller has made `lane.main` current; the range decoders run on the lane's
        decoder streams."""
        parsed, plans = self.plan_regions(datas, regions, levels, seeks)
        blob, starts = _upload(datas, self.blueprint.device)
        self.region_counts = {'streams': 0, 'symbols': 0}          # of this call: every pass adds to them
        return self._decode_planned(blob, starts, [[st for (_, _, _, st) in p[1]] for p in parsed], plans, lane)

    def _decode_planned(self, blob, starts, streams_of, plans, lane=None):
        """The region plans of containers uploaded to blob (container n at starts[n], its streams streams_of[n] as
        parse_container lists them per scale) in passes (region.plan_passes) -> the regions in plan order."""
        from .region import pass_streams, plan_passes
        ragged = REGION_RAGGED_PASS and self.net.windows_unsupported() is None
        outs = [None] * len(plans)
        for idxs, is_ragged in plan_passes(plans, ragged):
            sel = [plans[i] for i in idxs]
            offs, lens = pass_streams(sel, [streams_of[i] for i in idxs], np.asarray(starts)[idxs])
            for i, res in zip(idxs, self.decode_region_pass(blob, offs, lens, sel, is_ragged, lane=lane)):
                outs[i] = res
        return outs

    @_on_device
    def decode_region_pass(self, blob, offs, lens, plans, ragged, lane=None):
        """_decode_scales for the region plans of one pass (DESIGN §4.8; region.plan_passes): offs / lens int64
        [N][streams] from region.pass_streams.  Every scale decodes the tiles of each plan's rectangle (a plane that
        tile_grid cuts like the full one), its decoder network runs on the plans' windows of the coarser scale
        (symbols and, with dec.skip, features cut out of the coarser scale's) and its rows are built from the used
        rectangle of that output in place.
        ragged False: plans of equal shape_key, a batch of equal windows at per-image origins (l3c_crop_rect,
        l3c_dmll_build_table_window, l3c_reorder_tiles).
        ragged True ("Batches"; f16 / f16x2): plans of one pass_key and different shapes.  Every tensor is padded to
        the pass's largest, plan n top-left (get_P_nhwc(windows=)), and the kernels take per-image rectangles
        (l3c_crop_rects, l3c_dmll_build_table_windows, l3c_reorder_tiles_images); each plan's per-channel tile streams
        are padded with empty ones to the pass's largest tile count (stream_layout(pad_tiles=True)).
        Band plans of seek-indexed reference-layout containers (tile None, DESIGN §4.13 "Regions"): every scale's
        rectangle is a full-width band, one stream per channel whose segments over ScalePlan.seg are decoded
        (_SegmentDecode), laid out for the kernels as one tile (region.band_tile); the RGB scale builds coarse records
        (l3c_dmll_build_coarse_windows) where the whole-file decode does (f16, L = 256, K = 10), and the band's symbols
        before its seek point stay zero.
        -> [uint8 [1, C, h_n, w_n]], the regions.  lane: as in decode_device."""
        dev = blob.device
        N = len(plans)
        p0 = plans[0]
        tile = p0.tile
        band = tile is None
        K = self.net.config_ms.prob.K

        def size(r):
            return r[2] - r[0], r[3] - r[1]

        def pad(sizes):
            return max(h for h, _ in sizes), max(w for _, w in sizes)

        def rows_dev(rows):
            return E._to_device_async(np.array(rows, np.int32).reshape(N, -1), dev)

        def crop(src, origins, sizes, nhwc, split=False):
            """The sizes[n] rectangle at origins[n] of image n of src; split: one tensor per image."""
            if ragged:
                hp, wp = pad(sizes)
                return E.crop_rects(src, rows_dev([o + s for o, s in zip(origins, sizes)]), hp, wp, nhwc=nhwc,
                                    sizes=sizes if split else None)
            h, w = sizes[0]
            out = E.crop_rect(src, rows_dev(origins), h, w, nhwc=nhwc)
            return [out[n:n + 1] for n in range(N)] if split else out

        rects_of = [[(sp.C,) + size(sp.rect) for sp in p.scales] for p in plans]

        def ktile(idx):
            # the tile the layout kernels see: the container's, or for bands one that puts them in raster order
            if not band:
                return tile
            from .region import band_tile
            return band_tile(plans, idx)

        def coarse(dmll):
            # as decode_device's coarse(): the RGB scale of a seek-indexed decode in f16 from coarse records
            return band and dmll.rgb_scale and dmll.L == 256 and K == 10 and E.f16_mode()

        def network(idx, scale, bn8, F):
            wins = [size(p.scales[idx].window) for p in plans]
            l, F = self.net.get_P_nhwc(scale, bn8, F, windows=wins if len(set(wins)) > 1 else None)
            hm, wm = pad(wins)
            return l, F, (2 * hm, 2 * wm)

        def rows(idx, dmll, l, Sp, table, d, steps):
            C, plane = Sp.shape[1:]
            tg = dmll.targets(dev)
            ext = [r[idx][1:] for r in rects_of]
            if coarse(dmll):
                geo = rows_dev([p.scales[idx].out[:2] + e for p, e in zip(plans, ext)])
                max_hw = max(h * w for h, w in ext)
                return steps(lambda c: E.dmll_build_coarse_windows(l, geo, max_hw, plane, Sp, tg, K, dmll.L, c, table))
            if ragged:
                geo = rows_dev([p.scales[idx].out[:2] + e for p, e in zip(plans, ext)])
                max_hw = max(h * w for h, w in ext)
                steps(lambda c: E.dmll_build_table_windows(l, geo, max_hw, plane, Sp, tg, C, K, dmll.L, c >= 0, c,
                                                           table, ktile(idx)))
            else:
                (oy, ox), (H, W) = p0.scales[idx].out[:2], ext[0]
                steps(lambda c: E.dmll_build_table_window(l, oy, ox, Sp, tg, C, K, dmll.L, c >= 0, c, table, H, W,
                                                          ktile(idx)))

        def raster(idx, Sp):
            ext = [r[idx][1:] for r in rects_of]
            H, W = pad(ext)
            if ragged:
                return E.reorder_tiles_images(Sp, rows_dev(ext), H, W, ktile(idx))   # [N][C][H][W], zero-padded
            if band:
                return Sp.view(N, Sp.shape[1], H, W)                              # a band's stream order is raster
            return E.reorder_tiles(Sp, H, W, tile, False).view(N, Sp.shape[1], H, W)

        # the finer networks' inputs: their windows of this scale's symbols and, where they fuse them, of its features
        def symbols(idx, S):
            wins = [p.scales[idx + 1].window for p in plans]
            return crop(S, [(w[0] - p.scales[idx].rect[0], w[1] - p.scales[idx].rect[1]) for w, p in zip(wins, plans)],
                        [size(w) for w in wins], nhwc=False)

        def features(idx, F):
            if not p0.scales[idx + 1].fused:
                return None
            wins = [p.scales[idx + 1].window for p in plans]
            return crop(F.f, [(w[0] - 2 * p.scales[idx].window[0], w[1] - 2 * p.scales[idx].window[1])
                              for w, p in zip(wins, plans)], [size(w) for w in wins], nhwc=True)

        layout = stream_layout(rects_of, tile, pad_tiles=ragged)
        self.region_counts['streams'] += int((layout[2] > 0).sum())        # the empty ones that pad a ragged pass aside
        self.region_counts['symbols'] += sum(p.symbols for p in plans)
        streams = None
        if band:
            # per stream (plan, scale, channel: the container's first streams, in order) its band's symbols
            rng = np.array([[(sp.rect[0] * sp.W,) + sp.seg for sp in p.scales for _ in range(sp.C)] for p in plans],
                           np.int64)
            streams = _SegmentDecode(blob, offs, [p.seek for p in plans],
                                     (rng[:, :, 0], rng[:, :, 1], rng[:, :, 2])).decode
        S = self._decode_scales(blob, offs, lens, layout, [r[0] for r in rects_of[0]], p0.recursive, lane,
                                network, rows, raster, symbols, features,
                                row_pitch=lambda dmll: E.COARSE_PITCH if coarse(dmll) else E.table_pitch(dmll.L),
                                streams=streams, zero=band)
        return crop(S, [(p.region[0] - p.scales[-1].rect[0], p.region[1] - p.scales[-1].rect[1]) for p in plans],
                    [size(p.region) for p in plans], nhwc=False, split=True)

    # ------------------------------------------------------------------------------------------
    def _update_patch(self, patch):
        """The patch of update_region as uint8 [1, 3, h, w] on the codec's device; ValueError for anything else."""
        if not torch.is_tensor(patch) or patch.dtype not in (torch.uint8, torch.int64):
            raise ValueError('patch must be a uint8 or int64 tensor, got %s' % (
                patch.dtype if torch.is_tensor(patch) else type(patch).__name__))
        if patch.dim() == 4 and patch.shape[0] == 1:
            patch = patch[0]
        if patch.dim() != 3 or patch.shape[0] != 3:
            raise ValueError('patch must be [3, h, w] or [1, 3, h, w] (3 channels), got %s' % (tuple(patch.shape),))
        if patch.shape[1] < 1 or patch.shape[2] < 1:
            raise ValueError('empty patch %s' % (tuple(patch.shape),))
        if patch.dtype != torch.uint8 and (int(patch.min()) < 0 or int(patch.max()) > 255):
            raise ValueError('patch values must lie in 0..255')
        return patch.to(self.blueprint.device, torch.uint8).contiguous().unsqueeze(0)

    @_on_device
    def update_region(self, data, pos, patch):
        """A tiled L3C container with the pixels at pos = (y, x) (unpadded image coordinates) replaced by `patch`
        (uint8 / int64 [3, h, w] or [1, 3, h, w], 0..255, any device) -> the new container bytes, byte-identical to
        encoding the edited image (DESIGN §4.12).  Only the tile streams the edit can change are re-encoded
        (region.plan_update): the old pixels of the plan's window P_0 come from decode_regions, the encoder runs on
        its planned window of every scale, the decoder networks on their windows, the intervals of every re-encoded
        rectangle come from l3c_dmll_intervals_rect, and one range-coder launch codes every new stream; the host
        splices them into the old container.  A window of more than TILED_ENCODE_BAND_PIXELS pixels takes the whole
        path instead: decode the container, paste, encode the image (both banded where large).  update_counts says
        what ran.  ValueError, before any GPU work, for the reference layout, a container this model did not write,
        the RGB baselines, an empty patch or one not in the unpadded image, and a patch that is not 3-channel."""
        from .region import plan_update
        tile = container_tile(data)
        if tile is None:
            raise ValueError('region update needs a tiled container (written with Bitcoding(..., tile=(th, tw))): '
                             'the streams of the reference layout are serial')
        pad_tuple, parsed = parse_container(data)
        shapes = [(C, H, W) for (C, H, W, _) in parsed]
        try:
            self._check_shapes(shapes)
        except ValueError as err:
            raise ValueError('the container was not written by this model: %s' % err)
        if len(pos) != 2:
            raise ValueError('pos must be (y, x), got %r' % (pos,))
        patch = self._update_patch(patch)
        y, x = (int(v) for v in pos)
        h, w = patch.shape[2:]
        plan = plan_update(shapes, pad_tuple, tile, self.net, (y, x, h, w))
        left, _, top, _ = pad_tuple
        if plan.window_pixels > TILED_ENCODE_BAND_PIXELS:
            img, _ = self.decode_batch([data], to_host=False)
            img[:, :, top + y:top + y + h, left + x:left + x + w] = patch
            out = self.encode_batch(img, pad_tuple, tile=tile)[0][0]
            self.update_counts = {'streams': plan.total_streams, 'total': plan.total_streams,
                                  'window_pixels': img.shape[2] * img.shape[3], 'whole': True}
            return out
        return self._update_window(data, parsed, pad_tuple, tile, plan, patch)

    def _update_window(self, data, parsed, pad_tuple, tile, plan, patch):
        """update_region's window path (DESIGN §4.12)."""
        from .region import rect_streams
        dev = self.blueprint.device
        left, right, top, bottom = pad_tuple
        _, Hf, Wf = parsed[-1][:3]

        # ---- the pixels of P_0: the old ones (the padding is zero), the patch pasted in
        P = plan.window
        img = torch.zeros(1, 3, P[2] - P[0], P[3] - P[1], dtype=torch.uint8, device=dev)
        u = (max(P[0], top), max(P[1], left), min(P[2], Hf - bottom), min(P[3], Wf - right))
        old = self.decode_regions([data], [(u[0] - top, u[1] - left, u[2] - u[0], u[3] - u[1])])[0]
        img[:, :, u[0] - P[0]:u[2] - P[0], u[1] - P[1]:u[3] - P[1]] = old
        e = plan.edit
        img[:, :, e[0] - P[0]:e[2] - P[0], e[1] - P[1]:e[3] - P[1]] = patch
        del old

        # ---- encoder phase, fine to coarse: every scale's encoder on its planned window, all of its output kept
        walk = []
        for sp in plan.scales[::-1][:-1]:                       # scales 0 .. num_scales - 1
            a = sp.enc
            D = (a[0] // 2, a[1] // 2, -(-a[2] // 2), -(-a[3] // 2))
            walk.append((D, [(a, D)]))
        enc = self._encode_windows(img, P[:2], walk)

        # ---- coding phase, coarse to fine: the intervals of every R_s in its tile order, then one range-coder launch
        rects = []
        for sp in plan.scales:
            D = None if sp.window is None else tuple(2 * v for v in sp.window)      # the decoder's features: all kept
            rects.append((D, [(sp, D)]))
        layout = stream_layout([[s[:3] for s in parsed]], tile)
        ivs, cols, n_sym, ptrs = [], [], [], []
        for idx, sp, iv in self._code_rects(rects, enc, tile):
            c, n, elem = rect_streams(layout, idx, sp)
            ivs.append(iv)
            cols.append(c)
            n_sym.append(n[0])
            ptrs.append(iv.data_ptr() + elem[0] * 4)
        del enc
        cols = np.concatenate(cols)
        caps, slots, desc = _enc_descs(np.concatenate(ptrs), np.concatenate(n_sym), dev)
        _, lens_dev = E.ac_encode_streams(desc, dev)
        lens_h = torch.empty(lens_dev.shape, dtype=lens_dev.dtype, pin_memory=True)
        slots_h = torch.empty(slots.shape, dtype=torch.uint8, pin_memory=True)
        lens_h.copy_(lens_dev, non_blocking=True)
        slots_h.copy_(slots, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        del ivs
        lens = _host_lens(lens_h.numpy())
        _check_lens(lens, caps)
        slot_off = desc['out'].astype(np.int64) - slots.data_ptr()

        # ---- splice: the old streams' bytes, the new ones in their places, laid out afresh
        old_off = np.array([o for (_, _, _, st) in parsed for (o, _) in st], np.int64)
        old_len = np.array([n for (_, _, _, st) in parsed for (_, n) in st], np.int64)
        new_len = old_len.copy()
        new_len[cols] = lens
        layout = ContainerLayout([(i, C, H, W) for i, (C, H, W, _) in enumerate(parsed)], tile)
        total, pieces, new_off = layout.header_and_offsets(new_len, pad_tuple)
        new_off = np.asarray(new_off, np.int64)
        buf = np.empty(total, np.uint8)
        for o, b in pieces:
            buf[o:o + len(b)] = np.frombuffer(b, np.uint8)
        src = np.frombuffer(data, np.uint8)
        changed = np.sort(cols)
        # a run of unchanged streams keeps its bytes and the headers between them: one copy per run
        for a, b in zip(np.concatenate([[0], changed + 1]), np.concatenate([changed, [old_len.size]])):
            if b > a:
                buf[new_off[a]:new_off[b - 1] + new_len[b - 1]] = src[old_off[a]:old_off[b - 1] + old_len[b - 1]]
        sl = slots_h.numpy()
        for k, col in enumerate(cols):
            buf[new_off[col]:new_off[col] + lens[k]] = sl[slot_off[k]:slot_off[k] + lens[k]]
        self.update_counts = {'streams': int(cols.size), 'total': plan.total_streams,
                              'window_pixels': plan.window_pixels, 'whole': False}
        return buf.tobytes()

    def plan_updates(self, datas, edits):
        """Parse, validate and plan every container and edit of an update_regions call, before any GPU work: -> one
        _UpdateJob per container.  ValueError naming the container (and the edit) for every refusal of update_region."""
        from .region import merge_update_plans, plan_update
        if len(edits) != len(datas):
            raise ValueError('%d edit lists for %d containers' % (len(edits), len(datas)))
        jobs = []
        for i, (data, ed) in enumerate(zip(datas, edits)):
            tile = container_tile(data)
            if tile is None:
                raise ValueError('container %d: region update needs a tiled container (written with Bitcoding(..., '
                                 'tile=(th, tw))): the streams of the reference layout are serial' % i)
            try:
                pad_tuple, parsed = parse_container(data)
                shapes = [(C, H, W) for (C, H, W, _) in parsed]
                self._check_shapes(shapes)
            except ValueError as err:
                raise ValueError('container %d was not written by this model: %s' % (i, err))
            if self.net._rgb:
                raise ValueError('container %d: region update is not supported by the RGB baselines: their bicubic '
                                 'encoder has no planned windows' % i)
            rects, patches = [], []
            for j, e in enumerate(ed):
                try:
                    if len(e) != 2:
                        raise ValueError('an edit is (pos, patch), got %d items' % len(e))
                    pos, patch = e
                    if len(pos) != 2:
                        raise ValueError('pos must be (y, x), got %r' % (pos,))
                    patch = self._update_patch(patch)
                    rect = (int(pos[0]), int(pos[1])) + tuple(patch.shape[2:])
                    plan_update(shapes, pad_tuple, tile, self.net, rect)        # its refusals, edit by edit
                except ValueError as err:
                    raise ValueError('container %d, edit %d: %s' % (i, j, err))
                rects.append(rect)
                patches.append(patch)
            plans = merge_update_plans(shapes, pad_tuple, tile, self.net, rects)
            whole = any(p.window_pixels > TILED_ENCODE_BAND_PIXELS for p, _ in plans)
            jobs.append(_UpdateJob(data, pad_tuple, parsed, tile, rects, patches, plans, whole))
        return jobs

    @_on_device
    def update_regions(self, datas, edits):
        """update_region for many containers and many edits each: edits[i] = [(pos, patch)] for datas[i], applied in
        list order (a later patch overwrites an earlier one where they overlap) -> the new container bytes in input
        order, result i byte-identical to encoding decode(datas[i]) with every patch pasted in order (DESIGN §4.12,
        "Batches of updates").  An empty edit list returns the container unchanged.  The edits of one container are
        planned (region.merge_update_plans); a container whose merged window exceeds TILED_ENCODE_BAND_PIXELS takes the
        whole path (decode, paste every patch, encode), the others the window path (_update_windows).  updates_counts:
        one dict per container, update_counts' keys and `plans`, the number of plans after merging.  ValueError,
        before any GPU work, for every refusal of update_region, naming the container and the edit."""
        t0 = time.perf_counter()
        jobs = self.plan_updates(datas, edits)
        self.updates_stage_ms = {'parse': (time.perf_counter() - t0) * 1e3, 'upload': 0.0, 'gpu': 0.0, 'splice': 0.0,
                                 'whole': 0.0}
        outs, counts, window = [None] * len(jobs), [None] * len(jobs), []
        for i, job in enumerate(jobs):
            if not job.plans:
                outs[i] = bytes(job.data)
                counts[i] = _host_counts(job)
            elif job.whole:
                t0 = time.perf_counter()
                outs[i] = self._whole_begin(job).finish()[0][0]
                counts[i] = _host_counts(job)
                self.updates_stage_ms['whole'] += (time.perf_counter() - t0) * 1e3
            else:
                window.append(i)
        if window:
            for i, out, c in zip(window, *self._update_windows([jobs[i] for i in window])):
                outs[i], counts[i] = out, c
        self.updates_counts = counts
        return outs

    def _whole_begin(self, job, lane=None):
        """update_regions' whole path for one container, queued: decode it (lane: as in decode_batch), paste every
        patch in order, encode_begin the image -> its EncodeJob."""
        left, _, top, _ = job.pad_tuple
        img, _ = self.decode_batch([job.data], to_host=False, lane=lane)
        for (y, x, h, w), patch in zip(job.rects, job.patches):
            img[:, :, top + y:top + y + h, left + x:left + x + w] = patch
        return self.encode_begin(img, job.pad_tuple, tile=job.tile)

    @_on_device
    def update_regions_begin(self, datas, edits, lane=None):
        """update_regions queued without a host wait (DESIGN §4.12, "Serving updates") -> UpdateJob, whose finish()
        returns the bytes update_regions returns and whose `counts` are the call's updates_counts (this codec's
        updates_counts and updates_stage_ms are left as they are).  The host parse and plan (plan_updates) run here and
        raise every ValueError of update_regions before any launch.  Everything else is queued on the current stream:
        the window path up to the new stream lengths (_enqueue_windows), then l3c_update_layout lays out and
        l3c_splice_streams_dev splices every new container from those lengths in device memory, and the sizes and the
        error flag start on their way to the host; a whole-path container is decoded, pasted and encode_begin'd.
        lane: as in decode_regions -- the caller has made `lane.main` current, and the old-pixel decodes run their range
        decoders on the lane's decoder streams.  Buffers the queued work reads stay alive on the job until finish()."""
        jobs = self.plan_updates(datas, edits)
        cur = torch.cuda.current_stream()
        outs, counts, whole, window = [None] * len(jobs), [None] * len(jobs), [], []
        for i, job in enumerate(jobs):
            for patch in job.patches:
                patch.record_stream(cur)            # the caller's tensor, read on this stream
            if not job.plans:
                outs[i] = bytes(job.data)
                counts[i] = _host_counts(job)
            elif job.whole:
                whole.append((i, self._whole_begin(job, lane)))
                counts[i] = _host_counts(job)
            else:
                window.append(i)
        tail = None
        if window:
            sel = [jobs[i] for i in window]
            w = self._enqueue_windows(sel, lane, hold=True)
            conts, streams, starts, size = update_layout_inputs(
                [(job.parsed, job.tile, w.starts[k], len(job.data), w.cols[k], w.sl[k]) for k, job in enumerate(sel)],
                w.caps)
            out = torch.empty(max(size, 1), dtype=torch.uint8, device=w.blob.device)
            info, keep = E.update_splice(conts, streams, w.lens_dev, w.slot_off[:-1], w.caps, w.blob, w.slots, out)
            info_host = torch.empty(info.shape, dtype=torch.int64, pin_memory=True)
            info_host.copy_(info, non_blocking=True)
            ready = torch.cuda.Event()
            ready.record(cur)
            for i, c in zip(window, w.counts):
                counts[i] = c
            tail = (window, starts, out, info_host, ready, cur, (jobs, w, keep, info))
        return UpdateJob(self, outs, counts, whole, tail)

    def _update_windows(self, jobs):
        """update_regions' window path (DESIGN §4.12, "Batches of updates") for the jobs of one call -> ([bytes],
        [counts]).  _enqueue_windows queues everything up to the new stream lengths; they come to the host, and one
        l3c_splice_streams launch assembles every new container from host-made segments and one copy brings them to
        the host."""
        stage = self.updates_stage_ms
        w = self._enqueue_windows(jobs)
        stage['upload'] = w.upload_ms
        t0 = w.t_enqueue
        # ---- the new stream lengths, in the call's stream order, to the host (the layout depends on them)
        lens_h = torch.empty(w.lens_dev.shape, dtype=torch.int32, pin_memory=True)
        lens_h.copy_(w.lens_dev, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        lens = _host_lens(lens_h.numpy())
        _check_lens(lens, w.caps)
        stage['gpu'] = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        # ---- splice: every container's segments, one launch, one copy to the host
        segs, sizes, out_starts, pos = [], [], [], 0
        for k, job in enumerate(jobs):
            cols, sl = w.cols[k], w.sl[k]
            layout = ContainerLayout([(i, C, H, W) for i, (C, H, W, _) in enumerate(job.parsed)], job.tile)
            old_len = np.concatenate([np.asarray(st, np.int64).reshape(-1, 2)[:, 1] for (_, _, _, st) in job.parsed])
            _, old_off = layout.offsets(old_len)
            new_len = old_len.copy()
            new_len[cols] = lens[sl]
            total, new_off = layout.offsets(new_len)
            segs.append(splice_segments(old_off, old_len, len(job.data), new_off, cols, lens[sl], w.slot_off[sl],
                                        w.starts[k], pos))
            sizes.append(total)
            out_starts.append(pos)
            pos += (total + 15) & ~15
        out = torch.empty(pos, dtype=torch.uint8, device=w.blob.device)
        E.splice_streams(w.blob, w.slots, np.concatenate(segs), out)
        host = torch.empty(out.shape, dtype=torch.uint8, pin_memory=True)
        host.copy_(out, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        buf = host.numpy()
        outs = [buf[s:s + n].tobytes() for s, n in zip(out_starts, sizes)]
        stage['splice'] = (time.perf_counter() - t0) * 1e3
        return outs, w.counts

    def _enqueue_windows(self, jobs, lane=None, hold=False):
        """The part of update_regions' window path that runs without a host wait, shared by update_regions and
        update_regions_begin: everything up to the new stream lengths in device memory.  One upload of the containers,
        read by the old-pixel decodes and the splice.  The plans are grouped into passes of one tile size whose windows
        fit TILED_ENCODE_BAND_PIXELS (region.plan_update_passes).  Per pass: the old pixels of every window from region
        passes (_decode_planned; on the lane's decoder streams with `lane`), the patches pasted in order, then per plan
        the encoders and the coding on its windows (_encode_windows, _code_rects) and one range-coder launch for every
        new stream of the pass.  A stream that two separate plans re-encode is coded once (both give the same bytes).
        hold: keep every pass's intervals alive in `keep` (they are freed after each pass otherwise).
        -> _WindowWork: blob and starts (_upload), upload_ms and t_enqueue (the host clock after the upload), caps and
        slot_off (int64 per new stream, in the call's stream order), slots, lens_dev (int32 on the device) and, per
        job, cols (the ascending columns of its re-encoded streams), sl (their indices into lens_dev) and counts."""
        from .region import plan_region, plan_update_passes, rect_streams
        dev = self.blueprint.device
        w = _WindowWork()
        t0 = time.perf_counter()
        w.blob, w.starts = _upload([job.data for job in jobs], dev)
        w.t_enqueue = time.perf_counter()
        w.upload_ms = (w.t_enqueue - t0) * 1e3
        w.keep = []
        geo = self._geometry()
        # ---- host: every plan's streams (duplicates across a container's plans dropped) and its slot in one buffer
        items = []
        for k, job in enumerate(jobs):
            layout = stream_layout([[s[:3] for s in job.parsed]], job.tile)
            seen = np.zeros(layout[2].shape[1], bool)
            for plan, _ in job.plans:
                keep = {}
                for sp in plan.scales:
                    cols, n, elem = rect_streams(layout, sp.idx, sp)
                    new = ~seen[cols]
                    seen[cols] = True
                    ch = np.repeat(np.arange(sp.C), len(sp.tiles))
                    keep[sp.idx] = (cols[new], n[0][new], elem[0][new], ch[new])
                items.append((k, plan, keep))
        caps = _slot_cap(np.concatenate([kp[1] for _, _, keep in items for _, kp in sorted(keep.items())]))
        slot_off = np.concatenate([[0], np.cumsum(caps)])
        slots = torch.empty(max(int(slot_off[-1]), 1), dtype=torch.uint8, device=dev)
        w.caps, w.slot_off, w.slots = caps, slot_off, slots
        passes = plan_update_passes([plan for _, plan, _ in items], TILED_ENCODE_BAND_PIXELS)
        first = np.zeros(len(items) + 1, np.int64)          # each plan's first stream in the call's stream order
        first[1:] = np.cumsum([sum(kp[0].size for kp in keep.values()) for _, _, keep in items])
        lens_parts = []
        for ps in passes:
            # ---- old pixels of every window (the padding is zero), then the patches in order
            imgs, rplans = [], []
            for t in ps:
                k, plan, _ = items[t]
                job, P = jobs[k], plan.window
                left, right, top, bottom = job.pad_tuple
                _, Hf, Wf = job.parsed[-1][:3]
                u = (max(P[0], top), max(P[1], left), min(P[2], Hf - bottom), min(P[3], Wf - right))
                rplans.append(plan_region([s[:3] for s in job.parsed], job.pad_tuple, job.tile, geo,
                                          (u[0] - top, u[1] - left, u[2] - u[0], u[3] - u[1])))
                imgs.append((u, torch.zeros(1, 3, P[2] - P[0], P[3] - P[1], dtype=torch.uint8, device=dev)))
            olds = self._decode_planned(w.blob, w.starts[[items[t][0] for t in ps]],
                                        [[st for (_, _, _, st) in jobs[items[t][0]].parsed] for t in ps], rplans, lane)
            for t, (u, img), old in zip(ps, imgs, olds):
                k, plan, _ = items[t]
                job, P = jobs[k], plan.window
                img[:, :, u[0] - P[0]:u[2] - P[0], u[1] - P[1]:u[3] - P[1]] = old
                left, _, top, _ = job.pad_tuple
                for (y, x, h, w_), patch in zip(job.rects, job.patches):
                    e = (y + top, x + left, y + top + h, x + left + w_)
                    c = (max(e[0], P[0]), max(e[1], P[1]), min(e[2], P[2]), min(e[3], P[3]))
                    if c[0] < c[2] and c[1] < c[3]:
                        img[:, :, c[0] - P[0]:c[2] - P[0], c[1] - P[1]:c[3] - P[1]] = \
                            patch[:, :, c[0] - e[0]:c[2] - e[0], c[1] - e[1]:c[3] - e[1]]
            del olds
            # ---- encoder phase fine to coarse, coding phase coarse to fine: the whole pass as one ragged batch of
            # windows where the network runs one, else plan after plan as update_region's window path
            if self.net.ragged_unsupported() is None:
                coded = self._code_pass_ragged([items[t][1] for t in ps], [img for _, img in imgs], jobs[items[ps[0]][0]].tile)
            else:
                coded = self._code_pass_serial([items[t][1] for t in ps], [img for _, img in imgs],
                                               [jobs[items[t][0]].tile for t in ps])
            del imgs
            descs, order, keep_alive, nxt = [], [], [], {t: first[t] for t in ps}
            for n, idx, sp, iv, plane in coded:
                t = ps[n]
                cols, cnt, elem, ch = items[t][2][idx]
                if plane is not None:           # image n's planes of a [N][C][plane] batch of interval planes
                    elem = (n * sp.C + ch) * plane + elem - ch * (sp.rect[2] - sp.rect[0]) * (sp.rect[3] - sp.rect[1])
                s0 = nxt[t]
                d = np.zeros(cols.size, dtype=_lib.ENC_STREAM_DTYPE)
                d['intervals'] = iv.data_ptr() + elem * 4
                d['n_sym'] = cnt
                d['out_cap'] = caps[s0:s0 + cols.size]
                d['out'] = slots.data_ptr() + slot_off[s0:s0 + cols.size]
                nxt[t] = s0 + cols.size
                descs.append(d)
                order.append(np.arange(s0, s0 + cols.size))
                keep_alive.append(iv)
            # ---- one range-coder launch for every new stream of the pass
            desc = np.concatenate(descs)
            if desc.size:
                lens_parts.append((np.concatenate(order), E.ac_encode_streams(desc, dev)[1]))
            if hold:
                w.keep.extend(keep_alive)
            del keep_alive, coded
        # ---- the new stream lengths in the call's stream order
        w.lens_dev = torch.empty(int(first[-1]), dtype=torch.int32, device=dev)
        for order, ln in lens_parts:
            w.lens_dev[E._to_device_async(order, dev)] = ln
        # ---- per job: its re-encoded streams in container order, where their lengths are, and the call's counts
        w.cols, w.sl, w.counts = [], [], []
        for k in range(len(jobs)):
            mine = [t for t, it in enumerate(items) if it[0] == k]
            cols = np.concatenate([kp[0] for t in mine for _, kp in sorted(items[t][2].items())])
            sl = np.concatenate([np.arange(first[t], first[t + 1]) for t in mine])
            order = np.argsort(cols, kind='stable')
            w.cols.append(cols[order])
            w.sl.append(sl[order])
            w.counts.append({'streams': int(cols.size), 'total': items[mine[0]][1].total_streams,
                             'window_pixels': sum(items[t][1].window_pixels for t in mine), 'whole': False,
                             'plans': len(mine)})
        return w

    def _code_pass_serial(self, plans, imgs, tiles):
        """The encoders and the coding of the update plans of one pass, plan after plan, on their windows as update_region
        does (_encode_windows, _code_rects).  imgs[n]: the pixels of plans[n]'s P_0, uint8 [1][3][h][w].  Yields (n, idx,
        sp, intervals int32 [1][C][h * w] of sp.rect in its tile order, None) as each rectangle's intervals are queued."""
        for n, (plan, img, tile) in enumerate(zip(plans, imgs, tiles)):
            walk = []
            for sp in plan.scales[::-1][:-1]:
                a = sp.enc
                D = (a[0] // 2, a[1] // 2, -(-a[2] // 2), -(-a[3] // 2))
                walk.append((D, [(a, D)]))
            enc = self._encode_windows(img, plan.window[:2], walk)
            rects = [(None if sp.window is None else tuple(2 * v for v in sp.window),
                      [(sp, None if sp.window is None else tuple(2 * v for v in sp.window))]) for sp in plan.scales]
            for idx, sp, iv in self._code_rects(rects, enc, tile):
                yield n, idx, sp, iv, None
            del enc

    def _code_pass_ragged(self, plans, imgs, tile):
        """_code_pass_serial for a pass of plans of one tile size as ONE ragged batch of their windows (f16: the network
        runs padded batches of differently sized images, ragged_unsupported).  Fine to coarse, each scale's head and
        encoder run once on a padded batch of the plans' encoder windows, window n top-left, under ragged_extents
        (l3c_crop_rects cuts them out of the finer scale's padded batch).  Coarse to fine, each decoder runs once on the
        plans' decoder windows (get_P_nhwc(windows=)) and l3c_dmll_intervals_rects codes every plan's R_s to its own
        stream planes; the uniform-prior scale codes each plan's rectangle with lut_intervals in its own tile order.
        Yields (n, idx, sp, intervals, plane): intervals int32 [N][C][plane] shared by the plans of a scale (plane None:
        [1][C][h * w] of plan n alone)."""
        net, dev, N = self.net, self.blueprint.device, len(plans)
        K = net.config_ms.prob.K
        by = [{sp.scale: sp for sp in p.scales} for p in plans]

        def rows_dev(rows):
            return E._to_device_async(np.array(rows, np.int32).reshape(N, -1), dev)

        def size(r):
            return r[2] - r[0], r[3] - r[1]

        # the scale-0 symbols: every P_0, padded, window n top-left
        P = [p.window for p in plans]
        X = torch.zeros(N, 3, max(size(r)[0] for r in P), max(size(r)[1] for r in P), dtype=torch.uint8, device=dev)
        for n, img in enumerate(imgs):
            X[n, :, :img.shape[2], :img.shape[3]] = img[0]
        enc = [([r[:2] for r in P], X, None)]                 # by scale: (origin of window n, symbols, values NHWC)
        x, xo = X, [r[:2] for r in P]
        for s in range(net.scales):
            A = [b[s].enc for b in by]
            # A window that ends on an odd row or column is one longer in the batch, so that every resolution of the
            # encoder is an exact half of the one before (E.extents_at).  The window starts on an even row and column
            # (encoder_rect), and where it ends on an odd one that end is not the plane's edge, whose size is even, so it
            # ends inside the image: the extra row or column is a zero the single-window run also reads there (its
            # tensor's border), and it reaches only outputs within the window's planned margins, which the plan never
            # reads.  Every output the plan reads is the same bits as update_region's.
            ext = [(h + h % 2, w + w % 2) for h, w in map(size, A)]
            hp, wp = max(h for h, _ in ext), max(w for _, w in ext)
            Hx, Wx = (x.shape[1], x.shape[2]) if s > 0 else (x.shape[2], x.shape[3])
            hc, wc = min(hp, Hx), min(wp, Wx)            # a crop is at most its source; a rounded window may be longer
            inp = E.crop_rects(x, rows_dev([(a[0] - o[0], a[1] - o[1]) + size(a) for a, o in zip(A, xo)]), hc, wc,
                               nhwc=s > 0)
            if (hc, wc) != (hp, wp):
                grown = inp.new_zeros((N, hp, wp, inp.shape[3]) if s > 0 else (N, inp.shape[1], hp, wp))
                (grown[:, :hc, :wc] if s > 0 else grown[:, :, :hc, :wc]).copy_(inp)
                inp = grown
            with E.ragged_extents(ext, hp, wp):
                if s == 0:
                    inp = net._rgb_head_input(inp)
                    hd = inp if isinstance(inp, E.Act) else net.heads[0](inp)
                else:
                    hd = net.heads[s](self._operand_act(inp))
                eo = net.nets[s].enc(hd)
            xo = [(a[0] // 2, a[1] // 2) for a in A]
            enc.append((xo, eo.S.contiguous(), eo.bn_q))
            if s + 1 < net.scales:
                x = eo.F.r if E.tensor_core_mode() else eo.F.f
            del eo, hd, inp
        F = None                                              # (origins, features) the next finer decoder adds
        for idx, (scale, dmll, uniform) in enumerate(self.iter_scale_dmll(0)):
            o, Ssym, _ = enc[scale]
            sps = [b[scale] for b in by]
            if uniform:
                for n, sp in enumerate(sps):
                    h, w = size(sp.rect)
                    sym = _crop(Ssym[n:n + 1], o[n], sp.rect, nhwc=False)
                    yield n, idx, sp, E.reorder_tiles(E.lut_intervals(sym, self._uniform(dmll.L, dev)[0]), h, w, tile,
                                                      True), None
                continue
            ob, _, bq = enc[scale + 1]
            wins = [sp.window for sp in sps]
            wsz = [size(w) for w in wins]
            hm, wm = max(h for h, _ in wsz), max(w for _, w in wsz)
            win = E.crop_rects(bq, rows_dev([(w[0] - b[0], w[1] - b[1]) + sz for w, b, sz in zip(wins, ob, wsz)]), hm,
                               wm, nhwc=True)
            Fw = None
            if net.fuses(scale):
                Fw = E.crop_rects(F[1], rows_dev([(w[0] - f[0], w[1] - f[1]) + sz for w, f, sz in zip(wins, F[0], wsz)]),
                                  hm, wm, nhwc=True)
            l, Fo = net.get_P_nhwc(scale, win, Fw, windows=wsz if len(set(wsz)) > 1 else None)
            del win, Fw
            geo = [sp.out[:2] + (sp.rect[0] - on[0], sp.rect[1] - on[1]) + size(sp.rect) + tuple(on) + (sp.H, sp.W)
                   for sp, on in zip(sps, o)]
            iv = E.dmll_intervals_rects(l, Ssym, geo, dmll.targets(dev), sps[0].C, K, dmll.L, dmll.rgb_scale, tile)
            del l
            for n, sp in enumerate(sps):
                yield n, idx, sp, iv, iv.shape[2]
            F = ([(2 * w[0], 2 * w[1]) for w in wins], Fo.f) if scale >= 1 and net.fuses(scale - 1) else None
            del Fo

    # stage timing of a decode (bench.py / tools): set `codec.stage_events = []` before decode_device,
    # synchronise, then read stage_ms()
    stage_events = None

    def _mark(self, name):
        if self.stage_events is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.stage_events.append((name, ev))

    def stage_ms(self):
        """{stage: ms} of the decode recorded since `stage_events = []` (call after a synchronize)."""
        evs, self.stage_events = self.stage_events or [], None
        out = {}
        for (_, a), (name, b) in zip(evs[:-1], evs[1:]):
            out[name] = out.get(name, 0.0) + a.elapsed_time(b)
        return out

    def _check_shapes(self, shapes):
        """C, H, W of every scale come straight from the (untrusted) file, while the kernels index with
        the shapes the MODEL produces (each scale twice the size of the coarser one, C = 3 for the image
        and the RGB baselines, q.C for bottlenecks).  A crafted, truncated or wrong-config container must
        fail here, before any buffer is sized from it (the reference fails with a torch shape error).
        -> R, the number of recursive scales (DESIGN §4.7): the scales beyond the model's num_scales + 1, allowed
        for the RGB baselines only."""
        cfg = self.net.config_ms
        n = len(shapes)
        R = n - (self.net.scales + 1)
        if R < 0:
            raise ValueError('container has %d scales, model expects %d' % (n, self.net.scales + 1))
        if R > 0 and not self.net._rgb:
            raise ValueError('container has %d scales, model expects %d: recursive containers are written by the '
                             'RGB baselines only' % (n, self.net.scales + 1))
        for idx, (C, H, W) in enumerate(shapes):
            scale = n - 1 - idx
            want_C = 3 if (scale == 0 or self.net._rgb) else cfg.q.C
            if C != want_C:
                raise ValueError('container scale %d has %d channels, model expects %d' % (scale, C, want_C))
            if H < 1 or W < 1:
                raise ValueError('container scale %d has an empty shape %dx%d' % (scale, H, W))
            check_plane(H, W, 'container scale %d' % scale)
            if idx > 0:
                Hc, Wc = shapes[idx - 1][1:]
                if (H, W) != (2 * Hc, 2 * Wc):
                    raise ValueError('container scale %d is %dx%d, expected twice the coarser scale (%dx%d)'
                                     % (scale, H, W, 2 * Hc, 2 * Wc))
        return R

    def _symbol_values(self, scale, dmll, dev):
        """Value of every symbol of bottleneck `scale`: the `levels` LUT of the quantiser that produced
        it (nets[scale-1].enc.levels, a checkpoint parameter: net.py:123-127) so that the decoder feeds
        its nets exactly what the encoder fed (SURVEY finding 1); plain 0..255 for the RGB baselines."""
        if self.net._rgb:
            return dmll.values(dev)
        return self.net.nets[scale - 1].enc.levels.detach().float().contiguous()
