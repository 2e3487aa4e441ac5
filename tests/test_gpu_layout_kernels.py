"""The data-movement kernels (include/l3c_b200.h) element for element against numpy restatements of their header text:
l3c_reorder_tiles, l3c_reorder_tiles_images, l3c_crop_rect, l3c_crop_rects, l3c_ragged_zero_halo, l3c_ragged_pack,
l3c_pack_streams and l3c_lut_intervals.

A layout that is wrong in the same way in both directions still round-trips, and a write past a plane or a slot
usually lands where a later kernel overwrites it.  So every destination here is a view into a larger allocation filled
with a canary -- NaN bit patterns where the kernel moves 4-byte words, 0xA5 where it moves bytes -- and the whole
allocation is compared byte for byte: the documented output region against the restatement, where zeros are +0 (not
-0), and everything else against the canary.

The restatements are written from the header's words; the host tests at the top pin each of them to cases worked out
by hand, so a misreading the restatement shared with a kernel would show there.  The refusals are checked in a
process that sees no CUDA device: an argument check that is missing then fails the call with L3C_ECUDA instead of
launching a kernel on arguments outside its contract.
"""
import ctypes
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu

CANARY_WORD = 0x7FA5A5A5            # a NaN bit pattern
NEG_ZERO = 0x80000000               # -0.0
CANARY_BYTE = 0xA5
GUARD = 8192                        # canary bytes on each side of every source and destination


# ---------------------------------------------------------------------------------------------
# restatements of the header (numpy, host)
# ---------------------------------------------------------------------------------------------
def tile_order(H, W, th, tw):
    """raster index of every position of the tile order of an H x W plane: th x tw tiles in row-major tile order,
    smaller at the right and bottom edges, pixels row-major inside a tile"""
    idx = np.arange(H * W, dtype=np.int64).reshape(H, W)
    return np.concatenate([idx[y:y + th, x:x + tw].ravel() for y in range(0, H, th) for x in range(0, W, tw)])


def tile_position(y, x, H, W, th, tw):
    """the inverse of tile_order for arrays (numpy or torch int64) of raster coordinates: the tile rows above hold
    ty * th * W pixels, the tiles to the left in this tile row tx * tw * (height of this tile row)"""
    ty, tx = y // th, x // tw
    hh, ww = (H - ty * th).clip(max=th), (W - tx * tw).clip(max=tw)
    return ty * th * W + tx * tw * hh + (y - ty * th) * ww + (x - tx * tw)


def crop(src, y, x, h, w):
    """src [..., H, W, e] -> the h x w rectangle at (y, x)"""
    return src[..., y:y + h, x:x + w, :]


def pad_top_left(a, hp, wp):
    """a [..., h, w, e] -> [..., hp, wp, e], a top-left and +0 elsewhere"""
    out = np.zeros(a.shape[:-3] + (hp, wp, a.shape[-1]), a.dtype)
    out[..., :a.shape[-3], :a.shape[-2], :] = a
    return out


def compact(plane, h, w, compact_len):
    """one padded plane [H, W, e] -> its h x w image row-major, then zeros up to compact_len elements"""
    out = np.zeros((compact_len, plane.shape[-1]), plane.dtype)
    out[:h * w] = plane[:h, :w].reshape(h * w, -1)
    return out


def uncompact(c, h, w, H, W):
    """one compact plane [compact_len, e] -> the padded H x W plane, zeros outside the h x w image"""
    out = np.zeros((H, W, c.shape[-1]), c.dtype)
    out[:h, :w] = c[:h * w].reshape(h, w, -1)
    return out


def halo_band(H, W, h, w, halo):
    """bool [H, W]: [h, h + halo) x [0, w + halo) and [0, h) x [w, w + halo), clipped to the tensor"""
    m = np.zeros((H, W), bool)
    m[h:h + halo, :w + halo] = True
    m[:h, w:w + halo] = True
    return m


def pack_blob(blob, slots, lens, caps, offs):
    """the first min(len, cap) bytes of every slot to blob[off:]"""
    out = blob.copy()
    for s, n, c, o in zip(slots, lens, caps, offs):
        k = min(int(n), int(c))
        out[o:o + k] = s[:k]
    return out


def uniform_row(L):
    """the shared CDF row of the uniform prior (bitcoding.py:297-323): fp32 1/L, fp32 running sum, times 2^16,
    rounded half to even; the top entry is 2^16 (the reference's int16 cast wraps it to 0, the coder never reads it)"""
    c = np.add.accumulate(np.full(L, np.float32(1) / np.float32(L), np.float32), dtype=np.float32)
    row = np.concatenate([[0], np.rint(c * np.float32(65536)).astype(np.int64)])
    row[L] = 65536
    return row


def uniform_lut(L):
    """256 coding intervals c_low | (c_high - 1) << 16 of symbols 0..L-1 under uniform_row(L), 0 past L"""
    row = uniform_row(L)
    lut = np.zeros(256, np.int64)
    lut[:L] = row[:L] + ((row[1:L + 1] - 1) << 16)
    return lut


# ---------------------------------------------------------------------------------------------
# host self-tests of the restatements: cases worked out by hand
# ---------------------------------------------------------------------------------------------
def test_tile_order_of_5x7_plane_in_2x3_tiles():
    # tiles (rows x cols): [0,2)x[0,3) [0,2)x[3,6) [0,2)x[6,7) | [2,4)x.. | [4,5)x[0,3) [4,5)x[3,6) [4,5)x[6,7)
    want = [0, 1, 2, 7, 8, 9, 3, 4, 5, 10, 11, 12, 6, 13,
            14, 15, 16, 21, 22, 23, 17, 18, 19, 24, 25, 26, 20, 27,
            28, 29, 30, 31, 32, 33, 34]
    assert tile_order(5, 7, 2, 3).tolist() == want


def test_tile_order_edges_by_hand():
    assert tile_order(2, 3, 5, 5).tolist() == [0, 1, 2, 3, 4, 5]             # one tile larger than the plane
    assert tile_order(2, 3, 1, 1).tolist() == [0, 1, 2, 3, 4, 5]             # 1 x 1 tiles: raster order
    assert tile_order(3, 2, 9, 1).tolist() == [0, 2, 4, 1, 3, 5]             # column tiles
    assert tile_order(1, 5, 4, 2).tolist() == [0, 1, 2, 3, 4]
    assert tile_order(3, 3, 2, 2).tolist() == [0, 1, 3, 4, 2, 5, 6, 7, 8]


@pytest.mark.parametrize('H,W', [(1, 1), (1, 9), (9, 1), (5, 7), (8, 8), (13, 6)])
def test_tile_position_inverts_tile_order(H, W):
    for th in range(1, H + 3):
        for tw in range(1, W + 3):
            order = tile_order(H, W, th, tw)
            assert sorted(order.tolist()) == list(range(H * W))
            y, x = np.divmod(order, W)
            assert tile_position(y, x, H, W, th, tw).tolist() == list(range(H * W)), (th, tw)


def test_crop_compact_and_halo_by_hand():
    a = np.arange(12).reshape(3, 4, 1)
    assert crop(a, 1, 2, 2, 2)[..., 0].tolist() == [[6, 7], [10, 11]]
    assert pad_top_left(crop(a, 1, 2, 2, 2), 3, 3)[..., 0].tolist() == [[6, 7, 0], [10, 11, 0], [0, 0, 0]]
    assert compact(a, 2, 3, 8)[:, 0].tolist() == [0, 1, 2, 4, 5, 6, 0, 0]
    assert uncompact(np.arange(1, 9).reshape(8, 1), 2, 3, 3, 4)[..., 0].tolist() == \
        [[1, 2, 3, 0], [4, 5, 6, 0], [0, 0, 0, 0]]
    # a 2 x 3 image in a 5 x 6 tensor, halo 2: columns 3..4 beside it, rows 2..3 below it (columns 0..4)
    assert halo_band(5, 6, 2, 3, 2).astype(int).tolist() == [[0, 0, 0, 1, 1, 0],
                                                             [0, 0, 0, 1, 1, 0],
                                                             [1, 1, 1, 1, 1, 0],
                                                             [1, 1, 1, 1, 1, 0],
                                                             [0, 0, 0, 0, 0, 0]]
    assert not halo_band(4, 4, 4, 4, 3).any()                                  # extent = tensor: no band
    assert halo_band(4, 4, 3, 4, 3)[3].all() and halo_band(4, 4, 3, 4, 3).sum() == 4    # clipped right and bottom


def test_stream_packing_by_hand():
    blob = np.full(12, 0xA5, np.uint8)
    slots = [np.array([1, 2, 3, 4], np.uint8), np.array([5, 6, 7, 8], np.uint8), np.array([9], np.uint8)]
    got = pack_blob(blob, slots, lens=[2, 9, 0], caps=[4, 4, 4], offs=[1, 5, 11])
    assert got.tolist() == [0xA5, 1, 2, 0xA5, 0xA5, 5, 6, 7, 8, 0xA5, 0xA5, 0xA5]


def test_uniform_lut_by_hand():
    assert uniform_row(2).tolist() == [0, 32768, 65536]
    assert uniform_row(4).tolist() == [0, 16384, 32768, 49152, 65536]
    # fp32(1/3) = 0.3333333433..., 2 * that = 0.6666666865...: 21845.33 -> 21845, 43690.67 -> 43691
    assert uniform_row(3).tolist() == [0, 21845, 43691, 65536]
    assert uniform_lut(3)[:4].tolist() == [0 | 21844 << 16, 21845 | 43690 << 16, 43691 | 65535 << 16, 0]
    for L in (2, 4, 8, 16, 32, 64, 128, 256):                     # powers of two are exact
        assert uniform_row(L).tolist() == [65536 * i // L for i in range(L + 1)]
    for L in range(2, 257):                                       # every symbol keeps a nonempty interval
        row = uniform_row(L)
        assert (np.diff(row) > 0).all() and np.abs(row * L - 65536 * np.arange(L + 1)).max() <= L


def test_uniform_row_of_the_library_is_the_restated_row():
    from l3c_pytorch_b200 import engine as E
    for L in range(2, 257):
        lib_row = E.uniform_cdf_row(L).astype(np.int64)
        assert lib_row[L] == 0                                   # the int16 wrap of 2^16, as in the reference
        assert lib_row[:L].tolist() == uniform_row(L)[:L].tolist(), L


# ---------------------------------------------------------------------------------------------
# refusals: host checks, no launch (run where no device is visible)
# ---------------------------------------------------------------------------------------------
_REFUSALS = r'''
import ctypes, json, sys
sys.path.insert(0, %(root)r)
from l3c_pytorch_b200._lib import lib
V, P, Q, A = ctypes.c_void_p, ctypes.c_void_p(4096), ctypes.c_void_p(8192), ctypes.c_void_p(12288)
O = ctypes.c_void_p(12292)                                   # 4-byte but not 16-byte aligned
null, s = None, None
big = 1 << 40
cases = {
  'reorder_tiles': [
    lambda: lib.l3c_reorder_tiles(null, Q, 1, 1, 4, 4, 2, 2, 1, s),
    lambda: lib.l3c_reorder_tiles(P, null, 1, 1, 4, 4, 2, 2, 1, s),
    lambda: lib.l3c_reorder_tiles(P, P, 1, 1, 4, 4, 2, 2, 1, s),
    lambda: lib.l3c_reorder_tiles(P, Q, 2, 1, 4, 4, 2, 2, 1, s),
    lambda: lib.l3c_reorder_tiles(P, Q, 8, 1, 4, 4, 2, 2, 1, s),
    lambda: lib.l3c_reorder_tiles(P, Q, 0, 1, 4, 4, 2, 2, 1, s),
    lambda: lib.l3c_reorder_tiles(P, Q, 1, 0, 4, 4, 2, 2, 1, s),
    lambda: lib.l3c_reorder_tiles(P, Q, 1, 65536, 4, 4, 2, 2, 1, s),
    lambda: lib.l3c_reorder_tiles(P, Q, 1, 1, 0, 4, 2, 2, 1, s),
    lambda: lib.l3c_reorder_tiles(P, Q, 1, 1, 4, 4, 0, 2, 1, s),
    lambda: lib.l3c_reorder_tiles(P, Q, 1, 1, 4, 4, 2, -1, 1, s),
    lambda: lib.l3c_reorder_tiles(P, Q, 1, 1, 46341, 46341, 8, 16, 1, s),     # H * W > 2^31 - 1
    lambda: lib.l3c_reorder_tiles(P, Q, 4, 1, 65536, 32768, 8, 16, 0, s),     # H * W = 2^31
  ],
  'reorder_tiles_images': [
    lambda: lib.l3c_reorder_tiles_images(null, Q, 1, 1, 16, 4, 4, A, 2, 2, s),
    lambda: lib.l3c_reorder_tiles_images(P, null, 1, 1, 16, 4, 4, A, 2, 2, s),
    lambda: lib.l3c_reorder_tiles_images(P, Q, 1, 1, 16, 4, 4, null, 2, 2, s),
    lambda: lib.l3c_reorder_tiles_images(P, P, 1, 1, 16, 4, 4, A, 2, 2, s),
    lambda: lib.l3c_reorder_tiles_images(P, Q, 0, 1, 16, 4, 4, A, 2, 2, s),
    lambda: lib.l3c_reorder_tiles_images(P, Q, 3, 21846, 16, 4, 4, A, 2, 2, s),   # N * planes = 65538
    lambda: lib.l3c_reorder_tiles_images(P, Q, 1, 1, 0, 4, 4, A, 2, 2, s),
    lambda: lib.l3c_reorder_tiles_images(P, Q, 1, 1, 16, 4, 0, A, 2, 2, s),
    lambda: lib.l3c_reorder_tiles_images(P, Q, 1, 1, 16, 4, 4, A, 0, 2, s),
    lambda: lib.l3c_reorder_tiles_images(P, Q, 1, 1, 16, 46341, 46341, A, 8, 16, s),   # hp * wp > 2^31 - 1
  ],
  'crop_rect': [
    lambda: lib.l3c_crop_rect(null, Q, 4, 1, 1, 8, 8, A, 2, 2, s),
    lambda: lib.l3c_crop_rect(P, null, 4, 1, 1, 8, 8, A, 2, 2, s),
    lambda: lib.l3c_crop_rect(P, Q, 4, 1, 1, 8, 8, null, 2, 2, s),
    lambda: lib.l3c_crop_rect(P, P, 4, 1, 1, 8, 8, A, 2, 2, s),
    lambda: lib.l3c_crop_rect(P, Q, 0, 1, 1, 8, 8, A, 2, 2, s),
    lambda: lib.l3c_crop_rect(P, Q, -4, 1, 1, 8, 8, A, 2, 2, s),
    lambda: lib.l3c_crop_rect(P, Q, 4, 0, 1, 8, 8, A, 2, 2, s),
    lambda: lib.l3c_crop_rect(P, Q, 4, 256, 256, 8, 8, A, 2, 2, s),           # N * planes = 65536
    lambda: lib.l3c_crop_rect(P, Q, 4, 1, 1, 8, 8, A, 9, 2, s),               # taller than the plane
    lambda: lib.l3c_crop_rect(P, Q, 4, 1, 1, 8, 8, A, 2, 9, s),               # wider than the plane
    lambda: lib.l3c_crop_rect(P, Q, 4, 1, 1, 8, 8, A, 0, 2, s),
    lambda: lib.l3c_crop_rect(P, Q, 1, 1, 1, 1 << 20, 1 << 20, A, 1 << 20, 1 << 20, s),   # 2^40 bytes: grid.x
    lambda: lib.l3c_crop_rect(P, Q, 1 << 30, 1, 1, 1 << 16, 1 << 16, A, 1 << 16, 1 << 16, s),
  ],
  'crop_rects': [
    lambda: lib.l3c_crop_rects(null, Q, 4, 1, 1, 8, 8, A, null, 2, 2, s),
    lambda: lib.l3c_crop_rects(P, null, 4, 1, 1, 8, 8, A, null, 2, 2, s),
    lambda: lib.l3c_crop_rects(P, Q, 4, 1, 1, 8, 8, null, null, 2, 2, s),
    lambda: lib.l3c_crop_rects(P, P, 4, 1, 1, 8, 8, A, null, 2, 2, s),
    lambda: lib.l3c_crop_rects(P, Q, 4, 1, 1, 8, 8, O, null, 2, 2, s),        # rects not 16-byte aligned
    lambda: lib.l3c_crop_rects(P, Q, 0, 1, 1, 8, 8, A, null, 2, 2, s),
    lambda: lib.l3c_crop_rects(P, Q, 4, 1, 65536, 8, 8, A, null, 2, 2, s),
    lambda: lib.l3c_crop_rects(P, Q, 4, 1, 1, 8, 8, A, null, 9, 2, s),
    lambda: lib.l3c_crop_rects(P, Q, 4, 1, 1, 8, 8, A, Q, 2, 9, s),
    lambda: lib.l3c_crop_rects(P, Q, 4, 1, 1, 8, 8, A, null, 0, 2, s),
    lambda: lib.l3c_crop_rects(P, Q, 3, 1, 1, 1 << 20, 1 << 20, A, null, 1 << 20, 1 << 20, s),
  ],
  'ragged_zero_halo': [
    lambda: lib.l3c_ragged_zero_halo(null, 4, 1, 8, 8, A, 1, s),
    lambda: lib.l3c_ragged_zero_halo(P, 4, 1, 8, 8, null, 1, s),
    lambda: lib.l3c_ragged_zero_halo(P, 6, 1, 8, 8, A, 1, s),
    lambda: lib.l3c_ragged_zero_halo(P, 2, 1, 8, 8, A, 1, s),
    lambda: lib.l3c_ragged_zero_halo(P, 0, 1, 8, 8, A, 1, s),
    lambda: lib.l3c_ragged_zero_halo(P, 4, 0, 8, 8, A, 1, s),
    lambda: lib.l3c_ragged_zero_halo(P, 4, 65536, 8, 8, A, 1, s),
    lambda: lib.l3c_ragged_zero_halo(P, 4, 1, 0, 8, A, 1, s),
    lambda: lib.l3c_ragged_zero_halo(P, 4, 1, 8, 8, A, -1, s),
    lambda: lib.l3c_ragged_zero_halo(P, 4, 1, 1 << 30, 1 << 30, A, 1 << 30, s),   # band of 2^61 pixels: grid.x
    lambda: lib.l3c_ragged_zero_halo(P, 1 << 24, 1, 1 << 16, 1 << 16, A, 8, s),      # 2^20 pixels of 2^22 words
  ],
  'ragged_pack': [
    lambda: lib.l3c_ragged_pack(null, Q, 4, 1, 1, 8, 8, A, 64, 1, s),
    lambda: lib.l3c_ragged_pack(P, null, 4, 1, 1, 8, 8, A, 64, 1, s),
    lambda: lib.l3c_ragged_pack(P, Q, 4, 1, 1, 8, 8, null, 64, 1, s),
    lambda: lib.l3c_ragged_pack(P, P, 4, 1, 1, 8, 8, A, 64, 0, s),
    lambda: lib.l3c_ragged_pack(P, Q, 0, 1, 1, 8, 8, A, 64, 1, s),
    lambda: lib.l3c_ragged_pack(P, Q, 4, 0, 1, 8, 8, A, 64, 1, s),
    lambda: lib.l3c_ragged_pack(P, Q, 4, 65535, 2, 8, 8, A, 64, 1, s),
    lambda: lib.l3c_ragged_pack(P, Q, 4, 1, 1, 0, 8, A, 64, 1, s),
    lambda: lib.l3c_ragged_pack(P, Q, 4, 1, 1, 8, 8, A, 0, 1, s),
    lambda: lib.l3c_ragged_pack(P, Q, 1, 1, 1, 8, 8, A, big, 1, s),              # 2^40 compact elements
    lambda: lib.l3c_ragged_pack(P, Q, 8, 1, 1, 1 << 30, 1 << 30, A, 64, 0, s),   # 2^61 padded words
  ],
  'pack_streams': [
    lambda: lib.l3c_pack_streams(null, Q, A, 1, P, s),
    lambda: lib.l3c_pack_streams(P, null, A, 1, Q, s),
    lambda: lib.l3c_pack_streams(P, Q, null, 1, A, s),
    lambda: lib.l3c_pack_streams(P, Q, A, 1, null, s),
    lambda: lib.l3c_pack_streams(P, Q, A, -1, O, s),
  ],
  'lut_intervals': [
    lambda: lib.l3c_lut_intervals(null, Q, 16, A, s),
    lambda: lib.l3c_lut_intervals(P, null, 16, A, s),
    lambda: lib.l3c_lut_intervals(P, Q, 16, null, s),
    lambda: lib.l3c_lut_intervals(P, Q, 16, P, s),                          # intervals over the symbols
    lambda: lib.l3c_lut_intervals(P, Q, 16, Q, s),                          # intervals over the LUT
    lambda: lib.l3c_lut_intervals(P, Q, -1, A, s),
    lambda: lib.l3c_lut_intervals(P, Q, big, A, s),                         # 2^32 CTAs
  ],
}
out = {}
for name, calls in cases.items():
    res = []
    for call in calls:
        lib.l3c_launch_log(None, 0, 1)
        rc = call()
        res.append((rc, lib.l3c_launch_log(None, 0, 0), (lib.l3c_last_error() or b'').decode()))
    out[name] = res
print(json.dumps(out))
'''


@pytest.fixture(scope='module')
def refusals():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    p = subprocess.run([sys.executable, '-c', _REFUSALS % {'root': ROOT}], capture_output=True, text=True, env=env,
                       timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize('entry', ['reorder_tiles', 'reorder_tiles_images', 'crop_rect', 'crop_rects',
                                   'ragged_zero_halo', 'ragged_pack', 'pack_streams', 'lut_intervals'])
def test_arguments_outside_the_header_are_refused_before_any_launch(refusals, entry):
    for i, (rc, launches, msg) in enumerate(refusals[entry]):
        assert (rc, launches) == (-1, 0), (entry, i, rc, launches, msg)      # L3C_EINVAL, nothing launched
        assert msg.startswith('l3c_' + entry), (entry, i, msg)


# ---------------------------------------------------------------------------------------------
# device helpers
# ---------------------------------------------------------------------------------------------
def _lib():
    from l3c_pytorch_b200._lib import lib
    return lib


def _stream():
    from l3c_pytorch_b200 import engine as E
    return E._stream_ptr()


def _ok(rc):
    from l3c_pytorch_b200._lib import check
    check(rc)
    torch.cuda.synchronize()


def _canary(nbytes, words):
    """host bytes of the canary pattern"""
    if words:
        assert nbytes % 4 == 0
        return np.full(nbytes // 4, CANARY_WORD, np.uint32).view(np.uint8)
    return np.full(nbytes, CANARY_BYTE, np.uint8)


class Guarded:
    """`nbytes` of device memory at byte GUARD of an allocation of GUARD + nbytes + GUARD bytes, all of it filled with
    the canary (or with `fill`, host bytes of the whole allocation)"""

    def __init__(self, nbytes, words, fill=None):
        self.n, self.words = int(nbytes), words
        self.host = _canary(GUARD + ((self.n + 3) // 4) * 4 + GUARD, words) if fill is None else fill
        self.buf = torch.from_numpy(self.host.copy()).cuda()

    @property
    def ptr(self):
        return ctypes.c_void_p(self.buf.data_ptr() + GUARD)

    def expect(self, region):
        """host bytes the whole allocation must hold when the region (bytes) is the documented output"""
        want = self.host.copy()
        want[GUARD:GUARD + self.n] = np.asarray(region, np.uint8).reshape(-1)
        return want

    def check(self, want, what):
        got = self.buf.cpu().numpy()
        if not np.array_equal(got, want):
            i = int(np.nonzero(got != want)[0][0])
            where = 'before the output' if i < GUARD else 'after the output' if i >= GUARD + self.n else \
                'in the output at byte %d' % (i - GUARD)
            raise AssertionError('%s: first differing byte %s: got %#x, want %#x (%d bytes differ)'
                                 % (what, where, got[i], want[i], int((got != want).sum())))


def _dev(a):
    """a copy of the host array on the device, between GUARD canary bytes on each side"""
    t = torch.from_numpy(np.ascontiguousarray(a))
    raw = torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8))
    buf = torch.full((GUARD + raw.numel() + GUARD,), CANARY_BYTE, dtype=torch.uint8, device='cuda')
    buf[GUARD:GUARD + raw.numel()] = raw.cuda()
    return buf[GUARD:GUARD + raw.numel()].view(t.dtype).view(t.shape)


def _rand_bytes(rng, shape):
    return rng.integers(0, 256, size=shape, dtype=np.uint8)


WIDTHS = [1, 2, 3, 4, 8, 12, 128, 480]       # bytes per element: byte path (1, 2, 3), word path (4, 8, 12, ...)


# ---------------------------------------------------------------------------------------------
# l3c_reorder_tiles
# ---------------------------------------------------------------------------------------------
TILE_CASES = [
    (5, 7, 2, 3),          # the hand-worked plane
    (1, 1, 1, 1), (1, 1, 8, 16),
    (1, 17, 4, 5), (17, 1, 4, 5),                      # H or W = 1
    (9, 13, 1, 1),                                     # 1 x 1 tiles
    (6, 8, 16, 16), (6, 40, 16, 8), (40, 6, 8, 16),    # tiles larger than the plane in both, H only, W only
    (33, 47, 8, 16),                                   # partial tiles on both edges
    (64, 64, 8, 16), (7, 300, 3, 64), (130, 3, 64, 2),
]


@gpu
@pytest.mark.parametrize('H,W,th,tw', TILE_CASES)
@pytest.mark.parametrize('elem', [1, 4])
def test_reorder_tiles_is_the_tile_order(H, W, th, tw, elem):
    lib = _lib()
    rng = np.random.default_rng(H * 1000 + W + th * 7 + tw)
    planes = 3
    src_np = _rand_bytes(rng, (planes, H * W, elem))
    src = _dev(src_np)
    perm = tile_order(H, W, th, tw)
    for to_tiles in (1, 0):
        dst = Guarded(planes * H * W * elem, elem == 4)
        _ok(lib.l3c_reorder_tiles(ctypes.c_void_p(src.data_ptr()), dst.ptr, elem, planes, H, W, th, tw, to_tiles,
                                  _stream()))
        want = np.empty_like(src_np)
        if to_tiles:
            want[:, :] = src_np[:, perm]
        else:
            want[:, perm] = src_np
        dst.check(dst.expect(want), ('to_tiles' if to_tiles else 'to_raster', H, W, th, tw, elem))


# ---------------------------------------------------------------------------------------------
# l3c_reorder_tiles_images
# ---------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('tile', [(8, 16), (1, 1), (3, 5), (64, 64)])
def test_reorder_tiles_images_is_each_images_tile_order(tile):
    lib = _lib()
    rng = np.random.default_rng(tile[0] * 100 + tile[1])
    hp, wp = 37, 45
    ext = [(37, 45), (1, 1), (1, 45), (37, 1), (20, 33), (8, 16), (9, 17)]
    N, P = len(ext), 2
    plane_len = hp * wp + 13                                  # garbage after each image's h * w bytes
    src_np = _rand_bytes(rng, (N, P, plane_len))
    src, ext_dev = _dev(src_np), _dev(np.array(ext, np.int32))
    dst = Guarded(N * P * hp * wp, False)
    _ok(lib.l3c_reorder_tiles_images(ctypes.c_void_p(src.data_ptr()), dst.ptr, P, N, plane_len, hp, wp,
                                     ctypes.c_void_p(ext_dev.data_ptr()), tile[0], tile[1], _stream()))
    want = np.zeros((N, P, hp, wp), np.uint8)
    for n, (h, w) in enumerate(ext):
        perm = tile_order(h, w, *tile)
        for q in range(P):
            img = np.empty(h * w, np.uint8)
            img[perm] = src_np[n, q, :h * w]
            want[n, q, :h, :w] = img.reshape(h, w)
    dst.check(dst.expect(want), ('reorder_tiles_images', tile))


# ---------------------------------------------------------------------------------------------
# l3c_crop_rect / l3c_crop_rects
# ---------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('elem', WIDTHS)
def test_crop_rect_is_the_rectangle(elem):
    lib = _lib()
    rng = np.random.default_rng(elem)
    N, P, H, W = 3, 2, 13, 11
    src_np = _rand_bytes(rng, (N, P, H, W, elem))
    src = _dev(src_np)
    for (h, w), org in [((13, 11), [(0, 0)] * 3),                            # the whole plane
                        ((1, 1), [(0, 0), (12, 10), (6, 3)]),                # 1 x 1, in the far corner
                        ((4, 7), [(9, 4), (0, 0), (5, 2)]),                  # flush with the bottom right
                        ((13, 1), [(0, 10), (0, 0), (0, 5)])]:
        org_dev = _dev(np.array(org, np.int32))
        dst = Guarded(N * P * h * w * elem, elem % 4 == 0)
        _ok(lib.l3c_crop_rect(ctypes.c_void_p(src.data_ptr()), dst.ptr, elem, P, N, H, W,
                              ctypes.c_void_p(org_dev.data_ptr()), h, w, _stream()))
        want = np.stack([crop(src_np[n], y, x, h, w) for n, (y, x) in enumerate(org)])
        dst.check(dst.expect(want), ('crop_rect', elem, h, w))


RECTS = [(0, 0, 13, 11), (12, 10, 1, 1), (3, 2, 5, 9), (9, 0, 4, 11), (0, 7, 13, 4)]


@gpu
@pytest.mark.parametrize('elem', WIDTHS)
def test_crop_rects_padded_is_each_rectangle_top_left_and_zeros(elem):
    lib = _lib()
    rng = np.random.default_rng(100 + elem)
    N, P, H, W = len(RECTS), 2, 13, 11
    src_np = _rand_bytes(rng, (N, P, H, W, elem))
    src = _dev(src_np)
    rects_dev = _dev(np.array(RECTS, np.int32))
    dst = Guarded(N * P * H * W * elem, elem % 4 == 0)                       # hp x wp = the plane
    _ok(lib.l3c_crop_rects(ctypes.c_void_p(src.data_ptr()), dst.ptr, elem, P, N, H, W,
                           ctypes.c_void_p(rects_dev.data_ptr()), None, H, W, _stream()))
    want = np.stack([pad_top_left(crop(src_np[n], y, x, h, w), H, W) for n, (y, x, h, w) in enumerate(RECTS)])
    dst.check(dst.expect(want), ('crop_rects padded', elem))
    # hp x wp larger than every rectangle: a zero margin right of and below all of them
    rects = [(y, x, min(h, 9), min(w, 7)) for (y, x, h, w) in RECTS]
    rects_dev = _dev(np.array(rects, np.int32))
    dst = Guarded(N * P * 10 * 8 * elem, elem % 4 == 0)
    _ok(lib.l3c_crop_rects(ctypes.c_void_p(src.data_ptr()), dst.ptr, elem, P, N, H, W,
                           ctypes.c_void_p(rects_dev.data_ptr()), None, 10, 8, _stream()))
    want = np.stack([pad_top_left(crop(src_np[n], y, x, h, w), 10, 8) for n, (y, x, h, w) in enumerate(rects)])
    dst.check(dst.expect(want), ('crop_rects padded, margin', elem))


@gpu
@pytest.mark.parametrize('elem', WIDTHS)
def test_crop_rects_compacted_goes_to_dst_off_and_nowhere_else(elem):
    lib = _lib()
    rng = np.random.default_rng(200 + elem)
    N, P, H, W = len(RECTS), 3, 13, 11
    src_np = _rand_bytes(rng, (N, P, H, W, elem))
    src = _dev(src_np)
    rects_dev = _dev(np.array(RECTS, np.int32))
    # image n's planes follow each other from element dst_off[n]; gaps of canary between (and before) the images,
    # the images in an order other than n
    sizes = [P * h * w for (_, _, h, w) in RECTS]
    order, off, offs = [2, 0, 4, 1, 3], 5, [0] * N
    for n in order:
        offs[n] = off
        off += sizes[n] + 3
    dst = Guarded(off * elem, elem % 4 == 0)
    off_dev = _dev(np.array(offs, np.int64))
    _ok(lib.l3c_crop_rects(ctypes.c_void_p(src.data_ptr()), dst.ptr, elem, P, N, H, W,
                           ctypes.c_void_p(rects_dev.data_ptr()), ctypes.c_void_p(off_dev.data_ptr()), 13, 11,
                           _stream()))
    region = dst.host[GUARD:GUARD + off * elem].copy().reshape(off, elem)
    for n, (y, x, h, w) in enumerate(RECTS):
        region[offs[n]:offs[n] + sizes[n]] = crop(src_np[n], y, x, h, w).reshape(-1, elem)
    dst.check(dst.expect(region), ('crop_rects compacted', elem))


# ---------------------------------------------------------------------------------------------
# l3c_ragged_pack
# ---------------------------------------------------------------------------------------------
PACK_EXT = [(13, 11), (1, 1), (1, 11), (13, 1), (7, 5), (12, 10)]


@gpu
@pytest.mark.parametrize('elem', WIDTHS)
@pytest.mark.parametrize('tail', [0, 9])
def test_ragged_pack_both_ways(elem, tail):
    lib = _lib()
    rng = np.random.default_rng(300 + elem + tail)
    N, P, H, W = len(PACK_EXT), 2, 13, 11
    clen = max(h * w for h, w in PACK_EXT) + tail               # tail > 0: longer than every h * w
    ext_dev = _dev(np.array(PACK_EXT, np.int32))
    words = elem % 4 == 0
    # padded -> compact
    pad_np = _rand_bytes(rng, (N, P, H, W, elem))
    src = _dev(pad_np)
    dst = Guarded(N * P * clen * elem, words)
    _ok(lib.l3c_ragged_pack(ctypes.c_void_p(src.data_ptr()), dst.ptr, elem, P, N, H, W,
                            ctypes.c_void_p(ext_dev.data_ptr()), clen, 1, _stream()))
    want = np.stack([[compact(pad_np[n, q], h, w, clen) for q in range(P)] for n, (h, w) in enumerate(PACK_EXT)])
    dst.check(dst.expect(want), ('to_compact', elem, tail))
    # compact -> padded (garbage in the compact tails is not read)
    cmp_np = _rand_bytes(rng, (N, P, clen, elem))
    src = _dev(cmp_np)
    dst = Guarded(N * P * H * W * elem, words)
    _ok(lib.l3c_ragged_pack(ctypes.c_void_p(src.data_ptr()), dst.ptr, elem, P, N, H, W,
                            ctypes.c_void_p(ext_dev.data_ptr()), clen, 0, _stream()))
    want = np.stack([[uncompact(cmp_np[n, q], h, w, H, W) for q in range(P)] for n, (h, w) in enumerate(PACK_EXT)])
    dst.check(dst.expect(want), ('to_padded', elem, tail))


# ---------------------------------------------------------------------------------------------
# l3c_ragged_zero_halo
# ---------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('px_bytes', [4, 12, 128, 256])
@pytest.mark.parametrize('halo', [1, 2, 4, 8])
def test_zero_halo_sets_exactly_the_band_to_plus_zero(px_bytes, halo):
    lib = _lib()
    H, W = 19, 23
    ext = [(19, 23),                   # the whole tensor: no band
           (1, 1), (9, 14),            # band inside the tensor
           (19 - halo // 2, 7),        # clipped at the bottom
           (5, 23 - halo // 2),        # clipped on the right
           (19 - halo // 2, 23 - halo // 2),   # clipped on both
           (19, 5), (3, 23)]           # touching an edge: only the other band
    N, wpp = len(ext), px_bytes // 4
    # -0.0 and NaN canaries alternating over the words, and in the guards
    words = GUARD // 4 + N * H * W * wpp + GUARD // 4
    host = np.where(np.arange(words) % 2 == 0, NEG_ZERO, CANARY_WORD).astype(np.uint32).view(np.uint8)
    x = Guarded(N * H * W * px_bytes, True, fill=host)
    ext_dev = _dev(np.array(ext, np.int32))
    _ok(lib.l3c_ragged_zero_halo(x.ptr, px_bytes, N, H, W, ctypes.c_void_p(ext_dev.data_ptr()), halo, _stream()))
    region = host[GUARD:GUARD + N * H * W * px_bytes].view(np.uint32).reshape(N, H, W, wpp).copy()
    for n, (h, w) in enumerate(ext):
        region[n][halo_band(H, W, h, w, halo)] = 0
    x.check(x.expect(region.view(np.uint8)), ('zero_halo', px_bytes, halo))


# ---------------------------------------------------------------------------------------------
# N * planes = 65535: the grid.y limit, every kernel that puts a plane or an image per grid row
# ---------------------------------------------------------------------------------------------
@gpu
def test_65535_planes_every_entry_point():
    lib = _lib()
    rng = np.random.default_rng(65535)
    NP, H, W = 65535, 3, 5
    src_np = _rand_bytes(rng, (NP, H, W))
    src = _dev(src_np)
    sp = ctypes.c_void_p(src.data_ptr())
    # l3c_reorder_tiles: 65535 planes
    dst = Guarded(NP * H * W, False)
    _ok(lib.l3c_reorder_tiles(sp, dst.ptr, 1, NP, H, W, 2, 3, 1, _stream()))
    dst.check(dst.expect(src_np.reshape(NP, H * W)[:, tile_order(H, W, 2, 3)]), 'reorder_tiles')
    # N = 65535 images of one plane each, every image its own rectangle / extent
    ext = np.stack([rng.integers(1, H + 1, NP), rng.integers(1, W + 1, NP)], 1).astype(np.int32)
    org = np.stack([rng.integers(0, H - ext[:, 0] + 1), rng.integers(0, W - ext[:, 1] + 1)], 1)
    rects = np.concatenate([org, ext], 1).astype(np.int32)
    orders = {(h, w): tile_order(h, w, 2, 3) for h in range(1, H + 1) for w in range(1, W + 1)}
    ext_dev, rects_dev = _dev(ext), _dev(rects)
    dst = Guarded(NP * 2 * 2, False)
    org_dev = _dev(np.stack([rng.integers(0, H - 1, NP), rng.integers(0, W - 1, NP)], 1).astype(np.int32))
    _ok(lib.l3c_crop_rect(sp, dst.ptr, 1, 1, NP, H, W, ctypes.c_void_p(org_dev.data_ptr()), 2, 2, _stream()))
    o = org_dev.cpu().numpy()
    dst.check(dst.expect(np.stack([src_np[n, y:y + 2, x:x + 2] for n, (y, x) in enumerate(o)])), 'crop_rect')
    dst = Guarded(NP * H * W, False)
    _ok(lib.l3c_crop_rects(sp, dst.ptr, 1, 1, NP, H, W, ctypes.c_void_p(rects_dev.data_ptr()), None, H, W,
                           _stream()))
    want = np.zeros((NP, H, W), np.uint8)
    for n, (y, x, h, w) in enumerate(rects):
        want[n, :h, :w] = src_np[n, y:y + h, x:x + w]
    dst.check(dst.expect(want), 'crop_rects')
    dst = Guarded(NP * H * W, False)
    _ok(lib.l3c_ragged_pack(sp, dst.ptr, 1, 1, NP, H, W, ctypes.c_void_p(ext_dev.data_ptr()), H * W, 1, _stream()))
    want = np.stack([compact(src_np[n][..., None], h, w, H * W)[:, 0] for n, (h, w) in enumerate(ext)])
    dst.check(dst.expect(want), 'ragged_pack')
    dst = Guarded(NP * H * W, False)
    _ok(lib.l3c_reorder_tiles_images(sp, dst.ptr, 1, NP, H * W, H, W, ctypes.c_void_p(ext_dev.data_ptr()), 2, 3,
                                     _stream()))
    want = np.zeros((NP, H, W), np.uint8)
    for n, (h, w) in enumerate(ext):
        img = np.empty(h * w, np.uint8)
        img[orders[(h, w)]] = src_np[n].reshape(-1)[:h * w]
        want[n, :h, :w] = img.reshape(h, w)
    dst.check(dst.expect(want), 'reorder_tiles_images')
    x = Guarded(NP * H * W * 4, True)
    _ok(lib.l3c_ragged_zero_halo(x.ptr, 4, NP, H, W, ctypes.c_void_p(ext_dev.data_ptr()), 2, _stream()))
    region = x.host[GUARD:GUARD + NP * H * W * 4].view(np.uint32).reshape(NP, H, W).copy()
    for n, (h, w) in enumerate(ext):
        region[n][halo_band(H, W, h, w, 2)] = 0
    x.check(x.expect(region.view(np.uint8)), 'zero_halo')


# ---------------------------------------------------------------------------------------------
# l3c_pack_streams
# ---------------------------------------------------------------------------------------------
def _enc_descs(outs, caps):
    from l3c_pytorch_b200 import _lib as L
    d = np.zeros(len(outs), L.ENC_STREAM_DTYPE)
    d['out'], d['out_cap'] = outs, caps
    return _dev(d.view(np.uint8))


@gpu
def test_pack_streams_over_two_launches_truncates_to_the_slot():
    lib = _lib()
    rng = np.random.default_rng(70001)
    n = 70001                                             # two launches: 65535 + 4466 streams
    caps = (rng.integers(0, 17, n) * 4).astype(np.int64)  # 0 to 64 bytes, multiples of 4
    caps[7] = 3 * 16384 * 64 + 4000                       # one slot beyond a grid row's stride (64 chunks of 16 KiB)
    lens = rng.integers(0, 70, n).astype(np.int64)
    lens[::11] = 0                                        # empty streams
    lens[5::13] = caps[5::13] + rng.integers(1, 9, len(lens[5::13]))   # streams that outgrew their slot
    lens[7], lens[65534], lens[65535], lens[n - 1] = caps[7] - 3, caps[65534] + 1, caps[65535], caps[n - 1] + 8
    slot_off = np.concatenate([[0], np.cumsum(caps)[:-1]])
    slots_np = _rand_bytes(rng, int(caps.sum()))
    slots = _dev(slots_np)
    # odd byte offsets, each stream's bytes followed by a gap of 1 to 3 canary bytes, the streams out of order
    order = rng.permutation(n)
    step = np.minimum(lens, caps)[order] + rng.integers(1, 4, n)
    offs = np.zeros(n, np.int64)
    offs[order] = 1 + np.concatenate([[0], np.cumsum(step)[:-1]])
    pos = 1 + int(step.sum())
    blob = Guarded(pos, False)
    descs = _enc_descs(slots.data_ptr() + slot_off, caps)
    lens_dev, offs_dev = _dev(lens.astype(np.uint32)), _dev(offs.astype(np.uint64))
    from l3c_pytorch_b200 import engine as E
    E.launch_log(reset=True)
    _ok(lib.l3c_pack_streams(ctypes.c_void_p(descs.data_ptr()), ctypes.c_void_p(lens_dev.data_ptr()),
                             ctypes.c_void_p(offs_dev.data_ptr()), n, ctypes.c_void_p(blob.buf.data_ptr() + GUARD),
                             _stream()))
    assert E.launch_log(reset=True)[0] == {'pack_streams_kernel': 2}
    region = pack_blob(blob.host[GUARD:GUARD + pos], [slots_np[o:o + c] for o, c in zip(slot_off, caps)], lens,
                       caps, offs)
    blob.check(blob.expect(region), 'pack_streams')


# ---------------------------------------------------------------------------------------------
# l3c_lut_intervals
# ---------------------------------------------------------------------------------------------
def _codec_lut(L):
    """the LUT the codec builds for the coarsest scale (BatchCodec._uniform)"""
    from l3c_pytorch_b200.codec import BatchCodec
    lut_dev, _ = BatchCodec._uniform(types.SimpleNamespace(_const={}), L, 'cuda')
    return lut_dev


@gpu
def test_lut_intervals_every_alphabet_and_symbol():
    lib = _lib()
    rng = np.random.default_rng(256)
    for L in range(2, 257):
        lut_dev = _codec_lut(L)
        assert lut_dev.cpu().numpy().view(np.uint32).astype(np.int64).tolist() == uniform_lut(L).tolist(), L
        n = 3 * 256 + 37 + L                               # not a multiple of 256
        sym_np = np.concatenate([np.arange(L), rng.integers(0, L, n - L)]).astype(np.uint8)
        rng.shuffle(sym_np)
        sym = _dev(sym_np)
        iv = Guarded(4 * n, True)
        _ok(lib.l3c_lut_intervals(ctypes.c_void_p(sym.data_ptr()), ctypes.c_void_p(lut_dev.data_ptr()), n, iv.ptr,
                                  _stream()))
        iv.check(iv.expect(uniform_lut(L)[sym_np].astype(np.uint32).view(np.uint8)), ('lut_intervals', L))


# ---------------------------------------------------------------------------------------------
# offsets past 2^31 elements and 2^32 bytes (each case under about 10 GiB of device memory)
# ---------------------------------------------------------------------------------------------
CHUNK = 1 << 24


def _pattern(i, salt):
    """a byte of data for int64 positions i (torch, on the device)"""
    return (((i * 0x9E3779B1 + salt * 0x85EBCA77) >> 17) & 0xFF).to(torch.uint8)


def _alloc_guarded(nbytes):
    """device uint8 GUARD + nbytes + GUARD, guards 0xA5 -> (allocation, the view in between)"""
    buf = torch.empty(GUARD + nbytes + GUARD, dtype=torch.uint8, device='cuda')
    buf[:GUARD] = CANARY_BYTE
    buf[GUARD + nbytes:] = CANARY_BYTE
    return buf, buf[GUARD:GUARD + nbytes]


def _nonzero(t):
    """nonzero elements of a large tensor, counted in slices along its first dimension"""
    step = max(1, CHUNK // max(1, t[0].numel()))
    return sum(int(torch.count_nonzero(t[a:a + step])) for a in range(0, t.shape[0], step))


def _guards_intact(buf, what):
    assert bool((buf[:GUARD] == CANARY_BYTE).all()) and bool((buf[-GUARD:] == CANARY_BYTE).all()), what


@pytest.fixture
def big_memory():
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.cuda.empty_cache()
    print('peak device memory: %.2f GiB' % (torch.cuda.max_memory_allocated() / 2 ** 30))


@gpu
def test_reorder_tiles_past_2_to_the_32_bytes(big_memory):
    lib = _lib()
    P, H, W, th, tw = 5, 29500, 29500, 999, 701           # 5 * 8.7e8 bytes: offsets past 2^31 and 2^32
    HW = H * W
    assert P * HW > 2 ** 32
    buf_s, src = _alloc_guarded(P * HW)
    buf_d, dst = _alloc_guarded(P * HW)
    dst.fill_(CANARY_BYTE)
    for q in range(P):
        for a in range(0, HW, CHUNK):
            src[q * HW + a:q * HW + min(a + CHUNK, HW)] = _pattern(torch.arange(a, min(a + CHUNK, HW),
                                                                                device='cuda'), q)
    _ok(lib.l3c_reorder_tiles(ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr()), 1, P, H, W, th, tw,
                              1, _stream()))
    _guards_intact(buf_d, 'to_tiles')
    for q in range(P):
        plane = dst[q * HW:(q + 1) * HW]
        for a in range(0, HW, CHUNK):
            p = torch.arange(a, min(a + CHUNK, HW), device='cuda')
            pos = tile_position(p // W, p % W, H, W, th, tw)
            assert torch.equal(plane[pos], _pattern(p, q)), (q, a)
    src.fill_(CANARY_BYTE)                                  # and back: every raster byte rewritten
    _ok(lib.l3c_reorder_tiles(ctypes.c_void_p(dst.data_ptr()), ctypes.c_void_p(src.data_ptr()), 1, P, H, W, th, tw,
                              0, _stream()))
    _guards_intact(buf_s, 'to_raster')
    for q in range(P):
        for a in range(0, HW, CHUNK):
            b = min(a + CHUNK, HW)
            assert torch.equal(src[q * HW + a:q * HW + b], _pattern(torch.arange(a, b, device='cuda'), q)), (q, a)


@gpu
def test_crops_pack_and_halo_past_2_to_the_31_words(big_memory):
    """one allocation of 4 planes of 13400 x 13400 pixels of 12 bytes (2.16e9 words, 8.6 GB), read by the crops and
    the ragged gather at their far end, then written whole by the ragged scatter and in place by the halo kernel"""
    lib = _lib()
    N, P, H, W, E3 = 2, 2, 13400, 13400, 3                 # E3 words per element
    words = N * P * H * W * E3
    assert words > 2 ** 31
    buf, big = _alloc_guarded(words * 4)
    bw = big.view(torch.int32).view(N, P, H, W, E3)
    g = torch.Generator(device='cuda').manual_seed(31)

    def rnd(*shape):
        return torch.randint(-2 ** 31, 2 ** 31, shape, generator=g, device='cuda', dtype=torch.int64).to(torch.int32)

    # crops at the far end of the last plane and elsewhere
    rects = [(100, 200, 37, 53), (H - 41, W - 29, 41, 29)]
    rects_np = np.array(rects, np.int32)
    for n, (y, x, h, w) in enumerate(rects):
        bw[n, :, y:y + h, x:x + w] = rnd(P, h, w, E3)
    org_dev = _dev(np.array([(y, x) for (y, x, _, _) in rects], np.int32))
    hh, ww = 37, 29
    out = Guarded(N * P * hh * ww * 12, True)
    _ok(lib.l3c_crop_rect(ctypes.c_void_p(big.data_ptr()), out.ptr, 12, P, N, H, W,
                          ctypes.c_void_p(org_dev.data_ptr()), hh, ww, _stream()))
    want = torch.stack([bw[n, :, y:y + hh, x:x + ww] for n, (y, x, _, _) in enumerate(rects)])
    out.check(out.expect(want.cpu().numpy().view(np.uint8)), 'crop_rect')
    rects_dev = _dev(rects_np)
    hp, wp = 41, 53
    out = Guarded(N * P * hp * wp * 12, True)
    _ok(lib.l3c_crop_rects(ctypes.c_void_p(big.data_ptr()), out.ptr, 12, P, N, H, W,
                           ctypes.c_void_p(rects_dev.data_ptr()), None, hp, wp, _stream()))
    want = np.stack([pad_top_left(bw[n, :, y:y + h, x:x + w].cpu().numpy(), hp, wp)
                     for n, (y, x, h, w) in enumerate(rects)])
    out.check(out.expect(want.view(np.uint8)), 'crop_rects padded')
    sizes = [P * h * w for (_, _, h, w) in rects]
    offs = np.array([sizes[1] + 1, 0], np.int64)
    off_dev = _dev(offs)
    out = Guarded((sum(sizes) + 1) * 12, True)
    _ok(lib.l3c_crop_rects(ctypes.c_void_p(big.data_ptr()), out.ptr, 12, P, N, H, W,
                           ctypes.c_void_p(rects_dev.data_ptr()), ctypes.c_void_p(off_dev.data_ptr()), hp, wp,
                           _stream()))
    region = out.host[GUARD:GUARD + (sum(sizes) + 1) * 12].view(np.uint32).reshape(-1, E3).copy()
    for n, (y, x, h, w) in enumerate(rects):
        region[offs[n]:offs[n] + sizes[n]] = bw[n, :, y:y + h, x:x + w].cpu().numpy().view(np.uint32).reshape(-1, E3)
    out.check(out.expect(region.view(np.uint8)), 'crop_rects compacted')
    # ragged gather: the last image's extent reaches the last rows of its planes
    ext = [(5, 7), (H, 5)]
    for n, (h, w) in enumerate(ext):
        bw[n, :, :h, :w] = rnd(P, h, w, E3)
    ext_dev = _dev(np.array(ext, np.int32))
    clen = H * 5 + 3
    out = Guarded(N * P * clen * 12, True)
    _ok(lib.l3c_ragged_pack(ctypes.c_void_p(big.data_ptr()), out.ptr, 12, P, N, H, W,
                            ctypes.c_void_p(ext_dev.data_ptr()), clen, 1, _stream()))
    cmp_np = np.stack([[compact(bw[n, q, :h, :w].cpu().numpy(), h, w, clen) for q in range(P)]
                       for n, (h, w) in enumerate(ext)])
    out.check(out.expect(cmp_np.view(np.uint8)), 'ragged_pack to_compact')
    # ragged scatter into the whole allocation: the images and +0 everywhere else
    big.fill_(CANARY_BYTE)
    cmp = _dev(cmp_np)
    _ok(lib.l3c_ragged_pack(ctypes.c_void_p(cmp.data_ptr()), ctypes.c_void_p(big.data_ptr()), 12, P, N, H, W,
                            ctypes.c_void_p(ext_dev.data_ptr()), clen, 0, _stream()))
    _guards_intact(buf, 'ragged_pack to_padded')
    for n, (h, w) in enumerate(ext):
        for q in range(P):
            img = cmp[n, q, :h * w].view(h, w, E3)
            assert torch.equal(bw[n, q, :h, :w], img), (n, q)
            assert _nonzero(bw[n, q]) == int(torch.count_nonzero(img)), (n, q)                     # +0 elsewhere
    # zero_halo in place on 4 images of 13400 x 13400 pixels of 12 bytes: -0.0 / NaN canaries by word of the pixel
    NI = N * P
    xw = big.view(torch.int32).view(NI, H, W, E3)
    canary = torch.tensor([NEG_ZERO - 2 ** 32, CANARY_WORD, NEG_ZERO - 2 ** 32], dtype=torch.int32, device='cuda')
    for i in range(NI):
        xw[i] = canary
    ext = [(H, W), (13000, 9000), (H - 3, 17), (13300, W - 5)]          # the last band lies past 2^31 words
    halo = 8
    ext_dev = _dev(np.array(ext, np.int32))
    _ok(lib.l3c_ragged_zero_halo(ctypes.c_void_p(big.data_ptr()), 12, NI, H, W, ctypes.c_void_p(ext_dev.data_ptr()),
                                 halo, _stream()))
    _guards_intact(buf, 'zero_halo')
    for i, (h, w) in enumerate(ext):
        img = xw[i]
        hb, wr = min(h + halo, H), min(w + halo, W)
        band = [img[h:hb, :wr], img[:h, w:wr]]
        rest = [img[:h, :w], img[:h, wr:], img[hb:], img[h:hb, wr:]]
        assert all(bool((b == 0).all()) for b in band), i
        assert all(bool((r == canary).all()) for r in rest), i


@gpu
def test_reorder_tiles_images_and_pack_streams_past_2_to_the_32_bytes(big_memory):
    lib = _lib()
    NP, hp, wp = 5, 41500, 41500                           # 5 planes of 1.7e9 bytes: offsets past 2^32
    total = NP * hp * wp
    buf, big = _alloc_guarded(total)
    big.fill_(CANARY_BYTE)
    ext = [(5, 41500), (300, 500), (1, 1), (41500, 7), (77, 41333)]
    plane_len = max(h * w for h, w in ext)
    g = torch.Generator(device='cuda').manual_seed(32)
    src = torch.randint(0, 256, (NP, plane_len), generator=g, device='cuda', dtype=torch.int64).to(torch.uint8)
    ext_dev = _dev(np.array(ext, np.int32))
    _ok(lib.l3c_reorder_tiles_images(ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(big.data_ptr()), 1, NP,
                                     plane_len, hp, wp, ctypes.c_void_p(ext_dev.data_ptr()), 64, 64, _stream()))
    _guards_intact(buf, 'reorder_tiles_images')
    dv = big.view(NP, hp, wp)
    for n, (h, w) in enumerate(ext):
        img = torch.empty(h * w, dtype=torch.uint8, device='cuda')
        img[torch.from_numpy(tile_order(h, w, 64, 64)).cuda()] = src[n, :h * w]
        img = img.view(h, w)
        assert torch.equal(dv[n, :h, :w], img), n
        assert _nonzero(dv[n]) == int(torch.count_nonzero(img)), n                                   # 0 elsewhere
    del src, dv
    # l3c_pack_streams: a slot of 2^32 - 4 bytes (the largest out_cap) whose stream is longer, copied to a byte
    # offset past 2^32 of the same allocation; two small streams beside it
    cap = 2 ** 32 - 4
    for a in range(0, cap, CHUNK):
        b = min(a + CHUNK, cap)
        big[a:b] = _pattern(torch.arange(a, b, device='cuda'), 7)
    big[cap:].fill_(CANARY_BYTE)
    d0 = 2 ** 32 + 1
    outs = np.array([big.data_ptr(), big.data_ptr() + 12, big.data_ptr() + 64], np.uint64)
    caps = np.array([cap, 8, 16], np.uint32)
    lens = np.array([2 ** 32 - 1, 9, 5], np.uint32)
    offs = np.array([d0, d0 + cap + 2, d0 + cap + 13], np.uint64)
    assert int(offs[-1]) + 5 < total
    descs = _enc_descs(outs, caps)
    lens_dev, offs_dev = _dev(lens), _dev(offs)
    _ok(lib.l3c_pack_streams(ctypes.c_void_p(descs.data_ptr()), ctypes.c_void_p(lens_dev.data_ptr()),
                             ctypes.c_void_p(offs_dev.data_ptr()), 3, ctypes.c_void_p(big.data_ptr()), _stream()))
    _guards_intact(buf, 'pack_streams')
    assert bool((big[cap:d0] == CANARY_BYTE).all())
    for a in range(0, cap, CHUNK):
        b = min(a + CHUNK, cap)
        assert torch.equal(big[d0 + a:d0 + b], _pattern(torch.arange(a, b, device='cuda'), 7)), a
    tail = big[d0 + cap:].cpu().numpy()
    want = np.full(len(tail), CANARY_BYTE, np.uint8)
    want[2:10] = big[12:20].cpu().numpy()
    want[13:18] = big[64:69].cpu().numpy()
    assert np.array_equal(tail, want)


@gpu
def test_lut_intervals_past_2_to_the_31_symbols(big_memory):
    lib = _lib()
    n = 2 ** 31 + 37                                       # sym 2 GiB, intervals 8 GiB: 10.0 GiB in all
    sym = torch.empty(n, dtype=torch.uint8, device='cuda')
    for a in range(0, n, CHUNK):
        b = min(a + CHUNK, n)
        sym[a:b] = _pattern(torch.arange(a, b, device='cuda'), 3)
    lut = _codec_lut(256)
    buf, iv = _alloc_guarded(4 * n)
    _ok(lib.l3c_lut_intervals(ctypes.c_void_p(sym.data_ptr()), ctypes.c_void_p(lut.data_ptr()), n,
                              ctypes.c_void_p(iv.data_ptr()), _stream()))
    _guards_intact(buf, 'lut_intervals')
    ivw = iv.view(torch.int32)
    lut64 = lut.long()
    for a in range(0, n, CHUNK):
        b = min(a + CHUNK, n)
        assert torch.equal(ivw[a:b], lut64[sym[a:b].long()].to(torch.int32)), a
