"""Adaptive cropping of large images into independently coded parts
(/root/reference/src/auto_crop.py:44-152): an image with H*W above the threshold is split 2x2
(floor halves), recursively and depth-first (TL, TR, BL, BR); `stitch` inverts it.

The threshold default (2000*1500) and the AC_NEEDS_CROP_DIM override are the reference's; on a
80 GB H100 the crops are not needed for memory any more, but they are part of the file format
(one `.partN` file per crop), so they are kept.  Crops of one image are coded as ONE batch."""
import math
import os

import torch

_DEFAULT = '2000,1500'


def _threshold():
    spec = os.environ.get('AC_NEEDS_CROP_DIM', _DEFAULT)
    out = 1
    for tok in spec.split(','):
        out *= int(tok)
    return out


def _check(img):
    if len(img.shape) != 4 or img.shape[1] != 3:
        raise ValueError('Expected BCHW image, got {}'.format(tuple(img.shape)))


def needs_crop(img, needs_crop_dim=None):
    _check(img)
    H, W = img.shape[-2:]
    return H * W > (_threshold() if needs_crop_dim is None else needs_crop_dim)


def _quadrants(img):
    H, W = img.shape[-2:]
    h, w = H // 2, W // 2
    return [img[..., :h, :w], img[..., :h, w:], img[..., h:, :w], img[..., h:, w:]]


def iter_crops(img, needs_crop_dim=None):
    _check(img)
    lim = _threshold() if needs_crop_dim is None else needs_crop_dim
    if not needs_crop(img, lim):
        yield img
        return
    for q in _quadrants(img):
        yield from iter_crops(q, lim)


def _crop_positions(side):
    """crop index (extraction order) -> row-major position in the side x side grid."""
    grid = torch.arange(side * side).reshape(1, 1, side, side).expand(1, 3, side, side)
    return [int(c[0, 0, 0, 0]) for c in iter_crops(grid, 1)]


def stitch(parts):
    side = int(round(math.sqrt(len(parts))))
    if side * side != len(parts):
        raise ValueError('Invalid number of parts {}'.format(len(parts)))
    pos = _crop_positions(side)
    ordered = [None] * len(parts)
    for i, part in enumerate(parts):
        ordered[pos[i]] = part
    rows = [torch.cat(ordered[r * side:(r + 1) * side], dim=3) for r in range(side)]
    return torch.cat(rows, dim=2)


def part_rects(shapes):
    """shapes: (H, W) of every part of an image, unpadded, in `stitch` order (the parts' file order) -> the (y, x, h, w)
    each one covers in the stitched image.  ValueError for anything `stitch` would not build as a grid: a part count
    that is not the square of a power of two, a grid row whose parts differ in height or a grid column whose parts differ in width."""
    shapes = [(int(h), int(w)) for (h, w) in shapes]
    side = math.isqrt(len(shapes))
    if not shapes or side * side != len(shapes) or side & (side - 1):
        # iter_crops splits in quadrants: a grid is 2^k x 2^k parts (stitch fails on any other square)
        raise ValueError('Invalid number of parts {}'.format(len(shapes)))
    pos = _crop_positions(side)
    grid = [None] * len(shapes)
    for i, p in enumerate(pos):
        grid[p] = shapes[i]
    heights = [{grid[r * side + c][0] for c in range(side)} for r in range(side)]
    widths = [{grid[r * side + c][1] for r in range(side)} for c in range(side)]
    for r, hs in enumerate(heights):
        if len(hs) != 1:
            raise ValueError('parts of grid row {} have different heights {}'.format(r, sorted(hs)))
    for c, ws in enumerate(widths):
        if len(ws) != 1:
            raise ValueError('parts of grid column {} have different widths {}'.format(c, sorted(ws)))
    ys, xs = [0], [0]
    for hs, ws in zip(heights, widths):
        ys.append(ys[-1] + hs.pop())
        xs.append(xs[-1] + ws.pop())
    return [(ys[p // side], xs[p % side]) + shapes[i] for i, p in enumerate(pos)]


class CropLossCombinator(object):
    """bpsp of several crops -> one bpsp, weighted by crop size (auto_crop.py:139-152)."""

    def __init__(self):
        self._bits = 0.
        self._subpixels = 0

    def add(self, bpsp, num_subpixels_crop):
        self._bits += bpsp * num_subpixels_crop
        self._subpixels += num_subpixels_crop

    def get_bpsp(self):
        assert self._subpixels > 0
        return self._bits / self._subpixels
