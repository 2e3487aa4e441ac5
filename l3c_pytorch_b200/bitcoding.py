"""Bitcoding: encode an image to a `.l3c` file and decode it back -- the reference's API
(/root/reference/src/bitcoding/bitcoding.py:39-161), byte-compatible container, on top of the
batched sm_90a pipeline of codec.py.

Kept from the reference: `Bitcoding(blueprint, times, compare_with_theory)`, `encode(img, pout) ->
bpsp` (int64 CHW/1CHW image; asserts `pout` does not exist; crops -> `pout.part{i}`; bpsp is
file bytes * 8 / PADDED sub-pixels, crops combined weighted by unpadded H*W, :63-71,108-110),
`decode(pin) -> int64 1CHW`, the helper functions for the header fields and the magic separator.

Added (H100-first): `encode_batch` / `decode_batch` for many images per call.  Where the codec supports ragged
batches (f16, learned bottlenecks, reference layout: BatchCodec.ragged_unsupported) images of any sizes share one
network pass and one range-coder launch (DESIGN §4.6); elsewhere images are grouped by shape.
"""
import os

import numpy as np
import torch

from . import auto_crop, pad, part_suffix_helper
from .blueprint import MultiscaleBlueprint
from .codec import BatchCodec, MAGIC, parse_container
from .times import NoOp

_MAGIC_VALUE_SEP = MAGIC
SEEK_SUFFIX = '.seek'          # a container's seek index beside it (DESIGN §4.13)

# Largest N * Hmax * Wmax (padded pixels of the batch tensor) coded in one ragged pass: 16 images of up to 768 x 768
# (tools/bench_mixed.py) -- the activations, mixture parameters and CDF rows of such a pass fit an 80 GB GPU.
RAGGED_PASS_PIXELS = 16 * 768 * 768


def plan_passes(shapes, budget=None, max_images=None):
    """shapes: padded (H, W) per image -> lists of image indices, one per ragged pass.  Images are sorted by shape
    (ties in input order) and consecutive ones share a pass while N * Hmax * Wmax stays within `budget` (default
    RAGGED_PASS_PIXELS) and N within `max_images` (default: no limit); an image larger than the budget is a pass of
    its own."""
    budget = RAGGED_PASS_PIXELS if budget is None else budget
    order = sorted(range(len(shapes)), key=lambda i: (tuple(shapes[i]), i))
    passes, cur, hm, wm = [], [], 0, 0
    for i in order:
        h, w = shapes[i]
        nh, nw = max(hm, h), max(wm, w)
        if cur and ((len(cur) + 1) * nh * nw > budget or (max_images is not None and len(cur) >= max_images)):
            passes.append(cur)
            cur, nh, nw = [], h, w
        cur.append(i)
        hm, wm = nh, nw
    if cur:
        passes.append(cur)
    return passes


def _groups(keys):
    """Indices of equal keys -- one group per (shape, padding tuple) where ragged passes are unsupported -- in
    order of first appearance."""
    groups = {}
    for i, k in enumerate(keys):
        groups.setdefault(k, []).append(i)
    return list(groups.values())


class Bitcoding(object):
    def __init__(self, blueprint, times=NoOp, compare_with_theory=False, tile=None, recursive=0, crop=True):
        """tile = (th, tw): write TILED containers (codec.ContainerLayout): every channel plane of every scale is
        cut into tiles coded as independent streams -- thousands of streams per batch instead of 18 per image,
        so encode and decode are no longer bound by one warp's serial chain.  Not readable by the reference and a
        few bytes per tile larger; decode() / decode_batch() recognise either layout.  Default: the reference's
        byte-compatible `.l3c` layout.
        recursive = R > 0 (RGB baselines only): write RECURSIVE containers (DESIGN §4.7): the last trained scale
        codes its own bicubic thumbnails R more times and only the 1 / 2**(num_scales + R) thumbnail is left for
        the uniform prior; images are padded to multiples of 2**(num_scales + R).  Not readable by the reference;
        decode() / decode_batch() read R from the file.  ValueError for anything but a non-negative int, and for
        R > 0 on an L3C model.
        crop = False (tiled containers only): encode() writes ONE container for an image of any size instead of the
        reference's auto-crop into `pout.partN` files (DESIGN §4.10); decode() of a large tiled container runs in
        bands of tile rows, and decode_region() reads any crop of it.  ValueError without tile=: the crops of the
        reference layout are part of its format, and its serial streams could not be decoded in bands."""
        if not crop and tile is None:
            raise ValueError('crop=False needs tile=(th, tw): the reference layout codes large images as crops')
        self.crop = bool(crop)
        self.blueprint = blueprint
        self.compare_with_theory = compare_with_theory
        self.times = times
        self.tile = tile
        self.codec = BatchCodec(blueprint)
        self.recursive = self.codec.check_recursive(recursive)

    def pad_factor(self):
        """Images are padded to multiples of this: 2**(num_scales + R)."""
        return 2 ** (self.blueprint.net.config_ms.num_scales + self.recursive)

    # ------------------------------------------------------------------------------------------
    def _device(self):
        return self.blueprint.device

    def _prepare(self, img, quiet=False):
        """-> (uint8 [1,3,H',W'] padded, on device; padding tuple)."""
        factor = self.pad_factor()
        if img.dim() == 3:
            img = img.unsqueeze(0)
        _, _, H, W = img.shape
        padding_tuple = (0, 0, 0, 0)
        if H % factor != 0 or W % factor != 0:
            if not quiet:
                print(f'*** INFO: image shape ({H}X{W}) not divisible by {factor}, will pad.')
            img, padding_tuple = pad.pad(img, fac=factor, mode=MultiscaleBlueprint.get_padding_mode())
        return img.to(torch.uint8).to(self._device()).contiguous(), padding_tuple

    def _passes(self, prepared):
        """Index groups of `prepared` [(uint8 [1,3,H,W], padding tuple)] coded in one pass each: ragged passes
        (plan_passes) where the codec supports them, else one group per (shape, padding tuple)."""
        if self.codec.ragged_unsupported(self.tile) is None:
            return plan_passes([tuple(t.shape[-2:]) for (t, _) in prepared])
        return _groups((tuple(t.shape), pt) for (t, pt) in prepared)

    def _begin_pass(self, prepared, idxs, seek=None):
        """Enqueue the encode of prepared[idxs] as one batch on the current stream -> codec EncodeJob.  Images of
        different shapes are placed top-left in a zero batch of the largest extent (a ragged batch)."""
        imgs = [prepared[i][0] for i in idxs]
        pts = [prepared[i][1] for i in idxs]
        shapes = [tuple(t.shape[-2:]) for t in imgs]
        if all(sh == shapes[0] for sh in shapes):
            batch = torch.cat(imgs, 0) if len(imgs) > 1 else imgs[0]
            pt = pts[0] if all(p == pts[0] for p in pts) else pts
            return self.codec.encode_begin(batch, pt, tile=self.tile, recursive=self.recursive, seek=seek)
        Hb, Wb = max(h for (h, _) in shapes), max(w for (_, w) in shapes)
        batch = torch.zeros(len(imgs), 3, Hb, Wb, dtype=torch.uint8, device=self._device())
        for k, t in enumerate(imgs):
            batch[k, :, :t.shape[2], :t.shape[3]] = t[0]
        return self.codec.encode_begin(batch, pts, tile=self.tile, extents=shapes, recursive=self.recursive, seek=seek)

    def encode(self, img, pout, seek=None):
        """img: int64 (or uint8) CHW / 1CHW tensor with values 0..255; writes `pout`; returns bpsp.
        seek = K (reference layout): also writes the container's seek index (DESIGN §4.13) to `pout + '.seek'`, and
        for auto-crops `pout.partN.seek` beside every part."""
        assert not os.path.isfile(pout)
        assert seek is None or not os.path.isfile(pout + SEEK_SUFFIX)
        if len(img.shape) == 3:
            img = img.unsqueeze(0)
        assert len(img.shape) == 4 and img.shape[0] == 1 and img.shape[1] == 3, img.shape
        assert img.dtype in (torch.int64, torch.uint8), img.dtype

        if self.crop and auto_crop.needs_crop(img):
            print('Need to encode individual crops!')
            combinator = auto_crop.CropLossCombinator()
            crops = list(auto_crop.iter_crops(img))
            pouts = [pout + part_suffix_helper.make_part_suffix(i) for i in range(len(crops))]
            # the reference recurses into encode() per part and asserts on every part path
            # (bitcoding.py:57,63-71); stale higher-numbered parts of an earlier encode would be picked
            # up by decode() and stitched into a wrong image
            stale = [q for q in part_suffix_helper.existing_parts(pout) if q not in pouts]
            assert not any(os.path.isfile(q) for q in pouts) and not stale, \
                'part files of {} already exist: {}'.format(pout, [q for q in pouts if os.path.isfile(q)] + stale)
            assert seek is None or not any(os.path.isfile(q + SEEK_SUFFIX) for q in pouts), \
                'seek indexes of the parts of {} already exist'.format(pout)
            bpsps = self._encode_many(crops, pouts, seek)
            for crop, bpsp in zip(crops, bpsps):
                combinator.add(bpsp, np.prod(crop.shape[-2:]))
            return combinator.get_bpsp()
        return self._encode_many([img], [pout], seek)[0]

    def _encode_many(self, imgs, pouts, seek=None):
        """Images are coded in ragged passes (any mix of shapes, plan_passes) where the codec supports them;
        otherwise, and with compare_with_theory, images of equal (padded) shape are coded as one batch."""
        prepared = [self._prepare(im) for im in imgs]
        if seek is not None or (not self.compare_with_theory and self.codec.ragged_unsupported(self.tile) is None):
            res = self._encode_prepared(prepared, seek).finish()
            for i, dta in enumerate(res[0]):
                with open(pouts[i], 'wb') as f:
                    f.write(dta)
                if seek is not None:
                    with open(pouts[i] + SEEK_SUFFIX, 'wb') as f:
                        f.write(res[2][i])
            return res[1]
        bpsps = [None] * len(imgs)
        for idxs in _groups((tuple(t.shape), pt) for (t, pt) in prepared):
            batch = torch.cat([prepared[i][0] for i in idxs], 0)
            pt = prepared[idxs[0]][1]
            # a large tiled batch is encoded in bands (DESIGN §4.10), which needs encode_begin to run the networks;
            # compare_with_theory needs every scale's parameters and keeps the whole-image forward
            banded = not self.compare_with_theory and self.codec.encode_banded(batch.shape, self.tile)
            with self.times.run('[-] encode forwardpass'):
                # without --compare_theory nobody reads the parameter tensors: the probability heads emit the
                # coding intervals directly (f16 mode; MultiscaleNetwork.forward(intervals_of=...))
                out = None if banded else self.blueprint.forward(batch, self.recursive) if self.compare_with_theory \
                    else self.blueprint.forward_for_coding(batch, self.recursive)
            if self.compare_with_theory:
                with self.times.run('[-] get loss'):
                    loss_out = self.blueprint.get_loss(out)
            with self.times.run('[-] entropy coding'):
                datas, info = self.codec.encode_batch(batch, pt, out=out, tile=self.tile, recursive=self.recursive)
            num_subpixels = int(np.prod(batch.shape[1:]))
            for k, i in enumerate(idxs):
                with open(pouts[i], 'wb') as f:
                    f.write(datas[k])
                bpsps[i] = len(datas[k]) * 8 / num_subpixels
            if self.compare_with_theory:
                total = sum(len(d) for d in datas) * 8 / (num_subpixels * len(idxs))
                # recursive containers code every scale of recursive_bpsps (the last one under the uniform prior)
                theory = loss_out.recursive_bpsps if self.recursive else loss_out.nonrecursive_bpsps
                print('Bitrates:\ntheory:  {} => {:.3f}\nactual:  => {:.3f}'.format(
                    ' | '.join('{:.3f}'.format(b) for b in theory), sum(theory), total))
        return bpsps

    def decode(self, pin, _recurse_part=True):
        """-> decoded image, int64 1CHW (on the GPU).  A seek index beside a file (`pin + '.seek'`, `pin.partN.seek`)
        is used (decode_batch(seeks=)); ValueError naming the index when it does not match its file."""
        if _recurse_part and part_suffix_helper.contains_part_suffix(pin):
            paths = part_suffix_helper.iter_part_suffixes(pin)
            parts = self._decode_many(paths)
            print(f'Stitching {len(parts)} parts...')
            return auto_crop.stitch(parts)
        return self._decode_many([pin])[0]

    def _decode_many(self, paths):
        from . import seek as _seek
        datas, seeks = [], []
        for p in paths:
            with open(p, 'rb') as f:
                datas.append(f.read())
            sk = None
            if os.path.isfile(p + SEEK_SUFFIX):
                with open(p + SEEK_SUFFIX, 'rb') as f:
                    sk = f.read()
                try:
                    _seek.parse_index(sk, datas[-1])
                except ValueError as e:
                    raise ValueError('%s: %s' % (p + SEEK_SUFFIX, e))
            seeks.append(sk)
        return self.decode_batch(datas, seeks if any(sk is not None for sk in seeks) else None)

    # ------------------------------------------------------------------------------------------
    # H100-first batch API
    def encode_batch(self, imgs_u8, seek=None):
        """imgs_u8: uint8 [N,3,H,W] (any device), or a list / tuple of uint8 [3,H,W] / [1,3,H,W] images of any
        sizes -> (list of container bytes, bpsp list) in input order.  seek = K (reference layout): -> (containers,
        bpsps, seek indexes), the containers the same bytes (BatchCodec.encode_begin)."""
        return self.encode_batch_begin(imgs_u8, seek=seek).finish()

    def _encode_prepared(self, prepared, seek=None):
        """Enqueue the passes of `prepared` on the current stream -> _ListEncodeJob."""
        jobs = [(idxs, self._begin_pass(prepared, idxs, seek)) for idxs in self._passes(prepared)]
        return _ListEncodeJob(jobs, [int(np.prod(t.shape[1:])) for (t, _) in prepared], seek is not None)

    def encode_batch_begin(self, imgs_u8, stream=None, seek=None):
        """Asynchronous encode_batch: enqueues the upload and the whole GPU side on `stream` (default:
        the current stream) and returns a job at once; job.finish() -> (containers, bpsps).  With
        `stream=self.side_stream(N)` the encode runs beside a decode_batch of another batch: the
        decode is bound by the serial range decoder and leaves most of the GPU idle.

        A list / tuple of images: each is padded on its own (as encode() does) and the images are coded in ragged
        passes (plan_passes): one network pass and one range-coder launch per pass, containers byte-identical to
        coding each image alone.  Where the codec does not support ragged batches (ragged_unsupported) images of
        different padded shapes raise NotImplementedError."""
        if isinstance(imgs_u8, (list, tuple)):
            stream = stream if stream is not None else torch.cuda.current_stream(self._device())
            with torch.cuda.stream(stream):
                prepared = [self._prepare(im, quiet=True) for im in imgs_u8]
                why = self.codec.ragged_unsupported(self.tile)
                if why is not None and len({tuple(t.shape) for (t, _) in prepared}) > 1:
                    raise NotImplementedError(why)
                return self._encode_prepared(prepared, seek)
        pt = pad.padding_tuple(imgs_u8.shape[-2], imgs_u8.shape[-1], self.pad_factor())
        stream = stream if stream is not None else torch.cuda.current_stream(self._device())
        with torch.cuda.stream(stream):
            x = imgs_u8.to(self._device(), non_blocking=True)
            if any(pt):
                x = torch.nn.functional.pad(x, pt, 'constant')
            x = x.contiguous()
            job = self.codec.encode_begin(x, pt, tile=self.tile, recursive=self.recursive, seek=seek)
        N = x.shape[0]
        return _ListEncodeJob([(list(range(N)), job)], [int(np.prod(x.shape[1:]))] * N, seek is not None)

    def side_stream(self, n_images, n_lanes=1):
        """Stream for encode_batch_begin() calls that should overlap decode_batch calls of `n_images` each."""
        return self.codec.encode_stream(self._device(), 3 * n_images, n_lanes)

    def decode_lanes(self, n_images, n_lanes=2):
        """Stream sets for `n_lanes` decode_batch calls in flight at the same time (codec.BatchCodec.lanes):
        `with torch.cuda.stream(lane.main): dec = bc.decode_batch(datas, lane=lane)` returns at once; the
        decode of one batch is bound by the serial chain of its range coder and leaves most of the GPU idle."""
        return self.codec.lanes(self._device(), 3 * n_images, n_lanes)[0]

    def decode_batch(self, datas, seeks=None, lane=None):
        """list of container bytes (any mix of shapes) -> list of int64 1CHW tensors (GPU).  Ragged passes
        (plan_passes) where the codec supports them, else one pass per shape.  seeks: a seek index (bytes) or None
        per container: the streams of an indexed container decode as parallel segments (DESIGN §4.13)."""
        if seeks is not None and len(seeks) != len(datas):
            raise ValueError('%d seek indexes for %d containers' % (len(seeks), len(datas)))
        from .codec import parse_container, container_tile
        parsed = [parse_container(d) for d in datas]
        if self.codec.ragged_unsupported(container_tile(datas[0]) if datas else None) is None and \
                all(len(p[1]) and container_tile(d) is None for p, d in zip(parsed, datas)):
            passes = plan_passes([p[1][-1][1:3] for p in parsed])
        else:
            passes = _groups((tuple((C, H, W) for (C, H, W, _) in scales), pt) for (pt, scales) in parsed)
        outs = [None] * len(datas)
        for idxs in passes:
            S, _ = self.codec.decode_batch([datas[i] for i in idxs], to_host=False, lane=lane,
                                           seeks=None if seeks is None else [seeks[i] for i in idxs])
            for k, i in enumerate(idxs):
                pt, scales = parsed[i]
                H, W = scales[-1][1:3] if scales else S.shape[-2:]
                img = S[k:k + 1, :, :H, :W].long()
                if any(pt):
                    img = pad.undo_pad(img, *pt)
                outs[i] = img
        return outs

    def seek_index(self, datas, every=None):
        """Seek indexes (sidecar bytes, DESIGN §4.13) of reference-layout containers, e.g. files the reference or an
        earlier encode wrote, from one serial decode (BatchCodec.seek_index); every = K, default 4096."""
        from . import seek as _seek
        every = _seek.DEFAULT_EVERY if every is None else every
        parsed = [parse_container(d) for d in datas]
        if self.codec.ragged_unsupported() is None and all(len(p[1]) for p in parsed):
            passes = plan_passes([p[1][-1][1:3] for p in parsed])
        else:
            passes = _groups(tuple((C, H, W) for (C, H, W, _) in scales) for (_, scales) in parsed)
        outs = [None] * len(datas)
        for idxs in passes:
            for i, sk in zip(idxs, self.codec.seek_index([datas[i] for i in idxs], every)):
                outs[i] = sk
        return outs

    def decode_region(self, data, region, level=0, lane=None, seek=None):
        """One region of a tiled container, or of a reference-layout one with its seek index `seek` (sidecar bytes;
        DESIGN §4.8, §4.13 "Regions") -> int64 1CHW tensor (GPU), equal bit for bit to the same crop of
        decode_batch([data])[0].  region = (y, x, h, w): at level 0 in the coordinates decode() returns (the unpadded
        image); at level k >= 1 (RGB baselines) in those of the stored scale-k thumbnail.  Only the tile streams (the
        segments of the row bands) and decoder windows the region depends on are decoded.  ValueError, before any GPU
        work, for a reference-layout container without an index, an index of another container, a container this model
        did not write, an empty region or one outside the image, and a level that does not exist.  lane: as in
        decode_batch (BatchCodec.lanes; the caller has made `lane.main` current)."""
        return self.decode_regions([data], [region], [level], lane=lane, seeks=None if seek is None else [seek])[0]

    def decode_regions(self, datas, regions, levels=None, lane=None, seeks=None):
        """decode_region for many (container, region[, level]) pairs -> list of int64 1CHW tensors in input order.
        seeks: None, or one seek index (bytes) or None per container.  In f16 and f16x2 the pairs of one level and tile
        size (or of indexed reference-layout containers) decode in one pass, whatever the shapes of their regions and
        images; in tf32 / fp32 pairs whose plans have equal window shapes share one pass and the others run one after
        another (BatchCodec.decode_regions)."""
        return [S.long() for S in self.codec.decode_regions(datas, regions, levels, lane=lane, seeks=seeks)]

    def decode_region_file(self, pin, region, level=0, lane=None):
        """decode_region of a file: a tiled container as it is; a reference-layout one with its seek index
        `pin + '.seek'`; an image the reference stored in parts (`pin.partN`, or `pin` when only the parts exist) from
        the parts the region touches, each with its own `.seek` index, in one decode_regions call, the crops stitched
        (auto_crop.part_rects).  -> int64 1CHW tensor (GPU), the same crop of decode(pin).  ValueError, before any GPU
        work, naming the file, for a missing or mismatched index and for tiled parts (a large tiled image is one
        container, crop=False); for level > 0 of an image in parts; and for what decode_regions refuses."""
        from . import seek as _seek
        from .codec import container_tile

        def read(p):
            with open(p, 'rb') as f:
                return f.read()

        def index_of(p, data):
            if not os.path.isfile(p + SEEK_SUFFIX):
                raise ValueError('{} is a reference-layout file: a region decode needs its seek index {} '
                                 '(`idx {}`)'.format(p, p + SEEK_SUFFIX, p))
            sk = read(p + SEEK_SUFFIX)
            try:
                _seek.parse_index(sk, data)
            except ValueError as e:
                raise ValueError('%s: %s' % (p + SEEK_SUFFIX, e))
            return sk

        if not os.path.isfile(pin) and os.path.isfile(pin + part_suffix_helper.make_part_suffix(0)):
            pin = pin + part_suffix_helper.make_part_suffix(0)
        if not part_suffix_helper.contains_part_suffix(pin):
            data = read(pin)
            if container_tile(data) is not None:
                return self.decode_region(data, region, level, lane)
            return self.decode_region(data, region, level, lane, seek=index_of(pin, data))
        paths = part_suffix_helper.iter_part_suffixes(pin)
        datas = [read(p) for p in paths]
        for p, d in zip(paths, datas):
            if container_tile(d) is not None:
                raise ValueError('{} is a tiled part: region decode of part files reads reference-layout parts with '
                                 'seek indexes (a large tiled image is one container, crop=False)'.format(p))
        if level != 0:
            raise ValueError('level {}: the parts of {} are crops of the image, not of its thumbnails'.format(
                level, pin))
        seeks = [index_of(p, d) for p, d in zip(paths, datas)]
        shapes = []
        for d in datas:
            (left, right, top, bottom), scales = parse_container(d)
            if not scales:
                raise ValueError('an empty part container')
            shapes.append((scales[-1][1] - top - bottom, scales[-1][2] - left - right))
        rects = auto_crop.part_rects(shapes)
        Ht, Wt = max(r[0] + r[2] for r in rects), max(r[1] + r[3] for r in rects)
        if len(region) != 4:
            raise ValueError('region must be (y, x, h, w), got %r' % (region,))
        y, x, h, w = (int(v) for v in region)
        if h < 1 or w < 1:
            raise ValueError('empty region %r' % (tuple(region),))
        if y < 0 or x < 0 or y + h > Ht or x + w > Wt:
            raise ValueError('region %r lies outside the %dx%d image' % (tuple(region), Ht, Wt))
        sel, subs = [], []
        for i, (py, px, ph, pw) in enumerate(rects):
            y0, x0, y1, x1 = max(y, py), max(x, px), min(y + h, py + ph), min(x + w, px + pw)
            if y0 < y1 and x0 < x1:
                sel.append(i)
                subs.append((y0 - py, x0 - px, y1 - y0, x1 - x0))
        pieces = self.decode_regions([datas[i] for i in sel], subs, lane=lane, seeks=[seeks[i] for i in sel])
        out = torch.empty(1, 3, h, w, dtype=torch.int64, device=self._device())
        for i, (sy, sx, sh, sw), piece in zip(sel, subs, pieces):
            oy, ox = rects[i][0] + sy - y, rects[i][1] + sx - x
            out[:, :, oy:oy + sh, ox:ox + sw] = piece
        return out

    def update_region(self, data, pos, patch):
        """A tiled container with the pixels at pos = (y, x) replaced by `patch` (DESIGN §4.12) -> the new container
        bytes, byte-identical to encoding the edited image.  pos is in the coordinates decode() returns (the unpadded
        image); patch: uint8 or int64 [3, h, w] or [1, 3, h, w], values 0..255, on any device.  Only the tile streams
        the edit can change are re-encoded, from a bounded window of the image (BatchCodec.update_region).
        ValueError, before any GPU work, for the reference layout, a container this model did not write, the RGB
        baselines, an empty patch or one not in the image, and a patch that is not 3-channel."""
        return self.codec.update_region(data, pos, patch)

    def update_regions(self, datas, edits):
        """update_region for many containers and many edits each: edits[i] = [(pos, patch)] for datas[i], applied in
        list order, so a later patch overwrites an earlier one where they overlap -> the new container bytes in input
        order, each byte-identical to encoding its decoded image with every patch pasted in order.  An empty edit list
        returns the container unchanged.  Edits whose windows do not meet are re-encoded from their own windows, the
        others from the window of their bounding rectangle; every container is parsed and uploaded once and spliced on
        the GPU (BatchCodec.update_regions, which records what ran in updates_counts).  ValueError, before any GPU
        work, for every refusal of update_region, naming the container and the edit."""
        return self.codec.update_regions(datas, edits)

    def update_regions_begin(self, datas, edits, lane=None):
        """update_regions without a host wait until job.finish(), which returns the same bytes (DESIGN §4.12, "Serving
        updates").  The parse, the plan and every ValueError of update_regions happen here, before any GPU work; the
        rest is queued on the current stream and the new containers are laid out and spliced on the GPU.  job.counts
        holds the call's per-container statistics.  lane: one of decode_lanes(...), as in decode_regions -- the caller
        has made `lane.main` current, and the old-pixel decodes use the lane's decoder streams, so updates run beside
        the region decodes and decode_batch calls of other lanes."""
        return self.codec.update_regions_begin(datas, edits, lane=lane)


class _ListEncodeJob:
    """encode_batch_begin: the codec jobs of its passes (one for a batch tensor); finish() -> (containers, bpsps) in
    input order."""

    def __init__(self, jobs, nsubs, seek=False):
        self.jobs, self.nsubs, self.seek = jobs, nsubs, seek

    def finish(self):
        """-> (containers, bpsps), and their seek indexes third when the encode records them"""
        datas = [None] * len(self.nsubs)
        seeks = [None] * len(self.nsubs)
        for idxs, job in self.jobs:
            d, info = job.finish(to_host=True)
            for k, i in enumerate(idxs):
                datas[i] = d[k]
                if self.seek:
                    seeks[i] = info['seeks'][k]
        bpsps = [len(d) * 8 / n for d, n in zip(datas, self.nsubs)]
        return (datas, bpsps, seeks) if self.seek else (datas, bpsps)


# --- header field helpers (bitcoding.py:326-375), little-endian -------------------------------
def write_bytes(f, ts, xs):
    for t, x in zip(ts, xs):
        f.write(t(x).tobytes())


def read_bytes(f, ts):
    return [np.frombuffer(f.read(t().itemsize), t, count=1)[0] for t in ts]


def write_shape(shape, fout):
    assert len(shape) == 4 and shape[0] == 1, shape
    C, H, W = shape[1:]
    assert C < 2 ** 8 and H < 2 ** 16 and W < 2 ** 16, shape
    write_bytes(fout, [np.uint8, np.uint16, np.uint16], (C, H, W))
    return 5


def read_shapes(fin):
    return tuple(map(int, read_bytes(fin, [np.uint8, np.uint16, np.uint16])))


def write_num_bytes_encoded(num_bytes, fout):
    assert num_bytes < 2 ** 32
    write_bytes(fout, [np.uint32], [num_bytes])
    return 2


def read_num_bytes_encoded(fin):
    return int(read_bytes(fin, [np.uint32])[0])


def write_padding_tuple(padding_tuple, fout):
    assert len(padding_tuple) == 4
    write_bytes(fout, [np.uint16] * 4, padding_tuple)


def read_padding_tuple(fin):
    return tuple(map(int, read_bytes(fin, [np.uint16] * 4)))
