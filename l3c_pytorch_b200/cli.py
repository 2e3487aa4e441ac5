"""Single-image command line: the encode/decode half of the reference's `l3c.py`
(/root/reference/src/l3c.py:74-129) on the H100 path.

    python -m l3c_pytorch_b200.cli --config cr --ckpt CKPT.pt enc IMG OUT.l3c [--overwrite] [--seek K]
    python -m l3c_pytorch_b200.cli --config cr --ckpt CKPT.pt idx IN.l3c [--every K]
    python -m l3c_pytorch_b200.cli --config cr --ckpt CKPT.pt dec IN.l3c OUT.png
    python -m l3c_pytorch_b200.cli --config cr_rgb_shared --ckpt CKPT.pt enc IMG OUT.l3c --recursive auto
    python -m l3c_pytorch_b200.cli --config cr --ckpt CKPT.pt dec IN.l3c OUT.png --region Y,X,H,W [--level K]
    python -m l3c_pytorch_b200.cli --config cr --ckpt CKPT.pt upd IN.l3c PATCH.png Y,X OUT.l3c [--overwrite]
                                                                  [--edit PATCH2.png Y2,X2 ...]

`enc --seek K` also writes OUT.l3c.seek, the file's seek index (DESIGN §4.13): the range coder's state every K
symbols, with which `dec` decodes every stream as parallel segments; the .l3c file itself is unchanged.  `idx`
writes the index of an existing file (one written by the reference, say).  With it, `dec --region` reads a crop of
a reference-layout file, or of an image stored in `.partN` parts, from the row bands the crop needs.

`upd --edit PATCH.png Y,X` (repeatable) applies more edits after the positional one, in order, in one call that
re-encodes every tile the edits reach once (DESIGN §4.12, "Batches of updates").

`--ckpt` is a checkpoint as written by the reference's Saver (`torch.save({'net': state_dict})`,
helpers/saver.py:168); the module tree here has the same parameter names, so it loads strict.
Without `--ckpt` the seed-0 default initialisation is used (only useful for testing).
Images larger than 2000x1500 are coded as crops into `OUT.l3c.part{i}` exactly as the reference does, unless
`enc --tile TH,TW` writes one tiled file for the whole image (DESIGN §4.10):

    python -m l3c_pytorch_b200.cli --config cr --ckpt CKPT.pt enc BIG.png OUT.l3c --tile 64,64
"""
import argparse
import os
import sys

import numpy as np
import torch

from . import codec
from .bitcoding import SEEK_SUFFIX


class EncodeError(Exception):
    pass


class DecodeError(Exception):
    pass


def load_blueprint(config_name, ckpt=None, precision=None, device='cuda:0'):
    from . import config, engine
    from .blueprint import MultiscaleBlueprint
    if precision:
        engine.set_conv_precision(precision)
    torch.manual_seed(0)
    bp = MultiscaleBlueprint(config.ms_config(config_name), device=device)
    bp.set_eval()
    if ckpt:
        state = torch.load(ckpt, map_location='cpu')
        bp.net.load_state_dict(state['net'] if 'net' in state else state, strict=True)   # saver.py:184-210
        bp.net.to(bp.device)
    return bp


def read_image(path, max_pixels=None):
    """PIL -> int64 1CHW, alpha dropped (multiscale_tester.py:411-422).  max_pixels: Pillow's decompression-bomb
    limit (Image.MAX_IMAGE_PIXELS) while reading; None keeps Pillow's default."""
    from PIL import Image
    if max_pixels is None:
        img = np.array(Image.open(path))
    else:
        old = Image.MAX_IMAGE_PIXELS
        Image.MAX_IMAGE_PIXELS = max_pixels
        try:
            img = np.array(Image.open(path))
        finally:
            Image.MAX_IMAGE_PIXELS = old
    if img.ndim == 2:
        img = np.stack([img] * 3, -1)
    img = img[..., :3]
    return torch.from_numpy(img).permute(2, 0, 1).unsqueeze(0).long()


def write_image(img_1chw, path):
    from PIL import Image
    assert path.endswith('.png'), 'decoded images are written as PNG (lossless)'
    arr = img_1chw[0].permute(1, 2, 0).to(torch.uint8).cpu().numpy()
    Image.fromarray(arr).save(path)


def encode(bc, img_p, pout, overwrite=False, seek=None):
    if os.path.isfile(pout) or os.path.isfile(pout + '.part0') or os.path.isfile(pout + SEEK_SUFFIX):
        if not overwrite:
            raise EncodeError('{} exists. Consider --overwrite.'.format(pout))
        # the parts and every seek index beside them: a stale index would no longer match its file
        for q in [pout] + [pout + '.part%d' % i for i in range(4096)]:
            if os.path.isfile(q + SEEK_SUFFIX):
                os.remove(q + SEEK_SUFFIX)
            if os.path.isfile(q):
                os.remove(q)
            elif q != pout:
                break
    # a tiled file holds one image of any size (DESIGN §4.10): read up to the largest plane the kernels index
    img = read_image(img_p, codec.MAX_PLANE_PIXELS if bc.tile is not None else None)
    try:
        bpsp = bc.encode(img, pout) if seek is None else bc.encode(img, pout, seek=seek)
    except ValueError as err:
        raise EncodeError(str(err))
    print('Encoded {} -> {}: {:.4f} bpsp'.format(img_p, pout, bpsp))
    return bpsp


def decode(bc, pin, png_out):
    if not os.path.isfile(pin):
        if os.path.isfile(pin + '.part0'):
            pin = pin + '.part0'
        else:
            raise DecodeError('File not found: {}'.format(pin))
    try:
        img = bc.decode(pin)
    except ValueError as err:
        raise DecodeError(str(err))
    write_image(img, png_out)
    print('Decoded {} -> {}'.format(pin, png_out))


def index(bc, pin, every=None, overwrite=False):
    """writes the seek index of pin (and of its .partN files) beside it -> the paths written"""
    from . import part_suffix_helper
    paths = [pin] if os.path.isfile(pin) else part_suffix_helper.existing_parts(pin)
    if not paths:
        raise DecodeError('File not found: {}'.format(pin))
    if not overwrite and any(os.path.isfile(q + SEEK_SUFFIX) for q in paths):
        raise EncodeError('{} exists. Consider --overwrite.'.format(paths[0] + SEEK_SUFFIX))
    datas = []
    for q in paths:
        with open(q, 'rb') as f:
            datas.append(f.read())
    try:
        seeks = bc.seek_index(datas, every)
    except ValueError as err:
        raise DecodeError(str(err))
    for q, sk in zip(paths, seeks):
        with open(q + SEEK_SUFFIX, 'wb') as f:
            f.write(sk)
        print('Indexed {} -> {}: {} bytes'.format(q, q + SEEK_SUFFIX, len(sk)))
    return [q + SEEK_SUFFIX for q in paths]


def recursive_of(args, config_ms):
    """R of `enc --recursive N|auto` (harness.parse_recursive_flag: 0 for L3C configs); 0 for `dec`."""
    from .harness import parse_recursive_flag
    return parse_recursive_flag(getattr(args, 'recursive', '0'), config_ms) if args.mode == 'enc' else 0


def build_parser():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument('--config', default='cr', help='cr | cr_rgb_shared | cr_rgb or a path to a .cf file')
    p.add_argument('--ckpt', default=None, help="checkpoint with {'net': state_dict}")
    p.add_argument('--precision', default=None, choices=['fp32', 'tf32', 'f16', 'f16x2'],
                   help='conv mode (default fp32; encoder and decoder must use the same one)')
    sub = p.add_subparsers(dest='mode', required=True)
    e = sub.add_parser('enc')
    e.add_argument('img')
    e.add_argument('out')
    e.add_argument('--overwrite', action='store_true')
    e.add_argument('--recursive', default='0', metavar='N|auto',
                   help='RGB baselines: code the last scale N more times on its own thumbnails (auto: 3 for '
                        'cr_rgb_shared); a recursive file, not readable by the reference.  Ignored for L3C.')
    e.add_argument('--tile', default=None, type=parse_tile, metavar='TH,TW',
                   help='write ONE tiled file (tiles of TH x TW coded as independent streams) for an image of any '
                        'size, no .partN crops; `dec` decodes it in bands and `dec --region` reads crops of it.  Not '
                        'readable by the reference')
    e.add_argument('--seek', default=None, type=int, metavar='K',
                   help='also write OUT.seek, a seek index of the coder state every K symbols (a multiple of 32; '
                        '4096 is a good default) with which `dec` decodes the streams in parallel')
    x = sub.add_parser('idx', help='write IN.l3c.seek, the seek index of an existing reference-layout file')
    x.add_argument('inp')
    x.add_argument('--every', default=None, type=int, metavar='K', help='symbols between seek points (4096)')
    x.add_argument('--overwrite', action='store_true')
    d = sub.add_parser('dec')
    d.add_argument('inp')
    d.add_argument('out_png')
    d.add_argument('--region', default=None, type=parse_region, metavar='Y,X,H,W',
                   help='decode only this crop, and only the tiles (DESIGN §4.8) or, for reference-layout files '
                        'and their .partN parts, the row bands of the seek index written by `idx` (§4.13) it '
                        'depends on')
    d.add_argument('--level', default=0, type=int, metavar='K',
                   help='with --region, RGB baselines: the crop is of the stored scale-K thumbnail (0 = the image)')
    u = sub.add_parser('upd', help='tiled L3C files: write OUT.l3c, IN.l3c with the pixels at Y,X replaced by '
                                   'PATCH.png (DESIGN §4.12), re-encoding only the tiles the edit can change')
    u.add_argument('inp')
    u.add_argument('patch')
    u.add_argument('pos', type=parse_pos, metavar='Y,X')
    u.add_argument('out')
    u.add_argument('--overwrite', action='store_true')
    u.add_argument('--edit', nargs=2, action='append', default=[], metavar=('PATCH.png', 'Y,X'),
                   help='one more edit, applied after the positional one and the --edit options before it (all in '
                        'one Bitcoding.update_regions call); may be repeated')
    return p


def parse_pos(text):
    """'Y,X' -> (y, x)."""
    try:
        vals = tuple(int(v) for v in text.split(','))
    except ValueError:
        vals = ()
    if len(vals) != 2:
        raise argparse.ArgumentTypeError('the position takes Y,X (two integers), got %r' % text)
    return vals


def parse_tile(text):
    """'TH,TW' -> (th, tw), each 1 .. 65535 (the container stores them as u16)."""
    try:
        vals = tuple(int(v) for v in text.split(','))
    except ValueError:
        vals = ()
    if len(vals) != 2 or not all(1 <= v <= 65535 for v in vals):
        raise argparse.ArgumentTypeError('--tile takes TH,TW (two integers 1..65535), got %r' % text)
    return vals


def parse_region(text):
    """'Y,X,H,W' -> (y, x, h, w)."""
    try:
        vals = tuple(int(v) for v in text.split(','))
    except ValueError:
        vals = ()
    if len(vals) != 4:
        raise argparse.ArgumentTypeError('--region takes Y,X,H,W (four integers), got %r' % text)
    return vals


def decode_region(bc, pin, png_out, region, level=0):
    """`dec --region`: one crop of a tiled file, of a reference-layout file with its seek index (`idx IN.l3c` writes
    it), or of an image the reference stored in parts (`.partN` files, each with its index) --
    Bitcoding.decode_region_file.  ValueError for what that refuses, e.g. a missing index or tiled parts."""
    if not os.path.isfile(pin) and not os.path.isfile(pin + '.part0'):
        raise DecodeError('File not found: {}'.format(pin))
    img = bc.decode_region_file(pin, region, level)
    write_image(img, png_out)
    print('Decoded region {} (level {}) of {} -> {}'.format(region, level, pin, png_out))


def update_region(bc, pin, patch_p, pos, pout, overwrite=False, more=()):
    """`upd`: IN.l3c with the pixels at pos replaced by the image PATCH, written to OUT; more = [(PATCH, 'Y,X')] (the
    --edit options): edits applied after it, in order, in one Bitcoding.update_regions call.  ValueError for crop files
    (`.partN`, an image coded in parts), an existing OUT without --overwrite, a malformed --edit position and what
    Bitcoding.update_region(s) refuses."""
    from . import part_suffix_helper
    if not os.path.isfile(pin):
        if os.path.isfile(pin + '.part0'):
            raise ValueError('{} is stored in parts ({}.part0, ...): region update of part files is not '
                             'supported'.format(pin, pin))
        raise DecodeError('File not found: {}'.format(pin))
    if part_suffix_helper.contains_part_suffix(pin):
        raise ValueError('{} is one part of an image coded in parts: region update of part files is not '
                         'supported'.format(pin))
    if os.path.isfile(pout) and not overwrite:
        raise ValueError('{} exists. Consider --overwrite.'.format(pout))
    with open(pin, 'rb') as f:
        data = f.read()
    if more:
        edits = [(pos, read_image(patch_p))]
        for p, text in more:
            try:
                edits.append((parse_pos(text), read_image(p)))
            except argparse.ArgumentTypeError as err:
                raise ValueError('--edit %s %s: %s' % (p, text, err))
        out = bc.update_regions([data], [edits])[0]
    else:
        out = bc.update_region(data, pos, read_image(patch_p))
    with open(pout, 'wb') as f:
        f.write(out)
    print('Updated {} at {} with {} -> {}'.format(pin, pos, patch_p, pout))
    for p, text in more:
        print('  and at {} with {}'.format(text, p))


def main(argv=None):
    a = build_parser().parse_args(argv)
    from .bitcoding import Bitcoding
    bp = load_blueprint(a.config, a.ckpt, a.precision)
    tile = getattr(a, 'tile', None) if a.mode == 'enc' else None        # dec: the layout is read from the file
    bc = Bitcoding(bp, recursive=recursive_of(a, bp.net.config_ms), tile=tile, crop=tile is None)
    try:
        if a.mode == 'enc':
            encode(bc, a.img, a.out, a.overwrite, a.seek)
        elif a.mode == 'idx':
            index(bc, a.inp, a.every, a.overwrite)
        elif a.mode == 'upd':
            try:
                update_region(bc, a.inp, a.patch, a.pos, a.out, a.overwrite, a.edit)
            except ValueError as err:
                raise EncodeError(str(err))
        elif a.region is not None:
            try:
                decode_region(bc, a.inp, a.out_png, a.region, a.level)
            except ValueError as err:
                raise DecodeError(str(err))
        else:
            decode(bc, a.inp, a.out_png)
    except (EncodeError, DecodeError) as err:
        print('*** ERROR: {}'.format(err))
        return 1
    return 0


if __name__ == '__main__':
    sys.exit(main())
