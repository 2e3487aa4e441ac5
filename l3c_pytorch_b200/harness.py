"""Test harness over experiment directories and image folders: the `test.py` / `MultiscaleTester` side
of the reference (SURVEY.md section 8, row f1) on the H100 path.

    python -m l3c_pytorch_b200.harness LOG_DIR LOG_DATES IMAGES [--write_to_files DIR] [--compare_theory]
                                       [--time_report PATH] [--crop N] [--restore_itr I] [--names A,B] ...

What it mirrors (flag names and meaning as in /root/reference/src/test.py:44-141):
  * experiment lookup: `LOG_DIR/<MMDD_HHMM> <ms config> <dl config> [r@...] [postfix]`, the config file is
    found under CONFIGS/ms/ with '@' standing for a path separator and '*' for exactly one character
    (helpers/logdir_helpers.py:71-108, helpers/paths.py:44-60);
  * checkpoint choice: `ckpts/ckpt_<itr>.pt[.tmp]`, newest for -1, else the closest one not after the
    requested iteration (helpers/saver.py:57-84); loaded strict into the same-named module tree
    (helpers/saver.py:184-210);
  * test sets: a folder of images or one image, optional name filter / evenly spaced subsample
    (helpers/testset.py:33-80), optional centre crop;
  * default mode: theoretical bpsp per image from the network's own likelihoods, crops of large images
    weighted by their sub-pixel counts (test/multiscale_tester.py:283-345), cached per (test set, itr);
  * --write_to_files: every image through the real coder to `<name>.l3c`, decoded again and compared,
    real bpsp reported, per-stage times collected (test/multiscale_tester.py:347-373).  With --recursive N|auto
    on an RGB baseline the files are recursive containers (DESIGN §4.7), which the reference cannot write
    (multiscale_tester.py:187-188 raises); --compare_theory then prints the recursive theory.
--sample writes the ground truth and three sampled images per test image (row f3).

H100-first difference: in the default mode up to `--batch` images (default 16) share one network pass instead
of going one at a time.  Where the network runs ragged batches (precision f16, learned bottlenecks, no
--recursive; DESIGN §4.6) every crop is padded on its own and crops of ANY sizes are planned into passes
(bitcoding.plan_passes), each placed top-left in a zero batch: the bpsp of every image is bit-identical to
evaluating it alone.  Elsewhere (fp32 / tf32 / f16x2, the RGB baselines, --recursive) only crops of equal shape
share a pass.
"""
import argparse
import fnmatch
import json
import os
import re
import sys
from collections import OrderedDict

import numpy as np
import torch

IMAGE_EXTS = ('.png', '.jpg', '.jpeg', '.bmp', '.ppm', '.tif', '.tiff')
FILE_EXT = '.l3c'
_LOG_DATE = re.compile(r'^\d{4}_\d{4}$')


# --------------------------------------------------------------------------------------------------
# experiment directories, configs, checkpoints
# --------------------------------------------------------------------------------------------------
def is_log_date(s):
    return bool(_LOG_DATE.match(s))


def find_experiment_dir(log_dir, log_date):
    """The one sub-directory of `log_dir` whose name starts with `log_date`."""
    if not is_log_date(log_date):
        raise ValueError('Not a log date (MMDD_HHMM): {!r}'.format(log_date))
    hits = [d for d in sorted(os.listdir(log_dir))
            if d.split(' ')[0] == log_date and os.path.isdir(os.path.join(log_dir, d))]
    if len(hits) != 1:
        raise ValueError('Expected exactly one experiment for {} in {}, found {}'.format(log_date, log_dir, hits))
    return os.path.join(log_dir, hits[0])


def _resolve_config(base_dir, token, ext='.cf'):
    """`token` is a config path relative to `base_dir` with os.sep written as '@' and line-breaking
    characters written as '*' (each '*' stands for exactly ONE character)."""
    rel = token.replace('@', os.sep) + ext
    want_dir, want_name = os.path.split(os.path.join(base_dir, rel))
    if not os.path.isdir(want_dir):
        raise ValueError('Cannot find config on disk: {}'.format(os.path.join(base_dir, rel)))
    pat = want_name.replace('*', '?')
    hits = [f for f in sorted(os.listdir(want_dir)) if len(f) == len(want_name) and fnmatch.fnmatchcase(f, pat)]
    if len(hits) != 1:
        raise ValueError('Cannot find config on disk: {} (matches: {})'.format(os.path.join(base_dir, rel), hits))
    return os.path.join(want_dir, hits[0])


def configs_of_experiment(experiment_dir, configs_dir, base_dirs=('ms', 'dl')):
    """-> (config paths, one per base dir; postfix tokens).  Directory name format:
    `<log date> <config> <config> [r@<restored log date>] [postfix ...]`."""
    comps = os.path.basename(experiment_dir.rstrip(os.sep)).split(' ')
    if not comps or not is_log_date(comps[0]):
        raise ValueError('Invalid log_dir: {}'.format(experiment_dir))
    if len(comps) <= len(base_dirs):
        raise ValueError('Expected a config for each of {}, got {}'.format(base_dirs, comps))
    tokens = comps[1:1 + len(base_dirs)]
    rest = [c for c in comps[1 + len(base_dirs):] if not c.startswith('r@')]
    # only the first tree (the network config) is needed to test; the data-loader configs of the
    # reference's training side are resolved when their tree exists and reported as None otherwise
    paths = tuple(_resolve_config(os.path.join(configs_dir, b), t)
                  if (i == 0 or os.path.isdir(os.path.join(configs_dir, b))) else None
                  for i, (b, t) in enumerate(zip(base_dirs, tokens)))
    return paths, tuple(rest)


def list_checkpoints(experiment_dir, prefix='ckpt_'):
    """[(iteration, path)] ascending; temporary (`.tmp`) checkpoints count, as in the reference."""
    d = os.path.join(experiment_dir, 'ckpts')
    if not os.path.isdir(d):
        raise ValueError('No ckpts directory in {}'.format(experiment_dir))
    out = []
    for f in sorted(os.listdir(d)):
        if f.startswith(prefix):
            digits = ''.join(c for c in os.path.splitext(f.replace('.tmp', ''))[0][len(prefix):] if c.isdigit())
            if digits:
                out.append((int(digits), os.path.join(d, f)))
    out.sort()
    if not out:
        raise ValueError('No ckpts found in {}'.format(d))
    return out


def checkpoint_for_itr(ckpts, itr):
    """Newest checkpoint for itr == -1, else the latest one with iteration <= itr."""
    if itr == -1:
        return ckpts[-1]
    older = [c for c in ckpts if c[0] <= itr]
    if not older:
        raise ValueError('Earliest ckpt {} is after {}'.format(ckpts[0][0], itr))
    return older[-1]


def restore(blueprint, ckpt_path):
    """Load `{'net': state_dict}` (helpers/saver.py:168) strictly into blueprint.net."""
    print('Restoring {}... (strict=True)'.format(ckpt_path))
    state = torch.load(ckpt_path, map_location='cpu')
    blueprint.net.load_state_dict(state['net'] if 'net' in state else state, strict=True)
    blueprint.net.to(blueprint.device)
    return blueprint


# --------------------------------------------------------------------------------------------------
# test sets
# --------------------------------------------------------------------------------------------------
class Testset(object):
    def __init__(self, root_dir_or_img, max_imgs=None, append_id=None):
        self.root = root_dir_or_img
        if os.path.isdir(root_dir_or_img):
            self.name = os.path.basename(root_dir_or_img.rstrip('/'))
            ps = sorted(os.path.join(root_dir_or_img, f) for f in os.listdir(root_dir_or_img)
                        if f.lower().endswith(IMAGE_EXTS))
            if max_imgs and max_imgs < len(ps):
                print('Subsampling to use {} imgs of {}...'.format(max_imgs, self.name))
                ps = [ps[i] for i in np.linspace(0, len(ps) - 1, max_imgs).astype(int)]
            if not ps:
                raise ValueError('No images found in {}'.format(root_dir_or_img))
            self.ps = ps
            self.id = '{}_{}'.format(self.name, len(ps))
        else:
            if not os.path.isfile(root_dir_or_img):
                raise FileNotFoundError('Does not exist: {}'.format(root_dir_or_img))
            self.name = os.path.basename(root_dir_or_img)
            self.ps = [root_dir_or_img]
            self.id = root_dir_or_img
        if append_id:
            self.id += append_id

    def filter_filenames(self, keep):
        self.ps = [p for p in self.ps if os.path.splitext(os.path.basename(p))[0] in keep]
        if not self.ps:
            raise ValueError('No files after filtering for {}'.format(keep))

    def __len__(self):
        return len(self.ps)

    def __repr__(self):
        return 'Testset({}): {} image(s)'.format(self.name, len(self.ps))


def read_image_chw(path, crop=None):
    """uint8 CHW (alpha dropped, grey replicated), optionally centre-cropped to crop x crop."""
    from PIL import Image
    a = np.array(Image.open(path))
    if a.ndim == 2:
        a = np.stack([a] * 3, -1)
    if a.shape[2] == 4:
        print('*** WARN: Will discard 4th (alpha) channel.')
    elif a.shape[2] != 3:
        raise ValueError('Image has {} channels, expected 3 or 4.'.format(a.shape[2]))
    a = a[..., :3]
    if crop:
        h, w = a.shape[:2]
        if h < crop or w < crop:
            raise ValueError('{} ({}x{}) is smaller than --crop {}'.format(path, h, w, crop))
        t, l = int(round((h - crop) / 2.)), int(round((w - crop) / 2.))
        a = a[t:t + crop, l:l + crop]
    return torch.from_numpy(np.ascontiguousarray(a)).permute(2, 0, 1).contiguous()


def save_png(img_1chw, path):
    """1CHW tensor with values in [0, 255] -> PNG (uint8 truncation as in multiscale_tester.py:425-434)."""
    from PIL import Image
    assert img_1chw.shape[0] == 1 and img_1chw.shape[1] == 3, img_1chw.shape
    a = img_1chw[0].detach().float().cpu().numpy().transpose(1, 2, 0).astype(np.uint8)
    Image.fromarray(np.ascontiguousarray(a)).save(path)


def ragged_theory_bpsps(blueprint, crops, fac, batch_max):
    """Theoretical bpsp of every crop (uint8 CHW, any sizes) in ragged passes (DESIGN §4.6): each crop is padded on
    its own to a multiple of `fac`, the padded shapes are planned into passes of at most `batch_max` images
    (bitcoding.plan_passes), each pass is placed top-left in a zero batch and run with forward(extents=).  The bpsp
    counts the crop's unpadded sub-pixels and is bit-identical to evaluating the crop alone.  -> [float] per crop."""
    from .bitcoding import plan_passes
    padded_shapes = [(c.shape[1] + (-c.shape[1]) % fac, c.shape[2] + (-c.shape[2]) % fac) for c in crops]
    bpsps = [None] * len(crops)
    for idxs in plan_passes(padded_shapes, max_images=batch_max):
        padded = [blueprint.unpack_batch_pad(crops[i].unsqueeze(0), fac=fac)[0] for i in idxs]
        shapes = [tuple(t.shape[-2:]) for t in padded]
        assert shapes == [padded_shapes[i] for i in idxs], shapes
        Hb, Wb = max(h for h, _ in shapes), max(w for _, w in shapes)
        batch = torch.zeros(len(idxs), 3, Hb, Wb, dtype=padded[0].dtype, device=padded[0].device)
        for k, t in enumerate(padded):
            batch[k, :, :t.shape[2], :t.shape[3]] = t[0]
        out = blueprint.forward(batch, 0, extents=shapes)
        n_sub = [crops[i].numel() for i in idxs]
        for i, bpsp in zip(idxs, blueprint.get_loss_per_image(out, num_subpixels_before_pad=n_sub)):
            bpsps[i] = float(bpsp)
    return bpsps


class TestResult(object):
    def __init__(self, metric_name='bpsp'):
        self.metric_name = metric_name
        self.per_img = OrderedDict()

    def __setitem__(self, name, value):
        self.per_img[name] = float(value)

    def mean(self):
        return float(np.mean(list(self.per_img.values())))


# --------------------------------------------------------------------------------------------------
# the tester
# --------------------------------------------------------------------------------------------------
def default_configs_dir():
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), 'configs')


DEFAULT_RECURSIVE_FOR_RGB = 3        # multiscale_tester.py:50


def parse_recursive_flag(recursive, config_ms):
    """multiscale_tester.py:123-132: only the RGB baselines are evaluated recursively; 'auto' = 3 more
    applications of the shared scale for RGB-shared (one trained scale)."""
    if not config_ms.rgb_bicubic_baseline:
        return 0
    if recursive == 'auto':
        if config_ms.rgb_bicubic_baseline and config_ms.num_scales == 1:
            return DEFAULT_RECURSIVE_FOR_RGB
    try:
        return int(recursive)
    except ValueError:
        return 0


class Tester(object):
    """One experiment (log date) at one checkpoint.  `make_blueprint(config_ms)` / `make_bitcoding(blueprint,
    times, compare_with_theory)` are injection points (defaults: the H100 classes)."""

    def __init__(self, log_date, flags, restore_itr, configs_dir=None, make_blueprint=None, make_bitcoding=None):
        from . import config as config_parser
        self.flags = flags
        self.experiment_dir = find_experiment_dir(flags.log_dir, log_date)
        self.log_date = log_date
        (ms_path, _dl_path), _postfix = configs_of_experiment(self.experiment_dir, configs_dir or default_configs_dir())
        self.config_ms = config_parser.parse(ms_path)[0]
        self.recursive = parse_recursive_flag(getattr(flags, 'recursive', '0'), self.config_ms)
        if self.recursive:
            print('--recursive={}'.format(self.recursive))
        if make_blueprint is None:
            from .blueprint import MultiscaleBlueprint
            make_blueprint = MultiscaleBlueprint
        self.blueprint = make_blueprint(self.config_ms)
        self.blueprint.set_eval()
        self.restore_itr, ckpt_p = checkpoint_for_itr(list_checkpoints(self.experiment_dir), restore_itr)
        restore(self.blueprint, ckpt_p)
        self.test_log_dir = os.path.join(flags.log_dir.rstrip(os.sep) + '_test', os.path.basename(self.experiment_dir))
        os.makedirs(self.test_log_dir, exist_ok=True)
        self.cache_p = os.path.join(self.test_log_dir, 'results.json')
        if getattr(flags, 'reset_entire_cache', False) and os.path.isfile(self.cache_p):
            os.remove(self.cache_p)
        self.times = None
        self.bc = None
        if flags.write_to_files:
            from .times import StackTimeLogger
            self.times = StackTimeLogger()
            if make_bitcoding is None:
                from .bitcoding import Bitcoding
                make_bitcoding = Bitcoding
            # --write_to_files --recursive: recursive containers (DESIGN §4.7), which the reference cannot write
            # (multiscale_tester.py:187-188); without --recursive the call is the reference's
            kw = dict(recursive=self.recursive) if self.recursive else {}
            self.bc = make_bitcoding(self.blueprint, times=self.times, compare_with_theory=flags.compare_theory, **kw)

    # ---- cache of theoretical results: {"<testset id>@<itr>": {"metric": .., "per_img": {..}}}
    def _cache(self):
        if os.path.isfile(self.cache_p):
            with open(self.cache_p) as f:
                return json.load(f)
        return {}

    def _cache_put(self, key, result):
        c = self._cache()
        c[key] = {'metric': result.metric_name, 'per_img': result.per_img}
        tmp = self.cache_p + '.tmp'
        with open(tmp, 'w') as f:
            json.dump(c, f)
        os.replace(tmp, self.cache_p)

    def test_all(self, testsets):
        results = [self.test(ts) for ts in testsets]
        if self.flags.write_to_files:
            return []
        return [(ts, self.log_date, self.restore_itr, '{}={}'.format(r.metric_name, r.mean()))
                for ts, r in zip(testsets, results)]

    def test(self, testset):
        key = '{}@{}'.format(testset.id, self.restore_itr)
        if not self.flags.write_to_files and not getattr(self.flags, 'overwrite_cache', False):
            hit = self._cache().get(key)
            if hit:
                print('*** Found cached: {}'.format(key))
                r = TestResult(hit['metric'])
                r.per_img.update(hit['per_img'])
                return r
        print('Testing {}'.format(testset))
        with torch.no_grad():
            if self.flags.write_to_files:
                self._write_all(testset)
                return None
            result = self._theory(testset)
        self._cache_put(key, result)
        return result

    # ---- default mode: theoretical bpsp, images of any sizes (ragged passes) or of equal size batched
    def _ragged(self):
        """True when the blueprint evaluates ragged batches (MultiscaleNetwork.ragged_unsupported is None)."""
        why = getattr(self.blueprint.net, 'ragged_unsupported', None)
        return why is not None and why(self.recursive) is None

    def _theory(self, testset):
        result = TestResult('bpsp recursive' if self.recursive else 'bpsp')
        # multiscale_tester.py:222-225: every recursion halves the image once more
        fac = 2 ** (self.recursive + 1) if self.recursive else 2 ** self.config_ms.num_scales
        batch_max = max(1, int(getattr(self.flags, 'batch', 16) or 1))
        if self._ragged():
            combos = self._theory_ragged(testset, fac, batch_max)
        else:
            combos = self._theory_by_shape(testset, fac, batch_max)
        for name, comb in combos.items():
            result[name] = comb.get_bpsp()
        print('{}: {} images: mean {}={}'.format(self.log_date, len(combos), result.metric_name, result.mean()))
        return result

    def _theory_ragged(self, testset, fac, batch_max):
        """Every crop of the test set through ragged passes (ragged_theory_bpsps); crops combined in test-set
        order."""
        from . import auto_crop
        combos = OrderedDict()                  # image name -> CropLossCombinator
        crops = []                              # [(name, crop uint8 CHW)] in test-set order
        for p in testset.ps:
            name = os.path.splitext(os.path.basename(p))[0]
            img = read_image_chw(p, self.flags.crop)
            combos[name] = auto_crop.CropLossCombinator()
            crops += [(name, crop[0]) for crop in auto_crop.iter_crops(img.unsqueeze(0))]
        bpsps = ragged_theory_bpsps(self.blueprint, [c for _, c in crops], fac, batch_max)
        for (name, crop), bpsp in zip(crops, bpsps):
            combos[name].add(bpsp, crop.numel())
        if getattr(self.flags, 'sample', None):            # multiscale_tester.py:327-328 (one image at a time)
            for (name, crop) in crops:
                self._sample(name, crop, fac)
        return combos

    def _theory_by_shape(self, testset, fac, batch_max):
        """Crops of equal shape share a pass of at most `batch_max` images."""
        from . import auto_crop
        combos = OrderedDict()                  # image name -> CropLossCombinator
        pending = OrderedDict()                 # (C,H,W) -> [(name, crop uint8 CHW)]

        def flush(shape):
            items = pending.pop(shape, [])
            if not items:
                return
            raw = torch.stack([c for _, c in items])                       # N,C,H,W uint8
            n_sub = int(np.prod(raw.shape[1:]))
            img_batch, _ = self.blueprint.unpack_batch_pad(raw, fac=fac)
            out = self.blueprint.forward(img_batch, self.recursive)
            per_image = self.blueprint.get_loss_per_image(out, num_subpixels_before_pad=n_sub)
            for (name, _), bpsp in zip(items, per_image):
                combos[name].add(float(bpsp), n_sub)
            if getattr(self.flags, 'sample', None):        # multiscale_tester.py:327-328 (one image at a time)
                for (name, crop) in items:
                    self._sample(name, crop, fac)

        for p in testset.ps:
            name = os.path.splitext(os.path.basename(p))[0]
            img = read_image_chw(p, self.flags.crop)
            combos[name] = auto_crop.CropLossCombinator()
            for crop in auto_crop.iter_crops(img.unsqueeze(0)):
                shape = tuple(crop.shape[1:])
                pending.setdefault(shape, []).append((name, crop[0]))
                if len(pending[shape]) >= batch_max:
                    flush(shape)
        for shape in list(pending):
            flush(shape)
        return combos

    # ---- --sample: images sampled from the model (multiscale_tester.py:436-448)
    def _sample(self, name, raw_u8, fac):
        out_dir = os.path.join(self.flags.sample, self.log_date)
        os.makedirs(out_dir, exist_ok=True)
        self._n_sampled = getattr(self, '_n_sampled', -1) + 1
        prefix = '{}_{}'.format(self._n_sampled, name)
        if any(f.startswith(prefix) for f in os.listdir(out_dir)):
            raise FileExistsError('Previous sample outputs found in {}. Please remove.'.format(out_dir))
        img_batch, _ = self.blueprint.unpack_batch_pad(raw_u8.unsqueeze(0), fac=fac)
        out = self.blueprint.forward(img_batch)
        bpsps = self.blueprint.get_loss(out).nonrecursive_bpsps
        save_png(img_batch, os.path.join(out_dir, '{}_{:.3f}_gt.png'.format(prefix, sum(bpsps))))
        for style, sample_scales in (('rgb', []),               # sample the RGB scale (final scale)
                                     ('rgb+bn0', [0]),          # RGB + z^(1)
                                     ('rgb+bn0+bn1', [0, 1])):  # RGB + z^(1) + z^(2)
            sampled = self.blueprint.sample_forward(img_batch, sample_scales)
            bpsp_sample = sum(bpsps[len(sample_scales) + 1:])
            save_png(sampled, os.path.join(out_dir, '{}_{}_{:.3f}.png'.format(prefix, style, bpsp_sample)))

    # ---- --write_to_files: real files through the coder, decoded back and compared
    def _write_all(self, testset):
        from . import part_suffix_helper
        out_dir = self.flags.write_to_files
        os.makedirs(out_dir, exist_ok=True)
        result = TestResult('bpsp')
        for i, p in enumerate(testset.ps):
            name = os.path.splitext(os.path.basename(p))[0]
            print('***', name)
            img = read_image_chw(p, self.flags.crop).unsqueeze(0).long().to(self.blueprint.device)
            out_p = os.path.join(out_dir, name + FILE_EXT)
            for q in [out_p] + [out_p + part_suffix_helper.make_part_suffix(j) for j in range(64)]:
                if os.path.isfile(q):
                    os.remove(q)
            with self.times.skip(i == 0):                                   # first image = warm-up
                with self.times.run('=== bc.encode'):
                    bpsp = self.bc.encode(img, pout=out_p)
                part0 = out_p + part_suffix_helper.make_part_suffix(0)
                pin = part0 if (not os.path.isfile(out_p) and os.path.isfile(part0)) else out_p
                with self.times.run('=== bc.decode'):
                    back = self.bc.decode(pin=pin)
            if not torch.equal(back.to(img.device), img):
                raise AssertionError('{}: decoded image differs from the input'.format(name))
            result[name] = bpsp
            print('{}: {} ({: 10d}): mean {}={}'.format(self.log_date, name, i, result.metric_name, result.mean()))
            if self.times.records:
                print('\n'.join(self.times.get_last_strs()))
            if self.flags.time_report:
                with open(self.flags.time_report, 'w') as f:
                    f.write('Average times:\n')
                    f.write('\n'.join(self.times.get_mean_strs()))
        return result


# --------------------------------------------------------------------------------------------------
# command line
# --------------------------------------------------------------------------------------------------
def build_parser():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument('log_dir', help='Directory of experiments; test outputs go to LOG_DIR_test.')
    p.add_argument('log_dates', help='Comma-separated log dates (MMDD_HHMM) of the experiments to test.')
    p.add_argument('images', help='Comma-separated image directories and/or single images.')
    p.add_argument('--match_filenames', '-fns', nargs='+', metavar='FILTER')
    p.add_argument('--max_imgs_per_folder', '-m', type=int, metavar='MAX')
    p.add_argument('--crop', type=int, help='Centre-crop all images to CROP x CROP.')
    p.add_argument('--names', '-n', type=str, help='Comma-separated display names, one per log date.')
    p.add_argument('--overwrite_cache', '-f', action='store_true')
    p.add_argument('--reset_entire_cache', action='store_true')
    p.add_argument('--restore_itr', '-i', default='-1', help='-1 = newest; else closest checkpoint not after it.')
    p.add_argument('--recursive', default='0')
    p.add_argument('--sample', type=str, metavar='SAMPLE_OUT_DIR')
    p.add_argument('--write_to_files', type=str, metavar='WRITE_OUT_DIR')
    p.add_argument('--compare_theory', action='store_true')
    p.add_argument('--time_report', type=str, metavar='TIME_REPORT_PATH')
    p.add_argument('--sort_output', '-s', choices=['testset', 'exp', 'itr', 'res'], default='testset')
    p.add_argument('--configs_dir', default=None, help='Root of the ms/ and dl/ config trees (default: the package\'s).')
    p.add_argument('--batch', type=int, default=16,
                   help='Most images per network pass (default mode): images of any sizes share a pass where the '
                        'network runs ragged batches (precision f16, learned bottlenecks, no --recursive), '
                        'else only images of equal size.')
    return p


def check_flags(flags):
    if flags.compare_theory and not flags.write_to_files:
        raise ValueError('Cannot have --compare_theory without --write_to_files.')
    if flags.write_to_files and flags.sample:
        raise ValueError('Cannot have --write_to_files and --sample.')
    if flags.time_report and not flags.write_to_files:
        raise ValueError('--time_report only valid with --write_to_files.')


def format_table(rows):
    """Left-aligned columns, two spaces apart."""
    widths = [max(len(str(r[c])) for r in rows) for c in range(len(rows[0]))]
    return '\n'.join('  '.join(str(v).ljust(w) for v, w in zip(r, widths)).rstrip() for r in rows)


def main(argv=None, tester_cls=Tester):
    flags = build_parser().parse_args(argv)
    check_flags(flags)
    testsets = [Testset(s.rstrip('/'), flags.max_imgs_per_folder,
                        append_id='_crop{}'.format(flags.crop) if flags.crop else None)
                for s in flags.images.split(',')]
    if flags.match_filenames:
        for ts in testsets:
            ts.filter_filenames(flags.match_filenames)
    splitter = ',' if ',' in flags.log_dates else '|'
    log_dates = flags.log_dates.split(splitter)
    results = []
    for log_date in log_dates:
        for restore_itr in map(int, flags.restore_itr.split(',')):
            print('Testing {} at {} ---'.format(log_date, restore_itr))
            tester = tester_cls(log_date, flags, restore_itr, configs_dir=flags.configs_dir)
            results += tester.test_all(testsets)
    if flags.names:
        names = flags.names.split(splitter)
        shown = {d: '{} ({})'.format(n, d) for d, n in zip(log_dates, names)}
    else:
        shown = {d: d for d in log_dates}
    if not flags.write_to_files:
        print('*** Summary:')
        key = {'testset': lambda r: r[0].id, 'exp': lambda r: r[1], 'itr': lambda r: r[2], 'res': lambda r: r[3]}
        rows = [('Testset', 'Experiment', 'Itr', 'Result')]
        for ts, log_date, itr, res in sorted(results, key=key[flags.sort_output]):
            rows.append((ts.id, shown[log_date], str(itr), res))
        print(format_table(rows))
    return 0


if __name__ == '__main__':
    sys.exit(main())
