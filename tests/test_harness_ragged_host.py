"""CPU: the harness's theoretical-bpsp mode with ragged passes (DESIGN §4.6) -- the pass plan, the `--batch` cap,
auto-cropped images, the per-crop sub-pixel counts, and results equal to the one-pass-per-shape path -- with a
stand-in blueprint that supports ragged batches (the real one needs a GPU: tests/test_gpu_ragged_theory.py)."""
import json
import os

import numpy as np
import pytest
import torch

from l3c_pytorch_b200 import harness as H
from l3c_pytorch_b200 import pad as _pad
from l3c_pytorch_b200.bitcoding import plan_passes

FAC = 8                                     # 2 ** num_scales of configs/ms/cr.cf
SIZES = {'a': (16, 24), 'b': (16, 24), 'c': (8, 8), 'd': (20, 12), 'e': (40, 40), 'f': (33, 17)}


def _png(path, h, w, seed):
    from PIL import Image
    rng = np.random.default_rng(seed)
    Image.fromarray(rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)).save(path)


def _padded(h, w):
    return h + (-h) % FAC, w + (-w) % FAC


class _Net(torch.nn.Module):
    ragged = True

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))

    def ragged_unsupported(self, auto_recurse=0):
        return None if _Net.ragged and not auto_recurse else 'no ragged batches here'


class _Out(object):
    def __init__(self, batch, extents):
        self.batch, self.extents = batch, extents


class _RaggedBlueprint(object):
    """bpsp of an image := sum of its padded pixels / its unpadded sub-pixels + w / 1e6; a ragged pass sums inside
    each extent only, so an image gets the same number in any pass."""
    made = []

    def __init__(self, config_ms):
        self.config_ms, self.net, self.device = config_ms, _Net(), torch.device('cpu')
        self.passes, self.subpixels = [], []
        _RaggedBlueprint.made.append(self)

    def set_eval(self):
        return self

    def unpack_batch_pad(self, raw, fac):
        assert raw.dim() == 4 and raw.dtype == torch.uint8 and fac == FAC
        x, _ = _pad.pad(raw, fac, mode='constant')
        return x.float(), x.long()

    def forward(self, batch, auto_recurse=0, extents=None):
        assert auto_recurse == 0
        self.passes.append((tuple(batch.shape), None if extents is None else list(extents)))
        if extents is not None:
            for n, (h, w) in enumerate(extents):
                assert (batch[n, :, h:, :] == 0).all() and (batch[n, :, :, w:] == 0).all()
        return _Out(batch, extents)

    def get_loss_per_image(self, out, num_subpixels_before_pad=None):
        N, _, Hb, Wb = out.batch.shape
        ext = out.extents or [(Hb, Wb)] * N
        sub = num_subpixels_before_pad
        sub = list(sub) if np.ndim(sub) > 0 else [sub] * N
        self.subpixels.append(sub)
        return [float(out.batch[n, :, :h, :w].double().sum()) / s + self.net.w.item() / 1e6
                for n, ((h, w), s) in enumerate(zip(ext, sub))]


def _tester(log_date, flags, restore_itr, configs_dir=None):
    return H.Tester(log_date, flags, restore_itr, configs_dir=configs_dir, make_blueprint=_RaggedBlueprint)


@pytest.fixture
def tree(tmp_path):
    logs, cfgs, imgs = tmp_path / 'logs', tmp_path / 'configs', tmp_path / 'imgs'
    for d in (cfgs / 'ms', imgs):
        d.mkdir(parents=True)
    here = os.path.join(os.path.dirname(H.__file__), 'configs', 'ms', 'cr.cf')
    (cfgs / 'ms' / 'cr.cf').write_text(open(here).read())
    exp = logs / '0306_0001 cr oi'
    (exp / 'ckpts').mkdir(parents=True)
    torch.save({'net': {'w': torch.tensor([7.])}}, str(exp / 'ckpts' / 'ckpt_0000000010.pt'))
    for i, (name, (h, w)) in enumerate(sorted(SIZES.items())):
        _png(str(imgs / (name + '.png')), h, w, i)
    _Net.ragged = True
    yield dict(logs=str(logs), cfgs=str(cfgs), imgs=str(imgs), root=tmp_path)
    _Net.ragged = True


def _run(tree, *extra):
    _RaggedBlueprint.made.clear()
    argv = [tree['logs'], '0306_0001', tree['imgs'], '--configs_dir', tree['cfgs'], '--overwrite_cache'] + list(extra)
    assert H.main(argv, tester_cls=_tester) == 0
    with open(os.path.join(tree['logs'] + '_test', '0306_0001 cr oi', 'results.json')) as f:
        return _RaggedBlueprint.made[-1], json.load(f)['imgs_6@10']['per_img']


def test_plan_passes_caps_the_images_per_pass():
    shapes = [(16, 24), (16, 24), (8, 8), (24, 16), (40, 40), (40, 24)]
    assert sorted(i for p in plan_passes(shapes) for i in p) == list(range(6))
    assert len(plan_passes(shapes)) == 1
    capped = plan_passes(shapes, max_images=2)
    assert [len(p) for p in capped] == [2, 2, 2]
    assert capped == [[2, 0], [1, 3], [5, 4]]                     # sorted by shape, ties in input order
    assert plan_passes(shapes, max_images=1) == [[i] for i in (2, 0, 1, 3, 5, 4)]
    assert plan_passes(shapes, budget=2 * 40 * 40, max_images=16)[-1] == [5, 4]


def test_ragged_passes_of_the_test_set(tree):
    bp, per_img = _run(tree, '--batch', '4')
    assert sorted(per_img) == sorted(SIZES)
    order = sorted(SIZES)                                         # test-set order: file names sorted
    padded = [_padded(*SIZES[n]) for n in order]
    want = plan_passes(padded, max_images=4)
    assert len(bp.passes) == len(want) == 2
    for (shape, ext), idxs in zip(bp.passes, want):
        assert ext == [padded[i] for i in idxs]                   # every crop padded on its own
        assert shape == (len(idxs), 3, max(h for h, _ in ext), max(w for _, w in ext))
        assert len(idxs) <= 4
    assert len({e for _, ext in bp.passes for e in ext}) > len(bp.passes)   # shapes really share passes
    # d (20 x 12) and f (33 x 17) are padded; their bpsp counts the unpadded sub-pixels
    assert bp.subpixels == [[3 * SIZES[order[i]][0] * SIZES[order[i]][1] for i in idxs] for idxs in want]


def test_crops_of_one_image_share_a_pass(tree, monkeypatch):
    monkeypatch.setenv('AC_NEEDS_CROP_DIM', '40,40')
    _png(os.path.join(tree['imgs'], 'g.png'), 97, 61, 9)
    for f in os.listdir(tree['imgs']):
        if f != 'g.png':
            os.remove(os.path.join(tree['imgs'], f))
    _RaggedBlueprint.made.clear()
    argv = [tree['logs'], '0306_0001', tree['imgs'], '--configs_dir', tree['cfgs']]
    assert H.main(argv, tester_cls=_tester) == 0
    bp = _RaggedBlueprint.made[-1]
    crops = [(48, 30), (48, 31), (49, 30), (49, 31)]             # quadrants of 97 x 61
    assert len(bp.passes) == 1
    assert bp.passes[0][1] == [(48, 32), (48, 32), (56, 32), (56, 32)]
    assert bp.subpixels == [[3 * h * w for (h, w) in crops]]


def test_ragged_results_equal_the_per_shape_path(tree):
    _, ragged = _run(tree, '--batch', '3')
    _, ragged1 = _run(tree, '--batch', '1')
    _Net.ragged = False
    bp, by_shape = _run(tree, '--batch', '3')
    assert all(ext is None for _, ext in bp.passes)
    assert sorted(shape[2:] for shape, _ in bp.passes) == sorted({_padded(*s) for s in SIZES.values()})
    assert ragged == by_shape == ragged1
