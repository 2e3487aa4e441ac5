"""CPU: host logic of recursive containers (DESIGN §4.7) -- how R is inferred from a container's scale list and
validated, the padding factor and the bpsp denominators, the `--recursive` flag of the CLI, and the harness
passing `recursive=` to the bit-coder only when it is non-zero."""
import os

import numpy as np
import pytest
import torch

from l3c_pytorch_b200 import harness as H
from tests import util


def _codec(cfg):
    from l3c_pytorch_b200.codec import BatchCodec
    return BatchCodec(util.blueprint(cfg, device='cpu'))


def test_check_shapes_infers_and_validates_recursion():
    rgbs, rgb, l3c = _codec('cr_rgb_shared'), _codec('cr_rgb'), _codec('cr')
    assert rgbs._check_shapes([(3, 32, 32), (3, 64, 64)]) == 0
    assert rgbs._check_shapes([(3, 4, 3), (3, 8, 6), (3, 16, 12), (3, 32, 24), (3, 64, 48)]) == 3
    assert rgb._check_shapes([(3, 2, 2), (3, 4, 4), (3, 8, 8), (3, 16, 16), (3, 32, 32), (3, 64, 64)]) == 2
    for bad in ([(3, 64, 64)],                                                # fewer scales than the model's
                [(3, 4, 4), (3, 8, 8), (3, 16, 12), (3, 32, 24)],              # a scale not half the finer one
                [(3, 4, 4), (5, 8, 8), (3, 16, 16), (3, 32, 32)],              # C != 3 at a recursive scale
                [(5, 4, 4), (3, 8, 8), (3, 16, 16), (3, 32, 32)],              # C != 3 at the uniform scale
                [(3, 0, 0), (3, 0, 0), (3, 0, 0)]):
        with pytest.raises(ValueError):
            rgbs._check_shapes(bad)
    # learned bottlenecks: one scale more than the model has is a recursive container, refused with the reason
    with pytest.raises(ValueError, match='RGB baselines'):
        l3c._check_shapes([(5, 2, 2), (5, 4, 4), (5, 8, 8), (5, 16, 16), (3, 32, 32)])
    l3c._check_shapes([(5, 4, 4), (5, 8, 8), (5, 16, 16), (3, 32, 32)])


def test_scale_walk_and_recursion_argument():
    c = _codec('cr_rgb_shared')
    walk = list(c.iter_scale_dmll(3))
    assert [s for s, _, _ in walk] == [4, 3, 2, 1, 0] and [u for _, _, u in walk] == [True] + [False] * 4
    assert all(d is c.blueprint.losses.loss_dmol_rgb for _, d, _ in walk)
    assert [s for s, _, _ in c.iter_scale_dmll()] == [1, 0]
    for bad in (-1, 1.5, True, '2', None):
        with pytest.raises(ValueError):
            c.check_recursive(bad)
    assert c.check_recursive(np.int64(2)) == 2
    with pytest.raises(ValueError, match='RGB baselines'):
        _codec('cr').check_recursive(1)
    assert _codec('cr').check_recursive(0) == 0


def test_bitcoding_padding_factor_and_bpsp_denominator():
    from l3c_pytorch_b200 import pad
    from l3c_pytorch_b200.bitcoding import Bitcoding, _ListEncodeJob
    bp = util.blueprint('cr_rgb_shared', device='cpu')
    assert Bitcoding(bp).pad_factor() == 2 and Bitcoding(bp, recursive=3).pad_factor() == 16
    assert Bitcoding(util.blueprint('cr_rgb', device='cpu'), recursive=2).pad_factor() == 32
    for bad in (-1, 2.0, False, 'auto'):
        with pytest.raises(ValueError):
            Bitcoding(bp, recursive=bad)
    with pytest.raises(ValueError, match='RGB baselines'):
        Bitcoding(util.blueprint('cr', device='cpu'), recursive=2)
    assert Bitcoding(util.blueprint('cr', device='cpu'), recursive=0).recursive == 0
    img = util.make_image(0, 40, 28)
    x, pt = Bitcoding(bp, recursive=3)._prepare(img, quiet=True)
    assert tuple(x.shape) == (1, 3, 48, 32) and torch.equal(pad.undo_pad(x, *pt)[0], img)
    assert int(x.sum()) == int(img.long().sum())                            # zero padding
    x0, pt0 = Bitcoding(bp)._prepare(img, quiet=True)
    assert tuple(x0.shape) == (1, 3, 40, 28) and pt0 == (0, 0, 0, 0) and any(pt)

    class _Job(object):
        def finish(self, to_host=True):
            return [b'x' * 100, b'y' * 60], None
    # bpsp = bytes * 8 / PADDED sub-pixels (the reference's denominator), per image
    datas, bpsps = _ListEncodeJob([([1, 0], _Job())], [3 * 48 * 32, 3 * 16 * 16]).finish()
    assert datas == [b'y' * 60, b'x' * 100]
    assert bpsps == [60 * 8 / (3 * 48 * 32), 100 * 8 / (3 * 16 * 16)]


def test_cli_recursive_flag():
    from l3c_pytorch_b200 import cli, config
    p = cli.build_parser()
    rgbs, rgb, l3c = (config.ms_config(n) for n in ('cr_rgb_shared', 'cr_rgb', 'cr'))
    a = p.parse_args(['--config', 'cr_rgb_shared', 'enc', 'i.png', 'o.l3c', '--recursive', 'auto'])
    assert a.recursive == 'auto' and cli.recursive_of(a, rgbs) == 3 and cli.recursive_of(a, l3c) == 0
    assert cli.recursive_of(a, rgb) == 0                                   # 'auto' is 3 for one trained scale only
    a = p.parse_args(['enc', 'i.png', 'o.l3c', '--recursive', '2'])
    assert cli.recursive_of(a, rgb) == 2 and cli.recursive_of(a, l3c) == 0
    assert cli.recursive_of(p.parse_args(['enc', 'i.png', 'o.l3c']), rgbs) == 0
    d = p.parse_args(['--config', 'cr_rgb_shared', 'dec', 'o.l3c', 'x.png'])
    assert cli.recursive_of(d, rgbs) == 0                                  # decode reads R from the file
    with pytest.raises(SystemExit):
        p.parse_args(['dec', 'o.l3c', 'x.png', '--recursive', '2'])


class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(1))


class _Blueprint(object):
    def __init__(self, config_ms):
        self.config_ms, self.net, self.device = config_ms, _Net(), torch.device('cpu')

    def set_eval(self):
        return self


class _Bitcoding(object):
    calls = []

    def __init__(self, blueprint, **kw):
        _Bitcoding.calls.append(kw)


@pytest.mark.parametrize('cfg,flag,want', [('cr_rgb_shared', 'auto', 3), ('cr_rgb_shared', '2', 2),
                                           ('cr_rgb_shared', '0', None), ('cr_rgb', '1', 1),
                                           ('cr_rgb', 'auto', None), ('cr', 'auto', None), ('cr', '2', None)])
def test_harness_passes_recursive_only_when_nonzero(tmp_path, cfg, flag, want):
    exp = tmp_path / 'logs' / ('0306_0001 %s oi' % cfg)
    (exp / 'ckpts').mkdir(parents=True)
    torch.save({'net': {'w': torch.tensor([1.])}}, str(exp / 'ckpts' / 'ckpt_0000000010.pt'))
    argv = [str(tmp_path / 'logs'), '0306_0001', str(tmp_path), '--write_to_files', str(tmp_path / 'out'),
            '--recursive', flag]
    flags = H.build_parser().parse_args(argv)
    H.check_flags(flags)
    _Bitcoding.calls.clear()
    t = H.Tester('0306_0001', flags, -1, make_blueprint=_Blueprint, make_bitcoding=_Bitcoding)
    assert t.recursive == (want or 0)
    kw = _Bitcoding.calls[-1]
    assert set(kw) == ({'times', 'compare_with_theory', 'recursive'} if want else {'times', 'compare_with_theory'})
    assert kw.get('recursive') == want
    assert os.path.isdir(t.test_log_dir)
