"""Host side of the 3x3 convolutions' backward (DESIGN §4.11): the C ABI refuses every bad call before any GPU work,
the switch `train.FUSED_CONV` is off by default and CPU tensors keep the torch path bit for bit, and the layers it
covers in `cr.cf` are exactly the 3x3 / 64-input-channel ones.  No device is needed: a refused call returns
L3C_EINVAL from its argument checks, where any CUDA call on a machine without a GPU would fail with L3C_ECUDA."""
import ctypes

import pytest
import torch

EINVAL = -1
P0, P1, P2, P3, P4 = (ctypes.c_void_p(0x10000 * (i + 1)) for i in range(5))   # never dereferenced
ODD = ctypes.c_void_p(0x10000 + 4)             # one fp32 element past an aligned address: not a 64-bit offset


def _lib():
    from l3c_pytorch_b200._lib import lib
    return lib


def _err():
    return _lib().l3c_last_error().decode()


def _dgrad(dy=P0, w=P1, dx=P2, N=2, H=16, W=16, Cin=64, Cout=64, d=1):
    return _lib().l3c_conv3x3_dgrad(dy, w, N, H, W, Cin, Cout, d, dx, None)


def _wgrad(x=P0, dy=P1, dw=P2, db=P3, work=P4, N=2, H=16, W=16, Cin=64, Cout=64, d=1, work_bytes=1 << 40):
    return _lib().l3c_conv3x3_wgrad(x, dy, N, H, W, Cin, Cout, d, dw, db, work, work_bytes, None)


BAD = [
    ('null dy / x', dict(dy=None), dict(x=None), 'null pointer'),
    ('null w / dy', dict(w=None), dict(dy=None), 'null pointer'),
    ('null dx / dw', dict(dx=None), dict(dw=None), 'null pointer'),
    ('cin', dict(Cin=32), dict(Cin=32), 'Cin=32'),
    ('cout 128', dict(Cout=128), dict(Cout=128), 'Cout=128'),
    ('cout 3', dict(Cout=3), dict(Cout=3), 'Cout=3'),
    ('dilation 3', dict(d=3), dict(d=3), 'dilation=3'),
    ('dilation 0', dict(d=0), dict(d=0), 'dilation=0'),
    ('plane above 2^30', dict(H=32769, W=32768), dict(H=32769, W=32768), 'plane is above'),
    ('N 0', dict(N=0), dict(N=0), 'N=0'),
    ('unaligned dy / x', dict(dy=ODD), dict(x=ODD), 'not 16-byte aligned'),
    ('unaligned dx / db', dict(dx=ODD), dict(db=ODD), 'not 16-byte aligned'),
]


@pytest.mark.parametrize('case', BAD, ids=[b[0] for b in BAD])
def test_backward_refusals_before_launch(case):
    _, dkw, wkw, msg = case
    assert _dgrad(**dkw) == EINVAL
    assert msg in _err(), _err()
    assert _wgrad(**wkw) == EINVAL
    assert msg in _err(), _err()


def test_wgrad_refuses_null_bias_grad_and_workspace():
    for kw in (dict(db=None), dict(work=None)):
        assert _wgrad(**kw) == EINVAL and 'null pointer' in _err()
    need = _lib().l3c_conv3x3_wgrad_workspace(2, 16, 16, 64)
    assert need > 0
    assert _wgrad(work_bytes=need - 4) == EINVAL and 'workspace' in _err()


def test_wgrad_workspace_follows_the_shape():
    lib = _lib()
    # one chunk per tile up to the CTA target, partial dW (64 x 576) and db (64) per chunk
    assert lib.l3c_conv3x3_wgrad_workspace(1, 9, 7, 64) == 2 * 64 * 577 * 4
    assert lib.l3c_conv3x3_wgrad_workspace(1, 33, 17, 64) == 10 * 64 * 577 * 4
    assert lib.l3c_conv3x3_wgrad_workspace(1, 33, 17, 256) == 10 * 256 * 577 * 4
    for bad in ((0, 8, 8, 64), (1, 8, 8, 128), (1, 32769, 32768, 64)):
        assert lib.l3c_conv3x3_wgrad_workspace(*bad) == 0


def test_round_refusals():
    lib = _lib()
    assert lib.l3c_round_tf32(None, P1, 16, None) == EINVAL
    assert lib.l3c_round_tf32(P0, ODD, 16, None) == EINVAL
    assert lib.l3c_round_tf32(P0, P1, -1, None) == EINVAL
    assert lib.l3c_round_tf32(P0, P1, 0, None) == 0          # nothing to do, nothing launched


def test_switch_is_off_by_default():
    from l3c_pytorch_b200 import train
    assert train.FUSED_CONV is False


def test_in_scope_layers_of_cr():
    """the 3x3 / 64-input-channel layers of cr.cf, and nothing else"""
    from l3c_pytorch_b200 import MultiscaleBlueprint, config, train
    torch.manual_seed(0)
    net = MultiscaleBlueprint(config.ms_config('cr'), device='cpu').net
    convs = {n: m for n, m in net.named_modules() if isinstance(m, torch.nn.Conv2d)}
    scope = {n for n, m in convs.items() if train.conv3x3_in_scope(m)}
    for n, m in convs.items():
        k, cin = m.kernel_size[0], m.in_channels
        assert (n in scope) == (k == 3 and cin == 64 and m.stride[0] == 1), n
    assert any(n.endswith('tail.0') for n in scope)
    assert sorted({convs[n].dilation[0] for n in scope}) == [1, 2, 4]
    assert sorted({convs[n].out_channels for n in scope}) == [64, 256]
    assert not any(n.startswith('heads.0') for n in scope)          # the RGB head (3 -> 64) stays on cuDNN


def test_cpu_tensors_keep_the_torch_path_exactly():
    """FUSED_CONV on CPU tensors: the same loss, gradients and step bit for bit as with the switch off"""
    from l3c_pytorch_b200 import MultiscaleBlueprint, config, train
    from tests import util
    imgs = torch.stack([util.make_image(i, 32, 32) for i in range(2)]).float()
    out = {}
    for fused in (False, True):
        torch.manual_seed(0)
        bp = MultiscaleBlueprint(config.ms_config('cr'), device='cpu')
        bp.net.float().cpu()
        bp.net.train()
        opt = train.make_optimizer(bp)
        old = train.FUSED_CONV
        train.FUSED_CONV = fused
        try:
            bp.net.zero_grad()
            loss, bpsps = train.training_loss(bp, imgs)
            loss.backward()
            grads = {k: p.grad.clone() for k, p in bp.net.named_parameters() if p.grad is not None}
            opt.step()
        finally:
            train.FUSED_CONV = old
        out[fused] = (float(loss.detach()), bpsps, grads, {k: p.detach().clone() for k, p in bp.net.named_parameters()})
    (l0, b0, g0, p0), (l1, b1, g1, p1) = out[False], out[True]
    assert l0 == l1 and b0 == b1
    assert g0.keys() == g1.keys()
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    for k in p0:
        assert torch.equal(p0[k], p1[k]), k
