"""CPU: which kernel engine.conv2d gives a layer in each precision mode (engine.on_tensor_cores), and that conv2d
hands that route to the library: the descriptor it fills for a recording stand-in of libl3c_b200.so."""
import types

import pytest
import torch

FP32, TF32, F16, F16X2 = 0, 1, 2, 3


def _conv(cin, cout, k, stride=1, dil=1):
    return types.SimpleNamespace(kernel_size=(k, k), stride=(stride, stride), dilation=(dil, dil), in_channels=cin,
                                 out_channels=cout)


# (conv, cin read, x pitch, y pitch, y offset, pixel shuffle, residual) -> tensor cores in (tf32, f16, f16x2)
ROUTES = {
    '3x3': ((_conv(64, 64, 3), 64, 64, 64, 0, False, False), (True, True, True)),
    '3x3 dilation 4': ((_conv(64, 64, 3, dil=4), 64, 64, 64, 0, False, False), (True, True, True)),
    '3x3 residual': ((_conv(64, 64, 3), 64, 64, 64, 0, False, True), (True, True, True)),
    '3x3 slice at offset 66': ((_conv(64, 64, 3), 64, 64, 192, 66, False, False), (False, True, True)),
    '3x3 output pitch 66': ((_conv(64, 64, 3), 64, 64, 66, 0, False, False), (False, True, True)),
    '3x3 slice at offset 64': ((_conv(64, 64, 3), 64, 64, 192, 64, False, False), (True, True, True)),
    '3x3 Cout 120': ((_conv(64, 120, 3), 64, 64, 120, 0, False, False), (False, False, False)),
    '3x3 Cin 192': ((_conv(192, 64, 3), 192, 192, 64, 0, False, False), (False, False, False)),
    '3x3 pixel shuffle': ((_conv(64, 256, 3), 64, 64, 64, 0, True, False), (True, True, True)),
    '3x3 pixel shuffle + residual': ((_conv(64, 256, 3), 64, 64, 64, 0, True, True), (True, True, False)),
    '3x3 x pitch 128': ((_conv(64, 64, 3), 64, 128, 64, 0, False, False), (False, False, False)),
    'RGB head, cin 3 in pitch 4': ((_conv(3, 64, 3), 3, 4, 64, 0, False, False), (False, False, False)),
    'cin 3 on a Cin-5 head': ((_conv(5, 64, 1), 3, 8, 64, 0, False, False), (False, False, False)),
    'decoder head, Cin 5 in pitch 8': ((_conv(5, 64, 1), 5, 8, 64, 0, False, True), (False, False, False)),
    'cin 64 of a Cin-128 1x1': ((_conv(128, 64, 1), 64, 128, 64, 0, False, False), (False, False, False)),
    '5x5/s2': ((_conv(64, 64, 5, stride=2), 64, 64, 64, 0, False, False), (False, True, False)),
    '5x5/s2 residual': ((_conv(64, 64, 5, stride=2), 64, 64, 64, 0, False, True), (False, True, False)),
    '5x5/s2 pixel shuffle': ((_conv(64, 64, 5, stride=2), 64, 64, 16, 0, True, False), (False, False, False)),
    '5x5/s2 dilation 2': ((_conv(64, 64, 5, stride=2, dil=2), 64, 64, 64, 0, False, False), (False, False, False)),
    '5x5/s2 Cout 120': ((_conv(64, 120, 5, stride=2), 64, 64, 120, 0, False, False), (False, False, False)),
    '1x1 192 -> 120': ((_conv(192, 120, 1), 192, 192, 120, 0, False, False), (True, True, True)),
    '1x1 128 -> 256': ((_conv(128, 256, 1), 128, 128, 256, 0, False, False), (True, True, True)),
    '1x1 odd Cout': ((_conv(192, 151, 1), 192, 192, 151, 0, False, False), (True, False, False)),
    '1x1 Cout 320': ((_conv(192, 320, 1), 192, 192, 320, 0, False, False), (True, False, False)),
    '1x1 residual': ((_conv(192, 120, 1), 192, 192, 120, 0, False, True), (True, False, False)),
    '1x1 pixel shuffle': ((_conv(192, 120, 1), 192, 192, 30, 0, True, False), (False, False, False)),
    '1x1 Cin 96': ((_conv(96, 64, 1), 96, 96, 64, 0, False, False), (False, False, False)),
}


@pytest.mark.parametrize('case', sorted(ROUTES))
def test_route_of_each_mode(case):
    from l3c_pytorch_b200 import engine as E
    args, want = ROUTES[case]
    assert not E.on_tensor_cores(FP32, *args)
    got = tuple(E.on_tensor_cores(mode, *args) for mode in (TF32, F16, F16X2))
    assert got == want, (case, got, want)


class _RecordingLib(object):
    """Stands in for libl3c_b200.so: records the conv descriptors and the splits, launches nothing."""

    def __init__(self):
        self.convs, self.splits = [], []

    def l3c_conv2d(self, desc, stream):
        d = desc._obj
        self.convs.append({f: getattr(d, f) for f, _ in d._fields_})
        return 0

    def l3c_split_f16x2(self, x, rows, C, out, stream):
        self.splits.append((x.value, out.value))
        return 0


@pytest.fixture
def host_engine(monkeypatch):
    from l3c_pytorch_b200 import engine as E
    rec = _RecordingLib()
    monkeypatch.setattr(E, 'lib', rec)
    monkeypatch.setattr(E, 'require_cuda', lambda t, name: t.is_cuda)
    monkeypatch.setattr(E, '_stream_ptr', lambda: None)
    return E, rec


def _layer(cin, cout, k):
    torch.manual_seed(0)
    return torch.nn.Conv2d(cin, cout, k, padding=k // 2)


def test_f16x2_reads_a_split_only_input_on_the_tensor_cores(host_engine):
    """Act(None, split image): the input pitch is half the image's, so the 3x3 and 1x1 layers take the split kernels
    on that image as it is; an fp32-only input is split first."""
    E, rec = host_engine
    x = torch.randn(2, 6, 10, 64)
    img = torch.cat(E._split_host(x), -1).contiguous()
    E.conv2d(_layer(64, 64, 3), E.Act(None, img), precision=F16X2)
    d = rec.convs[-1]
    assert (d['precision'], d['x_h'], d['x_pitch'], d['ksize']) == (F16X2, img.data_ptr(), 128, 3)
    E.conv2d(_layer(64, 120, 1), E.Act(None, img), precision=F16X2)
    d = rec.convs[-1]
    assert (d['precision'], d['x_h'], d['x_pitch'], d['ksize']) == (F16X2, img.data_ptr(), 128, 1)
    assert not rec.splits
    E.conv2d(_layer(64, 64, 3), x, precision=F16X2)
    assert len(rec.splits) == 1 and rec.splits[0][0] == x.data_ptr()
    assert rec.convs[-1]['x_h'] == rec.splits[0][1]


@pytest.mark.parametrize('mode', [FP32, TF32, F16, F16X2])
def test_ffma_layers_read_the_fp32_activation(host_engine, mode):
    """A Cin = 5 layer in a pitch-8 buffer runs on the FFMA kernel (precision fp32 in the descriptor) in every mode,
    reading x.f."""
    E, rec = host_engine
    x = torch.zeros(2, 6, 10, 8)
    E.conv2d(_layer(5, 64, 1), x, precision=mode)
    d = rec.convs[-1]
    assert (d['precision'], d['x'], d['x_pitch'], d['x_h']) == (FP32, x.data_ptr(), 8, None)
