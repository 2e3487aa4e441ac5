"""GPU: recursive containers of the RGB baselines (DESIGN §4.7): the last trained scale codes its own bicubic
thumbnails R more times, and only the 1 / 2**(num_scales + R) thumbnail is left for the uniform prior.

* Stream identity: every recursive scale's streams equal, byte for byte, the RGB-scale streams of the ordinary
  container of that thumbnail coded as an image -- which pins the recursive scales to code paths already tested
  against the reference.
* Round trips in every precision, with padding, batches and tiles; the decoder's symbols and parameters at every
  scale against the forward pass; launch shape; refusals before any kernel runs; async paths; the harness."""
import contextlib
import os
import re
import struct

import numpy as np
import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def _precision(mode):
    from l3c_pytorch_b200 import engine as E
    old = E.get_conv_precision()
    E.set_conv_precision(mode)
    try:
        yield
    finally:
        E.set_conv_precision(old)


def _launches(name, kernels):
    return sum(n for k, n in kernels.items() if name in k)


def _streams(data):
    """[(C, H, W, [stream bytes])] coarse -> fine of one container."""
    from l3c_pytorch_b200.codec import parse_container
    _, scales = parse_container(data)
    return [(C, H, W, [bytes(data[o:o + n]) for (o, n) in st]) for (C, H, W, st) in scales]


@pytest.mark.parametrize('mode', ['f16', 'f16x2'])
@pytest.mark.parametrize('R', [1, 2, 3])
def test_recursive_streams_equal_the_containers_of_the_thumbnails(mode, R):
    from l3c_pytorch_b200.codec import BatchCodec
    bp = util.blueprint('cr_rgb_shared')
    codec = BatchCodec(bp)
    x = util.make_image(70 + R, 64, 48).unsqueeze(0).cuda()
    with _precision(mode):
        rec = _streams(codec.encode_batch(x, recursive=R)[0][0])
        out = bp.forward(x, auto_recurse=R)
        assert len(rec) == R + 2 and [s[:3] for s in rec] == [tuple(S.shape[1:]) for S in reversed(out.S_u8)]
        for k in range(1, R + 1):
            S_k = out.S_u8[k].contiguous()
            plain = _streams(codec.encode_batch(S_k)[0][0])                     # uniform S_{k+1} | RGB scale S_k
            assert len(plain) == 2 and plain[1][:3] == rec[R + 1 - k][:3]
            assert plain[1][3] == rec[R + 1 - k][3], 'recursive scale %d differs from its thumbnail\'s container' % k
            if k == R:
                assert plain[0] == rec[0], 'uniform thumbnail differs'


@pytest.mark.parametrize('mode', ['f16', 'f16x2', 'tf32', 'fp32'])
@pytest.mark.parametrize('R', [1, 2, 3])
def test_recursive_round_trip_rgb_shared(mode, R):
    from l3c_pytorch_b200 import Bitcoding
    bp = util.blueprint('cr_rgb_shared')
    with _precision(mode):
        bc = Bitcoding(bp, recursive=R)
        pair = [util.make_image(80 + i, 40, 28) for i in range(2)]              # padded to multiples of 2**(1+R)
        datas, bpsps = bc.encode_batch(pair)
        fac = 2 ** (1 + R)
        hp, wp = 40 + (-40) % fac, 28 + (-28) % fac
        for d, b in zip(datas, bpsps):
            assert len(_streams(d)) == R + 2 and b == len(d) * 8 / (3 * hp * wp)    # padded sub-pixels
        for im, back in zip(pair, bc.decode_batch(datas)):
            assert torch.equal(back[0].cpu(), im.long())
        big = util.make_image(90 + R, 136, 72)
        datas, _ = bc.encode_batch(big.unsqueeze(0))
        assert torch.equal(bc.decode_batch(datas)[0][0].cpu(), big.long())
        # tiled containers
        bt = Bitcoding(bp, tile=(16, 16), recursive=R)
        batch = torch.stack([util.make_image(95 + i, 64, 48) for i in range(3)])
        datas, _ = bt.encode_batch(batch)
        for i, back in enumerate(Bitcoding(bp).decode_batch(datas)):              # R and tile come from the file
            assert torch.equal(back[0].cpu(), batch[i].long())


@pytest.mark.parametrize('mode', ['f16', 'fp32'])
@pytest.mark.parametrize('R', [1, 2])
def test_recursive_round_trip_rgb(mode, R):
    from l3c_pytorch_b200 import Bitcoding
    bp = util.blueprint('cr_rgb')
    with _precision(mode):
        bc = Bitcoding(bp, recursive=R)
        imgs = torch.stack([util.make_image(100 + i, 72, 40) for i in range(2)])
        datas, _ = bc.encode_batch(imgs)
        assert all(len(_streams(d)) == 3 + R + 1 for d in datas)
        for i, back in enumerate(bc.decode_batch(datas)):
            assert torch.equal(back[0].cpu(), imgs[i].long())


@pytest.mark.parametrize('mode', ['f16', 'fp32'])
@pytest.mark.parametrize('cfg,R', [('cr_rgb_shared', 3), ('cr_rgb', 2)])
def test_decoder_reproduces_every_scale_of_the_forward(monkeypatch, cfg, R, mode):
    """The decoded symbols of every scale equal forward(auto_recurse=R).S_u8, the decoder's parameters equal its
    P_nhwc bit for bit, and so does the get_P_nhwc chain run from the forward's own bottlenecks."""
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200.codec import BatchCodec
    bp = util.blueprint(cfg)
    net = bp.net
    ns = net.scales
    codec = BatchCodec(bp)
    x = torch.stack([util.make_image(110 + i, 64, 64) for i in range(2)]).cuda()
    with _precision(mode):
        out = bp.forward(x, auto_recurse=R)
        # the get_P_nhwc chain with MultiscaleNetwork._forward's fusion rule
        F = None
        for k in reversed(range(ns + R)):
            fuse = net._fuse_feat and k < ns - 1
            l, F = net.get_P_nhwc(k, out.bn8[k + 1], F if fuse else None)
            assert torch.equal(l, out.P_nhwc[k]), 'get_P_nhwc differs at scale %d' % k
        # the decoder: symbols fed to the next finer scale and the parameters it builds
        datas, _ = codec.encode_batch(x, recursive=R)
        seen_S, seen_P = {}, {}
        to_values, get_P = E.symbols_to_values, net.get_P_nhwc

        def spy_values(S, *a, **kw):
            seen_S[S.shape[-1]] = S.clone()
            return to_values(S, *a, **kw)

        def spy_P(scale, *a, **kw):
            l, F = get_P(scale, *a, **kw)
            seen_P[scale] = l.clone()
            return l, F
        monkeypatch.setattr(E, 'symbols_to_values', spy_values)
        monkeypatch.setattr(net, 'get_P_nhwc', spy_P)
        S0, _ = codec.decode_batch(datas, to_host=False)
        monkeypatch.undo()
    assert torch.equal(S0, x)
    for k in range(1, ns + R + 1):
        assert torch.equal(seen_S[out.S_u8[k].shape[-1]], out.S_u8[k]), 'decoded scale %d differs' % k
    assert sorted(seen_P) == list(range(ns + R))
    for k in range(ns + R):
        assert torch.equal(seen_P[k].view(out.P_nhwc[k].shape), out.P_nhwc[k]), 'decoder parameters of scale %d' % k


def test_recursive_launch_shape():
    from l3c_pytorch_b200 import Bitcoding, engine as E
    bc = Bitcoding(util.blueprint('cr_rgb_shared'), recursive=3)
    batch = torch.stack([util.make_image(120 + i, 64, 64) for i in range(4)])
    with _precision('f16'):
        bc.encode_batch(batch)                                                  # warm-up
        torch.cuda.synchronize()
        E.launch_log(reset=True)
        datas, _ = bc.encode_batch(batch)
        torch.cuda.synchronize()
        enc, _ = E.launch_log(reset=True)
        assert _launches('ac_encode_kernel', enc) == 1, enc
        # fused heads at all four DMLL scales: no parameter tensor, no separate interval kernel
        assert _launches('lin_dmll_f16_kernel', enc) >= 4 and _launches('dmll_intervals_kernel', enc) == 0, enc
        back = bc.decode_batch(datas)
        torch.cuda.synchronize()
        dec, _ = E.launch_log(reset=True)
    for i in range(4):
        assert torch.equal(back[i][0].cpu(), batch[i].long())
    assert _launches('dmll_table_kernel', dec) == 0, dec                       # coarse records at every RGB scale
    assert _launches('dmll_coarse_kernel', dec) >= 3 * 4, dec


def _no_kernel_runs(fn):
    from l3c_pytorch_b200 import engine as E
    torch.cuda.synchronize()
    E.launch_log(reset=True)
    with pytest.raises(ValueError) as err:
        fn()
    kernels, total = E.launch_log(reset=True)
    assert total == 0, kernels
    return str(err.value)


def test_recursive_refusals_raise_before_any_kernel():
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200.codec import parse_container
    bcs = Bitcoding(util.blueprint('cr_rgb_shared'), recursive=3)
    bcl = Bitcoding(util.blueprint('cr'))
    img = util.make_image(130, 64, 64).unsqueeze(0)
    datas, _ = bcs.encode_batch(img)
    good = datas[0]
    assert 'RGB baselines' in _no_kernel_runs(lambda: bcl.decode_batch([good]))
    _, scales = parse_container(good)
    assert [s[:3] for s in scales] == [(3, 4, 4), (3, 8, 8), (3, 16, 16), (3, 32, 32), (3, 64, 64)]
    # header of the recursive 16x16 scale: u8 C, u16 H, u16 W right before its first stream-length field
    off = scales[2][3][0][0] - 4 - 5
    assert struct.unpack_from('<BHH', good, off) == (3, 16, 16)
    bad = bytearray(good)
    struct.pack_into('<BHH', bad, off, 3, 16, 12)
    assert 'twice the coarser' in _no_kernel_runs(lambda: bcs.decode_batch([bytes(bad)]))
    bad = bytearray(good)
    struct.pack_into('<BHH', bad, off, 1, 16, 16)                               # C = 1: the file no longer parses
    _no_kernel_runs(lambda: bcs.decode_batch([bytes(bad)]))
    with pytest.raises(ValueError):
        Bitcoding(util.blueprint('cr'), recursive=2)
    with pytest.raises(ValueError):
        bcl.codec.encode_batch(img.cuda(), recursive=1)
    assert torch.equal(bcs.decode_batch([good])[0][0].cpu(), img[0].long())


def test_recursive_zero_is_the_ordinary_container():
    from l3c_pytorch_b200 import Bitcoding
    bp = util.blueprint('cr_rgb_shared')
    batch = torch.stack([util.make_image(140 + i, 40, 28) for i in range(2)])
    for mode in ('f16', 'fp32'):
        with _precision(mode):
            assert Bitcoding(bp, recursive=0).encode_batch(batch) == Bitcoding(bp).encode_batch(batch)


def test_recursive_encode_on_the_side_stream_beside_a_recursive_decode():
    from l3c_pytorch_b200 import Bitcoding
    bc = Bitcoding(util.blueprint('cr_rgb_shared'), recursive=2)
    a = torch.stack([util.make_image(150 + i, 96, 64) for i in range(3)])
    b = torch.stack([util.make_image(160 + i, 96, 64) for i in range(3)])
    with _precision('f16'):
        datas_a, _ = bc.encode_batch(a)
        want_b, _ = bc.encode_batch(b)
        side = bc.side_stream(3)
        lane = bc.decode_lanes(3, n_lanes=1)[0]
        cur = torch.cuda.current_stream()
        job = bc.encode_batch_begin(b.pin_memory(), stream=side)
        lane.main.wait_stream(cur)
        with torch.cuda.stream(lane.main):
            dec_a = bc.decode_batch(datas_a, lane=lane)
        assert job.finish()[0] == want_b
        cur.wait_stream(lane.main)
        torch.cuda.synchronize()
    for i in range(3):
        assert torch.equal(dec_a[i][0].cpu(), a[i].long())


def test_harness_writes_and_decodes_recursive_files(tmp_path, capsys):
    from PIL import Image
    from l3c_pytorch_b200 import harness as H
    bp0 = util.blueprint('cr_rgb_shared')
    exp = tmp_path / 'logs' / '0306_0001 cr_rgb_shared oi'
    (exp / 'ckpts').mkdir(parents=True)
    torch.save({'net': {k: v.detach().cpu() for k, v in bp0.net.state_dict().items()}},
               str(exp / 'ckpts' / 'ckpt_0000000010.pt'))
    imgs = tmp_path / 'imgs'
    imgs.mkdir()
    for name, (h, w), seed in (('a', (64, 64), 1), ('b', (40, 28), 2)):
        Image.fromarray(util.make_image(seed, h, w).permute(1, 2, 0).contiguous().numpy()).save(
            str(imgs / (name + '.png')))
    out_dir = str(tmp_path / 'l3c_out')
    assert H.main([str(tmp_path / 'logs'), '0306_0001', str(imgs), '--write_to_files', out_dir, '--recursive', 'auto',
                   '--compare_theory']) == 0                                    # lossless: checked inside
    out = capsys.readouterr().out
    assert '--recursive=3' in out
    assert sorted(os.listdir(out_dir)) == ['a.l3c', 'b.l3c']
    for name in ('a', 'b'):
        with open(os.path.join(out_dir, name + '.l3c'), 'rb') as f:
            assert len(_streams(f.read())) == 1 + 3 + 1
    theory = re.findall(r'theory:  (.*) =>', out)
    assert len(theory) == 2 and all(len(t.split(' | ')) == 1 + 3 + 1 for t in theory), theory


def test_cli_encodes_recursively_and_decodes_from_the_file(tmp_path):
    from PIL import Image
    from l3c_pytorch_b200 import cli
    from l3c_pytorch_b200.codec import parse_container
    ck = str(tmp_path / 'ckpt.pt')
    torch.save({'net': util.cpu_state_dict(util.blueprint('cr_rgb_shared'))}, ck)
    src, out, back = str(tmp_path / 'a.png'), str(tmp_path / 'a.l3c'), str(tmp_path / 'back.png')
    img = util.make_image(170, 40, 28)
    Image.fromarray(img.permute(1, 2, 0).contiguous().numpy()).save(src)
    base = ['--config', 'cr_rgb_shared', '--ckpt', ck, '--precision', 'f16']
    assert cli.main(base + ['enc', src, out, '--recursive', 'auto']) == 0
    with open(out, 'rb') as f:
        assert len(parse_container(f.read())[1]) == 1 + 3 + 1
    assert cli.main(base + ['dec', out, back]) == 0
    assert np.array_equal(np.array(Image.open(back)), img.permute(1, 2, 0).numpy())
