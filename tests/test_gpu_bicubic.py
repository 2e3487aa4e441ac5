"""GPU: the RGB baselines' encoder, l3c_bicubic_half_u8 (csrc/bicubic.cu via engine.bicubic_half), bit for bit
against Pillow and against the integer restatement of test_bicubic_host.py, at every size the codec hands it.

A. every (H, W) in 2..40 x 2..40, three contents per call;
B. output widths across the 128-thread blocks of the x grid, tall narrow and wide flat images (the tall ones run
   the vertical pass first, as Pillow does);
C. batches of 1, 2, 7 and 64 images: each equals its own single-image call (the plane index in gridDim.z);
D. the grid limits: the largest accepted H and plane count are correct, anything past them, and H or W below 2,
   raises RuntimeError before any launch and leaves the output alone;
E. 12-megapixel images, as tiled and crop=False containers hand them whole;
F. side streams: on a torch side stream while the default stream is busy, behind an input written late on its
   own stream, and on Bitcoding.side_stream;
G. every bicubic call of every RGB-baseline entry point (batches, padding, recursion, tiles, the banded crop=False
   encode, the CLI, the harness), recorded and compared; and the forward's thumbnails at every scale against
   oracle.model.encoder_side, whose chain runs in real Pillow."""
import numpy as np
import pytest
import torch

from tests import util
from tests.test_bicubic_host import SIDES, families, pil_half, pillow_half, stack

pytestmark = pytest.mark.gpu


def _dev(imgs):
    """uint8 [N, H, W, 3] numpy -> uint8 [N, 3, H, W] on the GPU."""
    return torch.from_numpy(np.ascontiguousarray(imgs)).permute(0, 3, 1, 2).contiguous().cuda()


def _restate(imgs):
    if imgs[0].size > 4 * 10 ** 6:                          # image by image: the int64 sums of a batch are large
        return np.stack([pillow_half(im)[0] for im in imgs])
    return pillow_half(imgs)[0]


def _check(got, imgs, what):
    """got: the kernel's uint8 [N, 3, H/2, W/2]; imgs: its input, uint8 [N, H, W, 3] numpy."""
    got = got.permute(0, 2, 3, 1).cpu()
    want = torch.from_numpy(_restate(imgs))
    pil = torch.from_numpy(pil_half(imgs))
    r, p = torch.equal(got, want), torch.equal(got, pil)
    if r and p:
        return
    ref = want if not r else pil
    where = (got != ref).nonzero()[:4].tolist() if got.shape == ref.shape else 'shape %s' % (tuple(got.shape),)
    raise AssertionError('%s: the kernel matches %s (restatement == Pillow: %s); first differences at %s'
                         % (what, 'the restatement only' if r else 'Pillow only' if p else 'neither',
                            torch.equal(want, pil), where))


def _half(imgs):
    from l3c_pytorch_b200 import engine as E
    return E.bicubic_half(_dev(imgs))


# ---- A. sweep -------------------------------------------------------------------------------------------------
def test_sweep_every_small_shape():
    names = list(families(2, 2))
    for H in SIDES:
        for W in SIDES:
            # noise, and two edge families rotating over the sweep so that every family meets every residue
            k = H * 41 + W
            imgs = stack(H, W, ['noise', names[1 + k % (len(names) - 1)], names[1 + (k * 7 + 3) % (len(names) - 1)]])
            _check(_half(imgs), imgs, (H, W))


# ---- B. block edges of the x grid, tall and flat ---------------------------------------------------------------
@pytest.mark.parametrize('H', [5, 6])
def test_output_widths_across_x_blocks(H):
    for W in list(range(254, 260)) + list(range(510, 516)):
        imgs = stack(H, W, ['noise', 'blocks', 'stripes_x3'], seed=2)
        _check(_half(imgs), imgs, (H, W))


@pytest.mark.parametrize('n', [2, 3, 4, 5])
def test_tall_narrow_and_wide_flat(n):
    for H, W in ((4099, n), (n, 4099)):
        imgs = stack(H, W, ['noise', 'blocks', 'hot'], seed=3)
        _check(_half(imgs), imgs, (H, W))


# ---- C. batches -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('N,H,W', [(1, 300, 517), (2, 67, 259), (7, 130, 206), (64, 33, 257)])
def test_batches_equal_single_image_calls(N, H, W):
    names = list(families(2, 2))
    pool = families(H, W, seed=N)
    imgs = np.stack([pool[names[i % len(names)]] if i % 3 else families(H, W, seed=100 + i)['noise']
                     for i in range(N)])
    got = _half(imgs)
    _check(got, imgs, (N, H, W))
    for i in range(N):
        assert torch.equal(_half(imgs[i:i + 1])[0], got[i]), 'image %d of %d differs from its own call' % (i, N)


# ---- D. limits --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('N,H,W', [(1, 65535, 4), (1, 65535, 656), (21845, 2, 2), (21845, 3, 3)])
def test_largest_grids_are_correct(N, H, W):
    """H = 65535 on both pass orders (65535 x 4 runs the vertical pass first; at W = 656 the horizontal pass runs
    first with gridDim.y = 65535), and 3 * 21845 = 65535 planes in gridDim.z."""
    from l3c_pytorch_b200 import engine as E
    if N == 1:
        imgs = stack(H, W, ['noise'], seed=4)
    else:
        imgs = np.random.default_rng(N + H).integers(0, 256, (N, H, W, 3), dtype=np.uint8)
        imgs[::5] = np.where(np.indices((H, W)).sum(0) % 2 == 0, 255, 0).astype(np.uint8)[..., None]
    E.launch_log(reset=True)
    got = _half(imgs)
    torch.cuda.synchronize()
    assert E.launch_log(reset=True)[1] == 2
    _check(got, imgs, (N, H, W))


@pytest.mark.parametrize('N,H,W', [(1, 65536, 4), (21846, 2, 2), (1, 1, 8), (1, 8, 1), (2, 1, 1)])
def test_refused_before_any_launch(N, H, W):
    from l3c_pytorch_b200 import engine as E
    x = torch.zeros(N, 3, H, W, dtype=torch.uint8, device='cuda')
    out = torch.full((N, 3, max(H // 2, 1), max(W // 2, 1)), 77, dtype=torch.uint8, device='cuda')
    torch.cuda.synchronize()
    E.launch_log(reset=True)
    with pytest.raises(RuntimeError, match='l3c_bicubic_half_u8'):
        E.check(E.lib.l3c_bicubic_half_u8(E._ptr(x), N, H, W, E._ptr(out), E._stream_ptr()))
    with pytest.raises(RuntimeError, match='l3c_bicubic_half_u8'):
        E.bicubic_half(x)
    torch.cuda.synchronize()
    assert E.launch_log(reset=True)[1] == 0
    assert bool((out == 77).all()), 'a refused call wrote its output'


# ---- E. large ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H,W', [(3000, 4000), (2999, 4001)])
def test_large_images(H, W):
    imgs = stack(H, W, ['noise', 'blocks'], seed=5)
    _check(_half(imgs), imgs, (H, W))


# ---- F. streams -------------------------------------------------------------------------------------------------
def test_side_streams():
    from l3c_pytorch_b200 import Bitcoding, engine as E
    imgs = stack(130, 517, ['noise', 'blocks', 'hot'], seed=6)
    src = _dev(imgs)
    want = E.bicubic_half(src)
    _check(want, imgs, 'default stream')
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    # the default stream busy with other work while the side stream runs the kernel
    torch.cuda._sleep(200 * 1000 * 1000)
    with torch.cuda.stream(side):
        got = E.bicubic_half(src)
    side.synchronize()
    assert torch.equal(got.cpu(), want.cpu()), 'side stream beside a busy default stream'
    torch.cuda.synchronize()
    # the input written late on the side stream itself: the kernel must run behind that write
    for stream in (side, Bitcoding(util.blueprint('cr_rgb_shared')).side_stream(3)):
        x = torch.zeros_like(src)
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(50 * 1000 * 1000)
            x.copy_(src)
            got = E.bicubic_half(x)
            got_host = got.to('cpu', non_blocking=False)
        stream.synchronize()
        assert torch.equal(got_host, want.cpu()), 'input written late on %r' % (stream,)
    torch.cuda.synchronize()


# ---- G. every call the codec makes ------------------------------------------------------------------------------
class _Recorder(object):
    """engine.bicubic_half wrapped: every (input, output) of every call, as the codec made it."""

    def __init__(self, monkeypatch):
        from l3c_pytorch_b200 import engine as E
        self.calls = []
        orig = E.bicubic_half

        def bicubic_half(img_u8):
            out = orig(img_u8)
            self.calls.append((img_u8.clone(), out.clone()))
            return out
        monkeypatch.setattr(E, 'bicubic_half', bicubic_half)

    def verify(self, n_calls, smallest, largest, wide=True):
        """The case recorded what it claims (call count, smallest and largest input H x W, an output wider than
        one 128-thread block of the x grid), and every recorded output is Pillow's x0.5 of its input."""
        sizes = [tuple(i.shape[-2:]) for i, _ in self.calls]
        assert len(self.calls) == n_calls, sizes
        assert min(sizes, key=lambda s: s[0] * s[1]) == smallest, sizes
        assert max(sizes, key=lambda s: s[0] * s[1]) == largest, sizes
        assert any(o.shape[-1] > 128 for _, o in self.calls) == wide, sizes
        for k, (img, out) in enumerate(self.calls):
            _check(out, img.permute(0, 2, 3, 1).cpu().numpy(), 'call %d of %d, input %s' % (k, n_calls, tuple(img.shape)))


def _pyramid(H, W, n):
    """input sizes of n successive x0.5 calls from H x W: (smallest, largest)."""
    return (H >> (n - 1), W >> (n - 1)), (H, W)


def _images(N, H, W, seed):
    return torch.stack([util.make_image(seed + i, H, W) for i in range(N)])


def _pad_to(v, fac):
    return v + (-v) % fac


CASES = ['batch_n1', 'batch_n3', 'batch_rgb', 'padded_odd', 'recursive_shared_1', 'recursive_shared_2',
         'recursive_shared_3', 'recursive_rgb_1', 'recursive_rgb_2', 'tiled', 'banded_no_crop', 'cli', 'harness']


@pytest.mark.parametrize('case', CASES)
def test_every_codec_call(case, monkeypatch, tmp_path):
    from l3c_pytorch_b200 import Bitcoding
    shared, rgb = util.blueprint('cr_rgb_shared'), util.blueprint('cr_rgb')
    if case in ('batch_n1', 'batch_n3'):
        N, H, W = (1, 64, 520) if case == 'batch_n1' else (3, 72, 300)
        rec = _Recorder(monkeypatch)
        Bitcoding(shared).encode_batch(_images(N, H, W, 10))
        assert rec.calls[0][0].shape[0] == N
        rec.verify(1, (H, W), (H, W))
    elif case == 'batch_rgb':
        rec = _Recorder(monkeypatch)
        Bitcoding(rgb).encode_batch(_images(2, 64, 520, 20))
        rec.verify(3, *_pyramid(64, 520, 3))
    elif case == 'padded_odd':
        rec = _Recorder(monkeypatch)
        Bitcoding(shared).encode_batch(_images(1, 129, 205, 30))          # padded to 130 x 206
        rec.verify(1, (130, 206), (130, 206), wide=False)
        assert tuple(rec.calls[0][1].shape[-2:]) == (65, 103)
    elif case.startswith('recursive_'):
        R = int(case[-1])
        bp, ns, (H, W) = (shared, 1, (48, 520)) if 'shared' in case else (rgb, 3, (40, 600))
        fac = 2 ** (ns + R)
        rec = _Recorder(monkeypatch)
        Bitcoding(bp, recursive=R).encode_batch(_images(2, H, W, 40 + R))
        Hp, Wp = _pad_to(H, fac), _pad_to(W, fac)
        rec.verify(ns + R, *_pyramid(Hp, Wp, ns + R))
        deepest = tuple(rec.calls[-1][1].shape[-2:])
        assert deepest == (Hp // fac, Wp // fac)
        if case in ('recursive_shared_3', 'recursive_rgb_1', 'recursive_rgb_2'):
            assert deepest[0] <= 3, deepest
    elif case == 'tiled':
        rec = _Recorder(monkeypatch)
        Bitcoding(shared, tile=(16, 32), recursive=2).encode_batch(_images(2, 64, 520, 50))
        rec.verify(3, *_pyramid(64, 520, 3))
    elif case == 'banded_no_crop':
        from l3c_pytorch_b200 import auto_crop, codec
        H, W = 1800, 2000
        img = util.make_image(60, H, W)
        assert auto_crop.needs_crop(img.unsqueeze(0))                     # crop=True would code four crops
        monkeypatch.setattr(codec, 'TILED_ENCODE_BAND_PIXELS', 1 << 20)
        banded = []
        orig = codec.BatchCodec._encode_banded
        monkeypatch.setattr(codec.BatchCodec, '_encode_banded',
                            lambda self, *a, **kw: banded.append(1) or orig(self, *a, **kw))
        rec = _Recorder(monkeypatch)
        Bitcoding(shared, tile=(16, 32), recursive=1, crop=False).encode(img, str(tmp_path / 'big.l3c'))
        assert banded == [1]
        rec.verify(2, *_pyramid(H, W, 2))
    elif case == 'cli':
        from PIL import Image
        from l3c_pytorch_b200 import cli
        ck = str(tmp_path / 'ckpt.pt')
        torch.save({'net': util.cpu_state_dict(shared)}, ck)
        src = str(tmp_path / 'a.png')
        Image.fromarray(util.make_image(70, 40, 520).permute(1, 2, 0).contiguous().numpy()).save(src)
        rec = _Recorder(monkeypatch)
        assert cli.main(['--config', 'cr_rgb_shared', '--ckpt', ck, '--precision', 'f16',
                         'enc', src, str(tmp_path / 'a.l3c'), '--recursive', '2']) == 0
        rec.verify(3, *_pyramid(40, 520, 3))
    elif case == 'harness':
        from PIL import Image
        from l3c_pytorch_b200 import harness as Hs
        exp = tmp_path / 'logs' / '0306_0001 cr_rgb_shared oi'
        (exp / 'ckpts').mkdir(parents=True)
        torch.save({'net': util.cpu_state_dict(shared)}, str(exp / 'ckpts' / 'ckpt_0000000010.pt'))
        imgs = tmp_path / 'imgs'
        imgs.mkdir()
        for name, (h, w), seed in (('a', (64, 520), 80), ('b', (40, 300), 81)):
            Image.fromarray(util.make_image(seed, h, w).permute(1, 2, 0).contiguous().numpy()).save(
                str(imgs / (name + '.png')))
        rec = _Recorder(monkeypatch)
        assert Hs.main([str(tmp_path / 'logs'), '0306_0001', str(imgs), '--recursive', 'auto']) == 0
        # --recursive auto = 3 on cr_rgb_shared: one forward of 4 calls per image shape, padded to multiples of 16
        rec.verify(8, (6, 38), (64, 528))


@pytest.mark.parametrize('cfg,R,H,W', [('cr_rgb_shared', 3, 64, 528), ('cr_rgb', 2, 64, 544)])
def test_forward_thumbnails_equal_the_oracle_chain(cfg, R, H, W):
    """forward(auto_recurse=R).S_u8 at every scale against oracle.model.encoder_side, which downsamples with
    Pillow itself (pillow_bicubic_half) from the oracle's own sub_rgb_mean."""
    from oracle import model as om
    bp = util.blueprint(cfg)
    ns = bp.net.scales
    x = torch.stack([util.make_image(90, H, W), torch.from_numpy(stack(H, W, ['blocks'])[0]).permute(2, 0, 1)])
    out = bp.forward(x.cuda(), auto_recurse=R)
    assert len(out.S_u8) == ns + R + 1
    sd = {k: v.detach().cpu().double() for k, v in bp.net.state_dict().items()}
    cfg_o = om.CFG_RGB_SHARED._replace(num_scales=ns + R)
    S, _ = om.encoder_side(sd, cfg_o, om._conv(sd, 'sub_rgb_mean', x.double()))
    for k in range(ns + R):
        got = out.S_u8[k + 1].cpu()
        assert torch.equal(got.long(), S[k]), 'scale %d' % (k + 1)
