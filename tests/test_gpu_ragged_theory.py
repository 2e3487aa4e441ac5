"""GPU: theoretical bpsp of ragged batches (DESIGN §4.6) -- the per-image NLL over each image's extent
(l3c_dmll_nll_ragged), the per-image losses of a ragged forward, and the harness evaluating a test set of many
sizes in ragged passes.  Every number must carry the bits of evaluating the image alone."""
import math

import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture
def f16():
    from l3c_pytorch_b200 import engine as E
    old = E.get_conv_precision()
    E.set_conv_precision('f16')
    yield
    E.set_conv_precision(old)


# ---------------------------------------------------------------------------------------------
# kernel
# ---------------------------------------------------------------------------------------------
# 8 x 8; widths that are not multiples of 16; (40, 56) spans 18 blocks of 128 pixels, the others at most 8
NLL_EXT = [(8, 8), (24, 40), (40, 56), (16, 24), (8, 40)]


def _nll_case(dm, C, seed):
    """NaN-filled padded parameters and garbage symbols around random ones inside NLL_EXT; a quarter of the
    pixels has log-scales at the -7 clamp or just below it (peaked mixtures)."""
    g = torch.Generator().manual_seed(seed)
    K = 10
    Kp = (4 if dm.rgb_scale else 3) * C * K
    H, W = max(h for h, _ in NLL_EXT), max(w for _, w in NLL_EXT)
    N = len(NLL_EXT)
    l = torch.full((N, H, W, Kp), float('nan'))
    sym = torch.full((N, C, H, W), 255, dtype=torch.uint8)
    for n, (h, w) in enumerate(NLL_EXT):
        p = torch.randn(h, w, Kp, generator=g)
        p[..., C * K:2 * C * K] = p[..., C * K:2 * C * K] * (dm.x_max - dm.x_min) / 4 + (dm.x_max + dm.x_min) / 2
        ls = torch.rand(h, w, C * K, generator=g) * 4 - 3
        peaked = torch.rand(h, w, 1, generator=g) < 0.25
        ls = torch.where(peaked, -7.25 + torch.rand(h, w, C * K, generator=g) * 0.5, ls)
        p[..., 2 * C * K:3 * C * K] = ls
        l[n, :h, :w] = p
        sym[n, :, :h, :w] = torch.randint(0, dm.L, (C, h, w), generator=g, dtype=torch.uint8)
    return l.cuda(), sym.cuda()


@pytest.mark.parametrize('scale', ['rgb', 'bottleneck'])
def test_ragged_nll_equals_per_image_nll(scale):
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    dm, C = (bp.losses.loss_dmol_rgb, 3) if scale == 'rgb' else (bp.losses.loss_dmol_n, 5)
    l, sym = _nll_case(dm, C, 11 if scale == 'rgb' else 12)
    got = dm.nll_sum(sym, l, extents=NLL_EXT)
    assert got.dtype == torch.float64 and got.shape == (len(NLL_EXT),)
    for n, (h, w) in enumerate(NLL_EXT):
        want = dm.nll_sum(sym[n:n + 1, :, :h, :w].contiguous(), l[n:n + 1, :h, :w].contiguous())
        assert torch.isfinite(want).all(), (scale, n)
        assert torch.equal(got[n:n + 1], want), (scale, n, float(got[n]), float(want[0]))
    # a batch whose images fill the plane gives what the equal-size kernel gives
    H, W = l.shape[1:3]
    lf, sf = l.nan_to_num(0.5), torch.where(sym < dm.L, sym, torch.zeros_like(sym))
    assert torch.equal(dm.nll_sum(sf, lf, extents=[(H, W)] * len(NLL_EXT)), dm.nll_sum(sf, lf))
    # extents that do not fit the batch are refused before anything is launched ...
    for bad in ([(0, 8)] + NLL_EXT[1:], [(H + 1, 8)] + NLL_EXT[1:], [(8, W + 8)] + NLL_EXT[1:], NLL_EXT[:-1]):
        with pytest.raises(ValueError):
            dm.nll_sum(sym, l, extents=bad)
    # ... and the native entry point reads nothing of such an image: it reports NaN for it alone
    vals = dm.values(l.device)
    ext = torch.tensor([(H + 8, 8)] + NLL_EXT[1:], dtype=torch.int32, device=l.device)
    out = torch.zeros(len(NLL_EXT), dtype=torch.float64, device=l.device)
    E.check(E.lib.l3c_dmll_nll_ragged(E._ptr(l), E._ptr(sym), E._ptr(vals), len(NLL_EXT), H, W, C, 10, dm.L,
                                      int(dm.rgb_scale), float(dm.x_min), float(dm.x_max), E._ptr(ext), E._ptr(out),
                                      E._stream_ptr()))
    assert math.isnan(float(out[0])) and torch.equal(out[1:], got[1:])


# ---------------------------------------------------------------------------------------------
# model
# ---------------------------------------------------------------------------------------------
SHAPES = [(32, 32), (48, 24), (16, 64), (64, 40), (8, 8)]


def _batch(shapes, seed=0):
    Hb, Wb = max(h for h, _ in shapes), max(w for _, w in shapes)
    imgs = [util.make_image(seed + i, h, w) for i, (h, w) in enumerate(shapes)]
    batch = torch.zeros(len(shapes), 3, Hb, Wb, dtype=torch.uint8)
    for n, im in enumerate(imgs):
        batch[n, :, :im.shape[1], :im.shape[2]] = im
    return imgs, batch.cuda()


def test_ragged_losses_equal_per_image_losses(f16):
    bp = util.blueprint('cr')
    imgs, batch = _batch(SHAPES, seed=30)
    out = bp.forward(batch, extents=SHAPES)
    assert out.extents == SHAPES
    got = bp.get_loss_per_image(out)
    explicit = [3 * (h - 3) * w for (h, w) in SHAPES]                  # e.g. the sub-pixels before padding
    got_explicit = bp.get_loss_per_image(out, num_subpixels_before_pad=explicit)
    nats, subpixels = 0.0, 0
    for n, im in enumerate(imgs):
        one = bp.forward(im.unsqueeze(0).cuda())
        assert one.extents is None
        assert got[n] == bp.get_loss_per_image(one)[0], n
        assert got_explicit[n] == bp.get_loss_per_image(one, num_subpixels_before_pad=explicit[n])[0], n
        nats += got[n] * math.log(2.) * 3 * SHAPES[n][0] * SHAPES[n][1]
        subpixels += 3 * SHAPES[n][0] * SHAPES[n][1]
    # get_loss sums the images' own costs, never the padding (all scales incl. the uniform one)
    total = float(sum(bp.get_loss(out).nonrecursive_bpsps))
    assert abs(total - nats / (math.log(2.) * subpixels)) < 1e-9 * total
    # the equal-size path is untouched: an Out without extents prices the whole tensor
    eq = bp.forward(batch)
    assert eq.extents is None and bp.get_loss_per_image(eq)[-1] != got[-1]


# ---------------------------------------------------------------------------------------------
# harness
# ---------------------------------------------------------------------------------------------
# (32, 32) and (64, 64) need no padding; (44, 36), (20, 36), (33, 17) do; 97 x 61 exceeds the 64 x 64 crop
# threshold and is cut into 48 x 30, 48 x 31, 49 x 30, 49 x 31 crops: padded, 48 x 32 and 56 x 32
HARNESS_SIZES = {'a': (64, 64), 'b': (44, 36), 'c': (32, 32), 'd': (20, 36), 'e': (33, 17), 'f': (97, 61),
                 'g': (32, 32)}


@pytest.fixture
def experiment(tmp_path, monkeypatch):
    from PIL import Image
    monkeypatch.setenv('AC_NEEDS_CROP_DIM', '64,64')
    bp0 = util.blueprint('cr')
    exp = tmp_path / 'logs' / '0306_0001 cr oi'
    (exp / 'ckpts').mkdir(parents=True)
    torch.save({'net': {k: v.detach().cpu() for k, v in bp0.net.state_dict().items()}},
               str(exp / 'ckpts' / 'ckpt_0000000010.pt'))
    imgs = tmp_path / 'imgs'
    imgs.mkdir()
    for i, (name, (h, w)) in enumerate(sorted(HARNESS_SIZES.items())):
        Image.fromarray(util.make_image(40 + i, h, w).permute(1, 2, 0).contiguous().numpy()).save(
            str(imgs / (name + '.png')))
    return str(tmp_path / 'logs'), str(imgs)


def _theory(logs, imgs, batch):
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200 import harness as H
    flags = H.build_parser().parse_args([logs, '0306_0001', imgs, '--overwrite_cache', '--batch', str(batch)])
    tester = H.Tester('0306_0001', flags, -1)
    calls = []
    fwd = tester.blueprint.forward

    def counting_forward(*a, **kw):
        calls.append(kw.get('extents'))
        return fwd(*a, **kw)
    tester.blueprint.forward = counting_forward
    E.launch_log(reset=True)
    res = tester.test(H.Testset(imgs))
    return res.per_img, calls, E.launch_log(reset=True)[0].get('rgb_im2col_kernel', 0)


def _crop_shapes(fac=8):
    from l3c_pytorch_b200 import auto_crop
    out = []
    for name, (h, w) in sorted(HARNESS_SIZES.items()):
        for c in auto_crop.iter_crops(torch.zeros(1, 3, h, w, dtype=torch.uint8)):
            out.append(tuple(c.shape[2:]))
    return out, [(h + (-h) % fac, w + (-w) % fac) for (h, w) in out]


def test_harness_evaluates_a_test_set_in_ragged_passes(experiment, f16):
    from l3c_pytorch_b200.bitcoding import plan_passes
    logs, imgs = experiment
    crops, padded = _crop_shapes()
    assert len(set(padded)) >= 5 and len(crops) == len(HARNESS_SIZES) + 3
    plan = plan_passes(padded, max_images=4)
    per_img, calls, passes = _theory(logs, imgs, 4)
    assert sorted(per_img) == sorted(HARNESS_SIZES)
    assert passes == len(calls) == len(plan) < len(set(padded)), (passes, len(calls), plan)
    assert [sorted(c) for c in calls] == [sorted(padded[i] for i in p) for p in plan]
    assert any(len(set(c)) > 1 for c in calls)
    # --batch 1: every crop evaluated alone
    alone, calls1, passes1 = _theory(logs, imgs, 1)
    assert passes1 == len(crops) and all(len(c) == 1 for c in calls1)
    for name in HARNESS_SIZES:
        assert per_img[name] == alone[name], (name, per_img[name], alone[name])
        assert math.isfinite(per_img[name]) and per_img[name] > 30.0, (name, per_img[name])


def test_harness_in_fp32_keeps_one_pass_per_shape(experiment):
    from l3c_pytorch_b200 import engine as E
    logs, imgs = experiment
    old = E.get_conv_precision()
    E.set_conv_precision('fp32')
    try:
        crops, _ = _crop_shapes()
        per_img, calls, _ = _theory(logs, imgs, 4)
        assert all(c is None for c in calls) and len(calls) == len(set(crops))
        alone, calls1, _ = _theory(logs, imgs, 1)
        assert len(calls1) == len(crops)
        for name in HARNESS_SIZES:
            assert per_img[name] == alone[name], (name, per_img[name], alone[name])
    finally:
        E.set_conv_precision(old)
