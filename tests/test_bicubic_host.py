"""CPU: an integer restatement of Pillow's x0.5 BICUBIC resize, pinned bit for bit to the installed Pillow.

The RGB baselines' encoder is Pillow's `Image.resize((int(w * 0.5), int(h * 0.5)), BICUBIC)` of the uint8 image
(csrc/bicubic.cu restates it on the GPU).  Pillow is an unpinned dependency, so `pillow_half` below restates its
published two-pass algorithm (libImaging/Resample.c) in int64 numpy, written from the algorithm rather than from
bicubic.cu:

* Keys cubic with a = -0.5, support 2 * scale, filter argument (x + xmin - center + 0.5) * (1 / scale);
* xmin = (int)(center - support + 0.5), xmax = (int)(center + support + 0.5): C truncation, then clipped to the input;
* weights normalised by their sum (summed in tap order, as the C loop does), then rounded half away from zero to
  22-bit fixed point;
* accumulator started at 2**21, arithmetic shift by 22, clamp to [0, 255];
* the horizontal pass first, with a uint8 intermediate -- except for images more than 100 times taller than wide
  (H > 100 * W), which Pillow 12 resizes vertically first, again through a uint8 intermediate
  (test_tall_images_run_the_vertical_pass_first pins where it switches).

This file checks the restatement against Pillow on every (H, W) in 2..40 x 2..40 and on the large and extreme shapes
the codec hands the kernel, shows that the content families drive the pre-clamp sums past both ends in both passes,
and that each plausible mis-restatement differs from Pillow.  test_gpu_bicubic.py checks the kernel against both."""
import functools
import math

import numpy as np
import pytest

PRECISION_BITS = 22
SIDES = range(2, 41)


def _cubic(x):
    """Keys cubic, a = -0.5, in the operation order of Pillow's bicubic_filter (double precision)."""
    a = -0.5
    x = np.abs(x)
    return np.where(x < 1.0, ((a + 2.0) * x - (a + 3.0)) * x * x + 1,
                    np.where(x < 2.0, (((x - 5) * x + 8) * x - 4) * a, 0.0))


@functools.lru_cache(maxsize=None)
def _taps(in_size, out_size, bound=np.trunc, scaled_support=True, rounded=True):
    """-> (idx, kk): int64 [out_size, ksize] input index and fixed-point coefficient of every tap (0 past the
    window).  The keywords select the mutants of test_mutants_differ_from_pillow."""
    scale = in_size / out_size
    fscale = max(scale, 1.0)
    support = 2.0 * fscale if scaled_support else 2.0
    ksize = int(math.ceil(support)) * 2 + 1
    center = (np.arange(out_size) + 0.5) * scale
    xmin = np.maximum(bound(center - support + 0.5).astype(np.int64), 0)
    xmax = np.minimum(bound(center + support + 0.5).astype(np.int64), in_size) - xmin
    t = np.arange(ksize)
    inside = t[None, :] < xmax[:, None]
    k = np.where(inside, _cubic(((t[None, :] + xmin[:, None]) - center[:, None] + 0.5) * (1.0 / fscale)), 0.0)
    ww = np.zeros(out_size)
    for j in range(ksize):                                  # sequential, not numpy's pairwise sum
        ww = ww + k[:, j]
    k = np.where(ww[:, None] != 0.0, k / np.where(ww == 0.0, 1.0, ww)[:, None], k)
    fixed = k * (1 << PRECISION_BITS)
    if rounded:
        kk = np.where(k < 0, np.trunc(-0.5 + fixed), np.trunc(0.5 + fixed))
    else:
        kk = np.trunc(fixed)
    idx = np.minimum(xmin[:, None] + t[None, :], in_size - 1)
    return idx, np.where(inside, kk, 0).astype(np.int64)


def _half(img, acc0=1 << (PRECISION_BITS - 1), vertical_first=None, mid='u8', **taps):
    """Both passes over the H and W axes of [..., H, W, C], in Pillow's order unless vertical_first is given;
    the pre-clamp sums are returned horizontal pass first whatever the order.  mid: what the first pass hands the second -- 'u8'
    (Pillow: shifted and clamped), 'int' (shifted, not clamped) or 'float' (the exact quotient, no rounding).
    -> (uint8 output, pre-clamp shifted sums of the horizontal pass, of the vertical pass)."""
    x = np.asarray(img)                                     # the products below are int64
    H, W = x.shape[-3], x.shape[-2]
    passes = [(-2, W, int(W * 0.5)), (-3, H, int(H * 0.5))]
    if H > 100 * W if vertical_first is None else vertical_first:
        passes.reverse()
    pre = []
    for p, (axis, n_in, n_out) in enumerate(passes):
        idx, kk = _taps(n_in, n_out, **taps)
        acc = acc0
        for t in range(kk.shape[1]):
            w = kk[:, t].reshape((-1,) + (1,) * (-axis - 1))
            acc = acc + np.take(x, idx[:, t], axis=axis) * w
        shifted = acc >> PRECISION_BITS if acc.dtype == np.int64 else np.floor(acc / (1 << PRECISION_BITS))
        pre.append(shifted)
        if p == 0 and mid == 'float':
            x = (acc - acc0) / float(1 << PRECISION_BITS)
        elif p == 0 and mid == 'int':
            x = shifted
        else:
            x = np.clip(shifted, 0, 255)
    ph, pv = pre if passes[0][0] == -2 else pre[::-1]
    return x.astype(np.uint8), ph, pv


def pillow_half(img_hwc_u8):
    """Pillow's x0.5 BICUBIC of uint8 [..., H, W, C] (any leading batch axes) -> (uint8 [..., H//2, W//2, C],
    int64 pre-clamp sums of the horizontal pass [..., H, W//2, C] and of the vertical pass [..., H//2, W//2, C])."""
    return _half(img_hwc_u8)


def pil_half(img_hwc_u8):
    """The installed Pillow on uint8 [..., H, W, 3], image by image, at the size the reference's resize_bicubic
    asks for: (int(w * 0.5), int(h * 0.5))."""
    from PIL import Image
    a = np.asarray(img_hwc_u8)
    flat = a.reshape((-1,) + a.shape[-3:])
    outs = []
    for im in flat:
        p = Image.fromarray(np.ascontiguousarray(im))
        w, h = p.size
        outs.append(np.asarray(p.resize((int(w * 0.5), int(h * 0.5)), Image.BICUBIC)))
    return np.stack(outs).reshape(a.shape[:-3] + outs[0].shape)


# ---------------------------------------------------------------------------------------------------------------
# content
# ---------------------------------------------------------------------------------------------------------------
def _planes(H, W):
    """name -> uint8 [H, W] of every content family except noise."""
    y, x = np.mgrid[0:H, 0:W]
    hot = np.zeros((H, W), np.uint8)
    hot[H // 2, W // 2] = 255
    return {
        'checker': np.where((x + y) % 2 == 0, 255, 0),
        'stripes_x2': np.where(x % 2 == 0, 255, 0),
        'stripes_y2': np.where(y % 2 == 0, 255, 0),
        'stripes_x3': np.where(x % 3 == 0, 255, 0),
        'stripes_y3': np.where(y % 3 == 0, 255, 0),
        'hot': hot,
        'cold': 255 - hot,
        'blocks': np.where((x // 8 + y // 8) % 2 == 0, 255, 0),
        'ramp_x': (x * 255) // max(W - 1, 1),
        'ramp_y': (y * 255) // max(H - 1, 1),
        'ramp_xy': ((x + y) * 255) // max(H + W - 2, 1),
        'zero': np.zeros((H, W)),
        'full': np.full((H, W), 255),
    }


def families(H, W, seed=0):
    """name -> uint8 [H, W, 3]: noise and the edge families.  The channels differ (the pattern, its transpose-like
    roll and its complement) so that a kernel mixing up channels fails."""
    rng = np.random.default_rng(seed * 100003 + H * 4099 + W)
    out = {'noise': rng.integers(0, 256, (H, W, 3), dtype=np.uint8)}
    for name, p in _planes(H, W).items():
        p = p.astype(np.uint8)
        out[name] = np.stack([p, np.roll(p, (1, 1), (0, 1)), 255 - p], -1)
    return out


FAMILIES = list(families(2, 2))


def stack(H, W, names=None, seed=0):
    f = families(H, W, seed)
    return np.stack([f[n] for n in (names or FAMILIES)])


# ---------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def sweep():
    """Every (H, W) in 2..40 x 2..40, every family: [(H, W, images [F, H, W, 3], Pillow's outputs)]."""
    return [(H, W, imgs, pil_half(imgs)) for H in SIDES for W in SIDES for imgs in [stack(H, W)]]


def test_restatement_equals_pillow_on_the_sweep(sweep):
    bad = []
    lo = [np.inf, np.inf]
    hi = [-np.inf, -np.inf]
    for H, W, imgs, want in sweep:
        got, ph, pv = pillow_half(imgs)
        assert got.shape == want.shape == (len(FAMILIES), H // 2, W // 2, 3)
        if not np.array_equal(got, want):
            bad.append((H, W))
        for i, p in enumerate((ph, pv)):
            lo[i], hi[i] = min(lo[i], p.min()), max(hi[i], p.max())
    n = sum(len(imgs) for _, _, imgs, _ in sweep)
    print('restatement vs Pillow: %d images, %d shapes, %d mismatching shapes; pre-clamp range h [%d, %d], '
          'v [%d, %d]' % (n, len(sweep), len(bad), lo[0], hi[0], lo[1], hi[1]))
    assert not bad, 'restatement differs from Pillow at %d shapes, e.g. %s' % (len(bad), bad[:8])
    # both clamps are reached in both passes: the test is not only about interior values
    assert lo[0] < 0 and hi[0] > 255 and lo[1] < 0 and hi[1] > 255, (lo, hi)


@pytest.mark.parametrize('name', ['hot', 'cold', 'blocks'])
def test_edge_families_reach_both_clamps(name):
    """A hot pixel, a cold pixel and 8x8 blocks (each with its complement in another channel) drive the pre-clamp
    sums below 0 and above 255 in both passes.  Period-2 patterns do not: x0.5 flattens them to about 128."""
    _, ph, pv = pillow_half(stack(16, 16, [name]))
    assert ph.min() < 0 and ph.max() > 255 and pv.min() < 0 and pv.max() > 255, (ph.min(), ph.max(), pv.min(), pv.max())


@pytest.mark.parametrize('H,W', [(257, 515), (130, 206), (65, 103), (3, 4099), (4099, 3), (2001, 3003)])
def test_restatement_equals_pillow_on_large_and_extreme_shapes(H, W):
    names = ['noise', 'checker', 'stripes_x3', 'hot', 'blocks'] if H * W < 10 ** 6 else ['noise', 'blocks']
    imgs = stack(H, W, names, seed=1)
    got, ph, pv = pillow_half(imgs)
    want = pil_half(imgs)
    mism = np.argwhere(got != want)
    assert mism.size == 0, '%d mismatches, first at %s' % (len(mism), mism[:4].tolist())
    # both clamps in every pass that runs along an axis long enough to hold a block edge
    for p, n in ((ph, W), (pv, H)):
        assert n < 16 or (p.min() < 0 and p.max() > 255), (H, W, n, p.min(), p.max())


# Each plausible mis-restatement, as the keywords of _half.
MUTANTS = {
    'accumulator starts at 0': dict(acc0=0),
    'vertical pass first': dict(vertical_first=True),
    'horizontal pass first on tall images too': dict(vertical_first=False),
    'coefficients truncated': dict(rounded=False),
    'no clamp between passes': dict(mid='int'),
    'float intermediate': dict(mid='float'),
    'support not scaled': dict(scaled_support=False),
}


# Shapes on both sides of Pillow's switch to the vertical pass first (H > 100 * W).
TALL = [(H, W) for W in (2, 3, 5) for H in (100 * W, 100 * W + 1)] + [(4099, 3), (4099, 40)]


@pytest.fixture(scope='module')
def tall():
    return [(H, W, imgs, pil_half(imgs)) for (H, W) in TALL for imgs in [stack(H, W, ['noise', 'blocks', 'hot'])]]


def test_tall_images_run_the_vertical_pass_first(tall):
    """Pillow 12 resizes an image with H > 100 * W vertically first and every other image horizontally first: on
    each side of the switch exactly one order reproduces it."""
    for H, W, imgs, want in tall:
        v_first = H > 100 * W
        assert np.array_equal(pillow_half(imgs)[0], want), (H, W)
        assert np.array_equal(_half(imgs, vertical_first=v_first)[0], want), (H, W)
        assert not np.array_equal(_half(imgs, vertical_first=not v_first)[0], want), (H, W)


@pytest.mark.parametrize('mutant', sorted(MUTANTS))
def test_mutants_differ_from_pillow(sweep, tall, mutant):
    kw = MUTANTS[mutant]
    bad = sum(not np.array_equal(_half(imgs, **kw)[0], want) for _, _, imgs, want in sweep + tall)
    print('%s: differs from Pillow at %d of %d shapes' % (mutant, bad, len(sweep) + len(tall)))
    assert bad > 0, '%s is indistinguishable from Pillow on the sweep' % mutant


def test_floor_for_the_window_start_is_equivalent(sweep):
    """floor instead of truncation for xmin / xmax cannot change the result: the two differ only on negative
    arguments, which the clip to the input maps to 0 either way (center + support + 0.5 is always positive).  So
    this variant is not a mutant any test can reject; this pins that it is indeed the same on the whole sweep."""
    assert all(np.array_equal(_half(imgs, bound=np.floor)[0], want) for _, _, imgs, want in sweep)
