"""Ragged batches (DESIGN §4.6), host side: the pass policy, the stream layout shared by all batches, and Python
models of the index maps of the two ragged kernels (ragged.cu) -- which pixels l3c_ragged_zero_halo writes and how
l3c_ragged_pack moves elements."""
import numpy as np
import pytest

from l3c_pytorch_b200.bitcoding import plan_passes


# ---------------------------------------------------------------------------------------------
# models of ragged.cu (thread -> element maps restated)
# ---------------------------------------------------------------------------------------------
def zero_halo_pixels(H, W, ext, halo):
    """pixels (n, y, x) zero_halo_kernel writes, in thread order"""
    out = []
    for n, (h, w) in enumerate(ext):
        h, w = min(h, H), min(w, W)
        wr, hb = min(w + halo, W), min(h + halo, H)
        right = h * (wr - w)
        count = right + (hb - h) * wr
        for px in range(halo * (H + W)):             # the grid bound of l3c_ragged_zero_halo
            if px >= count:
                break
            if px < right:
                y, x = px // (wr - w), w + px % (wr - w)
            else:
                j = px - right
                y, x = h + j // wr, j % wr
            out.append((n, y, x))
    return out


def pack(src, ext, compact_len, to_compact, H, W):
    """ragged_pack_kernel on [N*planes] planes (one element per entry)"""
    planes = src.shape[0] // len(ext)
    if to_compact:
        dst = np.full((src.shape[0], compact_len), -1, src.dtype)
        for pl in range(src.shape[0]):
            h, w = ext[pl // planes]
            for e in range(compact_len):
                dst[pl, e] = src[pl, (e // w) * W + e % w] if e < h * w else 0
    else:
        dst = np.full((src.shape[0], H * W), -1, src.dtype)
        for pl in range(src.shape[0]):
            h, w = ext[pl // planes]
            for e in range(H * W):
                y, x = e // W, e % W
                dst[pl, e] = src[pl, y * w + x] if (y < h and x < w) else 0
    return dst


EXTENTS = [(16, 16), (8, 24), (24, 8), (3, 5), (24, 24), (1, 1)]


@pytest.mark.parametrize('halo', [1, 2, 4])
def test_zero_halo_writes_exactly_the_band(halo):
    H, W = 24, 24
    got = zero_halo_pixels(H, W, EXTENTS, halo)
    assert len(got) == len(set(got))                                   # every pixel written once
    want = {(n, y, x) for n, (h, w) in enumerate(EXTENTS) for y in range(H) for x in range(W)
            if not (y < h and x < w) and y < h + halo and x < w + halo}
    assert set(got) == want


def test_pack_round_trips_and_zero_fills():
    rng = np.random.default_rng(0)
    H, W, planes = 24, 24, 2
    ext = [(16, 16), (8, 24), (24, 8), (24, 24)]
    src = rng.integers(1, 1000, (len(ext) * planes, H * W)).astype(np.int64)
    plen = max(h * w for (h, w) in ext)
    comp = pack(src, ext, plen, True, H, W)
    for pl in range(src.shape[0]):
        h, w = ext[pl // planes]
        img = src[pl].reshape(H, W)[:h, :w].reshape(-1)
        assert np.array_equal(comp[pl, :h * w], img)                   # row-major image, stream order
        assert not comp[pl, h * w:].any()
    back = pack(comp, ext, plen, False, H, W)
    for pl in range(src.shape[0]):
        h, w = ext[pl // planes]
        m = np.zeros((H, W), bool)
        m[:h, :w] = True
        assert np.array_equal(back[pl].reshape(H, W)[m], src[pl].reshape(H, W)[m])
        assert not back[pl].reshape(H, W)[~m].any()


# ---------------------------------------------------------------------------------------------
# stream layout (codec.stream_layout): the one rule the encode and decode descriptors are built from
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', ['equal', 'tiled', 'ragged'])
def test_stream_layout_follows_the_container_order(case):
    from l3c_pytorch_b200 import codec as C
    fin, tile = {'equal': ([(32, 48)] * 3, None),
                 'tiled': ([(40, 56)] * 3, (16, 24)),                   # edge tiles of every scale are partial
                 'ragged': ([(40, 24), (16, 48), (40, 48), (8, 8)], None)}[case]
    # cr-like: three 5-channel bottlenecks over the 3-channel image, coarse -> fine
    shapes_of = [[(s, 3 if s == 0 else 5, h >> s, w >> s) for s in (3, 2, 1, 0)] for (h, w) in fin]
    si, elem, n_sym, plane = C.stream_layout([[sh[1:] for sh in shs] for shs in shapes_of], tile)
    N = len(fin)
    assert si.shape == elem.shape == n_sym.shape and si.shape[0] == N
    assert plane.tolist() == [max(h * w for (_, _, h, w) in (shs[k] for shs in shapes_of)) for k in range(4)]
    for n, shs in enumerate(shapes_of):
        # the order ContainerLayout writes and parse_container reads: scale, channel, tile (row-major), each tile
        # holding min(th, rows left) x min(tw, columns left) symbols
        want = []
        for k, (_, Cc, h, w) in enumerate(shs):
            th, tw = tile or (h, w)
            offs = np.cumsum([0] + [min(th, h - y) * min(tw, w - x) for y in range(0, h, th) for x in range(0, w, tw)])
            want += [(k, c, o, m) for c in range(Cc) for (o, m) in zip(offs[:-1], np.diff(offs))]
        lens = np.arange(len(want)) % 5
        total, pieces, _ = C.ContainerLayout(shs, tile).header_and_offsets(lens, (0, 0, 0, 0))
        buf = bytearray(total)
        for (o, b) in pieces:
            buf[o:o + len(b)] = b
        _, scales = C.parse_container(bytes(buf))
        assert [k for k, (_, _, _, st) in enumerate(scales) for _ in st] == [k for (k, _, _, _) in want]
        assert si[n].tolist() == [k for (k, _, _, _) in want]
        assert n_sym[n].tolist() == [m for (_, _, _, m) in want]
        # equal-size and tiled batches: the element index the descriptors used before stream_layout existed
        if case != 'ragged':
            assert elem[n].tolist() == [(n * Cc + c) * shs[k][2] * shs[k][3] + o for (k, c, o, _) in want
                                        for Cc in [shs[k][1]]]
    # the streams of every scale cover disjoint ranges of [N][C][plane], image n channel c from (n*C + c) * plane on
    for k in range(4):
        Cc = shapes_of[0][k][1]
        m = si == k
        lo, hi = elem[m], elem[m] + n_sym[m]
        order = np.argsort(lo)
        assert (hi[order][:-1] <= lo[order][1:]).all() and lo.min() >= 0 and hi.max() <= N * Cc * plane[k]
        for n, shs in enumerate(shapes_of):
            covered = sorted(zip(elem[n][si[n] == k], n_sym[n][si[n] == k]))
            for c in range(Cc):
                start = (n * Cc + c) * plane[k]
                mine = [(a, b) for (a, b) in covered if start <= a < start + plane[k]]
                assert mine[0][0] == start and sum(b for (_, b) in mine) == shs[k][2] * shs[k][3]
                assert all(a + b == a2 for (a, b), (a2, _) in zip(mine, mine[1:]))        # one contiguous run


# ---------------------------------------------------------------------------------------------
# pass policy
# ---------------------------------------------------------------------------------------------
def test_pass_policy_sorts_packs_and_splits():
    shapes = [(64, 96), (32, 32), (768, 768), (40, 32), (32, 32), (512, 256)]
    # one pass: every index once
    p = plan_passes(shapes, budget=10 ** 9)
    assert p == [sorted(range(6), key=lambda i: (shapes[i], i))]
    # sorted by shape, ties in input order
    assert p[0][:2] == [1, 4]
    # budget: N * Hmax * Wmax of every pass within it, consecutive in sorted order
    for budget in (32 * 32 * 2, 64 * 96 * 3, 768 * 768, 768 * 768 * 2 - 1):
        passes = plan_passes(shapes, budget=budget)
        flat = [i for q in passes for i in q]
        assert flat == sorted(range(6), key=lambda i: (shapes[i], i))
        for q in passes:
            n = len(q) * max(shapes[i][0] for i in q) * max(shapes[i][1] for i in q)
            assert n <= budget or len(q) == 1                          # an oversized image goes alone
    assert plan_passes(shapes, budget=1) == [[i] for i in sorted(range(6), key=lambda i: (shapes[i], i))]
    assert plan_passes([]) == []


def test_default_budget_makes_the_mixed_benchmark_one_pass():
    from l3c_pytorch_b200 import bitcoding
    assert len(plan_passes([(768, 768)] * 16)) == 1
    assert len(plan_passes([(768, 768)] * 17)) == 2
    assert bitcoding.RAGGED_PASS_PIXELS == 16 * 768 * 768
