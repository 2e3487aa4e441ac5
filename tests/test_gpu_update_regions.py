"""GPU: batches of region updates (DESIGN §4.12, "Batches of updates"), BatchCodec.update_regions /
Bitcoding.update_regions.

* Result i is byte for byte encode(decode(datas[i]) with every patch pasted in order) and decodes losslessly to it:
  `cr` in f16, f16x2, tf32 and fp32, tiles (16, 16), (16, 24) and (64, 64), containers of different sizes in one call;
  edits far apart (kept as separate plans), overlapping (the later wins) and whose windows meet (merged); edges,
  corners, a 1 x 1 edit, an edit equal to the old pixels (bytes unchanged) and an empty edit list.
* The whole path (budget monkeypatched) for one container in the same call as window-path containers.
* The same bytes as the edits applied one after another with update_region.
* In f16 a call whose plans fit one pass makes one range-coder launch and one splice launch, runs the pass as one
  ragged batch of windows (l3c_dmll_intervals_rects) and gives the bytes of the plans run one after another.
* l3c_dmll_intervals_rects equals l3c_dmll_intervals_rect run per image, bit for bit; its refusals launch nothing.
* l3c_splice_streams equals the numpy splice (codec.splice_segments), guard bytes around the output intact; its
  refusals launch nothing.
* Every refusal raises, naming container and edit, before any kernel launch; the CLI `upd --edit` round trip."""
import os

import numpy as np
import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu

MODES = ['f16', 'f16x2', 'tf32', 'fp32']


@pytest.fixture
def mode():
    from l3c_pytorch_b200 import engine as E
    old = E.get_conv_precision()
    yield E.set_conv_precision
    E.set_conv_precision(old)


def _bc(tile, cfg='cr'):
    from l3c_pytorch_b200.bitcoding import Bitcoding
    return Bitcoding(util.blueprint(cfg, device='cuda:0'), tile=tile, crop=tile is None)


def _image(seed, H, W):
    """A seeded image with smooth structure and noise (uint8 [3, H, W] on the GPU)."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32),
                            indexing='ij')
    base = torch.stack([(yy * 0.37 + xx * 0.11) % 256, (xx * 0.29) % 256, (yy * 0.21 + 60) % 256])
    img = (base + torch.randint(-20, 21, (3, H, W), generator=g)).clamp(0, 255).to(torch.uint8)
    return img.cuda()


def _encode(bc, img):
    return bc.encode_batch([img])[0][0]


def _patch(seed, h, w):
    return torch.randint(0, 256, (3, h, w), generator=torch.Generator().manual_seed(seed), dtype=torch.int64)


def _edited(img, edits):
    out = img.clone()
    for (y, x), p in edits:
        p = p[0] if p.dim() == 4 else p
        out[:, y:y + p.shape[1], x:x + p.shape[2]] = p.to(torch.uint8).cuda()
    return out


def _case():
    """(images, edit lists): containers of different sizes and every kind of edit list."""
    imgs = [_image(1, 517, 389), _image(2, 301, 255), _image(3, 256, 4096), _image(4, 131, 97)]
    edits = [
        # overlapping (the second wins), an edge, a corner, a single pixel: one merged plan
        [((100, 90), _patch(1, 40, 33)), ((120, 100), _patch(2, 30, 30)), ((0, 150), _patch(3, 5, 17)),
         ((508, 378), _patch(4, 9, 11)), ((250, 0), _patch(5, 1, 1))],
        [],
        # far apart: two plans; the third edit lies inside the first one's window and is merged with it
        [((10, 50), _patch(6, 20, 30)), ((200, 3950), _patch(7, 30, 40)), ((40, 300), _patch(8, 8, 8))],
        # the old pixels themselves: the container comes back unchanged
        [((30, 20), imgs[3][:, 30:70, 20:61].unsqueeze(0))],
    ]
    return imgs, edits


def _check(bc, imgs, datas, edits, outs):
    for img, data, ed, got in zip(imgs, datas, edits, outs):
        edited = _edited(img, ed)
        assert got == _encode(bc, edited)
        assert torch.equal(bc.decode_batch([got])[0][0].to(torch.uint8), edited)


@pytest.mark.parametrize('prec', MODES)
@pytest.mark.parametrize('tile', [(16, 16), (16, 24), (64, 64)])
def test_updates_equal_encode_of_the_edited_images(mode, prec, tile):
    mode(prec)
    bc = _bc(tile)
    imgs, edits = _case()
    datas = [_encode(bc, img) for img in imgs]
    outs = bc.update_regions(datas, edits)
    _check(bc, imgs, datas, edits, outs)
    assert outs[1] == datas[1] and outs[3] == datas[3]
    c = bc.codec.updates_counts
    assert [x['plans'] for x in c] == [1, 0, 2, 1] and not any(x['whole'] for x in c)
    assert c[1]['streams'] == 0 and all(x['streams'] <= x['total'] for x in c)
    assert 0 < c[2]['streams'] < c[2]['total']


def test_same_bytes_as_sequential_updates():
    bc = _bc((16, 16))
    imgs, edits = _case()
    datas = [_encode(bc, img) for img in imgs]
    outs = bc.update_regions(datas, edits)
    for data, ed, got in zip(datas, edits, outs):
        for pos, patch in ed:
            data = bc.update_region(data, pos, patch)
        assert got == data


def test_whole_path_beside_window_paths(monkeypatch):
    from l3c_pytorch_b200 import codec
    bc = _bc((16, 24))
    imgs, edits = _case()
    imgs, edits = [imgs[i] for i in (0, 1, 3)], [edits[i] for i in (0, 1, 3)]
    datas = [_encode(bc, img) for img in imgs]
    bc.update_regions(datas, edits)
    big = bc.codec.updates_counts[0]['window_pixels']
    assert big > max(c['window_pixels'] for c in bc.codec.updates_counts[1:])
    monkeypatch.setattr(codec, 'TILED_ENCODE_BAND_PIXELS', big - 1)       # container 0's window exceeds the budget
    outs = bc.update_regions(datas, edits)
    c = bc.codec.updates_counts
    assert [x['whole'] for x in c] == [True, False, False]
    assert c[0]['streams'] == c[0]['total']
    _check(bc, imgs, datas, edits, outs)


def test_one_range_coder_launch_per_pass_in_f16(mode):
    from l3c_pytorch_b200 import engine as E
    mode('f16')
    bc = _bc((16, 16))
    imgs, edits = _case()
    datas = [_encode(bc, img) for img in imgs]
    torch.cuda.synchronize()
    E.launch_log(reset=True)
    outs = bc.update_regions(datas, edits)
    kernels, _ = E.launch_log(reset=True)
    assert kernels.get('ac_encode_kernel') == 1 and kernels.get('splice_streams_kernel') == 1, kernels
    _check(bc, imgs, datas, edits, outs)


def _numpy_splice(old, slots, seg, out):
    for src, so, d, n in seg.tolist():
        out[d:d + n] = (slots if src else old)[so:so + n]
        if src:
            out[d - 4:d] = np.frombuffer(np.uint32(n).tobytes(), np.uint8)


def test_splice_kernel_against_numpy():
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200.codec import ContainerLayout, splice_segments
    rng = np.random.default_rng(5)
    dev = torch.device('cuda:0')
    layout = ContainerLayout([(0, 5, 8, 12), (1, 5, 16, 24), (2, 3, 32, 48)], (8, 8))
    n = 5 * 2 + 5 * 6 + 3 * 24
    old_len = rng.integers(0, 300, n)
    total_old, old_off = layout.offsets(old_len)
    old = rng.integers(0, 256, total_old + 40, dtype=np.uint8)       # 40 bytes of another container before it
    cols = np.sort(rng.choice(n, 20, replace=False))
    lens = rng.integers(0, 400, cols.size)
    slot_off = np.concatenate([[0], np.cumsum(lens + 3)])[:-1]
    slots = rng.integers(0, 256, int(slot_off[-1] + lens[-1] + 16), dtype=np.uint8)
    new_len = old_len.copy()
    new_len[cols] = lens
    total, new_off = layout.offsets(new_len)
    seg = splice_segments(old_off, old_len, total_old, new_off, cols, lens, slot_off, src0=40, dst0=32)
    want = np.full(total + 64, 0xA5, np.uint8)
    _numpy_splice(old, slots, seg, want)
    old_d, slots_d = torch.from_numpy(old).to(dev), torch.from_numpy(slots).to(dev)
    out = torch.full((total + 64,), 0xA5, dtype=torch.uint8, device=dev)
    E.splice_streams(old_d, slots_d, seg, out)
    got = out.cpu().numpy()
    assert np.array_equal(got, want)
    assert (got[:32] == 0xA5).all() and (got[32 + total:] == 0xA5).all()
    E.launch_log(reset=True)
    bad = []
    assert seg[0, 3] > 0 and seg[1, 0] == 1
    for k, v in [((0, 0), 2), ((0, 3), -1), ((0, 1), total_old + 41), ((1, 1), len(slots)), ((1, 2), 2),
                 ((0, 2), total + 64)]:
        s = seg.copy()
        s[k] = v
        if k == (1, 1):
            s[1, 3] = max(s[1, 3], 1)                                # at least one byte past the slots' end
        bad.append(s)
    overlap = seg.copy()
    overlap[1, 2] = overlap[0, 2] + 1                                # a new stream over the run before it
    bad.append(overlap)
    for s in bad:
        with pytest.raises(RuntimeError):
            E.splice_streams(old_d, slots_d, s, out)
    seg_dev = torch.empty(5 * seg.shape[0] + 1, dtype=torch.int64, device=dev)
    assert E.lib.l3c_splice_streams(None, old_d.numel(), slots_d.data_ptr(), slots_d.numel(), seg.ctypes.data,
                                    seg_dev.data_ptr(), seg.shape[0], out.data_ptr(), out.numel(), None) != 0
    assert E.lib.l3c_splice_streams(old_d.data_ptr(), old_d.numel(), slots_d.data_ptr(), slots_d.numel(),
                                    seg.ctypes.data, None, seg.shape[0], out.data_ptr(), out.numel(), None) != 0
    assert E.launch_log()[1] == 0


def test_refusals_before_any_launch():
    from l3c_pytorch_b200 import engine as E
    bc = _bc((16, 16))
    img = _image(6, 64, 72)
    data = _encode(bc, img)
    ref_data = _encode(_bc(None), img)
    rgb = _bc((16, 16), 'cr_rgb_shared')
    rgb_data = _encode(rgb, img)
    ok = torch.zeros(3, 4, 4, dtype=torch.uint8)
    good = [((0, 0), ok)]
    cases = [(bc, [data, ref_data], [good, good], r'container 1: .*tiled container'),
             (bc, [rgb_data], [good], 'container 0 was not written by this model'),
             (rgb, [data, rgb_data], [[], []], 'container 0 was not written by this model'),
             (rgb, [rgb_data], [[]], 'container 0: .*RGB baselines'),
             (bc, [data, data], [good, good + [((0, 0), torch.zeros(3, 0, 4, dtype=torch.uint8))]],
              'container 1, edit 1: empty'),
             (bc, [data], [good + [((62, 0), ok)]], 'container 0, edit 1: .*outside'),
             (bc, [data], [[((0, -1), ok)]], 'container 0, edit 0: .*outside'),
             (bc, [data], [good * 3 + [((0, 0), torch.zeros(1, 4, 4, dtype=torch.uint8))]],
              'container 0, edit 3: .*3 channels'),
             (bc, [data], [[((0, 0), torch.full((3, 4, 4), 256, dtype=torch.int64))]], 'edit 0: .*0..255'),
             (bc, [data], [[((0, 0), torch.zeros(3, 4, 4, dtype=torch.float32))]], 'edit 0: .*uint8 or int64'),
             (bc, [data], [[((0, 0, 0), ok)]], r'edit 0: pos must be \(y, x\)'),
             (bc, [data], [good, good], '2 edit lists for 1 containers')]
    torch.cuda.synchronize()
    E.launch_log(reset=True)
    for b, ds, eds, match in cases:
        with pytest.raises(ValueError, match=match):
            b.update_regions(ds, eds)
    assert E.launch_log()[1] == 0


def test_cli_update_with_edits_round_trip(tmp_path):
    from PIL import Image
    from l3c_pytorch_b200 import cli
    img = _image(9, 131, 97)
    src = str(tmp_path / 'img.png')
    Image.fromarray(img.permute(1, 2, 0).cpu().numpy()).save(src)
    patches = []
    for k, (h, w) in enumerate([(20, 30), (10, 12), (7, 5)]):
        p = torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(k))
        path = str(tmp_path / ('patch%d.png' % k))
        Image.fromarray(p.numpy()).save(path)
        patches.append((path, p.permute(2, 0, 1)))
    enc, upd = str(tmp_path / 'a.l3c'), str(tmp_path / 'b.l3c')
    assert cli.main(['--config', 'cr', 'enc', src, enc, '--tile', '16,16']) == 0
    assert cli.main(['--config', 'cr', 'upd', enc, patches[0][0], '40,50', upd, '--edit', patches[1][0], '45,55',
                     '--edit', patches[2][0], '120,90']) == 0
    edited = _edited(img, [((40, 50), patches[0][1]), ((45, 55), patches[1][1]), ((120, 90), patches[2][1])])
    bc = _bc((16, 16))
    with open(upd, 'rb') as f:
        assert f.read() == _encode(bc, edited)
    assert cli.main(['--config', 'cr', 'upd', enc, patches[0][0], '40,50', upd, '--overwrite', '--edit',
                     patches[1][0], '130,0']) == 1                                    # outside the image
    assert cli.main(['--config', 'cr', 'upd', enc, patches[0][0], '40,50', upd, '--overwrite', '--edit',
                     patches[1][0], '1']) == 1                                        # not Y,X


@pytest.mark.parametrize('rgb', [True, False])
def test_rects_kernel_equals_the_rect_kernel_per_image(rgb):
    from l3c_pytorch_b200 import engine as E
    dev = torch.device('cuda:0')
    bp = util.blueprint('cr', device='cuda:0')
    dm = bp.losses.loss_dmol_rgb if rgb else bp.losses.loss_dmol_n
    C, K, L = (3 if rgb else 5), 10, dm.L
    Kp = (4 if rgb else 3) * C * K
    N, H, W, tile = 4, 48, 40, (16, 8)
    g = torch.Generator().manual_seed(9)
    l = (torch.randn(N, H + 6, W + 4, Kp, generator=g) * 2).to(dev).contiguous()
    sym = torch.randint(0, L, (N, C, H, W), generator=g, dtype=torch.uint8).to(dev)
    win = sym[:, :, 8:, 8:].contiguous()                             # a symbol window at (8, 8) of every plane
    tg = dm.targets(dev)
    # per image: (oy, ox, y0, x0, h, w, sy, sx, Hf, Wf)
    cases = [[(3, 2, 16, 8, 16, 16, 0, 0, H, W), (0, 0, 0, 0, H, W, 0, 0, H, W), (5, 4, 32, 32, 16, 8, 0, 0, H, W),
              (1, 3, 16, 0, 32, 40, 0, 0, H, W)],
             [(2, 1, 8, 0, 16, 16, 8, 8, H, W), (0, 0, 8, 8, 32, 16, 8, 8, H, W), (6, 4, 24, 24, 16, 8, 8, 8, H, W),
              (3, 3, 8, 8, 16, 24, 8, 8, H, W)]]
    for geo, s in zip(cases, (sym, win)):
        plane = max(r[4] * r[5] for r in geo) + 8
        out = torch.full((N * C * plane,), -7, dtype=torch.int32, device=dev)
        got = E.dmll_intervals_rects(l, s, geo, tg, C, K, L, rgb, tile, plane=plane, out=out)
        for n, (oy, ox, y0, x0, h, w, sy, sx, Hf, Wf) in enumerate(geo):
            want = E.dmll_intervals_rect(l[n:n + 1].contiguous(), oy, ox, s[n:n + 1].contiguous(), (y0, x0, h, w), tg,
                                         C, K, L, rgb, tile, origin=(sy, sx), plane=(Hf, Wf))
            assert torch.equal(got[n, :, :h * w], want[0]), (n, geo[n])
            assert (got[n, :, h * w:] == -7).all()                    # nothing past the rectangle's planes
    ok = list(cases[0])
    E.launch_log(reset=True)
    for n, bad in [(1, (0, 0, 8, 0, 16, 16, 0, 0, H, W)),              # not aligned
                   (2, (0, 0, 0, 4, 16, 8, 0, 0, H, W)),
                   (3, (0, 0, 40, 0, 16, 8, 0, 0, H, W)),              # outside the symbols
                   (0, (H, 0, 0, 0, 16, 8, 0, 0, H, W)),               # outside the parameters
                   (1, (0, 0, 0, 0, 16, 8, 40, 0, H, W)),              # outside the plane
                   (2, (0, 0, 0, 0, 0, 8, 0, 0, H, W))]:               # empty
        geo = list(ok)
        geo[n] = bad
        with pytest.raises(RuntimeError, match='image %d' % n):
            E.dmll_intervals_rects(l, sym, geo, tg, C, K, L, rgb, tile)
    with pytest.raises(RuntimeError):                                   # planes smaller than a rectangle
        E.dmll_intervals_rects(l, sym, ok, tg, C, K, L, rgb, tile, plane=16 * 16)
    with pytest.raises(RuntimeError):
        E.dmll_intervals_rects(l, sym, ok, tg, C, 4, L, rgb, tile)
    geo = np.array(ok, np.int32)
    iv = torch.empty(N * C * H * W, dtype=torch.int32, device=dev)
    gd = torch.empty(N * 10, dtype=torch.int32, device=dev)
    assert E.lib.l3c_dmll_intervals_rects(l.data_ptr(), H + 6, W + 4, sym.data_ptr(), H, W, None, gd.data_ptr(), H * W,
                                          tg.data_ptr(), N, C, K, L, int(rgb), 16, 8, iv.data_ptr(), None) != 0
    assert E.lib.l3c_dmll_intervals_rects(l.data_ptr(), H + 6, W + 4, sym.data_ptr(), H, W, geo.ctypes.data, None,
                                          H * W, tg.data_ptr(), N, C, K, L, int(rgb), 16, 8, iv.data_ptr(), None) != 0
    assert E.launch_log()[1] == 0


def test_ragged_pass_equals_serial_pass(mode):
    """In f16 a pass runs as one ragged batch of windows; forced plan after plan it gives the same bytes."""
    from l3c_pytorch_b200 import engine as E
    mode('f16')
    bc = _bc((16, 24))
    imgs, edits = _case()
    datas = [_encode(bc, img) for img in imgs]
    E.launch_log(reset=True)
    ragged = bc.update_regions(datas, edits)
    kernels, _ = E.launch_log(reset=True)
    assert kernels.get('dmll_intervals_rects_kernel') == 3 and 'dmll_intervals_rect_kernel' not in kernels, kernels
    codec = bc.codec
    plans = [codec.updates_counts[i]['plans'] for i in range(4)]
    serial = codec._code_pass_serial
    try:
        codec._code_pass_ragged = lambda plans_, imgs_, tile: serial(plans_, imgs_, [tile] * len(plans_))
        assert bc.update_regions(datas, edits) == ragged
    finally:
        del codec._code_pass_ragged
    assert [codec.updates_counts[i]['plans'] for i in range(4)] == plans
    _check(bc, imgs, datas, edits, ragged)
