"""GPU: region decodes of seek-indexed reference-layout containers (DESIGN §4.13 "Regions").
* Regions of `cr` and `cr_rgb_shared` (R = 0 and 1) containers in f16, f16x2, tf32 and fp32, at K = 32, 4096 and one
  above every stream's length, equal bit for bit the same crop of the indexed decode, of the serial decode and of the
  image: corners, the middle, the whole image, 1x1, a single row, a full-width strip, bands starting on and just after
  a seek point, padded images, and levels >= 1 of the baselines.
* Mixed lists of tiled and indexed containers of different sizes equal each region alone; in f16 and f16x2 they run as
  one ragged pass per pass key.
* The launch log: segment launches only, the coarse window builder on the RGB scale in f16, and region_counts equal to
  the plan's (below the container's total for a middle region).
* l3c_dmll_build_coarse_windows equals l3c_dmll_build_coarse on a copied rectangle, bit for bit; its refusals launch
  nothing.
* Regions on a decode lane beside another lane's decode and an encode; junk and reference-written containers with their
  seek_index(); images stored in parts through decode_region_file and the command line."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def precision(mode):
    from l3c_pytorch_b200 import engine
    old = engine.get_conv_precision()
    engine.set_conv_precision(mode)
    try:
        yield
    finally:
        engine.set_conv_precision(old)


def _regions(H, W, Wp, K, top):
    """Regions of an H x W image (padded width Wp, `top` rows of padding above): corners, middle, whole, 1x1, a row, a
    full-width strip, and bands whose first symbol is a seek point and one symbol after one."""
    out = [(0, 0, 13, 13), (H - 5, W - 21, 5, 21), (H // 2 - 9, W // 2 - 13, 17, 23), (0, 0, H, W),
           (H // 2, W // 2, 1, 1), (H // 3, 5, 1, W - 7), (H // 4, 0, 9, W)]
    for r in range(top + 1, H + top - 4):               # a row whose first symbol is a seek point, if there is one
        if r * Wp % K == 0:
            out.append((r - top, 3, 4, 10))
            break
    for r in range(top + 1, H + top - 2):                # a row that starts just after one
        if 0 < r * Wp % K <= Wp // 2 and (r * Wp) // K > 0:
            out.append((r - top, 0, 2, W))
            break
    return out


def _check(bc, datas, seeks, refs, regions):
    for d, sk, ref in zip(datas, seeks, refs):
        for reg in regions:
            y, x, h, w = reg
            got = bc.decode_region(d, reg, seek=sk)
            assert got.dtype == torch.int64 and tuple(got.shape) == (1, 3, h, w) and got.is_cuda
            for r in ref:
                assert torch.equal(got, r[:, :, y:y + h, x:x + w]), reg


CASES = [  # (config, recursive, precision, K)
    ('cr', 0, 'f16', 32), ('cr', 0, 'f16', 4096), ('cr', 0, 'f16', None), ('cr', 0, 'f16x2', 32),
    ('cr', 0, 'tf32', 4096), ('cr', 0, 'fp32', 32), ('cr_rgb_shared', 0, 'f16', 32),
    ('cr_rgb_shared', 0, 'f16x2', 4096), ('cr_rgb_shared', 1, 'f16', 32), ('cr_rgb_shared', 1, 'fp32', None)]


@pytest.mark.parametrize('case', CASES, ids=lambda c: '%s-R%d-%s-K%s' % (c[0], c[1], c[2], c[3] or 'big'))
def test_regions_equal_crops(case):
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200.codec import parse_container
    cfg, R, mode, K = case
    bp = util.blueprint(cfg, 'cuda:0')
    bc = Bitcoding(bp, recursive=R)
    H, W = 150, 196                                          # padded on both axes
    imgs = [util.make_image(500, H, W), util.make_image(501, H, W)]
    with precision(mode):
        datas, _ = bc.encode_batch(imgs)
        pt, scales = parse_container(datas[0])
        Hp, Wp = scales[-1][1:3]
        K = K or -(-(Hp * Wp + 1) // 32) * 32                # above every stream's length: no seek point
        seeks = bc.seek_index(datas, every=K)
        full = bc.decode_batch(datas, seeks=seeks)
        serial = bc.decode_batch(datas)
        for f, s, im in zip(full, serial, imgs):
            assert torch.equal(f, s) and torch.equal(f[0].cpu(), im.long())
        _check(bc, datas, seeks, list(zip(full, serial)), _regions(H, W, Wp, K, pt[2]))
        if bp.net._rgb:                                       # the stored thumbnails, levels >= 1
            x, _ = bc._prepare(imgs[0], quiet=True)
            thumbs = bp.forward(x, auto_recurse=R).S_u8
            for k in range(1, len(scales)):
                Hk, Wk = thumbs[k].shape[-2:]
                for reg in [(Hk // 2 - 3, Wk // 2 - 2, 5, 4), (0, 0, Hk, Wk), (Hk - 1, 0, 1, Wk)]:
                    y, x0, h, w = reg
                    got = bc.decode_region(datas[0], reg, level=k, seek=seeks[0])
                    assert torch.equal(got, thumbs[k][:, :, y:y + h, x0:x0 + w].long()), (k, reg)


@pytest.mark.parametrize('mode', ['f16', 'f16x2', 'fp32'])
def test_mixed_lists_and_passes(mode):
    from l3c_pytorch_b200 import Bitcoding, codec
    bp = util.blueprint('cr', 'cuda:0')
    ref_bc, tiled_bc = Bitcoding(bp), Bitcoding(bp, tile=(32, 32))
    with precision(mode):
        imgs = [util.make_image(510, 128, 160), util.make_image(511, 96, 80), util.make_image(512, 150, 196)]
        ref = [ref_bc.encode_batch([im], seek=96) for im in imgs]
        datas = [r[0][0] for r in ref] + [tiled_bc.encode_batch([imgs[0]])[0][0]]
        seeks = [r[2][0] for r in ref] + [None]
        fulls = [ref_bc.decode_batch([d])[0] for d in datas]
        order = [0, 1, 3, 2, 0, 3]
        regions = [(40, 70, 20, 30), (10, 10, 30, 30), (40, 70, 20, 30), (0, 0, 150, 196), (100, 0, 28, 160),
                   (5, 5, 3, 3)]
        _, plans = ref_bc.codec.plan_regions([datas[i] for i in order], regions, seeks=[seeks[i] for i in order])
        calls = []
        orig = codec.BatchCodec.decode_region_pass

        def counting(self, blob, offs, lens, plans, ragged, lane=None):
            calls.append((ragged, {p.pass_key() for p in plans}))
            return orig(self, blob, offs, lens, plans, ragged, lane=lane)
        codec.BatchCodec.decode_region_pass = counting
        try:
            many = ref_bc.decode_regions([datas[i] for i in order], regions, seeks=[seeks[i] for i in order])
        finally:
            codec.BatchCodec.decode_region_pass = orig
        for i, reg, got in zip(order, regions, many):
            y, x, h, w = reg
            assert torch.equal(got, fulls[i][:, :, y:y + h, x:x + w]), (i, reg)
            assert torch.equal(got, ref_bc.decode_region(datas[i], reg, seek=seeks[i])), (i, reg)
        assert all(len(keys) == 1 for _, keys in calls)      # reference and tiled plans never share a pass
        if mode in ('f16', 'f16x2'):
            assert len(calls) == len({p.pass_key() for p in plans}) == 2
            assert all(ragged for ragged, _ in calls)


def test_launches_and_counts():
    from l3c_pytorch_b200 import Bitcoding, engine as E, seek
    from l3c_pytorch_b200.codec import parse_container
    bp = util.blueprint('cr', 'cuda:0')
    bc = Bitcoding(bp)
    with precision('f16'):
        img = util.make_image(520, 256, 320)
        datas, _, seeks = bc.encode_batch([img], seek=256)
        region = (128, 160, 16, 16)
        _, plans = bc.codec.plan_regions(datas, [region], seeks=seeks)
        torch.cuda.synchronize()
        E.launch_log(reset=True)
        got = bc.decode_region(datas[0], region, seek=seeks[0])
        torch.cuda.synchronize()
        kernels, _ = E.launch_log(reset=True)
        assert torch.equal(got[0].cpu(), img[:, 128:144, 160:176].long())
        dec = {k: n for k, n in kernels.items() if k.startswith('ac_decode')}
        # one segment launch per bottleneck scale, per RGB channel and for the uniform scale; nothing serial
        assert dec == {'ac_decode_segments': 2 + 1, 'ac_decode_segments_coarse': 3}, kernels
        assert kernels.get('dmll_coarse_windows_kernel') == 3 and 'dmll_coarse_kernel' not in kernels, kernels
        assert kernels.get('dmll_table_kernel') == 2, kernels                # the bottleneck scales' full rows
        counts = bc.codec.region_counts
        total = int(seek.stream_symbols(datas[0]).sum())
        assert counts == {'streams': plans[0].streams, 'symbols': plans[0].symbols}
        assert counts['symbols'] < total
        _, scales = parse_container(datas[0])
        assert plans[0].streams == sum(len(st) for (_, _, _, st) in scales)
        with precision('fp32'):
            E.launch_log(reset=True)
            bc.decode_region(datas[0], region, seek=seeks[0])
            torch.cuda.synchronize()
            kernels, _ = E.launch_log(reset=True)
            assert 'dmll_coarse_windows_kernel' not in kernels and 'ac_decode_segments_coarse' not in kernels


def test_coarse_window_records_equal_whole_plane_records():
    from l3c_pytorch_b200 import _lib, engine as E
    dev = torch.device('cuda:0')
    bp = util.blueprint('cr', 'cuda:0')
    tg = bp.losses.loss_dmol_rgb.targets(dev)
    g = torch.Generator(device=dev).manual_seed(3)
    N, Hl, Wl, Kp, P = 3, 21, 37, 120, E.COARSE_PITCH
    l = torch.randn(N, Hl, Wl, Kp, device=dev, generator=g) * 2
    for geo in ([(2, 3, 11, 30)] * N, [(0, 0, 21, 37), (5, 9, 1, 17), (20, 0, 1, 1)]):
        hw = [h * w for (_, _, h, w) in geo]
        plane = max(hw) + 5
        sym = torch.randint(0, 256, (N, 3, plane), dtype=torch.uint8, device=dev, generator=g)
        geo_dev = torch.tensor(geo, dtype=torch.int32, device=dev)
        for c in range(3):
            rec = torch.zeros(N * 3 * plane * P, dtype=torch.int16, device=dev)
            E.dmll_build_coarse_windows(l, geo_dev, max(hw), plane, sym, tg, 10, 256, c, rec)
            for n, (oy, ox, h, w) in enumerate(geo):
                lc = l[n:n + 1, oy:oy + h, ox:ox + w].contiguous()
                sc = sym[n:n + 1, :, :h * w].contiguous()
                want = torch.zeros(3 * h * w * P, dtype=torch.int16, device=dev)
                E.dmll_build_coarse(lc, sc, tg, 10, 256, c, want)
                got = rec.view(N, 3, plane * P)[n, c, :h * w * P]
                assert torch.equal(got, want[c * h * w * P:(c + 1) * h * w * P]), (geo, n, c)
    # refusals: nothing is launched
    torch.cuda.synchronize()
    E.launch_log(reset=True)
    geo_dev = torch.tensor([(0, 0, 4, 4)] * N, dtype=torch.int32, device=dev)
    rec = torch.zeros(N * 3 * 16 * P, dtype=torch.int16, device=dev)
    sym = torch.zeros(N, 3, 16, dtype=torch.uint8, device=dev)
    f = _lib.lib.l3c_dmll_build_coarse_windows
    p = ctypes.c_void_p
    base = dict(l=p(l.data_ptr()), geo=p(geo_dev.data_ptr()), max_hw=16, plane=16, sym=p(sym.data_ptr()),
                tg=p(tg.data_ptr()), L=256, c=1, rec=p(rec.data_ptr()))
    for bad in (dict(l=None), dict(geo=None), dict(rec=None), dict(tg=None), dict(L=255), dict(c=3), dict(c=-1),
                dict(c=1, sym=None), dict(max_hw=17), dict(max_hw=0)):
        a = dict(base, **bad)
        rc = f(a['l'], Hl, Wl, a['geo'], a['max_hw'], a['plane'], a['sym'], a['tg'], N, 10, a['L'], a['c'], a['rec'],
               None)
        assert rc != 0, bad
    assert E.launch_log(reset=True)[1] == 0


def test_regions_on_a_lane_beside_other_work():
    from l3c_pytorch_b200 import Bitcoding
    bp = util.blueprint('cr', 'cuda:0')
    bc = Bitcoding(bp)
    with precision('f16'):
        imgs_a = [util.make_image(530, 128, 128), util.make_image(531, 96, 112)]
        imgs_b = torch.stack([util.make_image(532 + i, 128, 128) for i in range(2)])
        da, _, sa = bc.encode_batch(imgs_a, seek=4096)
        db, _ = bc.encode_batch(imgs_b)
        regions = [(30, 20, 40, 50), (0, 0, 96, 112)]
        alone = bc.decode_regions(da, regions, seeks=sa)
        lanes = bc.decode_lanes(2, 2)
        side = bc.side_stream(2, 2)
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            job = bc.encode_batch_begin(imgs_b, stream=side)
        with torch.cuda.stream(lanes[0].main):
            got = bc.decode_regions(da, regions, seeks=sa, lane=lanes[0])
        with torch.cuda.stream(lanes[1].main):
            out_b = bc.decode_batch(db, lane=lanes[1])
        enc = job.finish()
        torch.cuda.synchronize()
    assert enc[0] == db
    for a, b in zip(got, alone):
        assert torch.equal(a, b)
    for a, b in zip(out_b, imgs_b):
        assert torch.equal(a.cpu(), b.unsqueeze(0).long())


@pytest.mark.parametrize('kind', ['cr_32', 'cr_40x28', 'rgbs_64'])
def test_junk_containers(kind):
    from l3c_pytorch_b200 import Bitcoding
    from tests.test_gpu_junk_containers import junk_sets
    from tests.test_malformed_containers_host import KINDS, build
    cfg, R = KINDS[kind][0], KINDS[kind][5]
    bc = Bitcoding(util.blueprint(cfg, 'cuda:0'), recursive=R)
    with precision('f16'):
        for name, payloads in junk_sets(kind).items():
            data = build(kind, payloads)[0]
            serial = bc.decode_batch([data])[0]
            sk = bc.seek_index([data], every=32)[0]
            H, W = serial.shape[-2:]
            for reg in [(0, 0, H, W), (H // 2, W // 3, max(1, H // 4), max(1, W // 3)), (H - 1, 0, 1, W)]:
                y, x, h, w = reg
                assert torch.equal(bc.decode_region(data, reg, seek=sk), serial[:, :, y:y + h, x:x + w]), (name, reg)


@pytest.mark.parametrize('name,cfg', [('l3c_32x32_i0', 'cr'), ('l3c_40x28_i1', 'cr'), ('rgbs_64x64_i0', 'cr_rgb_shared')])
def test_reference_written_containers(name, cfg):
    """The containers the reference wrote, indexed here: regions equal the crops of their serial decode, and of the
    golden image wherever that decode reproduces it (fp32, as the cross-decode test)."""
    from l3c_pytorch_b200 import Bitcoding
    g = util.golden_npz(name)
    bc = Bitcoding(util.blueprint(cfg, 'cuda:0'))
    ref = g['container'].tobytes()
    img = torch.from_numpy(g['img']).long()
    with precision('fp32'):
        serial = bc.decode_batch([ref])[0]
        sk = bc.seek_index([ref], every=32)[0]
        H, W = serial.shape[-2:]
        for reg in [(0, 0, H, W), (H // 2, 1, 3, W - 2), (H - 2, W - 3, 2, 3)]:
            y, x, h, w = reg
            got = bc.decode_region(ref, reg, seek=sk)
            assert torch.equal(got, serial[:, :, y:y + h, x:x + w]), reg
            if torch.equal(serial[0].cpu(), img):
                assert torch.equal(got[0].cpu(), img[:, y:y + h, x:x + w]), reg


def test_images_in_parts(tmp_path, monkeypatch, capsys):
    from PIL import Image
    from l3c_pytorch_b200 import Bitcoding, cli
    monkeypatch.setenv('AC_NEEDS_CROP_DIM', '100,100')
    bc = Bitcoding(util.blueprint('cr', 'cuda:0'))
    img = util.make_image(540, 150, 118)                  # 4 parts of 75 x 59 (padded to 80 x 64)
    p = str(tmp_path / 'big.l3c')
    with precision('f16'):
        bc.encode(img.long(), p, seek=96)
        whole = bc.decode(p + '.part0')
        assert torch.equal(whole[0].cpu(), img.long())
        for reg in [(10, 10, 20, 20), (60, 10, 30, 20), (10, 50, 20, 30), (70, 55, 10, 10), (0, 0, 150, 118),
                    (74, 0, 2, 118)]:
            y, x, h, w = reg
            got = bc.decode_region_file(p, reg)
            assert torch.equal(got, whole[:, :, y:y + h, x:x + w]), reg
            assert torch.equal(bc.decode_region_file(p + '.part2', reg), got)
        # the command line: the crop, and a missing sidecar refused naming it
        png = str(tmp_path / 'r.png')
        base = ['--config', 'cr', '--precision', 'f16']
        assert cli.main(base + ['dec', p, png, '--region', '70,50,20,30']) == 0
        assert np.array_equal(np.array(Image.open(png)), img.permute(1, 2, 0).numpy()[70:90, 50:80])
        import os
        os.remove(p + '.part3.seek')
        capsys.readouterr()
        assert cli.main(base + ['dec', p, png, '--region', '0,0,4,4']) == 1
        assert 'big.l3c.part3.seek' in capsys.readouterr().out
        # one reference file with its index through the command line
        q = str(tmp_path / 'one.l3c')
        small = util.make_image(541, 40, 56)
        bc.encode(small.long(), q, seek=32)
        assert cli.main(base + ['dec', q, png, '--region', '5,6,7,8']) == 0
        assert np.array_equal(np.array(Image.open(png)), small.permute(1, 2, 0).numpy()[5:12, 6:14])
