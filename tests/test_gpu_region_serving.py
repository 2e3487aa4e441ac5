"""GPU: serving region decodes (DESIGN §4.8 "Batches").  Regions of different shapes over containers of different
image sizes decode in one ragged pass per level and tile size (f16, f16x2), bit-identical to each region decoded alone
and to the crop of the full decode; tf32 / fp32 keep the per-shape groups.  Also: the f16x2 convs under ragged
extents, the per-image row-builder, reorder and crop entry points against per-image calls, empty padding streams,
region decodes on a decode lane beside other work, and a pass on 3 SMs."""
import contextlib

import numpy as np
import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu

TILE = (32, 48)


@contextlib.contextmanager
def _precision(mode):
    from l3c_pytorch_b200 import engine as E
    old = E.get_conv_precision()
    E.set_conv_precision(mode)
    try:
        yield
    finally:
        E.set_conv_precision(old)


def _mixed(H, W):
    """Regions of different sizes and clipping in an H x W image: interior, edges, corners, 1x1, the whole image."""
    return [(H // 2 - 9, W // 2 - 13, 17, 23), (0, W // 3, 11, 40), (H - 7, 5, 7, 30), (H // 3, W - 9, 25, 9),
            (0, 0, 13, 13), (H - 5, W - 21, 5, 21), (H // 2, W // 2, 1, 1), (0, 0, H, W)]


def _containers(bc, sizes, seed):
    imgs = [util.make_image(seed + i, h, w) for i, (h, w) in enumerate(sizes)]
    datas = [bc.encode_batch([im])[0][0] for im in imgs]
    fulls = [bc.decode_batch([d])[0] for d in datas]
    for im, f in zip(imgs, fulls):
        assert torch.equal(f[0].cpu(), im.long())
    return imgs, datas, fulls


def _request(datas, sizes):
    """A serving-like request list over every container: -> (datas, regions, container index)"""
    ds, regs, which = [], [], []
    for k, (h, w) in enumerate(sizes):
        for reg in _mixed(h, w)[k % 2::2] + [_mixed(h, w)[-1]]:
            ds.append(datas[k])
            regs.append(reg)
            which.append(k)
    return ds, regs, which


def _check_equal(bc, ds, regs, levels, got, want_of):
    for d, reg, lev, g in zip(ds, regs, levels, got):
        y, x, h, w = reg
        assert g.dtype == torch.int64 and tuple(g.shape) == (1, 3, h, w) and g.is_contiguous()
        assert torch.equal(g, bc.decode_region(d, reg, lev)), (reg, lev)
        assert torch.equal(g, want_of(d, lev)[:, :, y:y + h, x:x + w]), (reg, lev)


@pytest.mark.parametrize('cfg,mode', [('cr', 'f16'), ('cr', 'f16x2'), ('cr_rgb_shared', 'f16'),
                                      ('cr_rgb_shared', 'f16x2'), ('cr_rgb', 'f16')])
def test_mixed_regions_decode_in_one_pass_per_level(cfg, mode):
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint(cfg)
    sizes = [(150, 196), (96, 80)]                         # padded to 152 x 200 and 96 x 80 (cr)
    with _precision(mode):
        bc = Bitcoding(bp, tile=TILE)
        imgs, datas, fulls = _containers(bc, sizes, 400)
        ds, regs, which = _request(datas, sizes)
        levels = [0] * len(ds)
        want = {id(d): f for d, f in zip(datas, fulls)}
        thumbs = {}
        if cfg == 'cr_rgb_shared':
            # plus every level of a recursive container in the same call: one pass per level
            rbc = Bitcoding(bp, tile=(16, 16), recursive=2)
            rimg = util.make_image(410, 90, 70)
            rdata = rbc.encode_batch([rimg])[0][0]
            x, _ = rbc._prepare(rimg, quiet=True)
            pyr = bp.forward(x, auto_recurse=2).S_u8
            want[id(rdata)] = rbc.decode_batch([rdata])[0]
            for k in range(1, 4):
                thumbs[k] = pyr[k].long()
                Hk, Wk = pyr[k].shape[-2:]
                for reg in [(Hk // 2 - 3, Wk // 2 - 2, 5, 4), (0, 0, Hk, Wk), (Hk - 2, 0, 2, 3)]:
                    ds.append(rdata)
                    regs.append(reg)
                    levels.append(k)
            ds += [rdata] * 2
            regs += [(3, 4, 30, 20), (60, 50, 30, 20)]
            levels += [0, 0]
        _, plans = bc.codec.plan_regions(ds, regs, levels)
        assert len({p.shape_key() for p in plans}) > len(sizes)
        torch.cuda.synchronize()
        E.launch_log(reset=True)
        got = bc.decode_regions(ds, regs, levels)
        torch.cuda.synchronize()
        kernels, _ = E.launch_log(reset=True)
        assert kernels.get('zero_halo_kernel', 0) > 0 and kernels.get('crop_rects_kernel', 0) > 0, kernels
        if cfg == 'cr':                                     # one pass: one range-decoder launch per channel step
            dec = sum(n for k, n in kernels.items() if k.startswith('ac_decode'))
            assert dec == 1 + 2 + 3 and 'crop_rect_kernel' not in kernels, kernels

        def want_of(d, lev):
            return want[id(d)] if lev == 0 else thumbs[lev]
        _check_equal(bc, ds, regs, levels, got, want_of)


def test_mixed_list_launches_the_decoders_of_one_region():
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    sizes = [(150, 196), (96, 80), (128, 192)]
    with _precision('f16'):
        bc = Bitcoding(bp, tile=TILE)
        _, datas, fulls = _containers(bc, sizes, 420)
        ds = [datas[0], datas[1], datas[2], datas[0]]
        regs = [(70, 90, 17, 23), (0, 0, 40, 80), (100, 150, 28, 42), (149, 195, 1, 1)]
        _, plans = bc.codec.plan_regions(ds, regs)
        assert len({p.shape_key() for p in plans}) == len(regs)
        torch.cuda.synchronize()
        E.launch_log(reset=True)
        got = bc.decode_regions(ds, regs)
        torch.cuda.synchronize()
        kernels, _ = E.launch_log(reset=True)
        dec = sum(n for k, n in kernels.items() if k.startswith('ac_decode'))
        assert dec == 1 + 2 + 3, kernels                    # uniform, two bottleneck scales, R, G, B
        assert kernels.get('dmll_table_kernel', 0) == 2 + 3
        assert bc.codec.region_counts == {'streams': sum(p.streams for p in plans),
                                          'symbols': sum(p.symbols for p in plans)}
        for d, reg, g in zip(ds, regs, got):
            y, x, h, w = reg
            assert torch.equal(g, fulls[datas.index(d)][:, :, y:y + h, x:x + w]), reg


@pytest.mark.parametrize('mode', ['tf32', 'fp32'])
def test_tf32_fp32_keep_the_per_shape_groups(mode):
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    sizes = [(150, 196), (96, 80)]
    with _precision(mode):
        bc = Bitcoding(bp, tile=TILE)
        _, datas, fulls = _containers(bc, sizes, 430)
        ds, regs, _ = _request(datas, sizes)
        # two sizes inside the same tiles: equal rectangles and windows, different crops
        ds += [datas[1]] * 2
        regs += [(2, 3, 5, 4), (2, 3, 12, 9)]
        torch.cuda.synchronize()
        E.launch_log(reset=True)
        got = bc.decode_regions(ds, regs)
        torch.cuda.synchronize()
        kernels, _ = E.launch_log(reset=True)
        assert kernels.get('zero_halo_kernel', 0) == 0, kernels
        want = {id(d): f for d, f in zip(datas, fulls)}
        _check_equal(bc, ds, regs, [0] * len(ds), got, lambda d, lev: want[id(d)])


# ---------------------------------------------------------------------------------------------
# f16x2 convs of a padded batch
# ---------------------------------------------------------------------------------------------
EXT = [(24, 40), (8, 8), (16, 24), (40, 16), (32, 48)]
LIMITS = [(0, 0), (1, 0), (2, 0), (3, 0), (7, 0), (3, 112), (7, 160)]


def _ragged(ext, C, seed, scale=1):
    g = torch.Generator().manual_seed(seed)
    Hb, Wb = max(h for h, _ in ext) * scale, max(w for _, w in ext) * scale
    x = torch.full((len(ext), Hb, Wb, C), float('nan'))
    alone = []
    for n, (h, w) in enumerate(ext):
        v = torch.randn(1, h * scale, w * scale, C, generator=g) * 2
        x[n, :h * scale, :w * scale] = v[0]
        alone.append(v.cuda())
    return x.cuda(), alone


def _band_is_pos_zero(x, ext, halo):
    b = x.view(torch.int16) if x.dtype == torch.float16 else x.view(torch.int32)
    H, W = x.shape[1:3]
    for n, (h, w) in enumerate(ext):
        band = torch.zeros(H, W, dtype=torch.bool, device=x.device)
        band[:min(h + halo, H), :min(w + halo, W)] = True
        band[:h, :w] = False
        if not bool((b[n][band] == 0).all()):
            return False
    return True


@pytest.mark.parametrize('case', ['3x3_d1_relu', '3x3_d2', '3x3_d4', 'pixel_shuffle', 'ffma_head_residual'])
def test_f16x2_convs_of_a_ragged_batch_equal_per_image_launches(case):
    from l3c_pytorch_b200 import engine as E
    net = util.blueprint('cr').net
    conv, kw = {'3x3_d1_relu': (net.nets[0].dec.body[0].body[0], dict(relu=True)),
                '3x3_d2': (net.prob_clfs[0].atrous.atrous[1], {}),
                '3x3_d4': (net.prob_clfs[0].atrous.atrous[2], {}),
                'pixel_shuffle': (net.nets[0].dec.tail[0], dict(pixel_shuffle=True)),
                'ffma_head_residual': (net.nets[0].dec.head, {})}[case]
    ffma = case == 'ffma_head_residual'
    with _precision('f16x2'):
        x, alone = _ragged(EXT, 8 if ffma else 64, 11)
        if ffma:
            r, ralone = _ragged(EXT, conv.out_channels, 12)
            want = [E.conv2d(conv, a, residual=ra) for a, ra in zip(alone, ralone)]
        else:
            want = [E.conv2d(conv, E.Act(a, E.split_f16x2(a)), **kw) for a in alone]
        halo = conv.dilation[0] * (conv.kernel_size[0] // 2)
        f = 2 if kw.get('pixel_shuffle') else 1
        for max_sms, kb in LIMITS:
            with E.conv_launch_limits(max_sms=max_sms, conv_smem_kb=kb), E.ragged_extents(EXT, *x.shape[1:3]):
                if ffma:
                    xr = x.clone()
                    got = E.conv2d(conv, xr, residual=r)
                else:
                    xr = E.split_f16x2(x)
                    got = E.conv2d(conv, E.Act(x, xr), **kw)
            assert _band_is_pos_zero(xr, EXT, halo), (case, max_sms, kb)
            for n, (h, w) in enumerate(EXT):
                assert torch.equal(got[n, :h * f, :w * f], want[n][0]), (case, n, max_sms, kb)
            if ffma:
                break                                    # the FFMA kernel takes no launch limits


def test_f16x2_decoder_windows_equal_per_window_runs():
    """get_P_nhwc(windows=) in f16x2 on a NaN-padded batch: parameters and fused features equal per-window runs"""
    from l3c_pytorch_b200 import engine as E
    net = util.blueprint('cr').net
    wins = [(12, 20), (4, 4), (9, 13), (20, 8)]
    with _precision('f16x2'):
        bn, alone = _ragged(wins, 8, 13)
        Fp, Falone = _ragged(wins, net.config_ms.Cf, 14)
        for scale in (0, 1):
            want = [net.get_P_nhwc(scale, a, fa) for a, fa in zip(alone, Falone)]
            l, F = net.get_P_nhwc(scale, bn.clone(), Fp.clone(), windows=wins)
            for n, (h, w) in enumerate(wins):
                assert torch.equal(l[n, :2 * h, :2 * w], want[n][0][0]), (scale, n)
                if scale > 0:
                    assert torch.equal(F.f[n, :2 * h, :2 * w], want[n][1].f[0]), (scale, n)
    with _precision('tf32'), pytest.raises(NotImplementedError, match='tf32'):
        net.get_P_nhwc(1, bn, windows=wins)


# ---------------------------------------------------------------------------------------------
# the per-image entry points
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('rgb', [False, True])
def test_row_builder_windows_equal_per_image_calls(rgb):
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    dm = bp.losses.loss_dmol_rgb if rgb else bp.losses.loss_dmol_n
    C, K, L = (3 if rgb else 5), 10, dm.L
    Kp = (4 if rgb else 3) * C * K
    tile = (8, 16)
    # (oy, ox, H_n, W_n) inside parameter windows of (Hl_n, Wl_n), different tile counts
    geo = [(3, 5, 20, 37), (0, 0, 8, 16), (7, 1, 9, 3), (2, 9, 33, 40)]
    wl = [(26, 44), (8, 16), (20, 6), (40, 52)]
    Hl, Wl = max(h for h, _ in wl), max(w for _, w in wl)
    plane = max(h * w for _, _, h, w in geo)
    g = torch.Generator().manual_seed(21)
    l = torch.full((len(geo), Hl, Wl, Kp), float('nan'))
    for n, (h, w) in enumerate(wl):
        l[n, :h, :w] = torch.randn(h, w, Kp, generator=g) * 2
    l = l.cuda()
    sym = torch.randint(0, L, (len(geo), C, plane), generator=g, dtype=torch.uint8).cuda()
    pitch = E.table_pitch(L)
    tg = dm.targets(l.device)
    geo_dev = torch.tensor(geo, dtype=torch.int32).cuda()
    for c in (range(C) if rgb else [-1]):
        table = torch.full((len(geo) * C * plane * pitch,), -1, dtype=torch.int16, device='cuda')
        E.dmll_build_table_windows(l, geo_dev, max(h * w for _, _, h, w in geo), plane, sym, tg, C, K, L, rgb, c,
                                   table, tile)
        tv = table.view(len(geo), C, plane, pitch)
        for n, (oy, ox, h, w) in enumerate(geo):
            ln = l[n:n + 1, :wl[n][0], :wl[n][1]].contiguous()
            sn = sym[n:n + 1, :, :h * w].contiguous()
            ref = torch.full((C * h * w * pitch,), -1, dtype=torch.int16, device='cuda')
            E.dmll_build_table_window(ln, oy, ox, sn, tg, C, K, L, rgb, c, ref, h, w, tile)
            rv = ref.view(C, h * w, pitch)
            for cc in ([c] if c >= 0 else range(C)):
                assert torch.equal(tv[n, cc, :h * w], rv[cc]), (n, cc)
                assert bool((tv[n, cc, h * w:] == -1).all()), (n, cc)      # nothing written past the rectangle


def test_reorder_and_crop_entry_points_equal_per_image_calls():
    from l3c_pytorch_b200 import engine as E
    g = torch.Generator().manual_seed(22)
    tile = (8, 16)
    ext = [(20, 37), (8, 16), (9, 3), (33, 40)]
    N, P = len(ext), 3
    plane = max(h * w for h, w in ext)
    Hm, Wm = max(h for h, _ in ext), max(w for _, w in ext)
    src = torch.randint(0, 256, (N, P, plane), generator=g, dtype=torch.uint8).cuda()     # garbage past h_n * w_n
    got = E.reorder_tiles_images(src, torch.tensor(ext, dtype=torch.int32).cuda(), Hm, Wm, tile)
    for n, (h, w) in enumerate(ext):
        ref = E.reorder_tiles(src[n, :, :h * w].contiguous(), h, w, tile, False).view(P, h, w)
        assert torch.equal(got[n, :, :h, :w], ref), n
        pad = torch.ones(Hm, Wm, dtype=torch.bool, device='cuda')
        pad[:h, :w] = False
        assert bool((got[n][:, pad] == 0).all()), n
    # crops: planes of bytes, NHWC of fp32 words; NaN outside the rectangles that are read
    rects = [(1, 2, 9, 30), (0, 0, 8, 16), (5, 0, 4, 3), (10, 7, 23, 33)]
    rects_dev = torch.tensor(rects, dtype=torch.int32).cuda()
    hm, wm = max(r[2] for r in rects), max(r[3] for r in rects)
    planes = torch.randint(0, 256, (N, P, 40, 44), generator=g, dtype=torch.uint8).cuda()
    feats = torch.full((N, 40, 44, 20), float('nan'))
    for n, (y, x, h, w) in enumerate(rects):
        feats[n, y:y + h, x:x + w] = torch.randn(h, w, 20, generator=g)
    feats = feats.cuda()
    padded = E.crop_rects(planes, rects_dev, hm, wm, nhwc=False)
    fpad = E.crop_rects(feats, rects_dev, hm, wm, nhwc=True)
    compact = E.crop_rects(planes, rects_dev, hm, wm, nhwc=False, sizes=[r[2:] for r in rects])
    for n, (y, x, h, w) in enumerate(rects):
        org = torch.tensor([[y, x]], dtype=torch.int32).cuda()
        want = E.crop_rect(planes[n:n + 1].contiguous(), org, h, w, nhwc=False)
        fwant = E.crop_rect(feats[n:n + 1].contiguous(), org, h, w, nhwc=True)
        assert torch.equal(padded[n:n + 1, :, :h, :w], want) and torch.equal(compact[n], want), n
        assert compact[n].is_contiguous() and tuple(compact[n].shape) == (1, P, h, w)
        assert torch.equal(fpad[n:n + 1, :h, :w], fwant), n
        out = torch.ones(hm, wm, dtype=torch.bool, device='cuda')
        out[:h, :w] = False
        assert bool((padded[n][:, out] == 0).all()) and bool((fpad[n][out] == 0).all()), n


def test_empty_padding_streams_leave_the_real_streams_unchanged():
    from l3c_pytorch_b200 import Bitcoding, _lib
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200.codec import _upload, parse_container
    bp = util.blueprint('cr')
    with _precision('f16'):
        bc = Bitcoding(bp, tile=(8, 8))
        data = bc.encode_batch([util.make_image(440, 96, 80)])[0][0]
    _, scales = parse_container(data)
    C, H, W, streams = scales[0]                               # the uniform-prior scale: 5 x 12 x 10, 2 x 2 tiles
    L = bp.losses.loss_dmol_n.L
    dev = torch.device('cuda')
    blob, _ = _upload([data], dev)
    row = bc.codec._uniform(L, dev)[1]
    n_real = len(streams)
    cnt = 64                                                   # symbols per output slot (tiles hold <= 64)

    def run(with_empty):
        out = torch.full(((2 * n_real) * cnt,), 0xAB, dtype=torch.uint8, device=dev)
        descs = []
        for k, (off, ln) in enumerate(streams):
            t = k % (len(streams) // C)
            th = min(8, H - (t // 2) * 8)
            tw = min(8, W - (t % 2) * 8)
            descs.append((off, ln, th * tw, 2 * k * cnt))
            if with_empty:                                     # an empty stream writing into the guard slot
                descs.append((0, 0, 0, (2 * k + 1) * cnt))
        d = np.zeros(len(descs), dtype=_lib.DEC_STREAM_DTYPE)
        d['in'] = [blob.data_ptr() + o for (o, _, _, _) in descs]
        d['in_len'] = [ln for (_, ln, _, _) in descs]
        d['n_sym'] = [n for (_, _, n, _) in descs]
        d['sym_out'] = [out.data_ptr() + s for (_, _, _, s) in descs]
        d['table'] = row.data_ptr()
        d['row_pitch'] = 0
        E.ac_decode_streams(d, dev, L)
        torch.cuda.synchronize()
        return out

    plain, padded = run(False), run(True)
    assert torch.equal(plain, padded)
    assert bool((padded.view(2 * n_real, cnt)[1::2] == 0xAB).all())           # the empty streams wrote nothing


# ---------------------------------------------------------------------------------------------
# lanes and side streams
# ---------------------------------------------------------------------------------------------
def test_regions_on_a_lane_beside_a_decode_and_an_encode():
    from l3c_pytorch_b200 import Bitcoding
    bp = util.blueprint('cr')
    sizes = [(150, 196), (96, 80)]
    with _precision('f16'):
        bc = Bitcoding(bp, tile=TILE)
        _, datas, _ = _containers(bc, sizes, 450)
        ds, regs, _ = _request(datas, sizes)
        want_regions = bc.decode_regions(ds, regs)
        batch_a = torch.stack([util.make_image(460 + i, 64, 96) for i in range(3)])
        batch_b = torch.stack([util.make_image(470 + i, 64, 96) for i in range(3)])
        datas_a, _ = bc.encode_batch(batch_a)
        want_b, _ = bc.encode_batch(batch_b)
        want_a = bc.decode_batch(datas_a)
        torch.cuda.synchronize()
        lanes = bc.decode_lanes(3, n_lanes=2)
        side = bc.side_stream(3, n_lanes=2)
        cur = torch.cuda.current_stream()
        job = bc.encode_batch_begin(batch_b.pin_memory(), stream=side)
        for ln in lanes:
            ln.main.wait_stream(cur)
        with torch.cuda.stream(lanes[0].main):
            got_regions = bc.decode_regions(ds, regs, lane=lanes[0])
        with torch.cuda.stream(lanes[1].main):
            got_a = bc.decode_batch(datas_a, lane=lanes[1])
        assert job.finish()[0] == want_b
        for ln in lanes:
            cur.wait_stream(ln.main)
        torch.cuda.synchronize()
    for g, w in zip(got_regions, want_regions):
        assert torch.equal(g, w)
    for g, w in zip(got_a, want_a):
        assert torch.equal(g, w)


def test_mixed_pass_on_three_sms():
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr_rgb_shared')
    sizes = [(150, 196), (96, 80)]
    with _precision('f16'):
        bc = Bitcoding(bp, tile=TILE)
        _, datas, fulls = _containers(bc, sizes, 480)
        ds, regs, which = _request(datas, sizes)
        with E.conv_launch_limits(max_sms=3):
            got = bc.decode_regions(ds, regs)
    for k, reg, g in zip(which, regs, got):
        y, x, h, w = reg
        assert torch.equal(g, fulls[k][:, :, y:y + h, x:x + w]), reg
