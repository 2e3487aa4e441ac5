"""GPU: the banded encode of large tiled images (DESIGN §4.10).

* With codec.TILED_ENCODE_BAND_PIXELS patched small (four or more bands at the finest scale, the last one partial),
  the banded encode writes the same bytes as the whole-image encode: `cr` in all four precision modes, `cr_rgb_shared`
  with recursive=2 in f16 and f16x2, tiles (16, 16) and (16, 24), one image and a batch of three.  The band kernels
  run, and the containers decode losslessly.  The same bytes when it runs on a side stream beside a decode lane.
* The band interval kernels (the fused f16 one, and the rectangle kernel on full-width rectangles) equal the
  whole-plane kernels followed by reorder_tiles, restricted to the band.
* Every encoder-side kernel the windows rely on is position independent in all four modes.
* Peak encode memory grows with the band, not with the image height; an 8000 x 6000 image encodes under a 24 GB cap."""
import contextlib

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


def _encode(bc, imgs, budget, monkeypatch):
    from l3c_pytorch_b200 import codec
    from l3c_pytorch_b200 import engine as E
    monkeypatch.setattr(codec, 'TILED_ENCODE_BAND_PIXELS', budget)
    E.launch_log(reset=True)
    datas, _ = bc.encode_batch(imgs)
    return datas, E.launch_log(reset=True)[0]


@pytest.mark.parametrize('cfg,mode,R', [('cr', 'f16', 0), ('cr', 'f16x2', 0), ('cr', 'tf32', 0), ('cr', 'fp32', 0),
                                        ('cr_rgb_shared', 'f16', 2), ('cr_rgb_shared', 'f16x2', 2)])
def test_banded_encode_equals_the_whole_image_encode(cfg, mode, R, monkeypatch):
    from l3c_pytorch_b200 import Bitcoding
    from l3c_pytorch_b200.region import plan_bands
    from l3c_pytorch_b200.codec import parse_container
    bp = util.blueprint(cfg)
    H, W = 200, 136
    imgs = torch.stack([util.make_image(500 + i, H, W) for i in range(3)])
    with _precision(mode):
        for tile in ((16, 16), (16, 24)):
            bc = Bitcoding(bp, tile=tile, recursive=R)
            for N in (1, 3):
                whole, k_whole = _encode(bc, imgs[:N], 1 << 62, monkeypatch)
                # three tile rows per band at the finest scale: 5 bands, the last one 8 rows high
                banded, k_band = _encode(bc, imgs[:N], 3 * N * tile[0] * W, monkeypatch)
                shapes = [(C, h, w) for (C, h, w, _) in parse_container(whole[0])[1]]
                bands = plan_bands(shapes, tile, bp.net, len(shapes) - 1, 3)
                assert len(bands) >= 4 and bands[-1].rect[2] - bands[-1].rect[0] < 3 * tile[0]
                assert banded == whole, (tile, N)
                band_kernel = 'lin_dmll_band_f16_kernel' if mode == 'f16' else 'dmll_intervals_rect_kernel'
                assert k_band.get(band_kernel, 0) >= len(bands), k_band
                assert k_whole.get(band_kernel, 0) == 0
                outs = bc.decode_batch(banded)
                assert all(torch.equal(o[0].cpu().to(torch.uint8), imgs[n]) for n, o in enumerate(outs))


def test_banded_encode_beside_a_decode_lane(monkeypatch):
    from l3c_pytorch_b200 import Bitcoding
    bp = util.blueprint('cr')
    H, W, tile = 200, 136, (16, 16)
    imgs = torch.stack([util.make_image(600 + i, H, W) for i in range(3)])
    with _precision('f16'):
        bc = Bitcoding(bp, tile=tile)
        ref, _ = _encode(bc, imgs, 3 * 3 * tile[0] * W, monkeypatch)
        other = bc.encode_batch(torch.stack([util.make_image(700 + i, 256, 256) for i in range(3)]))[0]
        lane = bc.decode_lanes(3, 1)[0]
        with torch.cuda.stream(lane.main):
            S = bc.codec.decode_batch(other, to_host=False, lane=lane)[0]
        job = bc.encode_batch_begin(imgs, stream=bc.side_stream(3))
        got, _ = job.finish()
        torch.cuda.current_stream().wait_stream(lane.main)
        torch.cuda.synchronize()
        assert got == ref
        assert S.shape[0] == 3


@pytest.mark.parametrize('rgb', [True, False])
@pytest.mark.parametrize('N', [1, 3])
def test_band_interval_kernels_equal_the_whole_plane_kernels(rgb, N):
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    net, losses, dev = bp.net, bp.losses, bp.device
    dm = losses.loss_dmol_rgb if rgb else losses.loss_dmol_n
    C = 3 if rgb else net.config_ms.q.C
    K = net.config_ms.prob.K
    lin = net.prob_clfs[0 if rgb else 1].atrous.lin
    H, W, tile = 40, 52, (16, 24)                      # partial last tile row, 24 does not divide 52
    g = torch.Generator(device='cpu').manual_seed(7 + N)
    sym = torch.randint(0, dm.L, (N, C, H, W), generator=g).to(torch.uint8).to(dev)
    cat = (torch.randn(N, H, W, lin.in_channels, generator=g) * 0.5).half().to(dev)
    l = (torch.randn(N, H, W, lin.out_channels, generator=g) * 0.5).to(dev)
    tg = dm.targets(dev)
    with _precision('f16'):
        whole_a = E.reorder_tiles(E.lin_dmll_intervals(lin, cat, sym, tg, C, K, dm.L, rgb), H, W, tile, True)
    whole_b = E.reorder_tiles(E.dmll_intervals(l, sym, tg, C, K, dm.L, rgb), H, W, tile, True)
    for (y0, y1) in ((0, 16), (16, 40), (0, 40)):
        h = y1 - y0
        for oy, ox, extra in ((0, 0, 0), (5, 0, 3), (3, 4, 0)):
            # a window plane holding the band's rows at (oy, ox)
            Hl = oy + h + extra
            catw = torch.zeros(N, Hl, W, lin.in_channels, dtype=torch.float16, device=dev)
            catw[:, oy:oy + h] = cat[:, y0:y1]
            lw = torch.full((N, Hl, W + ox + 2, lin.out_channels), float('nan'), device=dev)
            lw[:, oy:oy + h, ox:ox + W] = l[:, y0:y1]
            with _precision('f16'):
                a = E.lin_dmll_intervals_band(lin, catw, oy, sym, y0, h, tg, C, K, dm.L, rgb, tile)
            b = E.dmll_intervals_rect(lw, oy, ox, sym, (y0, 0, h, W), tg, C, K, dm.L, rgb, tile)
            assert torch.equal(a, whole_a[:, :, y0 * W:y1 * W]), (y0, y1, oy)
            assert torch.equal(b, whole_b[:, :, y0 * W:y1 * W]), (y0, y1, oy, ox)


def test_band_interval_kernels_refuse_bad_rectangles():
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    dev = bp.device
    dm = bp.losses.loss_dmol_rgb
    sym = torch.zeros(1, 3, 32, 16, dtype=torch.uint8, device=dev)
    l = torch.zeros(1, 20, 16, 120, device=dev)
    lin = bp.net.prob_clfs[0].atrous.lin
    cat = torch.zeros(1, 20, 16, 192, dtype=torch.float16, device=dev)
    for bad in (dict(oy=10, y0=0, h=16), dict(oy=0, y0=20, h=16)):
        with pytest.raises(Exception, match='outside|rows'):
            E.dmll_intervals_rect(l, bad['oy'], 0, sym, (bad['y0'], 0, bad['h'], 16), dm.targets(dev), 3, 10, 256,
                                  True, (16, 16))
        with pytest.raises(Exception, match='rows'):
            E.lin_dmll_intervals_band(lin, cat, bad['oy'], sym, bad['y0'], bad['h'], dm.targets(dev), 3, 10, 256,
                                      True, (16, 16))
    with pytest.raises(Exception, match='C==3'):
        E.dmll_intervals_rect(l, 0, 0, torch.zeros(1, 4, 32, 16, dtype=torch.uint8, device=dev), (0, 0, 16, 16),
                              dm.targets(dev), 4, 10, 256, True, (16, 16))


@pytest.mark.parametrize('mode', ['f16', 'f16x2', 'tf32', 'fp32'])
def test_encoder_kernels_are_position_independent(mode):
    """The interior of a run on a window equals the full run: the 5x5/s2 down conv at even offsets, the RGB head, the
    3x3 heads and quantize_head."""
    from l3c_pytorch_b200 import engine as E
    bp = util.blueprint('cr')
    net, dev = bp.net, bp.device
    H, W, a, b = 72, 40, 10, 58                     # window rows [a, b), a even
    g = torch.Generator(device='cpu').manual_seed(3)
    x = (torch.randn(2, H, W, 64, generator=g) * 0.5).to(dev)
    img = torch.randint(0, 256, (2, 3, H, W), generator=g).to(torch.uint8).to(dev)

    def f(t):
        return t.f if t.f is not None else t.r

    with _precision(mode):
        # 5x5 / stride 2: window output row i is full row a/2 + i where rows 2i-2 .. 2i+2 lie in the window
        down = net.nets[0].enc.down
        full = E.conv2d(down, E.as_operand(x), want='act')
        win = E.conv2d(down, E.as_operand(x[:, a:b].contiguous()), want='act')
        lo, hi = 1, (b - a - 3) // 2 + 1
        assert torch.equal(f(win)[:, lo:hi], f(full)[:, a // 2 + lo:a // 2 + hi])
        # the 3x3 heads
        head = net.heads[1].head
        full = E.conv2d(head, E.as_operand(x))
        win = E.conv2d(head, E.as_operand(x[:, a:b].contiguous()))
        assert torch.equal(win[:, 1:-1], full[:, a + 1:b - 1])
        # the RGB head (f16: im2col + GEMM; otherwise the normalisation and the CUDA-core conv)
        full = net._rgb_head_input(img)
        win = net._rgb_head_input(img[:, :, a:b].contiguous())
        if not isinstance(full, E.Act):
            full, win = net.heads[0](full), net.heads[0](win)
        full, win = (t if torch.is_tensor(t) else f(t) for t in (full, win))
        assert torch.equal(win[:, 1:-1], full[:, a + 1:b - 1])
        # quantize_head (per pixel)
        sym_f, bq_f = E.quantize_head(x, net.nets[0].enc.to_q[0], net.nets[0].enc.levels)
        sym_w, bq_w = E.quantize_head(x[:, a:b].contiguous(), net.nets[0].enc.to_q[0], net.nets[0].enc.levels)
        assert torch.equal(sym_w, sym_f[:, :, a:b]) and torch.equal(bq_w, bq_f[:, a:b])


@pytest.mark.parametrize('cfg,R', [('cr', 0), ('cr_rgb_shared', 2)])
def test_encode_peak_follows_the_band(cfg, R, monkeypatch):
    """With the band fixed, doubling the image height must add less than 128 B per added pixel.  What stays whole
    (DESIGN §4.10), per pixel of the image: the image (3 B), the symbol planes of the coarser scales (< 2), the
    bottleneck values (< 11), the range coder's slots (< 9) and, in the encoder phase, F_1 as the FP16 operand (32); in
    the coding phase of scale 1, the fp32 features of the decoders of scales 2 (16) and 1 (64): under 105 B in the larger
    phase, against about 750 for the whole-image encode.  Both heights give every scale at least two bands, so the band
    windows (and what one band takes) are the same."""
    from l3c_pytorch_b200 import Bitcoding, codec
    bp = util.blueprint(cfg)
    W, tile = 1024, (64, 64)
    monkeypatch.setattr(codec, 'TILED_ENCODE_BAND_PIXELS', 256 * 1024)
    peaks = []
    with _precision('f16'):
        bc = Bitcoding(bp, tile=tile, recursive=R)
        for H in (2048, 4096):
            img = util.make_image(800, H, W).unsqueeze(0).to(bp.device)
            bc.encode_batch(img)                      # warm-up: weight images, plans
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            bc.encode_batch(img)
            torch.cuda.synchronize()
            peaks.append(torch.cuda.max_memory_allocated() - base)
            del img
    growth = (peaks[1] - peaks[0]) / (2048 * W)
    assert growth < 128, (peaks, growth)


def test_large_image_encodes_under_a_memory_cap(tmp_path):
    from l3c_pytorch_b200 import Bitcoding
    bp = util.blueprint('cr')
    H, W = 6000, 8000
    g = torch.Generator(device='cpu').manual_seed(11)
    # a smooth image with noise: like a photograph, not like the network's worst case
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing='ij')
    base = ((yy // 7 + xx // 5) % 200).to(torch.int16)
    img = (base.unsqueeze(0).repeat(3, 1, 1) + torch.randint(0, 40, (3, H, W), generator=g, dtype=torch.int16))
    img = img.clamp(0, 255).to(torch.uint8).unsqueeze(0)
    total = torch.cuda.get_device_properties(bp.device).total_memory
    path = str(tmp_path / 'big.l3c')
    with _precision('f16'):
        bc = Bitcoding(bp, tile=(64, 64), crop=False)
        torch.cuda.empty_cache()
        torch.cuda.set_per_process_memory_fraction(min(1.0, 24e9 / total), bp.device)
        try:
            bc.encode(img, path)
        finally:
            torch.cuda.set_per_process_memory_fraction(1.0, bp.device)
        torch.cuda.empty_cache()
        out = bc.decode(path)
    assert torch.equal(out.cpu().to(torch.uint8), img)
