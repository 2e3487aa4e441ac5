"""GPU: seek indexes (DESIGN §4.13).
* The recording encoder (l3c_ac_encode_streams_seek) writes the oracle's bytes and, at every seek point, the state of
  the restated reference decoder (test_seek_host.record_points), on flat, peaked, straddling (more than 31 owed bits),
  uniform (span 2^32 at every point at L = 256) and 1-symbol streams; l3c_ac_decode_segments decodes their segments
  to the symbols.
* The codec: encode_batch(seek=K) writes the containers encode_batch() writes and the indexes seek_index() builds from
  them, byte for byte (cr and cr_rgb_shared with R = 0 and 1, equal-size and ragged batches, K = 32, 96, 4096 and one
  above every stream's length); decode_batch(datas, seeks) equals the serial decode and the images in f16 (coarse
  records), f16x2 and fp32, on a decode lane beside another lane's decode and an encode, with segment launches only.
* Junk containers decode with their seek_index() to the serial decode's symbols.
* A stream past 2^32 code bits decodes from seek points beyond 2^32 bits.
* The command line: enc --seek, dec and idx round-trip; a stale or mismatched sidecar is refused."""
import contextlib
import os

import numpy as np
import pytest
import torch

from tests import util
from tests.test_gpu_coder_launches import _intervals, make_stream
from tests.test_seek_host import record_points

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


def _pack_words(w):
    """l3c_ac_encode_streams_seek's point words -> (low, high, flip, bits)"""
    w = w.astype(np.int64)
    return w[:, 0], w[:, 1], w[:, 3] & 0x80000000, w[:, 2] | ((w[:, 3] & 0x7FFFFFFF) << 32)


@pytest.mark.parametrize('L', [5, 25, 100, 256])
def test_recording_encoder_and_segment_decoder(L):
    from oracle import ac
    from l3c_pytorch_b200 import _lib, codec, engine as E, seek
    dev = torch.device('cuda:0')
    rng = np.random.default_rng(900 + L)
    ss = [make_stream(rng, k, n, L) for (k, n) in
          [('flat', 700), ('peaked', 1501), ('straddle-run', 999), ('uniform', 640), ('tail', 1), ('flat', 64)]]
    n = np.array([s.n for s in ss], np.int64)
    iv = torch.from_numpy(np.concatenate([_intervals(s, L) for s in ss]).view(np.int32)).to(dev)
    pitch = E.table_pitch(L)
    rows = np.zeros((int(n.sum()), pitch), np.uint16)
    rows[:, :L] = np.concatenate([s.cdf[:, :L] for s in ss])
    table = torch.from_numpy(rows.view(np.int16)).to(dev)
    for every in (32, 96, 4096):
        caps = np.array([codec._slot_cap(int(k)) for k in n], np.int64)
        slots = torch.zeros(int(caps.sum()) + 16, dtype=torch.uint8, device=dev)
        desc = np.zeros(len(ss), _lib.ENC_STREAM_DTYPE)
        desc['intervals'] = iv.data_ptr() + 4 * (np.cumsum(n) - n)
        desc['out'] = slots.data_ptr() + np.cumsum(caps) - caps
        desc['n_sym'], desc['out_cap'] = n, caps
        counts = seek.point_counts(n, every)
        pts = torch.zeros(max(1, int(counts.sum())), 4, dtype=torch.int32, device=dev)
        _, lens, _ = E.ac_encode_streams_seek(desc, dev, every, pts, np.cumsum(counts) - counts)
        lens = lens.cpu().numpy().astype(np.int64)
        host = slots.cpu().numpy()
        words = pts.cpu().numpy().view(np.uint32)
        low, high, flip, bits = _pack_words(words)
        k0 = 0
        for i, s in enumerate(ss):
            data = host[desc['out'][i] - slots.data_ptr():][:lens[i]].tobytes()
            assert data == ac.encode(s.cdf, s.sym), (s.kind, every)
            want, _ = record_points(s.cdf, data, L, every)
            got = list(zip(*(a[k0:k0 + counts[i]].tolist() for a in (low, high, flip, bits))))
            assert got == [tuple(p) for p in want], (s.kind, every)
            k0 += counts[i]
        # every segment of every stream in one launch, from the recorded points
        idx = seek.SeekIndex(every, counts, low[:k0], high[:k0], flip[:k0], bits[:k0])
        states = torch.from_numpy(np.concatenate([idx.state_words().reshape(-1), [0]]).astype(np.uint32)
                                  .view(np.int32)).to(dev)
        out = torch.full((int(n.sum()),), 0xEE, dtype=torch.uint8, device=dev)
        dd = np.zeros(len(ss), _lib.DEC_STREAM_DTYPE)
        dd['in'] = desc['out']
        dd['in_len'] = lens
        dd['n_sym'] = n
        dd['table'] = table.data_ptr() + 2 * pitch * (np.cumsum(n) - n)
        dd['sym_out'] = out.data_ptr() + np.cumsum(n) - n
        dd['row_pitch'] = pitch
        segs = seek.plan_segments(dd, np.sort(dd['in'].astype(np.int64)), np.full(len(ss), every, np.int64)
                                  [np.argsort(dd['in'].astype(np.int64))], idx.first[np.argsort(dd['in'].astype(
                                      np.int64))], states.data_ptr())
        assert segs.size == int(np.maximum(1, -(-n // every)).sum())
        E.ac_decode_segments(segs, dev, L)
        got = out.cpu().numpy()
        assert np.array_equal(got, np.concatenate([s.sym for s in ss]).astype(np.uint8)), every


# ----------------------------------------------------------------------------------------------
# the codec
# ----------------------------------------------------------------------------------------------
def _images(ragged, size, n=2):
    if ragged:
        return [util.make_image(40 + i, size - 16 * i, size - 8 * i) for i in range(n)]
    return torch.stack([util.make_image(40 + i, size, size) for i in range(n)])


CODEC_CASES = [
    # (config, recursive, precision, ragged, image size, K values)
    ('cr', 0, 'f16', False, 128, (32, 96, 4096, 1 << 20)),
    ('cr', 0, 'f16', True, 96, (96, 4096)),
    ('cr', 0, 'f16x2', False, 64, (96,)),
    ('cr', 0, 'fp32', False, 64, (96,)),
    ('cr_rgb_shared', 0, 'f16', False, 64, (32, 96)),
    ('cr_rgb_shared', 1, 'f16', False, 64, (96,)),
]


@pytest.mark.parametrize('case', CODEC_CASES, ids=lambda c: '%s-R%d-%s-%s' % (c[0], c[1], c[2],
                                                                           'ragged' if c[3] else 'equal'))
def test_codec_encode_index_decode(case):
    from l3c_pytorch_b200 import Bitcoding, engine
    cfg, R, mode, ragged, size, Ks = case
    bp = util.blueprint(cfg, 'cuda:0')
    bc = Bitcoding(bp, recursive=R)
    imgs = _images(ragged, size)
    with precision(mode):
        datas, bpsps = bc.encode_batch(imgs)
        serial = bc.decode_batch(datas)
        want = [im.unsqueeze(0).long() for im in imgs]
        for a, b in zip(serial, want):
            assert torch.equal(a.cpu(), b)
        for K in Ks:
            d2, bpsps2, seeks = bc.encode_batch(imgs, seek=K)
            assert d2 == datas and bpsps2 == bpsps, K
            assert seeks == bc.seek_index(datas, every=K), K
            engine.launch_log(reset=True)
            dec = bc.decode_batch(datas, seeks=seeks)
            kernels, _ = engine.launch_log(reset=True)
            for a, b in zip(dec, want):
                assert torch.equal(a.cpu(), b), K
            assert 'ac_decode_kernel' not in kernels, kernels          # no serial or pipelined decoder launch
            assert any(k.startswith('ac_decode_segments') for k in kernels), kernels
            if mode == 'f16' and not ragged and cfg == 'cr':
                assert 'ac_decode_segments_coarse' in kernels, kernels
        # a batch where one container has no index decodes it serially
        mixed = bc.decode_batch(datas, seeks=[seeks[0], None])
        for a, b in zip(mixed, want):
            assert torch.equal(a.cpu(), b)


def test_decode_with_seeks_on_a_lane_beside_other_work():
    from l3c_pytorch_b200 import Bitcoding, codec
    bp = util.blueprint('cr', 'cuda:0')
    bc = Bitcoding(bp)
    with precision('f16'):
        imgs_a = _images(False, 128)
        imgs_b = torch.stack([util.make_image(70 + i, 128, 128) for i in range(2)])
        da, _, sa = bc.encode_batch(imgs_a, seek=4096)
        db, _ = bc.encode_batch(imgs_b)
        calls = []
        orig = codec.BatchCodec._decode_rgb_pipelined
        codec.BatchCodec._decode_rgb_pipelined = lambda self, *a, **k: (calls.append(1), orig(self, *a, **k))[1]
        try:
            lanes = bc.decode_lanes(2, 2)
            side = bc.side_stream(2, 2)
            torch.cuda.synchronize()
            with torch.cuda.stream(side):
                job = bc.encode_batch_begin(imgs_b, stream=side)
            with torch.cuda.stream(lanes[0].main):
                out_a = bc.decode_batch(da, seeks=sa, lane=lanes[0])
            n_seek = len(calls)
            with torch.cuda.stream(lanes[1].main):
                out_b = bc.decode_batch(db, lane=lanes[1])
            enc = job.finish()
            torch.cuda.synchronize()
        finally:
            codec.BatchCodec._decode_rgb_pipelined = orig
        assert n_seek == 0 and len(calls) == 1               # the indexed decode never took the pipelined path
        assert enc[0] == db
        for out, imgs in ((out_a, imgs_a), (out_b, imgs_b)):
            for a, b in zip(out, imgs):
                assert torch.equal(a.cpu(), b.unsqueeze(0).long())


def test_refusals():
    from l3c_pytorch_b200 import Bitcoding
    bp = util.blueprint('cr', 'cuda:0')
    imgs = _images(False, 64)
    with precision('f16'):
        with pytest.raises(ValueError):
            Bitcoding(bp, tile=(32, 32)).encode_batch(imgs, seek=96)
        bc = Bitcoding(bp)
        for K in (0, 48, 1 << 25):
            with pytest.raises(ValueError):
                bc.encode_batch(imgs, seek=K)
        datas, _, seeks = bc.encode_batch(imgs, seek=96)
        with pytest.raises(ValueError):
            bc.decode_batch(datas, seeks=[seeks[1], seeks[0]])     # each index names its container
        with pytest.raises(ValueError):
            bc.decode_batch(datas, seeks=[seeks[0]])


# ----------------------------------------------------------------------------------------------
# junk containers
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', ['cr_32', 'cr_40x28', 'rgbs_64', 'rgbs_r2'])
def test_junk_containers_decode_with_their_index(kind):
    from l3c_pytorch_b200 import Bitcoding
    from tests.test_gpu_junk_containers import junk_sets
    from tests.test_malformed_containers_host import KINDS, build
    cfg, R = KINDS[kind][0], KINDS[kind][5]
    bc = Bitcoding(util.blueprint(cfg, 'cuda:0'), recursive=R)
    with precision('f16'):
        for name, payloads in junk_sets(kind).items():
            data = build(kind, payloads)[0]
            serial = bc.decode_batch([data])[0]
            seeks = bc.seek_index([data], every=32)
            assert torch.equal(bc.decode_batch([data], seeks=seeks)[0], serial), name


# ----------------------------------------------------------------------------------------------
# a stream past 2^32 code bits
# ----------------------------------------------------------------------------------------------
def test_segments_past_2_32_bits():
    """At L = 256 under the uniform prior every symbol is its own 8 code bits and leaves the coder in its initial
    state, so a stream of n random bytes followed by the terminator byte 0x40 codes n symbols, and the seek point
    before symbol j is (0, 2^32 - 1, no flip, 32 + 8 j)."""
    from l3c_pytorch_b200 import _lib, engine as E, seek
    dev = torch.device('cuda:0')
    n = (1 << 29) + 5000                                        # 2^32 + 40000 code bits
    g = torch.Generator(device=dev).manual_seed(5)
    buf = torch.randint(0, 256, (n + 16,), dtype=torch.uint8, device=dev, generator=g)
    buf[n] = 0x40
    row = torch.from_numpy(E.uniform_cdf_row(256).astype(np.uint16).view(np.int16)[:256].copy()).to(dev)
    firsts = np.array([(1 << 29) - 4096, (1 << 29) + 96, n - 1000], np.int64)   # the last segment ends the stream
    lens = np.array([8192, 4096, 1000], np.int64)
    bits = 32 + 8 * firsts
    assert (bits[1:] > (1 << 32)).all()
    words = np.zeros((3, seek.STATE_WORDS), np.uint32)
    words[:, 1] = 0xFFFFFFFF
    words[:, 3], words[:, 4] = bits & 0xFFFFFFFF, bits >> 32
    states = torch.from_numpy(words.reshape(-1).view(np.int32).copy()).to(dev)
    out = torch.zeros(int(lens.sum()), dtype=torch.uint8, device=dev)
    segs = np.zeros(3, _lib.DEC_STREAM_DTYPE)
    segs['in'], segs['in_len'] = buf.data_ptr(), n + 1
    segs['table'], segs['row_pitch'] = row.data_ptr(), 0
    segs['sym_out'] = out.data_ptr() + np.cumsum(lens) - lens
    segs['n_sym'] = lens
    segs['state'] = states.data_ptr() + 4 * seek.STATE_WORDS * np.arange(3)
    E.ac_decode_segments(segs, dev, 256)
    got = out.cpu().numpy()
    src = buf.cpu().numpy()
    want = np.concatenate([src[f:f + k] for f, k in zip(firsts, lens)])
    assert np.array_equal(got, want)
    del buf


# ----------------------------------------------------------------------------------------------
# command line
# ----------------------------------------------------------------------------------------------
def test_cli_seek_round_trip(tmp_path, capsys):
    from PIL import Image
    from l3c_pytorch_b200 import cli
    img = util.make_image(9, 64, 48)
    png = str(tmp_path / 'in.png')
    Image.fromarray(img.permute(1, 2, 0).numpy().astype(np.uint8)).save(png)
    out, dec = str(tmp_path / 'a.l3c'), str(tmp_path / 'a.png')
    base = ['--config', 'cr', '--precision', 'f16']
    with precision('f16'):                                  # restored after the calls set it
        _cli_round_trip(cli, base, tmp_path, png, out, dec, capsys)


def _cli_round_trip(cli, base, tmp_path, png, out, dec, capsys):
    from PIL import Image
    assert cli.main(base + ['enc', png, out, '--seek', '96']) == 0
    with open(out + '.seek', 'rb') as f:
        written = f.read()
    assert cli.main(base + ['dec', out, dec]) == 0
    assert np.array_equal(np.array(Image.open(dec)), np.array(Image.open(png)))
    assert cli.main(base + ['idx', out, '--every', '96']) == 1              # an index exists: no overwrite
    assert cli.main(base + ['idx', out, '--every', '96', '--overwrite']) == 0
    with open(out + '.seek', 'rb') as f:
        assert f.read() == written
    # an index of another container beside the file is refused, naming it
    other = str(tmp_path / 'b.l3c')
    img2 = util.make_image(10, 64, 48)
    png2 = str(tmp_path / 'in2.png')
    Image.fromarray(img2.permute(1, 2, 0).numpy().astype(np.uint8)).save(png2)
    assert cli.main(base + ['enc', png2, other, '--seek', '96']) == 0
    os.replace(other + '.seek', out + '.seek')
    capsys.readouterr()
    assert cli.main(base + ['dec', out, dec]) == 1
    assert out + '.seek' in capsys.readouterr().out
    # enc refuses a stale sidecar without --overwrite and removes it with it
    os.remove(out)
    assert cli.main(base + ['enc', png, out]) == 1
    assert cli.main(base + ['enc', png, out, '--overwrite']) == 0
    assert not os.path.isfile(out + '.seek')
    assert cli.main(base + ['dec', out, dec]) == 0
