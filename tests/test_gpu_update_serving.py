"""GPU: region updates in flight (DESIGN §4.12, "Serving updates"), BatchCodec.update_regions_begin /
Bitcoding.update_regions_begin.

* begin(...).finish() is byte for byte update_regions(...) and the encode of the edited images, with the same counts:
  one edit, many edits, overlapping edits, containers of different tile sizes in one call, an empty edit list and a
  whole-path container; in f16 (one ragged pass) and fp32 (plan after plan).
* begin does not wait for the GPU: with a long sleep queued ahead of it, on the current stream or on a decode lane, it
  returns while the sleep still runs, and no torch operation in it synchronises.
* Two jobs on two decode lanes beside a decode_batch on a third, finished in reverse order, are all correct.
* Every refusal of update_regions is raised by begin with no launch.
* l3c_update_layout and l3c_splice_streams_dev against the numpy restatement of tests/test_update_layout_host.py:
  segments, chunk prefixes, sizes, flag and bytes, with guard bytes around every container's upper bound; a length
  handed to the layout above its cap sets the flag and that container is not written."""
import numpy as np
import pytest
import torch

from tests import util
from tests.test_gpu_update_regions import _bc, _edited, _encode, _image, _patch
from tests.test_update_layout_host import CASES, build_call, restate_layout

pytestmark = pytest.mark.gpu


@pytest.fixture
def mode():
    from l3c_pytorch_b200 import engine as E
    old = E.get_conv_precision()
    yield E.set_conv_precision
    E.set_conv_precision(old)


def _call(bc16, bc24):
    """Containers of two tile sizes (two Bitcodings of one model) and their edit lists."""
    imgs = [_image(11, 517, 389), _image(12, 301, 255), _image(13, 131, 97), _image(14, 256, 1024)]
    edits = [
        [((100, 90), _patch(1, 40, 33))],                                                   # one edit
        [((10, 20), _patch(2, 30, 30)), ((25, 30), _patch(3, 20, 20)),                      # overlapping, the later wins
         ((200, 100), _patch(4, 9, 11)), ((0, 0), _patch(5, 1, 1))],
        [],                                                                                 # no edit
        [((10, 50), _patch(6, 20, 30)), ((200, 950), _patch(7, 30, 40)), ((100, 500), _patch(8, 8, 8))],
    ]
    bcs = [bc16, bc24, bc16, bc24]
    datas = [_encode(b, img) for b, img in zip(bcs, imgs)]
    return imgs, edits, bcs, datas


def _device_edits(edits):
    return [[(pos, p.to(torch.uint8).cuda()) for pos, p in ed] for ed in edits]


def _check_bytes(bcs, imgs, edits, outs):
    for b, img, ed, got in zip(bcs, imgs, edits, outs):
        assert got == _encode(b, _edited(img, ed))


@pytest.mark.parametrize('prec', ['f16', 'fp32'])
def test_begin_finish_equals_update_regions(mode, prec):
    mode(prec)
    bc16, bc24 = _bc((16, 16)), _bc((16, 24))
    imgs, edits, bcs, datas = _call(bc16, bc24)
    want = bc16.update_regions(datas, edits)
    counts = bc16.codec.updates_counts
    stage = dict(bc16.codec.updates_stage_ms)
    job = bc16.update_regions_begin(datas, edits)
    assert bc16.codec.updates_counts is counts and bc16.codec.updates_stage_ms == stage
    got = job.finish()
    assert got == want
    assert job.counts == counts and [c['plans'] > 0 for c in counts] == [True, True, False, True]
    assert got[2] == datas[2]
    _check_bytes(bcs, imgs, edits, got)
    with pytest.raises(RuntimeError, match='called before'):
        job.finish()


def test_whole_path_container_in_flight(monkeypatch):
    from l3c_pytorch_b200 import codec
    bc16, bc24 = _bc((16, 16)), _bc((16, 24))
    imgs, edits, bcs, datas = _call(bc16, bc24)
    bc16.update_regions(datas, edits)
    big = bc16.codec.updates_counts[0]['window_pixels']
    monkeypatch.setattr(codec, 'TILED_ENCODE_BAND_PIXELS', big - 1)       # container 0's window exceeds the budget
    want = bc16.update_regions(datas, edits)
    whole = [c['whole'] for c in bc16.codec.updates_counts]
    assert whole[0] and not whole[1] and not whole[2]
    job = bc16.update_regions_begin(datas, edits)
    got = job.finish()
    assert got == want and job.counts == bc16.codec.updates_counts
    _check_bytes(bcs, imgs, edits, got)
    # a call of whole-path containers only
    job = bc16.update_regions_begin(datas[:1], edits[:1])
    assert job.finish() == want[:1]


def _sleep_ahead(stream):
    """A sleep of about a second queued on `stream`, and an event recorded after it."""
    with torch.cuda.stream(stream):
        torch.cuda._sleep(2 * 10 ** 9)
        ev = torch.cuda.Event()
        ev.record()
    return ev


@pytest.mark.parametrize('on_lane', [False, True])
def test_begin_does_not_wait(mode, on_lane):
    mode('f16')
    bc16, bc24 = _bc((16, 16)), _bc((16, 24))
    imgs, edits, bcs, datas = _call(bc16, bc24)
    datas, edits = datas[1:2], _device_edits(edits[1:2])     # few launches: none waits for room in the stream's queue
    want = bc16.update_regions(datas, edits)
    lane = bc16.decode_lanes(4, n_lanes=1)[0] if on_lane else None
    stream = lane.main if on_lane else torch.cuda.current_stream()
    bc16.update_regions_begin(datas, edits, lane=lane).finish()            # every stream and kernel warmed up
    torch.cuda.synchronize()
    ev = _sleep_ahead(stream)
    with torch.cuda.stream(stream):
        torch.cuda.set_sync_debug_mode('error')
        try:
            job = bc16.update_regions_begin(datas, edits, lane=lane)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert not ev.query(), 'update_regions_begin waited for the work queued before it'
    assert job.finish() == want
    assert ev.query()


def test_two_jobs_on_two_lanes_beside_a_decode(mode):
    mode('f16')
    bc16, bc24 = _bc((16, 16)), _bc((16, 24))
    imgs, edits, bcs, datas = _call(bc16, bc24)
    edits_b = [[((5, 7), _patch(20 + i, 12, 17)), ((60, 40), _patch(30 + i, 25, 6))] for i in range(len(datas))]
    want_a = bc16.update_regions(datas, edits)
    want_b = bc16.update_regions(datas, edits_b)
    batch = torch.stack([util.make_image(500 + i, 64, 96) for i in range(3)])
    coded, _ = bc16.encode_batch(batch)
    want_dec = bc16.decode_batch(coded)
    ea, eb = _device_edits(edits), _device_edits(edits_b)
    torch.cuda.synchronize()
    lanes = bc16.decode_lanes(4, n_lanes=3)
    cur = torch.cuda.current_stream()
    for ln in lanes:
        ln.main.wait_stream(cur)
    with torch.cuda.stream(lanes[0].main):
        job_a = bc16.update_regions_begin(datas, ea, lane=lanes[0])
    with torch.cuda.stream(lanes[1].main):
        job_b = bc16.update_regions_begin(datas, eb, lane=lanes[1])
    with torch.cuda.stream(lanes[2].main):
        got_dec = bc16.decode_batch(coded, lane=lanes[2])
    assert job_b.finish() == want_b
    assert job_a.finish() == want_a
    for ln in lanes:
        cur.wait_stream(ln.main)
    torch.cuda.synchronize()
    for g, w in zip(got_dec, want_dec):
        assert torch.equal(g, w)


def test_refusals_from_begin_before_any_launch():
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
    lane = bc.decode_lanes(1, n_lanes=1)[0]
    torch.cuda.synchronize()
    E.launch_log(reset=True)
    for b, ds, eds, match in cases:
        with pytest.raises(ValueError, match=match):
            b.update_regions_begin(ds, eds)
        with pytest.raises(ValueError, match=match):
            b.update_regions_begin(ds, eds, lane=lane)
    assert E.launch_log()[1] == 0


def _run_kernels(c, new_len):
    """l3c_update_layout and l3c_splice_streams_dev on one call of build_call: -> (info, segments and chunk prefix,
    output with 64 guard bytes on each side of the call's upper bound)."""
    from l3c_pytorch_b200 import engine as E
    dev = torch.device('cuda:0')
    blob = torch.from_numpy(c['blob']).to(dev)
    slots = torch.from_numpy(c['slots']).to(dev)
    guard = torch.full((c['out_bytes'] + 128,), 0xA5, dtype=torch.uint8, device=dev)
    out = guard[64:64 + c['out_bytes']]
    lens = torch.from_numpy(new_len.astype(np.int32)).to(dev)
    info, keep = E.update_splice(c['conts'], c['streams'], lens, c['slot_off'], c['caps'], blob, slots, out)
    torch.cuda.synchronize()
    return info.cpu().numpy(), keep[1].cpu().numpy(), guard.cpu().numpy()


@pytest.mark.parametrize('case', range(len(CASES)))
def test_layout_and_splice_kernels_against_the_restatement(case):
    from tests.test_update_layout_host import apply_segments
    c = build_call(np.random.default_rng(200 + case), CASES[case])
    seg, chunk0, sizes, flag, _ = restate_layout(c['conts'], c['streams'], c['new_len'], c['slot_off'], c['caps'])
    info, seg_dev, got = _run_kernels(c, c['new_len'])
    n_seg = seg.shape[0]
    assert np.array_equal(info[:-1], sizes) and info[-1] == flag == 0
    assert np.array_equal(seg_dev[:4 * n_seg].reshape(-1, 4), seg)
    assert np.array_equal(seg_dev[4 * n_seg:], chunk0)
    want = np.full(c['out_bytes'] + 128, 0xA5, np.uint8)
    apply_segments(c['blob'], c['slots'], seg + np.array([0, 0, 64, 0]), want)
    assert np.array_equal(got, want)


def test_a_length_above_its_cap_is_flagged_and_not_spliced():
    """Lengths handed to the layout kernel directly: no range coder runs and nothing is written out of bounds."""
    c = build_call(np.random.default_rng(7), [((8, 8), 'some'), ((16, 24), 'all')])
    new_len = c['new_len'].copy()
    k = c['conts'][0]['n_new'] - 1
    new_len[k] = c['caps'][k] + 1
    seg, chunk0, sizes, flag, _ = restate_layout(c['conts'], c['streams'], new_len, c['slot_off'], c['caps'])
    info, seg_dev, got = _run_kernels(c, new_len)
    assert info[-1] == flag == 1 and np.array_equal(info[:-1], sizes)
    n_seg = seg.shape[0]
    assert np.array_equal(seg_dev[4 * n_seg:], chunk0)
    c0, c1 = c['conts']
    assert (got[64 + c0['out_base']:64 + c0['out_base'] + c0['out_cap']] == 0xA5).all()    # container 0: untouched
    want = np.full(c['out_bytes'] + 128, 0xA5, np.uint8)
    from tests.test_update_layout_host import apply_segments
    apply_segments(c['blob'], c['slots'], seg[c1['first_seg']:] + np.array([0, 0, 64, 0]), want)
    assert np.array_equal(got, want)
