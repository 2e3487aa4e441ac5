"""CPU: the layout of region updates from device-resident lengths (DESIGN §4.12, "Serving updates").

`restate_layout` restates the contract of l3c_update_layout (include/l3c_b200.h) in numpy: per container,
new_off = fixed_off + exclusive_scan(len), the size, the 2 n_new + 1 splice segments, their chunk prefix and the error
flag.  On containers built with ContainerLayout (tiles of several sizes, several containers in one call, re-encoded
sets that are empty, everything, the first or the last stream, or scattered), fed through codec.update_layout_inputs:
* the restated offsets and sizes are ContainerLayout.offsets of the new lengths;
* the restated segments, applied in numpy, write exactly the bytes of splice_segments applied in numpy, which are
  ContainerLayout's container of the new streams, inside each container's upper bound;
* a length above its cap sets bit 0 of the flag and gives its container no chunks.
tests/test_gpu_update_serving.py runs the kernels against the same restatement."""
import numpy as np
import pytest

from l3c_pytorch_b200.codec import (ContainerLayout, parse_container, splice_segments, tile_grid,
                                    update_layout_inputs)

CHUNK = 4096


def restate_layout(conts, streams, new_len, slot_off, caps):
    """l3c_update_layout in numpy -> (segments int64 [n_seg][4], chunk0 [n_seg + containers], sizes, flag,
    [new_off of each container's streams])."""
    n_seg = int((2 * conts['n_new'] + 1).sum())
    seg = np.zeros((n_seg, 4), np.int64)
    chunk0 = np.zeros(n_seg + len(conts), np.int64)
    sizes, offs, flag = np.zeros(len(conts), np.int64), [], 0
    for k, c in enumerate(conts):
        st = streams[c['first_stream']:c['first_stream'] + c['n_streams']]
        j = np.flatnonzero(st['src'] >= 0)
        src = st['src'][j]
        ln = st['old_len'].copy()
        ln[j] = new_len[src]
        err = int((ln[j] > caps[src]).any())
        new_off = st['fixed_off'] + np.concatenate([[0], np.cumsum(ln)[:-1]])
        total = c['fixed_total'] + ln.sum()
        if total > c['out_cap'] or j.size != c['n_new']:
            err |= 2
        s = seg[c['first_seg']:c['first_seg'] + 2 * j.size + 1]
        s[1::2] = np.stack([np.ones_like(j), slot_off[src], c['out_base'] + new_off[j], ln[j]], 1)
        s[2::2, :3] = np.stack([np.zeros_like(j), c['old_base'] + st['old_off'][j] + st['old_len'][j],
                                c['out_base'] + new_off[j] + ln[j]], 1)
        s[0, :3] = (0, c['old_base'], c['out_base'])
        s[0::2, 3] = np.concatenate([c['out_base'] + new_off[j] - 4, [c['out_base'] + total]]) - s[0::2, 2]
        if (s[0::2, 3] < 0).any():
            err |= 2
        n = np.where(s[:, 3] > 0, -(-s[:, 3] // CHUNK), s[:, 0]) * (err == 0)
        ch = chunk0[c['first_seg'] + k:c['first_seg'] + k + s.shape[0] + 1]
        ch[1:] = np.cumsum(n)
        sizes[k] = total
        offs.append(new_off)
        flag |= err
    return seg, chunk0, sizes, flag, offs


def apply_segments(old, slots, seg, out):
    """l3c_splice_streams' copy in numpy."""
    for src, so, d, n in seg.tolist():
        out[d:d + n] = (slots if src else old)[so:so + n]
        if src:
            out[d - 4:d] = np.frombuffer(np.uint32(n).tobytes(), np.uint8)


def make_container(rng, shapes, tile, lens=None, pad=(1, 2, 3, 4)):
    """A container of ContainerLayout with random stream bytes -> (bytes, scales (parse_container), stream bytes)."""
    layout = ContainerLayout([(i, C, H, W) for i, (C, H, W) in enumerate(shapes)], tile)
    n = sum(C * len(tile_grid(H, W, tile)) for C, H, W in shapes)
    lens = rng.integers(0, 120, n) if lens is None else lens
    total, pieces, offs = layout.header_and_offsets(lens, pad)
    buf = np.zeros(total, np.uint8)
    for o, b in pieces:
        buf[o:o + len(b)] = np.frombuffer(b, np.uint8)
    body = [rng.integers(0, 256, int(ln), dtype=np.uint8) for ln in lens]
    for o, b in zip(offs, body):
        buf[o:o + len(b)] = b
    data = buf.tobytes()
    pt, scales = parse_container(data)
    assert pt == pad
    return data, scales, body


def make_container_from(shapes, tile, body, pad):
    layout = ContainerLayout([(i, C, H, W) for i, (C, H, W) in enumerate(shapes)], tile)
    total, pieces, offs = layout.header_and_offsets([len(b) for b in body], pad)
    buf = np.zeros(total, np.uint8)
    for o, b in pieces:
        buf[o:o + len(b)] = np.frombuffer(b, np.uint8)
    for o, b in zip(offs, body):
        buf[o:o + len(b)] = b
    return buf


SHAPES = [(5, 8, 12), (5, 16, 24), (3, 32, 48)]


def build_call(rng, specs):
    """specs: [(tile, which)] with which in 'none', 'all', 'first', 'last', 'some'.  -> everything of one call: the
    uploaded blob, the containers' (shapes, tile, body, cols, lens), new lengths, caps, slots, slot offsets and the
    inputs of l3c_update_layout."""
    datas, per = [], []
    call_lens, call_caps = [], []
    for tile, which in specs:
        data, scales, body = make_container(rng, SHAPES, tile)
        n = len(body)
        cols = {'none': np.zeros(0, np.int64), 'all': np.arange(n), 'first': np.array([0]),
                'last': np.array([n - 1])}.get(which)
        if cols is None:
            cols = np.sort(rng.choice(n, max(2, n // 5), replace=False))
        caps = rng.integers(0, 200, cols.size) + 4
        lens = np.minimum(rng.integers(0, 220, cols.size), caps)
        lens[::3] = caps[::3]                                  # some fill their slot exactly
        src = np.arange(cols.size) + sum(c.size for c in call_lens)
        call_lens.append(lens)
        call_caps.append(caps)
        datas.append(data)
        per.append((scales, tile, body, cols, lens, src))
    new_len = np.concatenate(call_lens).astype(np.int64) if call_lens else np.zeros(0, np.int64)
    caps = np.concatenate(call_caps).astype(np.int64)
    slot_off = np.concatenate([[0], np.cumsum(caps)])[:-1] + 8
    slots = rng.integers(0, 256, int(caps.sum()) + 16, dtype=np.uint8)
    starts = np.zeros(len(datas), np.int64)
    pos = 0
    for k, d in enumerate(datas):
        starts[k] = pos
        pos += (len(d) + 15) & ~15
    blob = np.zeros(pos + 16, np.uint8)
    for k, d in enumerate(datas):
        blob[starts[k]:starts[k] + len(d)] = np.frombuffer(d, np.uint8)
    conts, streams, out_starts, out_bytes = update_layout_inputs(
        [(scales, tile, starts[k], len(datas[k]), cols, src) for k, (scales, tile, _, cols, _, src) in enumerate(per)],
        caps)
    return dict(datas=datas, per=per, new_len=new_len, caps=caps, slots=slots, slot_off=slot_off, blob=blob,
                starts=starts, conts=conts, streams=streams, out_starts=out_starts, out_bytes=out_bytes)


CASES = [[((8, 8), 'some')], [((16, 24), 'none')], [((4, 12), 'all')], [((64, 64), 'first')], [((8, 8), 'last')],
         [((8, 8), 'some'), ((16, 24), 'none'), ((4, 12), 'all'), ((64, 64), 'first'), ((8, 8), 'last'),
          ((16, 24), 'some')]]


@pytest.mark.parametrize('case', range(len(CASES)), ids=['some', 'none', 'all', 'first', 'last', 'six'])
def test_restated_layout_gives_the_container_layout(case):
    specs = CASES[case]
    rng = np.random.default_rng(100 + case)
    c = build_call(rng, specs)
    seg, chunk0, sizes, flag, offs = restate_layout(c['conts'], c['streams'], c['new_len'], c['slot_off'], c['caps'])
    assert flag == 0
    out = np.full(c['out_bytes'] + 32, 0xA5, np.uint8)
    apply_segments(c['blob'], c['slots'], seg, out)
    want_out = np.full_like(out, 0xA5)
    for k, (scales, tile, body, cols, lens, src) in enumerate(c['per']):
        layout = ContainerLayout([(i, C, H, W) for i, (C, H, W, _) in enumerate(scales)], tile)
        old_len = np.array([len(b) for b in body], np.int64)
        new_len = old_len.copy()
        new_len[cols] = lens
        total, new_off = layout.offsets(new_len)
        assert np.array_equal(offs[k], new_off) and sizes[k] == total
        assert total <= c['conts'][k]['out_cap'] and c['conts'][k]['out_cap'] % 16 == 0
        # splice_segments' bytes, applied the same way
        _, old_off = layout.offsets(old_len)
        s = splice_segments(old_off, old_len, len(c['datas'][k]), new_off, cols, lens, c['slot_off'][src],
                            c['starts'][k], c['out_starts'][k])
        apply_segments(c['blob'], c['slots'], s, want_out)
        # and the container itself: the old streams with the new ones in their places
        new_body = list(body)
        for col, ln, so in zip(cols, lens, c['slot_off'][src]):
            new_body[col] = c['slots'][so:so + ln]
        s0 = c['out_starts'][k]
        assert np.array_equal(out[s0:s0 + total], make_container_from(SHAPES, tile, new_body, (1, 2, 3, 4)))
        # chunks: every byte of the container in one 4 KB chunk of its segment, one chunk per empty new stream
        ns = 2 * cols.size + 1
        ch = chunk0[c['conts'][k]['first_seg'] + k:][:ns + 1]
        sg = seg[c['conts'][k]['first_seg']:][:ns]
        assert ch[0] == 0 and ch[-1] == sum(-(-n // CHUNK) if n else src_ for src_, _, _, n in sg.tolist())
    assert np.array_equal(out, want_out)


def test_a_length_above_its_cap_flags_the_container_and_gives_it_no_chunks():
    rng = np.random.default_rng(3)
    c = build_call(rng, [((8, 8), 'some'), ((16, 24), 'all')])
    new_len = c['new_len'].copy()
    k = c['conts'][0]['n_new'] - 1                                 # the last new stream of container 0
    new_len[k] = c['caps'][k] + 1
    seg, chunk0, sizes, flag, _ = restate_layout(c['conts'], c['streams'], new_len, c['slot_off'], c['caps'])
    assert flag == 1
    n0 = 2 * c['conts'][0]['n_new'] + 1
    assert (chunk0[:n0 + 1] == 0).all() and chunk0[n0 + 1 + 2 * c['conts'][1]['n_new'] + 1] > 0


def test_inputs_for_no_containers():
    conts, streams, starts, size = update_layout_inputs([], np.zeros(0, np.int64))
    assert conts.size == 0 and streams.size == 0 and starts.size == 0 and size == 0
