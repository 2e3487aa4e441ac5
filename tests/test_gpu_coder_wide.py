"""GPU: the range decoder for alphabets of 257 to 32768 symbols (range_coder.cu, wide::ac_decode_wide_kernel) against
the CPU oracle (oracle.ac, pinned to the reference at these alphabets by oracle/pin_oracle_wide.py): through the
drop-in torchac API, and batched through l3c_ac_decode_streams -- ragged streams decoded in place from odd byte
offsets, uint16 outputs at every 2-byte offset, junk and truncated streams in the same launches, several chunk
schedules with the saved state checked against the oracle after every launch."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ac
from tests.test_gpu_coder import _mixture_case
from tests.test_gpu_coder_launches import _encode_and_pack, _schedules, make_stream

DROPIN_L = (257, 258, 300, 511, 512, 513, 1024, 4095, 4096, 4097, 32768)
KINDS = ('flat', 'peaked', 'tail', 'straddle', 'uniform', 'mix')
TABLE_BYTES = 64 << 20            # per drop-in table


def _stream(rng, kind, n, L):
    """make_stream, with kinds whose rows cannot be strictly increasing at this L (the straddling rows hold
    2^14-count ranges) replaced by flat ones"""
    s = make_stream(rng, kind, n, L)
    if not (np.diff(s.cdf[:, :L].astype(np.int64), axis=1) > 0).all():
        s = make_stream(rng, 'flat', n, L)
        s.kind = kind + '->flat'
    assert (np.diff(s.cdf[:, :L].astype(np.int64), axis=1) > 0).all()
    return s


def _t_cdf(cdf):
    return torch.from_numpy(np.ascontiguousarray(cdf).view(np.int16).copy()).reshape(1, 1, cdf.shape[0], -1)


@pytest.mark.gpu
@pytest.mark.parametrize('L', DROPIN_L)
def test_dropin_round_trip_and_corrupt_input_match_oracle(L):
    """encode_cdf / decode_cdf at lengths 1 .. a few thousand (tables capped at 64 MB): the bytes equal the oracle's,
    the decode returns the symbols, and junk, truncated and empty input decode to the oracle's symbols"""
    from l3c_pytorch_b200 import torchac
    rng = np.random.default_rng(900 + L)
    n_max = min(3000, TABLE_BYTES // (2 * (L + 1)))
    for n in sorted({1, 2, 9, 64, n_max // 3, n_max}):
        for kind in KINDS:
            s = _stream(rng, kind, n, L)
            t = _t_cdf(s.cdf)
            data = torchac.encode_cdf(t, torch.from_numpy(s.sym))
            assert data == ac.encode(s.cdf, s.sym), (L, n, s.kind)
            assert (torchac.decode_cdf(t, data).numpy() == s.sym).all(), (L, n, s.kind)
            if kind in ('flat', 'tail'):
                junk = bytes(rng.integers(0, 256, len(data)).astype(np.uint8))
                for what, b in (('junk', junk), ('half', data[:len(data) // 2]), ('all but one', data[:-1]),
                                ('empty', b'')):
                    got = torchac.decode_cdf(t, b).numpy()
                    assert (got == ac.decode(s.cdf, b)).all(), (L, n, s.kind, what)


def _check_wide_launches(L, lengths):
    from l3c_pytorch_b200 import _lib, engine as E
    dev = torch.device('cuda')
    rng = np.random.default_rng(300 + L)
    ss = [_stream(rng, k, n, L) for n in lengths for k in KINDS]
    order = rng.permutation(len(ss))
    ss = [ss[i] for i in order]
    for s in ss:
        s.want = ac.encode(s.cdf, s.sym)
        s.sym = s.sym.astype(np.int64)          # _intervals forms sym + 1, which int16 cannot hold at L = 32768
    n_all = len(ss)
    n = np.array([s.n for s in ss], np.int64)
    lens, dst, blob, _ = _encode_and_pack(ss, L, dev)
    hb = blob.cpu().numpy()
    for i, s in enumerate(ss):
        assert hb[dst[i]:dst[i] + lens[i]].tobytes() == s.want, (L, i, s.kind)
    long_ = [i for i in range(n_all) if n[i] >= 64]
    junk, trunc = long_[:3], dict(zip(long_[3:8], (0.0, 0.33, -1, 1, 0.9)))
    in_len = lens.copy()
    for i in junk:
        blob[int(dst[i]):int(dst[i] + lens[i])] = torch.from_numpy(rng.integers(0, 256, int(lens[i]), np.uint8))
    for i, f in trunc.items():
        in_len[i] = lens[i] - 1 if f == -1 else (f if f == 1 else int(lens[i] * f))
    hb = blob.cpu().numpy()
    want_sym, trace = [], []
    for i, s in enumerate(ss):
        sym, tr = ac.decode_trace(s.cdf, hb[dst[i]:dst[i] + in_len[i]].tobytes())
        if i not in junk and i not in trunc:
            assert (sym == s.sym).all(), (L, i)
        want_sym.append(sym.astype(np.uint16))
        trace.append(tr)
    pitch = E.table_pitch(L)
    tab = np.zeros((int(n.sum()), pitch), np.uint16)
    tab[:, :L] = np.concatenate([s.cdf[:, :L] for s in ss])
    tab_dev = torch.from_numpy(tab.view(np.int16)).to(dev)
    row0 = np.concatenate([[0], np.cumsum(n)[:-1]])
    # uint16 outputs at +0/+2/+4/+6 bytes from an 8-byte boundary, each followed by 8 guard bytes
    slot = (2 * n + 8 + 7) // 8 * 8 + 8
    out0 = np.concatenate([[0], np.cumsum(slot)[:-1]]) + 2 * (np.arange(n_all) % 4)
    out = torch.empty(int(slot.sum()), dtype=torch.uint8, device=dev)
    state = torch.empty(4 * n_all, dtype=torch.int32, device=dev)
    dd = np.zeros(n_all, dtype=_lib.DEC_STREAM_DTYPE)
    dd['table'] = tab_dev.data_ptr() + 2 * pitch * row0
    dd['in'] = blob.data_ptr() + dst
    dd['sym_out'] = out.data_ptr() + out0
    dd['state'] = state.data_ptr() + 16 * np.arange(n_all)
    dd['row_pitch'] = pitch
    dd['n_sym'] = n
    dd['in_len'] = in_len
    desc_dev = E._desc_to_device(dd, dev)
    for k, (sched_name, sched) in enumerate(_schedules(rng, int(n.max()))):
        n_use = n_all - k % 3                    # streams past n_use must stay untouched
        out.fill_(0xA5)
        state.fill_(-1)
        E.launch_log(reset=True)
        for (first, count) in sched:
            E.ac_decode_streams(dd, dev, L, first, count, desc_dev=desc_dev, n=n_use)
            st = state.cpu().numpy().view(np.uint32).reshape(n_all, 4)
            for i in range(n_use):
                if first >= n[i]:
                    continue
                want = trace[i][min(first + count, int(n[i]) - 1)]
                assert (st[i] == want).all(), ('L=%d, schedule "%s", launch (%d, %d), stream %d (%s, n=%d, in_len=%d/%d):'
                                               ' saved state %s, oracle %s' % (L, sched_name, first, count, i,
                                                                               ss[i].kind, n[i], in_len[i], lens[i],
                                                                               st[i].tolist(), want.tolist()))
        kernels, _ = E.launch_log(reset=True)
        assert kernels == {'ac_decode_wide_kernel': len(sched)}, kernels
        got = out.cpu().numpy()
        for i in range(n_all):
            o = int(out0[i])
            seg = got[o:o + 2 * int(n[i])].view(np.uint16)
            guard = got[o + 2 * int(n[i]):o + 2 * int(n[i]) + 8]
            if i >= n_use:
                assert (got[o:o + 2 * int(n[i])] == 0xA5).all(), (L, sched_name, 'stream outside the launch', i)
                continue
            bad = np.flatnonzero(seg != want_sym[i])
            assert bad.size == 0, ('L=%d, schedule "%s", stream %d (%s, n=%d, in_len=%d/%d): %d wrong symbols, first '
                                   'at %d' % (L, sched_name, i, ss[i].kind, n[i], in_len[i], lens[i], bad.size,
                                              bad[0]))
            assert (guard == 0xA5).all(), (L, sched_name, 'write past the end of stream', i)
    del tab_dev, blob


@pytest.mark.gpu
@pytest.mark.parametrize('L,lengths', [(257, (1, 2, 7, 8, 9, 33, 65, 700, 1501)), (1000, (1, 8, 9, 65, 700)),
                                       (4097, (1, 9, 65, 700)), (32768, (1, 9, 65, 130))])
def test_batched_chunked_ragged_wide_decode_matches_oracle(L, lengths):
    """ragged streams of every kind in one descriptor array, decoded in place from odd byte offsets into uint16
    outputs at +0/+2/+4/+6 bytes, under five chunk schedules, with 3 junk and 5 truncated streams in the same
    launches: every stream decodes to the oracle's symbols for the bytes it was given, its saved state equals the
    oracle's after every launch, nothing is written past its symbols or for streams outside the launch, and only
    the wide kernel is launched"""
    _check_wide_launches(L, lengths)


@pytest.mark.gpu
def test_shared_row_pitch_0_decodes_the_uniform_kat():
    """row_pitch 0 (one shared row) at L = 1024: the uniform KAT of pin_oracle_wide decodes"""
    from l3c_pytorch_b200 import _lib, engine as E
    from oracle import pin_oracle_wide as pw
    dev = torch.device('cuda')
    data = bytes.fromhex('003ff80001ff84da014d00000fffe740')
    n = len(pw.KAT_SYM)
    assert ac.encode(pw.kat_row(), np.array(pw.KAT_SYM, np.int16)) == data
    row = torch.from_numpy(pw.kat_row()[:1024].view(np.int16).copy()).to(dev)
    blob = torch.zeros(64, dtype=torch.uint8, device=dev)
    blob[5:5 + len(data)] = torch.tensor(list(data), dtype=torch.uint8)
    out = torch.zeros(n + 4, dtype=torch.int16, device=dev)
    dd = np.zeros(1, dtype=_lib.DEC_STREAM_DTYPE)
    dd['table'], dd['in'], dd['sym_out'] = row.data_ptr(), blob.data_ptr() + 5, out.data_ptr()
    dd['row_pitch'], dd['n_sym'], dd['in_len'] = 0, n, len(data)
    E.ac_decode_streams(dd, dev, 1024)
    got = out.cpu().numpy()
    assert got[:n].tolist() == pw.KAT_SYM and (got[n:] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize('K,H,W,L', [(10, 16, 24, 1024, ), (3, 9, 11, 4096)])
def test_logistic_mixture_dropin_wide_vs_oracle(K, H, W, L):
    """encode_logistic_mixture / decode_logistic_mixture at Lp = 1025 and 4097, to the bar of
    test_gpu_coder.test_logistic_mixture_dropin_vs_oracle: an exact round trip; the GPU decoder decodes the oracle's
    stream, and the bytes are identical, whenever the integers of every coded interval agree; sizes agree"""
    from l3c_pytorch_b200 import torchac
    rng = np.random.default_rng(K * H * W + L)
    targets, mu, ls, pi = _mixture_case(rng, K, H, W, L, 0., float(L - 1))
    n = H * W
    cdf_o = ac.mixture_cdf(targets.numpy(), mu.reshape(K, n).numpy(), ls.reshape(K, n).numpy(),
                           pi.reshape(K, n).numpy())
    assert (np.diff(cdf_o[:, :L].astype(np.int64), axis=1) > 0).all()
    sym = rng.integers(0, L, size=n).astype(np.int16)
    dev = [t.cuda() for t in (targets, mu, ls, pi)]
    data = torchac.encode_logistic_mixture(*dev, torch.from_numpy(sym))
    back = torchac.decode_logistic_mixture(*dev, data).numpy()
    assert (back == sym).all()
    data_o = ac.encode(cdf_o, sym)
    if data_o == data:
        assert (torchac.decode_logistic_mixture(*dev, data_o).numpy() == sym).all()
    assert abs(len(data) - len(data_o)) <= max(2, len(data_o) // 1000)


@pytest.mark.gpu
def test_wide_alphabet_errors():
    from l3c_pytorch_b200 import _lib, engine as E, torchac
    from l3c_pytorch_b200._lib import lib
    rng = np.random.default_rng(3)
    s = make_stream(rng, 'flat', 4, 32768)
    bad = np.concatenate([s.cdf, np.zeros((4, 1), np.uint16)], 1)             # Lp = 32770
    with pytest.raises(RuntimeError, match=r'\[2,32769\]'):
        torchac.encode_cdf(_t_cdf(bad), torch.from_numpy(s.sym))
    with pytest.raises(RuntimeError, match=r'\[2,32769\]'):
        torchac.decode_cdf(_t_cdf(bad), b'\x12\x34')
    s = make_stream(rng, 'flat', 4, 1024)                                    # (int16 cannot hold 32768)
    sym = s.sym.copy()
    sym[2] = 1024                                                            # = Lp - 1
    with pytest.raises(RuntimeError, match='outside'):
        torchac.encode_cdf(_t_cdf(s.cdf), torch.from_numpy(sym))
    # l3c_ac_decode_streams: L = 32769, and row pitches a wide alphabet cannot use
    dev = torch.device('cuda')
    tab = torch.zeros(4 * 1040, dtype=torch.int16, device=dev)
    out = torch.zeros(16, dtype=torch.int16, device=dev)
    blob = torch.zeros(64, dtype=torch.uint8, device=dev)
    for L, pitch, ok in [(32769, 32776, False), (1000, 1004, False), (1000, 992, False), (1000, 1001, False),
                         (1000, 1000, True), (1000, 1040, True), (1000, 0, True)]:
        dd = np.zeros(1, dtype=_lib.DEC_STREAM_DTYPE)
        dd['table'], dd['in'], dd['sym_out'] = tab.data_ptr(), blob.data_ptr(), out.data_ptr()
        dd['row_pitch'], dd['n_sym'], dd['in_len'] = pitch, 4, 8
        d = E._desc_to_device(dd, dev)
        rc = lib.l3c_ac_decode_streams(ctypes.c_void_p(d.data_ptr()), 1, L, 0, 4, None)
        assert rc == (0 if ok else -1), (L, pitch, rc)
        torch.cuda.synchronize()


@pytest.mark.gpu
def test_launch_log_names_the_decoder_per_alphabet():
    """decode_cdf launches repitch_kernel and ac_decode_kernel for L <= 256, as before, and repitch_kernel and
    ac_decode_wide_kernel above"""
    from l3c_pytorch_b200 import engine as E, torchac
    rng = np.random.default_rng(4)
    for L, dec in [(25, 'ac_decode_kernel'), (100, 'ac_decode_kernel'), (256, 'ac_decode_kernel'),
                   (257, 'ac_decode_wide_kernel'), (32768, 'ac_decode_wide_kernel')]:
        s = make_stream(rng, 'peaked', 50, L)
        t = _t_cdf(s.cdf)
        data = torchac.encode_cdf(t, torch.from_numpy(s.sym))
        E.launch_log(reset=True)
        assert (torchac.decode_cdf(t, data).numpy() == s.sym).all()
        kernels, total = E.launch_log(reset=True)
        assert kernels == {'repitch_kernel': 1, dec: 1}, (L, kernels)
