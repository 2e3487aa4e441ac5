"""GPU: the batched torchac calls (l3c_pytorch_b200.torchac.*_batch) against the CPU oracle (oracle.ac) and the
one-stream functions: shuffled streams of every kind and alphabet in one call, CPU and CUDA inputs, corrupt input,
launch counts, chunked decodes under a small scratch cap, mixtures, errors and stream ordering."""
import numpy as np
import pytest
import torch

from oracle import ac
from tests.test_gpu_coder import _mixture_case
from tests.test_gpu_coder_wide import _stream, _t_cdf

ALPHABETS = (2, 3, 25, 32, 33, 100, 255, 256, 257, 300, 1024, 4097, 32768)
KINDS = ('flat', 'peaked', 'tail', 'straddle', 'uniform', 'mix')
LENGTHS = (1, 2, 9, 64, 700, 5003)
TABLE_BYTES = 64 << 20            # per table


def _mixed_streams(seed):
    """every kind at every alphabet, lengths 1 .. 5003 (tables capped at TABLE_BYTES), shuffled"""
    rng = np.random.default_rng(seed)
    ss = []
    for i, L in enumerate(ALPHABETS):
        for k, kind in enumerate(KINDS):
            n = min(LENGTHS[(i + k) % len(LENGTHS)], TABLE_BYTES // (2 * (L + 1)))
            s = _stream(rng, kind, n, L)
            s.L = L
            s.want = ac.encode(s.cdf, s.sym)
            ss.append(s)
    return [ss[i] for i in rng.permutation(len(ss))]


_CASE = {}


def _case():
    if 'ss' not in _CASE:
        _CASE['ss'] = _mixed_streams(11)
    return _CASE['ss']


def _inputs(ss, device):
    cdfs = [_t_cdf(s.cdf).to(device) for s in ss]
    syms = [torch.from_numpy(s.sym).to(device) for s in ss]
    return cdfs, syms


def _corrupt(ss, datas, rng):
    """junk, truncated and empty strings for some of the longer streams"""
    strings = list(datas)
    long_ = [i for i, s in enumerate(ss) if s.n >= 9]
    for j, i in enumerate(long_[:12]):
        d = datas[i]
        strings[i] = [bytes(rng.integers(0, 256, len(d)).astype(np.uint8)), d[:len(d) // 2], d[:-1], b''][j % 4]
    return strings


@pytest.mark.gpu
@pytest.mark.parametrize('device', ['cpu', 'cuda'])
def test_mixed_tables_match_oracle_and_one_stream_calls(device):
    """One call codes every kind of stream at L = 2 .. 32768 (all three decoder classes), lengths 1 .. 5003: the
    bytes equal the oracle's and encode_cdf's, the decode returns the symbols on the tables' device, and junk,
    truncated and empty strings in the same call decode to the oracle's symbols"""
    from l3c_pytorch_b200 import torchac
    ss = _case()
    cdfs, syms = _inputs(ss, device)
    datas = torchac.encode_cdf_batch(cdfs, syms)
    assert len(datas) == len(ss)
    for i, s in enumerate(ss):
        assert datas[i] == s.want, (i, s.kind, s.L, s.n)
    if device == 'cpu':
        for i, s in enumerate(ss):
            assert torchac.encode_cdf(cdfs[i], syms[i]) == datas[i], (i, s.kind, s.L, s.n)
    back = torchac.decode_cdf_batch(cdfs, datas)
    for i, s in enumerate(ss):
        assert back[i].device.type == device and back[i].dtype == torch.int16 and back[i].shape == (s.n,)
        assert (back[i].cpu().numpy() == s.sym).all(), (i, s.kind, s.L, s.n)
    strings = _corrupt(ss, datas, np.random.default_rng(12))
    got = torchac.decode_cdf_batch(cdfs, strings)
    for i, s in enumerate(ss):
        want = ac.decode(s.cdf, strings[i])
        assert (got[i].cpu().numpy() == want).all(), (i, s.kind, s.L, s.n, len(strings[i]), len(datas[i]))
        if device == 'cpu' and strings[i] != datas[i]:
            assert torch.equal(got[i], torchac.decode_cdf(cdfs[i], strings[i]))


def _decoder_name(L):
    return 'ac_decode_wide_kernel' if L > 256 else 'ac_decode_kernel'


def _expected_decode_launches(n, L, cap=None):
    from l3c_pytorch_b200 import torchac
    plan = torchac.plan_decode(n, L, cap)
    want = {'batch_rows_kernel': len(plan)}
    for act, _, _ in plan:
        for a in set(L[act].tolist()):
            want[_decoder_name(a)] = want.get(_decoder_name(a), 0) + 1
    return plan, want


@pytest.mark.gpu
def test_launch_counts():
    """encode: one interval launch, one encoder launch and one pack, whatever the number of streams; decode: one
    row launch per chunk and one decoder launch per alphabet in it"""
    from l3c_pytorch_b200 import engine as E, torchac
    ss = _case()
    cdfs, syms = _inputs(ss, 'cuda')
    n = np.array([s.n for s in ss])
    L = np.array([s.L for s in ss])
    E.launch_log(reset=True)
    datas = torchac.encode_cdf_batch(cdfs, syms)
    kernels, _ = E.launch_log(reset=True)
    assert kernels == {'batch_intervals_kernel': 1, 'ac_encode_kernel': 1, 'pack_streams_kernel': 1}, kernels
    torchac.decode_cdf_batch(cdfs, datas)
    kernels, _ = E.launch_log(reset=True)
    plan, want = _expected_decode_launches(n, L)
    assert len(plan) == 1
    assert kernels == want, (kernels, want)
    # many short streams: still one launch of each
    rng = np.random.default_rng(13)
    short = [_stream(rng, 'peaked', int(rng.integers(1, 4)), 25) for _ in range(3000)]
    cdfs = [_t_cdf(s.cdf) for s in short]
    datas = torchac.encode_cdf_batch(cdfs, [torch.from_numpy(s.sym) for s in short])
    kernels, _ = E.launch_log(reset=True)
    assert kernels == {'batch_intervals_kernel': 1, 'ac_encode_kernel': 1, 'pack_streams_kernel': 1}, kernels
    back = torchac.decode_cdf_batch(cdfs, datas)
    kernels, _ = E.launch_log(reset=True)
    assert kernels == {'batch_rows_kernel': 1, 'ac_decode_kernel': 1}, kernels
    for s, d, b in zip(short, datas, back):
        assert d == ac.encode(s.cdf, s.sym) and (b.numpy() == s.sym).all()


@pytest.mark.gpu
def test_a_hundred_thousand_short_streams():
    """10^5 streams of 1 to 3 symbols in one call (more than one grid dimension's 65535 blocks): bytes equal the
    oracle's, the decode returns the symbols"""
    from l3c_pytorch_b200 import torchac
    rng = np.random.default_rng(14)
    m = 100_000
    n = rng.integers(1, 4, m)
    L = np.where(rng.random(m) < 0.5, 25, 300)
    cdfs, syms, want = [], [], []
    base = {a: _stream(rng, 'flat', 3, a) for a in (25, 300)}
    for i in range(m):
        b = base[int(L[i])]
        k = int(n[i])
        sym = rng.integers(0, int(L[i]), k).astype(np.int16)
        cdfs.append(_t_cdf(b.cdf[:k]))
        syms.append(torch.from_numpy(sym))
        want.append((b.cdf[:k], sym))
    datas = torchac.encode_cdf_batch(cdfs, syms)
    idx = rng.choice(m, 2000, replace=False)
    for i in idx:
        assert datas[i] == ac.encode(*want[i]), i
    back = torchac.decode_cdf_batch(cdfs, datas)
    for i in range(m):
        assert (back[i].numpy() == want[i][1]).all(), i


@pytest.mark.gpu
def test_chunked_decode_under_a_small_cap(monkeypatch):
    """With the scratch cap small enough for at least three chunks (a wide stream among them) the results are
    identical, the launches follow the plan, and the torch allocator's peak during the call stays under the cap plus
    a fixed overhead"""
    from l3c_pytorch_b200 import engine as E, torchac
    rng = np.random.default_rng(15)
    ss = [_stream(rng, k, n, L) for (k, n, L) in [('peaked', 1000, 32768), ('mix', 5003, 256), ('flat', 3000, 1024),
                                                   ('tail', 700, 25), ('straddle', 64, 300), ('uniform', 1, 2),
                                                   ('peaked', 2500, 32768)]]
    for s, L in zip(ss, (32768, 256, 1024, 25, 300, 2, 32768)):
        s.L = L
    cdfs, syms = _inputs(ss, 'cuda')
    datas = torchac.encode_cdf_batch(cdfs, syms)
    whole = torchac.decode_cdf_batch(cdfs, datas)
    cap = 1 << 20
    monkeypatch.setattr(torchac, 'BATCH_SCRATCH_BYTES', cap)
    n = np.array([s.n for s in ss])
    L = np.array([s.L for s in ss])
    plan, want = _expected_decode_launches(n, L, cap)
    assert len(plan) >= 3 and sum(1 for act, _, _ in plan if (L[act] == 32768).any()) >= 3
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    E.launch_log(reset=True)
    got = torchac.decode_cdf_batch(cdfs, datas)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    kernels, _ = E.launch_log(reset=True)
    assert kernels == want
    overhead = 4 * int(n.sum()) + sum(len(d) for d in datas) + (1 << 20)
    assert peak <= cap + overhead, (peak, cap, overhead)
    for i, s in enumerate(ss):
        assert torch.equal(got[i], whole[i]) and (got[i].cpu().numpy() == s.sym).all(), i
    # encode groups under the same cap: same bytes
    assert torchac.encode_cdf_batch(cdfs, syms) == datas


@pytest.mark.gpu
def test_mixtures_of_every_k_and_lp_in_one_call():
    """K in {1, 3, 10} and Lp in {3, 26, 257, 1025} in one call: the bytes equal encode_logistic_mixture per stream,
    the decode returns the symbols (CUDA tensors), with CPU and CUDA symbols"""
    from l3c_pytorch_b200 import torchac
    rng = np.random.default_rng(16)
    cases = []
    for K in (1, 3, 10):
        for Lp in (3, 26, 257, 1025):
            H, W = [(1, 1), (5, 7), (16, 24), (9, 40)][int(rng.integers(0, 4))]
            L = Lp - 1
            t, mu, ls, pi = _mixture_case(rng, K, H, W, L, 0., float(L - 1) if L > 1 else 1.)
            sym = rng.integers(0, L, size=H * W).astype(np.int16)
            cases.append(([x.cuda() for x in (t, mu, ls, pi)], sym))
    order = rng.permutation(len(cases))
    cases = [cases[i] for i in order]
    args = [list(x) for x in zip(*[c[0] for c in cases])]
    for where in ('cpu', 'cuda'):
        syms = [torch.from_numpy(c[1]).to(where) for c in cases]
        datas = torchac.encode_logistic_mixture_batch(*args, syms)
        for i, (p, sym) in enumerate(cases):
            assert datas[i] == torchac.encode_logistic_mixture(*p, torch.from_numpy(sym)), i
    back = torchac.decode_logistic_mixture_batch(*args, datas)
    for i, (p, sym) in enumerate(cases):
        assert back[i].is_cuda and (back[i].cpu().numpy() == sym).all(), i


@pytest.mark.gpu
def test_wide_mixture_decodes_within_the_scratch_cap():
    """L = 32768, 192 x 192 symbols: its full rows would take 2.4 GB; the decode stays under the cap plus a fixed
    overhead and returns the symbols; the bytes equal encode_logistic_mixture's"""
    from l3c_pytorch_b200 import torchac
    rng = np.random.default_rng(17)
    L, H, W = 32768, 192, 192
    assert H * W * 2 * L > 2 << 30
    p = [x.cuda() for x in _mixture_case(rng, 1, H, W, L, 0., float(L - 1))]
    sym = rng.integers(0, L, size=H * W).astype(np.int16)
    data = torchac.encode_logistic_mixture_batch(*[[x] for x in p], [torch.from_numpy(sym)])[0]
    assert data == torchac.encode_logistic_mixture(*p, torch.from_numpy(sym))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    back = torchac.decode_logistic_mixture_batch(*[[x] for x in p], [data])[0]
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak <= torchac.BATCH_SCRATCH_BYTES + (16 << 20), peak
    assert (back.cpu().numpy() == sym).all()


@pytest.mark.gpu
def test_errors():
    from l3c_pytorch_b200 import torchac
    rng = np.random.default_rng(18)
    ss = [_stream(rng, 'flat', 6, L) for L in (25, 300, 25)]
    cdfs = [_t_cdf(s.cdf) for s in ss]
    syms = [torch.from_numpy(s.sym) for s in ss]
    for f in (torchac.encode_cdf_batch, torchac.decode_cdf_batch, torchac.encode_logistic_mixture_batch,
              torchac.decode_logistic_mixture_batch):
        assert f(*([[]] * (2 if 'cdf' in f.__name__ else 5))) == []
    with pytest.raises(ValueError):
        torchac.encode_cdf_batch([cdfs[0], cdfs[1].cuda(), cdfs[2]], syms)
    with pytest.raises(ValueError):
        torchac.encode_cdf_batch(cdfs, [syms[0], syms[1].cuda(), syms[2]])
    with pytest.raises(ValueError):
        torchac.encode_cdf_batch(cdfs, [s.cuda() for s in syms])
    with pytest.raises(ValueError):
        torchac.decode_cdf_batch([cdfs[0].cuda(), cdfs[1]], [b'', b''])
    with pytest.raises(RuntimeError, match='stream 1: sym has 5 entries'):
        torchac.encode_cdf_batch(cdfs, [syms[0], syms[1][:5], syms[2]])
    for where in ('cpu', 'cuda'):
        for j, pos, bad in ((2, 3, 25), (0, 0, -1), (1, 5, 300)):          # 25 and 300: Lp - 1
            ss_sym = [s.clone() for s in syms]
            ss_sym[j][pos] = bad
            with pytest.raises(RuntimeError, match='stream %d: symbol %d at position %d outside' % (j, bad, pos)):
                torchac.encode_cdf_batch([c.to(where) for c in cdfs], [s.to(where) for s in ss_sym])
    t, mu, ls, pi = _mixture_case(rng, 2, 3, 4, 25, 0., 24.)
    dev = [x.cuda() for x in (t, mu, ls, pi)]
    sym = torch.zeros(12, dtype=torch.int16)
    with pytest.raises(ValueError):
        torchac.encode_logistic_mixture_batch(*[[x, y] for x, y in zip(dev, [t, mu, ls, pi])], [sym, sym])
    with pytest.raises(RuntimeError, match='stream 1: Invalid size for means'):
        torchac.encode_logistic_mixture_batch(*[[x, x[0] if k == 1 else x] for k, x in enumerate(dev)], [sym, sym])
    with pytest.raises(RuntimeError, match=r'stream 0: Lp=32770 not in \[2,32769\]'):
        torchac.decode_logistic_mixture_batch([torch.zeros(32770).cuda()], *[[x] for x in dev[1:]], [b''])
    bad = sym.clone()
    bad[7] = 25
    with pytest.raises(RuntimeError, match='stream 1: symbol 25 at position 7 outside'):
        torchac.encode_logistic_mixture_batch(*[[x, x] for x in dev], [sym.cuda(), bad.cuda()])


@pytest.mark.gpu
def test_call_on_a_side_stream():
    """A call made under torch.cuda.stream(side) on inputs produced on that stream is correct"""
    from l3c_pytorch_b200 import torchac
    ss = _case()
    rng = np.random.default_rng(19)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        cdfs = [(_t_cdf(s.cdf).cuda(non_blocking=True) + 0) for s in ss]
        syms = [torch.from_numpy(s.sym).cuda(non_blocking=True) * 1 for s in ss]
        datas = torchac.encode_cdf_batch(cdfs, syms)
        back = torchac.decode_cdf_batch(cdfs, datas)
        t, mu, ls, pi = _mixture_case(rng, 3, 8, 8, 256, 0., 255.)
        p = [x.cuda(non_blocking=True) * 1 for x in (t, mu, ls, pi)]
        sym = rng.integers(0, 256, 64).astype(np.int16)
        d = torchac.encode_logistic_mixture_batch(*[[x] for x in p], [torch.from_numpy(sym).cuda() + 0])
        bm = torchac.decode_logistic_mixture_batch(*[[x] for x in p], d)[0]
        bm_host = bm.cpu()
    side.synchronize()
    assert all(d0 == s.want for d0, s in zip(datas, ss))
    assert all((b.cpu().numpy() == s.sym).all() for b, s in zip(back, ss))
    assert (bm_host.numpy() == sym).all()
    assert d[0] == torchac.encode_logistic_mixture(*p, torch.from_numpy(sym))
