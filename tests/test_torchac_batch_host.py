"""Host: the planner of the batched torchac calls (l3c_pytorch_b200.torchac.plan_decode / plan_encode) and the
argument checks that run before anything reaches the GPU."""
import numpy as np
import pytest
import torch

from l3c_pytorch_b200 import torchac as T


def _cases():
    rng = np.random.default_rng(5)
    alphabets = np.array([2, 25, 32, 33, 255, 256, 257, 1000, 4097, 32768])
    for k in range(40):
        m = int(rng.integers(1, 60))
        n = rng.integers(1, 6000, m)
        n[rng.random(m) < 0.2] = 1
        L = rng.choice(alphabets, m)
        cap = int(rng.choice([70_000, 300_000, 2 << 20, 64 << 20, 1 << 30]))
        yield n, L, cap


def test_plan_decode_covers_every_symbol_once_in_order_within_the_cap():
    """Every symbol of every stream is decoded exactly once, the chunks of a stream are in order and contiguous,
    the rows of every chunk fit the cap, and the streams of a chunk are sorted by L (one decoder launch per
    alphabet reads a contiguous run of descriptors)"""
    for n, L, cap in _cases():
        plan = T.plan_decode(n, L, cap)
        pos = np.zeros(n.size, np.int64)
        for act, first, count in plan:
            assert count >= 1 and act.size >= 1
            assert (pos[act] == first).all(), (first, count)
            assert (n[act] > first).all()
            rows = np.minimum(n[act] - first, count) * T.row_bytes(L[act])
            assert rows.sum() <= cap, (rows.sum(), cap)
            assert (np.diff(L[act]) >= 0).all()
            pos[act] = np.minimum(n[act], first + count)
        assert (pos == n).all()


def test_plan_decode_splits_streams_that_exceed_the_cap_together():
    """Eight L = 32768 streams whose rows for MIN_CHUNK_SYMBOLS symbols do not fit together are decoded in groups
    of streams, one group after the other; with a large cap they share every chunk"""
    n = np.full(8, 1000)
    L = np.full(8, 32768)
    row = int(T.row_bytes(32768))
    cap = 2 * T.MIN_CHUNK_SYMBOLS * row
    plan = T.plan_decode(n, L, cap)
    groups = []
    for act, first, _ in plan:
        if first == 0:
            groups.append(set(act.tolist()))
    assert len(groups) == 4 and all(len(g) == 2 for g in groups)
    assert set().union(*groups) == set(range(8))
    one = T.plan_decode(n, L, 1 << 30)
    assert len(one) == 1 and one[0][0].size == 8 and one[0][2] == 1000


def test_plan_decode_chunks_short_and_long_streams():
    """Streams that end early leave the later chunks, whose counts then grow; a cap smaller than one row is an
    error"""
    n = np.array([10, 5000, 3, 5000])
    L = np.array([25, 300, 25, 1024])
    cap = 200_000
    plan = T.plan_decode(n, L, cap)
    assert len(plan) >= 3
    assert set(plan[0][0].tolist()) == {0, 1, 2, 3}
    assert set(plan[-1][0].tolist()) <= {1, 3}
    with pytest.raises(ValueError, match='one row'):
        T.plan_decode([5], [32768], 60_000)
    assert T.plan_decode([], [], cap) == []


def test_plan_encode_groups_in_order_under_the_cap():
    rng = np.random.default_rng(6)
    for _ in range(30):
        n = rng.integers(1, 200_000, int(rng.integers(1, 50)))
        cap = int(rng.choice([100_000, 1 << 20, 1 << 30]))
        groups = T.plan_encode(n, cap)
        assert np.concatenate(groups).tolist() == list(range(n.size))
        for g in groups:
            need = int(T.enc_scratch_bytes(n[g]).sum())
            assert need <= cap or g.size == 1
    assert T.enc_scratch_bytes(1000) == 4000 + ((17000 + 7) // 8 + 64 + 3) // 4 * 4


def _cdf(n, Lp):
    return torch.zeros(1, 1, n, Lp, dtype=torch.int16)


def test_argument_errors_name_the_stream_before_any_work():
    assert T.encode_cdf_batch([], []) == []
    assert T.decode_cdf_batch([], []) == []
    assert T.encode_logistic_mixture_batch([], [], [], [], []) == []
    assert T.decode_logistic_mixture_batch([], [], [], [], []) == []
    ok = _cdf(4, 26)
    s = torch.zeros(4, dtype=torch.int16)
    with pytest.raises(RuntimeError, match='stream 1: Invalid size for cdf! Expected 1HWLp'):
        T.encode_cdf_batch([ok, ok[0]], [s, s])
    with pytest.raises(RuntimeError, match='stream 0: cdf must be int16'):
        T.decode_cdf_batch([ok.int(), ok], [b'', b''])
    with pytest.raises(RuntimeError, match=r'stream 2: Lp=32770 not in \[2,32769\]'):
        T.encode_cdf_batch([ok, ok, _cdf(1, 32770)], [s, s, s[:1]])
    with pytest.raises(RuntimeError, match=r'stream 1: Lp=1 not in \[2,32769\]'):
        T.decode_cdf_batch([ok, _cdf(3, 1)], [b'', b''])
    with pytest.raises(RuntimeError, match='stream 0: n_sym=0'):
        T.decode_cdf_batch([_cdf(0, 26)], [b''])
    with pytest.raises(ValueError, match='one entry per stream'):
        T.encode_cdf_batch([ok, ok], [s])
