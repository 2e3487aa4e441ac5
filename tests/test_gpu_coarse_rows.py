"""Coarse CDF rows of the RGB scale (L = 256, f16 mode; DESIGN §4.3 / §4.4): l3c_dmll_build_coarse writes each
sub-pixel's mixture parameters and every 8th CDF entry, and l3c_ac_decode_streams_coarse evaluates the 7 entries of
the bracket it lands in on demand.

* The coarse entries equal dmll_table_kernel's full rows at indices 8 i, on peaked (trained-like), broad
  (random-init-like) and mixed parameters, for all three channels with their R / G coupling.
* Streams encoded by the oracle on the full rows decode from the coarse records to the oracle's symbols, and the
  saved coder state after every launch equals the oracle's at that symbol, under chunk sizes from 1 symbol to 3 x
  the plane, on ragged stream lengths and on junk and truncated input, for every streams-per-CTA variant.  With one
  symbol per launch the state after every symbol is compared: both bounds of every decoded interval -- coarse or
  evaluated on demand -- are the full row's.
* l3c_decode_rgb_pipelined with coarse records gives the full-row path's planes, symbol for symbol."""
import numpy as np
import pytest
import torch

from oracle import ac
from tests.test_gpu_coder_launches import _rgb_case, _rgb_descs, _rgb_pipelined

H, W = 12, 20
HW = H * W
C, K, L = 3, 10, 256
NS = np.array([HW, HW - 37, 9, 1], np.int64)     # stream lengths: ragged, compact planes of HW
N = len(NS)
KINDS = ('peaked', 'broad', 'mixed')


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def _params(kind, rng, N=N, H=H, W=W):
    """l [N, H, W, 4 C K] and symbols [N, C, HW]: 'peaked' = one dominant component with log-scales down to and below
    the -7 clamp (most entries saturated); 'broad' = random-init-like logits, means around the middle of [0, 255] and
    log-scales around 2-4 (few entries saturated); 'mixed' = either, per pixel."""
    HW = H * W
    shp = (N, HW, C, K)
    dom = rng.integers(0, K, (N, HW, C))
    logit = rng.normal(0, 1, shp)
    mean = rng.uniform(-60, 315, shp)
    logs = rng.uniform(-9, 1.5, shp)
    np.put_along_axis(logit, dom[..., None], rng.uniform(4, 12, dom.shape)[..., None], axis=3)
    np.put_along_axis(logs, dom[..., None], rng.uniform(-9.5, -2, dom.shape)[..., None], axis=3)
    b_logit, b_mean, b_logs = rng.normal(0, 0.5, shp), rng.normal(128, 40, shp), rng.uniform(2, 4, shp)
    if kind == 'broad':
        logit, mean, logs = b_logit, b_mean, b_logs
    elif kind == 'mixed':
        pick = (rng.random((N, HW, 1, 1)) < 0.5)
        logit, mean, logs = (np.where(pick, b, a) for a, b in ((logit, b_logit), (mean, b_mean), (logs, b_logs)))
    coef = rng.normal(0, 2, shp)
    l = np.stack([logit, mean, logs, coef], axis=2).reshape(N, H, W, 4 * C * K).astype(np.float32)
    mu = np.take_along_axis(mean, dom[..., None], axis=3)[..., 0]
    sym = np.zeros((N, C, HW), np.int64)
    for c in range(C):
        m = mu[:, :, c] + (sym[:, 0] * _sigmoid(coef[:, :, 0, 0]) if c > 0 else 0)
        s = np.clip(np.rint(m + rng.normal(0, 0.4, m.shape)), 0, 255)
        u = rng.random(m.shape)
        s = np.where(u < 0.3, rng.integers(0, 256, m.shape), s)
        s = np.where((u >= 0.3) & (u < 0.33), 0, s)
        sym[:, c] = np.where((u >= 0.33) & (u < 0.36), 255, s)
    return l, sym.astype(np.uint8)


CASES = {}


def _case(kind):
    """full rows and coarse records of all three channels, built from the true symbols, and one oracle stream per
    (image, channel) on the full rows"""
    if kind in CASES:
        return CASES[kind]
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    dev = torch.device('cuda')
    rng = np.random.default_rng(7 + KINDS.index(kind))
    l, sym = _params(kind, rng)
    l_dev = torch.from_numpy(l).to(dev)
    sym_dev = torch.from_numpy(sym.reshape(N, C, H, W)).to(dev)
    tg = DiscretizedMixLogisticLoss(True, 0, 255, L).targets(dev)
    table = torch.zeros(N * C * HW * L, dtype=torch.int16, device=dev)
    rec = torch.zeros(N * C * HW * E.COARSE_PITCH, dtype=torch.int16, device=dev)
    for c in range(C):
        E.dmll_build_table(l_dev, sym_dev, tg, C, K, L, True, c, table)
        E.dmll_build_coarse(l_dev, sym_dev, tg, K, L, c, rec)
    rows = table.cpu().numpy().view(np.uint16).reshape(N, C, HW, L)
    recs = rec.cpu().numpy().view(np.uint16).reshape(N, C, HW, E.COARSE_PITCH)
    streams = [[ac.encode(np.concatenate([rows[n, c, :NS[n]], np.zeros((NS[n], 1), np.uint16)], 1),
                          sym[n, c, :NS[n]]) for c in range(C)] for n in range(N)]
    CASES[kind] = dict(l=l_dev, sym=sym, tg=tg, rows=rows, recs=recs, rec=rec, streams=streams)
    return CASES[kind]


@pytest.mark.gpu
@pytest.mark.parametrize('kind', KINDS)
def test_coarse_entries_equal_full_rows(kind):
    cs = _case(kind)
    rows, recs = cs['rows'], cs['recs']
    got = recs[..., 64:96]
    want = rows[..., ::8]
    bad = np.argwhere(got != want)
    assert bad.size == 0, '%s: %d coarse entries differ from the full row, first at %s' % (kind, len(bad), bad[0])
    assert (recs[..., 60:64] == 0).all()                   # the two padding words
    # not every entry is saturated: some rows need the transcendentals
    frac = np.mean(np.diff(rows.astype(np.int64), axis=-1) > 1)
    print('%s: %.1f %% of the entry steps are wider than one count' % (kind, 100 * frac))


def _schedules(n_max):
    out = []
    for chunk in (1, 5, 8, 13, HW, 3 * HW):
        out.append((chunk, [(f, chunk) for f in range(0, n_max, chunk)]))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('spc', [1, 2, 4])
@pytest.mark.parametrize('kind', KINDS)
def test_coarse_decode_matches_oracle(kind, spc):
    from l3c_pytorch_b200 import _lib, engine as E
    dev = torch.device('cuda')
    cs = _case(kind)
    rng = np.random.default_rng(99)
    # one stream per (image, channel), then junk and truncated copies of some of them
    items = [(n, c, cs['streams'][n][c]) for n in range(N) for c in range(C)]
    junk = [(0, 0, rng.integers(0, 256, len(cs['streams'][0][0]), np.uint8).tobytes()),
            (1, 2, rng.integers(0, 256, 40, np.uint8).tobytes())]
    trunc = [(0, 1, cs['streams'][0][1][:len(cs['streams'][0][1]) // 2]), (1, 0, cs['streams'][1][0][:3]),
             (0, 2, b'')]
    items += junk + trunc
    n_all = len(items)
    n_sym = np.array([NS[n] for n, _, _ in items], np.int64)
    want_sym, trace = [], []
    for i, (n, c, data) in enumerate(items):
        full = np.concatenate([cs['rows'][n, c, :NS[n]], np.zeros((NS[n], 1), np.uint16)], 1)
        s, tr = ac.decode_trace(full, data)
        if i < N * C:
            assert (s == cs['sym'][n, c, :NS[n]]).all(), (kind, n, c)
        want_sym.append(s.astype(np.uint8))
        trace.append(tr)
    # streams packed at odd offsets, outputs at +0..+3 with guard bytes
    offs = np.cumsum([0] + [len(d) + 3 for _, _, d in items])[:-1] + 1
    blob_h = np.zeros(int(offs[-1] + len(items[-1][2]) + 16), np.uint8)
    for i, (_, _, d) in enumerate(items):
        blob_h[offs[i]:offs[i] + len(d)] = np.frombuffer(d, np.uint8)
    blob = torch.from_numpy(blob_h).to(dev)
    slot = (n_sym + 8 + 3) // 4 * 4 + 4
    out0 = np.concatenate([[0], np.cumsum(slot)[:-1]]) + np.arange(n_all) % 4
    out = torch.empty(int(slot.sum()), dtype=torch.uint8, device=dev)
    state = torch.empty(4 * n_all, dtype=torch.int32, device=dev)
    dd = np.zeros(n_all, dtype=_lib.DEC_STREAM_DTYPE)
    plane = np.array([n * C + c for n, c, _ in items], np.int64)
    dd['table'] = cs['rec'].data_ptr() + 2 * E.COARSE_PITCH * HW * plane
    dd['row_pitch'] = E.COARSE_PITCH
    dd['in'] = blob.data_ptr() + offs
    dd['in_len'] = [len(d) for _, _, d in items]
    dd['n_sym'] = n_sym
    dd['sym_out'] = out.data_ptr() + out0
    dd['state'] = state.data_ptr() + 16 * np.arange(n_all)
    desc_dev = E._desc_to_device(dd, dev)
    with E.decoder_streams_per_cta(spc):
        for chunk, sched in _schedules(int(n_sym.max())):
            out.fill_(0xA5)
            state.fill_(-1)
            for first, count in sched:
                E.ac_decode_streams_coarse(dd, dev, cs['tg'], first, count, desc_dev=desc_dev, n=n_all)
                st = state.cpu().numpy().view(np.uint32).reshape(n_all, 4)
                for i in range(n_all):
                    if first >= n_sym[i]:
                        continue
                    last = min(first + count, int(n_sym[i]))
                    want = trace[i][min(last, int(n_sym[i]) - 1)]
                    assert (st[i] == want).all(), ('%s, SPC %d, chunk %d, launch (%d, %d), stream %d: saved state %s, '
                                                   'oracle %s' % (kind, spc, chunk, first, count, i, st[i].tolist(),
                                                                  want.tolist()))
            got = out.cpu().numpy()
            for i in range(n_all):
                o = int(out0[i])
                seg, guard = got[o:o + int(n_sym[i])], got[o + int(n_sym[i]):o + int(n_sym[i]) + 8]
                bad = np.flatnonzero(seg != want_sym[i])
                assert bad.size == 0, ('%s, SPC %d, chunk %d, stream %d: %d wrong symbols, first at %d'
                                       % (kind, spc, chunk, i, bad.size, bad[0]))
                assert (guard == 0xA5).all(), (kind, spc, chunk, 'write past the end of stream', i)


@pytest.mark.gpu
@pytest.mark.parametrize('spc', [1, 4])
def test_pipelined_coarse_decode_matches_full_rows(spc):
    """l3c_decode_rgb_pipelined on coarse records (ragged stream lengths HW, HW-37, 9, 1; chunks of 1, 13, HW and
    3 HW pixels) against the same call on full rows."""
    from l3c_pytorch_b200 import engine as E
    dev = torch.device('cuda')
    cs = _rgb_case(dev)
    n_px = cs.N * cs.C * cs.H * cs.W
    bld = [torch.cuda.Stream(device=dev) for _ in range(3)]
    dec = [torch.cuda.Stream(device=dev) for _ in range(3)]
    with E.decoder_streams_per_cta(spc):
        for chunk in (1, 13, cs.H * cs.W, 3 * cs.H * cs.W):
            full = _rgb_pipelined(cs, dev, chunk, bld, dec)
            S = torch.zeros(cs.N, cs.C, cs.H, cs.W, dtype=torch.uint8, device=dev)
            rec = torch.zeros(n_px * E.COARSE_PITCH, dtype=torch.int16, device=dev)
            state = torch.full((cs.N * cs.C * 4,), -1, dtype=torch.int32, device=dev)
            d = _rgb_descs(cs, dev, S, rec, state)
            plane = np.arange(cs.N)[:, None] * cs.C + np.arange(cs.C)[None]
            d['table'] = rec.data_ptr() + 2 * E.COARSE_PITCH * cs.H * cs.W * plane
            d['row_pitch'] = E.COARSE_PITCH
            descs = [E._desc_to_device(np.ascontiguousarray(d[:, c]), dev) for c in range(cs.C)]
            E.decode_rgb_pipelined(cs.l, S, cs.tg, cs.K, cs.L, rec, descs, chunk, torch.cuda.current_stream(), bld,
                                   dec, coarse=True)
            torch.cuda.synchronize()
            got = S.cpu().numpy().reshape(cs.N, cs.C, -1)
            for nn in range(cs.N):
                k = int(cs.ns[nn])
                assert (got[nn, :, :k] == cs.sym[nn, :, :k]).all(), (spc, chunk, nn)
                bad = np.flatnonzero((got[nn, :, :k] != full[nn, :, :k]).reshape(-1))
                assert bad.size == 0, ('SPC %d, chunk %d, image %d: %d sub-pixels differ from the full-row path'
                                       % (spc, chunk, nn, bad.size))
