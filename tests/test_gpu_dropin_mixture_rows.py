"""The torchac drop-in's logistic-mixture CDFs, entry by entry against the float64 restatement, at every alphabet.

The drop-in (torchac.encode/decode_logistic_mixture and their _batch forms) builds its CDF integers in four kernels:
plane_intervals_kernel and plane_table_kernel for one stream (capi.cu), batch_intervals_kernel and batch_rows_kernel
for many (torchac_batch.cu).  They take log-scales unclamped and weights as given, as the reference's torchac does,
so the parameters reach further than the codec's: log-scales from -30 to +20, weights that do not sum to one.

* Restatement: test_gpu_cdf_rows.restate on the kernels' fp32 parameters, with inv_s recomputed from the log-scale
  (u_rel = U_REL_EXPF), scale 65536 - (Lp - 1) and the reference's rounding -- lrintf to a 64-bit integer, + l,
  the low 16 bits.  Where |V| >= 2^31 (weights summing to thousands) only that rounding gives the reference's entry.
* Parameter grid: Lp in LPS (every decoder pitch class, pitches one either side of a multiple of 8), K in {1, 3, 10,
  17}, evenly spaced and log-spaced targets and means exactly on targets, and the families in FAMILIES.  Symbols
  hit 0, Lp - 2 (the interval that ends at 65536) and random entries.
* Rows (l3c_batch_rows): every entry l < L is one of the restatement's values, entries L .. pitch - 1 are 0, and
  nothing outside the rows is written; also for one launch of 300 short ragged streams among long ones, with first
  != 0 and counts that end mid-stream.
* Intervals (l3c_batch_intervals, encode_logistic_mixture): the restated rows' intervals; the bytes are those of
  oracle.ac.encode on the kernel's rows; an out-of-range symbol reports the stream's first bad position.
* decode_logistic_mixture returns the symbols of oracle streams coded on those rows.  That is the only view the
  suite has of plane_table_kernel's integers: a decode checks an entry only where a coded value lies next to it.
* Codability: where the parameters are finite, expf(-log_scale) is finite, pi >= 0 and sum(pi) <= 1 + 2^-20, every
  row is strictly increasing with its last entry <= 65535 (in_domain).  Outside, per-entry agreement is all that is
  asserted: garbage in gives the reference's garbage out.
* float64, float16 and non-contiguous inputs code like the float32 contiguous call on the same values.
* CPU self-tests: a float32 model of the kernels passes the checks, and four planted mis-restatements fail them."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ac
from tests.test_gpu_cdf_rows import NEG_LOG2E, U_REL_EXPF, check_rows, emulate, f2i_rn, f2ll_rn, restate

LPS = [2, 3, 26, 33, 256, 257, 258, 264, 265, 1025, 4097, 32769]
KS = [1, 3, 10, 17]
TARGETS = ('even', 'log', 'on')
FAMILIES = ('trained', 'wide', 'logscale', 'far', 'pi_underflow', 'sum_pi', 'nonfinite', 'unnorm', 'unnorm_big')
# restatement work per call, in [row, entry, component] elements: tens of rows at L = 32768
CHUNK_ELEMS = 1 << 21
GUARD = 4096                        # canary bytes on each side of the rows
CANARY = 0xA5
TWO31 = 2.0 ** 31


def n_rows(Lp):
    L = Lp - 1
    return 48 if L <= 32 else 24 if L <= 256 else 12 if L <= 1024 else 6 if L <= 4096 else 3


# ---------------------------------------------------------------------------------------------------------------------
# streams
# ---------------------------------------------------------------------------------------------------------------------
def targets(kind, Lp):
    """float32 [Lp] strictly increasing bin edges: evenly spaced over [-1, 1] (half a bin beyond), or log-spaced
    (bins growing by e^4 from the first to the last)"""
    L = Lp - 1
    if kind == 'log':
        g = 4.0
        t = -1.0 + 2.0 * np.expm1(g * np.arange(Lp) / max(L, 1)) / np.expm1(g)
    else:
        bw = 2.0 / max(L - 1, 1)
        t = np.linspace(-1 - bw / 2, 1 + bw / 2, Lp)
    t = t.astype(np.float32)
    assert (np.diff(t) > 0).all()
    return t


def _softmax32(logit):
    e = np.exp(logit - logit.max(1, keepdims=True))
    return (e / e.sum(1, keepdims=True)).astype(np.float32)


def _ramp_weights(rng, pi, scale, L, lo, hi):
    """rows of weights whose fp32 in-order sum, times scale, rounds to c with c mod 2^16 <= 65536 - L: a row whose
    every term is saturated low is then c + l, strictly increasing and codable"""
    for _ in range(64):
        acc = np.zeros(pi.shape[0], np.float32)
        for k in range(pi.shape[1]):
            acc = acc + pi[:, k]
        c = np.rint((acc * np.float32(scale)).astype(np.float64)).astype(np.int64) & 0xFFFF
        redo = c > 65536 - L
        if not redo.any():
            break
        pi[redo] = np.sign(pi[redo]) * rng.uniform(lo, hi, pi[redo].shape).astype(np.float32)
    return pi


def make_stream(family, Lp, K, tkind, rng, n=None):
    """-> dict: t [Lp], mu / ls / pi float32 [n, K], sym int16 [n] (0, Lp - 2, then random), the parameters of the
    family (tkind 'on': a third of the finite means moved onto targets)"""
    L = Lp - 1
    n = n_rows(Lp) if n is None else n
    t = targets('log' if tkind == 'log' else 'even', Lp)
    tt = t[:L]
    x0, x1 = float(tt[0]), float(tt[-1])
    R = max(x1 - x0, 2.0 / 32768)
    bw = R / max(L - 1, 1)
    logit = rng.normal(0, 1, (n, K))
    logit[np.arange(n), rng.integers(0, K, n)] += rng.uniform(3, 10, n)
    mu = rng.uniform(x0 - 0.2 * R, x1 + 0.2 * R, (n, K)).astype(np.float32)
    ls = (np.log(bw) + rng.uniform(-4, 3, (n, K))).astype(np.float32)
    pi = None
    sel = rng.random((n, K)) < 0.5
    if family == 'wide':
        ls = rng.choice(np.linspace(8, 20, 13), (n, K)).astype(np.float32)
    elif family == 'logscale':
        ls = rng.uniform(-30, 20, (n, K)).astype(np.float32)
        ls[sel] = rng.choice(np.float32([-30, -7, 0, 20]), int(sel.sum()))
    elif family == 'far':
        mu[sel] = rng.choice(np.float32([1e6, -1e6, 3e38, -3e38]), int(sel.sum()))
    elif family == 'pi_underflow':
        logit[sel] = -rng.uniform(80, 400, int(sel.sum()))          # fp32 subnormal below -87.3, 0 below -103.3
        logit[:, 0] = 0
    elif family == 'sum_pi':
        pi = np.full((n, K), np.float32(1.0 / K), np.float32)
        up = rng.random(n) < 0.5
        pi[up] = (pi[up] * np.float32(1 + 2.0 ** -21)).astype(np.float32)
    elif family == 'nonfinite':
        pi = _softmax32(logit)
        for arr, vals in ((pi, [np.nan, np.inf, -np.inf]), (mu, [np.nan, np.inf, -np.inf]),
                          (ls, [np.nan, np.inf, -np.inf, -100, -1e30])):
            pick = rng.random((n, K)) < 0.15
            arr[pick] = rng.choice(np.float32(vals), int(pick.sum()))
        # inf * 0: an infinite mean under a +inf log-scale (inv_s = -0) makes u NaN at every target
        r, k = rng.integers(0, n, max(1, n // 6)), rng.integers(0, K, max(1, n // 6))
        mu[r, k], ls[r, k] = rng.choice(np.float32([np.inf, -np.inf]), r.size), np.inf
    elif family in ('unnorm', 'unnorm_big'):
        # every term saturated or at u = 0, so the restatement decides every entry: narrow components, means on a
        # target or a quarter of a bin or more away from every target; half the rows below every target (c + l)
        scale = 65536 - L
        lo, hi = (200.0, 1900.0) if family == 'unnorm' else (1.05 * TWO31 / scale / K, 8.0 * TWO31 / scale / K)
        sign = np.where(rng.random((n, 1)) < 0.7, 1.0, -1.0) if family == 'unnorm_big' else \
            np.where(rng.random((n, K)) < 0.7, 1.0, -1.0)
        pi = (sign * rng.uniform(lo, hi, (n, K))).astype(np.float32)
        if family == 'unnorm_big':
            big = rng.random(n) < 0.2
            pi[big] = (pi[big] * np.float32(1e4)).astype(np.float32)
        ls = rng.uniform(-30, -25, (n, K)).astype(np.float32)
        j = rng.integers(0, L, (n, K))
        frac = rng.choice([0.0, 0.25, 0.5, 0.75], (n, K)) * (tkind != 'on')
        nxt = t[np.minimum(j + 1, L)].astype(np.float64)
        mu = (tt[j] + frac * (nxt - tt[j])).astype(np.float32)
        ramp = rng.random(n) < 0.5
        mu[ramp] = (x0 - R - rng.uniform(0, 1, (int(ramp.sum()), K))).astype(np.float32)
        pi[ramp] = _ramp_weights(rng, pi[ramp], scale, L, lo, hi)
    if pi is None:
        pi = _softmax32(logit)
    if tkind == 'on' and family not in ('unnorm', 'unnorm_big'):
        on = (rng.random((n, K)) < 0.35) & np.isfinite(mu) & (np.abs(mu) < 1e6)
        mu[on] = tt[rng.integers(0, L, int(on.sum()))]
    sym = rng.integers(0, L, n)
    sym[0] = 0
    if n > 1:
        sym[1] = L - 1
    return dict(family=family, Lp=Lp, K=K, tkind=tkind, t=t, mu=np.ascontiguousarray(mu),
                ls=np.ascontiguousarray(ls), pi=np.ascontiguousarray(pi), sym=sym.astype(np.int16))


def grid_streams(family, Lp, seed=0):
    """one stream per K, the target kinds cycled so that every (Lp, K) pair and every (Lp, target kind) pair is met"""
    rng = np.random.default_rng(1000 * FAMILIES.index(family) + Lp + seed)
    li = LPS.index(Lp) if Lp in LPS else 0
    return [make_stream(family, Lp, K, TARGETS[(i + li) % 3], rng) for i, K in enumerate(KS)]


def in_domain(st):
    """[n] rows where a strictly increasing row with last entry <= 65535 is promised"""
    with np.errstate(over='ignore', invalid='ignore'):
        fin = np.isfinite(st['pi']) & np.isfinite(st['mu']) & np.isfinite(st['ls']) & \
            np.isfinite(np.exp(-st['ls'].astype(np.float64)).astype(np.float32))
        return fin.all(1) & (st['pi'] >= 0).all(1) & (st['pi'].astype(np.float64).sum(1) <= 1 + 2.0 ** -20)


# ---------------------------------------------------------------------------------------------------------------------
# restatement and checks
# ---------------------------------------------------------------------------------------------------------------------
def inv_s_unclamped(ls):
    """-log2(e) / sigma as the drop-in computes it from the raw log-scale (expf to within 2 ulp, then one rounding)"""
    with np.errstate(over='ignore', invalid='ignore'):
        return np.exp(-ls.astype(np.float64)).astype(np.float32) * NEG_LOG2E


def restate_stream(st, entries=None, defect=None):
    """restate() of every row of a stream over `entries` (default L) targets, in chunks of rows.  defect: a planted
    mis-restatement -- 'scale' (65536 - Lp), 'shift' (targets shifted by one) or 'round32' (a saturating 32-bit
    round)"""
    L = st['Lp'] - 1
    E = L if entries is None else entries
    t = st['t']
    kw = {'scale': 65536 - L}
    if defect == 'scale':
        kw['scale'] = 65536 - st['Lp']
    elif defect == 'shift':
        t = np.concatenate([t[1:], t[-1:] + (t[-1] - t[-2])]).astype(np.float32)
    elif defect == 'round32':
        kw['rnd'] = f2i_rn
    inv_s = inv_s_unclamped(st['ls'])
    n, K = st['pi'].shape
    step = max(1, CHUNK_ELEMS // (E * K))
    parts = [restate(st['pi'][a:a + step], st['mu'][a:a + step], inv_s[a:a + step], t, E, U_REL_EXPF, **kw)
             for a in range(0, n, step)]
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0] if k != 'u'}


def sub_ref(ref, rows):
    return {k: v[rows] for k, v in ref.items()}


def check_stream_rows(got, ref, st, what):
    """got uint16 [r, L]: per entry against the restatement -> stats (band, |V| >= 2^31 entries)"""
    try:
        stt = check_rows(got, ref, what)
    except AssertionError as e:
        bad = np.argwhere((got.astype(np.int64) != ref['lo']) & (got.astype(np.int64) != ref['hi']))
        r, l = bad[0]
        raise AssertionError('%s\n  first bad entry: row %d l %d, |V| = %.6g (%s 2^31), family %s K %d targets %s'
                             % (e, r, l, abs(ref['V'][r, l]), '>=' if abs(ref['V'][r, l]) >= TWO31 else '<',
                                st['family'], st['K'], st['tkind'])) from None
    with np.errstate(invalid='ignore'):
        stt['n_big'] = int((np.abs(ref['V']) >= TWO31).sum())
    stt['n_band'] = int(ref['band'].sum())
    return stt


def restated_intervals(ref, sym, L, top=None):
    """acceptable packed intervals lo | (hi - 1) << 16 of each symbol: (lo_a, lo_b, hm1_a, hm1_b); hi = 65536 for
    symbol L - 1 unless top ([n, 2] acceptable values of the entry at target L) is given"""
    r = np.arange(len(sym))
    s = sym.astype(np.int64)
    lo_a, lo_b = ref['lo'][r, s], ref['hi'][r, s]
    nx = np.minimum(s + 1, L - 1)
    hi_a, hi_b = ref['lo'][r, nx], ref['hi'][r, nx]
    last = s == L - 1
    ta, tb = (65536, 65536) if top is None else (top[:, 0], top[:, 1])
    hi_a, hi_b = np.where(last, ta, hi_a), np.where(last, tb, hi_b)
    return lo_a, lo_b, (hi_a - 1) & 0xFFFF, (hi_b - 1) & 0xFFFF


def check_intervals(iv, ref, sym, L, what, top=None):
    iv = np.asarray(iv).view(np.uint32).astype(np.int64)
    lo_a, lo_b, h_a, h_b = restated_intervals(ref, sym, L, top)
    lo, hm1 = iv & 0xFFFF, iv >> 16
    ok = ((lo == lo_a) | (lo == lo_b)) & ((hm1 == h_a) | (hm1 == h_b))
    bad = np.flatnonzero(~ok)
    assert bad.size == 0, '%s: %d of %d intervals outside the restated rows; first symbol %d (value %d): got %d..%d' \
        % (what, bad.size, ok.size, bad[0], sym[bad[0]], lo[bad[0]], hm1[bad[0]] + 1)


def row_intervals(rows, sym):
    """packed intervals from rows [n, L] (what the coder is handed for these rows)"""
    L = rows.shape[1]
    s = sym.astype(np.int64)
    r = np.arange(len(s))
    lo = rows[r, s].astype(np.int64)
    hi = np.where(s == L - 1, 65536, rows[r, np.minimum(s + 1, L - 1)].astype(np.int64))
    return (lo | (((hi - 1) & 0xFFFF) << 16)).astype(np.uint32)


def top_entry(st):
    """[n, 2] acceptable values of the entry at target L (what the reference computes there; the drop-in codes
    symbol Lp - 2 up to 65536 instead)"""
    L = st['Lp'] - 1
    ref = restate_stream(st, entries=L + 1)
    return np.stack([ref['lo'][:, L], ref['hi'][:, L]], 1)


def codable(rows):
    """[n] rows whose intervals are all at least one count wide"""
    return (np.diff(rows.astype(np.int64), axis=1) >= 1).all(1)


def check_codable(rows, ref, st, what):
    """in the domain: strictly increasing, last entry <= 65535 before the 16-bit wrap -> number of rows checked"""
    dom = in_domain(st)
    r = rows[dom].astype(np.int64)
    bad = np.flatnonzero(~codable(r))
    assert bad.size == 0, '%s: %d rows in the domain are not strictly increasing, first %d' % (
        what, bad.size, np.flatnonzero(dom)[bad[0]])
    last = r[:, -1]
    lo_raw, hi_raw = ref['lo_raw'][dom, -1], ref['hi_raw'][dom, -1]
    assert ((last == lo_raw) | (last == hi_raw)).all() and (hi_raw <= 65535).all(), \
        '%s: a last entry wraps past 65535' % what
    return int(dom.sum())


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the checks pass a float32 model of the kernels and reject planted mis-restatements
# ---------------------------------------------------------------------------------------------------------------------
SELF_LPS = [2, 26, 258, 1025]
DEFECTS = ('scale', 'shift', 'top', 'round32')


def _model(st, push):
    """plane_cdf_u16 in numpy float32 (the sigmoid pushed by push x SIG_ABS): rows uint16 [n, L], intervals"""
    L = st['Lp'] - 1
    rows = emulate(st['pi'], st['mu'], inv_s_unclamped(st['ls']), st['t'], L,
                   np.full(st['pi'].shape[:1] + (L,) + st['pi'].shape[1:], float(push)), rnd=f2ll_rn)
    return rows.astype(np.uint16), row_intervals(rows, st['sym'])


def _check_all(st, rows, iv, defect=None):
    L = st['Lp'] - 1
    ref = restate_stream(st, defect=None if defect == 'top' else defect)
    check_stream_rows(rows, ref, st, 'model')
    check_intervals(iv, ref, st['sym'], L, 'model', top_entry(st) if defect == 'top' else None)
    return ref


@pytest.mark.parametrize('Lp', SELF_LPS)
def test_restatement_accepts_the_kernel_model(Lp):
    n_big = n_exact = 0
    for fam in FAMILIES:
        for st in grid_streams(fam, Lp):
            for push in (-1, 1, 0):                  # codability below on the unpushed, monotone sigmoid
                rows, iv = _model(st, push)
                ref = _check_all(st, rows, iv)
            if fam not in ('nonfinite', 'unnorm', 'unnorm_big'):
                assert in_domain(st).all(), (fam, st['K'])
                check_codable(rows, ref, st, fam)
            if fam in ('unnorm', 'unnorm_big'):
                assert ref['exact'].all(), 'the unnormalised families must be decided entry by entry'
                assert codable(rows).any(), 'some unnormalised rows must be codable'
            with np.errstate(invalid='ignore'):
                n_big += int((np.abs(ref['V']) >= TWO31).sum())
            n_exact += int(ref['exact'].sum())
    assert n_big > 0 and n_exact > 0


@pytest.mark.parametrize('defect', DEFECTS)
@pytest.mark.parametrize('Lp', SELF_LPS)
def test_planted_misrestatement_is_rejected(defect, Lp):
    rejected = []
    for fam in FAMILIES:
        for st in grid_streams(fam, Lp):
            rows, iv = _model(st, 0)
            try:
                _check_all(st, rows, iv, defect)
            except AssertionError:
                rejected.append((fam, st['K']))
    assert rejected, 'the %s mis-restatement passed every stream at Lp=%d' % (defect, Lp)
    if defect == 'round32':
        assert {f for f, _ in rejected} == {'unnorm_big'}, rejected
    print('%s at Lp=%d: rejected on %d of %d streams' % (defect, Lp, len(rejected), 4 * len(FAMILIES)))


def test_families_reach_their_regimes():
    """the parameters are what the families claim: log-scales down to -30 unclamped, Lp - 2 coded, sums in the
    thousands and beyond 2^31 / scale, subnormal and zero weights, non-finite values"""
    for Lp in (258, 32769):
        scale = 65536 - (Lp - 1)
        s = {f: grid_streams(f, Lp) for f in FAMILIES}
        assert all(st['sym'][1] == Lp - 2 for f in FAMILIES for st in s[f])
        assert min(float(st['ls'].min()) for st in s['logscale']) <= -29.9
        sums = [np.abs(st['pi'].astype(np.float64).sum(1)) for st in s['unnorm']]
        assert max(float(x.max()) for x in sums) >= 1000 and max(float(x.max()) for x in sums) * scale < TWO31
        big = [np.abs(st['pi'].astype(np.float64).sum(1)) * scale for st in s['unnorm_big']]
        assert min(float(x.min()) for x in big) >= TWO31
        pu = np.concatenate([st['pi'].ravel() for st in s['pi_underflow']])
        assert (pu == 0).any() and ((pu > 0) & (pu < np.finfo(np.float32).tiny)).any()
        assert any((st['pi'].astype(np.float64).sum(1) > 1).any() for st in s['sum_pi'])
        nf = [x for st in s['nonfinite'] for x in (st['pi'], st['mu'], st['ls'])]
        assert any(np.isnan(x).any() for x in nf) and any(np.isinf(x).any() for x in nf)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _dev(st):
    """device tensors of the stream, in the drop-in's shapes: targets [Lp], planes 1 x K x 1 x n"""
    n, K = st['pi'].shape
    pl = [torch.from_numpy(np.ascontiguousarray(st[k].T)).reshape(1, K, 1, n).cuda() for k in ('mu', 'ls', 'pi')]
    return [torch.from_numpy(st['t']).cuda()] + pl


def _sources(devs):
    from l3c_pytorch_b200 import torchac
    return torchac._mixture_sources(*[list(x) for x in zip(*devs)])


def launch_rows(devs, first, count):
    """one l3c_batch_rows launch for symbols [first, first + count) of every stream, into a canary-guarded buffer
    -> [rows uint16 [r_j, pitch_j]]"""
    from l3c_pytorch_b200 import _lib, engine as E, torchac
    dev, src, n, Lp, keep = _sources(devs)
    r = np.clip(np.minimum(count, n - first), 0, None)
    pitch = torchac.row_bytes(Lp - 1) // 2
    row_off = np.concatenate([[0], np.cumsum(r * pitch)]).astype(np.int64)
    total = int(row_off[-1])
    buf = torch.full((GUARD + 2 * total + GUARD,), CANARY, dtype=torch.uint8, device=dev)
    src_dev, off_dev = E._desc_to_device(src, dev), E._to_device_async(row_off, dev)
    _lib.check(_lib.lib.l3c_batch_rows(E._ptr(src_dev), E._ptr(off_dev), len(devs), total, first,
                                       ctypes.c_void_p(buf.data_ptr() + GUARD), E._stream_ptr()))
    h = buf.cpu().numpy()
    assert (h[:GUARD] == CANARY).all() and (h[GUARD + 2 * total:] == CANARY).all(), 'rows written out of bounds'
    rows = h[GUARD:GUARD + 2 * total].view(np.uint16)
    return [rows[row_off[j]:row_off[j + 1]].reshape(int(r[j]), int(pitch[j])) for j in range(len(devs))]


def launch_intervals(devs, syms):
    """one l3c_batch_intervals launch -> ([iv uint32 [n_j]], bad int32 [streams])"""
    from l3c_pytorch_b200 import _lib, engine as E
    dev, src, n, Lp, keep = _sources(devs)
    sd = [torch.from_numpy(np.asarray(s, np.int16)).cuda() for s in syms]
    src['sym'] = [s.data_ptr() for s in sd]
    off = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    iv = torch.full((int(off[-1]),), -1, dtype=torch.int32, device=dev)
    bad = torch.empty(len(devs), dtype=torch.int32, device=dev)
    src_dev, off_dev = E._desc_to_device(src, dev), E._to_device_async(off, dev)
    _lib.check(_lib.lib.l3c_batch_intervals(E._ptr(src_dev), E._ptr(off_dev), len(devs), int(off[-1]), E._ptr(iv),
                                            E._ptr(bad), E._stream_ptr()))
    h = iv.cpu().numpy().view(np.uint32)
    return [h[off[j]:off[j + 1]] for j in range(len(devs))], bad.cpu().numpy()


def _substream(st, rows):
    out = dict(st)
    for k in ('mu', 'ls', 'pi'):
        out[k] = np.ascontiguousarray(st[k][rows])
    out['sym'] = st['sym'][rows]
    return out


def _oracle_bytes(rows, sym):
    return ac.encode(np.concatenate([rows, np.zeros((rows.shape[0], 1), np.uint16)], 1), sym)


STATS = {}


@pytest.mark.gpu
@pytest.mark.parametrize('Lp', LPS)
@pytest.mark.parametrize('family', FAMILIES)
def test_dropin_rows_intervals_and_streams(family, Lp):
    """rows and intervals of the four streams (K = 1, 3, 10, 17) of a family at one Lp against the restatement;
    the codable rows' streams: the oracle's bytes from both encoders, the symbols back from both decoders"""
    from l3c_pytorch_b200 import torchac
    L = Lp - 1
    streams = grid_streams(family, Lp)
    devs = [_dev(st) for st in streams]
    rows = launch_rows(devs, 0, max(len(st['sym']) for st in streams))
    ivs, bad = launch_intervals(devs, [st['sym'] for st in streams])
    assert (bad == -1).all()
    n_dom = n_cod = 0
    for st, dv, rw, iv in zip(streams, devs, rows, ivs):
        what = '%s Lp=%d K=%d %s' % (family, Lp, st['K'], st['tkind'])
        ref = restate_stream(st)
        got = rw[:, :L]
        stt = check_stream_rows(got, ref, st, what + ' batch_rows')
        assert (rw[:, L:] == 0).all(), '%s: the padding up to the pitch is not zero' % what
        agg = STATS.setdefault(Lp, [0, 0, 0])
        agg[0] += got.size
        agg[1] += stt['n_band']
        agg[2] += stt['n_big']
        check_intervals(iv, ref, st['sym'], L, what + ' batch_intervals')
        assert (iv == row_intervals(got, st['sym'])).all(), '%s: batch intervals differ from the rows' % what
        n_dom += check_codable(got, ref, st, what)
        if family not in ('nonfinite', 'unnorm', 'unnorm_big'):
            assert in_domain(st).all()
        # codable rows: one stream of them through the single-stream entry points and the batched ones
        ok = codable(got)
        if not ok.any():
            continue
        n_cod += int(ok.sum())
        sub = _substream(st, ok)
        sd = _dev(sub)
        sym = torch.from_numpy(sub['sym'])
        want = _oracle_bytes(got[ok], sub['sym'])
        data = torchac.encode_logistic_mixture(*sd, sym)
        assert data == want, '%s: encode_logistic_mixture differs from the oracle on the kernel rows' % what
        assert torchac.encode_logistic_mixture_batch(*[[x] for x in sd], [sym])[0] == want, what
        back = torchac.decode_logistic_mixture(*sd, want)
        assert (back.numpy() == sub['sym']).all(), '%s: decode_logistic_mixture lost symbols' % what
        back = torchac.decode_logistic_mixture_batch(*[[x] for x in sd], [want])[0]
        assert (back.cpu().numpy() == sub['sym']).all(), '%s: decode_logistic_mixture_batch lost symbols' % what
    if family in ('trained', 'wide', 'logscale', 'far', 'pi_underflow', 'sum_pi'):
        assert n_cod == n_dom == sum(len(st['sym']) for st in streams)
    if family == 'unnorm_big':
        assert n_cod > 0, 'no row above 2^31 was coded'
    print('%s Lp=%d: %d rows in the domain, %d codable rows coded; Lp totals (entries, in the band, |V| >= 2^31): %s'
          % (family, Lp, n_dom, n_cod, STATS[Lp]))


RAGGED_LPS = [2, 3, 26, 33, 256, 257, 258, 264, 265]


def _ragged_streams():
    """300 streams of 1 to 7 symbols (every family, Lp up to 265) and long streams at every Lp"""
    rng = np.random.default_rng(77)
    out = []
    for i in range(300):
        fam = FAMILIES[i % len(FAMILIES)]
        out.append(make_stream(fam, RAGGED_LPS[(i // len(FAMILIES)) % len(RAGGED_LPS)], KS[i % 4],
                               TARGETS[i % 3], rng, n=int(rng.integers(1, 8))))
    for Lp, n in [(257, 60), (1025, 23), (4097, 11), (32769, 4), (26, 200), (3, 300)]:
        out.insert(int(rng.integers(0, len(out))), make_stream(FAMILIES[Lp % len(FAMILIES)], Lp, 3, 'log', rng, n=n))
    return out


@pytest.mark.gpu
def test_ragged_launch_with_first_and_mid_stream_counts():
    """one launch over 306 streams, blocks spanning many streams: every (first, count) gives each stream's rows
    [first, first + count) clipped to its length, streams with no rows left included"""
    streams = _ragged_streams()
    devs = [_dev(st) for st in streams]
    refs = [restate_stream(st) for st in streams]
    n_max = max(len(st['sym']) for st in streams)
    for first, count in [(0, n_max), (0, 3), (2, 3), (5, 1), (6, n_max), (3, 7), (250, 40)]:
        rows = launch_rows(devs, first, count)
        for j, (st, ref, rw) in enumerate(zip(streams, refs, rows)):
            L = st['Lp'] - 1
            r = max(0, min(count, len(st['sym']) - first))
            assert rw.shape[0] == r
            if r == 0:
                continue
            what = 'stream %d (%s Lp=%d) first %d count %d' % (j, st['family'], st['Lp'], first, count)
            check_stream_rows(rw[:, :L], sub_ref(ref, slice(first, first + r)), st, what)
            assert (rw[:, L:] == 0).all(), what
    ivs, bad = launch_intervals(devs, [st['sym'] for st in streams])
    assert (bad == -1).all()
    for j, (st, ref, iv) in enumerate(zip(streams, refs, ivs)):
        check_intervals(iv, ref, st['sym'], st['Lp'] - 1, 'ragged stream %d' % j)


@pytest.mark.gpu
def test_out_of_range_symbols_report_the_first_bad_position():
    rng = np.random.default_rng(5)
    streams = [make_stream('trained', Lp, 3, 'even', rng, n=40) for Lp in (2, 26, 257, 1025, 32769, 258)]
    syms = [st['sym'].copy() for st in streams]
    # Lp - 1 (no interval ends past 65536) and negatives are out of range; 32767 at Lp = 32769 is Lp - 2
    plant = {0: [(3, 1)], 1: [(7, 25), (30, -1)], 2: [(0, -32768)], 3: [(39, 1024)], 4: [(12, 32767), (5, 32767)]}
    for j, hits in plant.items():
        for pos, v in hits:
            syms[j][pos] = v
    ivs, bad = launch_intervals([_dev(st) for st in streams], syms)
    want = [3, 7, 0, 39, -1, -1]
    assert bad.tolist() == want, bad.tolist()
    for j, (st, iv, s) in enumerate(zip(streams, ivs, syms)):
        L = st['Lp'] - 1
        bad_pos = (s < 0) | (s > L - 1)
        assert (iv[bad_pos] == 0).all()
        ref = restate_stream(st)
        ok = ~bad_pos
        check_intervals(iv[ok], sub_ref(ref, ok), s[ok], L, 'stream %d' % j)


@pytest.mark.gpu
@pytest.mark.parametrize('Lp,K', [(258, 10), (4097, 3), (26, 17)])
def test_input_forms_code_like_float32(Lp, K):
    """float64, float16 and non-contiguous parameters give the bytes of the float32 contiguous call on the values
    _check_mixture converts them to; the symbols come back"""
    from l3c_pytorch_b200 import torchac
    rng = np.random.default_rng(Lp + K)
    st = make_stream('trained', Lp, K, 'log', rng, n=64)
    base = _dev(st)
    sym = torch.from_numpy(st['sym'])
    d32 = torchac.encode_logistic_mixture(*base, sym)
    # float64 values off the float32 grid, float16 values
    jit = [x.double() * (1 + 1e-9 * torch.randn_like(x.double())) for x in base]
    f16 = [base[1].half(), base[2].half(), (base[3] * 0.99).half()]      # weights summing below 1 in float16
    forms = {
        'float64': (jit, [x.float() for x in jit]),
        'float16': ([base[0]] + f16, [base[0]] + [x.float() for x in f16]),
    }
    # non-contiguous: strided targets, planes as a slice of a wider tensor and as a transposed [n, K] array
    wide = [torch.stack([x, torch.zeros_like(x)], -1).reshape(1, K, 1, 2 * x.shape[-1])[..., ::2] for x in base[1:]]
    tr = [x.reshape(K, -1).t().contiguous().t().reshape(1, K, 1, -1) for x in base[1:]]
    t_str = torch.stack([base[0], base[0]], 1)[:, 0]
    forms['strided'] = ([t_str] + wide, base)
    forms['transposed'] = ([base[0]] + tr, base)
    for name, (given, as32) in forms.items():
        if name in ('strided', 'transposed'):
            assert not any(x.is_contiguous() for x in given[name == 'transposed':])
        want = torchac.encode_logistic_mixture(*as32, sym)
        if name in ('strided', 'transposed'):
            assert want == d32
        assert torchac.encode_logistic_mixture(*given, sym) == want, name
        assert torchac.encode_logistic_mixture_batch(*[[x] for x in given], [sym])[0] == want, name
        assert (torchac.decode_logistic_mixture(*given, want).numpy() == st['sym']).all(), name
        assert (torchac.decode_logistic_mixture_batch(*[[x] for x in given], [want])[0].cpu().numpy()
                == st['sym']).all(), name
