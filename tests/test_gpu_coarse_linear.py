"""Linear brackets of the coarse RGB decoder (DESIGN §4.4): bracket j of a coarse record is linear when every mixture
term is saturated on the same side at t[8 j] and t[8 j + 7] (dmll_math.cuh: mixture_linear); the decoder then takes
the bracket's entries as cdf[8 j] + e without evaluating them, and evaluates the other brackets term-parallel.

* Host: a numpy float32 model of the rule (the same IEEE-rounded subtraction and multiplication, the same compares)
  on random parameter sets -- sigma down to 1e-3 bins, means exactly on targets, u exactly on SAT_LO and SAT_HI --
  equals the explicit "same side at both ends" test, and wherever it marks a bracket linear, the row computed with
  the saturated-term definition is cdf[8 j] + e at every entry of the bracket.
* GPU: on the records l3c_dmll_build_coarse writes (peaked, broad and mixed parameters, plus an all-linear and a
  no-linear kind), every bracket the rule marks linear is exactly cdf[8 j] + e in dmll_table_kernel's full row.
* GPU: oracle streams decode from the records to the oracle's symbols and saved states after every launch, under
  every streams-per-CTA variant and chunk schedule (one symbol per launch included, so both bounds of every
  evaluated entry are compared), on linear-only, non-linear-only and mixed streams, junk and truncated input."""
import numpy as np
import pytest

SAT_LO, SAT_HI = np.float32(-25.0), np.float32(40.0)
SCALE = np.float32(65536 - 256)
K = 10
NEG_LOG2E = np.float32(-1.4426950408889634)


def _targets():
    """the RGB bin edges of DiscretizedMixLogisticLoss(True, 0, 255, 256).targets(): -0.5 .. 255.5"""
    return np.linspace(-0.5, 255.5, 257, dtype=np.float32)


def linear_mask(mu, inv_s, tg):
    """[..., 32] bool: bracket j linear for the parameter sets mu, inv_s [..., K] (float32)"""
    t0, t1 = tg[0:256:8], tg[7:256:8]
    u0 = (t0[:, None] - mu[..., None, :]) * inv_s[..., None, :]
    u1 = (t1[:, None] - mu[..., None, :]) * inv_s[..., None, :]
    return ((u0 <= SAT_LO) | (u1 >= SAT_HI)).all(-1)


def _side(u):
    return np.where(u <= SAT_LO, -1, np.where(u >= SAT_HI, 1, 0))


def _same_side_mask(mu, inv_s, tg):
    """the rule as stated: every term has the same nonzero side at both ends"""
    u0 = (tg[0:256:8][:, None] - mu[..., None, :]) * inv_s[..., None, :]
    u1 = (tg[7:256:8][:, None] - mu[..., None, :]) * inv_s[..., None, :]
    s0, s1 = _side(u0), _side(u1)
    return ((s0 != 0) & (s0 == s1)).all(-1)


def _saturated_row(pi, mu, inv_s, tg):
    """cdf[0..255] of one parameter set where every term of an entry is saturated (mixture_saturated: a sum of pi's,
    in term order, in float32), and which entries are"""
    u = (tg[:256, None] - mu[None]) * inv_s[None]
    lo, hi = u <= SAT_LO, u >= SAT_HI
    acc = np.zeros(256, np.float32)
    for k in range(K):
        acc = np.where(lo[:, k], acc + pi[k], acc).astype(np.float32)
    cdf = (np.rint(acc * SCALE).astype(np.int64) + np.arange(256)) & 0xFFFF
    return cdf, (lo | hi).all(1)


def _random_sets(rng, n):
    """n parameter sets (pi, mu, inv_s) [n, K] float32"""
    tg = _targets()
    logit = rng.normal(0, 2, (n, K))
    pi = np.exp(logit - logit.max(1, keepdims=True))
    pi = (pi / pi.sum(1, keepdims=True)).astype(np.float32)
    sigma = np.exp(rng.uniform(np.log(1e-3), np.log(30.0), (n, K)))        # bins
    inv_s = (NEG_LOG2E / sigma).astype(np.float32)
    mu = rng.uniform(-40, 300, (n, K)).astype(np.float32)
    pick = rng.random((n, K))
    on = pick < 0.2                                                         # means exactly on targets
    mu[on] = tg[rng.integers(0, 257, on.sum())]
    # u exactly on SAT_LO / SAT_HI at a bracket end: inv_s a power of two, mu = t - u / inv_s (exact)
    edge = (pick >= 0.2) & (pick < 0.5)
    ne = int(edge.sum())
    p2 = -(2.0 ** rng.integers(-3, 6, ne)).astype(np.float32)
    j = rng.integers(0, 32, ne)
    t = np.where(rng.random(ne) < 0.5, tg[8 * j], tg[8 * j + 7]).astype(np.float32)
    u = np.where(rng.random(ne) < 0.5, SAT_LO, SAT_HI).astype(np.float32)
    inv_s[edge] = p2
    mu[edge] = t - u / p2
    return pi, mu, inv_s


def test_linear_rule_host_model():
    rng = np.random.default_rng(11)
    tg = _targets()
    pi, mu, inv_s = _random_sets(rng, 3000)
    lin = linear_mask(mu, inv_s, tg)
    assert (lin == _same_side_mask(mu, inv_s, tg)).all()
    # the boundary cases land exactly on the thresholds
    u_ends = (tg[None, None, :256] - mu[..., None]) * inv_s[..., None]
    assert (u_ends == SAT_LO).any() and (u_ends == SAT_HI).any()
    n_lin = 0
    for i in range(len(pi)):
        cdf, sat = _saturated_row(pi[i], mu[i], inv_s[i], tg)
        for jj in np.flatnonzero(lin[i]):
            m = 8 * jj + np.arange(8)
            assert sat[m].all(), (i, jj)
            assert (cdf[m] == (cdf[8 * jj] + np.arange(8)) & 0xFFFF).all(), (i, jj, cdf[m])
            n_lin += 1
    # both outcomes occur
    assert 0 < n_lin < lin.size, n_lin


def test_linear_rule_never_marks_nan():
    tg = _targets()
    mu = np.full((1, K), -1000.0, np.float32)
    inv_s = np.full((1, K), -1.0, np.float32)
    assert linear_mask(mu, inv_s, tg).all()
    mu[0, 3] = np.nan
    assert not linear_mask(mu, inv_s, tg).any()


# ------------------------------------------------------------------------------------------------------------
# GPU: the builder's records against dmll_table_kernel's full rows, and the decoder against the oracle
# ------------------------------------------------------------------------------------------------------------
KINDS = ('peaked', 'broad', 'mixed', 'linear', 'nonlinear', 'split')


def _params_extra(kind, rng, N, HW, C):
    """'linear': every component's mean on the pixel value 8 j + 7 with the smallest scale, coupling off: each
    component saturated at every target, so every bracket is linear; 'nonlinear': broad components (sigma of e^3 to
    e^5 bins) unsaturated over the whole row, so none is; 'split': either, per pixel"""
    shp = (N, HW, C, K)
    lin = dict(logit=rng.normal(0, 2, shp), mean=(8 * rng.integers(0, 32, shp) + 7).astype(np.float64),
               logs=rng.uniform(-12, -7, shp), coef=np.full(shp, -40.0))
    non = dict(logit=rng.normal(0, 1, shp), mean=rng.uniform(-60, 315, shp), logs=rng.uniform(3, 5, shp),
               coef=rng.normal(0, 2, shp))
    if kind == 'linear':
        p = lin
    elif kind == 'nonlinear':
        p = non
    else:
        pick = rng.random((N, HW, 1, 1)) < 0.5
        p = {k: np.where(pick, lin[k], non[k]) for k in lin}
    return np.stack([p['logit'], p['mean'], p['logs'], p['coef']], axis=2).astype(np.float32)


def _case(kind):
    """test_gpu_coarse_rows' case (full rows, records, oracle streams) for any of KINDS; registered in that module's
    cache so that its oracle decode harness runs on it"""
    import torch
    from oracle import ac
    from tests import test_gpu_coarse_rows as CR
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    key = 'linear-' + kind
    if key in CR.CASES:
        return key, CR.CASES[key]
    dev = torch.device('cuda')
    N, H, W, HW, C, L = CR.N, CR.H, CR.W, CR.HW, CR.C, CR.L
    rng = np.random.default_rng(301 + KINDS.index(kind))
    if kind in CR.KINDS:
        l, sym = CR._params(kind, rng)
    else:
        l = _params_extra(kind, rng, N, HW, C).reshape(N, H, W, 4 * C * K)
        sym = rng.integers(0, 256, (N, C, HW)).astype(np.uint8)        # uniform symbols: every bracket is visited
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
    streams = [[ac.encode(np.concatenate([rows[n, c, :CR.NS[n]], np.zeros((CR.NS[n], 1), np.uint16)], 1),
                          sym[n, c, :CR.NS[n]]) for c in range(C)] for n in range(N)]
    CR.CASES[key] = dict(l=l_dev, sym=sym, tg=tg, rows=rows, recs=recs, rec=rec, streams=streams)
    return key, CR.CASES[key]


def _record_mask(cs):
    """the rule on the records' own parameters (float32 bits as the decoder reads them): [N, C, HW, 32]"""
    par = np.ascontiguousarray(cs['recs'][..., :64]).view(np.float32)
    return linear_mask(par[..., K:2 * K], par[..., 2 * K:3 * K], cs['tg'].cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize('kind', KINDS)
def test_linear_brackets_match_full_rows(kind):
    _, cs = _case(kind)
    rows = cs['rows'].astype(np.int64)
    lin = _record_mask(cs)
    head = rows[..., ::8]                                                    # [N, C, HW, 32]
    want = (head[..., None] + np.arange(8)) & 0xFFFF
    is_lin = (rows.reshape(rows.shape[:-1] + (32, 8)) == want).all(-1)
    bad = np.argwhere(lin & ~is_lin)
    assert bad.size == 0, '%s: %d brackets marked linear are not cdf[8 j] + e in the full row, first %s' % (
        kind, len(bad), bad[0])
    frac = lin.mean()
    print('%s: %.1f %% of the brackets linear (%.1f %% of the full rows\' brackets are)' % (
        kind, 100 * frac, 100 * is_lin.mean()))
    if kind == 'linear':
        assert lin.all()
    elif kind == 'nonlinear':
        assert not lin.any()
    elif kind == 'split':
        assert 0 < frac < 1


@pytest.mark.gpu
@pytest.mark.parametrize('spc', [1, 2, 4])
@pytest.mark.parametrize('kind', ('linear', 'nonlinear', 'split'))
def test_linear_and_term_parallel_decode_match_oracle(kind, spc):
    from tests import test_gpu_coarse_rows as CR
    key, cs = _case(kind)
    # the decoded symbols' brackets: all linear, none, or both
    lin = _record_mask(cs)
    n, c, p = np.meshgrid(np.arange(CR.N), np.arange(CR.C), np.arange(CR.HW), indexing='ij')
    hit = lin[n, c, p, cs['sym'].astype(np.int64) >> 3]
    assert hit.all() if kind == 'linear' else (not hit.any()) if kind == 'nonlinear' else (0 < hit.mean() < 1)
    CR.test_coarse_decode_matches_oracle(key, spc)
