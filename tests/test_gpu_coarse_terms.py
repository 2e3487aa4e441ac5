"""The coarse RGB decoder (DESIGN §4.4) on records whose brackets have a chosen number of varying mixture terms --
terms that are not saturated on the same side over the whole bracket, so that the decoder has to evaluate them --
and on records with NaN weights.

* Host: the number of varying terms per bracket, counted with the kernels' float32 operations, is what the
  parameters were built for: 0, 1, 2, 4, 5 or 10 at every bracket of a record.
* GPU: oracle streams on such records decode to the oracle's symbols and saved states after every launch, for every
  streams-per-CTA variant and chunk schedule, with junk and truncated input and write guards (test_gpu_coarse_rows'
  harness).  Every count occurs among the decoded symbols' brackets: linear ones (no evaluation) and brackets with
  one to ten evaluated terms.  About 3 % of the records come from a NaN logit, which makes all ten weights NaN (the
  softmax cannot give an infinite one); their full rows are cdf[m] = m and decode like any other."""
import numpy as np
import pytest

from tests.test_gpu_coarse_linear import K, SAT_HI, SAT_LO, NEG_LOG2E, _targets

NV = (0, 1, 2, 4, 5, 10)
NAN_FRAC = 0.03


def vary_counts(mu, inv_s, tg):
    """[..., 32]: varying terms of every bracket for the parameter sets mu, inv_s [..., K] (float32)"""
    u0 = ((tg[0:256:8][:, None] - mu[..., None, :]).astype(np.float32) * inv_s[..., None, :]).astype(np.float32)
    u1 = ((tg[7:256:8][:, None] - mu[..., None, :]).astype(np.float32) * inv_s[..., None, :]).astype(np.float32)
    return (~((u0 <= SAT_LO) | (u1 >= SAT_HI))).sum(-1)


def _params_vary(rng, N, HW, C):
    """per sub-pixel nv in NV broad components (sigma e^3 to e^5 bins: varying over the whole row) at random term
    positions, the others narrow (the smallest scale, mean on a pixel value 8 j + 7: saturated at every target), no
    channel coupling: every bracket of the record has exactly nv varying terms.  A few sub-pixels get a NaN logit."""
    shp = (N, HW, C, K)
    nv = rng.choice(NV, (N, HW, C))
    broad = np.argsort(rng.random(shp), -1) < nv[..., None]
    logit = rng.normal(0, 2, shp)
    mean = np.where(broad, rng.uniform(-60, 315, shp), 8 * rng.integers(0, 32, shp) + 7)
    logs = np.where(broad, rng.uniform(3, 5, shp), rng.uniform(-12, -7, shp))
    coef = np.full(shp, -40.0)
    logit[..., 0] = np.where(rng.random(shp[:3]) < NAN_FRAC, np.nan, logit[..., 0])
    return np.stack([logit, mean, logs, coef], axis=2).astype(np.float32), nv


def test_vary_counts_host_model():
    rng = np.random.default_rng(404)
    tg = _targets()
    l, nv = _params_vary(rng, 2, 500, 3)
    mean, logs = l[:, :, 1], l[:, :, 2]                                       # [N, HW, C, K]
    inv_s = (np.exp(-np.maximum(logs.astype(np.float64), -7.0)) * NEG_LOG2E).astype(np.float32)
    got = vary_counts(mean, inv_s, tg)                                        # [N, HW, C, 32]
    assert (got == nv[..., None]).all()


def _case():
    """test_gpu_coarse_rows' case (full rows, records, oracle streams), registered in that module's cache so that its
    oracle decode harness runs on it"""
    import torch
    from oracle import ac
    from tests import test_gpu_coarse_rows as CR
    from l3c_pytorch_b200 import engine as E
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    key = 'terms-vary'
    if key in CR.CASES:
        return key, CR.CASES[key]
    dev = torch.device('cuda')
    N, H, W, HW, C, L = CR.N, CR.H, CR.W, CR.HW, CR.C, CR.L
    rng = np.random.default_rng(404)
    l, _ = _params_vary(rng, N, HW, C)
    l = l.reshape(N, H, W, 4 * C * K)
    sym = rng.integers(0, 256, (N, C, HW)).astype(np.uint8)
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


@pytest.mark.gpu
@pytest.mark.parametrize('spc', [1, 2, 4])
def test_varying_terms_decode_match_oracle(spc):
    from tests import test_gpu_coarse_rows as CR
    key, cs = _case()
    par = np.ascontiguousarray(cs['recs'][..., :64]).view(np.float32)        # the records' own parameters
    nv = vary_counts(par[..., K:2 * K], par[..., 2 * K:3 * K], cs['tg'].cpu().numpy())
    hit = np.take_along_axis(nv, (cs['sym'].astype(np.int64) >> 3)[..., None], -1)[..., 0]
    assert set(NV) <= set(np.unique(hit).tolist()), np.unique(hit)
    nan_pi = np.isnan(par[..., :K]).all(-1)
    assert 0 < nan_pi.mean() < 0.1, nan_pi.mean()
    assert (cs['rows'][nan_pi] == np.arange(256)).all()
    CR.test_coarse_decode_matches_oracle(key, spc)
