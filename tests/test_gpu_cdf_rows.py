"""CDF rows and coding intervals of the DMLL head, entry by entry against float64, and their codability.

Lossless coding rests on one property of the 16-bit CDF rows: every row is strictly increasing over its L entries,
so every symbol has an interval at least one count wide.  For finite parameters every step of an entry,
cdf[l] = F2I(scale * sum_k fma(pi_k, sigma(u_k), acc)) + l with u_k = (t_l - mu_k) * inv_s_k, is monotone except the
sigmoid itself, MUFU.RCP(1 + MUFU.EX2(u)), whose monotonicity the PTX ISA does not promise.

* GPU sweep (l3c_dmll_probe_sigmoid): every finite fp32 u, in magnitude order.  sigmoid_from_log2 is non-increasing
  across (-25, 40); mixture_term is exactly 1 at u <= -25 and 0 at u >= 40; the largest absolute error against
  float64 1 / (1 + 2^u) is within SIG_ABS, the bound the per-entry budget below uses.
* Restatement: each entry in float64 from the kernel's own fp32 parameters, with an error budget B for the sigmoid,
  the fma chain and the final multiplication.  Outside a band of width B around a half-integer the entry must equal
  rint(V) + l (rounded to 64 bits, as the reference's lrintf); an entry whose terms are all saturated or at u = 0
  (sigma exactly 1/2) must equal the fp32 in-order sum of those terms, bit for bit.  A CPU self-test pushes a numpy float32 emulation of the kernel to both ends of the sigmoid bound and checks that it stays
  inside the budget, and that the band holds only a small share of the entries.
* Every builder is held to the restatement: dmll_table_kernel (pitch 32 and 256, RGB with R/G coupling, non-RGB
  with C = 1 and 5), its pixel chunks, its tiled variant, the coarse records and dmll_intervals_kernel.
* Adversarial parameter families (wide components, clamped and infinite log-scales, far and infinite means,
  underflowing pi, sum(pi) above 1, NaN everywhere, inf * 0, saturated coupling) give strictly increasing rows,
  intervals of width >= 1 equal to the rows' differences, the oracle's stream bytes from the GPU encoder, and the
  symbols back from full rows, tiled rows, coarse records and l3c_decode_rgb_pipelined (full and coarse).
* The fused FP16 head (one-hot FP16 pixels, weight columns = parameter vectors, non-finite values in the fp32 bias)
  gives, bit for bit, the intervals of the restated rows of the parameters it sees.
* The torchac drop-in (l3c_*_logistic_mixture), on finite parameters with log-scales >= -7, writes the oracle's
  stream on the restated rows and decodes it."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ac

K = 10
SAT_LO, SAT_HI = np.float32(-25.0), np.float32(40.0)
LOG_SCALES_MIN = np.float32(-7.0)
NEG_LOG2E = np.float32(-1.4426950408889634)
# |sigmoid_from_log2(u) - 1 / (1 + 2^u)| on (-25, 40): the bound the budget uses; test_sigmoid_sweep measures it
# (1.159e-7 at u = -5.829 on an H100)
SIG_ABS = 1.25e-7
# relative error of the u the restatement recomputes from a log-scale (expf <= 2 ulp, then one rounding)
U_REL_EXPF = 2.0 ** -20


# ---------------------------------------------------------------------------------------------------------------------
# float64 restatement
# ---------------------------------------------------------------------------------------------------------------------
def f2i_rn(x):
    """cvt.rni.s32.f32 on float arrays: round half to even, NaN -> 0, saturating"""
    x = np.asarray(x, np.float64)
    with np.errstate(invalid='ignore'):
        r = np.rint(np.where(np.isnan(x), 0.0, np.clip(x, -2.0 ** 31, 2.0 ** 31 - 1)))
    return r.astype(np.int64)


def f2ll_rn(x):
    """the reference's lrintf (torchac_kernel.cu:20-24; on the device lrint of the float as a double, cvt.rni.s64) on
    float arrays: round half to even to a 64-bit integer, saturating at +-2^63, NaN -> 0 (INT64_MIN, what some
    conversions give instead, has the same low 16 bits)"""
    x = np.asarray(x, np.float64)
    with np.errstate(invalid='ignore'):
        r = np.rint(np.where(np.isnan(x), 0.0, x))
        hi, lo = r >= 2.0 ** 63, r < -2.0 ** 63
        out = np.where(hi | lo, 0.0, r).astype(np.int64)
    return np.where(hi, np.iinfo(np.int64).max, np.where(lo, np.iinfo(np.int64).min, out))


def u32(t, mu, inv_s):
    """u [R, L, K] exactly as the kernels compute it: f32(f32(t - mu) * inv_s)"""
    with np.errstate(invalid='ignore', over='ignore'):
        return (t[None, :, None] - mu[:, None, :]) * inv_s[:, None, :]


def restate(pi, mu, inv_s, t, L, u_rel=0.0, scale=None, rnd=f2ll_rn):
    """pi, mu, inv_s float32 [R, K]; t float32 [>= L] bin edges -> dict of int64 [R, L] arrays:
    lo / hi  the acceptable entries (equal outside the rounding band), already + l and mod 2^16
    band     entry inside the rounding band;  exact  every term saturated or at u = 0 (bit-exact fp32 sum)
    and V (float64, before + l).  u_rel > 0: inv_s is known only to that relative precision (recomputed from the
    log-scale), which widens the budget and makes threshold-straddling terms non-exact.  An entry is
    rnd(V) + l mod 2^16 with scale (default 65536 - L) and rnd the reference's rounding to 64 bits; a 32-bit one
    (f2i_rn) gives the same entries while |V| < 2^31, which holds wherever sum(pi) <= 1."""
    scale = np.float32(65536 - L if scale is None else scale)
    t = np.asarray(t[:L], np.float32)
    u = u32(t, mu, inv_s)
    lo_s, hi_s = u <= SAT_LO, u >= SAT_HI
    mid = ~(lo_s | hi_s)
    # sigma(0) is exactly 1/2 (test_sigmoid_sweep), and fma(pi, 1/2, acc) = fp32(acc + pi / 2) unless pi / 2 rounds
    with np.errstate(invalid='ignore'):
        zero = (u == 0) & ~((pi != 0) & (np.abs(pi) < np.float32(2.0 ** -125)))[:, None, :]
    l_idx = np.arange(L, dtype=np.int64)[None, :]
    # bit-exact path: in-order fp32 sum of the pi's saturated low and the halves of those at u = 0
    acc32 = np.zeros(u.shape[:2], np.float32)
    with np.errstate(invalid='ignore', over='ignore'):
        for k in range(pi.shape[-1]):
            acc32 = np.where(lo_s[..., k], acc32 + pi[:, None, k],
                             np.where(zero[..., k], acc32 + pi[:, None, k] * np.float32(0.5), acc32))
        sat_val = rnd(acc32 * scale) + l_idx
    # float64 value and budget
    pi64 = pi.astype(np.float64)[:, None, :]
    u64 = u.astype(np.float64)
    with np.errstate(invalid='ignore', over='ignore'):
        sig = 1.0 / (1.0 + np.exp2(u64))
        term = np.where(lo_s, pi64, np.where(mid, pi64 * sig, 0.0))
    A = np.cumsum(term, axis=-1)                          # the accumulator after each term
    V = float(scale) * A[..., -1]
    with np.errstate(invalid='ignore', over='ignore'):
        # half an ulp of every fma result (terms saturated high add nothing, round nothing)
        half_ulp = 0.5 * np.spacing(np.abs(A * (1 + 1e-6)).astype(np.float32)).astype(np.float64)
        fma_err = np.where(hi_s, 0.0, half_ulp).sum(-1)
        sig_err = np.where(mid, np.abs(pi64), 0.0).sum(-1) * SIG_ABS
        B = float(scale) * (sig_err + fma_err) + 0.5 * np.spacing(np.abs(V).astype(np.float32)).astype(np.float64)
        straddle = np.zeros(V.shape, bool)
        if u_rel:
            # sigma moves by |sigma'(u)| |du| (sigma' = -ln2 sigma (1 - sigma)); a term within u_rel of a threshold
            # may be classified the other way, which moves it by < pi 2^-24
            du = np.abs(u64) * u_rel
            B += float(scale) * np.where(mid, np.abs(pi64) * np.log(2) * sig * (1 - sig) * du, 0.0).sum(-1)
            near = (np.abs(u64 - float(SAT_LO)) <= np.abs(u64) * u_rel) | \
                   (np.abs(u64 - float(SAT_HI)) <= np.abs(u64) * u_rel)
            straddle = near.any(-1)
            B += float(scale) * np.where(near, np.abs(pi64) * 2.0 ** -24, 0.0).sum(-1)
        B = B * 1.01 + 1e-9
        frac = V - np.floor(V)
        band = np.isfinite(V) & (np.abs(frac - 0.5) <= B)
    exact = ~(mid & ~zero).any(-1) & ~straddle
    assert not (np.isfinite(B) & (B >= 0.25) & ~exact).any(), 'budget too wide to decide an entry'
    r = rnd(V)
    lo = np.where(band, rnd(np.floor(V)), r) + l_idx
    hi = np.where(band, rnd(np.ceil(V)), r) + l_idx
    lo_raw, hi_raw = np.where(exact, sat_val, lo), np.where(exact, sat_val, hi)     # before the 16-bit wrap
    return dict(lo=lo_raw & 0xFFFF, hi=hi_raw & 0xFFFF, lo_raw=lo_raw, hi_raw=hi_raw, band=band & ~exact,
                exact=exact, V=V, u=u)


def check_rows(rows, ref, what, l_idx=None):
    """rows uint16/int64 [R, n] must be one of the two acceptable entries everywhere; l_idx: the entries' indices
    (default 0..n-1).  -> shares of the unsaturated entries in the band and off rint(V)"""
    rows = rows.astype(np.int64)
    l_idx = np.arange(rows.shape[1]) if l_idx is None else l_idx
    ok = (rows == ref['lo']) | (rows == ref['hi'])
    bad = np.argwhere(~ok)
    if bad.size:
        r, e = bad[0]
        raise AssertionError('%s: %d of %d entries outside the float64 restatement; first row %d entry %d: got %d, '
                             'want %d..%d (V = %.6f, exact %s)' % (what, len(bad), ok.size, r, e, rows[r, e],
                                                                  ref['lo'][r, e], ref['hi'][r, e], ref['V'][r, e],
                                                                  ref['exact'][r, e]))
    unsat = ~ref['exact']
    n_un = max(int(unsat.sum()), 1)
    off = unsat & (rows != (f2ll_rn(ref['V']) + l_idx) & 0xFFFF)
    return dict(band=float(ref['band'].sum()) / n_un, off_rint=float(off.sum()) / n_un, unsat=int(unsat.sum()))


def emulate(pi, mu, inv_s, t, L, sig_push, rnd=f2i_rn):
    """numpy float32 model of mixture_cdf_u16 (rnd = f2ll_rn: plane_cdf_u16) with the sigmoid replaced by
    sigma64 + sig_push (each term's push in [-1, 1] x SIG_ABS, rounded to fp32 and kept within SIG_ABS of sigma64;
    exactly 1 at u <= -25 and 1/2 at u = 0): [R, L] entries (+ l, mod 2^16)"""
    scale = np.float32(65536 - L)
    u = u32(np.asarray(t[:L], np.float32), mu, inv_s)
    with np.errstate(invalid='ignore', over='ignore'):
        s64 = 1.0 / (1.0 + np.exp2(u.astype(np.float64)))
        s32 = (s64 + sig_push * SIG_ABS).astype(np.float32)
        s32 = np.where(np.abs(s32 - s64) > SIG_ABS, np.nextafter(s32, s64.astype(np.float32)), s32)
        s32 = np.where(s32 > 0, s32, s64.astype(np.float32))          # the sigmoid is positive below u = 40
        s32 = np.where(u <= SAT_LO, np.float32(1), np.where(u == 0, np.float32(0.5), s32))
        acc = np.zeros(u.shape[:2], np.float32)
        for k in range(pi.shape[-1]):
            f = (pi[:, None, k].astype(np.float64) * s32[..., k] + acc.astype(np.float64)).astype(np.float32)
            f = np.where((u[..., k] <= SAT_LO) | (u[..., k] == 0), acc + pi[:, None, k] * s32[..., k], f)
            acc = np.where(u[..., k] >= SAT_HI, acc, f)
        return (rnd(acc * scale) + np.arange(L)[None, :]) & 0xFFFF


def inv_s_from_logs(logs):
    """-log2(e) / sigma from the raw log-scales, as channel_params computes it (expf to within 2 ulp)"""
    with np.errstate(over='ignore', invalid='ignore'):
        ls = np.fmax(logs.astype(np.float32), LOG_SCALES_MIN)
        return np.exp(-ls.astype(np.float64)).astype(np.float32) * NEG_LOG2E


# ---------------------------------------------------------------------------------------------------------------------
# parameters
# ---------------------------------------------------------------------------------------------------------------------
def _grid(rgb, L):
    """(x_min, x_max) of the value grid and its float32 bin edges (DiscretizedMixLogisticLoss.targets)"""
    from l3c_pytorch_b200.dmll import DiscretizedMixLogisticLoss
    x0, x1 = (0, 255) if rgb else (-1, 1)
    return x0, x1, DiscretizedMixLogisticLoss(rgb, x0, x1, L).targets('cpu').numpy()


def _trained_like(rng, N, HW, C, rgb, x0, x1, L):
    """l [N, HW, Kp]: one dominant narrow component per sub-pixel, or broad random-init-like mixtures"""
    bw = (x1 - x0) / (L - 1)
    shp = (N, HW, C, K)
    logit = rng.normal(0, 1, shp)
    mean = rng.uniform(x0 - 0.2 * (x1 - x0), x1 + 0.2 * (x1 - x0), shp)
    logs = np.log(bw) + rng.uniform(-4, 3, shp)
    dom = rng.integers(0, K, (N, HW, C, 1))
    np.put_along_axis(logit, dom, rng.uniform(3, 10, dom.shape), axis=3)
    parts = [logit, mean, logs]
    if rgb:
        parts.append(rng.normal(0, 2, shp))
    return np.stack(parts, axis=2).reshape(N, HW, len(parts) * C * K).astype(np.float32)


def _symbols(rng, N, C, HW, L):
    s = rng.integers(0, L, (N, C, HW))
    s[..., 0], s[..., -1] = 0, L - 1
    return s.astype(np.uint8)


class Built:
    """rows of every channel from dmll_table_kernel, plus the kernel's pi / mu (dmll_channel_params)"""

    def __init__(self, l, sym, rgb, C, L, H, W):
        from l3c_pytorch_b200 import engine as E
        self.dev = torch.device('cuda')
        self.l_np, self.sym, self.rgb, self.C, self.L, self.H, self.W = l, sym, rgb, C, L, H, W
        self.N, self.HW = l.shape[0], H * W
        self.x0, self.x1, self.t = _grid(rgb, L)
        self.tg = torch.from_numpy(self.t).to(self.dev)
        self.l = torch.from_numpy(l.reshape(self.N, H, W, -1)).to(self.dev)
        self.sym_dev = torch.from_numpy(sym.reshape(self.N, C, H, W)).to(self.dev)
        self.pitch = E.table_pitch(L)
        table = torch.zeros(self.N * C * self.HW * self.pitch, dtype=torch.int16, device=self.dev)
        for c in (range(C) if rgb else [-1]):
            E.dmll_build_table(self.l, self.sym_dev, self.tg, C, K, L, rgb, c, table)
        self.table = table
        self.rows = table.cpu().numpy().view(np.uint16).reshape(self.N, C, self.HW, self.pitch)[..., :L]
        x_dec = self.sym_dev.float().contiguous()
        self.pi, self.mu = [], []
        for c in range(C):
            pi, mu, _ = E.dmll_channel_params(self.l, x_dec, C, K, rgb, c)
            self.pi.append(pi.cpu().numpy().reshape(self.N, K, self.HW).transpose(0, 2, 1))
            self.mu.append(mu.cpu().numpy().reshape(self.N, K, self.HW).transpose(0, 2, 1))
        torch.cuda.synchronize()

    def logs(self, c):
        C, P = self.C, self.l_np.shape[-1]
        return self.l_np.reshape(self.N, self.HW, P)[..., 2 * C * K + c * K: 2 * C * K + (c + 1) * K]

    def restate(self, c, inv_s=None):
        """restatement of channel c's rows, [N * HW, L]; inv_s exact (coarse records) or recomputed"""
        pi = self.pi[c].reshape(-1, K)
        mu = self.mu[c].reshape(-1, K)
        if inv_s is None:
            return restate(pi, mu, inv_s_from_logs(self.logs(c)).reshape(-1, K), self.t, self.L, U_REL_EXPF)
        return restate(pi, mu, inv_s.reshape(-1, K), self.t, self.L)

    def coarse(self):
        from l3c_pytorch_b200 import engine as E
        rec = torch.zeros(self.N * 3 * self.HW * E.COARSE_PITCH, dtype=torch.int16, device=self.dev)
        for c in range(3):
            E.dmll_build_coarse(self.l, self.sym_dev, self.tg, K, self.L, c, rec)
        torch.cuda.synchronize()
        return rec, rec.cpu().numpy().view(np.uint16).reshape(self.N, 3, self.HW, E.COARSE_PITCH)


def _rec_params(recs, c):
    w = np.ascontiguousarray(recs[:, c, :, :64]).view(np.float32)       # [N, HW, 32]
    return w[..., :K], w[..., K:2 * K], w[..., 2 * K:3 * K], w[..., 3 * K:]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the budget holds the emulated kernel, and is tight enough to mean something
# ---------------------------------------------------------------------------------------------------------------------
def _host_params(rng, R, rgb, L):
    x0, x1, t = _grid(rgb, L)
    l = _trained_like(rng, 1, R, 1, False, x0, x1, L)[0]
    logit, mean, logs = l[:, :K], l[:, K:2 * K], l[:, 2 * K:3 * K]
    logs[:R // 3] = np.log((x1 - x0) / (L - 1)) + rng.uniform(-7, -3, (R // 3, K))     # narrow: mostly saturated
    e = np.exp(logit.astype(np.float64) - logit.max(1, keepdims=True))
    pi = (e / e.sum(1, keepdims=True)).astype(np.float32)
    return pi, mean.astype(np.float32), inv_s_from_logs(logs), t


@pytest.mark.parametrize('L', [2, 25, 256])
def test_budget_holds_emulated_kernel(L):
    rng = np.random.default_rng(11 + L)
    R = 1500 if L == 256 else 6000
    pi, mu, inv_s, t = _host_params(rng, R, L == 256, L)
    # plus rows with u exactly on the thresholds and sum(pi) above 1
    pi[:50] = np.float32(0.1)
    ref = restate(pi, mu, inv_s, t, L)
    pushes = [np.ones((R, L, K)), -np.ones((R, L, K)), rng.choice([-1.0, 1.0], (R, L, K)), rng.uniform(-1, 1, (R, L, K))]
    for push in pushes:
        got = emulate(pi, mu, inv_s, t, L, push)
        check_rows(got, ref, 'emulation, L=%d' % L)
    st = check_rows(emulate(pi, mu, inv_s, t, L, np.zeros((R, L, K))), ref, 'emulation')
    print('L=%d: %d unsaturated entries, %.2f %% in the rounding band, %.2f %% off rint(V) at sigma64'
          % (L, st['unsat'], 100 * st['band'], 100 * st['off_rint']))
    assert st['unsat'] > 0.2 * R * L, 'the parameters must exercise the transcendental path'
    assert st['band'] < 0.08, 'the budget must decide most entries: %.3f in the band' % st['band']
    # the bit-exact saturated path is taken, and an emulation that drops a low-saturated pi is caught
    assert ref['exact'].mean() > 0.05
    bad = emulate(pi, mu, inv_s, t, L, np.zeros((R, L, K)))
    bad = np.where(ref['exact'] & (ref['lo'] != 0), (bad + 1) & 0xFFFF, bad)
    with pytest.raises(AssertionError):
        check_rows(bad, ref, 'fault')


def test_budget_catches_a_shifted_sigmoid():
    """an emulation whose sigmoid is off by 4 x SIG_ABS leaves the budget somewhere"""
    rng = np.random.default_rng(5)
    pi, mu, inv_s, t = _host_params(rng, 2000, True, 256)
    ref = restate(pi, mu, inv_s, t, 256)
    with pytest.raises(AssertionError):
        check_rows(emulate(pi, mu, inv_s, t, 256, np.full((2000, 256, K), 4.0)), ref, 'shifted')


def tile_order_to_raster_py(H, W, th, tw):
    """raster pixel of every tile-order position, written out tile by tile"""
    out = []
    for ty in range(0, H, th):
        for tx in range(0, W, tw):
            for y in range(ty, min(ty + th, H)):
                for x in range(tx, min(tx + tw, W)):
                    out.append(y * W + x)
    return np.array(out, np.int64)


def test_tile_order_restatement_is_a_permutation():
    for H, W, th, tw in [(7, 11, 3, 4), (5, 6, 1, 1), (4, 5, 9, 13), (6, 9, 6, 2)]:
        p = tile_order_to_raster_py(H, W, th, tw)
        assert sorted(p.tolist()) == list(range(H * W))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the sigmoid, every finite fp32 argument
# ---------------------------------------------------------------------------------------------------------------------
CHUNK = 1 << 26
MAX_FINITE_BITS = 0x7F7FFFFF


def _probe(u):
    from l3c_pytorch_b200 import _lib, engine as E
    raw, term = torch.empty_like(u), torch.empty_like(u)
    _lib.check(_lib.lib.l3c_dmll_probe_sigmoid(ctypes.c_void_p(u.data_ptr()), ctypes.c_void_p(raw.data_ptr()),
                                               ctypes.c_void_p(term.data_ptr()), u.numel(), E._stream_ptr()))
    return raw, term


@pytest.mark.gpu
def test_sigmoid_sweep():
    dev = torch.device('cuda')
    rises, n_rises = [], 0
    max_abs, max_rel, at_abs, at_rel = 0.0, 0.0, None, None
    max_hi, n_seen = 0.0, 0
    for neg in (False, True):
        prev = None                                   # last raw inside (-25, 40), carried across chunks
        for start in range(0, MAX_FINITE_BITS + 1, CHUNK):
            bits = torch.arange(start, min(start + CHUNK, MAX_FINITE_BITS + 1), dtype=torch.int32, device=dev)
            if neg:
                bits = bits | torch.tensor(-2 ** 31, dtype=torch.int32, device=dev)
            u = bits.view(torch.float32)              # increasing magnitude
            n_seen += u.numel()
            raw, term = _probe(u)
            lo, hi = u <= -25.0, u >= 40.0
            mid = ~(lo | hi)
            if lo.any():
                assert bool((raw[lo] == 1).all()) and bool((term[lo] == 1).all()), 'u <= -25 must give exactly 1'
            if hi.any():
                assert bool((term[hi] == 0).all()), 'u >= 40 must add nothing'
                max_hi = max(max_hi, float(raw[hi].max()))
            if not mid.any():
                continue
            # (-25, 40) is a prefix of either magnitude-ordered sweep
            um, rm = u[mid], raw[mid]
            assert bool((term[mid] == rm).all()), 'mixture_term(0, 1, u) must be the raw sigmoid inside (-25, 40)'
            seq = torch.cat([prev, rm]) if prev is not None else rm
            useq = torch.cat([prev_u, um]) if prev is not None else um
            d = seq[1:] - seq[:-1]
            bad = (d < 0) if neg else (d > 0)         # away from 0: raw falls for u > 0, rises for u < 0
            if bad.any():
                idx = torch.nonzero(bad).flatten()
                n_rises += idx.numel()
                for i in idx[:50].tolist():
                    rises.append((float(useq[i]), float(useq[i + 1]), float(seq[i]), float(seq[i + 1])))
            prev, prev_u = rm[-1:], um[-1:]
            ref = 1.0 / (1.0 + torch.exp2(um.double()))
            err = (rm.double() - ref).abs()
            rel = err / ref
            i, j = int(err.argmax()), int(rel.argmax())
            if float(err[i]) > max_abs:
                max_abs, at_abs = float(err[i]), float(um[i])
            if float(rel[j]) > max_rel:
                max_rel, at_rel = float(rel[j]), float(um[j])
            del bits, u, raw, term, ref, err, rel
    assert n_seen == 2 * (MAX_FINITE_BITS + 1), n_seen       # every finite fp32 value, +0 and -0 included
    ends = torch.tensor([float('-inf'), float('inf'), 0.0, -0.0], device=dev)
    raw, term = _probe(ends)
    assert raw.tolist() == [1.0, 0.0, 0.5, 0.5] and term.tolist() == [1.0, 0.0, 0.5, 0.5]
    print('sigmoid_from_log2 over every finite fp32 u: %s; max |err| %.3e at u = %.9g, max rel err %.3e at u = %.9g, '
          'largest raw at u >= 40: %.6e (2^-40 = %.6e)'
          % ('monotone' if n_rises == 0 else '%d rises' % n_rises, max_abs, at_abs, max_rel, at_rel, max_hi,
             2.0 ** -40))
    assert n_rises == 0, 'sigmoid_from_log2 is not monotone: %d rises, e.g. (u0, u1, raw0, raw1) %s' % (n_rises,
                                                                                                     rises[:20])
    assert max_abs <= SIG_ABS, 'sigmoid error %.3e exceeds the budget\'s SIG_ABS %.1e' % (max_abs, SIG_ABS)
    assert max_hi <= 2.0 ** -40 * (1 + 2.0 ** -20)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: every builder against the restatement
# ---------------------------------------------------------------------------------------------------------------------
GRIDS = [  # (rgb, C, L)
    (False, 1, 2), (False, 5, 25), (False, 1, 32),
    (False, 5, 33), (False, 1, 100), (False, 5, 255), (False, 1, 256), (True, 3, 256)]
_BUILT = {}


def _built(rgb, C, L, H=9, W=31, N=2):
    key = (rgb, C, L, H, W, N)
    if key not in _BUILT:
        rng = np.random.default_rng(1000 + 7 * L + C + int(rgb))
        x0, x1, _ = _grid(rgb, L)
        l = _trained_like(rng, N, H * W, C, rgb, x0, x1, L)
        _BUILT[key] = Built(l, _symbols(rng, N, C, H * W, L), rgb, C, L, H, W)
    return _BUILT[key]


@pytest.mark.gpu
@pytest.mark.parametrize('rgb,C,L', GRIDS)
def test_table_rows_vs_restatement(rgb, C, L):
    b = _built(rgb, C, L)
    if rgb:
        _, recs = b.coarse()
    for c in range(C):
        if rgb:
            pi, mu, inv_s, pad = _rec_params(recs, c)
            assert (pi.view(np.uint32) == b.pi[c].view(np.uint32)).all(), 'record pi != dmll_channel_params'
            assert (mu.view(np.uint32) == b.mu[c].view(np.uint32)).all(), 'record mu != dmll_channel_params'
            assert (pad == 0).all()
            ref = b.restate(c, inv_s)
        else:
            ref = b.restate(c)
        st = check_rows(b.rows[:, c].reshape(-1, L), ref, 'dmll_table_kernel rgb=%d C=%d L=%d c=%d' % (rgb, C, L, c))
        print('rgb=%d C=%d L=%d c=%d: %d unsaturated entries, %.2f %% in the band, %.2f %% differ from rint(V)'
              % (rgb, C, L, c, st['unsat'], 100 * st['band'], 100 * st['off_rint']))
        assert st['unsat'] > 0
    # the unused tail of a pitch-32 / pitch-256 row is zero
    tail = b.table.cpu().numpy().view(np.uint16).reshape(b.N, C, b.HW, b.pitch)[..., L:]
    assert (tail == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize('rgb,C,L', [(True, 3, 256), (False, 5, 25), (False, 1, 100)])
def test_table_chunks_equal_one_launch(rgb, C, L):
    from l3c_pytorch_b200 import engine as E
    b = _built(rgb, C, L, H=20, W=31)
    for chunk in (1, 255, 256, 257):
        table = torch.full((b.N * C * b.HW * b.pitch,), -1, dtype=torch.int16, device=b.dev)
        for p0 in range(0, b.HW, chunk):
            for c in (range(C) if rgb else [-1]):
                E.dmll_build_table(b.l, b.sym_dev, b.tg, C, K, L, rgb, c, table, pix0=p0, npix=min(chunk, b.HW - p0))
        got = table.cpu().numpy().view(np.uint16).reshape(b.N, C, b.HW, b.pitch)[..., :L]
        bad = np.argwhere(got != b.rows)
        assert bad.size == 0, 'chunk %d: %d entries differ from one launch, first at %s' % (chunk, len(bad), bad[0])


@pytest.mark.gpu
@pytest.mark.parametrize('tile', [(2, 5), (3, 4), (1, 1), (9, 31), (40, 50), (4, 31), (9, 7)])
@pytest.mark.parametrize('rgb,C,L', [(True, 3, 256), (False, 5, 25)])
def test_tiled_rows_are_raster_rows(rgb, C, L, tile):
    from l3c_pytorch_b200 import engine as E
    b = _built(rgb, C, L)
    perm = tile_order_to_raster_py(b.H, b.W, *tile)
    sym_t = torch.from_numpy(np.ascontiguousarray(b.sym[..., perm])).to(b.dev)
    table = torch.full((b.N * C * b.HW * b.pitch,), -1, dtype=torch.int16, device=b.dev)
    for c in (range(C) if rgb else [-1]):
        E.dmll_build_table_tiled(b.l, sym_t, b.tg, C, K, L, rgb, c, table, tile)
    got = table.cpu().numpy().view(np.uint16).reshape(b.N, C, b.HW, b.pitch)[..., :L]
    bad = np.argwhere(got != b.rows[:, :, perm])
    assert bad.size == 0, 'tile %s: %d entries differ from the raster row, first at %s' % (tile, len(bad), bad[0])


@pytest.mark.gpu
def test_coarse_entries_vs_restatement():
    b = _built(True, 3, 256)
    _, recs = b.coarse()
    for c in range(3):
        pi, mu, inv_s, _ = _rec_params(recs, c)
        ref = b.restate(c, inv_s)
        sub = {k: ref[k][:, ::8] for k in ('lo', 'hi', 'band', 'exact', 'V')}
        st = check_rows(recs[:, c, :, 64:96].reshape(-1, 32), sub, 'coarse records c=%d' % c, np.arange(0, 256, 8))
        assert (recs[:, c, :, 64:96] == b.rows[:, c, :, ::8]).all()
        print('coarse c=%d: %.2f %% of unsaturated entries in the band' % (c, 100 * st['band']))


def _row_intervals(rows, sym):
    """[N, C, HW] uint32 interval lo | (hi - 1) << 16 of every coded symbol, from the rows"""
    s = sym.astype(np.int64)
    lo = np.take_along_axis(rows.astype(np.int64), s[..., None], -1)[..., 0]
    nxt = np.take_along_axis(rows.astype(np.int64), np.minimum(s + 1, rows.shape[-1] - 1)[..., None], -1)[..., 0]
    hi = np.where(s == rows.shape[-1] - 1, 65536, nxt)
    return lo, hi, (lo | ((hi - 1) << 16)).astype(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize('rgb,C,L', [(True, 3, 256), (False, 5, 25), (False, 1, 2), (False, 5, 255)])
def test_intervals_kernel_vs_rows(rgb, C, L):
    from l3c_pytorch_b200 import engine as E
    b = _built(rgb, C, L)
    iv = E.dmll_intervals(b.l, b.sym_dev, b.tg, C, K, L, rgb).cpu().numpy().view(np.uint32)
    _, _, want = _row_intervals(b.rows, b.sym)
    bad = np.argwhere(iv != want)
    assert bad.size == 0, '%d intervals differ from the rows, first at %s' % (len(bad), bad[0])


# ---------------------------------------------------------------------------------------------------------------------
# GPU: codability on adversarial parameters
# ---------------------------------------------------------------------------------------------------------------------
FAMILIES = ('wide', 'clamp', 'far', 'pi_underflow', 'sum_pi', 'nan', 'coupling', 'trained')
FH, FW, FN = 8, 32, 2


def _pidx(P, C, p, c, k):
    """index of parameter kind p (0 logit, 1 mean, 2 log-scale, 3 coupling block c) of channel c, component k"""
    return p * C * K + c * K + k


def _family(name, rgb, C, L, rng):
    """l [N, HW, Kp] float32, symbols, and the mask [N, HW, C] of the sub-pixels put into the family's regime"""
    HW = FH * FW
    x0, x1, _ = _grid(rgb, L)
    l = _trained_like(rng, FN, HW, C, rgb, x0, x1, L).reshape(FN, HW, -1, C, K)
    sym = _symbols(rng, FN, C, HW, L)
    sel = rng.random((FN, HW, C)) < 0.5
    logit, mean, logs = l[:, :, 0], l[:, :, 1], l[:, :, 2]

    def put(arr, vals):
        v = rng.choice(np.asarray(vals, np.float32), arr.shape)
        arr[sel] = v[sel]

    if name == 'wide':
        put(logs, np.concatenate([np.linspace(8, 20, 13), [np.inf]]))
    elif name == 'clamp':
        put(logs, [-7, -30, -1e30, -np.inf])
    elif name == 'far':
        put(mean, [1e6, -1e6, 3e38, -3e38, np.inf, -np.inf])
    elif name == 'pi_underflow':
        spread = rng.uniform(104, 400, logit.shape).astype(np.float32)
        logit[sel] = -spread[sel]
        logit[..., 0][sel] = 0
        extra = rng.random(sel.shape) < 0.3
        logit[..., 1][sel & extra] = rng.choice(np.float32([1e30, -1e30, np.inf, -np.inf]), (sel & extra).sum())
    elif name == 'sum_pi':
        logit[sel] = 0
        near = sel & (rng.random(sel.shape) < 0.5)
        logit[near] = rng.uniform(-1e-6, 1e-6, (near.sum(), K)).astype(np.float32)
    elif name == 'nan':
        for arr in (logit, mean, logs) + ((l[:, :, 3],) if rgb else ()):
            pick = sel & (rng.random(sel.shape) < 0.25)
            k = rng.integers(0, K, pick.sum())
            sub = arr[pick]
            sub[np.arange(len(k)), k] = np.nan
            arr[pick] = sub
        # inf * 0: an infinite mean under an infinite log-scale (inv_s = -0) makes u NaN at every target
        pick = sel & (rng.random(sel.shape) < 0.2)
        k = rng.integers(0, K, pick.sum())
        for arr, v in ((mean, rng.choice(np.float32([np.inf, -np.inf]), len(k))), (logs, np.float32(np.inf))):
            sub = arr[pick]
            sub[np.arange(len(k)), k] = v
            arr[pick] = sub
    elif name == 'coupling' and rgb:
        put(l[:, :, 3], [88, -88, np.inf, -np.inf, np.nan])
        edge = rng.random((FN, HW)) < 0.6
        sym[:, 0][edge] = rng.choice([0, 255], edge.sum())
        sym[:, 1][edge] = rng.choice([0, 255], edge.sum())
    elif name == 'coupling':
        sel[:] = False
    return np.ascontiguousarray(l.reshape(FN, HW, -1)), sym, sel


def _regimes(name, l, rgb, C, sel, b):
    """{sub-case: number of sub-pixels (or channels) in it}; every sub-case must be reached"""
    N, HW = l.shape[:2]
    P = 4 if rgb else 3
    q = l.reshape(N, HW, P, C, K)
    logit, mean, logs = q[:, :, 0], q[:, :, 1], q[:, :, 2]

    def has(arr, pred):
        with np.errstate(invalid='ignore'):
            return int((sel & pred(arr).any(-1)).sum())

    if name == 'wide':
        u_mid = [((b.ref[c]['u'] > SAT_LO) & (b.ref[c]['u'] < SAT_HI)).all((-1, -2)).reshape(N, HW) for c in range(C)]
        return {'no term saturated in the row': int((sel & np.stack(u_mid, -1)).sum()),
                'log-scale +inf': has(logs, np.isposinf), 'log-scale >= 8': has(logs, lambda a: a >= 8)}
    if name == 'clamp':
        return {'log-scale %g' % v: has(logs, lambda a, v=v: a == np.float32(v)) for v in (-7, -30, -1e30, -np.inf)}
    if name == 'far':
        return {'mean %g' % v: has(mean, lambda a, v=v: a == np.float32(v))
                for v in (1e6, -1e6, 3e38, -3e38, np.inf, -np.inf)}
    if name == 'pi_underflow':
        out = {'pi == 0': int((sel & np.stack([(b.pi[c] == 0).any(-1) for c in range(C)], -1)).sum())}
        out.update({'logit %g' % v: has(logit, lambda a, v=v: a == np.float32(v)) for v in (1e30, -1e30, np.inf,
                                                                                           -np.inf)})
        return out
    if name == 'sum_pi':
        return {'fp32 sum(pi) > 1': int((sel & np.stack([b.pi[c].sum(-1, dtype=np.float32) > 1 for c in range(C)],
                                                       -1)).sum())}
    if name == 'nan':
        out = {'NaN logit': has(logit, np.isnan), 'NaN mean': has(mean, np.isnan), 'NaN log-scale': has(logs, np.isnan),
               'inf mean under +inf log-scale': int((sel & (np.isinf(mean) & np.isposinf(logs)).any(-1)).sum())}
        if rgb:
            out['NaN coupling coefficient'] = has(q[:, :, 3], np.isnan)
        return out
    if name == 'coupling':
        co = q[:, :, 3]                               # [N, HW, 3 coefficient blocks, K]
        out = {'coefficient %g' % v: has(co, lambda a, v=v: a == np.float32(v)) for v in (88, -88, np.inf, -np.inf)}
        out['coefficient NaN'] = has(co, np.isnan)
        out['R and G at 0 or 255'] = int(((b.sym[:, 0] % 255 == 0) & (b.sym[:, 1] % 255 == 0)).sum())
        return out
    return {'trained-like': int(sel.sum())}


def _fused_bias(name, rgb, C):
    """fp32 bias of the fused head's 1x1 conv: the non-finite and out-of-FP16-range values of each family, one per
    parameter channel (the one-hot FP16 weight columns carry the finite per-pixel parts)"""
    P = 4 if rgb else 3
    b = np.zeros(P * C * K, np.float32)
    pi = lambda p, c, k: _pidx(P, C, p, c, k)        # noqa: E731
    if name == 'wide':
        for c in range(C):
            b[pi(2, c, 0)] = np.inf
    elif name == 'clamp':
        for c in range(C):
            b[pi(2, c, 1)], b[pi(2, c, 2)], b[pi(2, c, 3)] = -np.inf, -1e30, -30
    elif name == 'far':
        for c in range(C):
            b[pi(1, c, 0)], b[pi(1, c, 1)], b[pi(1, c, 2)], b[pi(1, c, 3)] = np.inf, -np.inf, 3e38, -1e6
    elif name == 'pi_underflow':
        for c in range(C):
            b[pi(0, c, 1)], b[pi(0, c, 2)] = -np.inf, -1e30
    elif name == 'nan':
        b[pi(0, 0, 4)] = np.nan                                            # NaN logit: channel 0 is the ramp row
        b[pi(1, 1, 6)] = np.inf                                            # inf mean under
        b[pi(2, 1, 6)] = np.inf                                            # a +inf log-scale: channel 1 is the ramp
        if rgb:
            b[_pidx(P, C, 3, 1, 2)] = np.nan                               # NaN coefficient: channel 2 is the ramp
        else:
            b[pi(2, 2, 3)] = np.nan                                        # NaN log-scale: clamped, not a ramp
            b[pi(1, 3, 0)] = np.nan                                        # NaN mean: channel 3 is the ramp
    elif name == 'coupling' and rgb:
        b[_pidx(P, C, 3, 0, 0)], b[_pidx(P, C, 3, 1, 1)], b[_pidx(P, C, 3, 2, 2)] = np.inf, -np.inf, np.nan
    return b


FUSED_CIN = 192


def _fused_head(name, l, sym, rgb, C, L, H, W):
    """drive l3c_lin_dmll_intervals with one-hot FP16 pixels: pixel i of the batch selects weight column i % 192,
    set to the FP16 value of the i-th parameter vector (0 where it is not finite or beyond FP16), plus the family's
    fp32 bias.  -> (the parameters the head sees, fp32 [N, HW, Kp], its intervals [N, C, HW] uint32)"""
    from l3c_pytorch_b200 import engine as E
    dev = torch.device('cuda')
    N, HW, Kp = l.shape
    flat = l.reshape(-1, Kp)
    cols = np.resize(np.arange(flat.shape[0]), FUSED_CIN)              # column j = vector j (cycled if fewer)
    with np.errstate(invalid='ignore'):
        wv = np.where(np.isfinite(flat[cols]) & (np.abs(flat[cols]) <= 65504), flat[cols], 0).astype(np.float16)
    bias = _fused_bias(name, rgb, C)
    conv = torch.nn.Conv2d(FUSED_CIN, Kp, 1).to(dev)
    with torch.no_grad():
        conv.weight.copy_(torch.from_numpy(wv.T.astype(np.float32)).reshape(Kp, FUSED_CIN, 1, 1))
        conv.bias.copy_(torch.from_numpy(bias))
    j = np.arange(N * HW) % FUSED_CIN
    x = np.zeros((N * HW, FUSED_CIN), np.float16)
    x[np.arange(N * HW), j] = 1
    cat = torch.from_numpy(x.reshape(N, H, W, FUSED_CIN)).to(dev)
    with np.errstate(invalid='ignore', over='ignore'):
        l_eff = (wv[j].astype(np.float32) + bias[None]).reshape(N, HW, Kp)
    sym_dev = torch.from_numpy(sym.reshape(N, C, H, W)).to(dev)
    _, _, tg = _grid(rgb, L)
    iv = E.lin_dmll_intervals(conv, cat, sym_dev, torch.from_numpy(tg).to(dev), C, K, L, rgb)
    return np.ascontiguousarray(l_eff), iv.cpu().numpy().view(np.uint32)


def _check_codable(b, what):
    """strict increase, restatement (exact inv_s from the coarse records on the RGB scale), ramp rows where a term is
    NaN at every target; stores the restatements in b.ref"""
    rows = b.rows.astype(np.int64)
    bad = np.argwhere(np.diff(rows, axis=-1) < 1)
    assert bad.size == 0, '%s: %d empty intervals, first at (n, c, p, l) = %s' % (what, len(bad), bad[0])
    if b.rgb:
        b.rec_t, b.recs = b.coarse()
    b.ref = []
    for c in range(b.C):
        ref = b.restate(c, _rec_params(b.recs, c)[2] if b.rgb else None)
        check_rows(b.rows[:, c].reshape(-1, b.L), ref, '%s c=%d' % (what, c))
        b.ref.append(ref)
        # a NaN pi or mu, or u NaN at every target (inf * 0), gives the ramp row cdf[l] = l
        ramp = (b.rows[:, c] == np.arange(b.L)).all(-1).reshape(-1)
        nan_all = np.isnan(ref['u']).all(1).any(-1) | np.isnan(b.pi[c].reshape(-1, K)).any(-1) | \
            np.isnan(b.mu[c].reshape(-1, K)).any(-1)
        assert ramp[nan_all].all(), '%s c=%d: %d NaN rows are not the ramp' % (what, c, int((~ramp[nan_all]).sum()))
        b.n_ramp = getattr(b, 'n_ramp', 0) + int(nan_all.sum())


def _encode(b, sym, iv):
    """GPU-encode one stream per (image, channel) from the intervals; each must be the oracle's bytes on the rows"""
    from l3c_pytorch_b200 import _lib, engine as E
    N, C, HW = b.N, b.C, b.HW
    n_st = N * C
    iv_dev = torch.from_numpy(iv.reshape(-1).view(np.int32)).to(b.dev)
    cap = ((HW * 17 + 7) // 8 + 64 + 3) & ~3
    slots = torch.zeros(n_st * cap, dtype=torch.uint8, device=b.dev)
    desc = np.zeros(n_st, dtype=_lib.ENC_STREAM_DTYPE)
    desc['intervals'] = iv_dev.data_ptr() + 4 * HW * np.arange(n_st)
    desc['out'] = slots.data_ptr() + cap * np.arange(n_st)
    desc['n_sym'] = HW
    desc['out_cap'] = cap
    _, lens_dev = E.ac_encode_streams(desc, b.dev)
    lens = lens_dev.cpu().numpy()
    hb = slots.cpu().numpy()
    streams = []
    for n in range(N):
        for c in range(C):
            i = n * C + c
            want = ac.encode(np.concatenate([b.rows[n, c], np.zeros((HW, 1), np.uint16)], 1), sym[n, c])
            assert hb[i * cap:i * cap + lens[i]].tobytes() == want, 'GPU stream (%d, %d) != oracle' % (n, c)
            streams.append(want)
    return streams


def _decode_streams(b, streams, tab, pitch, coarse=False):
    from l3c_pytorch_b200 import _lib, engine as E
    n_st, HW = len(streams), b.HW
    blob = torch.from_numpy(np.frombuffer(b''.join(streams) + b'\0' * 8, np.uint8).copy()).to(b.dev)
    offs = np.concatenate([[0], np.cumsum([len(s) for s in streams])[:-1]])
    out = torch.zeros(n_st * HW, dtype=torch.uint8, device=b.dev)
    state = torch.zeros(4 * n_st, dtype=torch.int32, device=b.dev)
    dd = np.zeros(n_st, dtype=_lib.DEC_STREAM_DTYPE)
    dd['table'] = tab.data_ptr() + 2 * pitch * HW * np.arange(n_st)
    dd['row_pitch'] = pitch
    dd['in'] = blob.data_ptr() + offs
    dd['in_len'] = [len(s) for s in streams]
    dd['n_sym'] = HW
    dd['sym_out'] = out.data_ptr() + HW * np.arange(n_st)
    dd['state'] = state.data_ptr() + 16 * np.arange(n_st)
    if coarse:
        E.ac_decode_streams_coarse(dd, b.dev, b.tg)
    else:
        E.ac_decode_streams(dd, b.dev, b.L)
    return out.cpu().numpy().reshape(b.N, b.C, HW)


def _decode_tiled(b, sym, tile):
    """rows in tile order from the tiled builder, one oracle stream per tile, decoded by the full-row decoder"""
    from l3c_pytorch_b200 import _lib, engine as E
    perm = tile_order_to_raster_py(b.H, b.W, *tile)
    sym_t = np.ascontiguousarray(sym[..., perm])
    table = torch.zeros(b.N * b.C * b.HW * b.pitch, dtype=torch.int16, device=b.dev)
    for c in (range(b.C) if b.rgb else [-1]):
        E.dmll_build_table_tiled(b.l, torch.from_numpy(sym_t).to(b.dev), b.tg, b.C, K, b.L, b.rgb, c, table, tile)
    rows_t = table.cpu().numpy().view(np.uint16).reshape(b.N, b.C, b.HW, b.pitch)[..., :b.L]
    sizes = [min(tile[0], b.H - y) * min(tile[1], b.W - x) for y in range(0, b.H, tile[0])
             for x in range(0, b.W, tile[1])]
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    items = []
    for n in range(b.N):
        for c in range(b.C):
            for s0, m in zip(starts, sizes):
                r = np.concatenate([rows_t[n, c, s0:s0 + m], np.zeros((m, 1), np.uint16)], 1)
                items.append(((n * b.C + c) * b.HW + s0, m, ac.encode(r, sym_t[n, c, s0:s0 + m])))
    blob = torch.from_numpy(np.frombuffer(b''.join(d for _, _, d in items) + b'\0' * 8, np.uint8).copy()).to(b.dev)
    offs = np.concatenate([[0], np.cumsum([len(d) for _, _, d in items])[:-1]])
    out = torch.zeros(b.N * b.C * b.HW, dtype=torch.uint8, device=b.dev)
    dd = np.zeros(len(items), dtype=_lib.DEC_STREAM_DTYPE)
    first = np.array([f for f, _, _ in items], np.int64)
    dd['table'] = table.data_ptr() + 2 * b.pitch * first
    dd['row_pitch'] = b.pitch
    dd['in'] = blob.data_ptr() + offs
    dd['in_len'] = [len(d) for _, _, d in items]
    dd['n_sym'] = [m for _, m, _ in items]
    dd['sym_out'] = out.data_ptr() + first
    E.ac_decode_streams(dd, b.dev, b.L)
    return out.cpu().numpy().reshape(b.N, b.C, b.HW), sym_t


def _decode_pipelined(b, streams, coarse, chunk):
    """l3c_decode_rgb_pipelined: rows (or coarse records) of G and B built from the symbols it has decoded"""
    from l3c_pytorch_b200 import _lib, engine as E
    N, C, HW = b.N, b.C, b.HW
    S = torch.zeros(N, C, b.H, b.W, dtype=torch.uint8, device=b.dev)
    pitch = E.COARSE_PITCH if coarse else b.L
    table = torch.zeros(N * C * HW * pitch, dtype=torch.int16, device=b.dev)
    state = torch.full((N * C * 4,), -1, dtype=torch.int32, device=b.dev)
    blob = torch.from_numpy(np.frombuffer(b''.join(streams) + b'\0' * 8, np.uint8).copy()).to(b.dev)
    offs = np.concatenate([[0], np.cumsum([len(s) for s in streams])[:-1]]).reshape(N, C)
    plane = np.arange(N)[:, None] * C + np.arange(C)[None]
    d = np.zeros((N, C), dtype=_lib.DEC_STREAM_DTYPE)
    d['in'] = blob.data_ptr() + offs
    d['in_len'] = np.array([len(s) for s in streams]).reshape(N, C)
    d['n_sym'] = HW
    d['sym_out'] = S.data_ptr() + HW * plane
    d['table'] = table.data_ptr() + 2 * pitch * HW * plane
    d['row_pitch'] = pitch
    d['state'] = state.data_ptr() + 16 * plane
    descs = [E._desc_to_device(np.ascontiguousarray(d[:, c]), b.dev) for c in range(C)]
    bld = [torch.cuda.Stream(device=b.dev) for _ in range(3)]
    dec = [torch.cuda.Stream(device=b.dev) for _ in range(3)]
    E.decode_rgb_pipelined(b.l, S, b.tg, K, b.L, table, descs, chunk, torch.cuda.current_stream(), bld, dec,
                           coarse=coarse)
    torch.cuda.synchronize()
    return S.cpu().numpy().reshape(N, C, HW)


FAMILY_GRIDS = [(True, 3, 256), (False, 5, 25), (False, 1, 100)]


def _family_case(family, rgb, C, L):
    rng = np.random.default_rng(100 * FAMILIES.index(family) + L + C)
    if family == 'trained':
        from tests import test_gpu_coarse_rows as cr
        if rgb:
            l, sym = cr._params('mixed', rng)
            H, W = cr.H, cr.W
            l = l.reshape(l.shape[0], H * W, -1)
        else:
            x0, x1, _ = _grid(rgb, L)
            H, W = FH, FW
            l = _trained_like(rng, FN, H * W, C, rgb, x0, x1, L)
            sym = _symbols(rng, FN, C, H * W, L)
        return l, sym, np.ones((l.shape[0], H * W, C), bool), H, W
    l, sym, sel = _family(family, rgb, C, L, rng)
    return l, sym, sel, FH, FW


@pytest.mark.gpu
@pytest.mark.parametrize('rgb,C,L', FAMILY_GRIDS)
@pytest.mark.parametrize('family', FAMILIES)
def test_rows_codable(family, rgb, C, L):
    from l3c_pytorch_b200 import engine as E
    if family == 'coupling' and not rgb:
        pytest.skip('coupling exists on the RGB scale only')
    l, sym, sel, H, W = _family_case(family, rgb, C, L)
    b = Built(l, sym, rgb, C, L, H, W)
    N, HW = b.N, b.HW
    _check_codable(b, family)
    regime = _regimes(family, l, rgb, C, sel, b)
    print('%s rgb=%d C=%d L=%d: %s; %d NaN ramp rows' % (family, rgb, C, L, regime, b.n_ramp))
    for case, n in regime.items():
        assert n >= 3, '%s: sub-case "%s" reached by %d sub-pixels only' % (family, case, n)
    if family == 'nan':
        assert b.n_ramp >= 10
    if family == 'sum_pi':
        # the last entry, before the 16-bit wrap, stays below 2^16 (and the row is the restatement's)
        for c in range(C):
            last = b.rows[:, c, :, -1].reshape(-1).astype(np.int64)
            lo_raw, hi_raw = b.ref[c]['lo_raw'][:, -1], b.ref[c]['hi_raw'][:, -1]
            assert ((last == lo_raw) | (last == hi_raw)).all() and (hi_raw <= 65535).all()
    # intervals: width >= 1, equal to the rows' differences, and what dmll_intervals_kernel computes
    lo, hi, want = _row_intervals(b.rows, sym)
    assert (hi - lo >= 1).all()
    iv = E.dmll_intervals(b.l, b.sym_dev, b.tg, C, K, L, rgb).cpu().numpy().view(np.uint32)
    assert (iv == want).all(), '%s: %d intervals differ from the rows' % (family, int((iv != want).sum()))
    streams = _encode(b, sym, want)
    # decode: full rows, tiled rows, and on the RGB scale the coarse records and the pipelined decoder
    got = _decode_streams(b, streams, b.table, b.pitch)
    assert (got == sym).all(), '%s: full-row decode: %d wrong symbols' % (family, int((got != sym).sum()))
    for tile in ((3, 5), (H, W)):
        got_t, sym_t = _decode_tiled(b, sym, tile)
        assert (got_t == sym_t).all(), '%s: tiled decode %s: %d wrong' % (family, tile, int((got_t != sym_t).sum()))
    if rgb:
        got = _decode_streams(b, streams, b.rec_t, E.COARSE_PITCH, coarse=True)
        assert (got == sym).all(), '%s: coarse decode: %d wrong symbols' % (family, int((got != sym).sum()))
        # the coarse decoder took both kinds of bracket: linear ones and term-parallel evaluated ones
        from tests.test_gpu_coarse_linear import linear_mask
        n_lin = n_eval = 0
        for c in range(C):
            pi_c, mu_c, is_c, _ = _rec_params(b.recs, c)
            with np.errstate(invalid='ignore', over='ignore'):
                lin = linear_mask(mu_c, is_c, b.t)                          # [N, HW, 32]
            at = np.take_along_axis(lin, (sym[:, c].astype(np.int64) // 8)[..., None], -1)[..., 0]
            n_lin, n_eval = n_lin + int(at.sum()), n_eval + int((~at).sum())
        print('coarse decode: %d symbols in linear brackets, %d in evaluated ones' % (n_lin, n_eval))
        assert n_lin > 0 and n_eval > 0
        for coarse in (False, True):
            for chunk in (1, 77, HW):
                got = _decode_pipelined(b, streams, coarse, chunk)
                assert (got == sym).all(), '%s: pipelined decode (coarse %s, chunk %d): %d wrong' % (
                    family, coarse, chunk, int((got != sym).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize('rgb,C,L', [(True, 3, 256), (False, 5, 25), (False, 5, 100)])
@pytest.mark.parametrize('family', FAMILIES)
def test_fused_head_codable(family, rgb, C, L):
    """the DMLL head fused into the 1x1 conv (the f16 encoder): its intervals equal, bit for bit, those of the rows
    built from the parameters it sees, and those rows are strictly increasing and the restatement's"""
    if family == 'coupling' and not rgb:
        pytest.skip('coupling exists on the RGB scale only')
    l, sym, _, H, W = _family_case(family, rgb, C, L)
    l_eff, iv = _fused_head(family, l, sym, rgb, C, L, H, W)
    b = Built(l_eff, sym, rgb, C, L, H, W)
    _check_codable(b, 'fused ' + family)
    lo, hi, want = _row_intervals(b.rows, sym)
    assert (hi - lo >= 1).all()
    bad = np.argwhere(iv != want)
    assert bad.size == 0, 'fused %s: %d intervals differ from the rows, first at %s' % (family, len(bad), bad[0])
    n_bias = int((~np.isfinite(_fused_bias(family, rgb, C))).sum() + (np.abs(_fused_bias(family, rgb, C)) > 65504).sum())
    print('fused %s rgb=%d C=%d L=%d: %d non-finite or beyond-FP16 bias channels, %d NaN ramp rows'
          % (family, rgb, C, L, n_bias, b.n_ramp))
    if family in ('wide', 'clamp', 'far', 'pi_underflow', 'nan', 'coupling'):
        assert n_bias > 0
    if family == 'nan':
        assert b.n_ramp >= 2 * b.N * b.HW


@pytest.mark.gpu
@pytest.mark.parametrize('rgb,C,L', [(True, 3, 256), (False, 5, 25), (False, 1, 100)])
@pytest.mark.parametrize('family', ['trained', 'wide', 'far'])
def test_dropin_on_clamped_parameters(family, rgb, C, L):
    """the torchac drop-in (l3c_*_logistic_mixture: plane_intervals_kernel / plane_table_kernel) on finite parameters
    with log-scales >= -7, the kernels' pi and mu: its stream is the oracle's on the restated rows of
    dmll_table_kernel, and it decodes back"""
    from l3c_pytorch_b200 import torchac
    l, sym, _, H, W = _family_case(family, rgb, C, L)
    with np.errstate(invalid='ignore'):
        l = np.where(np.isfinite(l), l, np.float32(7e5)).astype(np.float32)
    P = 4 if rgb else 3
    q = l.reshape(l.shape[0], H * W, P, C, K)
    q[:, :, 2] = np.clip(np.fmax(q[:, :, 2], LOG_SCALES_MIN), None, 20)
    b = Built(np.ascontiguousarray(q.reshape(l.shape)), sym, rgb, C, L, H, W)
    _check_codable(b, 'drop-in ' + family)
    N, HW = b.N, b.HW
    tg = torch.from_numpy(b.t).to(b.dev)
    for c in range(C):
        planes = [torch.from_numpy(np.ascontiguousarray(a.transpose(2, 0, 1).reshape(1, K, 1, N * HW))).to(b.dev)
                  for a in (b.mu[c], q[:, :, 2, c, :], b.pi[c])]
        s = torch.from_numpy(sym[:, c].reshape(-1).astype(np.int16))
        data = torchac.encode_logistic_mixture(tg, planes[0], planes[1], planes[2], s)
        rows = b.rows[:, c].reshape(N * HW, L)
        want = ac.encode(np.concatenate([rows, np.zeros((N * HW, 1), np.uint16)], 1), s.numpy())
        assert data == want, 'drop-in %s c=%d: stream differs from the oracle on the rows' % (family, c)
        back = torchac.decode_logistic_mixture(tg, planes[0], planes[1], planes[2], data)
        assert (back.numpy() == s.numpy()).all()
