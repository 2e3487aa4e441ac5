"""Every layer of the forward, checked on the exact operands it read, and its wiring checked against the oracle.

The end-to-end tests (test_gpu_model.py) hold the network to loose bounds: a quantiser flip budget, P at 8e-2 and
bpsp at 2e-3.  A wrong tap at a tile edge, a residual taken from the wrong tensor or an operand image rounded from
the wrong value costs compression long before it breaks those.  This file closes the gap in three parts.

1. Recorder.  The engine entry points network.py calls (conv2d, rgb_prep, rgb_head_f16, quantize_head,
   split_f16x2, symbols_to_values, bicubic_half) are wrapped.  Each call records the layer's state-dict name, its
   arguments, the operand image the kernel really read (`xa.r` for the tensor-core layers, `xa.f` for FFMA), every
   output, and the kernels it launched (engine.launch_log).  The routing is asserted from that log: in f16 every
   3x3 64-channel layer and every 5x5/s2 `down` runs a tensor-core kernel and `dec.head` runs FFMA; in f16x2
   `down` runs FFMA and is followed by split_f16x2.

2. Per-layer numerics (teacher forcing).  Each recorded conv is recomputed in float64 from the recorded operand
   and the weights as the kernel reads them: FP16 (clamped, RN), TF32 (RNA), the f16x2 split with the products the
   kernel forms (hi*hi + (hi*lo + lo*hi) / 2^11, no lo*lo term), or fp32 for FFMA.  Bias, ReLU, residual and pixel
   shuffle follow in the kernels' order.  Operand rounding therefore drops out; what remains is fp32 accumulation.
   Each output element gets the budget

       B = gamma * sum_i |t_i| + u_epi * (|after bias| + |after residual|) [+ u_epi * |combined| for f16x2],

   where t_i are the products and gamma = K * u_acc with K accumulation steps per output.  Each epilogue rounding
   (the bias add, the residual add, the f16x2 combine fma) is charged u_epi = 2^-22 of the value it produces: two
   full fp32 ulps, four times the half-ulp an RN rounding can reach, so that the margin of 2 also holds on outputs
   whose only error is that rounding (a residual that dominates the conv).
     * FFMA (conv_ffma_kernel): u_acc = 2^-24, one fma rounding per step of a sequential chain.  K is the fmas the
       kernel executes, Cin rounded up to its 32-channel chunk times k * k.  The zero-padded channels add exactly
       zero; counting them matters for the 3- and 5-channel layers (RGB head, decoder heads), whose error is decided
       by a handful of roundings and meets the K = Cin * k * k worst case to within 20 % somewhere among millions
       of outputs.
     * wgmma (conv3x3/5x5s2/1x1 f16, f16x2, tf32 kernels): K = Cin * k * k products, u_acc = 2^-23.  Hopper's
       tensor cores do not round each addition to nearest: a group of products is aligned to its largest
       exponent and truncated before it is added to the fp32 accumulator.  We charge every product one full fp32 ulp (truncation, not half an ulp) of the sum
       of magnitudes, which bounds the alignment loss of a group by its products and the accumulator's truncation
       by the running sum.
   Measured on an H100 SXM (80 GB, default power limit) over every case below, max |err| / B per kernel:
       conv_ffma_kernel 0.24      conv3x3_f16_kernel 0.0074     conv5x5s2_f16_kernel 0.0027
       conv1x1_f16_kernel 0.021   conv3x3_f16x2_kernel 0.0070   conv1x1_f16x2_kernel 0.012
       conv3x3_tf32_kernel 0.012  conv1x1_tf32_kernel 0.016
   Every layer must stay at or under 0.5 B, a margin of at least 2 on the constants (the test fails otherwise).
   One zeroed weight tap reads as err/B of about 2600.

   Operand images written beside an fp32 output must equal the documented rounding of that output bit for bit
   (f16: cvt.rn.satfinite = clamp to +-65504, RN, subnormals kept; f16x2: hi = satfinite RN(y), lo = satfinite
   RN((y - hi) * 2048); tf32: cvt.rna).  The next layer is teacher-forced, so this is the only check that sees a
   wrong twin.  An operand-only output (want='round') must be the rounding of some value within ref +- B.  The
   RGB im2col columns are checked against a float64 restatement of the two MeanShift affines, zero padding applied
   to the normalised value, entries 27..63 zero.  The quantiser's symbol must be the float64 argmin except where the
   two nearest levels are within budget of a tie, and bn_q must be exactly levels[sym].  symbols_to_values and
   split_f16x2 must be exact.

3. Dataflow.  oracle.model.forward (independent of network.py) is replayed in float64 with `_conv`, `quantize` and
   `pillow_bicubic_half` replaced by a shim that does not compute: it returns the GPU's recorded result for that
   name, undoing what the kernel fused (the residual is subtracted, the pixel-shuffled tail unshuffled, each atrous
   result taken from the slice that call wrote), so that the oracle's own graph redoes it.  First it asserts that
   the input the oracle's graph hands to the layer equals the operand the GPU layer read, within that operand's
   rounding, and that a fused residual equals the tensor the oracle adds.  Fused groups (sub_rgb_mean + MeanShift +
   RGB head; to_q + quantiser) are compared at the fused call's boundary.  The set of layer names the GPU called
   must equal the set the oracle called.  This runs for `cr` and `cr_rgb_shared`, the configurations the oracle
   restates; `cr_rgb` and the recursive scales get the per-layer checks only.

Planted defects (wrappers around the engine inside this file; nothing in the product changes) show that each check
can fail and names the right layer.  The host-only self-test shows the same for the budget itself.

Run with -s to print one line per layer: name, kernels, max err/B, share of outputs above 0.5 B, first failure.
"""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import util

U24 = 2.0 ** -24             # fp32 unit roundoff (RN)
U_FFMA = 2.0 ** -24          # per-product accumulation error of the sequential fma chain
U_WGMMA = 2.0 ** -23         # per-product accumulation error charged to Hopper's truncating wgmma accumulation
LO_SCALE = 2048.0            # f16x2: x = hi + lo / 2^11
F16_MAX = 65504.0
U_EPI = 2.0 ** -22           # charged per epilogue rounding (bias add, residual add, f16x2 combine): 2 full ulps
MARGIN = 0.5                 # every layer must stay at or under MARGIN * B

TC_KERNELS = {'f16': {3: 'conv3x3_f16_kernel', 5: 'conv5x5s2_f16_kernel', 1: 'conv1x1_f16_kernel'},
              'f16x2': {3: 'conv3x3_f16x2_kernel', 1: 'conv1x1_f16x2_kernel'},
              'tf32': {3: 'conv3x3_tf32_kernel', 1: 'conv1x1_tf32_kernel'}}
FFMA = 'conv_ffma_kernel'
SPLIT = 'split_f16x2_kernel'


# ----------------------------------------------------------------------------------------------------------------
# the roundings the kernels document, restated
# ----------------------------------------------------------------------------------------------------------------
def rnd16(y):
    """cvt.rn.satfinite.f16.f32: clamp to +-65504, round to nearest even, subnormals kept."""
    return y.float().clamp(-F16_MAX, F16_MAX).half()


def split16(y):
    """f16x2 operand image [.., 2C] = (hi | lo): hi = satfinite RN(y), lo = satfinite RN((y - hi) * 2048)."""
    y = y.float()
    hi = rnd16(y)
    return torch.cat([hi, rnd16((y - hi.float()) * LO_SCALE)], -1)


def rna_tf32(y):
    """cvt.rna.tf32.f32: keep 10 mantissa bits, ties away from zero (on the magnitude, sign kept)."""
    u = y.float().contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = (u & 0x80000000) | (((u & 0x7FFFFFFF) + 0x1000) & 0x7FFFE000)
    return torch.where(r >= 2 ** 31, r - 2 ** 32, r).to(torch.int32).view(torch.float32)


def _half_spacing(v, min_exp, mant_bits):
    """Half the spacing of the binade of |v| for a format with `mant_bits` stored bits and normal exponents down to
    min_exp (below: subnormal spacing)."""
    v = v.abs()
    e = torch.frexp(v)[1].to(torch.float64) - 1
    e = torch.where(v == 0, torch.full_like(e, min_exp), e).clamp(min=min_exp)
    return torch.pow(2.0, e - mant_bits - 1)


def hs16(v):
    return _half_spacing(v.double(), -14, 10)


def hs_tf32(v):
    return _half_spacing(v.double(), -126, 10)


def _bits_equal(a, b):
    if a.dtype == torch.float16:
        return a.view(torch.int16) == b.view(torch.int16)
    return a.view(torch.int32) == b.view(torch.int32)


# ----------------------------------------------------------------------------------------------------------------
# float64 reference of one conv and its budget (shared by the host self-test and the GPU checks)
# ----------------------------------------------------------------------------------------------------------------
def conv_reference(parts, bias, stride, dil, pad, n_products, u_acc, relu=False, residual=None,
                   pixel_shuffle=False, fma_combine=False):
    """parts: [(x NCHW float64, w OIHW float64, scale)] whose scaled convs sum to the accumulator (one part, or the
    three f16x2 products).  -> (reference, budget), NCHW float64, after bias / ReLU / residual / pixel shuffle."""
    acc = abs_sum = None
    for x, w, s in parts:
        a = F.conv2d(x, w, None, stride=stride, padding=pad, dilation=dil) * s
        m = F.conv2d(x.abs(), w.abs(), None, stride=stride, padding=pad, dilation=dil) * s
        acc = a if acc is None else acc + a
        abs_sum = m if abs_sum is None else abs_sum + m
    B = n_products * u_acc * abs_sum
    if fma_combine:                                   # acc1 = fma(acc2, 2^-11, acc1): one rounding
        B = B + U_EPI * (acc.abs() + B)
    v = acc + bias.view(1, -1, 1, 1)
    B = B + U_EPI * (v.abs() + B)
    if relu:
        v = v.clamp(min=0)
    if residual is not None:
        v = v + residual
        B = B + U_EPI * (v.abs() + B)
    if pixel_shuffle:
        v, B = F.pixel_shuffle(v, 2), F.pixel_shuffle(B, 2)
    return v, B


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


# ----------------------------------------------------------------------------------------------------------------
# host-only self-test of the budget: it holds for a faithful fp32 accumulation and fails on a missing tap
# ----------------------------------------------------------------------------------------------------------------
def _emulate_ffma(x16, w16, b32, skip_tap=None):
    """numpy: 3x3 conv (padding 1) of FP16 operands, products exact in fp32, accumulated sequentially in fp32 in
    the FFMA kernel's order (tap-major, then input channel), then + bias.  x16 [Cin,H,W], w16 [Cout,Cin,3,3]."""
    Cin, H, W = x16.shape
    xp = np.zeros((Cin, H + 2, W + 2), np.float32)
    xp[:, 1:-1, 1:-1] = x16.astype(np.float32)
    w = w16.astype(np.float32)
    out = np.zeros((w.shape[0], H, W), np.float32)
    for co in range(w.shape[0]):
        acc = np.zeros((H, W), np.float32)
        for tap in range(9):
            if tap == skip_tap:
                continue
            ky, kx = divmod(tap, 3)
            for ci in range(Cin):
                acc = (acc + xp[ci, ky:ky + H, kx:kx + W] * w[co, ci, ky, kx]).astype(np.float32)
        out[co] = (acc + b32[co]).astype(np.float32)
    return out


def test_budget_self_test_host():
    """No GPU: a faithful sequential fp32 accumulation stays within B; omitting one tap exceeds B by at least 4x on
    nearly every output (all of them depend on the centre tap)."""
    rng = np.random.default_rng(0)
    Cin, Cout, H, W = 16, 8, 9, 11
    x16 = (rng.standard_normal((Cin, H, W)) * 3).astype(np.float16)
    w16 = (rng.standard_normal((Cout, Cin, 3, 3)) * 0.1).astype(np.float16)
    b32 = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    ref, B = conv_reference([(torch.from_numpy(x16.astype(np.float64))[None],
                              torch.from_numpy(w16.astype(np.float64)), 1.0)],
                            torch.from_numpy(b32.astype(np.float64)), 1, 1, 1, Cin * 9, U_FFMA)
    ref, B = ref[0].numpy(), B[0].numpy()
    good = _emulate_ffma(x16, w16, b32)
    ratio = np.abs(good.astype(np.float64) - ref) / B
    assert ratio.max() <= MARGIN, ratio.max()
    bad = _emulate_ffma(x16, w16, b32, skip_tap=4)
    ratio = np.abs(bad.astype(np.float64) - ref) / B
    assert np.mean(ratio >= 4.0) >= 0.95, np.mean(ratio >= 4.0)


def test_roundings_host():
    """The restated roundings on hand-picked values: saturation, subnormals, ties."""
    y = torch.tensor([1e6, -1e6, 65519.0, 65520.0, 3e-6, -6e-8, 2.0 ** -25, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11])
    h = rnd16(y).float()
    assert h.tolist()[:4] == [65504.0, -65504.0, 65504.0, 65504.0]
    assert h[4].item() == 50 * 2.0 ** -24                                          # subnormal kept, RN
    assert h[6].item() == 0.0                                                      # 2^-25: tie to even (0)
    assert h[7].item() == 1.0 and h[8].item() == 1.0 + 2 * 2.0 ** -10             # ties to even
    t = rna_tf32(torch.tensor([1.0 + 2.0 ** -11, -(1.0 + 2.0 ** -11), 1.0 + 2.0 ** -12]))
    assert t.tolist() == [1.0 + 2.0 ** -10, -(1.0 + 2.0 ** -10), 1.0]               # ties away from zero
    s = split16(torch.tensor([[1.0 + 2.0 ** -13], [1e6]]))                        # rows: (hi | lo)
    assert s[0].float().tolist() == [1.0, 0.25] and s[1].float().tolist() == [65504.0, 65504.0]


# ----------------------------------------------------------------------------------------------------------------
# recorder
# ----------------------------------------------------------------------------------------------------------------
class Rec(object):
    def __init__(self, kind, name, **kw):
        self.kind, self.name = kind, name
        self.splits = []
        self.__dict__.update(kw)


def _expected_route(mode, conv, cin, want):
    """(route, kernels): which kernel a layer of this geometry runs in `mode`."""
    k, cin_all = conv.kernel_size[0], conv.in_channels
    tc = None
    if mode != 'fp32' and cin == cin_all:
        if k == 3 and cin == 64:
            tc = TC_KERNELS[mode][3]
        elif k == 5 and cin == 64:
            tc = TC_KERNELS[mode].get(5)
        elif k == 1 and cin % 64 == 0:
            tc = TC_KERNELS[mode][1]
    if tc is not None:
        return 'tc', {tc}
    return 'ffma', ({FFMA, SPLIT} if mode == 'f16x2' and want != 'plain' else {FFMA})


class Recorder(object):
    ENTRIES = ('conv2d', 'rgb_prep', 'rgb_head_f16', 'quantize_head', 'split_f16x2', 'symbols_to_values',
               'bicubic_half')

    def __init__(self, net):
        from l3c_pytorch_b200 import engine as E
        self.E = E
        self.names = {id(m): n for n, m in net.named_modules()}
        self.calls = []
        self._conv = None                  # the conv record a nested split_f16x2 belongs to

    def install(self, mp, inner=None, outer=None):
        """Wrap the engine: network -> outer -> recorder -> inner -> engine (plants go in `inner` when the recorder
        must see the caller's arguments, in `outer` when it must see what the kernel was given)."""
        E = self.E
        orig = {n: getattr(E, n) for n in self.ENTRIES}
        conv = orig['conv2d'] if inner is None else inner(orig['conv2d'])
        rec_conv = self._wrap_conv(conv)
        mp.setattr(E, 'conv2d', rec_conv if outer is None else outer(rec_conv))
        mp.setattr(E, 'split_f16x2', self._wrap_split(orig['split_f16x2']))
        mp.setattr(E, 'rgb_prep', self._wrap_rgb_prep(orig['rgb_prep']))
        mp.setattr(E, 'rgb_head_f16', self._wrap_rgb_head(orig['rgb_head_f16']))
        mp.setattr(E, 'quantize_head', self._wrap_quantize(orig['quantize_head']))
        mp.setattr(E, 'symbols_to_values', self._wrap_s2v(orig['symbols_to_values']))
        mp.setattr(E, 'bicubic_half', self._wrap_bicubic(orig['bicubic_half']))

    def _log(self):
        return set(self.E.launch_log(reset=True)[0])

    def _wrap_conv(self, fn):
        E = self.E

        def conv2d(conv, x, cin=None, relu=False, residual=None, pixel_shuffle=False, out=None, out_coff=0,
                   precision=None, want='plain'):
            assert precision is None
            mode = E.get_conv_precision()
            xa = x if isinstance(x, E.Act) else E.Act(x)
            cin_r = conv.in_channels if cin is None else cin
            route, kernels = _expected_route(mode, conv, cin_r, want)
            # the operand image the kernel reads (engine.conv2d's operand for each mode and route)
            op, opkind = None, None
            if route == 'ffma':
                op, opkind = xa.f[..., :cin_r].clone(), 'f32'
            elif mode == 'tf32':
                op, opkind = (xa.r if xa.r is not None else xa.f).clone(), 'tf32'
            elif mode == 'f16':
                r = xa.r if (xa.r is not None and xa.r.dtype == torch.float16) else None
                op, opkind = (r.clone() if r is not None else rnd16(xa.f)), 'f16'
            else:
                r = xa.r
                if r is not None and r.dtype == torch.float16 and r.shape[-1] == 2 * conv.in_channels:
                    op = r.clone()
                opkind = 'split'
            rec = Rec('conv', self.names[id(conv)], conv=conv, mode=mode, route=route, cin=cin_r, relu=relu,
                      residual=None if residual is None else residual.clone(), pixel_shuffle=pixel_shuffle,
                      out_coff=out_coff, has_out=out is not None, want=want, x=op, opkind=opkind,
                      expect_kernels=kernels)
            self._log()
            self._conv = rec
            try:
                ret = fn(conv, x, cin=cin, relu=relu, residual=residual, pixel_shuffle=pixel_shuffle, out=out,
                         out_coff=out_coff, want=want)
            finally:
                self._conv = None
            rec.kernels = self._log()
            if rec.x is None:                  # f16x2 operand split inside the call
                assert rec.splits, 'f16x2 tensor-core layer %s read no split image' % rec.name
                rec.x = rec.splits[0][1]
            cout = conv.out_channels // (4 if pixel_shuffle else 1)
            y = img = only = None
            if out is not None:
                if mode == 'f16x2' and want == 'round':
                    P = out.shape[-1] // 2
                    sl = torch.cat([out[..., out_coff:out_coff + cout], out[..., P + out_coff:P + out_coff + cout]], -1)
                else:
                    sl = out[..., out_coff:out_coff + cout]
                if want == 'round' and mode != 'fp32':
                    only = sl.clone()
                else:
                    y = sl.clone()
            elif want == 'plain':
                y = ret.clone()
            elif mode == 'fp32':
                y = ret.f.clone()
            elif want == 'round':
                only = (ret.f if mode == 'tf32' else ret.r).clone()
            else:
                y, img = ret.f.clone(), ret.r.clone()
            if route == 'ffma' and mode == 'f16x2' and want != 'plain':
                # the FFMA kernel's fp32 output, split by l3c_split_f16x2 (recorded below as its own check)
                assert len(rec.splits) == 1, rec.name
                y, img, only = rec.splits[0][0], rec.splits[0][1], None
            rec.y, rec.img, rec.only = y, img, only
            self.calls.append(rec)
            return ret
        return conv2d

    def _wrap_split(self, fn):
        def split_f16x2(x):
            top = self._conv is None
            if top:
                self._log()
            out = fn(x)
            if top:
                self.calls.append(Rec('split', 'split_f16x2', x=x.clone(), out=out.clone(), kernels=self._log()))
            else:
                self._conv.splits.append((x.clone(), out.clone()))
            return out
        return split_f16x2

    def _wrap_rgb_prep(self, fn):
        def rgb_prep(img_u8, conv1, conv2):
            self._log()
            xsub, t = fn(img_u8, conv1, conv2)
            self.calls.append(Rec('rgb_prep', self.names[id(conv2)], img=img_u8.clone(), conv1=conv1, conv2=conv2,
                                  xsub=None if xsub is None else xsub.clone(), t=None if t is None else t.clone(),
                                  kernels=self._log()))
            return xsub, t
        return rgb_prep

    def _wrap_rgb_head(self, fn):
        E = self.E

        def rgb_head_f16(img_u8, conv1, conv2, head_conv):
            self._log()
            ret = fn(img_u8, conv1, conv2, head_conv)
            kernels = self._log()
            # the columns the GEMM read: the same im2col kernel on the same image
            N, _, H, W = img_u8.shape
            prm = []
            for m in (conv1, conv2):
                prm += [m.weight.detach().float().reshape(9).contiguous(), m.bias.detach().float().contiguous()]
            cols = torch.empty(N, H, W, 64, dtype=torch.float16, device=img_u8.device)
            E.check(E.lib.l3c_rgb_im2col_f16(E._ptr(img_u8), *[E._ptr(p) for p in prm], N, H, W, E._ptr(cols),
                                             E._stream_ptr()))
            self._log()
            self.calls.append(Rec('rgb_head', self.names[id(head_conv)], img=img_u8.clone(), conv1=conv1,
                                  conv2=conv2, conv=head_conv, cols=cols, only=ret.r.clone(), kernels=kernels))
            return ret
        return rgb_head_f16

    def _wrap_quantize(self, fn):
        def quantize_head(f, to_q_conv, levels):
            self._log()
            sym, bnq = fn(f, to_q_conv, levels)
            self.calls.append(Rec('quantize', self.names[id(to_q_conv)], f=f.clone(), conv=to_q_conv,
                                  levels=levels.detach().float().clone(), sym=sym.clone(), bnq=bnq.clone(),
                                  kernels=self._log()))
            return sym, bnq
        return quantize_head

    def _wrap_s2v(self, fn):
        def symbols_to_values(sym, values, shift=None):
            self._log()
            out = fn(sym, values, shift)
            self.calls.append(Rec('s2v', 'symbols_to_values', sym=sym.clone(), values=values.clone(),
                                  shift=None if shift is None else shift.clone(), out=out.clone(),
                                  kernels=self._log()))
            return out
        return symbols_to_values

    def _wrap_bicubic(self, fn):
        def bicubic_half(img_u8):
            self._log()
            out = fn(img_u8)
            self.calls.append(Rec('bicubic', 'bicubic_half', img=img_u8.clone(), out=out.clone(), kernels=self._log()))
            return out
        return bicubic_half


# ----------------------------------------------------------------------------------------------------------------
# per-layer checks
# ----------------------------------------------------------------------------------------------------------------
class Report(object):
    """Per layer: kernels, max err/B, share above MARGIN * B, first failing index; and the failures (layer, check)."""

    def __init__(self):
        self.rows = {}
        self.fails = []          # (layer, check, message), in the order found

    def row(self, key, kernels):
        if key not in self.rows:
            self.rows[key] = dict(kernels=sorted(kernels), ratio=0.0, above=0, n=0, first=None)
        return self.rows[key]

    def ratio(self, key, kernels, ratio, what):
        r = self.row(key, kernels)
        ratio = ratio.reshape(-1)
        if ratio.numel():
            mx = float(ratio.max())
            r['ratio'] = max(r['ratio'], mx)
            r['above'] += int((ratio > MARGIN).sum())
            r['n'] += ratio.numel()
            if mx > 1.0:
                self.fail(key, 'numerics', '%s: max err/B %.3g' % (what, mx), ratio > 1.0)

    def fail(self, key, check, msg, mask=None):
        first = None
        if mask is not None:
            idx = torch.nonzero(mask.reshape(-1))
            first = int(idx[0]) if len(idx) else None
        self.fails.append((key, check, msg if first is None else '%s (first flat index %d)' % (msg, first)))
        r = self.rows.get(key)
        if r is not None and r['first'] is None:
            r['first'] = '%s@%s' % (check, first)

    def margins(self):
        for key, r in self.rows.items():
            if r['ratio'] > MARGIN and not any(f[0] == key and f[1] == 'numerics' for f in self.fails):
                self.fail(key, 'margin', 'max err/B %.3g above %.2g' % (r['ratio'], MARGIN))

    def table(self, title):
        lines = ['== %s' % title,
                 '%-44s %-44s %10s %10s  %s' % ('layer', 'kernels', 'max err/B', '>0.5B', 'first failure')]
        for key, r in self.rows.items():
            lines.append('%-44s %-44s %10.3e %10.2e  %s' % (key, ','.join(r['kernels']), r['ratio'],
                                                             r['above'] / max(r['n'], 1), r['first'] or '-'))
        return '\n'.join(lines)

    def per_kernel(self):
        out = {}
        for r in self.rows.values():
            for k in r['kernels']:
                if k != SPLIT:
                    out[k] = max(out.get(k, 0.0), r['ratio'])
        return out


def _weights_as_read(rec):
    """float64 OIHW weight parts (w, scale) of the conv as its kernel reads them."""
    w = rec.conv.weight.detach().float()
    if rec.route == 'ffma':
        return [(w.double(), 1.0)]
    if rec.mode == 'tf32':
        return [(rna_tf32(w).double(), 1.0)]
    wc = w.clamp(-F16_MAX, F16_MAX)
    hi = wc.half()
    if rec.mode == 'f16':
        return [(hi.double(), 1.0)]
    lo = ((wc - hi.float()) * LO_SCALE).half()
    return [(hi.double(), 1.0), (lo.double(), 1.0 / LO_SCALE)]


def layer_reference(rec):
    """-> (ref, B) NHWC float64 of a recorded conv, from its recorded operand."""
    conv = rec.conv
    k, stride, dil = conv.kernel_size[0], conv.stride[0], conv.dilation[0]
    pad = k // 2 if dil == 1 else dil
    ws = _weights_as_read(rec)
    if rec.opkind == 'split':
        C = rec.x.shape[-1] // 2
        hi, lo = _nchw(rec.x[..., :C]).double(), _nchw(rec.x[..., C:]).double()
        (whi, _), (wlo, s) = ws
        parts = [(hi, whi, 1.0), (hi, wlo, s), (lo, whi, s)]
    else:
        parts = [(_nchw(rec.x).double(), ws[0][0], 1.0)]
    if rec.route == 'ffma':
        # the fmas conv_ffma_kernel executes: Cin in chunks of 32 channels (zero padded), times k*k taps
        u_acc, steps = U_FFMA, -(-rec.cin // 32) * 32 * k * k
    else:
        u_acc, steps = U_WGMMA, rec.cin * k * k
    res = None if rec.residual is None else _nchw(rec.residual).double()
    ref, B = conv_reference(parts, conv.bias.detach().double(), stride, dil, pad, steps, u_acc,
                            relu=rec.relu, residual=res, pixel_shuffle=rec.pixel_shuffle,
                            fma_combine=rec.opkind == 'split')
    return _nhwc(ref), _nhwc(B)


def _check_only(rep, key, kernels, v, ref, B, fmt):
    """Operand-only output: the rounding (fmt) of some value within ref +- B."""
    if fmt == 'split':
        C = v.shape[-1] // 2
        hi, lo = v[..., :C].double(), v[..., C:].double()
        val, hs = hi + lo / LO_SCALE, hs16(lo) / LO_SCALE
        # hi must itself be the FP16 rounding of the value the pair stands for
        bad = (hi - val.clamp(-F16_MAX, F16_MAX)).abs() > hs16(hi) * (1 + 2.0 ** -9)
        if bool(bad.any()):
            rep.fail(key, 'image', 'split image: hi is not the FP16 rounding of hi + lo/2^11', bad)
    else:
        val = v.double()
        hs = hs16(val) if fmt == 'f16' else hs_tf32(val)
        if fmt == 'f16':
            ref = ref.clamp(-F16_MAX, F16_MAX)
    excess = ((val - ref).abs() - hs).clamp(min=0)
    rep.ratio(key, kernels, excess / B.clamp(min=1e-300), 'operand-only output')


def check_conv(rep, key, rec):
    if rec.kernels != rec.expect_kernels:
        rep.fail(key, 'routing', 'ran %s, expected %s' % (sorted(rec.kernels), sorted(rec.expect_kernels)))
    if rec.opkind == 'tf32' and not bool(_bits_equal(rna_tf32(rec.x), rec.x).all()):
        rep.fail(key, 'operand', 'tf32 operand is not TF32-representable')
    ref, B = layer_reference(rec)
    if rec.y is not None:
        assert rec.y.shape == ref.shape, (key, rec.y.shape, ref.shape)
        err = (rec.y.double() - ref).abs()
        rep.ratio(key, rec.kernels, err / B.clamp(min=1e-300), 'fp32 output')
    if rec.img is not None:
        want = {'f16': rnd16, 'f16x2': split16, 'tf32': rna_tf32}[rec.mode](rec.y)
        eq = _bits_equal(rec.img, want)
        if not bool(eq.all()):
            rep.fail(key, 'image', 'operand image != documented rounding of the fp32 output (%d elements)'
                     % int((~eq).sum()), ~eq)
    if rec.only is not None:
        fmt = {'f16': 'f16', 'tf32': 'tf32', 'f16x2': 'split'}[rec.mode]
        assert rec.only.shape[:3] == ref.shape[:3], key
        _check_only(rep, key, rec.kernels, rec.only, ref, B, fmt)
    for sx, sout in rec.splits:
        eq = _bits_equal(sout, split16(sx))
        if not bool(eq.all()):
            rep.fail(key, 'split', 'split_f16x2 output != documented split of its input', ~eq)


def _affines64(img_u8, conv1, conv2):
    """float64 restatement of the two MeanShift 1x1 convs -> (z NCHW, magnitude bound of the fp32 terms)."""
    x = img_u8.double()
    A1, b1 = conv1.weight.detach().double().reshape(3, 3), conv1.bias.detach().double()
    A2, b2 = conv2.weight.detach().double().reshape(3, 3), conv2.bias.detach().double()
    y = torch.einsum('cj,njhw->nchw', A1, x) + b1.view(1, 3, 1, 1)
    z = torch.einsum('cj,njhw->nchw', A2, y) + b2.view(1, 3, 1, 1)
    ym = torch.einsum('cj,njhw->nchw', A1.abs(), x) + b1.abs().view(1, 3, 1, 1)
    zm = torch.einsum('cj,njhw->nchw', A2.abs(), ym) + b2.abs().view(1, 3, 1, 1)
    return z, zm


def check_rgb_head(rep, key, rec):
    kernels = rec.kernels
    if kernels != {'rgb_im2col_kernel', TC_KERNELS['f16'][1]}:
        rep.fail(key, 'routing', 'ran %s' % sorted(kernels))
    z, zm = _affines64(rec.img, rec.conv1, rec.conv2)
    N, _, H, W = z.shape
    zp, zmp = F.pad(z, (1, 1, 1, 1)), F.pad(zm, (1, 1, 1, 1))      # zero padding of the NORMALISED image
    taps = [(zp[:, :, ky:ky + H, kx:kx + W], zmp[:, :, ky:ky + H, kx:kx + W]) for ky in range(3) for kx in range(3)]
    want = torch.cat([_nhwc(t) for t, _ in taps], -1)            # element tap*3 + c
    mag = torch.cat([_nhwc(m) for _, m in taps], -1)
    got = rec.cols[..., :27].double()
    bad = (got - want.clamp(-F16_MAX, F16_MAX)).abs() > hs16(got) + 16 * U24 * mag
    if bool(bad.any()):
        rep.fail(key, 'im2col', 'columns != FP16 rounding of the normalised 3x3 neighbourhood', bad)
    if not bool((rec.cols[..., 27:].view(torch.int16) == 0).all()):
        rep.fail(key, 'im2col', 'entries 27..63 of the columns are not +0')
    # the K = 64 GEMM on the columns, weights k = (ky*3 + kx)*3 + c as FP16
    w = rec.conv.weight.detach().float().clamp(-F16_MAX, F16_MAX).half().double()      # [Cf, 3, 3, 3]
    wk = w.permute(0, 2, 3, 1).reshape(w.shape[0], 27)
    cols = rec.cols[..., :27].double()
    acc = cols @ wk.t()
    A = cols.abs() @ wk.abs().t()
    ref = acc + rec.conv.bias.detach().double()
    B = 64 * U_WGMMA * A + U_EPI * (ref.abs() + 64 * U_WGMMA * A)
    _check_only(rep, key, kernels, rec.only, ref, B, 'f16')


def check_rgb_prep(rep, key, rec):
    if rec.kernels != {'rgb_prep_kernel'}:
        rep.fail(key, 'routing', 'ran %s' % sorted(rec.kernels))
    z, zm = _affines64(rec.img, rec.conv1, rec.conv2)
    got = rec.t.double()
    ratio = (got[..., :3] - _nhwc(z)).abs() / (16 * U24 * _nhwc(zm))
    rep.ratio(key, rec.kernels, ratio, 'rgb_prep')
    if not bool((rec.t[..., 3] == 0).all()):
        rep.fail(key, 'rgb_prep', 'padding channel 3 is not 0')


def check_quantize(rep, key, rec):
    if rec.kernels != {'quantize_head_kernel'}:
        rep.fail(key, 'routing', 'ran %s' % sorted(rec.kernels))
    C, Cf = rec.conv.out_channels, rec.conv.in_channels
    w = rec.conv.weight.detach().double().reshape(C, Cf)
    f = rec.f.double()
    q = f @ w.t() + rec.conv.bias.detach().double()
    Bq = Cf * U_FFMA * (f.abs() @ w.abs().t()) + U_EPI * q.abs()
    lev = rec.levels.double()
    d = (q.unsqueeze(-1) - lev).abs()
    ds, order = torch.sort(d, dim=-1, stable=True)
    sym = rec.sym.permute(0, 2, 3, 1).long()
    tie = (ds[..., 1] - ds[..., 0]) <= 2 * (Bq + 2.0 ** -20 * (1 + q.abs()))
    ok = (sym == order[..., 0]) | (tie & (sym == order[..., 1]))
    if not bool(ok.all()):
        rep.fail(key, 'quantizer', 'symbol is not the nearest level (%d)' % int((~ok).sum()), ~ok)
    rep.row(key, rec.kernels)['ties'] = int(tie.sum())
    if not (torch.equal(rec.bnq[..., :C], rec.levels[sym]) and bool((rec.bnq[..., C:] == 0).all())):
        rep.fail(key, 'quantizer', 'bn_q != levels[sym] (zero padded)')


def check_s2v(rep, key, rec):
    if rec.kernels != {'symbols_to_values_kernel'}:
        rep.fail(key, 'routing', 'ran %s' % sorted(rec.kernels))
    C = rec.sym.shape[1]
    want = rec.values[rec.sym.long()].permute(0, 2, 3, 1)
    if rec.shift is not None:
        want = want - rec.shift
    if not (torch.equal(rec.out[..., :C], want) and bool((rec.out[..., C:] == 0).all())):
        rep.fail(key, 's2v', 'symbols_to_values != values[sym] - shift')


def check_layers(rec):
    rep = Report()
    count = {}
    for r in rec.calls:
        n = count.get(r.name, 0)
        count[r.name] = n + 1
        key = r.name if n == 0 else '%s#%d' % (r.name, n)
        rep.row(key, r.kernels)
        if r.kind == 'conv':
            check_conv(rep, key, r)
        elif r.kind == 'rgb_head':
            check_rgb_head(rep, key, r)
        elif r.kind == 'rgb_prep':
            check_rgb_prep(rep, key, r)
        elif r.kind == 'quantize':
            check_quantize(rep, key, r)
        elif r.kind == 's2v':
            check_s2v(rep, key, r)
        elif r.kind == 'split':
            if not bool(_bits_equal(r.out, split16(r.x)).all()):
                rep.fail(key, 'split', 'split_f16x2 output != documented split of its input')
    rep.margins()
    return rep


# ----------------------------------------------------------------------------------------------------------------
# dataflow against oracle.model
# ----------------------------------------------------------------------------------------------------------------
def _undo(r):
    """The recorded result of conv `r` as the oracle's conv returns it: NCHW float64, residual subtracted, the
    pixel shuffle undone."""
    if r.y is not None:
        v = r.y.double()
        if r.residual is not None:
            v = v - r.residual.double()
    else:
        assert r.residual is None, r.name
        if r.mode == 'f16x2':
            C = r.only.shape[-1] // 2
            v = r.only[..., :C].double() + r.only[..., C:].double() / LO_SCALE
        else:
            v = r.only.double()
    v = _nchw(v)
    return F.pixel_unshuffle(v, 2) if r.pixel_shuffle else v


def _operand_bad(x, op, opkind):
    """x: NHWC float64 the oracle hands to the layer; op: the operand image the GPU read.  -> violation mask."""
    if opkind == 'f32':
        g = op.double()
        return (x - g).abs() > 2.0 ** -40 * (g.abs() + g.abs().max())
    if opkind == 'f16':
        g = op.double()
        return (x.clamp(-F16_MAX, F16_MAX) - g).abs() > hs16(g) * (1 + 2.0 ** -10)
    if opkind == 'tf32':
        g = op.double()
        return (x - g).abs() > hs_tf32(g) * (1 + 2.0 ** -10)
    C = op.shape[-1] // 2
    lo = op[..., C:].double()
    g = op[..., :C].double() + lo / LO_SCALE
    return (x - g).abs() > (hs16(lo) / LO_SCALE) * (1 + 2.0 ** -10) + 2.0 ** -40 * g.abs()


def _expected_residual_src(name, num_scales, dec_skip):
    """Name of the layer whose oracle input is the tensor the oracle adds after `name` (None: nothing is added)."""
    m = re.match(r'(nets\.\d+\.(?:enc|dec)\.body)\.(\d+)\.body\.2$', name)
    if m:
        return '%s.%s.body.0' % (m.group(1), m.group(2))
    m = re.match(r'(nets\.\d+\.(?:enc|dec)\.body)\.(\d+)$', name)
    if m:
        return '%s.0.body.0' % m.group(1)
    m = re.match(r'nets\.(\d+)\.dec\.head$', name)
    if m and dec_skip and int(m.group(1)) + 1 < num_scales:
        return 'prob_clfs.%d.atrous.atrous.0' % (int(m.group(1)) + 1)
    return None


def check_dataflow(rec, bp, cfg_name, imgs, mp):
    """Replay oracle.model.forward on the GPU's recorded results; -> Report of wiring failures, in oracle order."""
    from oracle import model as om
    rep = Report()
    cfg = util.oracle_cfg(cfg_name)
    dev = imgs.device
    sd = {k: v.detach().double() for k, v in bp.net.state_dict().items()}
    queues, quant, bicubic = {}, [], []
    front = None
    gpu_names = set()
    for r in rec.calls:
        if r.kind == 'conv':
            queues.setdefault(r.name, []).append(r)
            gpu_names.add(r.name)
        elif r.kind == 'quantize':
            quant.append(r)
            gpu_names.add(r.name)
        elif r.kind == 'bicubic':
            bicubic.append(r)
            gpu_names.add('sub_rgb_mean')
        elif r.kind == 'rgb_prep':
            front = r
            gpu_names.update({'sub_rgb_mean', 'heads.0.head.0'})
        elif r.kind == 'rgb_head':
            front = r
            gpu_names.update({'sub_rgb_mean', 'heads.0.head.0', 'heads.0.head.1.head'})
    seen, called = {}, set()

    def op_check(name, x, op, opkind):
        bad = _operand_bad(x, op, opkind)
        if bool(bad.any()):
            rep.fail(name, 'operand', 'input the oracle hands to the layer != operand the GPU read (%s, %d elements)'
                     % (opkind, int(bad.sum())), bad)

    def shim_conv(sd_, name, x, stride=1, rate=1):
        called.add(name)
        xh = _nhwc(x)
        seen.setdefault(name, xh)
        rep.row(name, [])
        if name == 'sub_rgb_mean':
            src = front.img if front is not None else bicubic[0].img
            if not torch.equal(x, src.double()):
                rep.fail(name, 'operand', 'image the oracle reads != image the GPU read')
            return F.conv2d(x, sd[name + '.weight'], sd[name + '.bias'])          # inside the fused call
        if name == 'heads.0.head.0':
            if front.kind == 'rgb_prep':
                return _nchw(front.t[..., :3]).double()
            return F.conv2d(x, sd[name + '.weight'], sd[name + '.bias'])          # inside rgb_head_f16
        if name == 'heads.0.head.1.head' and front is not None and front.kind == 'rgb_head':
            got = front.cols[..., 12:15].double()                                 # centre tap of the im2col
            bad = (xh.clamp(-F16_MAX, F16_MAX) - got).abs() > hs16(got) + 2.0 ** -20 * xh.abs()
            if bool(bad.any()):
                rep.fail(name, 'operand', 'normalised image != the im2col centre tap', bad)
            return _nchw(front.only).double()
        if name.endswith('.to_q.0'):
            q = quant[0]
            op_check(name, xh, q.f, 'f32')
            return torch.zeros(x.shape[0], q.conv.out_channels, x.shape[2], x.shape[3], dtype=x.dtype, device=dev)
        if not queues.get(name):
            rep.fail(name, 'missing', 'the oracle calls a layer the GPU did not run')
            w = sd[name + '.weight']
            pad = w.shape[-1] // 2 if rate == 1 else rate
            return F.conv2d(x, w, sd[name + '.bias'], stride=stride, padding=pad, dilation=rate)
        r = queues[name].pop(0)
        op_check(name, xh, r.x, r.opkind)
        src = _expected_residual_src(name, cfg.num_scales, cfg.dec_skip)
        if (src is None) != (r.residual is None):
            rep.fail(name, 'residual', 'GPU residual %s, oracle adds %s' % (r.residual is not None, src))
        elif src is not None:
            want = seen[src]
            g = r.residual.double()
            bad = (g - want).abs() > 2.0 ** -40 * (g.abs() + g.abs().max())
            if bool(bad.any()):
                rep.fail(name, 'residual', 'fused residual != the tensor the oracle adds (%s input, %d elements)'
                         % (src, int(bad.sum())), bad)
        return _undo(r)

    def shim_quantize(q_in, levels):
        q = quant.pop(0)
        C = q.conv.out_channels
        return q.sym.long(), _nchw(q.bnq[..., :C]).double()

    def shim_bicubic(u8):
        b = bicubic.pop(0)
        if not torch.equal(u8, b.img):
            rep.fail('bicubic_half', 'operand', 'image the oracle downsamples != image the GPU downsampled')
        return b.out

    mean255 = om._rgb_mean255
    with mp.context() as m:
        m.setattr(om, '_conv', shim_conv)
        m.setattr(om, 'quantize', shim_quantize)
        m.setattr(om, 'pillow_bicubic_half', shim_bicubic)
        m.setattr(om, '_rgb_mean255', lambda: mean255().to(dev))
        om.forward(sd, cfg, imgs.double())
    if called != gpu_names:
        rep.fail('<graph>', 'names', 'oracle-only %s, GPU-only %s' % (sorted(called - gpu_names),
                                                                       sorted(gpu_names - called)))
    left = [n for n, q in queues.items() if q] + (['quantize'] if quant else []) + (['bicubic'] if bicubic else [])
    if left:
        rep.fail('<graph>', 'names', 'GPU calls the oracle never consumed: %s' % left)
    return rep


# ----------------------------------------------------------------------------------------------------------------
# driver
# ----------------------------------------------------------------------------------------------------------------
def _fresh_blueprint(cfg_name):
    from l3c_pytorch_b200 import config
    from l3c_pytorch_b200.blueprint import MultiscaleBlueprint
    torch.manual_seed(0)
    return MultiscaleBlueprint(config.ms_config(cfg_name)).set_eval()


def run_case(mp, bp, cfg_name, prec, N, H, W, auto_recurse=0, max_sms=0, dataflow=True, inner=None, outer=None,
             title=None):
    """Forward once under the recorder -> (recorder, per-layer report, dataflow report or None)."""
    from l3c_pytorch_b200 import engine as E
    imgs = torch.stack([util.make_image(i, H, W) for i in range(N)]).cuda()
    old = E.get_conv_precision()
    E.set_conv_precision(prec)
    rec = Recorder(bp.net)
    try:
        with mp.context() as m:
            rec.install(m, inner=inner, outer=outer)
            with E.conv_launch_limits(max_sms=max_sms):
                bp.net(imgs, auto_recurse=auto_recurse)
            torch.cuda.synchronize()
    finally:
        E.set_conv_precision(old)
    assert rec.calls, 'the recorder saw no engine call'
    layers = check_layers(rec)
    flow = check_dataflow(rec, bp, cfg_name, imgs, mp) if dataflow else None
    title = title or '%s %s N=%d %dx%d%s%s' % (cfg_name, prec, N, H, W, ' recurse=%d' % auto_recurse
                                                if auto_recurse else '', ' max_sms=%d' % max_sms if max_sms else '')
    print()
    print(layers.table(title))
    print('   per kernel max err/B: %s' % ', '.join('%s %.3e' % kv for kv in sorted(layers.per_kernel().items())))
    if flow is not None:
        print('   dataflow: %d layers checked against oracle.model, %d failures' % (len(flow.rows), len(flow.fails)))
    return rec, layers, flow


def _failure_text(rep):
    return '\n'.join('%s [%s] %s' % f for f in rep.fails)


CASES = [
    # (cfg, precision, N, H, W, auto_recurse, max_sms, dataflow)
    ('cr', 'fp32', 2, 200, 296, 0, 0, True),     # every scale has partial 8x16 tiles, down to 25x37
    ('cr', 'tf32', 2, 200, 296, 0, 0, True),
    ('cr', 'f16', 2, 200, 296, 0, 0, True),
    ('cr', 'f16x2', 2, 200, 296, 0, 0, True),
    ('cr', 'f16', 2, 512, 512, 0, 0, True),      # the benchmark's shape
    ('cr', 'f16', 1, 200, 296, 0, 3, True),      # decode-lane regime: 3 SMs, many tiles per CTA
    ('cr_rgb_shared', 'f16x2', 2, 256, 256, 0, 0, True),   # the benchmark's case
    ('cr_rgb_shared', 'f16', 1, 130, 206, 0, 0, True),     # odd thumbnails
    ('cr_rgb_shared', 'f16x2', 2, 256, 256, 2, 0, False),  # recursive scales
    ('cr_rgb', 'f16', 1, 64, 96, 0, 0, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize('cfg_name,prec,N,H,W,recurse,max_sms,dataflow', CASES,
                         ids=['%s-%s-%dx%dx%d%s%s' % (c[0], c[1], c[2], c[3], c[4], '-rec%d' % c[5] if c[5] else '',
                                                     '-sms%d' % c[6] if c[6] else '') for c in CASES])
def test_layer_parity(monkeypatch, cfg_name, prec, N, H, W, recurse, max_sms, dataflow):
    bp = util.blueprint(cfg_name)
    rec, layers, flow = run_case(monkeypatch, bp, cfg_name, prec, N, H, W, recurse, max_sms, dataflow)
    fails = layers.fails + (flow.fails if flow is not None else [])
    assert not fails, '\n' + _failure_text(layers) + '\n' + (_failure_text(flow) if flow else '') + '\n' + \
        layers.table('failing case')
    # the case exercised what it claims
    kinds = {r.kind for r in rec.calls}
    if cfg_name == 'cr':
        assert ('rgb_head' if prec == 'f16' else 'rgb_prep') in kinds and 'quantize' in kinds
    else:
        assert {'bicubic', 's2v'} <= kinds
    if recurse:
        assert sum(r.name == 'prob_clfs.0.atrous.lin' for r in rec.calls) == 1 + recurse


@pytest.mark.gpu
def test_layer_parity_range(monkeypatch):
    """cr f16 with one encoder block scaled so that activations exceed 65504 (saturating FP16 twins) and the coarsest
    decoder head scaled into the FP16 subnormal range: the operand roundings and the kernels reading such operands."""
    bp = _fresh_blueprint('cr')
    net = bp.net
    big, tiny = net.nets[0].enc.body[0].body[2], net.nets[2].dec.head
    with torch.no_grad():
        big.weight.mul_(1e7)
        big.bias.mul_(1e7)
        tiny.weight.mul_(1e-5)
        tiny.bias.mul_(1e-5)
    rec, layers, _ = run_case(monkeypatch, bp, 'cr', 'f16', 1, 64, 96, dataflow=False, title='cr f16 range case')
    assert not layers.fails, '\n' + _failure_text(layers)
    by = {r.name: r for r in rec.calls}
    sat = by['nets.0.enc.body.0.body.2']
    assert bool((sat.y.abs() > F16_MAX).any()) and bool((sat.img.float().abs() == F16_MAX).any())
    assert bool((by['nets.0.enc.body.1.body.0'].x.float().abs() == F16_MAX).any())
    sub = by['nets.2.dec.head'].img.float().abs()
    assert bool(((sub > 0) & (sub < 2.0 ** -14)).float().mean() > 0.5)
    assert bool(((by['nets.2.dec.body.0.body.0'].x.float().abs() < 2.0 ** -14)
                 & (by['nets.2.dec.body.0.body.0'].x != 0)).any())


# ----------------------------------------------------------------------------------------------------------------
# planted defects: each must be reported against the right layer and the right check
# ----------------------------------------------------------------------------------------------------------------
PLANT_SHAPE = ('cr', 'f16', 1, 64, 96)


def _kinds(rep, exclude=('margin',)):
    return {(f[0], f[1]) for f in rep.fails if f[1] not in exclude}


@pytest.mark.gpu
def test_plant_zeroed_weight_tap(monkeypatch):
    """One tap of one 3x3 layer's packed FP16 weight image zeroed while the kernel runs: the per-layer numerics of
    exactly that layer fail."""
    from l3c_pytorch_b200 import engine as E
    target = 'nets.0.enc.body.1.body.2'

    def inner(fn):
        def conv2d(conv, x, **kw):
            if conv is not holder['conv']:
                return fn(conv, x, **kw)
            w_h = E._packed_obj(conv).get_f16()[0]
            saved = w_h[4].clone()
            w_h[4].zero_()
            try:
                return fn(conv, x, **kw)
            finally:
                w_h[4].copy_(saved)
        return conv2d
    holder = {}
    bp = _fresh_blueprint('cr')
    holder['conv'] = dict(bp.net.named_modules())[target]
    cfg_name, prec, N, H, W = PLANT_SHAPE
    _, layers, flow = run_case(monkeypatch, bp, cfg_name, prec, N, H, W, inner=inner, title='plant: zeroed tap')
    assert _kinds(layers) == {(target, 'numerics')}, _failure_text(layers)
    assert not flow.fails, _failure_text(flow)


@pytest.mark.gpu
def test_plant_residual_from_twin(monkeypatch):
    """A ResBlock's residual swapped for its input's FP16 operand twin: the dataflow check fails first at that
    layer's residual, while every layer's numerics (teacher-forced) still pass."""
    target = 'nets.0.dec.body.2.body.2'

    def outer(fn):
        def conv2d(conv, x, **kw):
            if conv is holder['conv']:
                kw['residual'] = rnd16(kw['residual']).float()
            return fn(conv, x, **kw)
        return conv2d
    holder = {}
    bp = _fresh_blueprint('cr')
    holder['conv'] = dict(bp.net.named_modules())[target]
    cfg_name, prec, N, H, W = PLANT_SHAPE
    _, layers, flow = run_case(monkeypatch, bp, cfg_name, prec, N, H, W, outer=outer, title='plant: residual')
    assert not _kinds(layers), _failure_text(layers)
    assert flow.fails and flow.fails[0][:2] == (target, 'residual'), _failure_text(flow)


@pytest.mark.gpu
def test_plant_swapped_atrous_slices(monkeypatch):
    """Two atrous convs write each other's channel slice of the concat buffer: the dataflow check fails at the 1x1
    `lin` conv that reads it, while the numerics of every layer pass."""
    def outer(fn):
        def conv2d(conv, x, **kw):
            if conv is holder['a0']:
                kw['out_coff'] = 64
            elif conv is holder['a1']:
                kw['out_coff'] = 0
            return fn(conv, x, **kw)
        return conv2d
    holder = {}
    bp = _fresh_blueprint('cr')
    mods = dict(bp.net.named_modules())
    holder['a0'], holder['a1'] = mods['prob_clfs.1.atrous.atrous.0'], mods['prob_clfs.1.atrous.atrous.1']
    cfg_name, prec, N, H, W = PLANT_SHAPE
    _, layers, flow = run_case(monkeypatch, bp, cfg_name, prec, N, H, W, outer=outer, title='plant: atrous slices')
    assert not _kinds(layers), _failure_text(layers)
    assert flow.fails and flow.fails[0][:2] == ('prob_clfs.1.atrous.lin', 'operand'), _failure_text(flow)


@pytest.mark.gpu
def test_plant_flipped_twin_bit(monkeypatch):
    """One bit of one FP16 element of an 'act' twin flipped after the kernel wrote it: the operand-image check of
    exactly that layer fails (the next layer, teacher-forced on the flipped operand, still passes its numerics)."""
    target = 'nets.1.enc.body.0.body.2'

    def inner(fn):
        def conv2d(conv, x, **kw):
            ret = fn(conv, x, **kw)
            if conv is holder['conv']:
                v = ret.r.view(torch.int16).view(-1)
                v[1234] ^= 0x0008
            return ret
        return conv2d
    holder = {}
    bp = _fresh_blueprint('cr')
    holder['conv'] = dict(bp.net.named_modules())[target]
    cfg_name, prec, N, H, W = PLANT_SHAPE
    _, layers, flow = run_case(monkeypatch, bp, cfg_name, prec, N, H, W, inner=inner, title='plant: flipped bit')
    assert _kinds(layers) == {(target, 'image')}, _failure_text(layers)
