"""Host mirror of DiscretizedMixLogisticLoss (/root/reference/src/criterion/logistic_mixture.py:
86-275): the value grid (x_min, x_max, L, bin_width), to_sym/to_bn, the per-channel CDF parameters
(`cdf_step_non_shared` -> CDFOut) and the NLL -- all evaluated by kernels of libl3c_b200.so.

Decode-side repair built in (SURVEY.md finding 1): `to_bn` maps symbols through the same
`linspace` LUT the encoder's quantizer uses, instead of `S*bin + x_min`, which differs by 1 ulp for
14 of the 25 levels and desynchronises the decoder in the unmodified reference.
"""
from collections import namedtuple

import torch
from torch import nn

from . import engine as E

_NUM_PARAMS_RGB = 4      # pi, mu, sigma, lambda
_NUM_PARAMS_OTHER = 3    # pi, mu, sigma
_LOG_SCALES_MIN = -7.

CDFOut = namedtuple('CDFOut', ['logit_probs_c_sm', 'means_c', 'log_scales_c', 'K', 'targets'])


def non_shared_get_Kp(K, C):
    return (_NUM_PARAMS_RGB if C == 3 else _NUM_PARAMS_OTHER) * C * K


def non_shared_get_K(Kp, C):
    return Kp // ((_NUM_PARAMS_RGB if C == 3 else _NUM_PARAMS_OTHER) * C)


class DiscretizedMixLogisticLoss(nn.Module):
    def __init__(self, rgb_scale, x_min=0, x_max=255, L=256):
        super(DiscretizedMixLogisticLoss, self).__init__()
        self.rgb_scale = rgb_scale
        self.x_min, self.x_max, self.L = x_min, x_max, L
        self.use_coeffs = rgb_scale
        self._num_params = _NUM_PARAMS_RGB if rgb_scale else _NUM_PARAMS_OTHER
        self.bin_width = (x_max - x_min) / (L - 1)
        self.x_lower_bound = x_min + 0.001
        self.x_upper_bound = x_max - 0.001
        self._cache = {}

    def extra_repr(self):
        return 'DMLL: x={}, L={}, coeffs={}, P={}, bin_width={}'.format(
            (self.x_min, self.x_max), self.L, self.use_coeffs, self._num_params, self.bin_width)

    # ---- constant tables (host computed once, cached per device) ---------------------------
    def values(self, device):
        """value of every symbol: linspace(x_min, x_max, L) -- identical to the quantiser levels
        (net.py:125) for the bottleneck scales and to 0..255 for RGB."""
        key = ('values', str(device))
        if key not in self._cache:
            self._cache[key] = torch.linspace(self.x_min, self.x_max, self.L,
                                              dtype=torch.float32).to(device)
        return self._cache[key]

    def targets(self, device):
        """bin edges, coders_helpers.py:44-46."""
        key = ('targets', str(device))
        if key not in self._cache:
            self._cache[key] = torch.linspace(self.x_min - self.bin_width / 2,
                                              self.x_max + self.bin_width / 2, self.L + 1,
                                              dtype=torch.float32).to(device)
        return self._cache[key]

    # ---- symbols <-> values --------------------------------------------------------------------
    def to_sym(self, x):
        """quantizer.py:38-41 (tiny host-side helper, torch elementwise)."""
        bin_size = (self.x_max - self.x_min) / (self.L - 1)
        return x.clamp(self.x_min, self.x_max).sub(self.x_min).div(bin_size).round().long()

    def to_bn(self, S):
        """values[S] through the shared LUT (see module docstring)."""
        return self.values(S.device)[S.long()]

    # ---- kernels -------------------------------------------------------------------------------
    def _nhwc(self, l):
        """accepts the reference's NKpHW tensors (any strides) or NHWC buffers."""
        if l.dim() == 4 and l.stride(1) == 1 and l.is_contiguous(memory_format=torch.channels_last):
            return l.permute(0, 2, 3, 1)            # already NHWC memory
        return l.permute(0, 2, 3, 1).contiguous()

    def cdf_step_non_shared(self, l, targets, c_cur, C, x_c=None):
        """logistic_mixture.py:134-141.  l: NKpHW-shaped tensor; x_c: NCHW values decoded so far."""
        assert c_cur < C
        lh = self._nhwc(l)
        K = non_shared_get_K(lh.shape[-1], C)
        xd = None
        if self.use_coeffs and c_cur > 0:
            assert x_c is not None
            xd = x_c.float().contiguous()
        pi, mu, ls = E.dmll_channel_params(lh, xd, C, K, self.rgb_scale, c_cur)
        return CDFOut(pi, mu, ls, K, targets.to(l.device))

    def sample(self, l, C, u_sel=None, u_x=None):
        """logistic_mixture.py:143-144,277-323: one sample per sub-pixel.  l: NKpHW-shaped tensor -> NCHW float
        (RGB: clamped to [0, 255], not rounded).  u_sel [N,C,K,H,W] / u_x [N,C,H,W]: the uniform random
        numbers (default: drawn here from the device generator, in [1e-5, 1 - 1e-5] as in the reference)."""
        lh = self._nhwc(l)
        N, H, W, Kp = lh.shape
        K = non_shared_get_K(Kp, C)
        if u_sel is None:
            u_sel = torch.empty(N, C, K, H, W, dtype=torch.float32, device=lh.device).uniform_(1e-5, 1. - 1e-5)
        if u_x is None:
            u_x = torch.empty(N, C, H, W, dtype=torch.float32, device=lh.device).uniform_(1e-5, 1. - 1e-5)
        return E.dmll_sample(lh.contiguous(), u_sel, u_x, C, K, self.use_coeffs)

    def nll_sum(self, sym_u8, l_nhwc, want_map=False, extents=None):
        """per-image NLL in nats (float64 [N]) of uint8 symbol planes under NHWC parameters.
        extents: [(h_n, w_n)] at this resolution -> a ragged batch: image n is summed over [0, h_n) x [0, w_n) only,
        bit-identical to its own call (no per-sub-pixel map)."""
        C = sym_u8.shape[1]
        K = non_shared_get_K(l_nhwc.shape[-1], C)
        if extents is not None:
            if want_map:
                raise NotImplementedError('per-sub-pixel NLL maps are not built for ragged batches')
            return E.dmll_nll_ragged(l_nhwc, sym_u8, self.values(l_nhwc.device), C, K, self.L, self.rgb_scale,
                                     self.x_min, self.x_max, extents)
        s, m = E.dmll_nll(l_nhwc, sym_u8, self.values(l_nhwc.device), C, K, self.L, self.rgb_scale,
                          self.x_min, self.x_max, want_map)
        return (s, m) if want_map else s

    def forward(self, x, l, scale=0):
        """logistic_mixture.py:146-207: x NCHW values on the grid, l NKpHW -> NCHW nats."""
        sym = self.to_sym(x).to(torch.uint8).contiguous()
        _, m = self.nll_sum(sym, self._nhwc(l), want_map=True)
        return m
