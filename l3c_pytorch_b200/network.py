"""Host-side mirror of the reference's model classes for the encode/decode path.

The module tree, constructor order and parameter names replicate the reference so that
  * `torch.manual_seed(s); MultiscaleBlueprint(cfg)` yields bit-identical default-init weights, and
  * released checkpoints (`{'net': state_dict}`, /root/reference/src/helpers/saver.py:168) load with
    `load_state_dict(strict=True)`.
The nn.Conv2d objects are *parameter containers only*: no torch operator ever runs on the hot path;
`forward` methods launch the sm_90a kernels of libl3c_b200.so on NHWC fp32 buffers.

Reference classes mirrored (under /root/reference/src/modules):
  multiscale_network.py:54-130 Out | :133-165 Losses | :168-322 MultiscaleNetwork
  net.py:36-43 EncOut/DecOut | :49-62 Net | :65-80 BicubicDownsamplingEnc | :89-148 EDSRLikeEnc |
  :151-184 EDSRDec;  edsr.py:52-60 MeanShift | :63-89 ResBlock | :92-119 Upsampler;
  head.py:26-59 RGBHead/Head;  prob_clf.py:29-74;  quantizer.py:50-90
"""
from collections import namedtuple

import numpy as np
import torch
from torch import nn

from . import engine as E
from .dmll import DiscretizedMixLogisticLoss, non_shared_get_Kp

EncOut = namedtuple('EncOut', ['bn', 'bn_q', 'S', 'L', 'F'])
DecOut = namedtuple('DecOut', ['F'])

RGB_MEAN = (0.4488, 0.4371, 0.4040)


def default_conv(in_channels, out_channels, kernel_size, bias=True, rate=1, stride=1):
    """pytorch_ext.py:57-61 (padding = k//2, or the dilation rate for atrous convs)."""
    padding = kernel_size // 2 if rate == 1 else rate
    return nn.Conv2d(in_channels, out_channels, kernel_size, stride=stride, dilation=rate,
                     padding=padding, bias=bias)


conv = default_conv


def nchw_view(x_nhwc, C=None):
    """NHWC buffer -> NCHW-shaped view (channels_last strides), optionally the first C channels."""
    if C is not None:
        x_nhwc = x_nhwc[..., :C]
    return x_nhwc.permute(0, 3, 1, 2)


def to_nhwc(x_nchw, pitch=None):
    """NCHW tensor (any strides) -> contiguous NHWC fp32, zero padded to `pitch` channels."""
    E.require_cuda(x_nchw, 'input')
    x = x_nchw.permute(0, 2, 3, 1)
    C = x.shape[-1]
    if pitch is not None and pitch != C:
        out = torch.zeros(*x.shape[:3], pitch, dtype=torch.float32, device=x.device)
        out[..., :C] = x
        return out
    return x.float().contiguous()


class MeanShift(nn.Conv2d):
    """1x1 conv initialised to x/std + sign*range*mean/std (edsr.py:52-60); trainable like any
    other parameter, so it is read from the state dict, not hard-coded."""

    def __init__(self, rgb_range, rgb_mean, rgb_std, sign=-1):
        super(MeanShift, self).__init__(3, 3, kernel_size=1)
        std = torch.Tensor(rgb_std)
        self.weight.data = torch.eye(3).view(3, 3, 1, 1)
        self.weight.data.div_(std.view(3, 1, 1, 1))
        self.bias.data = sign * rgb_range * torch.Tensor(rgb_mean)
        self.bias.data.div_(std)
        self.requires_grad = False


class ResBlock(nn.Module):
    def __init__(self, conv, n_feats, kernel_size, act=None):
        super(ResBlock, self).__init__()
        # body = [conv, act, conv] -> parameter names body.0.*, body.2.* as in edsr.py:69-79
        self.body = nn.Sequential(conv(n_feats, n_feats, kernel_size), act or nn.ReLU(True),
                                  conv(n_feats, n_feats, kernel_size))

    def forward(self, x):
        """x: engine.Act.  The intermediate only feeds the second conv -> TF32-rounded in place when
        the tensor cores are on; the block output feeds the next conv AND a residual add -> both."""
        r = E.conv2d(self.body[0], x, relu=True, want='round')
        return E.conv2d(self.body[2], r, residual=x.f, want='act')           # res += x


def _run_body(body, x):
    """Sequential of ResBlocks + final conv, plus the outer skip `body(x) + x` (net.py:144,181).
    x and the result are engine.Act."""
    y = x
    for m in list(body)[:-1]:
        y = m(y)
    return E.conv2d(body[-1], y, residual=x.f, want='act')


class Upsampler(nn.Sequential):
    """conv(n_feats -> 4 n_feats, 3x3) + PixelShuffle(2), fused into one kernel epilogue."""

    def __init__(self, conv, scale, n_feats):
        assert scale == 2
        super(Upsampler, self).__init__(conv(n_feats, 4 * n_feats, 3, True), nn.PixelShuffle(2))

    def forward(self, x, want='act'):
        return E.conv2d(self[0], x, pixel_shuffle=True, want=want)


class Head(nn.Module):
    def __init__(self, config_ms, Cin):
        super(Head, self).__init__()
        assert 'Subsampling' not in config_ms.enc.cls
        self.head = conv(Cin, config_ms.Cf, config_ms.kernel_size)

    def forward(self, x):
        # the head output feeds nothing but the encoder's down-sampling conv: in f16 mode (where that conv runs
        # on the tensor cores) only its FP16 operand image is written
        return E.conv2d(self.head, x, want='round' if E.f16_mode() else 'plain')


class RGBHead(nn.Module):
    def __init__(self, config_ms):
        super(RGBHead, self).__init__()
        assert 'Subsampling' not in config_ms.enc.cls
        self.head = nn.Sequential(MeanShift(0, (0., 0., 0.), (128., 128., 128.)),
                                  Head(config_ms, Cin=3))

    def forward(self, t4):
        """t4: NHWC [N,H,W,4] = second MeanShift already applied by engine.rgb_prep."""
        return E.conv2d(self.head[1].head, t4, cin=3, want='act' if E.f16_mode() else 'plain')


class Quantizer(nn.Module):
    """Hard (eval) path of quantizer.py:62-90; fused with the to_q conv in one kernel."""

    def __init__(self, levels, sigma=1.0):
        super(Quantizer, self).__init__()
        assert levels.dim() == 1
        self.levels = levels
        self.sigma = sigma
        self.L = self.levels.size()[0]


class _Identity(nn.Module):
    def forward(self, x):
        return x


class EDSRLikeEnc(nn.Module):
    def __init__(self, config_ms, scale):
        super(EDSRLikeEnc, self).__init__()
        self.scale = scale
        self.config_ms = config_ms
        Cf = config_ms.Cf
        C, self.L = config_ms.q.C, config_ms.q.L
        self.down = conv(Cf, Cf, kernel_size=5, stride=2)
        m_body = [ResBlock(conv, Cf, config_ms.kernel_size) for _ in range(config_ms.enc.num_blocks)]
        m_body.append(conv(Cf, Cf, config_ms.kernel_size))
        self.body = nn.Sequential(*m_body)
        # to_q.1 is the reference's (parameter-free) HistogramPlot slot; keep the index layout
        self.to_q = nn.Sequential(conv(Cf, C, 1), _Identity())
        lo, hi = config_ms.q.levels_range
        self.levels = nn.Parameter(torch.linspace(lo, hi, self.L), requires_grad=False)
        self.q = Quantizer(self.levels, config_ms.q.sigma)

    def quantize_x(self, x):
        """net.py:132-134: hard-quantised values levels[argmin_l |x - level_l|] of an NCHW tensor (sampling only)."""
        lev = self.levels.detach().float()
        return lev[(x.unsqueeze(-1) - lev).abs().argmin(-1)]

    def forward(self, x):
        x = E.conv2d(self.down, x, want='act')
        F = _run_body(self.body, x)                                # engine.Act
        sym, bnq = E.quantize_head(F.f, self.to_q[0], self.levels)
        return EncOut(bnq, bnq, sym, self.L, F)


class BicubicDownsamplingEnc(nn.Module):
    """RGB baselines (net.py:65-80): the "encoder" is a Pillow bicubic x0.5 of the uint8 image."""

    def __init__(self, *_):
        super(BicubicDownsamplingEnc, self).__init__()
        self.rgb_mean = torch.tensor(RGB_MEAN, dtype=torch.float32).mul(255.)
        self._values = None

    def _consts(self, device):
        if self._values is None or self._values.device != device:
            self._values = torch.arange(256, dtype=torch.float32, device=device)
            self.rgb_mean = self.rgb_mean.to(device)
        return self._values, self.rgb_mean

    def forward(self, img_u8):
        """img_u8: uint8 planes [N,3,H,W] (the clamp/round of x+mean in the reference is the
        identity on integer images)."""
        sym = E.bicubic_half(img_u8)
        values, mean = self._consts(img_u8.device)
        bn = E.symbols_to_values(sym, values, mean)
        return EncOut(bn, bn, sym, 256, None)


class EDSRDec(nn.Module):
    def __init__(self, config_ms, scale):
        super(EDSRDec, self).__init__()
        self.scale = scale
        Cf = config_ms.Cf
        self.head = conv(config_ms.q.C, Cf, 1)
        m_body = [ResBlock(conv, Cf, config_ms.kernel_size) for _ in range(config_ms.dec.num_blocks)]
        m_body.append(conv(Cf, Cf, config_ms.kernel_size))
        self.body = nn.Sequential(*m_body)
        self.tail = Upsampler(conv, 2, Cf)

    def forward(self, bn8, features_to_fuse=None, operand_only=False):
        """bn8: NHWC [N,h,w,8] (q.C channels used); features_to_fuse: engine.Act or tensor or None.
        operand_only: the features feed nothing but the probability classifier's tensor-core convs (finest
        scale) -> in f16 mode only their FP16 operand image is written."""
        fuse = features_to_fuse.f if isinstance(features_to_fuse, E.Act) else features_to_fuse
        x = E.conv2d(self.head, bn8, residual=fuse, want='act')       # head(x) + F_prev
        x = _run_body(self.body, x)
        return DecOut(self.tail(x, 'round' if (operand_only and E.f16_mode()) else 'act'))   # engine.Act


class Net(nn.Module):
    def __init__(self, config_ms, scale):
        super(Net, self).__init__()
        self.config_ms = config_ms
        self.enc = {'EDSRLikeEnc': EDSRLikeEnc,
                    'BicubicSubsampling': BicubicDownsamplingEnc}[config_ms.enc.cls](config_ms, scale)
        self.dec = {'EDSRDec': EDSRDec}[config_ms.dec.cls](config_ms, scale)

    def forward(self, x):
        raise NotImplementedError()  # call .enc / .dec


class StackedAtrousConvs(nn.Module):
    def __init__(self, atrous_rates_str, Cin, Cout, bias=True, kernel_size=3):
        super(StackedAtrousConvs, self).__init__()
        rates = [atrous_rates_str] if isinstance(atrous_rates_str, int) else \
            list(map(int, atrous_rates_str.split(',')))
        self.atrous = nn.ModuleList([conv(Cin, Cin, kernel_size, rate=r) for r in rates])
        self.lin = conv(len(rates) * Cin, Cout, 1, bias=bias)

    def forward(self, x, fused=None):
        """x: engine.Act -> NHWC parameter tensor; or, with fused = (sym uint8 planes, dmll) in f16 mode, the
        coding intervals of `sym` (the DMLL head runs in the 1x1 conv's epilogue: engine.lin_dmll_intervals); with
        fused = (sym, dmll, (oy, y0, h, tile, out)) those of one band of a banded encode, x being the band's decoder
        window (engine.lin_dmll_intervals_band)."""
        src = x.f if x.f is not None else x.r
        N, H, W = src.shape[:3]
        Cin = self.atrous[0].in_channels
        # f16 modes: the concat buffer IS the FP16 operand image of the 1x1 conv (f16x2: the split image, hi | lo)
        f16 = E.f16_mode() or E.f16x2_mode()
        cat = torch.empty(N, H, W, Cin * len(self.atrous) * (2 if E.f16x2_mode() else 1), device=src.device,
                          dtype=torch.float16 if f16 else torch.float32)
        for i, a in enumerate(self.atrous):
            # concat by channel slice; `cat` only feeds the 1x1 conv -> TF32-rounded in place when the
            # tensor cores are on
            E.conv2d(a, x, out=cat, out_coff=i * Cin, want='round')
        if fused is not None:
            sym, dm = fused[:2]
            C = sym.shape[1]
            K = self.lin.out_channels // ((4 if dm.rgb_scale else 3) * C)
            if len(fused) > 2:
                oy, y0, h, tile, out = fused[2]
                return E.lin_dmll_intervals_band(self.lin, cat, oy, sym, y0, h, dm.targets(cat.device), C, K, dm.L,
                                                 dm.rgb_scale, tile, out=out)
            return E.lin_dmll_intervals(self.lin, cat, sym, dm.targets(cat.device), C, K, dm.L, dm.rgb_scale)
        return E.conv2d(self.lin, E.Act(None, cat) if f16 else cat)


class AtrousProbabilityClassifier(nn.Module):
    def __init__(self, config_ms, C=3, atrous_rates_str='1,2,4'):
        super(AtrousProbabilityClassifier, self).__init__()
        K = config_ms.prob.K
        self.atrous = StackedAtrousConvs(atrous_rates_str, config_ms.Cf, non_shared_get_Kp(K, C),
                                         kernel_size=config_ms.kernel_size)

    def forward(self, x, fused=None):
        return self.atrous(x, fused)


class Out(object):
    """Outputs of the network, fine -> coarse (multiscale_network.py:54-130).  Public attributes
    follow the reference (NCHW-shaped tensors); the device-resident buffers the bit-coder consumes
    are kept beside them: `S_u8` uint8 planes [N,C,H,W], `bn8` NHWC pitch-8, `P_nhwc`."""

    def __init__(self, targets_style='S', auto_recursive_from=None):
        assert targets_style in ('S', 'bn')
        self.S_u8, self.bn8, self.P_nhwc, self.L = [], [], [], []
        self.IV = None          # per scale: coding intervals from the fused head (forward(intervals_of=...)), P is None then
        self.extents = None     # ragged batch (forward(extents=...)): [(h_n, w_n)] of every image at the finest scale
        self.auto_recursive_from = auto_recursive_from
        self.targets_style = targets_style

    # reference-shaped accessors
    @property
    def S(self):
        return [s.long() if s is not None else None for s in self.S_u8]

    @property
    def bn(self):
        out = []
        for b, s in zip(self.bn8, self.S_u8):
            out.append(None if b is None else nchw_view(b, s.shape[1]))
        return out

    @property
    def P(self):
        return [None if p is None else nchw_view(p) for p in self.P_nhwc]

    def append_input_image(self, img_u8):
        self.S_u8.append(img_u8)
        self.L.append(256)
        self.bn8.append(None)

    def append(self, enc_out, P, is_training=False):
        self.S_u8.append(enc_out.S)
        self.L.append(enc_out.L)
        self.P_nhwc.append(P)
        self.bn8.append(enc_out.bn_q)
        assert len(self.S_u8) == len(self.L) == len(self.bn8) == len(self.P_nhwc) + 1

    def extents_at(self, i):
        """Ragged batch: [(h_n, w_n)] of every image at the resolution of S_u8[i] (scale index, -1 the coarsest)."""
        s = i % len(self.S_u8)
        return [(h >> s, w >> s) for (h, w) in self.extents]

    def get_nat_count(self, i):
        if self.extents is not None:
            return float(self.get_nat_counts_per_image(i).sum())
        N, C, H, W = self.S_u8[i].shape
        return N * C * H * W * np.log(self.L[i])

    def get_nat_counts_per_image(self, i):
        """Uniform-prior nats of S_u8[i] for every image, float64 [N]: priced over each image's own extent in a
        ragged batch, exactly as get_nat_count() of that image alone."""
        N, C, H, W = self.S_u8[i].shape
        ext = self.extents_at(i) if self.extents is not None else [(H, W)] * N
        return np.array([C * h * w * np.log(self.L[i]) for (h, w) in ext], np.float64)


class Losses(nn.Module):
    def __init__(self, config_ms):
        super(Losses, self).__init__()
        self.loss_dmol_rgb = DiscretizedMixLogisticLoss(rgb_scale=True, x_min=0, x_max=255, L=256)
        if config_ms.rgb_bicubic_baseline:
            self.loss_dmol_n = self.loss_dmol_rgb
        else:
            x_min, x_max = config_ms.q.levels_range
            self.loss_dmol_n = DiscretizedMixLogisticLoss(rgb_scale=False, x_min=x_min, x_max=x_max,
                                                          L=config_ms.q.L)

    def get(self, out):
        """(per-scale costs in nats [python floats, summed over the batch], uniform-scale nats,
        number of sub-pixels) -- multiscale_network.py:145-165.  A ragged Out (Out.extents) counts every image over
        its own extent only, never the padding."""
        if out.extents is not None:
            costs, uniform, num_subpixels = self.get_per_image(out)
            return [float(c.sum()) for c in costs], float(uniform.sum()), int(num_subpixels.sum())
        costs = [float(self.loss_dmol_rgb.nll_sum(out.S_u8[0], out.P_nhwc[0]).sum())]
        for s in range(1, len(out.P_nhwc)):
            costs.append(float(self.loss_dmol_n.nll_sum(out.S_u8[s], out.P_nhwc[s]).sum()))
        final_idx = -1 if out.auto_recursive_from is None else out.auto_recursive_from
        return costs, out.get_nat_count(final_idx), int(np.prod(out.S_u8[0].shape))

    def get_per_image(self, out):
        """Same quantities as get(), kept apart per image of the batch: (per-scale nats as float64
        arrays [N], uniform-scale nats of ONE image, sub-pixels of ONE image).
        A ragged Out (Out.extents): every image over its own extent, (h_n >> s, w_n >> s) at scale s, bit-identical to
        the Out of that image alone; the uniform-scale nats and the sub-pixels are then arrays [N] as well."""
        if out.extents is not None:
            dms = [self.loss_dmol_rgb] + [self.loss_dmol_n] * (len(out.P_nhwc) - 1)
            costs = [dm.nll_sum(out.S_u8[s], out.P_nhwc[s], extents=out.extents_at(s)).double().cpu().numpy()
                     for s, dm in enumerate(dms)]
            final_idx = -1 if out.auto_recursive_from is None else out.auto_recursive_from
            subpixels = np.array([out.S_u8[0].shape[1] * h * w for (h, w) in out.extents], np.int64)
            return costs, out.get_nat_counts_per_image(final_idx), subpixels
        costs = [self.loss_dmol_rgb.nll_sum(out.S_u8[0], out.P_nhwc[0]).double().cpu().numpy()]
        for s in range(1, len(out.P_nhwc)):
            costs.append(self.loss_dmol_n.nll_sum(out.S_u8[s], out.P_nhwc[s]).double().cpu().numpy())
        final_idx = -1 if out.auto_recursive_from is None else out.auto_recursive_from
        n = out.S_u8[0].shape[0]
        return costs, out.get_nat_count(final_idx) / n, int(np.prod(out.S_u8[0].shape[1:]))


class MultiscaleNetwork(nn.Module):
    def __init__(self, config_ms):
        super(MultiscaleNetwork, self).__init__()
        self._rgb = config_ms.rgb_bicubic_baseline
        self._fuse_feat = config_ms.dec.skip
        self.sub_rgb_mean = MeanShift(255., RGB_MEAN, (1.0, 1.0, 1.0))
        self.scales = config_ms.num_scales
        self.config_ms = config_ms
        if not config_ms.rgb_bicubic_baseline:
            heads = [RGBHead(config_ms)] + [Head(config_ms, Cin=self.get_Cin_for_scale(s))
                                            for s in range(self.scales - 1)]
            nets = [Net(config_ms, s) for s in range(self.scales)]
            prob_clfs = [AtrousProbabilityClassifier(config_ms, C=3)] + \
                        [AtrousProbabilityClassifier(config_ms, config_ms.q.C)
                         for _ in range(self.scales - 1)]
        else:
            heads = [_Identity() for _ in range(self.scales)]
            nets = [Net(config_ms, s) for s in range(self.scales)]
            prob_clfs = [AtrousProbabilityClassifier(config_ms, C=3) for _ in range(self.scales)]
        self.heads = nn.ModuleList(heads)
        self.nets = nn.ModuleList(nets)
        self.prob_clfs = nn.ModuleList(prob_clfs)

    def get_losses(self):
        return Losses(self.config_ms)

    def get_Cin_for_scale(self, scale):
        return self.config_ms.Cf if self.config_ms.enc.feed_F else self.config_ms.q.C

    def fuses(self, scale):
        """Whether the decoder of `scale` adds the coarser decoder's features (dec.skip), by _forward's rule: no
        features cross into or out of a recursive scale (scale >= num_scales), and the coarsest trained scale gets
        none."""
        return bool(self._fuse_feat) and scale < self.scales - 1

    # ------------------------------------------------------------------------------------------
    @staticmethod
    def _as_u8_planes(x):
        """Accepts what the reference accepts (NCHW float/long 0..255) and uint8; returns
        contiguous uint8 planes on the device."""
        E.require_cuda(x, 'image batch')
        if x.dim() == 3:
            x = x.unsqueeze(0)
        if x.dtype != torch.uint8:
            x = x.round().clamp(0, 255).to(torch.uint8)
        return x.contiguous()

    def _rgb_head_input(self, img):
        """What feeds the first encoder: in f16 mode the OUTPUT of heads[0] (MeanShift x2 + 3 -> Cf conv, computed as
        im2col + tensor-core GEMM, engine.rgb_head_f16) as an engine.Act; otherwise the normalised image for
        heads[0] to convolve on the CUDA cores."""
        if E.f16_mode() and self.heads[0].head[1].head.out_channels % 2 == 0:
            return E.rgb_head_f16(img, self.sub_rgb_mean, self.heads[0].head[0], self.heads[0].head[1].head)
        return E.rgb_prep(img, self.sub_rgb_mean, self.heads[0].head[0])[1]

    def ragged_unsupported(self, auto_recurse=0):
        """Why this network cannot run a ragged batch (a message naming it), or None when it can."""
        if self._rgb:
            return 'ragged batches are not supported by the RGB baselines (bicubic encoder)'
        if auto_recurse:
            return 'ragged batches are not supported with auto_recurse'
        if not E.f16_mode():
            return 'ragged batches run in precision f16 only, not %s' % E.get_conv_precision()
        return None

    def windows_unsupported(self):
        """Why this network cannot run a decoder on a ragged batch of region windows (get_P_nhwc(windows=)), or None
        when it can.  Only the decoder and classifier convs run there, so unlike ragged_unsupported this allows the RGB
        baselines, recursive scales and f16x2."""
        if not (E.f16_mode() or E.f16x2_mode()):
            return 'ragged decoder windows run in precision f16 or f16x2 only, not %s' % E.get_conv_precision()
        return None

    def _check_ragged(self, extents, auto_recurse=0):
        why = None if extents is None else self.ragged_unsupported(auto_recurse)
        if why is not None:
            raise NotImplementedError(why)

    def forward(self, x, auto_recurse=0, intervals_of=None, extents=None):
        """intervals_of: a Losses object -> encode-side pass in f16 mode: the probability heads emit the coding
        intervals of the symbols directly (Out.IV) and no parameter tensor is materialised (Out.P entries None).

        extents: [(h_n, w_n)] -> `x` is a ragged batch (DESIGN §4.6, f16 only): image n occupies [0, h_n) x [0, w_n)
        of the padded batch (multiples of 2**num_scales, zero outside) and every output inside an image's extent at
        every scale is bit-identical to the forward of that image alone; outside it the outputs are unspecified.

        x: image batch NCHW in [0,255] (uint8 / long / float).  Eval-mode forward
        (multiscale_network.py:226-306) -> Out.  auto_recurse: how many times the last trained scale is
        applied again (theoretical-bpsp evaluation of the RGB-shared baseline, `--recursive`;
        multiscale_network.py:235-238,291-294); the extra scales use scale index -1, never fuse decoder
        features, and `Out.auto_recursive_from` marks where they start."""
        img = self._as_u8_planes(x)
        self._check_ragged(extents, auto_recurse)
        with E.ragged_extents(extents, img.shape[2], img.shape[3]):
            out = self._forward(img, auto_recurse, intervals_of)
        if extents is not None:
            out.extents = [(int(h), int(w)) for (h, w) in extents]
        return out

    def _forward(self, img, auto_recurse, intervals_of):
        forward_scales = list(range(self.scales)) + [-1] * int(auto_recurse)
        out = Out(targets_style='S' if self._rgb else 'bn',
                  auto_recursive_from=self.scales if auto_recurse > 0 else None)
        out.append_input_image(img)
        enc_outs = []
        if self._rgb:
            inp = img
            for s in forward_scales:
                eo = self.nets[s].enc(inp)
                enc_outs.append(eo)
                inp = eo.S
        else:
            inp = self._rgb_head_input(img)
            for i, s in enumerate(forward_scales):
                h = inp if (i == 0 and isinstance(inp, E.Act)) else self.heads[s](inp)
                eo = self.nets[s].enc(h)
                enc_outs.append(eo)
                inp = eo.F                                  # enc.feed_F
        dec_F = [None] * len(forward_scales)
        prev = None
        for i, s in reversed(list(enumerate(forward_scales))):
            # no fusion for: disabled / auto-recursive scales / the final trained scale
            fuse = prev if (self._fuse_feat and s != -1 and s != max(forward_scales)) else None
            # the features of scale 0 and of the recursive scales feed nothing but their probability classifier
            prev = self.nets[s].dec(enc_outs[i].bn_q, fuse, operand_only=(i == 0 or s == -1)).F
            dec_F[i] = prev
        fuse_iv = (intervals_of is not None and E.f16_mode() and
                   all(self.prob_clfs[s].atrous.lin.in_channels % 64 == 0 for s in forward_scales))
        if fuse_iv:
            out.IV = []
        for i, s in enumerate(forward_scales):
            if fuse_iv:
                dm = intervals_of.loss_dmol_rgb if i == 0 else intervals_of.loss_dmol_n
                C = out.S_u8[i].shape[1]
                if (dm.rgb_scale and C == 3) or (not dm.rgb_scale and C == 5):
                    out.IV.append(self.prob_clfs[s](dec_F[i], fused=(out.S_u8[i], dm)))
                    out.append(enc_outs[i], None)
                    continue
                out.IV.append(None)
            out.append(enc_outs[i], self.prob_clfs[s](dec_F[i]))
        return out

    def sample_forward(self, x, losses, sample_scales, partial_final=None, auto_recurse=0):
        """multiscale_network.py:328-406 (test.py --sample): encode x, then decode coarse -> fine, replacing
        the bottlenecks of the scales in `sample_scales` (and always the image itself) by samples from the
        predicted distributions; the coarsest sampled bottleneck is drawn uniformly.  Returns the sampled
        image, NCHW float in [0, 255]."""
        if auto_recurse != 0:
            raise NotImplementedError('Currently not supported for sampling: autorecurse={}'.format(auto_recurse))
        if self._rgb:
            raise NotImplementedError('sampling is built for the L3C configurations (learned bottlenecks)')
        print('-' * 40)
        print('- Sampling {}'.format(sample_scales))
        print('-' * 40)
        img = self._as_u8_planes(x)
        forward_scales = list(range(self.scales))
        enc_outs, Cs = [], [3]
        inp = self._rgb_head_input(img)
        for i, s in enumerate(forward_scales):
            eo = self.nets[s].enc(inp if (i == 0 and isinstance(inp, E.Act)) else self.heads[s](inp))
            Cs.append(eo.S.shape[1])
            enc_outs.append(eo)
            inp = eo.F
        prev_x, fuse = None, None
        for scale in reversed(forward_scales):
            loss_dmm = losses.loss_dmol_rgb if scale == 0 else losses.loss_dmol_n
            C = Cs[scale]
            if scale in sample_scales:
                if prev_x is None:
                    print('Sampling uniformly!')
                    last = enc_outs[-1]
                    n, c, h, w = last.S.shape
                    fake = torch.empty(n, c, h, w, dtype=torch.float32, device=img.device).uniform_(-1, 1)
                    prev_x = self.nets[-1].enc.quantize_x(fake)
                    if partial_final:
                        print('partial sampling')
                        bnq = nchw_view(enc_outs[scale].bn_q, c)
                        for ch in partial_final:
                            prev_x[:, ch, ...] = bnq[:, ch, ...]
                print('{}: Feeding sampled to decoder'.format(scale))
                dec_in = to_nhwc(prev_x, 8)
            else:
                print('{}: Feeding encoder output to decoder'.format(scale))
                dec_in = enc_outs[scale].bn_q
            F = self.nets[scale].dec(dec_in, fuse, operand_only=(scale == 0)).F
            if self._fuse_feat:
                fuse = F
            P = self.prob_clfs[scale](F)
            if scale == 0 or scale - 1 in sample_scales:
                print('{}: sampling N{}HW for next scale'.format(scale, C))
                prev_x = loss_dmm.sample(nchw_view(P), C=C)
        return prev_x

    def get_P_nhwc(self, scale, bn8, dec_F_prev=None, need_F=False, extents=None, windows=None, fused=None):
        """-> (parameters NHWC, decoder features as engine.Act for the next finer scale).  At scale 0 the
        features feed nothing else (need_F=True keeps their fp32 tensor for the reference-shaped get_P).
        extents: [(h_n, w_n)] at the FINEST scale -> bn8 is a ragged batch (forward()).
        windows: [(h_n, w_n)] at bn8's own resolution -> bn8 (and dec_F_prev) is a padded batch of region windows of
        different sizes (DESIGN §4.8), window n top-left; the outputs inside 2 x window n are bit-identical to a run
        on that window alone (windows_unsupported).
        scale >= num_scales: a recursive scale of forward(auto_recurse=R) (RGB baselines), num_scales + k the k-th
        extra application of the last trained scale: nets[-1] / prob_clfs[-1], no features in or out (like scale 0,
        its features feed nothing but its probability classifier).  The bit-coder decodes recursive scales of the
        RGB baselines only (codec.BatchCodec).
        fused: the probability classifier's `fused` argument (StackedAtrousConvs.forward): the first result is then the
        coding intervals instead of the parameters."""
        ns = self.config_ms.num_scales
        recursive = scale >= ns
        assert 0 <= scale, 'Out of range: {}'.format(scale)
        if recursive and dec_F_prev is not None:
            raise ValueError('recursive scale %d takes no decoder features' % scale)
        f = 2 ** (scale + 1)
        if windows is not None:
            assert extents is None, 'extents and windows exclude each other'
            why = self.windows_unsupported()
            if why is not None:
                raise NotImplementedError(why)
            extents, f = [(2 * int(h), 2 * int(w)) for (h, w) in windows], 2
        else:
            self._check_ragged(extents, int(recursive))
        s = -1 if recursive else scale
        with E.ragged_extents(extents, bn8.shape[1] * f, bn8.shape[2] * f):
            F = self.nets[s].dec(bn8, dec_F_prev, operand_only=((scale == 0 or recursive) and not need_F)).F
            return self.prob_clfs[s](F, fused), F

    def get_P(self, scale, bn_q, dec_F_prev=None):
        """multiscale_network.py:308-322 with NCHW-shaped tensors in and out."""
        bn8 = to_nhwc(bn_q, 8)
        Fp = None if dec_F_prev is None else to_nhwc(dec_F_prev)
        l, F = self.get_P_nhwc(scale, bn8, Fp, need_F=True)
        return nchw_view(l), nchw_view(F.f)
