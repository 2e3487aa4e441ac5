"""MultiscaleBlueprint: API facade of the model + losses
(/root/reference/src/blueprints/multiscale_blueprint.py:42-150), backed by the sm_90a kernels."""
from collections import namedtuple

import numpy as np
import torch
from torch import nn

from . import pad as _pad
from .network import MultiscaleNetwork, Out

MultiscaleLoss = namedtuple('MultiscaleLoss', ['loss_pc', 'nonrecursive_bpsps', 'recursive_bpsps'])

DEVICE = torch.device('cuda:0')


class MultiscaleBlueprint(nn.Module):
    def __init__(self, config_ms, device=None):
        super(MultiscaleBlueprint, self).__init__()
        net = MultiscaleNetwork(config_ms)          # default init on the CPU generator, as the reference
        self.device = torch.device(device) if device is not None else DEVICE
        if torch.cuda.is_available():
            net.to(self.device)
        self.net = net
        self.losses = net.get_losses()

    def set_eval(self):
        self.net.eval()
        self.losses.loss_dmol_rgb.eval()
        self.losses.loss_dmol_n.eval()
        return self

    def forward(self, in_batch, auto_recurse=0, extents=None) -> Out:
        """in_batch: NCHW 0..255 (float / long / uint8) on the GPU.  extents: [(h_n, w_n)] -> a ragged batch
        (MultiscaleNetwork.forward): the losses of the returned Out cover every image's own extent only."""
        if self.device.type != 'cuda':
            return self.net(in_batch, auto_recurse, extents=extents)   # raises: there is no CPU path
        with torch.cuda.device(self.device):          # kernels launch on the CURRENT device
            return self.net(in_batch, auto_recurse, extents=extents)

    def forward_for_coding(self, in_batch, auto_recurse=0) -> Out:
        """forward() for the bit-coder: in f16 mode the DMLL head is fused into the 1x1 convs of the probability
        classifiers and `Out.IV` holds the coding intervals instead of `Out.P` the parameters (recursive scales
        included)."""
        if self.device.type != 'cuda':
            return self.net(in_batch, auto_recurse, intervals_of=self.losses)
        with torch.cuda.device(self.device):
            return self.net(in_batch, auto_recurse, intervals_of=self.losses)

    def get_loss(self, out: Out, num_subpixels_before_pad=None) -> MultiscaleLoss:
        """Theoretical bpsp per scale, incl. the uniform-prior final scale
        (multiscale_blueprint.py:64-95)."""
        costs, final_cost_uniform, num_subpixels = self.losses.get(out)
        if num_subpixels_before_pad:
            assert num_subpixels_before_pad <= num_subpixels, num_subpixels_before_pad
            num_subpixels = num_subpixels_before_pad
        conversion = np.log(2.) * num_subpixels
        costs_bpsp = [cost / conversion for cost in costs]
        nonrecursive_bpsps = costs_bpsp[:out.auto_recursive_from] + [final_cost_uniform / conversion]
        recursive_bpsps = None
        if out.auto_recursive_from is not None:
            # non-recursive AND recursive scales, plus the uniform-prior cost of the very last scale
            recursive_bpsps = costs_bpsp + [out.get_nat_count(-1) / conversion]
        return MultiscaleLoss(sum(costs_bpsp), nonrecursive_bpsps, recursive_bpsps)

    def sample_forward(self, in_batch, sample_scales, partial_final=None):
        """multiscale_blueprint.py:97-98"""
        with torch.cuda.device(self.device):
            return self.net.sample_forward(in_batch, self.losses, sample_scales, partial_final)

    def get_loss_per_image(self, out: Out, num_subpixels_before_pad=None):
        """Total theoretical bpsp (all scales + the uniform-prior final scale) of every image of the
        batch, as a list of floats: what get_loss() gives for a batch of one, without running the
        images one at a time.  `num_subpixels_before_pad` counts ONE image (an int), or is one count per image (a
        sequence), e.g. the unpadded sub-pixels of every image of a ragged batch (Out.extents)."""
        costs, final_cost_uniform, num_subpixels = self.losses.get_per_image(out)
        if num_subpixels_before_pad is not None and np.ndim(num_subpixels_before_pad) > 0:
            num_subpixels_before_pad = np.asarray(num_subpixels_before_pad, np.int64)
            assert num_subpixels_before_pad.shape == (out.S_u8[0].shape[0],), num_subpixels_before_pad.shape
        if np.ndim(num_subpixels_before_pad) > 0 or num_subpixels_before_pad:
            assert np.all(num_subpixels_before_pad <= num_subpixels), num_subpixels_before_pad
            num_subpixels = num_subpixels_before_pad
        if out.auto_recursive_from is not None:                  # sum(recursive_bpsps): the last scale is the uniform one
            final_cost_uniform = out.get_nat_count(-1) / out.S_u8[0].shape[0]
        total = sum(costs) + final_cost_uniform                  # numpy float64 [N]
        return (total / (np.log(2.) * num_subpixels)).tolist()

    def unpack_batch_pad(self_or_raw, raw_or_fac=None, fac=None):
        """Reference signature `unpack_batch_pad(raw, fac)` (static, multiscale_blueprint.py:121-131: the
        module-level DEVICE); called on an instance (`bp.unpack_batch_pad(raw, fac)`) the batch goes to
        that blueprint's own device."""
        if isinstance(self_or_raw, MultiscaleBlueprint):
            device, raw = self_or_raw.device, raw_or_fac
        else:
            device, raw, fac = DEVICE, self_or_raw, (raw_or_fac if fac is None else fac)
        if len(raw.shape) == 3:
            raw = raw.unsqueeze(0)
        assert len(raw.shape) == 4
        raw = MultiscaleBlueprint.pad(raw, fac)
        raw = raw.to(device)
        return raw.float(), raw.long()

    @staticmethod
    def pad(raw, fac):
        raw, _ = _pad.pad(raw, fac, mode=MultiscaleBlueprint.get_padding_mode())
        return raw

    @staticmethod
    def get_padding_mode():
        return 'constant'
