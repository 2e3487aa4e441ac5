"""Thin Python wrappers over the C ABI: PyTorch tensors are only the *containers* (device memory,
streams); every computation on the hot path is a kernel of libl3c_b200.so.

Activation convention inside the package: NHWC fp32 contiguous tensors `[N, H, W, pitch]`.
"""
import contextlib
import ctypes
import os

import numpy as np
import torch

from . import _lib
from ._lib import lib, check, ConvDesc

# default conv precision: env L3C_CONV_PRECISION (fp32 | tf32 | f16); see set_conv_precision
LAUNCHES = {'n': 0}        # kernels of libl3c_b200.so launched through this module (bench.py reports it)
_PRECISION = {'mode': _lib.PRECISIONS[os.environ.get('L3C_CONV_PRECISION', 'fp32')]}


def set_conv_precision(name):
    """'fp32' (CUDA-core FFMA, bit-faithful ordering), 'tf32' (wgmma kind::tf32 on TF32-RN operands),
    'f16' (wgmma kind::f16 on FP16-RN operand images: same 10 mantissa bits, half the bytes and MMAs)."""
    _PRECISION['mode'] = _lib.PRECISIONS[name]


def get_conv_precision():
    return {v: k for k, v in _lib.PRECISIONS.items()}[_PRECISION['mode']]


def launch_log(reset=False):
    """-> ({kernel name: launches}, total) counted INSIDE libl3c_b200.so at its launch sites since the last
    reset (l3c_launch_log): which kernels really ran, e.g. per precision mode in smoke()."""
    buf = ctypes.create_string_buffer(8192)
    total = lib.l3c_launch_log(buf, len(buf), 1 if reset else 0)
    out = {}
    for line in buf.value.decode().splitlines():
        name, n = line.rsplit(' ', 1)
        out[name] = int(n)
    return out, int(total)


def _stream_ptr():
    # the raw handle of the current stream of the current device (torch.cuda.current_stream() builds a Python
    # Stream object per call: 12 us x ~600 launches per step on the host thread that feeds three decode lanes)
    return ctypes.c_void_p(torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice()))


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


_PARTITIONS = {}


def partition_streams(device, sm_a, n_a, n_b):
    """Streams confined to two disjoint SM groups of `device` (l3c_partition_streams):
    -> (streams_a, streams_b, sm_a, sm_b) as torch ExternalStreams, or None when the driver cannot
    partition (the caller then uses ordinary streams).  Cached per (device, sm_a)."""
    dev = torch.device(device)
    key = (dev.index if dev.index is not None else torch.cuda.current_device(), sm_a, n_a, n_b)
    if key not in _PARTITIONS:
        a = (ctypes.c_void_p * n_a)()
        b = (ctypes.c_void_p * n_b)()
        got_a, got_b = ctypes.c_int(0), ctypes.c_int(0)
        with torch.cuda.device(key[0]):
            rc = lib.l3c_partition_streams(sm_a, n_a, a, n_b, b, ctypes.byref(got_a), ctypes.byref(got_b))
        if rc == _lib.E_UNSUPPORTED:
            _PARTITIONS[key] = None
        else:
            check(rc)
            _PARTITIONS[key] = ([torch.cuda.ExternalStream(int(p), device=key[0]) for p in a],
                                [torch.cuda.ExternalStream(int(p), device=key[0]) for p in b],
                                got_a.value, got_b.value)
    return _PARTITIONS[key]


def partition_streams2(device, sm_a, n_a, n_b_high, n_b_low):
    """l3c_partition_streams2: -> (streams_a, streams_b_high, streams_b_low, sm_a, sm_b) or None."""
    dev = torch.device(device)
    key = (dev.index if dev.index is not None else torch.cuda.current_device(), sm_a, n_a, n_b_high, n_b_low, 'v2')
    if key not in _PARTITIONS:
        a = (ctypes.c_void_p * max(1, n_a))()
        bh = (ctypes.c_void_p * max(1, n_b_high))()
        bl = (ctypes.c_void_p * max(1, n_b_low))()
        got_a, got_b = ctypes.c_int(0), ctypes.c_int(0)
        with torch.cuda.device(key[0]):
            rc = lib.l3c_partition_streams2(sm_a, n_a, a, n_b_high, bh, n_b_low, bl, ctypes.byref(got_a),
                                            ctypes.byref(got_b))
        if rc == _lib.E_UNSUPPORTED:
            _PARTITIONS[key] = None
        else:
            check(rc)
            mk = lambda arr, n: [torch.cuda.ExternalStream(int(arr[i]), device=key[0]) for i in range(n)]
            _PARTITIONS[key] = (mk(a, n_a), mk(bh, n_b_high), mk(bl, n_b_low), got_a.value, got_b.value)
    return _PARTITIONS[key]


@contextlib.contextmanager
def conv_launch_limits(max_sms=0, conv_smem_kb=0):
    """Test knob (l3c_set_conv_launch_limits): inside the block the persistent tensor-core convolutions size their
    grid for at most `max_sms` SMs and choose their pipeline stages from a `conv_smem_kb` KB budget (0 = default).
    Process-wide; the defaults are restored on exit."""
    check(lib.l3c_set_conv_launch_limits(int(max_sms), int(conv_smem_kb)))
    try:
        yield
    finally:
        check(lib.l3c_set_conv_launch_limits(0, 0))


@contextlib.contextmanager
def conv_tile_schedule(mode):
    """Test and diagnosis knob (l3c_set_conv_tile_schedule): inside the block the persistent tensor-core
    convolutions hand out their tiles with schedule `mode`: 0 dynamic (the default), 1 the static stripe, 2 dynamic
    with odd CTAs starting 500 us late.  Every mode gives the same bits.  Process-wide; the default is restored on
    exit."""
    check(lib.l3c_set_conv_tile_schedule(int(mode)))
    try:
        yield
    finally:
        check(lib.l3c_set_conv_tile_schedule(0))


def conv_idle_ctas(reset=False):
    """l3c_conv_idle_ctas: CTAs of the current device that ran no tile under schedule 2 since the last reset
    (waits for the device)."""
    n = ctypes.c_longlong(0)
    check(lib.l3c_conv_idle_ctas(ctypes.byref(n), int(bool(reset))))
    return n.value


@contextlib.contextmanager
def decoder_streams_per_cta(spc):
    """Test knob (l3c_set_decoder_streams_per_cta): inside the block the range decoder of alphabets L > 32 packs `spc`
    streams (1, 2 or 4) into one CTA; 0 = the L3C_DEC_SPC / default choice.  Process-wide; the default is restored on
    exit."""
    check(lib.l3c_set_decoder_streams_per_cta(int(spc)))
    try:
        yield
    finally:
        check(lib.l3c_set_decoder_streams_per_cta(0))


@contextlib.contextmanager
def encoder_streams_per_cta(spc):
    """Test knob (l3c_set_encoder_streams_per_cta): inside the block the range encoder packs `spc` streams (1, 2 or 4),
    each a coding warp and an emitter warp, into one CTA; 0 = the L3C_ENC_SPC / default choice.  Process-wide; the
    default is restored on exit."""
    check(lib.l3c_set_encoder_streams_per_cta(int(spc)))
    try:
        yield
    finally:
        check(lib.l3c_set_encoder_streams_per_cta(0))


# ----------------------------------------------------------------------------------------------
# ragged batches (DESIGN §4.6)
# ----------------------------------------------------------------------------------------------
_RAGGED = {'v': None}       # inside ragged_extents(): (finest H, W, [(h_n, w_n)], {(H, W): device extents})


@contextlib.contextmanager
def ragged_extents(extents, H, W):
    """Inside the block the tensors of the conv stack are padded batches [N][H'][W'][..] of differently sized
    images: image n occupies [0, h_n) x [0, w_n) of the finest H x W (`extents` = [(h_n, w_n)]) and
    (h_n * H' / H, w_n * W' / W) at a coarser H' x W'.  Before every k x k conv the band of its halo around each
    image is set to +0 in the tensor it reads (l3c_ragged_zero_halo), so every output pixel inside an image is
    bit-identical to the per-image conv.  extents None: a no-op (equally sized images)."""
    if extents is None:
        yield
        return
    prev = _RAGGED['v']
    _RAGGED['v'] = (int(H), int(W), [(int(h), int(w)) for (h, w) in extents], {})
    try:
        yield
    finally:
        _RAGGED['v'] = prev


def ragged_active():
    return _RAGGED['v'] is not None


def extents_at(H, W, device):
    """Device int32 [N][2] extents of the active ragged batch at resolution H x W (cached per block)."""
    H0, W0, ext, cache = _RAGGED['v']
    key = (int(H), int(W), str(device))
    if key not in cache:
        fh, fw = H0 // H, W0 // W
        if fh * H != H0 or fw * W != W0:
            raise ValueError('ragged batch: a %dx%d tensor is not a scale of the %dx%d batch' % (H, W, H0, W0))
        arr = np.array([(h // fh, w // fw) for (h, w) in ext], np.int32)
        cache[key] = _to_device_async(arr, device)
    return cache[key]


def zero_halo(x, halo):
    """Ragged batch: +0 into the `halo`-pixel band around every image of the NHWC tensor x (in place)."""
    N, H, W = x.shape[:3]
    ext = extents_at(H, W, x.device)
    assert x.is_contiguous()
    check(lib.l3c_ragged_zero_halo(_ptr(x), x.shape[-1] * x.element_size(), N, H, W, _ptr(ext), int(halo),
                                   _stream_ptr()))
    LAUNCHES['n'] += 1


def ragged_pack(src, planes, H, W, extents_dev, compact_len, to_compact, out=None):
    """l3c_ragged_pack: padded planes [N][planes][H][W] of elements (trailing dims) <-> compact planes
    [N][planes][compact_len] of the same elements.  -> the new tensor."""
    assert src.is_contiguous()
    N = extents_dev.shape[0]
    elem = src.numel() // (N * planes * (compact_len if not to_compact else H * W))
    elem_bytes = elem * src.element_size()
    if out is None:
        shape = (N, planes, compact_len) if to_compact else (N, planes, H, W)
        out = torch.empty(shape + ((elem,) if elem > 1 else ()), dtype=src.dtype, device=src.device)
    check(lib.l3c_ragged_pack(_ptr(src), _ptr(out), elem_bytes, planes, N, H, W, _ptr(extents_dev),
                              int(compact_len), 1 if to_compact else 0, _stream_ptr()))
    LAUNCHES['n'] += 1
    return out


def _ragged_guard(kh, dil, x):
    """Before a k x k conv of a ragged batch: zero the halo band of the tensor it reads."""
    if _RAGGED['v'] is not None and kh > 1:
        zero_halo(x, dil * (kh // 2))


def require_cuda(t, name):
    if not t.is_cuda:
        raise ValueError('%s must be a CUDA tensor (l3c_pytorch_b200 has no CPU path)' % name)


# ----------------------------------------------------------------------------------------------
# weights
# ----------------------------------------------------------------------------------------------
class PackedConv(object):
    """The device-side weight images of one nn.Conv2d, each built on first use.  `get` checks the parameters' key
    (weight and bias pointer and version, device) and drops every image when it changed (load_state_dict, .to(),
    an in-place update).  The getters return the cached tensors themselves, with the padded bias."""

    def __init__(self, conv):
        self.conv = conv
        self._key = None
        self.w = self.b = self.w_tc = self.w_h = self.w_h2 = self.w_im2col = self.w_dgrad = None

    def _sync(self):
        """Drops every image when the parameters' key changed."""
        w, b = self.conv.weight, self.conv.bias
        key = (w.data_ptr(), w._version, b.data_ptr(), b._version, str(w.device))
        if key != self._key:
            require_cuda(w, 'conv weight')
            self.w = self.b = self.w_tc = self.w_h = self.w_h2 = self.w_im2col = self.w_dgrad = None
            self._key = key

    def _bias(self):
        """the bias padded to cout_pad"""
        self._sync()
        if self.b is None:
            b = self.conv.bias
            bp = torch.zeros((b.shape[0] + 63) // 64 * 64, dtype=torch.float32, device=b.device)
            bp[:b.shape[0]] = b.detach().float()
            self.b = bp
        return self.b

    def get(self):
        """FFMA image (conv_ffma.cu): OIHW -> [KH][KW][Cin][cout_pad] fp32, bias padded to cout_pad."""
        b = self._bias()
        if self.w is None:
            w = self.conv.weight
            cout, cin, kh, kw = w.shape
            wp = torch.zeros(kh, kw, cin, b.shape[0], dtype=torch.float32, device=w.device)
            wp[..., :cout] = w.detach().float().permute(2, 3, 1, 0)
            self.w = wp
        return self.w, b

    def get_tc(self):
        """TF32 tensor-core image (conv_tf32.cu): [tap][K-half = Cin/32][Cout padded to 64][32] fp32, K-major rows
        of 128 B that TMA drops into 128B-swizzled shared memory; values pre-rounded to TF32 (RN)."""
        b = self._bias()
        if self.w_tc is None:
            w = round_to_tf32(self.conv.weight.detach().float())
            cout, cin, kh, kw = w.shape
            cout_pad = (cout + 63) // 64 * 64
            assert cin % 64 == 0 and kh == kw and kh in (1, 3)
            img = torch.zeros(kh * kw, cin // 32, cout_pad, 32, dtype=torch.float32, device=w.device)
            img[:, :, :cout] = w.permute(2, 3, 0, 1).reshape(kh * kw, cout, cin // 32, 32).permute(0, 2, 1, 3)
            self.w_tc = img.contiguous()
        return self.w_tc, b

    def get_dgrad(self):
        """Data-gradient image of a 3x3 layer with Cin 64 (l3c_conv3x3_dgrad): the weights flipped spatially with Cin
        and Cout swapped, as Cout / 64 forward images of 64 -> 64 convs, [Cout/64][tap][K-half][64 ci][32 co] fp32,
        values rounded to TF32 (RN).  Rebuilt with the other images when the parameters change."""
        self._sync()
        if self.w_dgrad is None:
            w = self.conv.weight.detach().float()                              # [Cout, 64, 3, 3]
            cout, cin, kh, kw = w.shape
            assert cin == 64 and kh == kw == 3 and cout % 64 == 0
            # img[s][tap][kh][ci][j] = w[64 s + 32 kh + j][ci][2 - ky][2 - kx]
            img = w.flip(2, 3).reshape(cout // 64, 2, 32, 64, 9).permute(0, 4, 1, 3, 2).contiguous()
            check(lib.l3c_round_tf32(_ptr(img), _ptr(img), img.numel(), _stream_ptr()))
            LAUNCHES['n'] += 1
            self.w_dgrad = img
        return self.w_dgrad

    def get_f16(self):
        """F16 tensor-core image (conv_f16.cu): 3x3 / 5x5 -> [taps][cout_pad][64 cin] fp16, 1x1 ->
        [Cin/64][cout_pad][64] fp16; K-major rows of 128 B; values rounded to FP16 (RN, saturating)."""
        _, b = self.get()
        if self.w_h is None:
            w = self.conv.weight.detach().float().clamp(-65504.0, 65504.0)
            cout, cin, kh, kw = w.shape
            cout_pad = (cout + 63) // 64 * 64
            assert cin % 64 == 0 and kh == kw and kh in (1, 3, 5)
            if kh in (3, 5):
                assert cin == 64
                img = torch.zeros(kh * kh, cout_pad, 64, dtype=torch.float16, device=w.device)
                img[:, :cout] = w.permute(2, 3, 0, 1).reshape(kh * kh, cout, 64).half()
            else:
                img = torch.zeros(cin // 64, cout_pad, 64, dtype=torch.float16, device=w.device)
                img[:, :cout] = w.reshape(cout, cin // 64, 64).permute(1, 0, 2).half()
            self.w_h = img.contiguous()
        return self.w_h, b

    def get_f16x2(self):
        """Split image of precision mode 'f16x2' (conv_f16x2.cu): 3x3 -> [9][cout_pad][128] (hi | lo per row),
        1x1 -> [2 * Cin/64][cout_pad][64] (hi chunks, then lo chunks)."""
        _, b = self.get()
        if self.w_h2 is None:
            w = self.conv.weight.detach().float().clamp(-65504.0, 65504.0)
            cout, cin, kh, kw = w.shape
            cout_pad = (cout + 63) // 64 * 64
            assert cin % 64 == 0 and kh == kw and kh in (1, 3)
            if kh == 3:
                assert cin == 64
                hi, lo = _split_host(w.permute(2, 3, 0, 1).reshape(9, cout, 64))
                img = torch.zeros(9, cout_pad, 128, dtype=torch.float16, device=w.device)
                img[:, :cout, :64] = hi
                img[:, :cout, 64:] = lo
            else:
                hi, lo = _split_host(w.reshape(cout, cin // 64, 64).permute(1, 0, 2))
                img = torch.zeros(2 * (cin // 64), cout_pad, 64, dtype=torch.float16, device=w.device)
                img[:cin // 64, :cout] = hi
                img[cin // 64:, :cout] = lo
            self.w_h2 = img.contiguous()
        return self.w_h2, b

    def get_im2col(self):
        """FP16 image of the RGB head's 3 -> Cf 3x3 conv as the K = 64 GEMM over its im2col (rgb_head_f16):
        [1][cout_pad][64], k = (ky*3 + kx)*3 + c, zero for k >= 27."""
        _, b = self.get()
        if self.w_im2col is None:
            w = self.conv.weight.detach().float().clamp(-65504.0, 65504.0)        # [Cf, 3, 3, 3]
            cout = w.shape[0]
            assert tuple(w.shape[1:]) == (3, 3, 3) and cout % 2 == 0 and b.shape[0] <= 256
            img = torch.zeros(1, b.shape[0], 64, dtype=torch.float16, device=w.device)
            img[0, :cout, :27] = w.permute(0, 2, 3, 1).reshape(cout, 27).half()
            self.w_im2col = img.contiguous()
        return self.w_im2col, b


_LO_SCALE = 2048.0


def _split_host(w):
    """fp32 -> (hi, lo) FP16 pair with w ~= hi + lo / 2^11 (weight images; activations use l3c_split_f16x2)."""
    hi = w.half()
    lo = ((w - hi.float()) * _LO_SCALE).half()
    return hi, lo


def round_to_tf32(t):
    """fp32 tensor -> nearest TF32-representable fp32 (10-bit mantissa, ties away from zero like
    `cvt.rna.tf32.f32`).  Host-side preparation of the tensor-core weight image.  As the instruction does on sm_90a,
    only finite values are rounded; an inf or NaN keeps its upper 19 bits, so a NaN whose payload lies wholly in the
    low 13 bits becomes inf there and here.  (Adding the half ulp to a NaN could carry its payload into the sign bit
    and give +-0.)"""
    bits = t.contiguous().view(torch.int32)
    finite = (bits & 0x7F800000) != 0x7F800000
    return (torch.where(finite, bits + 0x1000, bits) & -8192).view(torch.float32)


class Act(object):
    """An activation: `f` = NHWC fp32 tensor, `r` = the operand image the next tensor-core conv reads --
    in tf32 mode an fp32 tensor rounded to TF32 (`r is f` when the tensor itself is rounded), in f16 mode
    an FP16 tensor of the same shape (conv_f16.cu); then `f` is None for activations that feed nothing but
    tensor-core convs (want='round')."""
    __slots__ = ('f', 'r')

    def __init__(self, f, r=None):
        self.f, self.r = f, r


def as_operand(x):
    """fp32 NHWC tensor -> Act that also carries the operand image the tensor cores read (its rounded twin)
    when the tensor-core mode is on.  For callers that feed a conv from outside the network (tests, bench)."""
    if not tensor_core_mode():
        return Act(x)
    if f16_mode():
        return Act(x, x.clamp(-65504.0, 65504.0).half())
    if f16x2_mode():
        return Act(x, split_f16x2(x))
    return Act(x, round_to_tf32(x))


def tensor_core_mode():
    return _PRECISION['mode'] != _lib.PREC_FP32


def f16_mode():
    return _PRECISION['mode'] == _lib.PREC_F16


def f16x2_mode():
    return _PRECISION['mode'] == _lib.PREC_F16X2


def split_f16x2(x):
    """fp32 NHWC [..., C] -> split operand image FP16 [..., 2C] (hi | lo) of precision mode 'f16x2'."""
    require_cuda(x, 'x')
    assert x.dtype == torch.float32 and x.is_contiguous()
    C = x.shape[-1]
    out = torch.empty(x.shape[:-1] + (2 * C,), dtype=torch.float16, device=x.device)
    check(lib.l3c_split_f16x2(_ptr(x), x.numel() // C, C, _ptr(out), _stream_ptr()))
    LAUNCHES['n'] += 1
    return out


def _packed_obj(conv):
    pc = conv.__dict__.get('_l3c_packed')
    if pc is None:
        pc = PackedConv(conv)
        conv.__dict__['_l3c_packed'] = pc
    return pc


# ----------------------------------------------------------------------------------------------
# conv stack
# ----------------------------------------------------------------------------------------------
def on_tensor_cores(mode, conv, cin, x_pitch, y_pitch, y_coff, pixel_shuffle, residual):
    """The route of a conv2d call: True for a tensor-core kernel, False for the fp32 FFMA kernel.  `conv` gives the
    geometry (kernel_size, stride, dilation, in_channels, out_channels), `cin` the channels read, `x_pitch` the
    input's pitch in values (half the split image's in f16x2), `y_pitch` / `y_coff` the output's, `residual` whether
    one is added.  A tensor-core layer reads all of a dense input, cin == x_pitch == in_channels, and then:
      fp32   never
      tf32   stride 1: 3x3 with Cin 64, Cout % 64 == 0, y_pitch and y_coff multiples of 4; or 1x1 with
             Cin % 64 == 0 and no pixel shuffle
      f16    3x3/s1 with Cin 64 and Cout % 64 == 0; 5x5/s2 with dilation 1, Cin 64, Cout % 64 == 0 and no pixel
             shuffle; 1x1/s1 with Cin % 64 == 0, no pixel shuffle, even Cout <= 256 and no residual
      f16x2  f16's 3x3 except with pixel shuffle and a residual together, and f16's 1x1
    The rows differ where the modes' kernels do (conv_tf32.cu, conv_f16.cu, conv_f16x2.cu)."""
    cin_all = conv.in_channels
    if mode == _lib.PREC_FP32 or cin != cin_all or x_pitch != cin_all:
        return False
    k, stride, cout = conv.kernel_size[0], conv.stride[0], conv.out_channels
    if k == 3:
        return stride == 1 and cin == 64 and cout % 64 == 0 and (
            y_pitch % 4 == 0 and y_coff % 4 == 0 if mode == _lib.PREC_TF32 else
            not (mode == _lib.PREC_F16X2 and pixel_shuffle and residual))
    if k == 1:
        return stride == 1 and cin % 64 == 0 and not pixel_shuffle and (
            mode == _lib.PREC_TF32 or (cout % 2 == 0 and cout <= 256 and not residual))
    return (k == 5 and mode == _lib.PREC_F16 and stride == 2 and conv.dilation[0] == 1 and cin == 64 and
            cout % 64 == 0 and not pixel_shuffle)


def conv2d(conv, x, cin=None, relu=False, residual=None, pixel_shuffle=False, out=None, out_coff=0,
           precision=None, want='plain'):
    """y = conv(x) [+ReLU] [+residual] on NHWC tensors, parameters taken from the nn.Conv2d `conv` (never called as
    a torch op), in precision mode `precision` (default: the process-wide mode).  `cin` < in_channels reads the
    first `cin` channels of the input; `out` / `out_coff` write a channel slice of a wider NHWC buffer (the atrous
    concat, prob_clf.py:71).

    x: tensor or Act.  The layer runs on the tensor cores or on the fp32 FFMA kernel (on_tensor_cores).  An FFMA
    layer reads `x.f`; a tensor-core layer reads the operand image `x.r`, made for this call's mode when it is
    missing.  y is the fp32 output, `want` picks what is returned:

      mode   tensor-core layer reads   'plain'  'act'                'round'
      fp32   -                         y        Act(y, None)         Act(y, None)
      tf32   x.r, else x.f as it is    y        Act(y, TF32 twin)    Act(y, y), y rounded to TF32 in place
      f16    x.r, else FP16 of x.f     y        Act(y, FP16 image)   Act(None, FP16 image)
      f16x2  x.r, else split of x.f    y        Act(y, split image)  Act(None, split image)

    The conv kernel writes the operand image beside y, except the f16x2 FFMA and 1x1 kernels: they write y and
    split_f16x2 splits it.  With want='round' in f16 / f16x2, `out` is the image's buffer (f16x2: a split buffer
    [.., 2 * C], channels out_coff.. of both halves, which only the 3x3 kernel can fill); otherwise it is y's."""
    xa = x if isinstance(x, Act) else Act(x)
    mode = _PRECISION['mode'] if precision is None else precision
    f16 = mode in (_lib.PREC_F16, _lib.PREC_F16X2)
    split = mode == _lib.PREC_F16X2
    if _RAGGED['v'] is not None and not f16:
        raise NotImplementedError('ragged batches run in precision f16 or f16x2 only, not %s'
                                  % {v: k for k, v in _lib.PRECISIONS.items()}[mode])
    src = xa.r if f16 and xa.f is None else xa.f
    require_cuda(src, 'x')
    assert (f16 or src.dtype == torch.float32) and src.is_contiguous() and src.dim() == 4
    N, H, W, xp = src.shape
    if split and xa.f is None:
        xp //= 2                                              # hi | lo halves
    kh, stride, dil = conv.kernel_size[0], conv.stride[0], conv.dilation[0]
    cin = conv.in_channels if cin is None else cin
    cout = conv.out_channels
    pad = kh // 2 if dil == 1 else dil
    Ho = (H + 2 * pad - dil * (kh - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dil * (kh - 1) - 1) // stride + 1
    shape = (N, Ho * 2, Wo * 2, cout // 4) if pixel_shuffle else (N, Ho, Wo, cout)
    flags = (_lib.CONV_RELU if relu else 0) | (_lib.CONV_PIXEL_SHUFFLE2 if pixel_shuffle else 0)
    tc = on_tensor_cores(mode, conv, cin, xp, shape[3] if out is None else out.shape[-1], out_coff, pixel_shuffle,
                         residual is not None)
    assert tc or xa.f is not None, 'an fp32 (CUDA-core) layer needs the fp32 activation'

    # y: the fp32 output; y_r: its operand image, written by the conv kernel when kernel_img
    kernel_img = mode in (_lib.PREC_TF32, _lib.PREC_F16) or (split and tc and kh == 3)
    image_out = f16 and want == 'round'
    y = y_r = None
    if out is not None:
        assert out.dtype == (torch.float16 if image_out else torch.float32)
        if image_out:
            y_r = out
        else:
            y = out
    # sizes as separate ints: torch.empty takes ~1.5 us longer to parse a tuple, on the thread that feeds the GPU
    if y is None and not (image_out and tc and kernel_img):
        y = torch.empty(*shape, dtype=torch.float32, device=src.device)
    if y_r is None and kernel_img and want in ('act', 'round'):
        if mode == _lib.PREC_TF32 and want == 'round':
            y_r, flags = y, flags | _lib.CONV_ROUND_TF32
        elif mode == _lib.PREC_TF32:
            y_r = torch.empty_like(y)
        else:
            y_r = torch.empty(*shape[:3], shape[3] * (2 if split else 1), dtype=torch.float16, device=src.device)
    if out is not None and y is not None and y_r is not None:
        assert split or y.shape == y_r.shape                  # an unsplit image has y's layout
    y_pitch = y.shape[-1] if y is not None else y_r.shape[-1] // (2 if split else 1)
    if residual is not None:                  # read in y's layout; the f16x2 3x3 kernel adds it to a new y only
        assert residual.dtype == torch.float32 and residual.is_contiguous()
        assert residual.shape == (y.shape if y is not None else y_r.shape[:3] + (y_pitch,))
        assert out is None or not (split and kernel_img)

    pc = _packed_obj(conv)
    if not tc:
        x_in = xa.f
        w, b = pc.get()
    elif mode == _lib.PREC_TF32:
        x_in = xa.r if xa.r is not None else xa.f
        w, b = pc.get_tc()
    elif split:
        x_in = xa.r
        if x_in is None or x_in.dtype != torch.float16 or x_in.shape[-1] != 2 * conv.in_channels:
            x_in = split_f16x2(xa.f)
        w, b = pc.get_f16x2()
    else:
        x_in = xa.r
        if x_in is None or x_in.dtype != torch.float16:
            x_in = xa.f.clamp(-65504.0, 65504.0).half()
        w, b = pc.get_f16()
    _ragged_guard(kh, dil, x_in)
    d = ConvDesc(bias=b.data_ptr(), residual=_dp(residual), y=_dp(y), N=N, H=H, W=W, Cin=cin,
                 x_pitch=2 * xp if split and tc else xp, Cout=cout, cout_pad=b.shape[0], y_pitch=y_pitch,
                 y_coff=out_coff, ksize=kh, stride=stride, dilation=dil, flags=flags,
                 precision=mode if tc else _lib.PREC_FP32)
    if f16 and tc:
        d.x_h, d.w_h = x_in.data_ptr(), w.data_ptr()
    else:
        d.x, d.w = x_in.data_ptr(), w.data_ptr()
    if kernel_img and y_r is not None and y_r is not y:
        if mode == _lib.PREC_TF32:
            d.y_tf32 = y_r.data_ptr()
        else:
            d.y_h = y_r.data_ptr()
            if split:
                d.yh_pitch, d.yh_lo_off = y_r.shape[-1], y_r.shape[-1] // 2
    check(lib.l3c_conv2d(ctypes.byref(d), _stream_ptr()))
    LAUNCHES['n'] += 1

    if not kernel_img and split and want in ('act', 'round'):
        assert out is None or want != 'round', 'a CUDA-core layer cannot fill a slice of a split buffer'
        y_r = split_f16x2(y)
    if want == 'plain':
        return y
    return Act(None if image_out else y, y_r)


def _dp(t):
    return t.data_ptr() if t is not None else None


def rgb_prep(img_u8, conv1, conv2):
    """uint8 planes [N,3,H,W] -> (x_sub NHWC [N,H,W,3] or None, t NHWC [N,H,W,4]); the two 1x1
    MeanShift convs are applied as per-pixel 3x3 affines (parameters read from the modules)."""
    require_cuda(img_u8, 'img')
    assert img_u8.dtype == torch.uint8 and img_u8.is_contiguous()
    if _RAGGED['v'] is not None:
        raise NotImplementedError('ragged batches need the f16 RGB head (precision f16)')
    N, _, H, W = img_u8.shape
    A1 = conv1.weight.detach().float().reshape(9).contiguous()
    b1 = conv1.bias.detach().float().contiguous()
    t = None
    A2 = b2 = None
    xsub = None
    if conv2 is not None:
        A2 = conv2.weight.detach().float().reshape(9).contiguous()
        b2 = conv2.bias.detach().float().contiguous()
        t = torch.empty(N, H, W, 4, dtype=torch.float32, device=img_u8.device)
    else:
        xsub = torch.empty(N, H, W, 3, dtype=torch.float32, device=img_u8.device)
    check(lib.l3c_rgb_prep(_ptr(img_u8), _ptr(A1), _ptr(b1), _ptr(A2), _ptr(b2), N, H * W,
                           _ptr(xsub), _ptr(t), _stream_ptr()))
    LAUNCHES['n'] += 1
    return xsub, t


def rgb_head_f16(img_u8, conv1, conv2, head_conv):
    """f16 mode: RGBHead (the two MeanShift affines + conv 3 -> Cf, 3x3) on the tensor cores: im2col of the
    normalised 3x3 neighbourhood (l3c_rgb_im2col_f16) + a K = 64 GEMM (conv1x1_f16_kernel).  -> Act carrying only
    the FP16 operand image of the head output (it feeds nothing but the encoder's down-sampling conv)."""
    require_cuda(img_u8, 'img')
    assert img_u8.dtype == torch.uint8 and img_u8.is_contiguous()
    N, _, H, W = img_u8.shape
    A1 = conv1.weight.detach().float().reshape(9).contiguous()
    b1 = conv1.bias.detach().float().contiguous()
    A2 = conv2.weight.detach().float().reshape(9).contiguous()
    b2 = conv2.bias.detach().float().contiguous()
    cols = torch.empty(N, H, W, 64, dtype=torch.float16, device=img_u8.device)
    if _RAGGED['v'] is not None:
        check(lib.l3c_rgb_im2col_f16_ragged(_ptr(img_u8), _ptr(A1), _ptr(b1), _ptr(A2), _ptr(b2), N, H, W,
                                            _ptr(extents_at(H, W, img_u8.device)), _ptr(cols), _stream_ptr()))
    else:
        check(lib.l3c_rgb_im2col_f16(_ptr(img_u8), _ptr(A1), _ptr(b1), _ptr(A2), _ptr(b2), N, H, W, _ptr(cols),
                                     _stream_ptr()))
    LAUNCHES['n'] += 1
    w_h, b = _packed_obj(head_conv).get_im2col()
    cout = head_conv.out_channels
    y_h = torch.empty(N, H, W, cout, dtype=torch.float16, device=img_u8.device)
    d = ConvDesc(x_h=cols.data_ptr(), w_h=w_h.data_ptr(), bias=b.data_ptr(), y_h=y_h.data_ptr(),
                 N=N, H=H, W=W, Cin=64, x_pitch=64, Cout=cout, cout_pad=b.shape[0], y_pitch=cout, y_coff=0,
                 ksize=1, stride=1, dilation=1, flags=0, precision=_lib.PREC_F16)
    check(lib.l3c_conv2d(ctypes.byref(d), _stream_ptr()))
    LAUNCHES['n'] += 1
    return Act(None, y_h)


def quantize_head(f, to_q_conv, levels):
    """F NHWC [N,H,W,Cf] -> (sym uint8 planes [N,C,H,W], bn_q NHWC [N,H,W,8] zero padded)."""
    N, H, W, Cf = f.shape
    C = to_q_conv.out_channels
    w = to_q_conv.weight.detach().float().reshape(C, Cf).t().contiguous()
    b = to_q_conv.bias.detach().float().contiguous()
    lev = levels.detach().float().contiguous()
    sym = torch.empty(N, C, H, W, dtype=torch.uint8, device=f.device)
    bnq = torch.empty(N, H, W, 8, dtype=torch.float32, device=f.device)
    check(lib.l3c_quantize_head(_ptr(f), _ptr(w), _ptr(b), _ptr(lev), N, H * W, Cf, C, lev.numel(),
                                _ptr(sym), _ptr(bnq), _stream_ptr()))
    LAUNCHES['n'] += 1
    return sym, bnq


def symbols_to_values(sym, values, shift=None):
    """uint8 planes [N,C,H,W] -> NHWC [N,H,W,8] of values[sym] - shift (zero padded)."""
    N, C, H, W = sym.shape
    out = torch.empty(N, H, W, 8, dtype=torch.float32, device=sym.device)
    check(lib.l3c_symbols_to_values(_ptr(sym), _ptr(values), _ptr(shift), N, H * W, C, values.numel(),
                                    _ptr(out), _stream_ptr()))
    LAUNCHES['n'] += 1
    return out


def bicubic_half(img_u8):
    if _RAGGED['v'] is not None:
        raise NotImplementedError('ragged batches are not supported by the RGB baselines (bicubic encoder)')
    N, C, H, W = img_u8.shape
    assert C == 3 and img_u8.dtype == torch.uint8 and img_u8.is_contiguous()
    out = torch.empty(N, 3, int(H * 0.5), int(W * 0.5), dtype=torch.uint8, device=img_u8.device)
    check(lib.l3c_bicubic_half_u8(_ptr(img_u8), N, H, W, _ptr(out), _stream_ptr()))
    LAUNCHES['n'] += 2
    return out


# ----------------------------------------------------------------------------------------------
# DMLL head
# ----------------------------------------------------------------------------------------------
def uniform_cdf_row(L):
    row = np.zeros(L + 1, np.uint16)
    check(lib.l3c_uniform_cdf_row(L, row.ctypes.data_as(ctypes.c_void_p)))
    return row


def dmll_intervals(l, sym, targets, C, K, L, rgb):
    """l NHWC [N,H,W,Kp]; sym uint8 [N,C,H,W] -> intervals uint32 (stored int32) [N,C,H*W]."""
    N, H, W, _ = l.shape
    iv = torch.empty(N, C, H * W, dtype=torch.int32, device=l.device)
    check(lib.l3c_dmll_intervals(_ptr(l), _ptr(sym), _ptr(targets), N, H * W, C, K, L, int(rgb),
                                 _ptr(iv), _stream_ptr()))
    LAUNCHES['n'] += 1
    return iv


def lut_intervals(sym, lut):
    iv = torch.empty(sym.shape[0], sym.shape[1], sym.shape[2] * sym.shape[3], dtype=torch.int32,
                     device=sym.device)
    check(lib.l3c_lut_intervals(_ptr(sym), _ptr(lut), sym.numel(), _ptr(iv), _stream_ptr()))
    LAUNCHES['n'] += 1
    return iv


def table_pitch(L):
    """row pitch (entries) of the decoder's CDF tables for alphabet L"""
    return 32 if L <= 32 else 256 if L <= 256 else (L + 7) // 8 * 8


def dmll_build_table(l, sym, targets, C, K, L, rgb, c, table, pix0=0, npix=None):
    N, H, W, _ = l.shape
    npix = H * W - pix0 if npix is None else npix
    check(lib.l3c_dmll_build_table(_ptr(l), _ptr(sym), _ptr(targets), N, H * W, C, K, L, int(rgb), c,
                                   pix0, npix, _ptr(table), table_pitch(L), _stream_ptr()))
    LAUNCHES['n'] += 1


def dmll_build_table_tiled(l, sym, targets, C, K, L, rgb, c, table, tile):
    """rows of channel c (all channels for c < 0) in TILE order; `sym` (decoded channels) also in tile order."""
    N, H, W, _ = l.shape
    check(lib.l3c_dmll_build_table_tiled(_ptr(l), _ptr(sym), _ptr(targets), N, H, W, C, K, L, int(rgb), c,
                                         tile[0], tile[1], _ptr(table), table_pitch(L), _stream_ptr()))
    LAUNCHES['n'] += 1


def dmll_build_table_window(l, oy, ox, sym, targets, C, K, L, rgb, c, table, H, W, tile):
    """dmll_build_table_tiled for the H x W symbol plane whose parameters are the rectangle at (oy, ox) of the
    wider plane l NHWC [N,Hl,Wl,Kp] (a decoder window's output, DESIGN §4.8); rows and `sym` in tile order."""
    N, Hl, Wl, _ = l.shape
    assert l.is_contiguous()
    check(lib.l3c_dmll_build_table_window(_ptr(l), Hl, Wl, int(oy), int(ox), _ptr(sym), _ptr(targets), N, H, W, C,
                                          K, L, int(rgb), c, tile[0], tile[1], _ptr(table), table_pitch(L),
                                          _stream_ptr()))
    LAUNCHES['n'] += 1


def crop_rect(src, origins_dev, h, w, nhwc):
    """l3c_crop_rect: the h x w rectangle at origins_dev[n] = (y, x) (int32 [N, 2] on the device) of image n, as a
    new tensor.  nhwc: src is NHWC [N, H, W, C]; otherwise planes [N, P, H, W]."""
    assert src.is_contiguous() and src.dim() == 4
    N = origins_dev.shape[0]
    if nhwc:
        H, W, planes = src.shape[1], src.shape[2], 1
        out = torch.empty(N, h, w, src.shape[3], dtype=src.dtype, device=src.device)
        elem_bytes = src.shape[3] * src.element_size()
    else:
        H, W, planes = src.shape[2], src.shape[3], src.shape[1]
        out = torch.empty(N, planes, h, w, dtype=src.dtype, device=src.device)
        elem_bytes = src.element_size()
    check(lib.l3c_crop_rect(_ptr(src), _ptr(out), elem_bytes, planes, N, H, W, _ptr(origins_dev), int(h), int(w),
                            _stream_ptr()))
    LAUNCHES['n'] += 1
    return out


def dmll_build_table_windows(l, geo_dev, max_hw, plane, sym, targets, C, K, L, rgb, c, table, tile):
    """dmll_build_table_window with a rectangle per image (l3c_dmll_build_table_windows): geo_dev int32 [N, 4] =
    (oy, ox, H_n, W_n) on the device; rows and `sym` in each image's own tile order, in planes of `plane` elements."""
    N, Hl, Wl, _ = l.shape
    assert l.is_contiguous() and geo_dev.shape == (N, 4) and geo_dev.dtype == torch.int32
    check(lib.l3c_dmll_build_table_windows(_ptr(l), Hl, Wl, _ptr(geo_dev), int(max_hw), int(plane), _ptr(sym),
                                           _ptr(targets), N, C, K, L, int(rgb), c, tile[0], tile[1], _ptr(table),
                                           table_pitch(L), _stream_ptr()))
    LAUNCHES['n'] += 1


def crop_rects(src, rects_dev, hp, wp, nhwc, sizes=None):
    """l3c_crop_rects: the rectangle rects_dev[n] = (y, x, h_n, w_n) (int32 [N, 4] on the device) of image n.
    sizes None: -> one tensor, [N, hp, wp, C] (nhwc) or [N, P, hp, wp], image n top-left and +0 elsewhere.
    sizes = [(h_n, w_n)] (planes only): -> [tensor [1, P, h_n, w_n]], contiguous views of one buffer."""
    assert src.is_contiguous() and src.dim() == 4
    N = rects_dev.shape[0]
    if nhwc:
        H, W, planes = src.shape[1], src.shape[2], 1
        elem_bytes = src.shape[3] * src.element_size()
        shape = (N, hp, wp, src.shape[3])
    else:
        H, W, planes = src.shape[2], src.shape[3], src.shape[1]
        elem_bytes = src.element_size()
        shape = (N, planes, hp, wp)
    off_dev, views = None, None
    if sizes is None:
        out = torch.empty(shape, dtype=src.dtype, device=src.device)
    else:
        assert not nhwc and len(sizes) == N
        n_el = [planes * h * w for (h, w) in sizes]
        offs = np.concatenate([[0], np.cumsum(n_el)]).astype(np.int64)
        out = torch.empty(int(offs[-1]), dtype=src.dtype, device=src.device)
        off_dev = _to_device_async(offs[:-1], src.device)
        views = [out[offs[n]:offs[n + 1]].view(1, planes, h, w) for n, (h, w) in enumerate(sizes)]
    check(lib.l3c_crop_rects(_ptr(src), _ptr(out), elem_bytes, planes, N, H, W, _ptr(rects_dev), _ptr(off_dev),
                             int(hp), int(wp), _stream_ptr()))
    LAUNCHES['n'] += 1
    return out if views is None else views


def reorder_tiles_images(src, extents_dev, hp, wp, tile):
    """uint8 [N, P, plane] in each image's own tile order (extents_dev int32 [N, 2] = (h_n, w_n) on the device) ->
    raster [N, P, hp, wp], image n top-left and 0 elsewhere (l3c_reorder_tiles_images)."""
    assert src.is_contiguous() and src.dtype == torch.uint8 and src.dim() == 3
    N, P, plane = src.shape
    dst = torch.empty(N, P, hp, wp, dtype=torch.uint8, device=src.device)
    check(lib.l3c_reorder_tiles_images(_ptr(src), _ptr(dst), P, N, plane, int(hp), int(wp), _ptr(extents_dev),
                                       tile[0], tile[1], _stream_ptr()))
    LAUNCHES['n'] += 1
    return dst


def reorder_tiles(src, H, W, tile, to_tiles, out=None):
    """[planes..., H*W or H, W] uint8 / int32 tensor: raster <-> tile order (l3c_reorder_tiles); new tensor, or `out`
    (a contiguous tensor of src's dtype and size) in src's shape."""
    assert src.is_contiguous() and src.dtype in (torch.uint8, torch.int32)
    planes = src.numel() // (H * W)
    dst = torch.empty_like(src) if out is None else out.view(src.shape)
    check(lib.l3c_reorder_tiles(_ptr(src), _ptr(dst), src.element_size(), planes, H, W, tile[0], tile[1],
                                1 if to_tiles else 0, _stream_ptr()))
    LAUNCHES['n'] += 1
    return dst


def dmll_nll(l, sym, values, C, K, L, rgb, x_min, x_max, want_map=False):
    """-> (per-image nats float64 [N], per-sub-pixel nats f32 [N,C,H,W] or None)."""
    N, H, W, _ = l.shape
    out = torch.empty(N, dtype=torch.float64, device=l.device)
    nmap = torch.empty(N, C, H, W, dtype=torch.float32, device=l.device) if want_map else None
    check(lib.l3c_dmll_nll(_ptr(l), _ptr(sym), _ptr(values), N, H * W, C, K, L, int(rgb),
                           float(x_min), float(x_max), _ptr(out), _ptr(nmap), _stream_ptr()))
    LAUNCHES['n'] += 2
    return out, nmap


def dmll_nll_ragged(l, sym, values, C, K, L, rgb, x_min, x_max, extents):
    """dmll_nll of a ragged batch: l NHWC [N,H,W,Kp] and sym [N,C,H,W] padded, image n occupies [0, h_n) x [0, w_n)
    (`extents` = [(h_n, w_n)] at this resolution).  -> per-image nats float64 [N], bit-identical to dmll_nll on each
    image alone; nothing outside an extent is read."""
    N, H, W, _ = l.shape
    ext = [(int(h), int(w)) for (h, w) in extents]
    if len(ext) != N:
        raise ValueError('%d extents for a batch of %d images' % (len(ext), N))
    for n, (h, w) in enumerate(ext):
        if not (1 <= h <= H and 1 <= w <= W):
            raise ValueError('extent %dx%d of image %d does not fit the %dx%d batch' % (h, w, n, H, W))
    assert tuple(sym.shape) == (N, C, H, W) and sym.dtype == torch.uint8, (tuple(sym.shape), sym.dtype)
    l, sym = l.contiguous(), sym.contiguous()
    ext_dev = _to_device_async(np.array(ext, np.int32).reshape(N, 2), l.device)
    out = torch.empty(N, dtype=torch.float64, device=l.device)
    check(lib.l3c_dmll_nll_ragged(_ptr(l), _ptr(sym), _ptr(values), N, H, W, C, K, L, int(rgb), float(x_min),
                                  float(x_max), _ptr(ext_dev), _ptr(out), _stream_ptr()))
    LAUNCHES['n'] += 2
    return out


def dmll_nll_train(l, x, K, rgb, half_bin, x_lower, x_upper, grad=None, want_dx=False):
    """The training loss of one scale on NCHW fp32 tensors (l3c_dmll_nll_train): l [N,Kp,H,W], x [N,C,H,W] targets,
    both contiguous.  grad None -> per-image nats float64 [N] (2 launches).  grad (0-dim f32 on the device, the
    gradient of the summed nats) -> (dl like l, dx like x or None) (1 launch); want_dx only where not rgb."""
    N, C, H, W = x.shape
    assert l.is_contiguous() and x.is_contiguous() and l.dtype == x.dtype == torch.float32
    assert l.shape[0] == N and l.shape[2:] == x.shape[2:]
    args = (_ptr(l), _ptr(x), N, H * W, C, K, int(rgb), float(half_bin), float(x_lower), float(x_upper))
    if grad is None:
        out = torch.empty(N, dtype=torch.float64, device=l.device)
        check(lib.l3c_dmll_nll_train(*args, _ptr(out), None, None, None, _stream_ptr()))
        LAUNCHES['n'] += 2
        return out
    dl = torch.empty_like(l)
    dx = torch.empty_like(x) if want_dx else None
    check(lib.l3c_dmll_nll_train(*args, None, _ptr(grad), _ptr(dl), _ptr(dx), _stream_ptr()))
    LAUNCHES['n'] += 1
    return dl, dx


def soft_quantize(q, levels, sigma, grad=None):
    """Soft quantiser of a contiguous fp32 tensor q onto fp32 levels [L] (l3c_soft_quantize).
    grad None -> (sym int64, value f32), both shaped like q.  grad (like q) -> dq = grad * 2 sigma Var_phi(levels)."""
    assert q.is_contiguous() and q.dtype == levels.dtype == torch.float32 and levels.is_contiguous()
    if grad is None:
        sym = torch.empty(q.shape, dtype=torch.int64, device=q.device)
        val = torch.empty_like(q)
        check(lib.l3c_soft_quantize(_ptr(q), q.numel(), _ptr(levels), levels.numel(), float(sigma), _ptr(sym),
                                    _ptr(val), None, None, _stream_ptr()))
        LAUNCHES['n'] += 1
        return sym, val
    assert grad.shape == q.shape and grad.is_contiguous() and grad.dtype == torch.float32
    dq = torch.empty_like(q)
    check(lib.l3c_soft_quantize(_ptr(q), q.numel(), _ptr(levels), levels.numel(), float(sigma), None, None,
                                _ptr(grad), _ptr(dq), _stream_ptr()))
    LAUNCHES['n'] += 1
    return dq


def round_tf32(x):
    """l3c_round_tf32: a new tensor of the contiguous fp32 CUDA tensor x rounded to TF32 (RN), the operand image the
    TF32 kernels read."""
    require_cuda(x, 'x')
    assert x.dtype == torch.float32 and x.is_contiguous()
    out = torch.empty_like(x)
    if x.numel():                 # an empty tensor has no storage: a null pointer the C entry point refuses
        check(lib.l3c_round_tf32(_ptr(x), _ptr(out), x.numel(), _stream_ptr()))
        LAUNCHES['n'] += 1
    return out


def _nhwc_args(t, what):
    require_cuda(t, what)
    assert t.dtype == torch.float32 and t.is_contiguous() and t.dim() == 4, (what, t.dtype, tuple(t.shape))


def conv3x3_train(conv, x):
    """Forward of a 3x3 / Cin 64 layer of the training step: x NHWC fp32 [N,H,W,64] -> y NHWC [N,H,W,Cout] in TF32
    (conv3x3_tf32_kernel on the TF32-rounded x, bias added, no epilogue)."""
    _nhwc_args(x, 'x')
    return conv2d(conv, Act(x, round_tf32(x)), precision=_lib.PREC_TF32)


def conv3x3_dgrad(conv, dy):
    """Data gradient of a 3x3 / Cin 64 layer (l3c_conv3x3_dgrad): dy NHWC fp32 [N,H,W,Cout] -> dx NHWC [N,H,W,64],
    dy rounded to TF32 first.  Cout / 64 launches of the forward TF32 kernel on PackedConv.get_dgrad."""
    _nhwc_args(dy, 'dy')
    N, H, W, cout = dy.shape
    assert cout == conv.out_channels
    dyr = round_tf32(dy)
    w = _packed_obj(conv).get_dgrad()
    dx = torch.empty(N, H, W, conv.in_channels, dtype=torch.float32, device=dy.device)
    check(lib.l3c_conv3x3_dgrad(_ptr(dyr), _ptr(w), N, H, W, conv.in_channels, cout, conv.dilation[0], _ptr(dx),
                                _stream_ptr()))
    LAUNCHES['n'] += cout // 64
    return dx


def conv3x3_wgrad(conv, x, dy):
    """Weight and bias gradient of a 3x3 / Cin 64 layer (l3c_conv3x3_wgrad): x NHWC fp32 [N,H,W,64] (the layer's
    input), dy NHWC [N,H,W,Cout] -> (dW [Cout,64,3,3] like conv.weight, db [Cout]).  Two launches, no atomics."""
    _nhwc_args(x, 'x')
    _nhwc_args(dy, 'dy')
    N, H, W, cout = dy.shape
    assert tuple(x.shape) == (N, H, W, conv.in_channels) and cout == conv.out_channels
    work = torch.empty(max(1, lib.l3c_conv3x3_wgrad_workspace(N, H, W, cout) // 4), dtype=torch.float32,
                       device=dy.device)
    dw = torch.empty(cout, conv.in_channels, 3, 3, dtype=torch.float32, device=dy.device)
    db = torch.empty(cout, dtype=torch.float32, device=dy.device)
    check(lib.l3c_conv3x3_wgrad(_ptr(x), _ptr(dy), N, H, W, conv.in_channels, cout, conv.dilation[0], _ptr(dw),
                                _ptr(db), _ptr(work), work.numel() * 4, _stream_ptr()))
    LAUNCHES['n'] += 2
    return dw, db


def dmll_channel_params(l, x_dec, C, K, rgb, c):
    """l NHWC; x_dec f32 [N,C,H,W] contiguous (values of already coded channels) or None.
    -> (softmax pi, mu, log sigma), each [N,K,H,W] f32."""
    N, H, W, _ = l.shape
    outs = [torch.empty(N, K, H, W, dtype=torch.float32, device=l.device) for _ in range(3)]
    check(lib.l3c_dmll_channel_params(_ptr(l), _ptr(x_dec), N, H * W, C, K, int(rgb), c,
                                      _ptr(outs[0]), _ptr(outs[1]), _ptr(outs[2]), _stream_ptr()))
    LAUNCHES['n'] += 1
    return outs


def lin_dmll_intervals(conv, cat_h, sym, targets, C, K, L, rgb):
    """1x1 `lin` conv of the probability classifier fused with the coding intervals (f16 mode, encode side):
    cat_h FP16 NHWC [N,H,W,Cin] -> intervals uint32 (stored int32) [N,C,H*W]; the parameters never reach HBM."""
    N, H, W, cin = cat_h.shape
    assert cat_h.dtype == torch.float16 and cat_h.is_contiguous() and cin == conv.in_channels
    assert conv.kernel_size[0] == 1 and conv.out_channels == (4 if rgb else 3) * C * K
    w_h, b = _packed_obj(conv).get_f16()
    iv = torch.empty(N, C, H * W, dtype=torch.int32, device=cat_h.device)
    check(lib.l3c_lin_dmll_intervals(_ptr(cat_h), _ptr(w_h), _ptr(b), _ptr(sym), _ptr(targets), N, H * W, cin, C, K,
                                     L, int(rgb), _ptr(iv), _stream_ptr()))
    LAUNCHES['n'] += 1
    return iv


def _band_out(out, N, C, n, device):
    if out is None:
        return torch.empty(N, C, n, dtype=torch.int32, device=device)
    assert out.dtype == torch.int32 and out.is_contiguous() and out.numel() == N * C * n
    return out.view(N, C, n)


def lin_dmll_intervals_band(conv, cat_h, oy, sym, y0, h, targets, C, K, L, rgb, tile, out=None):
    """lin_dmll_intervals for one band of a banded encode (l3c_lin_dmll_intervals_band): rows [oy, oy + h) of the FP16
    concat buffer cat_h [N,Hl,W,Cin] of a full-width decoder window, coding the symbols of rows [y0, y0 + h) of the
    whole planes sym uint8 [N,C,Hs,W] -> intervals int32 [N,C,h*W] in the tile order of an h x W plane (written to
    `out` when given: an int32 tensor of as many elements)."""
    N, Hl, W, cin = cat_h.shape
    assert cat_h.dtype == torch.float16 and cat_h.is_contiguous() and cin == conv.in_channels
    assert conv.kernel_size[0] == 1 and conv.out_channels == (4 if rgb else 3) * C * K
    assert sym.dtype == torch.uint8 and sym.is_contiguous() and tuple(sym.shape[:2]) == (N, C) and sym.shape[3] == W
    w_h, b = _packed_obj(conv).get_f16()
    iv = _band_out(out, N, C, h * W, cat_h.device)
    check(lib.l3c_lin_dmll_intervals_band(_ptr(cat_h), Hl, int(oy), _ptr(w_h), _ptr(b), _ptr(sym), sym.shape[2],
                                          int(y0), int(h), W, _ptr(targets), N, cin, C, K, L, int(rgb), tile[0],
                                          tile[1], _ptr(iv), _stream_ptr()))
    LAUNCHES['n'] += 1
    return iv


def dmll_intervals_rect(l, oy, ox, sym, rect, targets, C, K, L, rgb, tile, origin=(0, 0), plane=None, out=None):
    """dmll_intervals for one tile-aligned rectangle (l3c_dmll_intervals_rect), a band of a banded encode or an R_s of a
    region update: the parameters of the h x w rectangle at (oy, ox) of l NHWC [N,Hl,Wl,Kp], coding the symbols of
    rect = (y0, x0, h, w) of the window sym uint8 [N,C,Hs,Ws] -> intervals int32 [N,C,h*w] in the tile order of an h x w plane (to `out` when given).
    The window sits at `origin` of the container's plane of (H, W) = `plane` (default: sym is the whole plane), in
    which the rectangle must be tile-aligned."""
    N, Hl, Wl, _ = l.shape
    y0, x0, h, w = (int(v) for v in rect)
    Hs, Ws = sym.shape[2], sym.shape[3]
    Hf, Wf = (Hs, Ws) if plane is None else (int(plane[0]), int(plane[1]))
    assert l.is_contiguous() and l.dtype == torch.float32
    assert sym.dtype == torch.uint8 and sym.is_contiguous() and tuple(sym.shape[:2]) == (N, C)
    iv = _band_out(out, N, C, h * w, l.device)
    check(lib.l3c_dmll_intervals_rect(_ptr(l), Hl, Wl, int(oy), int(ox), _ptr(sym), Hs, Ws, y0, x0, h, w,
                                      int(origin[0]), int(origin[1]), Hf, Wf, _ptr(targets), N, C, K, L, int(rgb),
                                      tile[0], tile[1], _ptr(iv), _stream_ptr()))
    LAUNCHES['n'] += 1
    return iv


def dmll_intervals_rects(l, sym, geo, targets, C, K, L, rgb, tile, plane=None, out=None):
    """dmll_intervals_rect with one rectangle per image (l3c_dmll_intervals_rects): geo int32 [N][10] = (oy, ox, y0, x0,
    h, w, sy, sx, Hf, Wf) per image, l NHWC [N,Hl,Wl,Kp] and sym uint8 [N,C,Hs,Ws] padded batches -> intervals int32
    [N,C,plane] (plane default: the largest h * w), image n's in the tile order of its own h x w rectangle."""
    N, Hl, Wl, _ = l.shape
    geo = np.ascontiguousarray(geo, np.int32).reshape(N, 10)
    plane = int((geo[:, 4].astype(np.int64) * geo[:, 5]).max()) if plane is None else int(plane)
    assert l.is_contiguous() and l.dtype == torch.float32
    assert sym.dtype == torch.uint8 and sym.is_contiguous() and tuple(sym.shape[:2]) == (N, C)
    iv = _band_out(out, N, C, plane, l.device)
    geo_dev = torch.empty(geo.shape, dtype=torch.int32, device=l.device)
    check(lib.l3c_dmll_intervals_rects(_ptr(l), Hl, Wl, _ptr(sym), sym.shape[2], sym.shape[3],
                                       geo.ctypes.data_as(ctypes.c_void_p), _ptr(geo_dev), plane, _ptr(targets), N, C,
                                       K, L, int(rgb), tile[0], tile[1], _ptr(iv), _stream_ptr()))
    LAUNCHES['n'] += 1
    return iv


def dmll_sample(l, u_sel, u_x, C, K, rgb):
    """l NHWC [N,H,W,Kp]; u_sel f32 [N,C,K,H,W]; u_x f32 [N,C,H,W] -> sampled values f32 [N,C,H,W]."""
    N, H, W, _ = l.shape
    assert u_sel.shape == (N, C, K, H, W) and u_x.shape == (N, C, H, W)
    out = torch.empty(N, C, H, W, dtype=torch.float32, device=l.device)
    check(lib.l3c_dmll_sample(_ptr(l), _ptr(u_sel.contiguous()), _ptr(u_x.contiguous()), N, H * W, C, K, int(rgb),
                              _ptr(out), _stream_ptr()))
    LAUNCHES['n'] += 1
    return out


# ----------------------------------------------------------------------------------------------
# range coder
# ----------------------------------------------------------------------------------------------
def _to_device_async(arr, device):
    """numpy -> device through pinned staging, asynchronous on the current stream.  (A copy from pageable
    memory first waits for everything already queued on the stream: the host would stall behind the
    GPU at every descriptor upload and could never run ahead to feed a second stream.)"""
    return torch.from_numpy(np.ascontiguousarray(arr)).pin_memory().to(device, non_blocking=True)


def _desc_to_device(arr, device):
    return _to_device_async(arr.view(np.uint8).reshape(-1), device)


def ac_encode_streams(desc_np, device):
    """desc_np: numpy structured array (ENC_STREAM_DTYPE). Returns (desc_dev, lens_dev int32)."""
    n = desc_np.shape[0]
    desc = _desc_to_device(desc_np, device)
    lens = torch.empty(n, dtype=torch.int32, device=device)
    check(lib.l3c_ac_encode_streams(_ptr(desc), n, _ptr(lens), _stream_ptr()))
    LAUNCHES['n'] += 1
    return desc, lens


def ac_encode_slice(desc_dev, lens_dev, first, n):
    """l3c_ac_encode_streams on descriptors [first, first + n) of an uploaded array (as ac_encode_streams' desc_dev),
    their lengths to the same elements of lens_dev (int32)."""
    first, size = int(first), np.dtype(_lib.ENC_STREAM_DTYPE).itemsize
    check(lib.l3c_ac_encode_streams(ctypes.c_void_p(desc_dev.data_ptr() + first * size), int(n),
                                    ctypes.c_void_p(lens_dev.data_ptr() + first * 4), _stream_ptr()))
    LAUNCHES['n'] += 1


def pack_streams(desc_dev, lens_dev, dst_off_np, n, blob):
    off = _to_device_async(dst_off_np.astype(np.int64), blob.device)
    check(lib.l3c_pack_streams(_ptr(desc_dev), _ptr(lens_dev), _ptr(off), n, _ptr(blob), _stream_ptr()))
    LAUNCHES['n'] += -(-n // 65535)                 # one launch per 65535 streams


def splice_streams(old, slots, seg, out):
    """l3c_splice_streams: the segments seg int64 [n][4] (codec.splice_segments) from the uint8 device buffers old and
    slots into out, in one launch."""
    seg = np.ascontiguousarray(seg, np.int64).reshape(-1, 4)
    seg_dev = torch.empty(5 * seg.shape[0] + 1, dtype=torch.int64, device=out.device)
    check(lib.l3c_splice_streams(_ptr(old), old.numel(), _ptr(slots), slots.numel(),
                                 seg.ctypes.data_as(ctypes.c_void_p), _ptr(seg_dev), seg.shape[0], _ptr(out),
                                 out.numel(), _stream_ptr()))
    LAUNCHES['n'] += int(seg.shape[0] > 0)


def update_splice(conts, streams, new_len, slot_off, caps, old, slots, out):
    """l3c_update_layout, then l3c_splice_streams_dev: the containers conts (UPDATE_CONTAINER_DTYPE) with their streams
    (UPDATE_STREAM_DTYPE), numpy, are laid out from the device lengths new_len (int32) and spliced from the uint8 device
    buffers old and slots into out, without a host wait.  slot_off / caps: int64 numpy [new_len.numel()].  Everything
    host-side is uploaded in one asynchronous copy.  -> (info, keep): info int64 [len(conts) + 1] on the device, the
    new sizes and the error flag; keep: the device tensors the launches read, to be kept alive until they ran."""
    n_c, n_s, n_new = conts.shape[0], streams.shape[0], int(new_len.numel())
    n_seg = int((2 * conts['n_new'] + 1).sum())
    host = np.concatenate([conts.view(np.int64).reshape(-1), streams.view(np.int64).reshape(-1),
                           np.asarray(slot_off, np.int64), np.asarray(caps, np.int64)])
    up = _to_device_async(host, out.device)
    a, b = conts.size * 9, conts.size * 9 + streams.size * 4
    seg = torch.empty(4 * n_seg + n_seg + n_c, dtype=torch.int64, device=out.device)
    info = torch.empty(n_c + 1, dtype=torch.int64, device=out.device)
    ptr = lambda t, i: ctypes.c_void_p(t.data_ptr() + 8 * i)
    check(lib.l3c_update_layout(ptr(up, 0), n_c, ptr(up, a), n_s, _ptr(new_len), ptr(up, b), ptr(up, b + n_new), n_new,
                                _ptr(seg), ptr(seg, 4 * n_seg), n_seg, _ptr(info), _stream_ptr()))
    LAUNCHES['n'] += int(n_c > 0)
    # a container's chunks: one per 4 KB of its bytes, plus one per segment boundary
    max_chunks = int((conts['out_cap'] // 4096 + 2 * conts['n_new'] + 2).max()) if n_c else 0
    check(lib.l3c_splice_streams_dev(ptr(up, 0), n_c, _ptr(seg), ptr(seg, 4 * n_seg), n_seg, _ptr(old), old.numel(),
                                     _ptr(slots), slots.numel(), _ptr(out), out.numel(), max_chunks, ptr(info, n_c),
                                     _stream_ptr()))
    LAUNCHES['n'] += -(-n_c // 65535) if max_chunks else 0
    return info, (up, seg, new_len, old, slots, out)


COARSE_PITCH = 96     # uint16 per coarse record (l3c_dmll_build_coarse)


def dmll_build_coarse(l, sym, targets, K, L, c, rec, pix0=0, npix=None):
    """coarse records (parameters + cdf[8 i]) of RGB channel c, L = 256: rec int16 [N * 3 * H * W * COARSE_PITCH]"""
    N, H, W, _ = l.shape
    npix = H * W - pix0 if npix is None else npix
    check(lib.l3c_dmll_build_coarse(_ptr(l), _ptr(sym), _ptr(targets), N, H * W, K, L, c, pix0, npix, _ptr(rec),
                                    _stream_ptr()))
    LAUNCHES['n'] += 1


def dmll_build_coarse_windows(l, geo_dev, max_hw, plane, sym, targets, K, L, c, rec):
    """dmll_build_coarse on decoder windows (l3c_dmll_build_coarse_windows): image n's parameters are the rectangle
    geo_dev[n] = (oy, ox, H_n, W_n) (int32 [N, 4] on the device) of l NHWC [N,Hl,Wl,Kp]; its records and `sym` in the
    raster order of that rectangle, in planes of `plane` elements."""
    N, Hl, Wl, _ = l.shape
    assert l.is_contiguous() and geo_dev.shape == (N, 4) and geo_dev.dtype == torch.int32
    check(lib.l3c_dmll_build_coarse_windows(_ptr(l), Hl, Wl, _ptr(geo_dev), int(max_hw), int(plane), _ptr(sym),
                                            _ptr(targets), N, K, L, c, _ptr(rec), _stream_ptr()))
    LAUNCHES['n'] += 1


def ac_decode_streams_coarse(desc_np, device, targets, first=0, count=None, desc_dev=None, n=None):
    """ac_decode_streams (L = 256) for streams whose `table` points at coarse records (row_pitch COARSE_PITCH)."""
    if desc_dev is None:
        desc_dev = _desc_to_device(desc_np, device)
    if n is None:
        n = desc_np.shape[0]
    if count is None:
        count = int(desc_np['n_sym'].max()) if n else 0
    check(lib.l3c_ac_decode_streams_coarse(_ptr(desc_dev), n, _ptr(targets), first, count, _stream_ptr()))
    LAUNCHES['n'] += 1
    return desc_dev


def decode_rgb_pipelined(l, S, targets, K, L, table, descs_dev, chunk_px, cur, bld, dec, coarse=False):
    """l3c_decode_rgb_pipelined: the chunk-pipelined RGB scale of a decode in one native call.
    descs_dev: three device tensors (descriptor arrays of the R, G, B streams); cur / bld / dec: torch streams.
    coarse: `table` holds coarse records (pitch COARSE_PITCH) instead of 256-entry rows."""
    N, H, W, _ = l.shape
    HW = H * W
    pp = (ctypes.c_void_p * 3)(*[d.data_ptr() for d in descs_dev])
    sb = (ctypes.c_void_p * 3)(*[s.cuda_stream for s in bld])
    sd = (ctypes.c_void_p * 3)(*[s.cuda_stream for s in dec])
    check(lib.l3c_decode_rgb_pipelined(_ptr(l), _ptr(S), _ptr(targets), N, HW, K, L, _ptr(table),
                                       COARSE_PITCH if coarse else table_pitch(L), pp, int(chunk_px),
                                       ctypes.c_void_p(cur.cuda_stream), sb, sd, 1 if coarse else 0))
    LAUNCHES['n'] += 2 * 3 * (-(-HW // int(chunk_px)))


def ac_decode_streams(desc_np, device, L, first=0, count=None, desc_dev=None, n=None):
    """Decode symbols [first, first+count) of every stream.  Pass `desc_dev` (+ `n`) to reuse an
    uploaded descriptor array across chunked launches."""
    if desc_dev is None:
        desc_dev = _desc_to_device(desc_np, device)
    if n is None:
        n = desc_np.shape[0]
    if count is None:
        count = int(desc_np['n_sym'].max()) if n else 0
    check(lib.l3c_ac_decode_streams(_ptr(desc_dev), n, L, first, count, _stream_ptr()))
    LAUNCHES['n'] += 1
    return desc_dev


def ac_encode_streams_seek(desc_np, device, every, points_dev, point_off):
    """ac_encode_streams that also records seek points every `every` symbols (l3c_ac_encode_streams_seek): stream i's
    points go to points_dev (int32 [points][4]) from row point_off[i] on.  Returns (desc_dev, lens_dev int32)."""
    n = desc_np.shape[0]
    desc = _desc_to_device(desc_np, device)
    ptrs = _to_device_async(points_dev.data_ptr() + 16 * np.asarray(point_off, np.int64), device)
    lens = torch.empty(n, dtype=torch.int32, device=device)
    check(lib.l3c_ac_encode_streams_seek(_ptr(desc), n, _ptr(lens), int(every), _ptr(ptrs), _stream_ptr()))
    LAUNCHES['n'] += int(n > 0)
    return desc, lens, ptrs


def ac_decode_segments(segs_np, device, L, targets=None):
    """l3c_ac_decode_segments on the segment descriptors segs_np (DEC_STREAM_DTYPE); with `targets`, the coarse
    variant (tables of coarse records).  -> the uploaded descriptors (keep them alive until the launch ran)."""
    n = segs_np.shape[0]
    segs = _desc_to_device(segs_np, device)
    if targets is None:
        check(lib.l3c_ac_decode_segments(_ptr(segs), n, L, _stream_ptr()))
    else:
        check(lib.l3c_ac_decode_segments_coarse(_ptr(segs), n, _ptr(targets), _stream_ptr()))
    LAUNCHES['n'] += int(n > 0)
    return segs
