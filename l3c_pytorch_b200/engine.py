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
def decoder_streams_per_cta(spc):
    """Test knob (l3c_set_decoder_streams_per_cta): inside the block the L = 256 range decoder packs `spc` streams
    (1, 2 or 4) into one CTA; 0 = the L3C_DEC_SPC / default choice.  Process-wide; the default is restored on exit."""
    check(lib.l3c_set_decoder_streams_per_cta(int(spc)))
    try:
        yield
    finally:
        check(lib.l3c_set_decoder_streams_per_cta(0))


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
    """Device-side repack of one nn.Conv2d: OIHW -> [KH][KW][Cin][cout_pad] (+ padded bias).
    Re-packed automatically when the parameter is modified (load_state_dict, .to())."""

    def __init__(self, conv):
        self.conv = conv
        self._key = None
        self.w = self.b = None

    def get(self):
        w, b = self.conv.weight, self.conv.bias
        key = (w.data_ptr(), w._version, b.data_ptr(), b._version, str(w.device))
        if key != self._key:
            require_cuda(w, 'conv weight')
            cout, cin, kh, kw = w.shape
            cout_pad = (cout + 63) // 64 * 64
            wp = torch.zeros(kh, kw, cin, cout_pad, dtype=torch.float32, device=w.device)
            wp[..., :cout] = w.detach().float().permute(2, 3, 1, 0)
            bp = torch.zeros(cout_pad, dtype=torch.float32, device=w.device)
            bp[:cout] = b.detach().float()
            self.w, self.b, self._key = wp, bp, key
            self.w_tc = None
            self.w_h = None
            self.w_im2col = None
        return self.w, self.b

    def get_tc(self):
        """Tensor-core operand image: [tap][K-half = Cin/32][Cout padded to 64][32] fp32, K-major rows
        of 128 B that TMA drops into 128B-swizzled shared memory; values pre-rounded to TF32 (RN)."""
        _, b = self.get()
        if self.w_tc is None:
            w = round_to_tf32(self.conv.weight.detach().float())
            cout, cin, kh, kw = w.shape
            cout_pad = (cout + 63) // 64 * 64
            assert cin % 64 == 0 and kh == kw and kh in (1, 3)
            img = torch.zeros(kh * kw, cin // 32, cout_pad, 32, dtype=torch.float32, device=w.device)
            img[:, :, :cout] = w.permute(2, 3, 0, 1).reshape(kh * kw, cout, cin // 32, 32).permute(0, 2, 1, 3)
            self.w_tc = img.contiguous()
        return self.w_tc, b


def _get_f16(self):
    """F16 tensor-core operand image (conv_f16.cu): 3x3 / 5x5 -> [taps][cout_pad][64 cin] fp16, 1x1 ->
    [Cin/64][cout_pad][64] fp16; K-major rows of 128 B; values rounded to FP16 (RN, saturating)."""
    _, b = self.get()
    if getattr(self, 'w_h', None) is None:
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


PackedConv.get_f16 = _get_f16


_LO_SCALE = 2048.0


def _split_host(w):
    """fp32 -> (hi, lo) FP16 pair with w ~= hi + lo / 2^11 (weight images; activations use l3c_split_f16x2)."""
    hi = w.half()
    lo = ((w - hi.float()) * _LO_SCALE).half()
    return hi, lo


def _get_f16x2(self):
    """Split weight image of precision mode 'f16x2' (conv_f16x2.cu): 3x3 -> [9][cout_pad][128] (hi | lo per row),
    1x1 -> [2 * Cin/64][cout_pad][64] (hi chunks, then lo chunks)."""
    _, b = self.get()
    if getattr(self, 'w_h2', None) is None or self._key_h2 != self._key:
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
        self.w_h2, self._key_h2 = img.contiguous(), self._key
    return self.w_h2, b


PackedConv.get_f16x2 = _get_f16x2


def round_to_tf32(t):
    """fp32 tensor -> nearest TF32-representable fp32 (10-bit mantissa, ties away from zero like
    `cvt.rna.tf32.f32`).  Host-side preparation of the tensor-core weight image."""
    bits = t.contiguous().view(torch.int32)
    return ((bits + 0x1000) & -8192).view(torch.float32)


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


def packed(conv):
    return _packed_obj(conv).get()


def tc_eligible(conv, x_pitch, y_pitch, y_coff, pixel_shuffle=False):
    """Layers the wgmma kernel covers: 3x3 (any dilation) with 64 input channels and Cout % 64 == 0,
    and 1x1 with Cin % 64 == 0 (any Cout); stride 1, dense input pitch.  Everything else (5x5/s2,
    Cin = 3 or 5) runs on the fp32 FFMA kernel."""
    k, cin, cout = conv.kernel_size[0], conv.in_channels, conv.out_channels
    if conv.stride[0] != 1 or x_pitch != cin:
        return False
    if k == 3:
        return cin == 64 and cout % 64 == 0 and y_pitch % 4 == 0 and y_coff % 4 == 0
    if k == 1:
        return cin % 64 == 0 and not pixel_shuffle
    return False


# ----------------------------------------------------------------------------------------------
# conv stack
# ----------------------------------------------------------------------------------------------
def conv2d(conv, x, cin=None, relu=False, residual=None, pixel_shuffle=False, out=None, out_coff=0,
           precision=None, want='plain'):
    """y = conv(x) [+ReLU] [+residual] on NHWC tensors, parameters taken from the nn.Conv2d `conv`
    (never called as a torch op).  `out`/`out_coff` write a channel slice of a wider NHWC buffer
    (used for the atrous concat, prob_clf.py:71).

    x: tensor or Act.  want: 'plain' -> tensor; 'act' -> Act whose `.r` twin is produced when the
    tensor-core mode is on; 'round' -> Act whose only tensor is the operand image (for activations that
    feed nothing but a following tensor-core conv; then `out`, if given, is that image's buffer)."""
    xa = x if isinstance(x, Act) else Act(x)
    mode = _PRECISION['mode'] if precision is None else precision
    if mode == _lib.PREC_F16:
        return _conv2d_f16(conv, xa, cin, relu, residual, pixel_shuffle, out, out_coff, want)
    if _RAGGED['v'] is not None:
        raise NotImplementedError('ragged batches run in precision f16 only, not %s'
                                  % {v: k for k, v in _lib.PRECISIONS.items()}[mode])
    if mode == _lib.PREC_F16X2:
        return _conv2d_f16x2(conv, xa, cin, relu, residual, pixel_shuffle, out, out_coff, want)
    x = xa.f
    require_cuda(x, 'x')
    assert x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 4
    N, H, W, xp = x.shape
    kh = conv.kernel_size[0]
    stride, dil = conv.stride[0], conv.dilation[0]
    cin = conv.in_channels if cin is None else cin
    cout = conv.out_channels
    pad = kh // 2 if dil == 1 else dil
    Ho = (H + 2 * pad - dil * (kh - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dil * (kh - 1) - 1) // stride + 1
    flags = (_lib.CONV_RELU if relu else 0) | (_lib.CONV_PIXEL_SHUFFLE2 if pixel_shuffle else 0)
    if out is None:
        if pixel_shuffle:
            out = torch.empty(N, Ho * 2, Wo * 2, cout // 4, dtype=torch.float32, device=x.device)
        else:
            out = torch.empty(N, Ho, Wo, cout, dtype=torch.float32, device=x.device)
    prec = mode
    x_in = x
    if mode != _lib.PREC_FP32 and tc_eligible(conv, xp, out.shape[-1], out_coff, pixel_shuffle) and cin == conv.in_channels:
        w, b = _packed_obj(conv).get_tc()
        if xa.r is not None:
            x_in = xa.r                       # TF32-rounded operand image
    else:
        prec = _lib.PREC_FP32
        w, b = packed(conv)
    out_r = None
    if mode != _lib.PREC_FP32:
        if want == 'act':
            out_r = torch.empty_like(out)
        elif want == 'round':
            flags |= _lib.CONV_ROUND_TF32
    d = ConvDesc(x=x_in.data_ptr(), w=w.data_ptr(), bias=b.data_ptr(),
                 residual=residual.data_ptr() if residual is not None else None, y=out.data_ptr(),
                 y_tf32=out_r.data_ptr() if out_r is not None else None,
                 N=N, H=H, W=W, Cin=cin, x_pitch=xp, Cout=cout, cout_pad=b.shape[0],
                 y_pitch=out.shape[-1], y_coff=out_coff, ksize=kh, stride=stride, dilation=dil,
                 flags=flags, precision=prec)
    if residual is not None:
        assert residual.shape == out.shape and residual.is_contiguous()
    check(lib.l3c_conv2d(ctypes.byref(d), _stream_ptr()))
    LAUNCHES['n'] += 1
    if want == 'plain':
        return out
    if want == 'round':
        return Act(out, out if mode != _lib.PREC_FP32 else None)
    return Act(out, out_r)


def _conv2d_f16(conv, xa, cin, relu, residual, pixel_shuffle, out, out_coff, want):
    """conv2d in precision mode 'f16': tensor-core-eligible layers read the FP16 operand image `xa.r` and
    run conv_f16.cu; the others (Cin = 3 or 5) run the fp32 FFMA kernel on `xa.f`.  Either kernel
    writes what the consumers need: fp32 (`want` 'plain' / 'act') and / or the FP16 image ('act' / 'round')."""
    src = xa.f if xa.f is not None else xa.r
    require_cuda(src, 'x')
    assert src.is_contiguous() and src.dim() == 4
    N, H, W, xp = src.shape
    kh = conv.kernel_size[0]
    stride, dil = conv.stride[0], conv.dilation[0]
    cin = conv.in_channels if cin is None else cin
    cout = conv.out_channels
    pad = kh // 2 if dil == 1 else dil
    Ho = (H + 2 * pad - dil * (kh - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dil * (kh - 1) - 1) // stride + 1
    flags = (_lib.CONV_RELU if relu else 0) | (_lib.CONV_PIXEL_SHUFFLE2 if pixel_shuffle else 0)
    shape = (N, Ho * 2, Wo * 2, cout // 4) if pixel_shuffle else (N, Ho, Wo, cout)
    need_f, need_h = want in ('plain', 'act'), want in ('act', 'round')
    y = y_h = None
    if out is not None:                      # caller's buffer for the primary output (channel slice)
        if want == 'round':
            assert out.dtype == torch.float16
            y_h = out
        else:
            assert out.dtype == torch.float32
            y = out
    k = kh
    tc = (xp == conv.in_channels and cin == conv.in_channels and
          ((k == 3 and stride == 1 and cin == 64 and cout % 64 == 0) or
           (k == 5 and stride == 2 and dil == 1 and cin == 64 and cout % 64 == 0 and not pixel_shuffle) or
           (k == 1 and stride == 1 and cin % 64 == 0 and not pixel_shuffle and cout % 2 == 0 and cout <= 256 and
            residual is None)))
    if need_f and y is None:
        y = torch.empty(shape, dtype=torch.float32, device=src.device)
    if need_h and y_h is None:
        y_h = torch.empty(shape, dtype=torch.float16, device=src.device)
    ref = y if y is not None else y_h
    pc = _packed_obj(conv)
    if tc:
        if xa.r is None or xa.r.dtype != torch.float16:
            xa = as_operand(xa.f)                     # callers from outside the network (tests, bench)
        w_h, b = pc.get_f16()
        _ragged_guard(kh, dil, xa.r)
        d = ConvDesc(x_h=xa.r.data_ptr(), w_h=w_h.data_ptr(), bias=b.data_ptr(),
                     residual=residual.data_ptr() if residual is not None else None,
                     y=_dp(y), y_h=_dp(y_h), N=N, H=H, W=W, Cin=cin, x_pitch=xp, Cout=cout, cout_pad=b.shape[0],
                     y_pitch=ref.shape[-1], y_coff=out_coff, ksize=kh, stride=stride, dilation=dil,
                     flags=flags, precision=_lib.PREC_F16)
    else:
        assert xa.f is not None, 'an fp32 (CUDA-core) layer needs the fp32 activation'
        if y is None:                                 # the FFMA kernel always writes fp32
            y = torch.empty(shape, dtype=torch.float32, device=src.device)
        w, b = pc.get()
        _ragged_guard(kh, dil, xa.f)
        d = ConvDesc(x=xa.f.data_ptr(), w=w.data_ptr(), bias=b.data_ptr(),
                     residual=residual.data_ptr() if residual is not None else None,
                     y=_dp(y), y_h=_dp(y_h), N=N, H=H, W=W, Cin=cin, x_pitch=xp, Cout=cout, cout_pad=b.shape[0],
                     y_pitch=ref.shape[-1], y_coff=out_coff, ksize=kh, stride=stride, dilation=dil,
                     flags=flags, precision=_lib.PREC_FP32)
    if residual is not None:
        assert residual.dtype == torch.float32 and residual.shape == ref.shape and residual.is_contiguous()
    if y is not None and y_h is not None:
        assert y.shape == y_h.shape
    check(lib.l3c_conv2d(ctypes.byref(d), _stream_ptr()))
    LAUNCHES['n'] += 1
    if want == 'plain':
        return y
    if want == 'round':
        return Act(None, y_h)
    return Act(y, y_h)


def _conv2d_f16x2(conv, xa, cin, relu, residual, pixel_shuffle, out, out_coff, want):
    """conv2d in precision mode 'f16x2' (strict tensor-core mode, conv_f16x2.cu): the 64-channel 3x3 layers and
    the wide 1x1 layers read SPLIT operand images `xa.r` ([N,H,W,2*Cin] FP16, hi | lo) and accumulate hi*hi and
    hi*lo + lo*hi separately; the other layers (5x5/s2, Cin = 3 or 5) run the fp32 FFMA kernel on `xa.f`, and
    their output is split by l3c_split_f16x2 when a tensor-core layer follows ('act' / 'round')."""
    src = xa.f if xa.f is not None else xa.r
    require_cuda(src, 'x')
    assert src.is_contiguous() and src.dim() == 4
    N, H, W = src.shape[:3]
    kh = conv.kernel_size[0]
    stride, dil = conv.stride[0], conv.dilation[0]
    cin_all = conv.in_channels
    xp = src.shape[-1] if xa.f is not None else src.shape[-1] // 2
    cin = cin_all if cin is None else cin
    cout = conv.out_channels
    pad = kh // 2 if dil == 1 else dil
    Ho = (H + 2 * pad - dil * (kh - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dil * (kh - 1) - 1) // stride + 1
    flags = (_lib.CONV_RELU if relu else 0) | (_lib.CONV_PIXEL_SHUFFLE2 if pixel_shuffle else 0)
    co = cout // 4 if pixel_shuffle else cout
    shape = (N, Ho * 2, Wo * 2, co) if pixel_shuffle else (N, Ho, Wo, co)
    need_f, need_h = want in ('plain', 'act'), want in ('act', 'round')
    y = y_h = None
    if out is not None:
        if want == 'round':
            assert out.dtype == torch.float16      # split buffer [.., 2*Ctot]; this layer fills channels out_coff..
            y_h = out
        else:
            assert out.dtype == torch.float32
            y = out
    tc = (xp == cin_all and cin == cin_all and stride == 1 and
          ((kh == 3 and cin == 64 and cout % 64 == 0 and not (pixel_shuffle and residual is not None)) or
           (kh == 1 and cin % 64 == 0 and not pixel_shuffle and cout % 2 == 0 and cout <= 256 and residual is None)))
    k1 = tc and kh == 1
    pc = _packed_obj(conv)
    if need_f and y is None:
        y = torch.empty(shape, dtype=torch.float32, device=src.device)
    if tc and not k1:
        if need_h and y_h is None:
            y_h = torch.empty(shape[:3] + (2 * co,), dtype=torch.float16, device=src.device)
        if xa.r is None or xa.r.dtype != torch.float16 or xa.r.shape[-1] != 2 * cin_all:
            xa = Act(xa.f, split_f16x2(xa.f))
        w_h, b = pc.get_f16x2()
        yh_pitch = y_h.shape[-1] if y_h is not None else 0
        d = ConvDesc(x_h=xa.r.data_ptr(), w_h=w_h.data_ptr(), bias=b.data_ptr(),
                     residual=residual.data_ptr() if residual is not None else None,
                     y=_dp(y), y_h=_dp(y_h), N=N, H=H, W=W, Cin=cin, x_pitch=2 * cin_all, Cout=cout,
                     cout_pad=b.shape[0], y_pitch=y.shape[-1] if y is not None else yh_pitch // 2, y_coff=out_coff,
                     ksize=kh, stride=stride, dilation=dil, flags=flags, precision=_lib.PREC_F16X2,
                     yh_pitch=yh_pitch, yh_lo_off=yh_pitch // 2)
        if residual is not None:
            assert residual.dtype == torch.float32 and residual.is_contiguous() and out is None and \
                tuple(residual.shape) == tuple(shape)
        check(lib.l3c_conv2d(ctypes.byref(d), _stream_ptr()))
        LAUNCHES['n'] += 1
    else:
        if y is None:
            y = torch.empty(shape, dtype=torch.float32, device=src.device)
        if k1:
            if xa.r is None or xa.r.dtype != torch.float16 or xa.r.shape[-1] != 2 * cin_all:
                xa = Act(xa.f, split_f16x2(xa.f))
            w_h, b = pc.get_f16x2()
            d = ConvDesc(x_h=xa.r.data_ptr(), w_h=w_h.data_ptr(), bias=b.data_ptr(), y=y.data_ptr(),
                         N=N, H=H, W=W, Cin=cin, x_pitch=2 * cin_all, Cout=cout, cout_pad=b.shape[0],
                         y_pitch=y.shape[-1], y_coff=out_coff, ksize=1, stride=1, dilation=1, flags=flags,
                         precision=_lib.PREC_F16X2)
        else:
            assert xa.f is not None, 'an fp32 (CUDA-core) layer needs the fp32 activation'
            w, b = pc.get()
            d = ConvDesc(x=xa.f.data_ptr(), w=w.data_ptr(), bias=b.data_ptr(),
                         residual=residual.data_ptr() if residual is not None else None, y=y.data_ptr(),
                         N=N, H=H, W=W, Cin=cin, x_pitch=xa.f.shape[-1], Cout=cout, cout_pad=b.shape[0],
                         y_pitch=y.shape[-1], y_coff=out_coff, ksize=kh, stride=stride, dilation=dil, flags=flags,
                         precision=_lib.PREC_FP32)
            if residual is not None:
                assert residual.dtype == torch.float32 and residual.shape == y.shape and residual.is_contiguous()
        check(lib.l3c_conv2d(ctypes.byref(d), _stream_ptr()))
        LAUNCHES['n'] += 1
        if need_h:
            assert out is None or want != 'round', 'a CUDA-core layer cannot fill a slice of a split buffer'
            y_h = split_f16x2(y)
    if want == 'plain':
        return y
    if want == 'round':
        return Act(None, y_h)
    return Act(y, y_h)


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
    pc = _packed_obj(head_conv)
    _, b = pc.get()
    if getattr(pc, 'w_im2col', None) is None:
        w = head_conv.weight.detach().float().clamp(-65504.0, 65504.0)        # [Cf, 3, 3, 3]
        cout = w.shape[0]
        assert tuple(w.shape[1:]) == (3, 3, 3) and cout % 2 == 0 and b.shape[0] <= 256
        img = torch.zeros(1, b.shape[0], 64, dtype=torch.float16, device=w.device)
        img[0, :cout, :27] = w.permute(0, 2, 3, 1).reshape(cout, 27).half()   # k = (ky*3 + kx)*3 + c
        pc.w_im2col = img.contiguous()
    cout = head_conv.out_channels
    y_h = torch.empty(N, H, W, cout, dtype=torch.float16, device=img_u8.device)
    d = ConvDesc(x_h=cols.data_ptr(), w_h=pc.w_im2col.data_ptr(), bias=b.data_ptr(), y_h=y_h.data_ptr(),
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
    return 32 if L <= 32 else 256


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


def reorder_tiles(src, H, W, tile, to_tiles):
    """[planes..., H*W or H, W] uint8 / int32 tensor: raster <-> tile order (l3c_reorder_tiles); new tensor."""
    assert src.is_contiguous() and src.dtype in (torch.uint8, torch.int32)
    planes = src.numel() // (H * W)
    dst = torch.empty_like(src)
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


def pack_streams(desc_dev, lens_dev, dst_off_np, n, blob):
    off = _to_device_async(dst_off_np.astype(np.int64), blob.device)
    check(lib.l3c_pack_streams(_ptr(desc_dev), _ptr(lens_dev), _ptr(off), n, _ptr(blob), _stream_ptr()))
    LAUNCHES['n'] += 1


def decode_rgb_pipelined(l, S, targets, K, L, table, descs_dev, chunk_px, cur, bld, dec):
    """l3c_decode_rgb_pipelined: the chunk-pipelined RGB scale of a decode in one native call.
    descs_dev: three device tensors (descriptor arrays of the R, G, B streams); cur / bld / dec: torch streams."""
    N, H, W, _ = l.shape
    HW = H * W
    pp = (ctypes.c_void_p * 3)(*[d.data_ptr() for d in descs_dev])
    sb = (ctypes.c_void_p * 3)(*[s.cuda_stream for s in bld])
    sd = (ctypes.c_void_p * 3)(*[s.cuda_stream for s in dec])
    check(lib.l3c_decode_rgb_pipelined(_ptr(l), _ptr(S), _ptr(targets), N, HW, K, L, _ptr(table), table_pitch(L), pp,
                                       int(chunk_px), ctypes.c_void_p(cur.cuda_stream), sb, sd))
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
