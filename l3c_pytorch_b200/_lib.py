"""ctypes binding of libl3c_b200.so (C ABI declared in include/l3c_b200.h).

There is NO CPU fallback: if the shared library cannot be loaded (or built) importing this module
raises, and every entry point raises RuntimeError with the library's own message on failure --
the same exception type the reference's pybind module surfaces for AT_CHECK failures
(/root/reference/src/torchac/torchac_backend/torchac.cpp:133-135,242-245).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# L3C_CTA_TRACE=1: the diagnosis build (build.py --cta-trace), whose conv CTAs record their timeline
SO_PATH = os.path.join(_HERE, 'libl3c_b200_trace.so' if os.environ.get('L3C_CTA_TRACE') == '1' else 'libl3c_b200.so')

c_void_p, c_int, c_int64, c_size_t, c_uint32, c_float = (
    ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_float)


class ConvDesc(ctypes.Structure):
    """l3c_conv_t"""
    _fields_ = [('x', c_void_p), ('w', c_void_p), ('bias', c_void_p), ('residual', c_void_p),
                ('y', c_void_p), ('y_tf32', c_void_p), ('y_h', c_void_p), ('x_h', c_void_p), ('w_h', c_void_p),
                ('N', c_int), ('H', c_int), ('W', c_int), ('Cin', c_int), ('x_pitch', c_int),
                ('Cout', c_int), ('cout_pad', c_int), ('y_pitch', c_int), ('y_coff', c_int),
                ('ksize', c_int), ('stride', c_int), ('dilation', c_int),
                ('flags', ctypes.c_uint), ('precision', c_int), ('yh_pitch', c_int), ('yh_lo_off', c_int)]


CONV_RELU = 1
CONV_PIXEL_SHUFFLE2 = 2
CONV_ROUND_TF32 = 4
PREC_FP32, PREC_TF32, PREC_F16, PREC_F16X2 = 0, 1, 2, 3
E_UNSUPPORTED = -5          # L3C_EUNSUPPORTED
PRECISIONS = {'fp32': PREC_FP32, 'tf32': PREC_TF32, 'f16': PREC_F16, 'f16x2': PREC_F16X2}

# numpy dtypes of the stream descriptor structs (l3c_enc_stream_t / l3c_dec_stream_t)
ENC_STREAM_DTYPE = [('intervals', '<u8'), ('out', '<u8'), ('n_sym', '<u4'), ('out_cap', '<u4')]
DEC_STREAM_DTYPE = [('table', '<u8'), ('in', '<u8'), ('sym_out', '<u8'), ('state', '<u8'),
                    ('row_pitch', '<i8'), ('n_sym', '<u4'), ('in_len', '<u4')]
# uint32 words of a decoder stream's saved state that fit every stream: (low, high, value, code bits read: low word,
# high word); streams below 2^28 bytes use only the first 4
DEC_STATE_WORDS = 5
# l3c_update_stream_t / l3c_update_container_t (l3c_update_layout)
UPDATE_STREAM_DTYPE = [('fixed_off', '<i8'), ('old_off', '<i8'), ('old_len', '<i8'), ('src', '<i8')]
UPDATE_CONTAINER_DTYPE = [('first_stream', '<i8'), ('n_streams', '<i8'), ('fixed_total', '<i8'), ('old_base', '<i8'),
                          ('old_bytes', '<i8'), ('out_base', '<i8'), ('out_cap', '<i8'), ('first_seg', '<i8'),
                          ('n_new', '<i8')]
# l3c_code_src_t (section F)
CODE_SRC_DTYPE = [('table', '<u8'), ('targets', '<u8'), ('means', '<u8'), ('log_scales', '<u8'), ('probs', '<u8'),
                  ('sym', '<u8'), ('n_sym', '<i8'), ('Lp', '<i4'), ('K', '<i4')]

_SIGNATURES = {
    'l3c_last_error': (ctypes.c_char_p, []),
    'l3c_version': (c_int, []),
    'l3c_launch_log': (ctypes.c_longlong, [ctypes.c_char_p, c_size_t, c_int]),
    'l3c_cuda_supported': (c_int, []),
    'l3c_encode_cdf': (c_int, [c_void_p, c_int64, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    'l3c_decode_cdf': (c_int, [c_void_p, c_int64, c_int, c_void_p, c_size_t, c_void_p]),
    'l3c_encode_logistic_mixture': (c_int, [c_void_p] * 4 + [c_int, c_int64, c_int, c_void_p, c_void_p,
                                                             c_size_t, c_void_p]),
    'l3c_decode_logistic_mixture': (c_int, [c_void_p] * 4 + [c_int, c_int64, c_int, c_void_p, c_size_t,
                                                             c_void_p]),
    'l3c_ac_encode_streams': (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    'l3c_ac_decode_streams': (c_int, [c_void_p, c_int, c_int, c_uint32, c_uint32, c_void_p]),
    'l3c_ac_encode_streams_seek': (c_int, [c_void_p, c_int, c_void_p, c_uint32, c_void_p, c_void_p]),
    'l3c_ac_decode_segments': (c_int, [c_void_p, c_int, c_int, c_void_p]),
    'l3c_ac_decode_segments_coarse': (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    'l3c_uniform_cdf_row': (c_int, [c_int, c_void_p]),
    'l3c_lut_intervals': (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p]),
    'l3c_dmll_intervals': (c_int, [c_void_p] * 3 + [c_int] * 6 + [c_void_p, c_void_p]),
    'l3c_dmll_build_table': (c_int, [c_void_p] * 3 + [c_int] * 9 + [c_void_p, c_int, c_void_p]),
    'l3c_dmll_build_table_tiled': (c_int, [c_void_p] * 3 + [c_int] * 10 + [c_void_p, c_int, c_void_p]),
    'l3c_reorder_tiles': (c_int, [c_void_p, c_void_p] + [c_int] * 7 + [c_void_p]),
    'l3c_dmll_build_table_window': (c_int, [c_void_p] + [c_int] * 4 + [c_void_p] * 2 + [c_int] * 10 +
                                    [c_void_p, c_int, c_void_p]),
    'l3c_crop_rect': (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [c_void_p, c_int, c_int, c_void_p]),
    'l3c_dmll_build_table_windows': (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int] + [c_void_p] * 2 +
                                     [c_int] * 8 + [c_void_p, c_int, c_void_p]),
    'l3c_crop_rects': (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    'l3c_reorder_tiles_images': (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [c_void_p, c_int, c_int, c_void_p]),
    'l3c_dmll_nll': (c_int, [c_void_p] * 3 + [c_int] * 6 + [c_float, c_float, c_void_p, c_void_p, c_void_p]),
    'l3c_dmll_channel_params': (c_int, [c_void_p, c_void_p] + [c_int] * 6 + [c_void_p] * 4),
    'l3c_dmll_sample': (c_int, [c_void_p] * 3 + [c_int] * 5 + [c_void_p, c_void_p]),
    'l3c_conv2d': (c_int, [ctypes.POINTER(ConvDesc), c_void_p]),
    'l3c_lin_dmll_intervals': (c_int, [c_void_p] * 5 + [c_int] * 7 + [c_void_p, c_void_p]),
    'l3c_lin_dmll_intervals_band': (c_int, [c_void_p, c_int, c_int] + [c_void_p] * 3 + [c_int] * 4 + [c_void_p] +
                                    [c_int] * 8 + [c_void_p, c_void_p]),
    'l3c_dmll_intervals_rect': (c_int, [c_void_p] + [c_int] * 4 + [c_void_p] + [c_int] * 10 + [c_void_p] + [c_int] * 7 +
                                [c_void_p, c_void_p]),
    'l3c_dmll_intervals_rects': (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int,
                                         c_void_p] + [c_int] * 7 + [c_void_p, c_void_p]),
    'l3c_rgb_prep': (c_int, [c_void_p] * 5 + [c_int, c_int, c_void_p, c_void_p, c_void_p]),
    'l3c_split_f16x2': (c_int, [c_void_p, ctypes.c_longlong, c_int, c_void_p, c_void_p]),
    'l3c_rgb_im2col_f16': (c_int, [c_void_p] * 5 + [c_int] * 3 + [c_void_p, c_void_p]),
    'l3c_rgb_im2col_f16_ragged': (c_int, [c_void_p] * 5 + [c_int] * 3 + [c_void_p] * 3),
    'l3c_ragged_zero_halo': (c_int, [c_void_p] + [c_int] * 4 + [c_void_p, c_int, c_void_p]),
    'l3c_ragged_pack': (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [c_void_p, ctypes.c_longlong, c_int, c_void_p]),
    'l3c_dmll_nll_ragged': (c_int, [c_void_p] * 3 + [c_int] * 7 + [c_float, c_float] + [c_void_p] * 3),
    'l3c_quantize_head': (c_int, [c_void_p] * 4 + [c_int] * 5 + [c_void_p, c_void_p, c_void_p]),
    'l3c_symbols_to_values': (c_int, [c_void_p] * 3 + [c_int] * 4 + [c_void_p, c_void_p]),
    'l3c_bicubic_half_u8': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    'l3c_decode_rgb_pipelined': (c_int, [c_void_p] * 3 + [c_int] * 4 + [c_void_p, c_int, c_void_p, c_int, c_void_p,
                                         c_void_p, c_void_p, c_int]),
    'l3c_dmll_build_coarse': (c_int, [c_void_p] * 3 + [c_int] * 7 + [c_void_p, c_void_p]),
    'l3c_dmll_build_coarse_windows': (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int] + [c_void_p] * 2 +
                                      [c_int] * 4 + [c_void_p, c_void_p]),
    'l3c_ac_decode_streams_coarse': (c_int, [c_void_p, c_int, c_void_p, c_uint32, c_uint32, c_void_p]),
    'l3c_pack_streams': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    'l3c_splice_streams': (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_int, c_void_p, c_int64,
                                   c_void_p]),
    'l3c_update_layout': (c_int, [c_void_p, c_int, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_void_p,
                                  c_void_p, c_int64, c_void_p, c_void_p]),
    'l3c_splice_streams_dev': (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_void_p,
                                       c_int64, c_void_p, c_int64, c_int64, c_void_p, c_void_p]),
    'l3c_partition_streams': (c_int, [c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    'l3c_partition_streams2': (c_int, [c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    'l3c_set_conv_launch_limits': (c_int, [c_int, c_int]),
    'l3c_set_conv_tile_schedule': (c_int, [c_int]),
    'l3c_conv_idle_ctas': (c_int, [ctypes.POINTER(ctypes.c_longlong), c_int]),
    'l3c_cta_trace_register': (c_int, [c_void_p, c_int64]),
    'l3c_cta_trace_launches': (c_int, [ctypes.c_char_p, c_size_t, ctypes.POINTER(c_int64)]),
    'l3c_set_decoder_streams_per_cta': (c_int, [c_int]),
    'l3c_set_encoder_streams_per_cta': (c_int, [c_int]),
    'l3c_dmll_probe_sigmoid': (c_int, [c_void_p] * 3 + [c_int64, c_void_p]),
    'l3c_batch_intervals': (c_int, [c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p, c_void_p]),
    'l3c_batch_rows': (c_int, [c_void_p, c_void_p, c_int, c_int64, c_uint32, c_void_p, c_void_p]),
    'l3c_dmll_nll_train': (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [c_float] * 3 + [c_void_p] * 5),
    'l3c_soft_quantize': (c_int, [c_void_p, c_int64, c_void_p, c_int, c_float] + [c_void_p] * 5),
    'l3c_round_tf32': (c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    'l3c_conv3x3_dgrad': (c_int, [c_void_p, c_void_p] + [c_int] * 6 + [c_void_p, c_void_p]),
    'l3c_conv3x3_wgrad_workspace': (c_int64, [c_int] * 4),
    'l3c_conv3x3_wgrad': (c_int, [c_void_p, c_void_p] + [c_int] * 6 + [c_void_p] * 3 + [c_int64, c_void_p]),
}

EXPORTS = sorted(_SIGNATURES)


def _bind(path):
    lib = ctypes.CDLL(path)
    for name, (restype, argtypes) in _SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError here = header/library mismatch
        fn.restype = restype
        fn.argtypes = argtypes
    return lib


def _load():
    from . import build as _build
    if not os.path.isfile(SO_PATH):
        # in-tree build (nvcc cross-compiles without a GPU); raises if nvcc is missing
        _build.build()
    try:
        return _bind(SO_PATH)
    except AttributeError:
        # a library left over from an older source tree: rebuild once, then fail loudly
        _build.build(force=True)
        return _bind(SO_PATH)


lib = _load()


def check(rc):
    """0 -> ok; anything else -> RuntimeError carrying l3c_last_error()."""
    if rc != 0:
        msg = lib.l3c_last_error().decode('utf-8', 'replace')
        raise RuntimeError('libl3c_b200: %s (code %d)' % (msg, rc))


def cuda_supported():
    return bool(lib.l3c_cuda_supported())
