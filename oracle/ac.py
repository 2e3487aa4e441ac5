"""ctypes wrappers around oracle/_build/liboracle.so (ac_oracle.c).  TEST INFRASTRUCTURE ONLY."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, '_build', 'liboracle.so')
_lib = None


def build():
    src = os.path.join(_HERE, 'ac_oracle.c')
    if not os.path.isfile(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(['make', '-s', '-C', _HERE])
    return _SO


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
        _lib.oracle_ac_encode.restype = ctypes.c_size_t
        _lib.oracle_ac_encode.argtypes = [
            ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
            ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
        _lib.oracle_ac_decode.restype = None
        _lib.oracle_ac_decode.argtypes = [
            ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
            ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
        _lib.oracle_ac_decode_trace.restype = None
        _lib.oracle_ac_decode_trace.argtypes = [
            ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
            ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p]
        _lib.oracle_mixture_cdf.restype = None
        _lib.oracle_mixture_cdf.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int] * 3 + [ctypes.c_void_p]
    return _lib


def _as_cdf(cdf):
    cdf = np.ascontiguousarray(cdf)
    if cdf.dtype == np.int16:
        cdf = cdf.view(np.uint16)
    assert cdf.dtype == np.uint16, cdf.dtype
    return cdf


def encode(cdf, sym):
    """cdf: [n_sym, Lp] (or [Lp] = one shared row) uint16/int16; sym: [n_sym] int16 -> bytes."""
    cdf = _as_cdf(cdf)
    sym = np.ascontiguousarray(sym, dtype=np.int16).reshape(-1)
    Lp = cdf.shape[-1]
    stride = 0 if cdf.ndim == 1 else Lp
    if cdf.ndim > 1:
        cdf = cdf.reshape(-1, Lp)
        assert cdf.shape[0] == sym.size, (cdf.shape, sym.size)
    cap = 4 * sym.size + 64
    out = np.empty(cap, np.uint8)
    n = lib().oracle_ac_encode(cdf.ctypes.data, stride, sym.size, Lp, sym.ctypes.data,
                               out.ctypes.data, cap)
    assert n <= cap
    return out[:n].tobytes()


def decode(cdf, data, n_sym=None):
    """Inverse of encode -> int16 [n_sym]."""
    cdf = _as_cdf(cdf)
    Lp = cdf.shape[-1]
    if cdf.ndim == 1:
        stride = 0
        assert n_sym is not None
    else:
        cdf = cdf.reshape(-1, Lp)
        stride = Lp
        n_sym = cdf.shape[0]
    buf = np.frombuffer(bytes(data), np.uint8)
    out = np.empty(n_sym, np.int16)
    lib().oracle_ac_decode(cdf.ctypes.data, stride, n_sym, Lp,
                           buf.ctypes.data if buf.size else None, buf.size, out.ctypes.data)
    return out


def decode_trace(cdf, data):
    """decode() that also returns the coder state when each symbol is reached: uint32 [n_sym, 4] rows of
    (low, high, value, code bits read so far) -- what a decoder resumed at that symbol starts from."""
    cdf = _as_cdf(cdf)
    Lp = cdf.shape[-1]
    cdf = cdf.reshape(-1, Lp)
    n_sym = cdf.shape[0]
    buf = np.frombuffer(bytes(data), np.uint8)
    out = np.empty(n_sym, np.int16)
    trace = np.empty((n_sym, 4), np.uint32)
    lib().oracle_ac_decode_trace(cdf.ctypes.data, Lp, n_sym, Lp, buf.ctypes.data if buf.size else None, buf.size,
                                 out.ctypes.data, trace.ctypes.data)
    return out, trace


def mixture_cdf(targets, means, log_scales, probs):
    """targets [Lp] f32; means/log_scales/probs [K, N] f32 -> uint16 [N, Lp]
    (formula of torchac_kernel.cu:26-76)."""
    targets = np.ascontiguousarray(targets, np.float32)
    means = np.ascontiguousarray(means, np.float32)
    log_scales = np.ascontiguousarray(log_scales, np.float32)
    probs = np.ascontiguousarray(probs, np.float32)
    K, N = means.shape
    Lp = targets.size
    out = np.empty((N, Lp), np.uint16)
    lib().oracle_mixture_cdf(targets.ctypes.data, means.ctypes.data, log_scales.ctypes.data,
                             probs.ctypes.data, K, N, Lp, out.ctypes.data)
    return out


def uniform_cdf_row(L):
    """Shared CDF row of the uniform prior, as the reference builds it
    (src/bitcoding/bitcoding.py:297-323): round(cumsum(1/L) * 2^16) with a leading 0, wrapped to
    16 bits (last entry becomes 0 and is never read)."""
    pr = np.ones(L, np.float32) / np.float32(L)
    c = np.cumsum(pr, dtype=np.float32) * np.float32(65536.0)
    c = np.rint(c).astype(np.int64)
    row = np.concatenate([[0], c]) & 0xFFFF
    return row.astype(np.uint16)
