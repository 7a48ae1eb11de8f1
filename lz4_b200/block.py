"""One-shot block API: the Python face of the drop-in C functions (lib/lz4.h:191,208,236, lib/lz4hc.h:66,91).

Same names, argument meaning and error behaviour as the reference's C API; data are host bytes (bytes-like, or a uint8
ndarray of any shape: its bytes in C order).  A length, capacity, target, level or acceleration that does not fit the C
int the call takes raises ValueError before anything is called.
Each call is LZ4_* in liblz4_b200.so: host -> device copy, CUDA kernels, device -> host copy.
"""
import ctypes as C

import numpy as np

from . import _lib


def _u8(data):
    """data as one contiguous run of bytes: a uint8 ndarray of any shape is flattened (a call passes all its bytes), any
    other ndarray raises ValueError, anything else goes through bytes()"""
    if isinstance(data, np.ndarray):
        if data.dtype != np.uint8:
            raise ValueError("byte arrays must be uint8 (got %s)" % data.dtype)
        return np.ascontiguousarray(data).reshape(-1)
    return np.frombuffer(bytes(data), dtype=np.uint8)


def _c_int(name, v):
    """v as the C int the call takes; ValueError when it does not fit one (ctypes would cut it silently)"""
    v = int(v)
    if not -2 ** 31 <= v < 2 ** 31:
        raise ValueError("%s = %d does not fit a C int" % (name, v))
    return v


def LZ4_compressBound(input_size):
    return int(_lib.load().LZ4_compressBound(_c_int("input_size", input_size)))


def LZ4_compress_fast(src, dst_capacity=None, acceleration=1):
    """Returns (ret, bytes): ret bytes written, 0 on failure -- lz4.h:236."""
    lib = _lib.load()
    s = _u8(src)
    n, accel = _c_int("len(src)", len(s)), _c_int("acceleration", acceleration)
    cap = LZ4_compressBound(n) if dst_capacity is None else _c_int("dst_capacity", dst_capacity)
    dst = np.empty(max(cap, 1), dtype=np.uint8)
    r = int(lib.LZ4_compress_fast(s.ctypes.data if n else None, dst.ctypes.data, n, cap, accel))
    return r, dst[:max(r, 0)].tobytes()


def LZ4_compress_default(src, dst_capacity=None):
    """lz4.h:191."""
    lib = _lib.load()
    s = _u8(src)
    n = _c_int("len(src)", len(s))
    cap = LZ4_compressBound(n) if dst_capacity is None else _c_int("dst_capacity", dst_capacity)
    dst = np.empty(max(cap, 1), dtype=np.uint8)
    r = int(lib.LZ4_compress_default(s.ctypes.data if n else None, dst.ctypes.data, n, cap))
    return r, dst[:max(r, 0)].tobytes()


def LZ4_compress_destSize(src, target, acceleration=None):
    """Returns (ret, consumed, bytes): ret bytes written (<= target), consumed = what the call leaves in *srcSizePtr --
    lz4.h:272.  acceleration None calls LZ4_compress_destSize, an integer LZ4_compress_destSize_extState (lz4.h:617)."""
    lib = _lib.load()
    s = _u8(src)
    n, target = C.c_int(_c_int("len(src)", len(s))), _c_int("target", target)
    accel = None if acceleration is None else _c_int("acceleration", acceleration)
    dst = np.empty(max(target, 1), dtype=np.uint8)
    sp = s.ctypes.data if len(s) else None
    if accel is None:
        r = int(lib.LZ4_compress_destSize(sp, dst.ctypes.data, C.byref(n), target))
    else:
        state = np.empty(16416 // 8, dtype=np.uint64)          # LZ4_sizeofState(), 8-byte aligned
        r = int(lib.LZ4_compress_destSize_extState(state.ctypes.data, sp, dst.ctypes.data, C.byref(n), target, accel))
    return r, int(n.value), dst[:max(r, 0)].tobytes()


def LZ4_compress_HC(src, level=9, dst_capacity=None):
    """Returns (ret, bytes): ret bytes written at LZ4HC level `level`, 0 on failure -- lz4hc.h:66."""
    lib = _lib.load()
    s = _u8(src)
    n, level = _c_int("len(src)", len(s)), _c_int("level", level)
    cap = LZ4_compressBound(n) if dst_capacity is None else _c_int("dst_capacity", dst_capacity)
    dst = np.empty(max(cap, 1), dtype=np.uint8)
    r = int(lib.LZ4_compress_HC(s.ctypes.data if n else None, dst.ctypes.data, n, cap, level))
    return r, dst[:max(r, 0)].tobytes()


def LZ4_compress_HC_destSize(src, target, level=9):
    """Returns (ret, consumed, bytes): ret bytes written (<= target) at LZ4HC level `level`, consumed = what the call
    leaves in *srcSizePtr -- lz4hc.h:83-94."""
    lib = _lib.load()
    s = _u8(src)
    n, target, level = C.c_int(_c_int("len(src)", len(s))), _c_int("target", target), _c_int("level", level)
    dst = np.empty(max(target, 1), dtype=np.uint8)
    state = np.empty(lib.LZ4_sizeofStateHC() // 8, dtype=np.uint64)      # 8-byte aligned, like LZ4_streamHC_t
    r = int(lib.LZ4_compress_HC_destSize(state.ctypes.data, s.ctypes.data if len(s) else None, dst.ctypes.data,
                                         C.byref(n), target, level))
    return r, int(n.value), dst[:max(r, 0)].tobytes()


def LZ4_decompress_safe_partial(src, target, dst_capacity=None):
    """Returns (ret, bytes): the first min(target, dst_capacity) decoded bytes at most, ret their count or a negative
    error -- lz4.h:308.  dst_capacity None means target."""
    lib = _lib.load()
    s = _u8(src)
    n, target = _c_int("len(src)", len(s)), _c_int("target", target)
    cap = target if dst_capacity is None else _c_int("dst_capacity", dst_capacity)
    dst = np.empty(max(min(target, cap), 1), dtype=np.uint8)
    sp = s.ctypes.data if n else np.zeros(1, dtype=np.uint8).ctypes.data
    r = int(lib.LZ4_decompress_safe_partial(sp, dst.ctypes.data, n, target, cap))
    return r, dst[:max(r, 0)].tobytes()


def LZ4_decompress_safe(src, dst_capacity):
    """Returns (ret, bytes): ret decoded size or negative error -- lz4.h:208."""
    lib = _lib.load()
    s = _u8(src)
    n, cap = _c_int("len(src)", len(s)), _c_int("dst_capacity", dst_capacity)
    dst = np.empty(max(cap, 1), dtype=np.uint8)
    sp = s.ctypes.data if n else np.zeros(1, dtype=np.uint8).ctypes.data
    r = int(lib.LZ4_decompress_safe(sp, dst.ctypes.data, n, cap))
    return r, dst[:max(r, 0)].tobytes()
