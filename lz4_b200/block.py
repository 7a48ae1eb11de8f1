"""One-shot block API: the Python face of the drop-in C functions (lib/lz4.h:191,208,236, lib/lz4hc.h:66,91).

Same names, argument meaning and error behaviour as the reference's C API; data are host bytes.
Each call is LZ4_* in liblz4_b200.so: host -> device copy, CUDA kernels, device -> host copy.
"""
import ctypes as C

import numpy as np

from . import _lib


def _u8(data):
    if isinstance(data, np.ndarray):
        assert data.dtype == np.uint8
        return np.ascontiguousarray(data)
    return np.frombuffer(bytes(data), dtype=np.uint8)


def LZ4_compressBound(input_size):
    return int(_lib.load().LZ4_compressBound(int(input_size)))


def LZ4_compress_fast(src, dst_capacity=None, acceleration=1):
    """Returns (ret, bytes): ret bytes written, 0 on failure -- lz4.h:236."""
    lib = _lib.load()
    s = _u8(src)
    cap = LZ4_compressBound(len(s)) if dst_capacity is None else int(dst_capacity)
    dst = np.empty(max(cap, 1), dtype=np.uint8)
    r = int(lib.LZ4_compress_fast(s.ctypes.data if len(s) else None, dst.ctypes.data, len(s), cap, int(acceleration)))
    return r, dst[:max(r, 0)].tobytes()


def LZ4_compress_default(src, dst_capacity=None):
    """lz4.h:191."""
    lib = _lib.load()
    s = _u8(src)
    cap = LZ4_compressBound(len(s)) if dst_capacity is None else int(dst_capacity)
    dst = np.empty(max(cap, 1), dtype=np.uint8)
    r = int(lib.LZ4_compress_default(s.ctypes.data if len(s) else None, dst.ctypes.data, len(s), cap))
    return r, dst[:max(r, 0)].tobytes()


def LZ4_compress_destSize(src, target, acceleration=None):
    """Returns (ret, consumed, bytes): ret bytes written (<= target), consumed = what the call leaves in *srcSizePtr --
    lz4.h:272.  acceleration None calls LZ4_compress_destSize, an integer LZ4_compress_destSize_extState (lz4.h:617)."""
    lib = _lib.load()
    s = _u8(src)
    dst = np.empty(max(int(target), 1), dtype=np.uint8)
    n = C.c_int(len(s))
    sp = s.ctypes.data if len(s) else None
    if acceleration is None:
        r = int(lib.LZ4_compress_destSize(sp, dst.ctypes.data, C.byref(n), int(target)))
    else:
        state = np.empty(16416 // 8, dtype=np.uint64)          # LZ4_sizeofState(), 8-byte aligned
        r = int(lib.LZ4_compress_destSize_extState(state.ctypes.data, sp, dst.ctypes.data, C.byref(n), int(target),
                                                   int(acceleration)))
    return r, int(n.value), dst[:max(r, 0)].tobytes()


def LZ4_compress_HC(src, level=9, dst_capacity=None):
    """Returns (ret, bytes): ret bytes written at LZ4HC level `level`, 0 on failure -- lz4hc.h:66."""
    lib = _lib.load()
    s = _u8(src)
    cap = LZ4_compressBound(len(s)) if dst_capacity is None else int(dst_capacity)
    dst = np.empty(max(cap, 1), dtype=np.uint8)
    r = int(lib.LZ4_compress_HC(s.ctypes.data if len(s) else None, dst.ctypes.data, len(s), cap, int(level)))
    return r, dst[:max(r, 0)].tobytes()


def LZ4_compress_HC_destSize(src, target, level=9):
    """Returns (ret, consumed, bytes): ret bytes written (<= target) at LZ4HC level `level`, consumed = what the call
    leaves in *srcSizePtr -- lz4hc.h:83-94."""
    lib = _lib.load()
    s = _u8(src)
    dst = np.empty(max(int(target), 1), dtype=np.uint8)
    n = C.c_int(len(s))
    state = np.empty(lib.LZ4_sizeofStateHC() // 8, dtype=np.uint64)      # 8-byte aligned, like LZ4_streamHC_t
    r = int(lib.LZ4_compress_HC_destSize(state.ctypes.data, s.ctypes.data if len(s) else None, dst.ctypes.data,
                                         C.byref(n), int(target), int(level)))
    return r, int(n.value), dst[:max(r, 0)].tobytes()


def LZ4_decompress_safe_partial(src, target, dst_capacity=None):
    """Returns (ret, bytes): the first min(target, dst_capacity) decoded bytes at most, ret their count or a negative
    error -- lz4.h:308.  dst_capacity None means target."""
    lib = _lib.load()
    s = _u8(src)
    target = int(target)
    cap = target if dst_capacity is None else int(dst_capacity)
    dst = np.empty(max(min(target, cap), 1), dtype=np.uint8)
    sp = s.ctypes.data if len(s) else np.zeros(1, dtype=np.uint8).ctypes.data
    r = int(lib.LZ4_decompress_safe_partial(sp, dst.ctypes.data, len(s), target, cap))
    return r, dst[:max(r, 0)].tobytes()


def LZ4_decompress_safe(src, dst_capacity):
    """Returns (ret, bytes): ret decoded size or negative error -- lz4.h:208."""
    lib = _lib.load()
    s = _u8(src)
    cap = int(dst_capacity)
    dst = np.empty(max(cap, 1), dtype=np.uint8)
    sp = s.ctypes.data if len(s) else np.zeros(1, dtype=np.uint8).ctypes.data
    r = int(lib.LZ4_decompress_safe(sp, dst.ctypes.data, len(s), cap))
    return r, dst[:max(r, 0)].tobytes()
