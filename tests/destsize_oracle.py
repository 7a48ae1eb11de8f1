"""LZ4_compress_destSize on the CPU -- TEST INFRASTRUCTURE ONLY.

`DestSizeOracle()` builds tests/destsize_oracle.c together with oracle/lz4_oracle.c (gcc, into a temporary directory,
once per process) and wraps oracle_lz4_compress_destSize.  `reference_dest_size` calls the reference's own
LZ4_compress_destSize / LZ4_compress_destSize_extState in oracle/_ref/libref_lz4.so (an `oracle.pyoracle.Reference`).
"""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_DIR = os.path.join(os.path.dirname(HERE), "oracle")

# path codes of oracle_lz4_compress_destSize (tests/destsize_oracle.c)
PATHS = {0: "fast", 1: "empty", 2: "no_room", 3: "literals", 4: "next_match", 5: "reduced", 6: "last_literals",
         7: "filled", 8: "bad_size"}

_u8p = C.POINTER(C.c_uint8)
_ip = C.POINTER(C.c_int)
_lib = None


def _load():
    global _lib
    if _lib is None:
        gcc = shutil.which("gcc") or shutil.which("cc")
        if not gcc:
            raise RuntimeError("a C compiler (gcc) is needed to build the destSize oracle")
        tmp = tempfile.mkdtemp(prefix="destsize_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libdestsize_oracle.so")
        subprocess.run([gcc, "-O2", "-std=c99", "-Wall", "-shared", "-fPIC", "-I" + ORACLE_DIR, "-o", so,
                        os.path.join(HERE, "destsize_oracle.c"), os.path.join(ORACLE_DIR, "lz4_oracle.c")], check=True)
        lib = C.CDLL(so)
        lib.oracle_lz4_compress_destSize.restype = C.c_int
        lib.oracle_lz4_compress_destSize.argtypes = [_u8p, _u8p, _ip, C.c_int, C.c_int, _ip]
        _lib = lib
    return _lib


def _as_u8(data):
    if isinstance(data, np.ndarray):
        assert data.dtype == np.uint8
        return np.ascontiguousarray(data)
    return np.frombuffer(bytes(data), dtype=np.uint8)


def _call(fn, data, target):
    """fn(src pointer, dst pointer, c_int n) -> (ret, path); checks that nothing at or past dst + target was written.
    Returns (ret, consumed, bytes, path), consumed = what the call leaves in *srcSizePtr."""
    src = _as_u8(data)
    room = max(int(target), 0)
    dst = np.full(room + 64, 0xA5, dtype=np.uint8)
    n = C.c_int(len(src))
    r, path = fn(src.ctypes.data_as(_u8p) if len(src) else None, dst.ctypes.data_as(_u8p), n)
    assert (dst[room:] == 0xA5).all(), "destSize wrote at or past targetDstSize"
    return r, n.value, dst[:max(r, 0)].tobytes(), path


class DestSizeOracle:
    """compress_dest_size(data, target, acceleration=None): acceleration None is LZ4_compress_destSize, an integer
    LZ4_compress_destSize_extState; returns (ret, consumed, bytes, path code)."""

    def __init__(self):
        self.lib = _load()

    def compress_dest_size(self, data, target, acceleration=None):
        acc = 1 if acceleration is None else int(acceleration)

        def fn(sp, dp, n):
            path = C.c_int(-1)
            r = int(self.lib.oracle_lz4_compress_destSize(sp, dp, C.byref(n), int(target), acc, C.byref(path)))
            return r, path.value
        return _call(fn, data, target)


def reference_dest_size(ref, data, target, acceleration=None):
    """The reference's LZ4_compress_destSize (acceleration None) or LZ4_compress_destSize_extState; path is None."""
    lib = ref.lib
    if not getattr(lib, "_destsize_bound", False):
        lib.LZ4_compress_destSize.restype = C.c_int
        lib.LZ4_compress_destSize.argtypes = [_u8p, _u8p, _ip, C.c_int]
        lib.LZ4_compress_destSize_extState.restype = C.c_int
        lib.LZ4_compress_destSize_extState.argtypes = [C.c_void_p, _u8p, _u8p, _ip, C.c_int, C.c_int]
        lib._destsize_state = np.zeros(16416 // 8, dtype=np.uint64)     # sizeof(LZ4_stream_t), lz4.h:729-733
        lib._destsize_bound = True

    def fn(sp, dp, n):
        if acceleration is None:
            return int(lib.LZ4_compress_destSize(sp, dp, C.byref(n), int(target))), None
        return int(lib.LZ4_compress_destSize_extState(lib._destsize_state.ctypes.data, sp, dp, C.byref(n), int(target),
                                                      int(acceleration))), None
    return _call(fn, data, target)
