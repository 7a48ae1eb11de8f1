"""One-shot LZ4 frames of independent blocks (SURVEY.md section 8 f-1): the Python face of
LZ4B200_compressFrame_host / LZ4B200_decompressFrame_host (the roles of LZ4F_compressFrame,
lz4frame.h:224, and of a one-shot LZ4F_decompress, lz4frame.h:470)."""
import ctypes as C

import numpy as np

from . import _lib
from .block import _u8


class Lz4FrameError(RuntimeError):
    def __init__(self, code, what):
        names = {-1: "bad argument", -2: "CUDA error", -3: "malformed frame", -4: "unsupported frame feature",
                 -5: "destination too small"}
        super().__init__("%s: %s (%d)" % (what, names.get(int(code), "error"), int(code)))
        self.code = int(code)


def compress_frame(data, block_size_id=4, level=0, content_size=False):
    lib = _lib.load()
    src = _u8(data)
    cap = int(lib.LZ4B200_compressFrameBound(len(src), int(block_size_id)))
    if cap < 0:
        raise Lz4FrameError(cap, "LZ4B200_compressFrameBound")
    dst = np.empty(cap, dtype=np.uint8)
    r = int(lib.LZ4B200_compressFrame_host(src.ctypes.data if len(src) else None, len(src), dst.ctypes.data, cap,
                                           int(block_size_id), int(level), 1 if content_size else 0))
    if r < 0:
        raise Lz4FrameError(r, "LZ4B200_compressFrame_host")
    return dst[:r].tobytes()


def decompress_frame(frame, capacity):
    lib = _lib.load()
    src = _u8(frame)
    dst = np.empty(max(int(capacity), 1), dtype=np.uint8)
    consumed = C.c_int64(0)
    r = int(lib.LZ4B200_decompressFrame_host(src.ctypes.data, len(src), dst.ctypes.data, int(capacity), C.byref(consumed)))
    if r < 0:
        raise Lz4FrameError(r, "LZ4B200_decompressFrame_host")
    return dst[:r].tobytes()
