"""Generate tests/golden/compress_frames.json from the COMPILED REFERENCE (oracle/_ref/libref_lz4.so).

    python tests/golden/make_golden_compress_frames.py

For every case of tests/compress_frames_model.corpus_cases() -- levels -70 000 .. 13, block size IDs 0 and 4 .. 7, with
and without the content size, sizes 0 .. 2 x block size + 1, P50 and incompressible data -- it records
LZ4F_compressFrame's frame length and SHA-256 and LZ4F_compressFrameBound, for independent blocks without checksums,
autoFlush 1.  Frames of at most 160 bytes are kept verbatim (hex).  The inputs are rebuilt by the tests from their seeds
(the project's own datagen and numpy), so the tests never need the reference."""
import ctypes as C
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE), HERE]

import numpy as np                                  # noqa: E402

import compress_frames_model as M                   # noqa: E402
from oracle.pyoracle import Oracle, Reference       # noqa: E402


class FrameInfo(C.Structure):                       # LZ4F_frameInfo_t, lz4frame.h:175-183
    _fields_ = [("blockSizeID", C.c_int), ("blockMode", C.c_int), ("contentChecksumFlag", C.c_int),
                ("frameType", C.c_int), ("contentSize", C.c_ulonglong), ("dictID", C.c_uint),
                ("blockChecksumFlag", C.c_int)]


class Prefs(C.Structure):                           # LZ4F_preferences_t, lz4frame.h:192-198
    _fields_ = [("frameInfo", FrameInfo), ("compressionLevel", C.c_int), ("autoFlush", C.c_uint),
                ("favorDecSpeed", C.c_uint), ("reserved", C.c_uint * 3)]


def main():
    lib = Reference().lib
    lib.LZ4F_compressFrameBound.restype = C.c_size_t
    lib.LZ4F_compressFrameBound.argtypes = [C.c_size_t, C.c_void_p]
    lib.LZ4F_compressFrame.restype = C.c_size_t
    lib.LZ4F_compressFrame.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.LZ4F_isError.restype = C.c_uint
    lib.LZ4F_isError.argtypes = [C.c_size_t]
    orc = Oracle()
    frames = []
    for cid, kind, size, seed, bsid, level, cs in M.corpus_cases():
        data = np.frombuffer(M.corpus_data(orc, kind, size, seed), dtype=np.uint8).copy()
        p = Prefs()
        p.frameInfo.blockSizeID = bsid
        p.frameInfo.blockMode = 1                   # LZ4F_blockIndependent
        p.frameInfo.contentSize = size if cs else 0
        p.compressionLevel = level
        p.autoFlush = 1
        bound = int(lib.LZ4F_compressFrameBound(size, C.byref(p)))
        dst = np.empty(bound, dtype=np.uint8)
        r = lib.LZ4F_compressFrame(dst.ctypes.data, bound, data.ctypes.data if size else None, size, C.byref(p))
        assert not lib.LZ4F_isError(r), cid
        short = lib.LZ4F_compressFrame(dst.ctypes.data, bound - 1, data.ctypes.data if size else None, size, C.byref(p))
        assert lib.LZ4F_isError(short), cid         # dstMaxSize_tooSmall one byte below the bound
        out = dst[:r].tobytes()
        rec = {"id": cid, "kind": kind, "size": size, "seed": seed, "bsid": bsid, "level": level, "content_size": cs,
               "length": int(r), "sha256": hashlib.sha256(out).hexdigest(), "bound": bound}
        if r <= 160:
            rec["hex"] = out.hex()
        frames.append(rec)
    with open(os.path.join(HERE, "compress_frames.json"), "w") as fh:
        json.dump({"source": "lz4 v1.10.0: LZ4F_compressFrame and LZ4F_compressFrameBound (lib/lz4frame.c), blockMode "
                             "LZ4F_blockIndependent, no checksums, autoFlush 1",
                   "frames": frames}, fh, indent=0)
        fh.write("\n")


if __name__ == "__main__":
    main()
