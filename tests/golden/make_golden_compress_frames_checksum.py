"""Generate tests/golden/compress_frames_checksum.json from the COMPILED REFERENCE (oracle/_ref/libref_lz4.so and the
`lz4` tool oracle/_ref/lz4).

    python tests/golden/make_golden_compress_frames_checksum.py

1. For every case of tests/compress_frames_checksum_model.checksum_cases() -- levels -5, 0, 1, 2, 9, 10, 12, block
   size IDs 0 and 4 .. 7 (4 from level 2), with and without the content size, sizes 0, 1, block - 1, block, block + 1 and
   2 x block + 1, P50 and incompressible data -- and each of the flag combinations B (block checksums), C (content
   checksum) and BC, it records LZ4F_compressFrame's frame length and SHA-256 and LZ4F_compressFrameBound, for
   independent blocks, autoFlush 1.  It asserts that one byte below the bound is rejected.  Frames of at most 160
   bytes are kept verbatim (hex).
2. The `lz4` tool's output (`lz4 -q -c <args>`) for compress_frames_checksum_model.cli_data(), a multi-block input
   of more than 8 MB built from a seed, for every entry of CLI_RUNS.  Each must equal LZ4F_compressFrame with the matching prefs
   (independent blocks, no content size, the level, block size ID and checksum flags of the run); a reference for which
   that fails makes this script fail rather than record the difference.
The inputs are rebuilt by the tests from their seeds, so the tests never need the reference."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE), HERE]

import numpy as np                                  # noqa: E402

import compress_frames_checksum_model as M           # noqa: E402
from make_golden_compress_frames import Prefs       # noqa: E402
from oracle.pyoracle import Oracle, Reference       # noqa: E402


def lz4f(lib, data, bsid, level, cs, block_sum, content_sum):
    """(frame, bound) of LZ4F_compressFrame; asserts dstMaxSize_tooSmall one byte below the bound"""
    data = np.frombuffer(bytes(data), dtype=np.uint8).copy()
    size = len(data)
    p = Prefs()
    p.frameInfo.blockSizeID = bsid
    p.frameInfo.blockMode = 1                       # LZ4F_blockIndependent
    p.frameInfo.contentChecksumFlag = 1 if content_sum else 0
    p.frameInfo.blockChecksumFlag = 1 if block_sum else 0
    p.frameInfo.contentSize = size if cs else 0
    p.compressionLevel = level
    p.autoFlush = 1
    bound = int(lib.LZ4F_compressFrameBound(size, C.byref(p)))
    dst = np.empty(bound, dtype=np.uint8)
    src = data.ctypes.data if size else None
    r = lib.LZ4F_compressFrame(dst.ctypes.data, bound, src, size, C.byref(p))
    assert not lib.LZ4F_isError(r)
    assert lib.LZ4F_isError(lib.LZ4F_compressFrame(dst.ctypes.data, bound - 1, src, size, C.byref(p)))
    return dst[:r].tobytes(), bound


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
    for cid, kind, size, seed, bsid, level, cs in M.checksum_cases():
        data = M.corpus_data(orc, kind, size, seed)
        rec = {"id": cid, "kind": kind, "size": size, "seed": seed, "bsid": bsid, "level": level, "content_size": cs,
               "sums": {}}
        for name, (bsum, csum) in M.SUM_FLAGS.items():
            out, bound = lz4f(lib, data, bsid, level, cs, bsum, csum)
            assert bound == M.bound(size, bsid, bsum, csum), (cid, name)
            r = {"length": len(out), "sha256": hashlib.sha256(out).hexdigest(), "bound": bound}
            if len(out) <= 160:
                r["hex"] = out.hex()
            rec["sums"][name] = r
        frames.append(rec)

    tool = os.path.join(ROOT, "oracle", "_ref", "lz4")
    data = M.cli_data(orc)
    cli = []
    for args, bsid, level, bsum, csum in M.CLI_RUNS:
        out = subprocess.run([tool, "-q", "-c", *args], input=data, capture_output=True, check=True).stdout
        ref, _ = lz4f(lib, data, bsid, level, False, bsum, csum)
        assert out == ref, "lz4 %s differs from LZ4F_compressFrame with the matching prefs" % " ".join(args)
        cli.append({"args": args, "bsid": bsid, "level": level, "block_sum": bsum, "content_sum": csum,
                    "length": len(out), "sha256": hashlib.sha256(out).hexdigest()})

    with open(os.path.join(HERE, "compress_frames_checksum.json"), "w") as fh:
        json.dump({"source": "lz4 v1.10.0: LZ4F_compressFrame and LZ4F_compressFrameBound (lib/lz4frame.c), blockMode "
                             "LZ4F_blockIndependent, autoFlush 1, with blockChecksumFlag (B), contentChecksumFlag (C) or "
                             "both; and the lz4 command-line tool (programs/), lz4 -q -c <args>",
                   "cli_input": {"size": M.CLI_SIZE, "seed": M.CLI_SEED, "kind": "datagen P50"},
                   "frames": frames, "cli": cli}, fh, indent=0)
        fh.write("\n")


if __name__ == "__main__":
    main()
