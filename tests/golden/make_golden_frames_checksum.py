"""Generate tests/golden/frames_checksum.json from the COMPILED REFERENCE (oracle/_ref/libref_lz4.so and oracle/_ref/lz4).

    python tests/golden/make_golden_frames_checksum.py

It holds, for LZ4B200_decompress_frames_checksummed's tests (which never need the reference):
  - "xxh32": LZ4_XXH32 digests of datagen bytes at lengths 0 .. 100 and several MB, seeds 0 and 0x9E3779B1;
  - "frames": frames of LZ4F_compressFrame with independent blocks and each combination of the block and content checksum
    flags, at block sizes 64 KB .. 4 MB, with stored-raw blocks, with and without the content size: the content's
    recipe, the frame's length and SHA-256 (verbatim when small);
  - "cli": a frame the reference `lz4` tool writes with default options, verbatim, and its content's recipe;
  - "corrupted": for the corrupted corpus of some of those frames (tests/frame_checksum_model.py's mutations), the
    outcome of the reference's one-shot LZ4F_decompress with and without skipChecksums, at the capacity given.
"""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import frame_checksum_model as fm          # noqa: E402
from oracle.pyoracle import Reference      # noqa: E402


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


# [size, proba, seed, noise bytes], bsid, content size, block checksums, content checksum
FRAMES = []
for spec, bsid in [([200000, 0.5, 1, 70000], 4), ([600000, 0.3, 2, 300000], 5), ([1300000, 0.5, 3, 0], 6),
                   ([1500000, 0.9, 4, 1100000], 7)]:
    for k, (bsum, csum) in enumerate([(0, 1), (1, 0), (1, 1), (0, 0)]):
        FRAMES.append((spec, bsid, bool((k + bsid) % 2), bsum, csum))
FRAMES += [([(4 << 20) + 12345, 0.5, 5, 0], 7, True, 0, 1), ([(4 << 20) + 12345, 0.5, 5, 0], 7, False, 1, 1),
           ([0, 0.5, 0, 0], 4, False, 1, 1), ([1, 0.5, 0, 0], 4, True, 1, 1), ([17, 0.5, 6, 17], 4, False, 1, 1),
           ([33, 0.5, 7, 0], 5, True, 0, 1), ([65536, 0.5, 8, 0], 4, True, 1, 1), ([65537, 0.5, 9, 0], 4, False, 1, 1)]
CORRUPT = [0, 1, 2, 4, 5, 6, 13, 14, 18, 19, 23]       # indices of FRAMES whose corrupted corpus is recorded
CLI_SPEC = [20000, 0.5, 11, 3000]
SKIP_SEED = 0x9E3779B1


class _DOpts(C.Structure):                 # LZ4F_decompressOptions_t, lz4frame.h:374-383
    _fields_ = [("stableDst", C.c_uint), ("skipChecksums", C.c_uint), ("reserved1", C.c_uint), ("reserved0", C.c_uint)]


def one_shot(lib, frame, cap, skip):
    """one LZ4F_decompress call on the whole frame: {"error": name or "incomplete" or None, "size", "sha", "consumed"}"""
    ctx = C.c_void_p()
    assert not lib.LZ4F_isError(lib.LZ4F_createDecompressionContext(C.byref(ctx), 100))
    src = np.frombuffer(frame, dtype=np.uint8)
    dst = np.zeros(max(cap, 1), dtype=np.uint8)
    ssz, dsz = C.c_size_t(len(frame)), C.c_size_t(cap)
    opts = _DOpts(0, 1 if skip else 0, 0, 0)
    r = lib.LZ4F_decompress(ctx, dst.ctypes.data, C.byref(dsz), src.ctypes.data, C.byref(ssz), C.byref(opts))
    lib.LZ4F_freeDecompressionContext(ctx)
    if lib.LZ4F_isError(r):
        return {"error": lib.LZ4F_getErrorName(r).decode().replace("ERROR_", ""), "size": None, "sha": None, "consumed": None}
    if r != 0:
        return {"error": "incomplete", "size": None, "sha": None, "consumed": None}
    return {"error": None, "size": dsz.value, "sha": sha(dst[:dsz.value]), "consumed": ssz.value}


def bind(lib):
    lib.LZ4F_createDecompressionContext.restype = C.c_size_t
    lib.LZ4F_createDecompressionContext.argtypes = [C.POINTER(C.c_void_p), C.c_uint]
    lib.LZ4F_freeDecompressionContext.argtypes = [C.c_void_p]
    lib.LZ4F_decompress.restype = C.c_size_t
    lib.LZ4F_decompress.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t), C.c_void_p, C.POINTER(C.c_size_t),
                                    C.c_void_p]
    lib.LZ4F_isError.restype = C.c_uint
    lib.LZ4F_isError.argtypes = [C.c_size_t]
    lib.LZ4F_getErrorName.restype = C.c_char_p
    lib.LZ4F_getErrorName.argtypes = [C.c_size_t]
    lib.LZ4_XXH32.restype = C.c_uint
    lib.LZ4_XXH32.argtypes = [C.c_void_p, C.c_size_t, C.c_uint]


def main():
    ref = Reference()
    lib = ref.lib
    bind(lib)

    digests = []
    d = ref.datagen(3 << 20, 0.5, 42)
    for n in list(range(101)) + [(1 << 20) + 7, (3 << 20) - 5]:
        for seed in (0, SKIP_SEED):
            digests.append({"len": n, "seed": seed, "xxh32": int(lib.LZ4_XXH32(d.ctypes.data, n, seed))})

    frames, corrupted = [], []
    for i, (spec, bsid, csf, bsum, csum) in enumerate(FRAMES):
        data = fm.content(ref.datagen, spec)
        f = ref.compress_frame(data, bsid, 0, csf, content_checksum=csum, block_checksum=bsum)
        row = {"spec": spec, "bsid": bsid, "content_size": csf, "block_sum": bsum, "content_sum": csum,
               "frame_size": len(f), "frame_sha256": sha(f), "src_sha256": sha(data)}
        if len(f) <= 1200:
            row["frame_hex"] = f.hex()
        for skip in (0, 1):
            o = one_shot(lib, f, len(data), skip)
            assert o["error"] is None and o["size"] == len(data) and o["consumed"] == len(f), (i, o)
        frames.append(row)
        if i in CORRUPT:
            cap = len(data) + (1 << (8 + 2 * fm.optimal_bsid(bsid, len(data))))
            for name, m in fm.mutations(f):
                corrupted.append({"frame": i, "mutation": name, "cap": cap,
                                  "verify": one_shot(lib, m, cap, 0), "skip": one_shot(lib, m, cap, 1)})

    with tempfile.TemporaryDirectory() as tmp:
        data = fm.content(ref.datagen, CLI_SPEC)
        src = os.path.join(tmp, "in.bin")
        with open(src, "wb") as fh:
            fh.write(data)
        cli = subprocess.run([os.path.join(ROOT, "oracle", "_ref", "lz4"), "-q", "-c", src], capture_output=True,
                             check=True).stdout
    assert one_shot(lib, cli, len(data), 0)["sha"] == sha(data)

    with open(os.path.join(HERE, "frames_checksum.json"), "w") as fh:
        json.dump({"source": "lz4 v1.10.0: LZ4_XXH32, lib/lz4frame.c LZ4F_compressFrame and LZ4F_decompress (one call per "
                             "frame), programs/lz4 with default options",
                   "xxh32_data": [3 << 20, 0.5, 42], "xxh32": digests, "frames": frames,
                   "cli": {"spec": CLI_SPEC, "frame_hex": cli.hex(), "src_sha256": sha(data)},
                   "corrupted": corrupted}, fh, indent=0)
        fh.write("\n")


if __name__ == "__main__":
    main()
