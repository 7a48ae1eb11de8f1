"""Generate tests/golden/frames_scale.json from the COMPILED REFERENCE (oracle/_ref/libref_lz4.so).

    python tests/golden/make_golden_frames_scale.py

It holds the digests of the far frame of tests/test_frames_scale_rules.py (one 64 KB-class frame of 65 540 blocks whose
content is 2^32 + 3 x 65 536 + 19 bytes), which the tests rebuild and never need the reference for:
  - "sha256": the content's SHA-256;
  - "xxh32": LZ4_XXH32(content, 0) in one call, and "xxh32_streamed": LZ4_XXH32_reset + LZ4_XXH32_update in 64 KB steps +
    LZ4_XXH32_digest, as LZ4F_decompress computes the content checksum;
  - "frame_size", "frame_sha256": the frame with that content checksum;
  - "lz4f": the outcome of one LZ4F_decompress call on the whole frame at capacity = content size.
Needs about 9 GB of host memory (the content and the reference's output)."""
import ctypes as C
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE), HERE]

import test_frames_scale_rules as S                 # noqa: E402
from make_golden_frames_checksum import bind, one_shot   # noqa: E402
from oracle.pyoracle import Reference               # noqa: E402


def main():
    lib = Reference().lib
    bind(lib)
    lib.LZ4_XXH32_createState.restype = C.c_void_p
    lib.LZ4_XXH32_freeState.argtypes = [C.c_void_p]
    lib.LZ4_XXH32_reset.argtypes = [C.c_void_p, C.c_uint]
    lib.LZ4_XXH32_update.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    lib.LZ4_XXH32_digest.restype = C.c_uint
    lib.LZ4_XXH32_digest.argtypes = [C.c_void_p]

    content = S.far_content()
    at = content.ctypes.data
    one = int(lib.LZ4_XXH32(at, S.FAR_SIZE, 0))
    st = lib.LZ4_XXH32_createState()
    lib.LZ4_XXH32_reset(st, 0)
    for k in range(0, S.FAR_SIZE, S.BLOCK):
        lib.LZ4_XXH32_update(st, at + k, min(S.BLOCK, S.FAR_SIZE - k))
    streamed = int(lib.LZ4_XXH32_digest(st))
    lib.LZ4_XXH32_freeState(st)
    sha = hashlib.sha256(memoryview(content)).hexdigest()
    del content

    frame = S.far_frame(one)
    outcome = one_shot(lib, frame, S.FAR_SIZE, 0)
    assert outcome["sha"] == sha, outcome
    with open(os.path.join(HERE, "frames_scale.json"), "w") as fh:
        json.dump({"source": "lz4 v1.10.0: LZ4_XXH32 and LZ4_XXH32_update (lib/xxhash.c), LZ4F_decompress (lib/lz4frame.c, "
                             "one call on the whole frame)",
                   "content_size": S.FAR_SIZE, "blocks": S.FAR_BLOCKS, "sha256": sha, "xxh32": one,
                   "xxh32_streamed": streamed, "frame_size": len(frame),
                   "frame_sha256": hashlib.sha256(frame).hexdigest(),
                   "lz4f": {"error": outcome["error"], "size": outcome["size"], "consumed": outcome["consumed"]}},
                  fh, indent=1)
        fh.write("\n")


if __name__ == "__main__":
    main()
