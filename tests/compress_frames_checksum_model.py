"""TEST INFRASTRUCTURE: a host model of LZ4B200_compress_frames_checksummed -- the frame LZ4F_compressFrame writes for
independent blocks with XXH32 block checksums (lz4frame.c:904-907), a content checksum (lz4frame.c:1225-1229) or both
(FLG bits 4 and 2, lz4frame.c:781-809; the bound of lz4frame.c:376-417), on top of tests/compress_frames_model.py,
whose frame without checksums it extends -- and the seeded corpus of tests/golden/compress_frames_checksum.json and the
`lz4` tool's files in it.  With both flags off every function here is compress_frames_model's."""
import struct

from compress_frames_model import (ERR_ARG, ERR_DSTSIZE, ERR_LIMIT, block_bytes, block_codec, budget,  # noqa: F401
                                   corpus_data, frame_bsid, n_blocks, sha)
from frame_checksum_model import xxh32
from frame_oracle import xxh32_short

FLG_BLOCK_SUM, FLG_CONTENT_SUM = 1 << 4, 1 << 2


def bound(n, requested, block_sum=False, content_sum=False):
    """LZ4F_compressFrameBound(n, &prefs) at the frame's optimal block size ID: 19 + (4 + 4 B) x blocks + n + 4 + 4 C"""
    return 19 + (8 if block_sum else 4) * n_blocks(n, frame_bsid(requested, n)) + n + 4 + (4 if content_sum else 0)


def header(bsid, content_size, block_sum=False, content_sum=False):
    """the frame header: magic, FLG (with the checksum bits), BD, the content size when content_size > 0, the header
    checksum byte"""
    desc = bytes([(1 << 6) | (1 << 5) | (FLG_BLOCK_SUM if block_sum else 0) | ((1 if content_size > 0 else 0) << 3)
                  | (FLG_CONTENT_SUM if content_sum else 0), bsid << 4])
    if content_size > 0:
        desc += struct.pack("<Q", content_size)
    return struct.pack("<I", 0x184D2204) + desc + bytes([(xxh32_short(desc) >> 8) & 0xFF])


def frame(data, bsid, content_size, codec, payload=None, block_sum=False, content_sum=False, xxh=xxh32):
    """compress_frames_model.frame with the checksums: after every block the LE32 xxh(stored payload) with block_sum
    (the compressed bytes, or a stored-raw block's source bytes), after the EndMark the LE32 xxh(data) with
    content_sum.  xxh(bytes): XXH32 with seed 0 (default: the Python XXH32 of tests/frame_checksum_model.py)."""
    data = bytes(data)
    b = frame_bsid(bsid, len(data))
    bs = block_bytes(b)
    out = bytearray(header(b, len(data) if content_size else 0, block_sum, content_sum))
    for i, at in enumerate(range(0, len(data), bs)):
        blk = data[at:at + bs]
        r, c = payload(i, blk) if payload else codec(blk, len(blk) - 1)
        if r <= 0 or r >= len(blk):
            stored, word = blk, len(blk) | 0x80000000
        else:
            stored, word = bytes(c[:r]), r
        out += struct.pack("<I", word) + stored
        if block_sum:
            out += struct.pack("<I", xxh(stored))
    out += struct.pack("<I", 0)
    if content_sum:
        out += struct.pack("<I", xxh(data))
    return bytes(out)


def blocks(fr):
    """(stored raw, payload size) of every block of a frame, its block checksums skipped"""
    flg = fr[4]
    ip, out = 7 + (8 if flg & 8 else 0), []
    while True:
        h = struct.unpack_from("<I", fr, ip)[0]
        ip += 4
        if h == 0:
            return out
        out.append((h >> 31, h & 0x7FFFFFFF))
        ip += (h & 0x7FFFFFFF) + (4 if flg & FLG_BLOCK_SUM else 0)


def verdicts(sizes, caps, bsid, max_blocks, block_sum=False, content_sum=False):
    """per frame (result or None for a frame that passes, class, blocks, base in its class's table), in the call's order:
    LZ4B200_ERR_ARG, LZ4B200_ERR_DSTSIZE against the bound for the checksums, then the budget rule of
    LZ4B200_decompress_frames"""
    used = [0, 0, 0, 0]
    out = []
    for n, cap in zip(sizes, caps):
        if n < 0 or cap < 0:
            out.append((ERR_ARG, -1, 0, 0))
            continue
        b = frame_bsid(bsid, n)
        if cap < bound(n, bsid, block_sum, content_sum):
            out.append((ERR_DSTSIZE, -1, 0, 0))
            continue
        c, k = b - 4, n_blocks(n, b)
        base = used[c]
        used[c] += k
        out.append((ERR_LIMIT if base + k > max_blocks[c] else None, c, k, base))
    return out


# ------------------------------------------------------------------------------------------
# the checksummed corpus (tests/golden/compress_frames_checksum.json): every case is written with each of the three
# nonzero flag combinations
# ------------------------------------------------------------------------------------------
SUM_FLAGS = {"B": (True, False), "C": (False, True), "BC": (True, True)}
SUM_FAST_LEVELS = [-5, 0, 1]
SUM_HC_LEVELS = [2, 9, 10, 12]


def checksum_cases():
    """(id, kind, size, seed, block size ID, level, content size): sizes 0, 1, block - 1, block, block + 1 and
    2 x block + 1, with and without the content size, P50 and incompressible data in turn; block size IDs 0 and 4 .. 7
    below level 2, 4 (64 KB blocks: one thread parses an HC block) from level 2"""
    cases = []
    for level in SUM_FAST_LEVELS + SUM_HC_LEVELS:
        for bsid in ([4] if level >= 2 else [0, 4, 5, 6, 7]):
            bs = block_bytes(bsid or 4)
            for i, size in enumerate([0, 1, bs - 1, bs, bs + 1, 2 * bs + 1]):
                for cs in (False, True):
                    kind = ("p50", "rand")[(i + cs + bsid) % 2]
                    seed = (abs(level) * 257 + bsid * 19 + i * 11 + cs) % 100003
                    cases.append(("S%d_b%d_n%d_%s_%s" % (level, bsid, size, kind, "cs" if cs else "nocs"),
                                  kind, size, seed, bsid, level, cs))
    return cases


CLI_SIZE, CLI_SEED = 8 * (1 << 20) + 123457, 2024
# (arguments of the `lz4` tool, block size ID, level, block checksums, content checksum): -9 runs with -B4, because one
# thread parses an HC block and a 4 MB block takes it tens of seconds
CLI_RUNS = [([], 7, 1, False, True), (["-BX"], 7, 1, True, True), (["-9", "-B4"], 4, 9, False, True),
            (["-B4"], 4, 1, False, True), (["--no-frame-crc"], 7, 1, False, False)]


def cli_data(oracle):
    """the input of the `lz4` tool's frames: datagen P50 of CLI_SIZE bytes"""
    return oracle.datagen(CLI_SIZE, 0.5, CLI_SEED).tobytes()
