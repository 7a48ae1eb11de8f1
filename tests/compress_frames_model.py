"""TEST INFRASTRUCTURE: a host model of LZ4B200_compress_frames -- the frame LZ4F_compressFrame writes for independent
blocks without checksums (lz4frame.c:362-373, 406-498, 781-809, 883-921, 1222) at every level, with the block codecs of
the oracle (levels below 2) and of the host HC build (tests/hc_emul.py, levels 2 and up), the call's per-frame
verdicts and its budget rule -- and the seeded corpus of tests/golden/compress_frames.json."""
import hashlib
import struct

import numpy as np

from frame_oracle import optimal_bsid, xxh32_short

ERR_ARG, ERR_DSTSIZE, ERR_LIMIT = -1, -5, -6


def block_bytes(bsid):
    return 1 << (8 + 2 * bsid)


def frame_bsid(requested, n):
    """the block size ID a frame of n bytes is written with"""
    return optimal_bsid(requested or 4, max(n, 0))


def n_blocks(n, bsid):
    bs = block_bytes(bsid)
    return (n + bs - 1) // bs


def bound(n, requested):
    """LZ4F_compressFrameBound(n, &prefs) at the frame's optimal block size ID: 19 + 4 x blocks + n + 4"""
    return 19 + 4 * n_blocks(n, frame_bsid(requested, n)) + n + 4


def header(bsid, content_size):
    """the frame header: magic, FLG, BD, the content size when content_size > 0, the header checksum byte"""
    desc = bytes([(1 << 6) | (1 << 5) | ((1 if content_size > 0 else 0) << 3), bsid << 4])
    if content_size > 0:
        desc += struct.pack("<Q", content_size)
    return struct.pack("<I", 0x184D2204) + desc + bytes([(xxh32_short(desc) >> 8) & 0xFF])


def acceleration(level):
    """lz4frame.c:911-921 with LZ4_compress_fast's clamp (lz4.c:1386-1387)"""
    return 1 if level >= 0 else min(-level + 1, 65537)


def block_codec(oracle, level):
    """(block, capacity) -> (ret, bytes) of the block call LZ4F_makeBlock makes at `level`"""
    if level < 2:
        accel = acceleration(level)
        return lambda blk, cap: oracle.compress(blk, accel, cap)
    import hc_emul
    if level >= 10:
        return lambda blk, cap: hc_emul.host_hc_opt(blk, cap, min(level, 12))
    return lambda blk, cap: hc_emul.host_hc(blk, cap, level)


def frame(data, bsid, content_size, codec, payload=None):
    """the frame of `data` (bytes) at requested block size ID bsid.  codec(block, size - 1) -> (ret, bytes): a block
    whose ret is 0 is stored raw.  payload(i, block) -> (ret, bytes) replaces codec when given (the parallel parse's
    payloads, taken from another call)."""
    data = bytes(data)
    b = frame_bsid(bsid, len(data))
    bs = block_bytes(b)
    out = bytearray(header(b, len(data) if content_size else 0))
    for i, at in enumerate(range(0, len(data), bs)):
        blk = data[at:at + bs]
        r, c = payload(i, blk) if payload else codec(blk, len(blk) - 1)
        if r <= 0 or r >= len(blk):
            out += struct.pack("<I", len(blk) | 0x80000000) + blk
        else:
            out += struct.pack("<I", r) + c[:r]
    out += struct.pack("<I", 0)
    return bytes(out)


def blocks(fr):
    """(stored raw, payload size) of every block of a frame"""
    flg = fr[4]
    ip, out = 7 + (8 if flg & 8 else 0), []
    while True:
        h = struct.unpack_from("<I", fr, ip)[0]
        ip += 4
        if h == 0:
            return out
        out.append((h >> 31, h & 0x7FFFFFFF))
        ip += h & 0x7FFFFFFF


def verdicts(sizes, caps, bsid, max_blocks):
    """per frame (result or None for a frame that passes, class, blocks, base in its class's table), in the call's order:
    LZ4B200_ERR_ARG, LZ4B200_ERR_DSTSIZE, then the budget rule of LZ4B200_decompress_frames"""
    used = [0, 0, 0, 0]
    out = []
    for n, cap in zip(sizes, caps):
        if n < 0 or cap < 0:
            out.append((ERR_ARG, -1, 0, 0))
            continue
        b = frame_bsid(bsid, n)
        if cap < bound(n, bsid):
            out.append((ERR_DSTSIZE, -1, 0, 0))
            continue
        c, k = b - 4, n_blocks(n, b)
        base = used[c]
        used[c] += k
        out.append((ERR_LIMIT if base + k > max_blocks[c] else None, c, k, base))
    return out


def budget(sizes, bsid):
    """the blocks of every class the frames need"""
    need = [0, 0, 0, 0]
    for n in sizes:
        if n >= 0:
            b = frame_bsid(bsid, n)
            need[b - 4] += n_blocks(n, b)
    return need


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


# ------------------------------------------------------------------------------------------
# the golden corpus: seeded inputs the tests rebuild without the reference
# ------------------------------------------------------------------------------------------
FAST_LEVELS = [-70000, -5, 0, 1]
HC_LEVELS = [2, 3, 9, 10, 12, 13]
EDGE_SIZES = [0, 1, 15, 16, 65535, 65536, 65537]


def corpus_data(oracle, kind, size, seed):
    """P50 datagen (compressible, with stored-raw tails) or incompressible bytes"""
    if kind == "p50":
        return oracle.datagen(size, 0.5, seed).tobytes()
    return np.random.default_rng(seed).integers(0, 256, size, dtype=np.uint8).tobytes()


def corpus_cases():
    """(id, kind, size, seed, block size ID, level, content size) of every golden frame"""
    cases = []
    for level in FAST_LEVELS + HC_LEVELS:
        hc = level >= 2
        for bsid in ([0, 4, 5] if hc else [0, 4, 5, 6, 7]):
            bs = block_bytes(bsid or 4)
            if hc:                                     # HC blocks stay at or below 256 KB
                big = [2 * bs + 1] if bs == 65536 else [bs, bs + 1]
            else:
                big = [bs, bs + 1, 2 * bs, 2 * bs + 1]
            sizes = sorted(set(EDGE_SIZES + big))
            for i, size in enumerate(sizes):
                for cs in ([False, True] if not hc else [bool(i % 2)]):
                    kind = ("p50", "rand")[(i + cs + bsid) % 2]
                    seed = (abs(level) * 131 + bsid * 17 + i * 7 + cs) % 100003
                    cases.append(("L%d_b%d_n%d_%s_%s" % (level, bsid, size, kind, "cs" if cs else "nocs"),
                                  kind, size, seed, bsid, level, cs))
    return cases
