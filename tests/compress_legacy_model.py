"""TEST INFRASTRUCTURE: a host model of LZ4B200_compress_legacy -- the `lz4 -l` legacy stream the reference tool writes
(LZ4IO_compressLegacy_internal, programs/lz4io.c:766-910) at every level, with the block codecs of the oracle (levels
below 3) and of the host HC build (tests/hc_emul.py, levels 3 and up), the call's per-file verdicts and its budget
rule -- and the seeded corpus of tests/golden/compress_legacy.json."""
import hashlib
import struct

import numpy as np

ERR_ARG, ERR_DSTSIZE, ERR_LIMIT = -1, -5, -6
MAGIC = 0x184C2102
CHUNK = 8 << 20                 # LEGACY_BLOCKSIZE
MIB = 1 << 20


def compress_bound(n):
    return n + n // 255 + 16


def n_chunks(n):
    return (n + CHUNK - 1) // CHUNK


def bound(n):
    """4 + the sum over the chunks of 4 + LZ4_compressBound(chunk)"""
    return 4 + sum(4 + compress_bound(min(CHUNK, n - at)) for at in range(0, n, CHUNK))


def acceleration(level):
    """lz4io.c:788-794 with LZ4_compress_fast's reading of it (lz4.c:1386-1387): -level for negative levels, 0 -- read
    as 1 -- otherwise, at most 65537"""
    return min(-level, 65537) if level < 0 else 1


def block_codec(oracle, level):
    """(chunk, capacity) -> (ret, bytes) of the block call the tool makes at `level`"""
    if level < 3:
        accel = acceleration(level)
        return lambda blk, cap: oracle.compress(blk, accel, cap)
    import hc_emul
    if level >= 10:
        return lambda blk, cap: hc_emul.host_hc_opt(blk, cap, min(level, 12))
    return lambda blk, cap: hc_emul.host_hc(blk, cap, level)


def stream(data, codec):
    """the legacy stream of `data`: the magic, then per chunk its LE32 compressed size and block"""
    data = bytes(data)
    out = bytearray(struct.pack("<I", MAGIC))
    for at in range(0, len(data), CHUNK):
        blk = data[at:at + CHUNK]
        r, c = codec(blk, compress_bound(len(blk)))
        assert r > 0
        out += struct.pack("<I", r) + c[:r]
    return bytes(out)


def chunks(st):
    """the compressed size of every block of a stream"""
    ip, out = 4, []
    while ip < len(st):
        k = struct.unpack_from("<I", st, ip)[0]
        out.append(k)
        ip += 4 + k
    return out


def verdicts(sizes, caps, max_blocks):
    """per file (result or None for a file that passes, chunks, base in the table), in the call's order:
    LZ4B200_ERR_ARG, LZ4B200_ERR_DSTSIZE, then the budget rule"""
    used, out = 0, []
    for n, cap in zip(sizes, caps):
        if n < 0 or cap < 0:
            out.append((ERR_ARG, 0, 0))
        elif cap < bound(n):
            out.append((ERR_DSTSIZE, 0, 0))
        else:
            k = n_chunks(n)
            out.append((ERR_LIMIT if used + k > max_blocks else None, k, used))
            used += k
    return out


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


# ------------------------------------------------------------------------------------------
# the golden corpus: seeded inputs the tests rebuild without the reference
# ------------------------------------------------------------------------------------------
FAST_LEVELS = [-70000, -65537, -17, -2, -1, 0, 1, 2]       # --fast=70000 .. --fast=1, -0, -1, -2
HC_LEVELS = [3, 9, 10, 12, 13]
FAST_SIZES = [0, 1, 13, 4096, 65536, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK + 17]
HC_SIZES = [0, 1, 13, 4096, 65536, MIB]
KINDS = ["p50", "p90", "rand", "zero"]
SPLIT_TAIL = 100000             # the multi-block HC file: a random 8 MiB chunk, then this many P50 bytes


def corpus_data(oracle, kind, size, seed):
    """P50 or P90 datagen, incompressible bytes, zeros, or (split) a random chunk followed by P50 bytes"""
    if kind in ("p50", "p90"):
        return oracle.datagen(size, 0.5 if kind == "p50" else 0.9, seed).tobytes()
    if kind == "rand":
        return np.random.default_rng(seed).integers(0, 256, size, dtype=np.uint8).tobytes()
    if kind == "zero":
        return bytes(size)
    head = min(size, CHUNK)
    return (np.random.default_rng(seed).integers(0, 256, head, dtype=np.uint8).tobytes()
            + oracle.datagen(size - head, 0.5, seed).tobytes())


def cli_args(level):
    """the `lz4` options of a level"""
    return ["--fast=%d" % -level] if level < 0 else ["-%d" % level]


def corpus_cases():
    """(id, kind, size, seed, level) of every golden stream"""
    cases = []
    for level in FAST_LEVELS + HC_LEVELS:
        sizes = FAST_SIZES if level < 3 else HC_SIZES
        for i, size in enumerate(sizes):
            kind = KINDS[(i + abs(level)) % len(KINDS)]
            seed = (abs(level) * 131 + i * 7) % 100003
            cases.append(("L%d_n%d_%s" % (level, size, kind), kind, size, seed, level))
        if level < 3:
            cases.append(("L%d_n%d_rand" % (level, 20 * MIB), "rand", 20 * MIB, abs(level) % 1000 + 1, level))
    for level in (3, 10):
        size = CHUNK + SPLIT_TAIL
        cases.append(("L%d_n%d_split" % (level, size), "split", size, 77 + level, level))
    return cases
