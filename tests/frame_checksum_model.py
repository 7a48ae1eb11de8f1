"""TEST INFRASTRUCTURE: XXH32 and LZ4 frames with block and content checksums in Python, for
LZ4B200_decompress_frames_checksummed -- XXH32 from the published xxHash specification, a builder of the frames
LZ4F_compressFrame makes with checksums (on top of the oracle's block codec), the corrupted corpus, and a model of the
call's result for one frame in either checksum mode.  Pinned by tests/golden/frames_checksum.json, which
tests/golden/make_golden_frames_checksum.py writes from the reference."""
import struct

import numpy as np

import frame_corpus as fc

P1, P2, P3, P4, P5 = 2654435761, 2246822519, 3266489917, 668265263, 374761393
M = 0xFFFFFFFF
ERR_CHECKSUM = -7
FLG_BLOCK_SUM, FLG_CONTENT_SUM = 1 << 4, 1 << 2


def xxh32(data, seed=0):
    """XXH32 (xxHash specification): four lanes over 16-byte stripes, then the remaining words and bytes, the avalanche"""
    data = bytes(data)
    n, i = len(data), 0
    if n >= 16:
        v1, v2, v3, v4 = (seed + P1 + P2) & M, (seed + P2) & M, seed & M, (seed - P1) & M
        i = n & ~15
        for a, b, c, d in struct.iter_unpack("<4I", memoryview(data)[:i]):
            v1 = (v1 + a * P2) & M
            v1 = (((v1 << 13) | (v1 >> 19)) & M) * P1 & M
            v2 = (v2 + b * P2) & M
            v2 = (((v2 << 13) | (v2 >> 19)) & M) * P1 & M
            v3 = (v3 + c * P2) & M
            v3 = (((v3 << 13) | (v3 >> 19)) & M) * P1 & M
            v4 = (v4 + d * P2) & M
            v4 = (((v4 << 13) | (v4 >> 19)) & M) * P1 & M
        h = (((v1 << 1) | (v1 >> 31)) + ((v2 << 7) | (v2 >> 25)) + ((v3 << 12) | (v3 >> 20)) + ((v4 << 18) | (v4 >> 14))) & M
    else:
        h = (seed + P5) & M
    h = (h + n) & M
    while i + 4 <= n:
        h = (h + struct.unpack_from("<I", data, i)[0] * P3) & M
        h = (((h << 17) | (h >> 15)) & M) * P4 & M
        i += 4
    while i < n:
        h = (h + data[i] * P5) & M
        h = (((h << 11) | (h >> 21)) & M) * P1 & M
        i += 1
    h ^= h >> 15
    h = h * P2 & M
    h ^= h >> 13
    h = h * P3 & M
    return h ^ (h >> 16)


def content(datagen, spec):
    """the bytes of a golden frame's content: spec = [size, proba, seed, noise]; `noise` bytes of seeded random data
    (stored raw by the compressor) replace the middle of the datagen bytes"""
    size, proba, seed, noise = spec
    d = bytearray(datagen(size, proba, seed).tobytes() if size else b"")
    if noise:
        at = size // 3
        d[at:at + noise] = np.random.default_rng(seed).integers(0, 256, noise, dtype=np.uint8).tobytes()
    return bytes(d)


def optimal_bsid(requested, n):
    """LZ4F_optimalBSID (lz4frame.c:362-373)"""
    bsid, top = 4, 64 * 1024
    while requested > bsid:
        if n <= top:
            return bsid
        bsid += 1
        top <<= 2
    return requested


def compress_frame(oracle, data, bsid, content_size, block_sum, content_sum):
    """the frame LZ4F_compressFrame makes at level 0 with independent blocks and the given checksum flags"""
    data = bytes(data)
    bsid = optimal_bsid(bsid, len(data))
    bs = 1 << (8 + 2 * bsid)
    csf = content_size and len(data) > 0
    flg = (1 << 6) | (1 << 5) | (8 if csf else 0) | (FLG_BLOCK_SUM if block_sum else 0) | (FLG_CONTENT_SUM if content_sum else 0)
    out = bytearray(fc.header(flg, bsid << 4, len(data) if csf else None))
    for i in range(0, len(data), bs):
        blk = data[i:i + bs]
        r, c = oracle.compress(blk, 1, len(blk) - 1)
        payload, word = (blk, len(blk) | 0x80000000) if (r == 0 or r >= len(blk)) else (c, r)
        out += struct.pack("<I", word) + payload
        if block_sum:
            out += struct.pack("<I", xxh32(payload))
    out += struct.pack("<I", 0)
    if content_sum:
        out += struct.pack("<I", xxh32(data))
    return bytes(out)


def frame_of_blocks(oracle, pieces, bsid, raw=(), block_sum=False, content_sum=False, content_size=None):
    """a frame of one block per piece (stored raw when its index is in `raw`) with the given checksums"""
    flg = (1 << 6) | (1 << 5) | (8 if content_size is not None else 0)
    flg |= (FLG_BLOCK_SUM if block_sum else 0) | (FLG_CONTENT_SUM if content_sum else 0)
    out = bytearray(fc.header(flg, bsid << 4, content_size))
    for i, p in enumerate(pieces):
        p = bytes(p)
        if i in raw:
            payload, word = p, len(p) | 0x80000000
        else:
            r, payload = oracle.compress(p, 1)
            word = r
        out += struct.pack("<I", word) + payload
        if block_sum:
            out += struct.pack("<I", xxh32(payload))
    out += struct.pack("<I", 0)
    if content_sum:
        out += struct.pack("<I", xxh32(b"".join(bytes(p) for p in pieces)))
    return bytes(out)


def sums_of(frame):
    return (bool(frame[4] & FLG_BLOCK_SUM), bool(frame[4] & FLG_CONTENT_SUM))


def walk(frame):
    """([(offset, size, raw)], consumed) of a frame with a valid header and a chain with checksum fields, else None"""
    bsum, csum = sums_of(frame)
    bs = 1 << (8 + 2 * ((frame[5] >> 4) & 7))
    ip, blocks = fc.header_len(frame), []
    while True:
        if ip + 4 > len(frame):
            return None
        h = struct.unpack_from("<I", frame, ip)[0]
        ip += 4
        if h == 0:
            if not csum:
                return blocks, ip
            return (blocks, ip + 4) if ip + 4 <= len(frame) else None
        sz = h & 0x7FFFFFFF
        if sz > bs or ip + sz + (4 if bsum else 0) > len(frame):
            return None
        blocks.append((ip, sz, h >> 31))
        ip += sz + (4 if bsum else 0)


def mutations(frame):
    """(name, bytes) of the corrupted corpus of a checksummed frame: a flipped byte in a compressed payload, in a raw
    payload, in a block checksum (of a compressed and of a raw block), in the content checksum, the content-size field
    +-1 (header checksum fixed up), truncation inside the last block checksum and inside the content checksum"""
    bsum, csum = sums_of(frame)
    blocks, consumed = walk(frame)
    out = []

    def flip(name, at):
        b = bytearray(frame)
        b[at] ^= 0x20
        out.append((name, bytes(b)))

    comp = [blk for blk in blocks if not blk[2]]
    raw = [blk for blk in blocks if blk[2]]
    if comp:
        flip("compressedPayload", comp[0][0] + comp[0][1] // 2)
    if raw:
        flip("rawPayload", raw[0][0] + raw[0][1] // 2)
    if bsum:
        if comp:
            flip("compressedBlockSum", comp[0][0] + comp[0][1] + 1)
        if raw:
            flip("rawBlockSum", raw[0][0] + raw[0][1] + 2)
        if blocks:
            o, sz, _ = blocks[-1]
            out.append(("truncBlockSum", frame[:o + sz + 2]))
    if csum:
        flip("contentSum", consumed - 3)
        out.append(("truncContentSum", frame[:consumed - 2]))
    if frame[4] & 8:                              # (not to 0, which lz4frame reads as "no content size")
        hl = fc.header_len(frame)
        size = struct.unpack_from("<Q", frame, 6)[0]
        for delta in (1, -1) if size > 1 else (1,):
            b = bytearray(frame)
            struct.pack_into("<Q", b, 6, size + delta)
            b[hl - 1] = (xxh32(bytes(b[4:hl - 1])) >> 8) & 0xFF
            out.append(("contentSize%+d" % delta, bytes(b)))
    return out


# the reference's LZ4F errors (LZ4F_getErrorName without "ERROR_") and the library's code for them; "incomplete": the
# one-shot LZ4F_decompress stopped, asking for more input
REF_CLASS = {"blockChecksum_invalid": ERR_CHECKSUM, "contentChecksum_invalid": ERR_CHECKSUM}


def ref_class(outcome):
    """the library's result class for a reference outcome: decoded size, ERR_CHECKSUM or ERR_FRAME"""
    if outcome["error"] is None:
        return outcome["size"]
    return REF_CLASS.get(outcome["error"], fc.ERR_FRAME)


def decode(oracle, frame, cap, skip):
    """the result of LZ4B200_decompress_frames_checksummed on one frame alone: (result, bytes, consumed)"""
    if len(frame) < 7 or struct.unpack_from("<I", frame, 0)[0] != fc.MAGIC:
        return (fc.ERR_UNSUPPORTED if len(frame) >= 7 and (struct.unpack_from("<I", frame, 0)[0] & 0xFFFFFFF0) == 0x184D2A50
                else fc.ERR_FRAME), b"", 0
    flg, bd = frame[4], frame[5]
    hl = fc.header_len(frame)
    if (flg >> 6) != 1 or flg & 2 or len(frame) < hl or bd & 0x8F or ((bd >> 4) & 7) < 4:
        return fc.ERR_FRAME, b"", 0
    if (xxh32(frame[4:hl - 1]) >> 8) & 0xFF != frame[hl - 1]:
        return fc.ERR_FRAME, b"", 0
    if not flg & 0x20 or flg & 1:
        return fc.ERR_UNSUPPORTED, b"", 0
    w = walk(frame)
    if w is None:
        return fc.ERR_FRAME, b"", 0
    blocks, consumed = w
    bsum, csum = sums_of(frame)
    # a content-size field past 2^63 is a size no frame decodes to: the frame fails at its end (frameSize_wrong)
    csize = min(struct.unpack_from("<Q", frame, 6)[0], (1 << 63) - 1) if flg & 8 else -1
    bs = 1 << (8 + 2 * ((bd >> 4) & 7))
    out = bytearray()
    for o, sz, raw in blocks:
        payload = frame[o:o + sz]
        bad = bsum and not skip and xxh32(payload) != struct.unpack_from("<I", frame, o + sz)[0]
        if bad and not raw:
            return ERR_CHECKSUM, b"", consumed
        if raw:
            r, d = sz, payload
        else:
            r, d = oracle.decompress(payload, bs)
        if r < 0:
            return fc.ERR_FRAME, b"", consumed
        if len(out) + r > cap:
            return fc.ERR_DSTSIZE, b"", consumed
        if csize >= 0 and len(out) + r > csize:
            return fc.ERR_FRAME, b"", consumed
        if bad:
            return ERR_CHECKSUM, b"", consumed
        out += d
    if csize >= 0 and csize != len(out):
        return fc.ERR_FRAME, b"", consumed
    if csum and not skip and xxh32(out) != struct.unpack_from("<I", frame, consumed - 4)[0]:
        return ERR_CHECKSUM, b"", consumed
    return len(out), bytes(out), consumed
