"""TEST INFRASTRUCTURE: pure-Python restatement of the LZ4 frame container for independent-block,
checksum-free frames (doc/lz4_Frame_format.md; lz4frame.c:362-373, 781-809, 883-908, 1222), on top of
the oracle's block codec.  Pinned by tests/golden/frames.json (frames made by the reference's
LZ4F_compressFrame) in tests/test_frame.py."""
import struct

P1, P2, P3, P4, P5 = 2654435761, 2246822519, 3266489917, 668265263, 374761393
M = 0xFFFFFFFF


def xxh32_short(data, seed=0):
    """XXH32 for messages shorter than 16 bytes (xxHash specification)."""
    assert len(data) < 16
    h = (seed + P5 + len(data)) & M
    i = 0
    while i + 4 <= len(data):
        h = (h + struct.unpack_from("<I", data, i)[0] * P3) & M
        h = (((h << 17) | (h >> 15)) & M) * P4 & M
        i += 4
    while i < len(data):
        h = (h + data[i] * P5) & M
        h = (((h << 11) | (h >> 21)) & M) * P1 & M
        i += 1
    h ^= h >> 15
    h = h * P2 & M
    h ^= h >> 13
    h = h * P3 & M
    h ^= h >> 16
    return h


def optimal_bsid(requested, src_size):
    proposed, max_block = 4, 64 * 1024
    while requested > proposed:
        if src_size <= max_block:
            return proposed
        proposed += 1
        max_block <<= 2
    return requested


def compress_frame(oracle, data, block_size_id=4, level=0, content_size=False):
    data = bytes(data)
    bsid = optimal_bsid(block_size_id or 4, len(data))
    bs = 1 << (8 + 2 * bsid)
    accel = -level + 1 if level < 0 else 1
    csf = content_size and len(data) > 0
    desc = bytes([(1 << 6) | (1 << 5) | ((1 if csf else 0) << 3), bsid << 4])
    if csf:
        desc += struct.pack("<Q", len(data))
    out = bytearray(struct.pack("<I", 0x184D2204) + desc + bytes([(xxh32_short(desc) >> 8) & 0xFF]))
    for i in range(0, len(data), bs):
        blk = data[i:i + bs]
        r, c = oracle.compress(blk, accel, len(blk) - 1)
        if r == 0 or r >= len(blk):
            out += struct.pack("<I", len(blk) | 0x80000000) + blk
        else:
            out += struct.pack("<I", r) + c
    out += struct.pack("<I", 0)
    return bytes(out)


def frame_of_blocks(oracle, pieces, bsid, content_size=None, raw=()):
    """a frame of independent blocks without checksums, one block per piece (at most the block size of bsid): piece i
    stored raw when i is in `raw`, compressed otherwise; content_size: the header's content-size field (None: absent)"""
    desc = bytes([(1 << 6) | (1 << 5) | ((content_size is not None) << 3), bsid << 4])
    if content_size is not None:
        desc += struct.pack("<Q", content_size)
    out = bytearray(struct.pack("<I", 0x184D2204) + desc + bytes([(xxh32_short(desc) >> 8) & 0xFF]))
    for i, p in enumerate(pieces):
        p = bytes(p)
        assert 0 < len(p) <= 1 << (8 + 2 * bsid)
        if i in raw:
            out += struct.pack("<I", len(p) | 0x80000000) + p
        else:
            r, c = oracle.compress(p, 1)
            out += struct.pack("<I", r) + c
    return bytes(out + struct.pack("<I", 0))


def decompress_frame(oracle, frame):
    assert struct.unpack_from("<I", frame, 0)[0] == 0x184D2204
    flg, bd = frame[4], frame[5]
    hdr = 7 + (8 if flg & 8 else 0) + (4 if flg & 1 else 0)
    assert (xxh32_short(frame[4:hdr - 1]) >> 8) & 0xFF == frame[hdr - 1]
    bs = 1 << (8 + 2 * ((bd >> 4) & 7))
    ip, out = hdr, bytearray()
    while True:
        h = struct.unpack_from("<I", frame, ip)[0]
        ip += 4
        if h == 0:
            break
        sz = h & 0x7FFFFFFF
        if h >> 31:
            out += frame[ip:ip + sz]
        else:
            r, d = oracle.decompress(frame[ip:ip + sz], bs)
            assert r >= 0
            out += d
        ip += sz
    return bytes(out), ip
