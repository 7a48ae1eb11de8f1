"""TEST INFRASTRUCTURE: frames for the batched frame decode (LZ4B200_decompress_frames) -- good frames of every block
size, stored-raw blocks and content sizes, the header and chain corpus of mutated frames, a Python walk of the chain of
block headers, and the budget rule.  Used by tests/test_frames_batch_rules.py (CPU) and tests/test_gpu_frames.py."""
import struct

import numpy as np

import frame_oracle as fo

OK, ERR_ARG, ERR_FRAME, ERR_UNSUPPORTED, ERR_DSTSIZE, ERR_LIMIT = 0, -1, -3, -4, -5, -6
MAGIC = 0x184D2204
PAD = 16


def header(flg, bd, content_size=None):
    """a frame header with a correct checksum; content_size is written when FLG's bit 3 is set"""
    desc = bytes([flg, bd]) + (struct.pack("<Q", content_size or 0) if flg & 8 else b"")
    return struct.pack("<I", MAGIC) + desc + bytes([(fo.xxh32_short(desc) >> 8) & 0xFF])


def header_len(frame):
    flg = frame[4]
    return 7 + (8 if flg & 8 else 0) + (4 if flg & 1 else 0)


def walk_prefix(frame):
    """the chain of a frame whose header is valid: ([(offset, size, raw)] of its valid blocks, consumed or None when the
    chain breaks after them)"""
    bs = 1 << (8 + 2 * ((frame[5] >> 4) & 7))
    ip, blocks = header_len(frame), []
    while True:
        if ip + 4 > len(frame):
            return blocks, None
        h = struct.unpack_from("<I", frame, ip)[0]
        ip += 4
        if h == 0:
            return blocks, ip
        sz = h & 0x7FFFFFFF
        if sz > bs or ip + sz > len(frame):
            return blocks, None
        blocks.append((ip, sz, h >> 31))
        ip += sz


def walk(frame):
    """([(offset, size, raw)], consumed) of a frame with a valid header and chain, else None"""
    blocks, consumed = walk_prefix(frame)
    return None if consumed is None else (blocks, consumed)


def short_blocks_frame(oracle, d):
    """the hand-built frame of test_frame.py's irregular inputs: short middle blocks, as a flushing compressor makes"""
    hand = bytearray(header((1 << 6) | (1 << 5), 4 << 4))
    for pce in [d[:1000], d[1000:70000 - 3], d[70000 - 3:70000], d[70000:]]:
        for i in range(0, len(pce), 65536):
            blk = pce[i:i + 65536]
            r, c = oracle.compress(blk, 1, len(blk) - 1)
            hand += (struct.pack("<I", len(blk) | 0x80000000) + blk) if (r == 0 or r >= len(blk)) else (struct.pack("<I", r) + c)
    return bytes(hand + struct.pack("<I", 0))


def good_frames(oracle, seed=0, big=True):
    """(frame, source) pairs: every block size, shrunk block sizes, content size on and off, raw blocks, empty frames"""
    rng = np.random.default_rng(seed)
    out = []
    sizes = [0, 1, 1000, 65535, 65536, 65537, 200000] + ([700000, (1 << 20) + 5, (4 << 20) + 3] if big else [])
    for k, n in enumerate(sizes):
        d = oracle.datagen(n, float(rng.choice([0.3, 0.5, 0.9])), 100 + seed + k).tobytes() if n else b""
        for bsid in (4, 5, 6, 7):
            out.append((fo.compress_frame(oracle, d, bsid, 0, bool((k + bsid) % 2)), d))
    noise = rng.integers(0, 256, 150000, dtype=np.uint8).tobytes()
    out.append((fo.compress_frame(oracle, noise, 5, 0, True), noise))                  # stored-raw blocks (random bytes)
    d = oracle.datagen(140000, 0.5, 7).tobytes()
    pieces = [d[:65536], noise[:300], d[65536:131072], d[131072:]]
    out.append((fo.frame_of_blocks(oracle, pieces, 4, 65536 + 300 + 65536 + len(d) - 131072, raw=(1,)),
                b"".join(pieces)))
    for bsid in (6, 7):                             # small blocks under a large block size ID (not shrunk)
        out.append((fo.frame_of_blocks(oracle, [d[:5000], noise[:700], d[5000:9000]], bsid, 9700 if bsid == 6 else None,
                                       raw=(1,)), d[:5000] + noise[:700] + d[5000:9000]))
    d = oracle.datagen(200000, 0.5, 77).tobytes()
    out.append((short_blocks_frame(oracle, d), d))
    return out


def mutations(frame):
    """(name, bytes) of a valid frame's header and chain corpus: every truncation of the header and into the chain,
    flipped FLG and BD bits (with and without a fixed-up checksum), a bad checksum, a block above the maximum,
    a truncated chain, trailing bytes, a skippable frame"""
    hl = header_len(frame)
    out = [("trunc%d" % k, frame[:k]) for k in range(0, hl + 5)]
    for bit in range(8):
        for pos in (4, 5):
            b = bytearray(frame)
            b[pos] ^= 1 << bit
            out.append(("flip%d.%d" % (pos, bit), bytes(b)))
            nl = header_len(b)
            if nl + 4 <= len(b):
                b2 = bytearray(b)
                b2[nl - 1] = (fo.xxh32_short(bytes(b2[4:nl - 1])) >> 8) & 0xFF
                out.append(("flipfix%d.%d" % (pos, bit), bytes(b2)))
    b = bytearray(frame)
    b[hl - 1] ^= 0x5A
    out.append(("checksum", bytes(b)))
    bs = 1 << (8 + 2 * ((frame[5] >> 4) & 7))
    b = bytearray(frame)
    struct.pack_into("<I", b, hl, bs + 1)
    out.append(("oversize", bytes(b)))
    out.append(("noEndMark", frame[:-4]))
    out.append(("halfEndMark", frame[:-2]))
    w = walk(frame)
    if w and w[0]:
        off, sz, _ = w[0][-1]
        out.append(("cutLastBlock", frame[:off + sz // 2]))
    out.append(("trailing", frame + b"trailing bytes"))
    out.append(("skippable", struct.pack("<II", 0x184D2A53, 4) + b"abcd"))
    return out


def budget_rule(frames, status, cls, budget):
    """the statuses of the index passes under a budget, from the statuses and classes without one (cls >= 0: the header
    passed): the chain walk stops after budget + 1 blocks, then LZ4B200_ERR_LIMIT is assigned in frame order"""
    run = [0, 0, 0, 0]
    out = []
    for fr, st, c in zip(frames, status, cls):
        if c < 0:
            out.append(st)
            continue
        blocks, consumed = walk_prefix(fr)
        if len(blocks) > budget[c]:
            n = budget[c] + 1
        elif consumed is None:
            out.append(ERR_FRAME)
            continue
        else:
            n = len(blocks)
        out.append(ERR_LIMIT if run[c] + n > budget[c] else OK)
        run[c] += n
    return out


def layout(frames, align=1, gap=PAD, seed=0):
    """frames laid out in one buffer with `gap` bytes between them (PAD of readable padding at both ends); offsets start
    at odd positions when align == 1"""
    rng = np.random.default_rng(seed)
    buf, offs = bytearray(b"\xEE" * PAD), []
    for f in frames:
        buf += b"\xEE" * (int(rng.integers(0, 7)) * align)
        offs.append(len(buf))
        buf += f + b"\xEE" * gap
    buf += b"\xEE" * PAD
    return bytes(buf), offs
