"""TEST INFRASTRUCTURE: a Python model of LZ4B200_decompress_files -- the grammar of a .lz4 file as `lz4 -d` reads it
piped to its standard input (LZ4 frames, skippable frames, legacy streams), the unit and block budget, and the per-file
result, consumed offset, prefix and bytes -- on top of the oracle's block decoder and frame_checksum_model's XXH32.
Pinned by tests/golden/decompress_files.json, which tests/golden/make_golden_decompress_files.py writes by running the
reference `lz4` tool; used by tests/test_decompress_files_rules.py (CPU) and tests/test_gpu_decompress_files.py.

Every builder here (skippable frames, legacy streams) writes the bytes the reference tool writes or reads."""
import struct

import numpy as np

import frame_checksum_model as fm
import frame_corpus as fc

OK, ERR_ARG, ERR_FRAME, ERR_UNSUPPORTED, ERR_DSTSIZE, ERR_LIMIT = 0, -1, -3, -4, -5, -6
ERR_CHECKSUM = fm.ERR_CHECKSUM
LEGACY_MAGIC, SKIPPABLE_MAGIC = 0x184C2102, 0x184D2A50
LEGACY_BLOCK, LEGACY_BOUND = 8 << 20, 8421520             # LEGACY_BLOCKSIZE, LZ4_COMPRESSBOUND(8 MiB)
CLASSES, LEGACY_CLASS = 5, 4
INF = 1 << 62


def skippable(payload, nibble=0):
    """a skippable frame: magic 0x184D2A50 + nibble, LE32 size, the payload"""
    return struct.pack("<II", SKIPPABLE_MAGIC + nibble, len(payload)) + bytes(payload)


def legacy(compress, data):
    """`lz4 -l`'s stream of data: the magic, then per 8 MiB chunk LE32 size and LZ4_compress_default's block.  compress:
    bytes -> compressed bytes (the oracle's or the reference's level-1 block compressor)"""
    data = bytes(data)
    out = bytearray(struct.pack("<I", LEGACY_MAGIC))
    for i in range(0, len(data), LEGACY_BLOCK):
        c = compress(data[i:i + LEGACY_BLOCK])
        out += struct.pack("<I", len(c)) + c
    return bytes(out)


def _frame_unit(data, p, max_blocks, skip):
    """pass 1 of an LZ4 frame at p (fc_index_frame_mode): (status, cls, count, length or None)"""
    fr = data[p:]
    if len(fr) < 7:
        return ERR_FRAME, -1, 0, None
    flg, bd = fr[4], fr[5]
    hl = fc.header_len(fr)
    if (flg >> 6) != 1 or flg & 2 or len(fr) < hl or bd & 0x8F or ((bd >> 4) & 7) < 4:
        return ERR_FRAME, -1, 0, None
    if (fm.xxh32(fr[4:hl - 1]) >> 8) & 0xFF != fr[hl - 1]:
        return ERR_FRAME, -1, 0, None
    if not flg & 0x20 or flg & 1:
        return ERR_UNSUPPORTED, -1, 0, None
    cls = ((bd >> 4) & 7) - 4
    bsum, csum = fm.sums_of(fr)
    bs, ip, n = 1 << (8 + 2 * (cls + 4)), hl, 0
    while True:
        if ip + 4 > len(fr):
            return ERR_FRAME, cls, 0, None
        h = struct.unpack_from("<I", fr, ip)[0]
        ip += 4
        if h == 0:
            if csum:
                if ip + 4 > len(fr):
                    return ERR_FRAME, cls, 0, None
                ip += 4
            return OK, cls, n, ip
        sz = h & 0x7FFFFFFF
        if sz > bs or ip + sz + (4 if bsum else 0) > len(fr):
            return ERR_FRAME, cls, 0, None
        ip += sz + (4 if bsum else 0)
        n += 1
        if n > max_blocks[cls]:
            return OK, cls, n, None


def legacy_blocks(data, p):
    """the blocks [(offset, size)] of the legacy unit at p and its end, or (blocks so far, None) when it breaks"""
    ip, blocks = p + 4, []
    while True:
        if ip == len(data):
            return blocks, ip
        if ip + 4 > len(data):
            return blocks, None
        w = struct.unpack_from("<I", data, ip)[0]
        if w > LEGACY_BOUND:
            return blocks, ip
        if ip + 4 + w > len(data):
            return blocks, None
        blocks.append((ip + 4, w))
        ip += 4 + w


def next_unit(data, p, max_blocks, skip):
    """pass 1 of the unit at p (fc_next_unit): dict(off, kind, status, cls, count, length or None)"""
    u = dict(off=p, kind="bad", status=ERR_FRAME, cls=-1, count=0, length=None)
    rem = len(data) - p
    if rem < 4:
        return u
    magic = struct.unpack_from("<I", data, p)[0]
    if magic == fc.MAGIC:
        st, cls, n, ln = _frame_unit(data, p, max_blocks, skip)
        u.update(kind="frame", status=st, cls=cls if st == OK else -1, count=n, length=ln)
    elif magic & 0xFFFFFFF0 == SKIPPABLE_MAGIC:
        if rem >= 8 and 8 + struct.unpack_from("<I", data, p + 4)[0] <= rem:
            u.update(kind="skip", status=OK, length=8 + struct.unpack_from("<I", data, p + 4)[0])
    elif magic == LEGACY_MAGIC:
        blocks, end = legacy_blocks(data, p)
        u.update(kind="legacy", cls=LEGACY_CLASS)
        if len(blocks) > max_blocks[LEGACY_CLASS]:
            u.update(status=OK, count=max_blocks[LEGACY_CLASS] + 1)
        elif end is None:
            u.update(status=ERR_FRAME, cls=-1)
        else:
            u.update(status=OK, count=len(blocks), length=end - p)
    return u


def walk_file(data, max_units, max_blocks, skip):
    """fc_index_file: the units the walk takes"""
    p, units = 0, []
    while p < len(data) and len(units) <= max_units:
        u = next_unit(data, p, max_blocks, skip)
        units.append(u)
        if u["status"] != OK or u["length"] is None:
            break
        p += u["length"]
    return units


def _frame_decode(oracle, fr, room, skip, content):
    """one LZ4 frame that passed pass 1, at `room` bytes of room: frame_checksum_model.decode, and with content False
    the content checksum not compared"""
    if content:
        return fm.decode(oracle, fr, room, skip)[:2]
    r, out, _ = fm.decode(oracle, fr, room, skip)
    if r != ERR_CHECKSUM or skip or not fm.sums_of(fr)[1]:
        return r, out
    # a CHECKSUM result may be the content checksum's (when the frame has one): decode again with the content checksum
    # field made right
    blocks, consumed = fm.walk(fr)
    r2, out2, _ = fm.decode(oracle, fr, room, True)
    if r2 < 0:
        return r, out
    fixed = bytearray(fr)
    struct.pack_into("<I", fixed, consumed - 4, fm.xxh32(out2))
    return fm.decode(oracle, bytes(fixed), room, skip)[:2]


def _legacy_decode(oracle, data, u, room):
    out = bytearray()
    for o, w in legacy_blocks(data, u["off"])[0]:
        r, d = oracle.decompress(data[o:o + w], LEGACY_BLOCK) if w else (-1, b"")
        if r < 0:
            return ERR_FRAME, b""
        if len(out) + r > room:
            return ERR_DSTSIZE, b""
        out += d
    return len(out), bytes(out)


def decompress_files(oracle, files, caps, max_units, max_blocks, skip=False, size_only=False, content=True):
    """The call on a batch: [(result, consumed, prefix, bytes)] per file.  caps: per-file room (ignored when size_only).
    content=False: content checksums are not compared (size_only implies it)."""
    content = content and not size_only
    bad = [not size_only and cap < 0 for cap in caps]       # ERR_ARG: the walk takes no unit
    walks = [[] if b else walk_file(bytes(d), max_units, max_blocks, skip) for d, b in zip(files, bad)]
    index, used = 0, [0] * CLASSES
    for units in walks:                                   # unit index, block budget (fc_place_frame)
        for u in units:
            u["index"] = index
            index += 1
            u["limit"] = False
            if u["index"] < max_units and u["status"] == OK and u["cls"] >= 0:
                base = used[u["cls"]]
                used[u["cls"]] += u["count"]
                u["limit"] = base + u["count"] > max_blocks[u["cls"]]
    out = []
    for d, cap, units, b in zip(files, caps, walks, bad):
        d = bytes(d)
        if b:
            out.append((ERR_ARG, 0, 0, b""))
            continue
        room = INF if size_only else cap
        res, at, got = None, len(d), bytearray()
        for u in units:
            if u["index"] >= max_units:
                res, at = (u["status"] if u["status"] != OK else ERR_LIMIT), u["off"]
            elif u["status"] != OK:
                res, at = u["status"], u["off"]
            elif u["limit"]:
                res, at = ERR_LIMIT, u["off"]
            else:
                if u["kind"] == "skip":
                    r, b = 0, b""
                elif u["kind"] == "legacy":
                    r, b = _legacy_decode(oracle, d, u, room - len(got))
                else:
                    r, b = _frame_decode(oracle, d[u["off"]:u["off"] + u["length"]], room - len(got), skip, content)
                if r < 0:
                    res, at = r, u["off"]
                else:
                    got += b
            if res is not None:
                break
        out.append((len(got) if res is None else res, at, len(got), bytes(got)))
    return out


def budget_needed(files, skip=False):
    """(units, blocks per class) a batch needs so that no file gets ERR_LIMIT"""
    big = [1 << 40] * CLASSES
    units, blocks = 0, [0] * CLASSES
    for d in files:
        for u in walk_file(bytes(d), 1 << 40, big, skip):
            units += 1
            if u["status"] == OK and u["cls"] >= 0:
                blocks[u["cls"]] += u["count"]
    return units, blocks


def build_file(oracle, recipe):
    """the bytes of a corpus file from its recipe: {"parts": [...], "flip": [offsets] or None, "cut": length or None}:
    the parts, each byte at an offset in "flip" XORed with 0x20, the first "cut" bytes.  Parts:
      ["frame", spec, bsid, content size, block sums, content sum]  LZ4F_compressFrame's frame (frame_checksum_model)
      ["hex", "..."]                                                 verbatim bytes (frames the `lz4` tool wrote)
      ["skip", nibble, size, seed]                                   a skippable frame of seeded random bytes
      ["legacy", spec]                                               `lz4 -l`'s stream of the content
      ["word", value]                                                one LE32 word
    spec: frame_checksum_model.content's [size, proba, seed, noise]"""
    out = bytearray()
    for part in recipe["parts"]:
        kind = part[0]
        if kind == "frame":
            out += fm.compress_frame(oracle, fm.content(oracle.datagen, part[1]), *part[2:6])
        elif kind == "hex":
            out += bytes.fromhex(part[1])
        elif kind == "skip":
            out += skippable(np.random.default_rng(part[3]).integers(0, 256, part[2], dtype=np.uint8).tobytes(), part[1])
        elif kind == "legacy":
            out += legacy(lambda b: oracle.compress(b, 1)[1], fm.content(oracle.datagen, part[1]))
        elif kind == "word":
            out += struct.pack("<I", part[1])
        else:
            raise ValueError(kind)
    for at in recipe.get("flip") or ():               # corrupted bytes
        out[at] ^= 0x20
    cut = recipe.get("cut")
    return bytes(out if cut is None else out[:cut])
