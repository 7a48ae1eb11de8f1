"""TEST INFRASTRUCTURE: a seeded fuzz of the container calls -- the frame, checksummed-frame, legacy-stream and whole-file
writers and readers -- after the reference's tests/frametest.c: a case generator that draws preferences, sizes, data
and capacities, mutation operators that corrupt a valid file and name what they did, and judges that give the expected
(result, consumed, prefix, bytes) of every call.

The judges run the reference (oracle/_ref/libref_lz4.so: LZ4F_compressFrame, LZ4F_decompress, LZ4_compress_fast,
LZ4_compress_HC) where it is built, and the host models otherwise (compress_frames_checksum_model,
compress_legacy_model, frame_checksum_model, decompress_files_model).  Used by tests/test_container_fuzz_rules.py (the
models against the reference, and against the digests of tests/golden/container_fuzz.json) and
tests/test_gpu_container_fuzz.py (the GPU calls against the judges)."""
import ctypes as C
import hashlib
import os
import struct
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (os.path.dirname(HERE), HERE, os.path.join(HERE, "golden")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import compress_frames_checksum_model as CM  # noqa: E402
import compress_legacy_model as LM  # noqa: E402
import decompress_files_model as DM  # noqa: E402
import frame_checksum_model as FM  # noqa: E402
import frame_corpus as FC  # noqa: E402

OK, ERR_ARG, ERR_FRAME, ERR_UNSUPPORTED, ERR_DSTSIZE, ERR_LIMIT, ERR_CHECKSUM = 0, -1, -3, -4, -5, -6, -7
VERDICTS = {ERR_ARG: "ARG", ERR_FRAME: "FRAME", ERR_UNSUPPORTED: "UNSUPPORTED", ERR_DSTSIZE: "DSTSIZE",
            ERR_LIMIT: "LIMIT", ERR_CHECKSUM: "CHECKSUM"}
MIB = 1 << 20

LEVELS = [-70000, -17, -1, 0, 1, 2, 3, 9, 10, 12]
BSIDS = [0, 4, 5, 6, 7]
KINDS = ["p0", "p50", "p90", "p100", "p50lit", "rand", "zero", "period", "win65534", "win65535", "win65536",
         "win32768", "win70000", "copy65535", "copy65536", "copy65537", "rcopy65536", "noisy"]
MUTATIONS = ["magic", "flg_fixed", "flg_stale", "bd_fixed", "bd_stale", "csize_fixed", "csize_stale", "dictid",
             "linked", "raw_bit", "size0", "size_bs1", "size_past", "payload", "blocksum", "contentsum", "cut",
             "cut_edge", "garbage", "wrap", "swap"]


def verdict(r):
    return "OK" if r >= 0 else VERDICTS[r]


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


# ------------------------------------------------------------------------------------------
# data
# ------------------------------------------------------------------------------------------
def data(oracle, kind, n, seed):
    """n bytes of a data kind: datagen at match probability 0, 0.5, 0.9, 1 (p50lit: literal probability 0.2), random,
    zeros, a random period of 1 .. 8 bytes, random data repeated at a period around LZ4's 65 535-byte window (winP),
    datagen (copyD) or random data (rcopyD) with 5 000-byte copies D bytes back, and datagen with an incompressible
    middle third (stored-raw blocks next to compressed ones)"""
    rng = np.random.default_rng(seed)
    if n == 0:
        return b""
    if kind in ("p0", "p50", "p90", "p100"):
        return oracle.datagen(n, int(kind[1:]) / 100.0, seed).tobytes()
    if kind == "p50lit":
        return oracle.datagen(n, 0.5, seed, 0.2).tobytes()
    if kind == "rand":
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    if kind == "zero":
        return bytes(n)
    if kind == "period":
        return np.tile(rng.integers(0, 256, 1 + seed % 8, dtype=np.uint8), n // (1 + seed % 8) + 1)[:n].tobytes()
    if kind.startswith("win"):
        p = int(kind[3:])
        return np.tile(rng.integers(0, 256, p, dtype=np.uint8), n // p + 1)[:n].tobytes()
    if kind.startswith("copy") or kind.startswith("rcopy"):
        dist = int(kind.lstrip("rcopy"))
        d = bytearray(oracle.datagen(n, 0.5, seed).tobytes() if kind[0] == "c" else
                      rng.integers(0, 256, n, dtype=np.uint8).tobytes())
        for at in range(0, n - dist - 5000, 3 * dist + 12345):
            d[at + dist:at + dist + 5000] = d[at:at + 5000]
        return bytes(d)
    if kind == "noisy":
        d = bytearray(oracle.datagen(n, 0.5, seed).tobytes())
        d[n // 3:2 * n // 3] = rng.integers(0, 256, 2 * n // 3 - n // 3, dtype=np.uint8).tobytes()
        return bytes(d)
    raise ValueError(kind)


# ------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------
def block_bytes(bsid):
    return 1 << (8 + 2 * (bsid or 4))


def size_cap(level, legacy):
    """the largest source a case draws at a level: one thread parses an HC block (DESIGN 3.8)"""
    hc = level >= (3 if legacy else 2)
    if not hc:
        return 9 * MIB
    return 160 * 1024 if level >= 10 else 330 * 1024


def sizes_of(bs, cap):
    """the edge sizes of a block size: 0, 1, 12, 13, bs +- 1 and k x bs +- 1 for k up to 3, and the sizes that put a
    block edge on a 1 MiB group edge of the host pipelines -- those at most cap"""
    edges = {0, 1, 12, 13, MIB - 1, MIB, MIB + 1, 2 * MIB - 1, 2 * MIB + 1}
    for k in (1, 2, 3):
        edges |= {k * bs - 1, k * bs, k * bs + 1}
    return sorted(e for e in edges if e <= cap)


def case(seed, k):
    """case k of seed: one writer call's preferences and items.  The same (seed, k) always gives the same case.
    dict(legacy, level, bsid, cs, bsum, csum, parallel, items=[dict(kind, size, seed, cap)]): cap is "bound",
    "bound-1", "small" (a random capacity below the bound) or "neg" (-1)."""
    rng = np.random.default_rng([seed, k])
    legacy = k % 4 == 3                                  # every fourth case; the levels cycle case by case
    level = LEVELS[(k + seed) % len(LEVELS)]
    bsid = 0 if legacy else int(rng.choice(BSIDS))
    cs, bsum, csum = (False, False, False) if legacy else tuple(bool(x) for x in rng.integers(0, 2, 3))
    parallel = bool(not legacy and level < 2 and rng.random() < 0.3)
    cap = size_cap(level, legacy)
    edges = sizes_of(LM.CHUNK if legacy else block_bytes(bsid), cap)
    if legacy and level < 3:
        edges += [LM.CHUNK - 1, LM.CHUNK + 1]
    hc = level >= (3 if legacy else 2)
    n_items = int(rng.choice([1, 2, 3, 5, 8, 13] if hc else [1, 2, 5, 13, 40, 200]))
    budget = (2 if hc else 20) * MIB if n_items <= 40 else 4 * MIB
    items, total = [], 0
    for i in range(n_items):
        r = rng.random()
        if r < 0.5:
            size = int(rng.choice(edges))
        elif r < 0.8 or n_items > 40:
            size = int(rng.integers(0, min(cap, 70000) + 1))
        else:
            size = int(rng.integers(0, cap + 1))
        size = min(size, max(budget - total, 0))
        total += size
        capmode = str(rng.choice(["bound"] * 7 + ["bound-1", "small", "neg"]))
        items.append(dict(kind=str(rng.choice(KINDS)), size=size, seed=int(rng.integers(0, 1 << 30)), cap=capmode))
    return dict(legacy=legacy, level=level, bsid=bsid, cs=cs, bsum=bsum, csum=csum, parallel=parallel, items=items)


def bound(c, n):
    """the model's bound of an item of case c"""
    return LM.bound(n) if c["legacy"] else CM.bound(n, c["bsid"], c["bsum"], c["csum"])


def capacity(c, item, rng_seed):
    """the capacity an item is given"""
    b = bound(c, item["size"])
    mode = item["cap"]
    if mode == "bound":
        return b
    if mode == "bound-1":
        return b - 1
    if mode == "neg":
        return -1
    return int(np.random.default_rng(rng_seed).integers(0, b))


def case_data(oracle, c):
    return [data(oracle, it["kind"], it["size"], it["seed"]) for it in c["items"]]


# ------------------------------------------------------------------------------------------
# mutations: valid file -> (class, corrupted file)
# ------------------------------------------------------------------------------------------
def _fix_hc(b):
    hl = FC.header_len(b)
    b[hl - 1] = (FM.xxh32(bytes(b[4:hl - 1])) >> 8) & 0xFF


def mutate(fr, rng, cls=None, other=None, oracle=None):
    """a corrupted copy of the valid frame fr, by the operator cls (drawn when None): (cls, bytes).  other: a second
    valid frame with fr's preferences (for "swap"); oracle: the block compressor of "wrap"'s legacy stream."""
    cls = cls or str(rng.choice(MUTATIONS))
    b = bytearray(fr)
    hl = FC.header_len(fr)
    blocks = chain(fr)
    bsum, csum = FM.sums_of(fr)
    consumed = (blocks[-1][0] + blocks[-1][1] + (4 if bsum else 0) if blocks else hl) + 4 + (4 if csum else 0)
    bs = 1 << (8 + 2 * ((fr[5] >> 4) & 7))
    if cls == "magic":
        b[int(rng.integers(0, 4))] ^= int(rng.integers(1, 256))
    elif cls in ("flg_fixed", "flg_stale"):
        b[4] ^= 1 << int(rng.choice([1, 1, 1, 6, 7, 3, 2, 4]))   # reserved bit, version, content size and checksum flags
        if cls == "flg_fixed" and len(b) >= FC.header_len(b):
            _fix_hc(b)
    elif cls in ("bd_fixed", "bd_stale"):
        b[5] ^= 1 << int(rng.choice([0, 3, 4, 5, 6, 7]))
        if cls == "bd_fixed":
            _fix_hc(b)
    elif cls in ("csize_fixed", "csize_stale"):
        if not fr[4] & 8:
            return mutate(fr, rng, "flg_stale", other, oracle)
        b[6 + int(rng.integers(0, 8))] ^= 1 << int(rng.integers(0, 8))
        if cls == "csize_fixed":
            _fix_hc(b)
    elif cls == "dictid":
        b[4] |= 1
        b[hl - 1:hl - 1] = struct.pack("<I", int(rng.integers(0, 1 << 32)))
        _fix_hc(b)
    elif cls == "linked":
        b[4] &= ~0x20
        _fix_hc(b)
    elif cls in ("raw_bit", "size0", "size_bs1", "size_past"):
        if not blocks:
            return mutate(fr, rng, "cut", other, oracle)
        o, sz, raw = blocks[int(rng.integers(0, len(blocks)))]
        word = {"raw_bit": (sz | (0 if raw else 0x80000000)), "size0": 0 if rng.random() < 0.5 else 0x80000000,
                "size_bs1": bs + 1 | (0x80000000 if raw else 0),
                "size_past": min(len(fr) - o + int(rng.integers(0, 9)), bs) | (0x80000000 if raw else 0)}[cls]
        struct.pack_into("<I", b, o - 4, word)
    elif cls == "payload":
        if not blocks or not any(sz for _, sz, _ in blocks):
            return mutate(fr, rng, "magic", other, oracle)
        o, sz, _ = blocks[int(rng.integers(0, len(blocks)))]
        b[o + int(rng.integers(0, sz))] ^= 1 << int(rng.integers(0, 8))
    elif cls == "blocksum":
        if not bsum or not blocks:
            return mutate(fr, rng, "contentsum" if csum else "payload", other, oracle)
        o, sz, _ = blocks[int(rng.integers(0, len(blocks)))]
        b[o + sz + int(rng.integers(0, 4))] ^= 1 << int(rng.integers(0, 8))
    elif cls == "contentsum":
        if not csum:
            return mutate(fr, rng, "blocksum" if bsum else "payload", other, oracle)
        b[consumed - 4 + int(rng.integers(0, 4))] ^= 1 << int(rng.integers(0, 8))
    elif cls == "cut":
        b = b[:int(rng.integers(0, len(fr)))]
    elif cls == "cut_edge":
        edges = [hl] + [o - 4 for o, _, _ in blocks] + [o + sz for o, sz, _ in blocks] + [consumed - 4]
        b = b[:max(0, min(len(fr) - 1, int(rng.choice(edges)) + int(rng.integers(-1, 2))))]
    elif cls == "garbage":
        b += rng.integers(0, 256, int(rng.integers(1, 40)), dtype=np.uint8).tobytes()
    elif cls == "wrap":
        pre = DM.skippable(rng.integers(0, 256, int(rng.integers(0, 50)), dtype=np.uint8).tobytes(), int(rng.integers(16)))
        post = DM.legacy(lambda x: oracle.compress(x, 1)[1], rng.integers(0, 4, int(rng.integers(0, 3000)),
                                                                          dtype=np.uint8).tobytes())
        b = bytearray(pre) + b + post
    elif cls == "swap":
        ow = chain(other) if other is not None else None
        if not blocks or not ow:
            return mutate(fr, rng, "payload", other, oracle)
        o, sz, _ = blocks[int(rng.integers(0, len(blocks)))]
        p, psz, _ = ow[int(rng.integers(0, len(ow)))]
        extra = 4 if bsum else 0
        b = b[:o - 4] + bytearray(other[p - 4:p + psz + extra]) + b[o + sz + extra:]
    else:
        raise ValueError(cls)
    return cls, bytes(b)


# ------------------------------------------------------------------------------------------
# the reference
# ------------------------------------------------------------------------------------------
class _DOpts(C.Structure):                 # LZ4F_decompressOptions_t, lz4frame.h
    _fields_ = [("stableDst", C.c_uint), ("skipChecksums", C.c_uint), ("reserved1", C.c_uint), ("reserved0", C.c_uint)]


class _Ref:
    """the reference calls the judges make"""

    def __init__(self, reference):
        self.r = reference
        lib = self.lib = reference.lib
        lib.LZ4F_createDecompressionContext.restype = C.c_size_t
        lib.LZ4F_createDecompressionContext.argtypes = [C.POINTER(C.c_void_p), C.c_uint]
        lib.LZ4F_freeDecompressionContext.argtypes = [C.c_void_p]
        lib.LZ4F_decompress.restype = C.c_size_t
        lib.LZ4F_decompress.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t), C.c_void_p,
                                        C.POINTER(C.c_size_t), C.c_void_p]
        lib.LZ4F_isError.restype = C.c_uint
        lib.LZ4F_isError.argtypes = [C.c_size_t]
        lib.LZ4F_getErrorName.restype = C.c_char_p
        lib.LZ4F_getErrorName.argtypes = [C.c_size_t]
        lib.LZ4_compress_HC.restype = C.c_int
        lib.LZ4_compress_HC.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
        lib.LZ4_XXH32.restype = C.c_uint
        lib.LZ4_XXH32.argtypes = [C.c_char_p, C.c_size_t, C.c_uint]

    def xxh32(self, b):
        return int(self.lib.LZ4_XXH32(bytes(b), len(b), 0))

    def skipped_block_sums(self, fr):
        """fr with every compressed block's checksum made right: under skipChecksums the library compares none, while
        LZ4F_decompress still compares a compressed block's (tests/test_decompress_files_rules.py lists the deviation)"""
        w = chain(fr) if len(fr) >= 7 and len(fr) >= FC.header_len(fr) else None
        if w is None or not fr[4] & FM.FLG_BLOCK_SUM:
            return fr
        b = bytearray(fr)
        for o, sz, raw in w:
            if not raw:
                struct.pack_into("<I", b, o + sz, self.xxh32(fr[o:o + sz]))
        return bytes(b)

    def decompress(self, fr, room, skip):
        """one LZ4F_decompress call on the whole input: frame_checksum_model's outcome dict (error name or None)"""
        lib = self.lib
        ctx = C.c_void_p()
        assert not lib.LZ4F_isError(lib.LZ4F_createDecompressionContext(C.byref(ctx), 100))
        src = np.frombuffer(bytes(fr) + b"\0", dtype=np.uint8)
        dst = np.zeros(max(room, 1), dtype=np.uint8)
        ssz, dsz = C.c_size_t(len(fr)), C.c_size_t(room)
        r = lib.LZ4F_decompress(ctx, dst.ctypes.data, C.byref(dsz), src.ctypes.data, C.byref(ssz),
                                C.byref(_DOpts(0, 1 if skip else 0, 0, 0)))
        lib.LZ4F_freeDecompressionContext(ctx)
        if lib.LZ4F_isError(r):
            return dict(error=lib.LZ4F_getErrorName(r).decode().replace("ERROR_", ""), size=None, out=b"")
        if r != 0:
            return dict(error="incomplete", size=None, out=b"")
        return dict(error=None, size=dsz.value, out=dst[:dsz.value].tobytes(), consumed=ssz.value)

    def legacy_block(self, blk, level):
        """the block `lz4 -l` writes for an 8 MiB chunk at `level` (lz4io.c's LZ4IO_compressLegacy): LZ4_compress_fast
        with acceleration -level below level 3 (0, read as 1, from level 0), LZ4_compress_HC from level 3"""
        src = np.frombuffer(bytes(blk) + b"\0", dtype=np.uint8)
        cap = LM.compress_bound(len(blk))
        dst = np.zeros(cap + 1, dtype=np.uint8)
        if level < 3:
            r = self.lib.LZ4_compress_fast(src.ctypes.data_as(C.POINTER(C.c_uint8)), dst.ctypes.data_as(
                C.POINTER(C.c_uint8)), len(blk), cap, -level if level < 0 else 0)
        else:
            r = self.lib.LZ4_compress_HC(src.ctypes.data, dst.ctypes.data, len(blk), cap, level)
        assert r > 0
        return dst[:r].tobytes()


def chain(fr):
    """the judge's own walk of a frame's chain (the frame format, lz4frame.c): [(offset, size, raw)] of its blocks when
    every block header, payload and checksum field lies inside fr up to the EndMark and the content checksum, else
    None"""
    bsum, csum = fr[4] & FM.FLG_BLOCK_SUM, fr[4] & FM.FLG_CONTENT_SUM
    bs = 1 << (8 + 2 * ((fr[5] >> 4) & 7))
    ip, blocks = FC.header_len(fr), []
    while ip + 4 <= len(fr):
        h = struct.unpack_from("<I", fr, ip)[0]
        ip += 4
        if h == 0:
            return blocks if ip + (4 if csum else 0) <= len(fr) else None
        sz = h & 0x7FFFFFFF
        if sz > bs or ip + sz + (4 if bsum else 0) > len(fr):
            return None
        blocks.append((ip, sz, h >> 31))
        ip += sz + (4 if bsum else 0)
    return None


def chain_blocks(fr):
    """the block headers a frame's chain holds before it ends or breaks, checksum fields stepped over"""
    if len(fr) < 7 or len(fr) < FC.header_len(fr):
        return 0
    ip, n = FC.header_len(fr), 0
    while ip + 4 <= len(fr):
        h = struct.unpack_from("<I", fr, ip)[0]
        if h == 0:
            break
        ip += 4 + (h & 0x7FFFFFFF) + (4 if fr[4] & FM.FLG_BLOCK_SUM else 0)
        n += 1
    return n


def room(fr):
    """the most a frame's chain can decode to"""
    if len(fr) < 6:
        return 16
    return (chain_blocks(fr) + 1) * (1 << (8 + 2 * max((fr[5] >> 4) & 7, 4)))


def _frame_header_verdict(fr, xxh32):
    """ERR_UNSUPPORTED for a frame whose header is valid and that has linked blocks or a dictID (the library's
    deviation from LZ4F_decompress, which decodes them), else None"""
    if len(fr) < 7 or struct.unpack_from("<I", fr, 0)[0] != FC.MAGIC:
        return None
    flg, bd = fr[4], fr[5]
    hl = FC.header_len(fr)
    if (flg >> 6) != 1 or flg & 2 or len(fr) < hl or bd & 0x8F or ((bd >> 4) & 7) < 4:
        return None
    if (xxh32(fr[4:hl - 1]) >> 8) & 0xFF != fr[hl - 1]:
        return None
    return ERR_UNSUPPORTED if (not flg & 0x20 or flg & 1) else None


# ------------------------------------------------------------------------------------------
# the judges
# ------------------------------------------------------------------------------------------
class Judge:
    """expected results of the container calls, from the reference (use_reference True, or None and the reference
    built) or from the models"""

    def __init__(self, oracle, use_reference=None):
        from oracle.pyoracle import Reference, have_reference
        self.oracle = oracle
        if use_reference is None:
            use_reference = have_reference()
        self.ref = _Ref(Reference()) if use_reference else None
        self.name = "reference" if self.ref else "model"

    # --- writers: (result, bytes) ---
    def write_frame(self, d, c, cap):
        """LZ4B200_compress_frames(_checksummed) on one source at parallel = 0"""
        if cap < 0:
            return ERR_ARG, b""
        if self.ref is not None:
            r = self.ref.r
            try:
                fr = r.compress_frame(d, c["bsid"], c["level"], c["cs"], 1, int(c["csum"]), int(c["bsum"]),
                                      capacity=cap)
            except RuntimeError:
                return ERR_DSTSIZE, b""
            return len(fr), fr
        if cap < CM.bound(len(d), c["bsid"], c["bsum"], c["csum"]):
            return ERR_DSTSIZE, b""
        fr = CM.frame(d, c["bsid"], c["cs"], CM.block_codec(self.oracle, c["level"]), block_sum=c["bsum"],
                      content_sum=c["csum"])
        return len(fr), fr

    def write_legacy(self, d, level, cap):
        """LZ4B200_compress_legacy on one source"""
        if cap < 0:
            return ERR_ARG, b""
        if self.ref is not None:
            need = 4 + sum(4 + LM.compress_bound(min(LM.CHUNK, len(d) - at)) for at in range(0, len(d), LM.CHUNK))
            if cap < need:
                return ERR_DSTSIZE, b""
            out = bytearray(struct.pack("<I", LM.MAGIC))
            for at in range(0, len(d), LM.CHUNK):
                blk = self.ref.legacy_block(d[at:at + LM.CHUNK], level)
                out += struct.pack("<I", len(blk)) + blk
            return len(out), bytes(out)
        if cap < LM.bound(len(d)):
            return ERR_DSTSIZE, b""
        st = LM.stream(d, LM.block_codec(self.oracle, level))
        return len(st), st

    def write(self, d, c, cap):
        return self.write_legacy(d, c["level"], cap) if c["legacy"] else self.write_frame(d, c, cap)

    # --- readers ---
    def read_frame(self, fr, cap, skip, content=True):
        """LZ4B200_decompress_frames_checksummed on one frame alone: (result, bytes).  content=False: the content
        checksum is not compared (the file calls' size-only pass).  With the reference, LZ4F_decompress decides every
        frame; the call's deviations from it are applied on top of its outcome, and a frame it decodes that the model's
        chain walk rejects is an AssertionError (the model is wrong)."""
        if self.ref is None:
            return FM.decode(self.oracle, fr, cap, skip)[:2] if content else \
                DM._frame_decode(self.oracle, fr, cap, skip, False)
        if len(fr) >= 4 and struct.unpack_from("<I", fr, 0)[0] & 0xFFFFFFF0 == DM.SKIPPABLE_MAGIC:
            return (ERR_UNSUPPORTED if len(fr) >= 7 else ERR_FRAME), b""      # a frame call takes no skippable frame
        un = _frame_header_verdict(fr, self.ref.xxh32)
        if un is not None:
            return un, b""
        o = self.ref.decompress(self.ref.skipped_block_sums(fr) if skip else fr, room(fr), skip)
        if not content and o["error"] == "contentChecksum_invalid":
            o = self.ref.decompress(fr, room(fr), True)
        rc = FM.ref_class(o)
        framed = len(fr) >= 7 and struct.unpack_from("<I", fr, 0)[0] == FC.MAGIC and len(fr) >= FC.header_len(fr)
        if rc >= 0:
            assert not framed or FM.walk(fr) is not None, "the model's chain walk rejects a frame LZ4F_decompress decodes"
            return (ERR_DSTSIZE, b"") if rc > cap else (rc, o["out"])
        if framed and chain(fr) is None:
            return ERR_FRAME, b""       # the call walks the whole chain before it decodes or hashes a block
        return rc, b""

    def read_files(self, files, caps, max_units, max_blocks, skip=False, size_only=False):
        """LZ4B200_decompress_files: [(result, consumed, prefix, bytes)].  The grammar, verdict order, consumed count and
        prefix are decompress_files_model's; with the reference, every frame unit the model's walk takes is checked
        against the reference judge first -- its result at unlimited room for a unit the model accepts, its verdict for
        a unit the model rejects (AssertionError: the model is wrong)."""
        if self.ref is not None:
            for f in files:
                f = bytes(f)
                for u in DM.walk_file(f, 1 << 40, [1 << 40] * DM.CLASSES, skip):
                    if u["kind"] != "frame":
                        continue
                    if u["status"] == DM.OK:
                        fr = f[u["off"]:u["off"] + u["length"]]
                        m = DM._frame_decode(self.oracle, fr, DM.INF, skip, not size_only)
                        want = self.read_frame(fr, DM.INF, skip, not size_only)
                        assert m == want, ("model and reference disagree on a frame unit", m[0], want[0])
                    else:
                        want = self.read_frame(f[u["off"]:], DM.INF, skip, not size_only)
                        assert want[0] == u["status"], ("the model rejects a frame unit the reference judges",
                                                        u["status"], want[0])
        return DM.decompress_files(self.oracle, files, caps, max_units, max_blocks, skip, size_only,
                                   content=not size_only)


# ------------------------------------------------------------------------------------------
# the run digests of tests/golden/container_fuzz.json
# ------------------------------------------------------------------------------------------
DIGEST_SEEDS = [1, 2, 2026]
DIGEST_CASES = 16
DIGEST_CHUNK = 4
SMALL = 2 * MIB                 # the CPU checks draw the cases of at most this many source bytes


def small_cases(seed, n, max_total=SMALL):
    """the first n cases (k, case) of seed with at most max_total source bytes (8 x max_total for legacy streams, whose
    judges hash nothing in Python)"""
    k = 0
    while n:
        c = case(seed, k)
        if sum(it["size"] for it in c["items"]) <= max_total * (8 if c["legacy"] else 1):
            yield k, c
            n -= 1
        k += 1


def digest_run(judge, seed, n_cases=DIGEST_CASES, chunk=DIGEST_CHUNK):
    """the SHA-256 digests of seed's first n_cases small cases, one per chunk of cases, over every (result, consumed,
    bytes) run_case judges"""
    out, h = [], hashlib.sha256()
    for j, (k, c) in enumerate(small_cases(seed, n_cases)):
        for tag, r, b in run_case(judge, seed, k, c):
            h.update(repr((tag, r)).encode() + sha(b).encode())
        if j % chunk == chunk - 1:
            out.append(h.hexdigest())
            h = hashlib.sha256()
    return out


def written(judge, c, datas):
    """the items of case c as written at their bound: [bytes]"""
    return [judge.write(d, c, bound(c, len(d)))[1] for d in datas]


def run_case(judge, seed, k, c, datas=None):
    """every judged record of case k: (call, result, bytes) with call a tag"""
    datas = case_data(judge.oracle, c) if datas is None else datas
    recs = []
    for i, (d, it) in enumerate(zip(datas, c["items"])):
        r, b = judge.write(d, c, capacity(c, it, seed * 1000003 + k * 1009 + i))
        recs.append((("w", i), r, b))
    files = written(judge, c, datas)
    rng = np.random.default_rng([seed, k, 7])
    muts = mutated_files(judge.oracle, c, files, rng)
    if not c["legacy"]:
        for i, (cls, f) in enumerate(muts):
            for skip in (False, True):
                r, b = judge.read_frame(f, 1 << 40, skip)
                recs.append((("r", i, cls, skip), r, b))
    mu, mb = DM.budget_needed([f for _, f in muts])
    for skip in (False, True):
        for i, (r, con, pre, b) in enumerate(judge.read_files([f for _, f in muts], [1 << 40] * len(muts), mu, mb,
                                                              skip)):
            recs.append((("f", i, skip, con, pre), r, b))
    return recs


def mutated_files(oracle, c, files, rng):
    """(class, file) per written item: a valid file ("none") or one of the mutations; legacy streams are cut, padded
    with garbage or wrapped only"""
    out = []
    for i, f in enumerate(files):
        if rng.random() < 0.3:
            out.append(("none", f))
        elif c["legacy"]:
            cls = str(rng.choice(["cut", "garbage", "wrap_legacy"]))
            if cls == "cut":
                out.append((cls, f[:int(rng.integers(0, len(f)))]))
            elif cls == "garbage":
                out.append((cls, f + rng.integers(0, 256, int(rng.integers(1, 12)), dtype=np.uint8).tobytes()))
            else:
                out.append((cls, DM.skippable(b"x" * int(rng.integers(0, 9))) + f))
        else:
            out.append(mutate(f, rng, other=files[(i + 1) % len(files)], oracle=oracle))
    return out
