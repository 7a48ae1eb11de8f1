/*
 * lz4_frame_core.h -- the rules of an LZ4 frame of independent blocks, in one place: XXH32, the header checks and the
 * header checksum (LZ4F_decodeHeader, lz4frame.c:1340-1425), the chain of block headers with its checksum fields
 * (lz4frame.c:1729-1758) and the verdict on the decoded blocks and their checksums.  LZ4B200_decompressFrame_host (lz4_api.c, compiled as C99) and the batched frame decode
 * (lz4_kernels.cu, CUDA) both decide with these functions; tests/emul/frame_emul.cpp runs the batched call's index passes
 * on the host from the same text.  The writing side -- optimal block size ID, bound, header bytes and the index passes of
 * the batched frame encode -- serves LZ4B200_compressFrame_host and LZ4B200_compress_frames the same way
 * (tests/emul/compress_frames_emul.cpp).  The file layer of LZ4B200_decompress_files -- the units of a .lz4 file, their
 * placement and the fold of their results -- sits on the frame decode's rules (tests/emul/decompress_files_emul.cpp).
 * The legacy stream's writing rules serve LZ4B200_compress_legacy through the frame encode's passes
 * (tests/emul/compress_legacy_emul.cpp).  No CUDA runtime calls, no allocation.
 */
#ifndef LZ4_FRAME_CORE_H
#define LZ4_FRAME_CORE_H

#include <stddef.h>
#include <stdint.h>
#include "../../include/lz4_b200.h"

#if defined(__CUDACC__)
#define FC_FN static __host__ __device__ __forceinline__
#else
#define FC_FN static inline
#endif

#define FC_MAGIC           0x184D2204u     /* lz4frame.c: LZ4F_MAGICNUMBER */
#define FC_MAGIC_SKIPPABLE 0x184D2A50u     /* .. LZ4F_MAGIC_SKIPPABLE_START */
#define FC_MAGIC_LEGACY    0x184C2102u     /* lz4io.c: LEGACY_MAGICNUMBER, the `lz4 -l` format */

FC_FN uint32_t fc_rd_le32(const uint8_t* p)
{
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

FC_FN uint32_t fc_rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

/* XXH32, as published in the xxHash specification (https://github.com/Cyan4973/xxHash/blob/dev/doc/xxhash_spec.md): the
 * frame header checksum is the second byte of XXH32(descriptor, 0) (lz4frame.c:781-809), a block checksum XXH32(payload,
 * 0) and the content checksum XXH32(content, 0).  The kernels of the checksummed frame decode read their stripes their own
 * way and share the round, the merge and the end with fc_xxh32. */
#define FC_XXH_P1 2654435761u
#define FC_XXH_P2 2246822519u
#define FC_XXH_P3 3266489917u
#define FC_XXH_P4 668265263u
#define FC_XXH_P5 374761393u

FC_FN uint32_t fc_xxh32_round(uint32_t acc, uint32_t lane) { return fc_rotl32(acc + lane * FC_XXH_P2, 13) * FC_XXH_P1; }

/* the four accumulators after the last stripe, folded into one */
FC_FN uint32_t fc_xxh32_merge(uint32_t v1, uint32_t v2, uint32_t v3, uint32_t v4)
{
    return fc_rotl32(v1, 1) + fc_rotl32(v2, 7) + fc_rotl32(v3, 12) + fc_rotl32(v4, 18);
}

/* the end of a message of len bytes: h (the merged accumulators, or seed + P5 below 16 bytes), the len & 15 bytes after
 * the last stripe at p, the avalanche */
FC_FN uint32_t fc_xxh32_end(uint32_t h, const uint8_t* p, uint64_t len)
{
    const uint8_t* end = p + (len & 15);
    h += (uint32_t)len;
    while (p + 4 <= end) { h += fc_rd_le32(p) * FC_XXH_P3; h = fc_rotl32(h, 17) * FC_XXH_P4; p += 4; }
    while (p < end) { h += (uint32_t)(*p) * FC_XXH_P5; h = fc_rotl32(h, 11) * FC_XXH_P1; p++; }
    h ^= h >> 15; h *= FC_XXH_P2; h ^= h >> 13; h *= FC_XXH_P3; h ^= h >> 16;
    return h;
}

FC_FN uint32_t fc_xxh32(const uint8_t* p, uint64_t len, uint32_t seed)
{
    uint32_t h = seed + FC_XXH_P5;
    if (len >= 16) {
        uint32_t v1 = seed + FC_XXH_P1 + FC_XXH_P2, v2 = seed + FC_XXH_P2, v3 = seed, v4 = seed - FC_XXH_P1;
        const uint8_t* limit = p + (len & ~(uint64_t)15);
        for (; p < limit; p += 16) {
            v1 = fc_xxh32_round(v1, fc_rd_le32(p));      v2 = fc_xxh32_round(v2, fc_rd_le32(p + 4));
            v3 = fc_xxh32_round(v3, fc_rd_le32(p + 8));  v4 = fc_xxh32_round(v4, fc_rd_le32(p + 12));
        }
        h = fc_xxh32_merge(v1, v2, v3, v4);
    }
    return fc_xxh32_end(h, p, len);
}

/* XXH32 with seed 0 over a message that arrives in pieces (LZ4B200_decompress_files_host: a frame's content spans the
 * groups of its blocks): the four accumulators, the bytes taken so far and the 0 .. 15 bytes after the last full
 * stripe.  fc_xxh32_digest after any split of the message into fc_xxh32_update calls equals fc_xxh32(message, 0). */
typedef struct {
    uint32_t v[4];
    uint32_t tailLen;          /* bytes in tail: total & 15 */
    uint64_t total;
    uint8_t tail[16];
} fc_xxh32_state;

FC_FN void fc_xxh32_init(fc_xxh32_state* s)
{
    s->v[0] = FC_XXH_P1 + FC_XXH_P2; s->v[1] = FC_XXH_P2; s->v[2] = 0; s->v[3] = 0u - FC_XXH_P1;
    s->tailLen = 0; s->total = 0;
}

FC_FN void fc_xxh32_stripe(uint32_t v[4], const uint8_t* p)
{
    v[0] = fc_xxh32_round(v[0], fc_rd_le32(p));      v[1] = fc_xxh32_round(v[1], fc_rd_le32(p + 4));
    v[2] = fc_xxh32_round(v[2], fc_rd_le32(p + 8));  v[3] = fc_xxh32_round(v[3], fc_rd_le32(p + 12));
}

FC_FN void fc_xxh32_update(fc_xxh32_state* s, const uint8_t* p, uint64_t len)
{
    const uint8_t* end = p + len;
    s->total += len;
    if (s->tailLen) {                                                      /* complete the stripe the tail began */
        while (s->tailLen < 16 && p < end) s->tail[s->tailLen++] = *p++;
        if (s->tailLen < 16) return;
        fc_xxh32_stripe(s->v, s->tail);
        s->tailLen = 0;
    }
    for (; end - p >= 16; p += 16) fc_xxh32_stripe(s->v, p);
    while (p < end) s->tail[s->tailLen++] = *p++;
}

FC_FN uint32_t fc_xxh32_digest(const fc_xxh32_state* s)
{
    const uint32_t h = s->total >= 16 ? fc_xxh32_merge(s->v[0], s->v[1], s->v[2], s->v[3]) : FC_XXH_P5;
    return fc_xxh32_end(h, s->tail, s->total);
}

FC_FN int64_t fc_block_bytes(int bsid) { return (int64_t)1 << (8 + 2 * bsid); }   /* 4..7 -> 64 KB..4 MB (lz4frame.c:333-342) */

/* The block classes of the batched decode and encode: 0 .. 3 hold frame blocks of block size ID 4 + c, class 4 the blocks
 * of a legacy stream (LZ4B200_decompress_files and LZ4B200_compress_legacy; the frames calls give it a budget of 0). */
#define FC_CLASSES      5
#define FC_LEGACY_CLASS 4
#define FC_LEGACY_BLOCK (8 << 20)          /* lz4io.c: LEGACY_BLOCKSIZE, the capacity a legacy block decodes with and
                                              the chunk the tool compresses */
#define FC_LEGACY_BOUND 8421520            /* LZ4_COMPRESSBOUND(8 MiB): a larger block word ends a legacy unit */

/* the uniform capacity the blocks of class cls decode with */
FC_FN int64_t fc_class_bytes(int cls) { return cls == FC_LEGACY_CLASS ? FC_LEGACY_BLOCK : fc_block_bytes(4 + cls); }

/* ---------------------------------------------------------------------------------------------
 * Writing a frame of independent blocks (LZ4F_compressFrame, lz4frame.c:425-498): LZ4B200_compressFrame_host (no
 * checksums) and the batched LZ4B200_compress_frames and LZ4B200_compress_frames_checksummed take these rules from here.
 * ------------------------------------------------------------------------------------------- */
#define FC_BLOCK_SUM   1           /* FLG bit 4: 4 bytes of XXH32(payload) after every block */
#define FC_CONTENT_SUM 2           /* FLG bit 2: 4 bytes of XXH32(content) after the EndMark */

/* LZ4F_optimalBSID (lz4frame.c:362-373): the smallest block size ID from 4 up to `requested` (4 .. 7) whose blocks hold
 * srcSize bytes */
FC_FN int fc_optimal_bsid(int requested, int64_t srcSize)
{
    int proposed = 4;
    int64_t maxBlock = 64 * 1024;
    while (requested > proposed) {
        if (srcSize <= maxBlock) return proposed;
        proposed++;
        maxBlock <<= 2;
    }
    return requested;
}

/* blocks of a frame of srcSize >= 0 bytes at block size ID bsid: the full ones and a last partial one */
FC_FN int64_t fc_frame_blocks(int64_t srcSize, int bsid)
{
    const int64_t bs = fc_block_bytes(bsid);
    return srcSize / bs + (srcSize % bs != 0);
}

/* LZ4F_compressFrameBound (lz4frame.c:406-417 with LZ4F_compressBound_internal, lz4frame.c:376-403) for autoFlush and
 * independent blocks, at the block size ID the frame is written with, for a frame carrying the checksums `sums`
 * (FC_BLOCK_SUM | FC_CONTENT_SUM): the largest header (19 bytes), a 4-byte header and, with block checksums, a
 * 4-byte checksum per block, the source, the EndMark and, with a content checksum, its 4 bytes.  Saturates at
 * INT64_MAX. */
FC_FN int64_t fc_frame_bound_sums(int64_t srcSize, int bsid, int sums)
{
    const int64_t extra = 19 + (4 + ((sums & FC_BLOCK_SUM) ? 4 : 0)) * fc_frame_blocks(srcSize, bsid) + 4 +
                          ((sums & FC_CONTENT_SUM) ? 4 : 0);
    return srcSize > INT64_MAX - extra ? INT64_MAX : srcSize + extra;
}

/* the same without checksums */
FC_FN int64_t fc_frame_bound(int64_t srcSize, int bsid) { return fc_frame_bound_sums(srcSize, bsid, 0); }

/* The frame header (LZ4F_compressBegin, lz4frame.c:781-809) into h[0 .. 15): magic, FLG (version 01, independent
 * blocks, the block checksum bit 4, the content-size bit 3, the content checksum bit 2), BD, the content size when
 * contentSize > 0 (an empty frame has none, lz4frame.c:445-446), and the header checksum byte.  sums: FC_BLOCK_SUM |
 * FC_CONTENT_SUM.  Returns its length, 7 or 15. */
FC_FN int fc_frame_header_sums(uint8_t* h, int bsid, int64_t contentSize, int sums)
{
    int n = 6, i;
    const int withSize = contentSize > 0;
    h[0] = (uint8_t)FC_MAGIC; h[1] = (uint8_t)(FC_MAGIC >> 8); h[2] = (uint8_t)(FC_MAGIC >> 16); h[3] = (uint8_t)(FC_MAGIC >> 24);
    h[4] = (uint8_t)((1u << 6) | (1u << 5) | (((sums & FC_BLOCK_SUM) ? 1u : 0u) << 4) | ((withSize ? 1u : 0u) << 3) |
                     (((sums & FC_CONTENT_SUM) ? 1u : 0u) << 2));
    h[5] = (uint8_t)((uint32_t)bsid << 4);
    if (withSize) for (i = 0; i < 8; i++) h[n++] = (uint8_t)((uint64_t)contentSize >> (8 * i));
    h[n] = (uint8_t)(fc_xxh32(h + 4, (uint64_t)(n - 4), 0) >> 8);
    return n + 1;
}

/* the same without checksums */
FC_FN int fc_frame_header_bytes(uint8_t* h, int bsid, int64_t contentSize) { return fc_frame_header_sums(h, bsid, contentSize, 0); }

typedef struct {
    int64_t contentSize;       /* the header's content size, -1 without one; a field of 2^63 or more reads INT64_MAX, a
                                  size no frame here decodes to, so the frame fails as lz4frame.c's frameSize_wrong */
    int32_t hdrLen;            /* bytes of the header: the first block header starts here */
    int32_t bsid;              /* block size ID, 4 .. 7 */
    int32_t sums;              /* the checksums the frame carries: FC_BLOCK_SUM | FC_CONTENT_SUM */
} fc_header_t;

/* what the header rules do with FLG's checksum bits: reject them (LZ4B200_ERR_UNSUPPORTED; the host call and
 * LZ4B200_decompress_frames), or accept them and skip or verify the checksums (LZ4B200_decompress_frames_checksummed) */
#define FC_SUMS_REJECT 0
#define FC_SUMS_SKIP   1
#define FC_SUMS_VERIFY 2

#define FC_VERIFY      4           /* (fc_frame_rec.sums) the call compares them */

/* The verdict on a frame's arguments and header, in the order LZ4B200_decompressFrame_host decides them: LZ4B200_OK (h
 * filled in), LZ4B200_ERR_ARG (srcSize or dstCap negative), LZ4B200_ERR_FRAME (malformed header) or
 * LZ4B200_ERR_UNSUPPORTED (skippable frame, linked blocks, checksums under FC_SUMS_REJECT, dictID).  The header checksum
 * is checked in every mode (lz4frame.c:1418).  Reads src[0, min(srcSize, 19)). */
FC_FN int fc_frame_header(const uint8_t* src, int64_t srcSize, int64_t dstCap, int mode, fc_header_t* h)
{
    uint32_t flg, bd, hdrLen, magic;
    int bsid, i;
    if (srcSize < 0 || dstCap < 0) return LZ4B200_ERR_ARG;
    if (srcSize < 7) return LZ4B200_ERR_FRAME;                                        /* minFHSize, lz4frame.h:280 */
    magic = fc_rd_le32(src);
    if ((magic & 0xFFFFFFF0u) == FC_MAGIC_SKIPPABLE) return LZ4B200_ERR_UNSUPPORTED;
    if (magic != FC_MAGIC) return LZ4B200_ERR_FRAME;
    flg = src[4];
    if (((flg >> 6) & 3) != 1 || ((flg >> 1) & 1)) return LZ4B200_ERR_FRAME;          /* version, reserved bit */
    hdrLen = 7 + (((flg >> 3) & 1) ? 8 : 0) + ((flg & 1) ? 4 : 0);
    if (srcSize < (int64_t)hdrLen) return LZ4B200_ERR_FRAME;
    bd = src[5];
    bsid = (int)((bd >> 4) & 7);
    if ((bd >> 7) || (bd & 15) || bsid < 4) return LZ4B200_ERR_FRAME;                 /* lz4frame.c:1406-1412 */
    if ((uint8_t)(fc_xxh32(src + 4, hdrLen - 5, 0) >> 8) != src[hdrLen - 1]) return LZ4B200_ERR_FRAME;
    if (!((flg >> 5) & 1)) return LZ4B200_ERR_UNSUPPORTED;                            /* linked blocks */
    if (flg & 1) return LZ4B200_ERR_UNSUPPORTED;                                      /* dictID */
    h->sums = (((flg >> 4) & 1) ? FC_BLOCK_SUM : 0) | (((flg >> 2) & 1) ? FC_CONTENT_SUM : 0);
    if (h->sums && mode == FC_SUMS_REJECT) return LZ4B200_ERR_UNSUPPORTED;
    h->contentSize = -1;
    if ((flg >> 3) & 1) {
        uint64_t v = 0;
        for (i = 0; i < 8; i++) v |= (uint64_t)src[6 + i] << (8 * i);
        h->contentSize = v > (uint64_t)INT64_MAX ? INT64_MAX : (int64_t)v;
    }
    h->hdrLen = (int32_t)hdrLen;
    h->bsid = bsid;
    return LZ4B200_OK;
}

/* One step of the chain of block headers (lz4frame.c:1729-1758) from the block header at *ip, for blocks of at most bs
 * bytes in a frame carrying the checksums `sums`.  Returns 1 for a block (*at: its first byte, *size, *raw: stored raw;
 * *ip moves past it and its checksum), 0 at the EndMark (*ip moves past it and the content checksum: the frame's
 * length), LZ4B200_ERR_FRAME for a truncated chain -- a checksum field is part of the chain (lz4frame.c:1731, 1751) -- or
 * a block above bs (maxBlockSize_invalid, lz4frame.c:1745). */
FC_FN int fc_next_block(const uint8_t* src, int64_t srcSize, int64_t bs, int sums, int64_t* ip, int64_t* at, int64_t* size,
                        int* raw)
{
    const int64_t cs = (sums & FC_BLOCK_SUM) ? 4 : 0;
    uint32_t h;
    int64_t sz;
    if (*ip + 4 > srcSize) return LZ4B200_ERR_FRAME;
    h = fc_rd_le32(src + *ip);
    *ip += 4;
    if (h == 0) {                                                                     /* EndMark */
        if ((sums & FC_CONTENT_SUM) && *ip + 4 > srcSize) return LZ4B200_ERR_FRAME;
        if (sums & FC_CONTENT_SUM) *ip += 4;
        return 0;
    }
    sz = (int64_t)(h & 0x7FFFFFFFu);
    if (sz > bs || *ip + sz + cs > srcSize) return LZ4B200_ERR_FRAME;
    *at = *ip; *size = sz; *raw = (int)(h >> 31);
    *ip += sz + cs;
    return 1;
}

/* One step of a legacy unit's chain (LZ4IO_decodeLegacyStream, lz4io.c:1836-1883) from the block word at *ip: 0 when the
 * unit ends -- no bytes left, or a word above FC_LEGACY_BOUND, which is the next unit's magic (*ip stays on it) -- 1 for
 * a block of that many compressed bytes (*at, *size; *ip moves past it), LZ4B200_ERR_FRAME for 1 .. 3 bytes left or a
 * block cut short.  A block of 0 bytes is a block: its decode fails. */
FC_FN int fc_next_legacy_block(const uint8_t* src, int64_t srcSize, int64_t* ip, int64_t* at, int64_t* size)
{
    uint32_t w;
    if (*ip == srcSize) return 0;
    if (*ip + 4 > srcSize) return LZ4B200_ERR_FRAME;
    w = fc_rd_le32(src + *ip);
    if (w > FC_LEGACY_BOUND) return 0;
    if (*ip + 4 + (int64_t)w > srcSize) return LZ4B200_ERR_FRAME;
    *at = *ip + 4; *size = (int64_t)w;
    *ip += 4 + (int64_t)w;
    return 1;
}

/* the chain step of a block of class cls: a frame's (fc_next_block) or a legacy unit's, whose blocks are never raw */
FC_FN int fc_next_class_block(const uint8_t* src, int64_t srcSize, int cls, int sums, int64_t* ip, int64_t* at,
                              int64_t* size, int* raw)
{
    if (cls == FC_LEGACY_CLASS) { *raw = 0; return fc_next_legacy_block(src, srcSize, ip, at, size); }
    return fc_next_block(src, srcSize, fc_block_bytes(4 + cls), sums, ip, at, size, raw);
}

/* The verdict on one decoded block: r = its decoded size (a stored-raw block's size; negative: it failed to decode),
 * written at pos of a frame with dstCap bytes of room.  Decode failure, then the room, then the content size. */
FC_FN int fc_block_verdict(int64_t pos, int64_t r, int64_t dstCap, int64_t contentSize)
{
    if (r < 0) return LZ4B200_ERR_FRAME;
    if (pos + r > dstCap) return LZ4B200_ERR_DSTSIZE;
    if (contentSize >= 0 && pos + r > contentSize) return LZ4B200_ERR_FRAME;
    return LZ4B200_OK;
}

/* The same with the outcome of the block's checksum (sumBad: it does not match), where LZ4F_decompress judges it: a
 * compressed block's before its decode (lz4frame.c:1871-1883), a stored-raw block's after its bytes are placed
 * (lz4frame.c:1803-1830), so after the room and the content size. */
FC_FN int fc_block_sum_verdict(int64_t pos, int64_t r, int64_t dstCap, int64_t contentSize, int raw, int sumBad)
{
    int v;
    if (sumBad && !raw) return LZ4B200_ERR_CHECKSUM;
    v = fc_block_verdict(pos, r, dstCap, contentSize);
    return (v == LZ4B200_OK && sumBad) ? LZ4B200_ERR_CHECKSUM : v;
}

/* a frame whose every block passed: its result, total decoded bytes, or LZ4B200_ERR_FRAME when the content size differs
 * (frameSize_wrong, lz4frame.c:1984; the content checksum is judged after it, by the caller) */
FC_FN int64_t fc_frame_result(int64_t total, int64_t contentSize)
{
    return (contentSize >= 0 && contentSize != total) ? (int64_t)LZ4B200_ERR_FRAME : total;
}

/* ---------------------------------------------------------------------------------------------
 * The batched frame decode (LZ4B200_decompress_frames and LZ4B200_decompress_frames_checksummed): one record per frame,
 * one table of blocks per class (block size ID 4 + c), and the three steps that run one frame per thread.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
    int64_t count;             /* blocks the chain walk saw (at most maxBlocks[cls] + 1) */
    int64_t base;              /* the frame's first entry in its class's table */
    int64_t contentSize;       /* as fc_header_t */
    int64_t consumed;          /* the frame's length once its chain is walked to the EndMark, else 0 */
    int32_t status;            /* LZ4B200_OK or the frame's error code so far */
    int32_t cls;               /* block size ID - 4 (-1 before the header passed, and for a skippable frame);
                                  FC_LEGACY_CLASS for a legacy unit of LZ4B200_decompress_files */
    int32_t hdrLen;
    int32_t sums;              /* fc_header_t.sums, | FC_VERIFY when the call compares them */
} fc_frame_rec;

typedef struct {               /* a class's block table; entry b of every array belongs to one block */
    int64_t* srcOff;           /* absolute offset of the block's bytes in the call's source */
    int64_t* dstOff;           /* absolute offset of its decoded bytes in the call's destination (set by the verdict);
                                  before the verdict, under FC_VERIFY, the block checksum's state: FC_SUM_* */
    int32_t* srcSize;          /* bytes the decode gets: 0 for a stored-raw block, so that the scan rejects it */
    int32_t* outSize;          /* the decode's return value; -1 once the verdict has failed the block's frame */
    int32_t* rawLen;           /* a stored-raw block's size, -1 for a compressed block */
} fc_block_tab;

/* the block checksum's state in a table entry's dstOff before the verdict (FC_VERIFY only; the table is cleared to
 * FC_SUM_NONE first) */
#define FC_SUM_NONE    0           /* no checksum to compare, or it matches */
#define FC_SUM_PENDING 1           /* the fill found one; the block checksum kernel compares it */
#define FC_SUM_BAD     2           /* it does not match */

/* The chain walk of pass 1 from the end of r's header (r->cls, hdrLen and sums set), which stops after maxBlocks[cls] + 1
 * blocks (the frame is over its budget whatever follows): r->count, and r->consumed once the chain ends. */
FC_FN void fc_walk_chain(const uint8_t* src, int64_t srcSize, const int64_t* maxBlocks, fc_frame_rec* r)
{
    int64_t ip = r->hdrLen, at, sz, n = 0;
    int raw, s;
    while ((s = fc_next_class_block(src, srcSize, r->cls, r->sums, &ip, &at, &sz, &raw)) == 1)
        if (++n > maxBlocks[r->cls]) break;
    if (s < 0) { r->status = s; return; }
    r->count = n;
    if (s == 0) r->consumed = ip;
}

FC_FN void fc_clear_rec(fc_frame_rec* r)
{
    r->count = 0; r->base = 0; r->contentSize = -1; r->consumed = 0; r->cls = -1; r->hdrLen = 0; r->sums = 0;
    r->status = LZ4B200_OK;
}

/* Pass 1 (the index): the header rules under `mode` (FC_SUMS_*), then the chain walk.  src: the frame's first byte. */
FC_FN void fc_index_frame_mode(const uint8_t* src, int64_t srcSize, int64_t dstCap, const int64_t* maxBlocks, int mode,
                               fc_frame_rec* r)
{
    fc_header_t h;
    fc_clear_rec(r);
    r->status = fc_frame_header(src, srcSize, dstCap, mode, &h);
    if (r->status != LZ4B200_OK) return;
    r->cls = h.bsid - 4; r->contentSize = h.contentSize; r->hdrLen = h.hdrLen;
    r->sums = h.sums | ((h.sums && mode == FC_SUMS_VERIFY) ? FC_VERIFY : 0);
    fc_walk_chain(src, srcSize, maxBlocks, r);
}

/* pass 1 of LZ4B200_decompress_frames, which rejects checksums */
FC_FN void fc_index_frame(const uint8_t* src, int64_t srcSize, int64_t dstCap, const int64_t* maxBlocks, fc_frame_rec* r)
{
    fc_index_frame_mode(src, srcSize, dstCap, maxBlocks, FC_SUMS_REJECT, r);
}

/* the blocks frame r puts into its class's exclusive scan (a frame that failed pass 1 puts none) */
FC_FN int64_t fc_scan_count(const fc_frame_rec* r) { return r->status == LZ4B200_OK ? r->count : 0; }

/* After the scan: base = the blocks of the earlier frames of r's class that passed pass 1.  The frame gets
 * LZ4B200_ERR_LIMIT when those and its own exceed its class's budget. */
FC_FN void fc_place_frame(fc_frame_rec* r, int64_t base, const int64_t* maxBlocks)
{
    r->base = base;
    if (r->status == LZ4B200_OK && base + r->count > maxBlocks[r->cls]) { r->status = LZ4B200_ERR_LIMIT; r->consumed = 0; }
}

/* Pass 2 (the fill): walks the chain again and writes the frame's entries of its class's table, and marks the block
 * checksums to compare.  srcOff: the frame's offset in the call's source. */
FC_FN void fc_fill_frame(const uint8_t* src, int64_t srcOff, int64_t srcSize, const fc_frame_rec* r, fc_block_tab t)
{
    int64_t ip = r->hdrLen, at, sz, b = r->base;
    int raw;
    if (r->status != LZ4B200_OK || r->cls < 0) return;
    const int mark = (r->sums & FC_VERIFY) && (r->sums & FC_BLOCK_SUM);
    while (fc_next_class_block(src, srcSize, r->cls, r->sums, &ip, &at, &sz, &raw) == 1) {
        t.srcOff[b] = srcOff + at;
        t.srcSize[b] = raw ? 0 : (int32_t)sz;
        t.rawLen[b] = raw ? (int32_t)sz : -1;
        if (mark) t.dstOff[b] = FC_SUM_PENDING;
        b++;
    }
}

/* The verdict, between the scan and the expand: the block rules in block order on the scanned and the raw sizes and the
 * block checksums' outcomes, each block's tight offset (dstOff: the frame's), the frame's result and consumed length.
 * Every block of a frame that fails gets outSize -1 and rawLen -1, so that neither the expand nor the raw copy writes any
 * of its bytes.  The content checksum of a frame that passes is judged after its bytes are in place. */
FC_FN void fc_verdict_frame(const fc_frame_rec* r, int64_t dstOff, int64_t dstCap, fc_block_tab t, int64_t* result,
                            int64_t* consumed)
{
    int64_t pos = 0, res, k;
    int v = LZ4B200_OK;
    const int verifyBlocks = (r->sums & FC_VERIFY) && (r->sums & FC_BLOCK_SUM);
    if (consumed) *consumed = r->consumed;
    if (r->status != LZ4B200_OK) { *result = r->status; return; }
    for (k = 0; k < r->count && v == LZ4B200_OK; k++) {
        const int64_t b = r->base + k;
        const int64_t rb = t.rawLen[b] >= 0 ? t.rawLen[b] : t.outSize[b];
        v = fc_block_sum_verdict(pos, rb, dstCap, r->contentSize, t.rawLen[b] >= 0, verifyBlocks && t.dstOff[b] == FC_SUM_BAD);
        t.dstOff[b] = dstOff + pos;
        pos += rb;
    }
    res = v != LZ4B200_OK ? (int64_t)v : fc_frame_result(pos, r->contentSize);
    if (res < 0)
        for (k = 0; k < r->count; k++) { t.outSize[r->base + k] = -1; t.rawLen[r->base + k] = -1; }
    *result = res;
}

/* ---------------------------------------------------------------------------------------------
 * The batched file decode (LZ4B200_decompress_files): a .lz4 file is a sequence of units -- LZ4 frames, skippable frames
 * and legacy streams -- read as `lz4 -d` reads its standard input (selectDecoder, lz4io.c:2349-2405).  Every unit gets a
 * fc_frame_rec and runs through the frame decode's steps as a frame of its own; the steps below give the units their
 * records, their places in their file's output, and fold their results into one per file.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
    int64_t units;             /* units the walk took (at most maxUnits + 1), the one that failed pass 1 included */
    int64_t base;              /* the index of the file's first unit in the call's unit order (files, then units) */
    int64_t overOff;           /* the offset of the file's first unit at index maxUnits or above (set by the fill) */
    int32_t status;            /* LZ4B200_ERR_ARG (a negative size or room), else the pass-1 status of the last unit */
    int32_t pad;
} fc_file_rec;

/* Pass 1 of the unit at src, rem >= 1 bytes before the file's end: the record fc_index_frame_mode gives an LZ4 frame
 * (consumed 0: its chain was cut short by the budget), a record of no blocks for a skippable frame, a legacy unit of
 * class FC_LEGACY_CLASS walked as a chain, or LZ4B200_ERR_FRAME for fewer than 4 bytes, a skippable frame that runs
 * past the end (lz4io.c:2384-2391 on a pipe) and any other magic. */
FC_FN void fc_next_unit(const uint8_t* src, int64_t rem, const int64_t* maxBlocks, int mode, fc_frame_rec* r)
{
    uint32_t magic;
    fc_clear_rec(r);
    r->status = LZ4B200_ERR_FRAME;
    if (rem < 4) return;
    magic = fc_rd_le32(src);
    if (magic == FC_MAGIC) { fc_index_frame_mode(src, rem, 0, maxBlocks, mode, r); return; }
    if ((magic & 0xFFFFFFF0u) == FC_MAGIC_SKIPPABLE) {
        if (rem < 8 || 8 + (int64_t)fc_rd_le32(src + 4) > rem) return;
        r->status = LZ4B200_OK;
        r->consumed = 8 + (int64_t)fc_rd_le32(src + 4);
        return;
    }
    if (magic != FC_MAGIC_LEGACY) return;
    r->status = LZ4B200_OK;
    r->cls = FC_LEGACY_CLASS;
    r->hdrLen = 4;
    fc_walk_chain(src, rem, maxBlocks, r);
}

/* The walk of one file (srcSize bytes, dstCap of room; dstCap 0 when the call only sizes): unit after unit until the
 * end, a unit that fails pass 1 or stops short on its budget, or maxUnits + 1 units -- the file is then over the unit
 * budget whatever follows. */
FC_FN void fc_index_file(const uint8_t* src, int64_t srcSize, int64_t dstCap, int64_t maxUnits, const int64_t* maxBlocks,
                         int mode, fc_file_rec* f)
{
    fc_frame_rec r;
    int64_t p = 0;
    f->units = 0; f->base = 0; f->overOff = 0; f->status = LZ4B200_OK; f->pad = 0;
    if (srcSize < 0 || dstCap < 0) { f->status = LZ4B200_ERR_ARG; return; }
    while (p < srcSize && f->units <= maxUnits) {
        fc_next_unit(src + p, srcSize - p, maxBlocks, mode, &r);
        f->units++;
        if (r.status != LZ4B200_OK || r.consumed == 0) { f->status = r.status; return; }
        p += r.consumed;
    }
}

/* After the scan of the unit counts (f->base): the walk again, writing the record, absolute source offset and length
 * (the rest of the file for a unit whose end pass 1 did not reach) of every unit below index maxUnits. */
FC_FN void fc_fill_file(const uint8_t* src, int64_t srcOff, int64_t srcSize, int64_t maxUnits, const int64_t* maxBlocks,
                        int mode, fc_file_rec* f, fc_frame_rec* units, int64_t* uSrcOff, int64_t* uSrcSize)
{
    int64_t p = 0, k;
    for (k = 0; k < f->units; k++) {
        const int64_t u = f->base + k;
        if (u >= maxUnits) { f->overOff = p; return; }
        fc_next_unit(src + p, srcSize - p, maxBlocks, mode, &units[u]);
        uSrcOff[u] = srcOff + p;
        uSrcSize[u] = units[u].consumed ? units[u].consumed : srcSize - p;
        p += units[u].consumed;
    }
}

/* A unit's totals, after the scans of its blocks (and their checksums): the verdict of fc_verdict_frame with unlimited
 * room and no placement -- its decoded size, or its error code.  The content checksum is not part of it. */
FC_FN int64_t fc_totals_frame(const fc_frame_rec* r, fc_block_tab t)
{
    int64_t pos = 0, k;
    int v = LZ4B200_OK;
    const int verifyBlocks = (r->sums & FC_VERIFY) && (r->sums & FC_BLOCK_SUM);
    if (r->status != LZ4B200_OK) return r->status;
    for (k = 0; k < r->count && v == LZ4B200_OK; k++) {
        const int64_t b = r->base + k;
        const int64_t rb = t.rawLen[b] >= 0 ? t.rawLen[b] : t.outSize[b];
        v = fc_block_sum_verdict(pos, rb, INT64_MAX, r->contentSize, t.rawLen[b] >= 0, verifyBlocks && t.dstOff[b] == FC_SUM_BAD);
        pos += rb < 0 ? 0 : rb;
    }
    return v != LZ4B200_OK ? (int64_t)v : fc_frame_result(pos, r->contentSize);
}

/* The placement of a file's units (dstOff, dstCap: the file's), before the verdict: every recorded unit gets the next
 * free byte of the file's output and the room left, until the first whose totals fail or do not fit -- the verdict
 * gives it its code in the frame order.  The units after it get room -1, so that the verdict fails them before any of
 * their bytes is placed. */
FC_FN void fc_place_file(const fc_file_rec* f, int64_t dstOff, int64_t dstCap, int64_t maxUnits, const int64_t* totals,
                         int64_t* uDstOff, int64_t* uDstCap)
{
    int64_t pos = 0, k;
    int failed = 0;
    for (k = 0; k < f->units && f->base + k < maxUnits; k++) {
        const int64_t u = f->base + k, t = totals[u];
        uDstOff[u] = dstOff + pos;
        uDstCap[u] = failed ? -1 : dstCap - pos;
        if (failed) continue;
        if (t < 0 || t > dstCap - pos) failed = 1;
        else pos += t;
    }
}

/* The fold: the file's result (decoded bytes, or the code of its first failing unit in file order), consumed (srcSize,
 * or that unit's offset) and prefix (the decoded bytes of the units before it).  uResult: every recorded unit's result
 * (the verdict's, or its totals when the call only sizes).  A unit at index maxUnits or above has no record: it fails
 * pass 1 with its own code (the walk's last unit), else it is LZ4B200_ERR_LIMIT. */
FC_FN void fc_fold_file(const fc_file_rec* f, int64_t srcOff, int64_t srcSize, int64_t maxUnits, const int64_t* uResult,
                        const int64_t* uSrcOff, int64_t* result, int64_t* consumed, int64_t* prefix)
{
    int64_t pos = 0, at = srcSize, res = 0, k;
    if (f->status == LZ4B200_ERR_ARG) { res = LZ4B200_ERR_ARG; at = 0; }
    for (k = 0; k < f->units && res >= 0; k++) {
        const int64_t u = f->base + k;
        if (u >= maxUnits) {
            res = (k + 1 == f->units && f->status != LZ4B200_OK) ? (int64_t)f->status : (int64_t)LZ4B200_ERR_LIMIT;
            at = f->overOff;
        } else if (uResult[u] < 0) {
            res = uResult[u];
            at = uSrcOff[u] - srcOff;
        } else {
            pos += uResult[u];
        }
    }
    *result = res < 0 ? res : pos;
    if (consumed) *consumed = at;
    if (prefix) *prefix = pos;
}

/* ---------------------------------------------------------------------------------------------
 * The batched frame encode (LZ4B200_compress_frames, LZ4B200_compress_frames_checksummed, and LZ4B200_compress_legacy
 * in class FC_LEGACY_CLASS): the decode's frame record and budget scan (fc_scan_count, fc_place_frame), with a record
 * that holds the frame's source size in contentSize and the checksums it is written with in sums, and one table of
 * blocks per class.
 * ------------------------------------------------------------------------------------------- */
typedef struct {               /* a class's block table; entry b of every array belongs to one block */
    int64_t* srcOff;           /* absolute offset of the block's source bytes in the call's source */
    int32_t* srcSize;          /* its size (0 for an unused entry) */
    int64_t* slotOff;          /* offset of its slot in the call's workspace */
    int32_t* cap;              /* a frame block's size - 1 (one that does not compress into fewer bytes than it has is
                                  stored raw), a legacy block's LZ4_compressBound(size) */
} fc_cblock_tab;

/* The record of an encode's pass 1 before its verdicts: the source size in contentSize, the checksums in sums; 0 for a
 * negative size or capacity (LZ4B200_ERR_ARG), else 1 */
FC_FN int fc_cclear_rec(int64_t srcSize, int64_t dstCap, int sums, fc_frame_rec* r)
{
    r->count = 0; r->base = 0; r->contentSize = srcSize; r->consumed = 0; r->cls = -1; r->hdrLen = 0; r->sums = sums;
    r->status = (srcSize < 0 || dstCap < 0) ? LZ4B200_ERR_ARG : LZ4B200_OK;
    return r->status == LZ4B200_OK;
}

/* Pass 1 of the encode: the verdict on frame f's arguments and capacity, in LZ4F_compressFrame's order -- LZ4B200_ERR_ARG
 * (a negative size or capacity), LZ4B200_ERR_DSTSIZE (dstCap below the reference's bound at the frame's optimal block
 * size ID for the checksums `sums`, dstMaxSize_tooSmall, lz4frame.c:451-452) -- and its class, block count, header
 * length and checksums (r->sums).  bsid: 4 .. 7. */
FC_FN void fc_cindex_frame_sums(int64_t srcSize, int64_t dstCap, int bsid, int contentSizeFlag, int sums, fc_frame_rec* r)
{
    int b;
    if (!fc_cclear_rec(srcSize, dstCap, sums, r)) return;
    b = fc_optimal_bsid(bsid, srcSize);
    if (dstCap < fc_frame_bound_sums(srcSize, b, sums)) { r->status = LZ4B200_ERR_DSTSIZE; return; }
    r->cls = b - 4;
    r->count = fc_frame_blocks(srcSize, b);
    r->hdrLen = (contentSizeFlag && srcSize > 0) ? 15 : 7;
}

/* pass 1 of LZ4B200_compress_frames, which writes no checksums */
FC_FN void fc_cindex_frame(int64_t srcSize, int64_t dstCap, int bsid, int contentSizeFlag, fc_frame_rec* r)
{
    fc_cindex_frame_sums(srcSize, dstCap, bsid, contentSizeFlag, 0, r);
}

/* ---------------------------------------------------------------------------------------------
 * Writing an `lz4 -l` legacy stream (LZ4IO_compressLegacy_internal, lz4io.c:766-910): the LE32 magic FC_MAGIC_LEGACY,
 * then for every FC_LEGACY_BLOCK chunk of the source (the last one may be short) the LE32 compressed size and the
 * compressed block.  No EndMark, no checksum, no stored-raw block: an incompressible chunk is written compressed, larger
 * than it is.  An empty source gives the magic alone (lz4io.c:729-731).  LZ4B200_compress_legacy runs the frame
 * encode's steps with these rules in class FC_LEGACY_CLASS.
 * ------------------------------------------------------------------------------------------- */

/* LZ4_compressBound of a chunk of n <= FC_LEGACY_BLOCK bytes: the capacity the tool compresses it with never limits it
 * (lz4io.c:886), so its bytes are those at this capacity */
FC_FN int32_t fc_legacy_cap(int32_t n) { return n + n / 255 + 16; }

/* the chunks of a source of n >= 0 bytes */
FC_FN int64_t fc_legacy_blocks(int64_t n) { return n / FC_LEGACY_BLOCK + (n % FC_LEGACY_BLOCK != 0); }

/* The longest stream of a source of n >= 0 bytes: 4 + the sum over its chunks of 4 + LZ4_compressBound(chunk).
 * Saturates at INT64_MAX. */
FC_FN int64_t fc_legacy_bound(int64_t n)
{
    const int64_t last = n % FC_LEGACY_BLOCK;
    const int64_t extra = 4 + (n / FC_LEGACY_BLOCK) * (4 + FC_LEGACY_BOUND - FC_LEGACY_BLOCK) +
                          (last ? 4 + fc_legacy_cap((int32_t)last) - last : 0);
    return n > INT64_MAX - extra ? INT64_MAX : n + extra;
}

/* Pass 1 of the legacy encode: LZ4B200_ERR_ARG (a negative size or capacity), LZ4B200_ERR_DSTSIZE (dstCap below
 * fc_legacy_bound), else class FC_LEGACY_CLASS, the chunk count and the 4-byte magic as the header. */
FC_FN void fc_lindex_file(int64_t srcSize, int64_t dstCap, fc_frame_rec* r)
{
    if (!fc_cclear_rec(srcSize, dstCap, 0, r)) return;
    if (dstCap < fc_legacy_bound(srcSize)) { r->status = LZ4B200_ERR_DSTSIZE; return; }
    r->cls = FC_LEGACY_CLASS;
    r->count = fc_legacy_blocks(srcSize);
    r->hdrLen = 4;
}

/* Pass 2 of the encode: a frame that passed writes its entries of its class's table (t: that class's).  srcOff: the
 * frame's offset in the call's source; the class's slots are slotStride bytes apart from slotBase.  A frame block's
 * capacity is size - 1, a legacy block's LZ4_compressBound(size) (fc_legacy_cap). */
FC_FN void fc_cfill_frame(const fc_frame_rec* r, int64_t srcOff, int64_t slotBase, int64_t slotStride, fc_cblock_tab t)
{
    const int64_t bs = fc_class_bytes(r->cls);
    int64_t k;
    if (r->status != LZ4B200_OK) return;
    for (k = 0; k < r->count; k++) {
        const int64_t b = r->base + k, left = r->contentSize - k * bs;
        const int32_t sz = (int32_t)(left < bs ? left : bs);
        t.srcOff[b] = srcOff + k * bs;
        t.srcSize[b] = sz;
        t.slotOff[b] = slotBase + b * slotStride;
        t.cap[b] = r->cls == FC_LEGACY_CLASS ? fc_legacy_cap(sz) : sz - 1;
    }
}

#endif /* LZ4_FRAME_CORE_H */
