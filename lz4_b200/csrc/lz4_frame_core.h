/*
 * lz4_frame_core.h -- the rules of an LZ4 frame of independent blocks, in one place: the header checks and the header
 * checksum (LZ4F_decodeHeader, lz4frame.c:1340-1425), the chain of block headers (lz4frame.c:1729-1758) and the verdict
 * on the decoded blocks.  LZ4B200_decompressFrame_host (lz4_api.c, compiled as C99) and the batched frame decode
 * (lz4_kernels.cu, CUDA) both decide with these functions; tests/emul/frame_emul.cpp runs the batched call's index passes
 * on the host from the same text.  No CUDA runtime calls, no allocation.
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

FC_FN uint32_t fc_rd_le32(const uint8_t* p)
{
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

FC_FN uint32_t fc_rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

/* XXH32 of a short message (len < 16), as published in the xxHash specification; the frame header checksum is its second
 * byte (lz4frame.c:781-809: HC = (XXH32(descriptor, 0) >> 8) & 0xFF). */
FC_FN uint32_t fc_xxh32_short(const uint8_t* p, size_t len, uint32_t seed)
{
    const uint32_t P1 = 2654435761u, P2 = 2246822519u, P3 = 3266489917u, P4 = 668265263u, P5 = 374761393u;
    const uint8_t* end = p + len;
    uint32_t h = seed + P5 + (uint32_t)len;
    while (p + 4 <= end) { h += fc_rd_le32(p) * P3; h = fc_rotl32(h, 17) * P4; p += 4; }
    while (p < end) { h += (uint32_t)(*p) * P5; h = fc_rotl32(h, 11) * P1; p++; }
    h ^= h >> 15; h *= P2; h ^= h >> 13; h *= P3; h ^= h >> 16;
    return h;
}

FC_FN int64_t fc_block_bytes(int bsid) { return (int64_t)1 << (8 + 2 * bsid); }   /* 4..7 -> 64 KB..4 MB (lz4frame.c:333-342) */

typedef struct {
    int64_t contentSize;       /* the header's content size, -1 without one (a field of 2^63 or more reads negative too) */
    int32_t hdrLen;            /* bytes of the header: the first block header starts here */
    int32_t bsid;              /* block size ID, 4 .. 7 */
} fc_header_t;

/* The verdict on a frame's arguments and header, in the order LZ4B200_decompressFrame_host decides them: LZ4B200_OK (h
 * filled in), LZ4B200_ERR_ARG (srcSize or dstCap negative), LZ4B200_ERR_FRAME (malformed header) or
 * LZ4B200_ERR_UNSUPPORTED (skippable frame, linked blocks, checksums, dictID).  Reads src[0, min(srcSize, 19)). */
FC_FN int fc_frame_header(const uint8_t* src, int64_t srcSize, int64_t dstCap, fc_header_t* h)
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
    if ((uint8_t)(fc_xxh32_short(src + 4, hdrLen - 5, 0) >> 8) != src[hdrLen - 1]) return LZ4B200_ERR_FRAME;
    if (!((flg >> 5) & 1)) return LZ4B200_ERR_UNSUPPORTED;                            /* linked blocks */
    if (((flg >> 4) & 1) || ((flg >> 2) & 1) || (flg & 1)) return LZ4B200_ERR_UNSUPPORTED;   /* checksums, dictID */
    h->contentSize = -1;
    if ((flg >> 3) & 1) {
        uint64_t v = 0;
        for (i = 0; i < 8; i++) v |= (uint64_t)src[6 + i] << (8 * i);
        h->contentSize = (int64_t)v;
    }
    h->hdrLen = (int32_t)hdrLen;
    h->bsid = bsid;
    return LZ4B200_OK;
}

/* One step of the chain of block headers (lz4frame.c:1729-1758) from the block header at *ip, for blocks of at most bs
 * bytes.  Returns 1 for a block (*at: its first byte, *size, *raw: stored raw; *ip moves past it), 0 at the EndMark (*ip
 * moves past it: the frame's length), LZ4B200_ERR_FRAME for a truncated chain or a block above bs (maxBlockSize_invalid,
 * lz4frame.c:1745). */
FC_FN int fc_next_block(const uint8_t* src, int64_t srcSize, int64_t bs, int64_t* ip, int64_t* at, int64_t* size, int* raw)
{
    uint32_t h;
    int64_t sz;
    if (*ip + 4 > srcSize) return LZ4B200_ERR_FRAME;
    h = fc_rd_le32(src + *ip);
    *ip += 4;
    if (h == 0) return 0;                                                             /* EndMark */
    sz = (int64_t)(h & 0x7FFFFFFFu);
    if (sz > bs || *ip + sz > srcSize) return LZ4B200_ERR_FRAME;
    *at = *ip; *size = sz; *raw = (int)(h >> 31);
    *ip += sz;
    return 1;
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

/* a frame whose every block passed: its result, total decoded bytes, or LZ4B200_ERR_FRAME when the content size differs
 * (frameSize_wrong) */
FC_FN int64_t fc_frame_result(int64_t total, int64_t contentSize)
{
    return (contentSize >= 0 && contentSize != total) ? (int64_t)LZ4B200_ERR_FRAME : total;
}

/* ---------------------------------------------------------------------------------------------
 * The batched frame decode (LZ4B200_decompress_frames): one record per frame, one table of blocks per class (block size
 * ID 4 + c), and the three steps that run one frame per thread.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
    int64_t count;             /* blocks the chain walk saw (at most maxBlocks[cls] + 1) */
    int64_t base;              /* the frame's first entry in its class's table */
    int64_t contentSize;       /* as fc_header_t */
    int64_t consumed;          /* the frame's length once its chain is walked to the EndMark, else 0 */
    int32_t status;            /* LZ4B200_OK or the frame's error code so far */
    int32_t cls;               /* block size ID - 4 (-1 before the header passed) */
    int32_t hdrLen, pad;
} fc_frame_rec;

typedef struct {               /* a class's block table; entry b of every array belongs to one block */
    int64_t* srcOff;           /* absolute offset of the block's bytes in the call's source */
    int64_t* dstOff;           /* absolute offset of its decoded bytes in the call's destination (set by the verdict) */
    int32_t* srcSize;          /* bytes the decode gets: 0 for a stored-raw block, so that the scan rejects it */
    int32_t* outSize;          /* the decode's return value; -1 once the verdict has failed the block's frame */
    int32_t* rawLen;           /* a stored-raw block's size, -1 for a compressed block */
} fc_block_tab;

/* Pass 1 (the index): the header rules, then the chain walk, which stops after maxBlocks[cls] + 1 blocks (the frame is over
 * its budget whatever follows).  src: the frame's first byte. */
FC_FN void fc_index_frame(const uint8_t* src, int64_t srcSize, int64_t dstCap, const int64_t* maxBlocks, fc_frame_rec* r)
{
    fc_header_t h;
    int64_t ip, at, sz, n = 0;
    int raw, s;
    r->count = 0; r->base = 0; r->contentSize = -1; r->consumed = 0; r->cls = -1; r->hdrLen = 0; r->pad = 0;
    r->status = fc_frame_header(src, srcSize, dstCap, &h);
    if (r->status != LZ4B200_OK) return;
    r->cls = h.bsid - 4; r->contentSize = h.contentSize; r->hdrLen = h.hdrLen;
    ip = h.hdrLen;
    while ((s = fc_next_block(src, srcSize, fc_block_bytes(h.bsid), &ip, &at, &sz, &raw)) == 1)
        if (++n > maxBlocks[r->cls]) break;
    if (s < 0) { r->status = s; return; }
    r->count = n;
    if (s == 0) r->consumed = ip;
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

/* Pass 2 (the fill): walks the chain again and writes the frame's entries of its class's table.  srcOff: the frame's offset
 * in the call's source. */
FC_FN void fc_fill_frame(const uint8_t* src, int64_t srcOff, int64_t srcSize, const fc_frame_rec* r, fc_block_tab t)
{
    int64_t ip = r->hdrLen, at, sz, b = r->base;
    int raw;
    if (r->status != LZ4B200_OK) return;
    while (fc_next_block(src, srcSize, fc_block_bytes(r->cls + 4), &ip, &at, &sz, &raw) == 1) {
        t.srcOff[b] = srcOff + at;
        t.srcSize[b] = raw ? 0 : (int32_t)sz;
        t.rawLen[b] = raw ? (int32_t)sz : -1;
        b++;
    }
}

/* The verdict, between the scan and the expand: the block rules in block order on the scanned and the raw sizes, each
 * block's tight offset (dstOff: the frame's), the frame's result and consumed length.  Every block of a frame that fails
 * gets outSize -1 and rawLen -1, so that neither the expand nor the raw copy writes any of its bytes. */
FC_FN void fc_verdict_frame(const fc_frame_rec* r, int64_t dstOff, int64_t dstCap, fc_block_tab t, int64_t* result,
                            int64_t* consumed)
{
    int64_t pos = 0, res, k;
    int v = LZ4B200_OK;
    if (consumed) *consumed = r->consumed;
    if (r->status != LZ4B200_OK) { *result = r->status; return; }
    for (k = 0; k < r->count && v == LZ4B200_OK; k++) {
        const int64_t b = r->base + k;
        const int64_t rb = t.rawLen[b] >= 0 ? t.rawLen[b] : t.outSize[b];
        v = fc_block_verdict(pos, rb, dstCap, r->contentSize);
        t.dstOff[b] = dstOff + pos;
        pos += rb;
    }
    res = v != LZ4B200_OK ? (int64_t)v : fc_frame_result(pos, r->contentSize);
    if (res < 0)
        for (k = 0; k < r->count; k++) { t.outSize[r->base + k] = -1; t.rawLen[r->base + k] = -1; }
    *result = res;
}

#endif /* LZ4_FRAME_CORE_H */
