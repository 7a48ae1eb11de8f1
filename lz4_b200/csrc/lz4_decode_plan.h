/*
 * lz4_decode_plan.h -- the plan of one decode call: workspace layout, scan kernel, and which expand kernel takes which
 * block.  The host plans every call once (plan_decode) and passes the kernels the view of the workspace (WsView) by
 * value; the library's workspace sizes are the same plan's total.  Included by lz4_kernels.cu (inside its anonymous
 * namespace); the same text compiles for the host, where tests/emul/plan_emul.cpp checks it.  No CUDA runtime calls.
 */
#ifndef LZ4_DECODE_PLAN_H
#define LZ4_DECODE_PLAN_H

#include <stddef.h>
#include <stdint.h>
#include "lz4_scan_core.h"

#if defined(__CUDACC__)
#define DP_FN __host__ __device__ __forceinline__
#else
#define DP_FN static inline
#endif

constexpr int kTile = 61440;                       /* output bytes per tile of a block above 64 KB: 15 waves of 4096 */
constexpr int32_t kTileMaxCap = 64 << 20;          /* larger capacities take the generic kernel (the marks would need 2 x capacity) */
constexpr int64_t kSplitMaxBlocks = 8192;          /* largest batch the split scan is the default for (H100, see plan_decode) */
DP_FN uint32_t tiles_of(int32_t bytes) { return ((uint32_t)bytes + (uint32_t)kTile - 1u) / (uint32_t)kTile; }

enum DecodeKind { kDecodeFull, kDecodePartial };    /* LZ4_decompress_safe, or LZ4_decompress_safe_partial (capacity = target) */
enum DecodeScan { kScanThread, kScanPar, kScanSplit };

struct DecodePlan {
    bool wide;                 /* one capacity in (64 KB, 64 MB] and room for the wide marks: the tiles kernel decodes */
    uint32_t markStride;       /* mark words per block (0: no block has marks) */
    uint32_t tilesMax;         /* tiles per block of a wide batch, else 0 */
    DecodeScan scan;
    size_t nSeq, slowList, marks, scratch, used, tileFirst, tileFlag;   /* byte offsets; 0: no such region */
    size_t bytes;              /* the workspace the layout needs */
};

/* header (256 bytes) | nSeq[N] | slowList[N] | marks[N][markStride], then
 *   narrow: 2 x markStride words per block: the split scan's lists (scratch), or the input bytes each block's walk consumed
 *           (used: the partial call; absent without marks, when every block takes the generic kernel, which needs none);
 *   wide:   tileFirst[N][tilesMax + 1] (first sequence of every tile) | tileFlag[N][tilesMax + 1] (done flags, "gave up");
 * and 256 bytes of slack.  Every region starts on 256 bytes. */
DP_FN void plan_layout(DecodePlan& p, int64_t n, DecodeKind kind)
{
    const size_t lst = ((size_t)n * 4 + 255) / 256 * 256, mk = ((size_t)n * p.markStride * 4 + 255) / 256 * 256;
    const size_t tl = p.wide ? ((size_t)n * (p.tilesMax + 1) * 4 + 255) / 256 * 256 : 0;
    p.nSeq = 256;
    p.slowList = p.nSeq + lst;
    p.marks = p.slowList + lst;
    const size_t tail = p.marks + mk;
    p.scratch = !p.wide && kind == kDecodeFull ? tail : 0;
    p.used = !p.wide && kind == kDecodePartial && p.markStride ? tail : 0;
    p.tileFirst = p.wide ? tail : 0;
    p.tileFlag = p.wide ? tail + tl : 0;
    p.bytes = tail + (p.wide ? 2 * tl : 2 * mk) + 256;
}

/* The plan of a call of nBlocks blocks with per-block capacities or one capacity dstCap for all, on a workspace of
 * workspaceBytes.  The library's sizes are plans too: SIZE_MAX bytes gives the size that enables the tiles kernel, 0 the
 * smallest a call accepts. */
DP_FN DecodePlan plan_decode(int64_t nBlocks, bool perBlockCaps, int32_t dstCap, size_t workspaceBytes, DecodeKind kind)
{
    DecodePlan p;
    /* wide marks: two words per sequence; a block of capacity c has at most c / 4 + 1 sequences (all but the last make
     * >= 4 bytes) and the scan visits at most one more.  The partial call never decodes in tiles. */
    p.wide = kind == kDecodeFull && !perBlockCaps && dstCap > 65536 && dstCap <= kTileMaxCap;
    if (p.wide) {
        p.markStride = 2u * ((uint32_t)dstCap / 4u + 2u);
        p.tilesMax = tiles_of(dstCap);
        plan_layout(p, nBlocks, kind);
        p.wide = workspaceBytes >= p.bytes;           /* too small: the narrow layout, and the generic kernel */
    }
    if (!p.wide) {                                    /* marks for the blocks the rows kernel may take (capacity <= 64 KB) */
        const uint32_t s = (uint32_t)dstCap / 4u + 2u;
        p.markStride = perBlockCaps ? (uint32_t)kMaxSeqFast    /* capacities live on the device: the worst case */
                     : (dstCap <= 0 || dstCap > 65536) ? 0u : (s < (uint32_t)kMaxSeqFast ? s : (uint32_t)kMaxSeqFast);
        p.tilesMax = 0;
        plan_layout(p, nBlocks, kind);
    }
    /* The lanes of the parallel scan re-walk their segments several times (fix-up rounds), many times the instructions of
     * the one-thread scan, so it only pays for blocks far beyond 64 KB (lz4frame's 4 MB blocks: 150 000 dependent steps
     * for one thread); it is also the only scan that writes wide marks.  Blocks of 16..64 KB: kSsLanes merging lanes per
     * block (smaller blocks have too few sequences to split).  Measured on an H100 SXM at a 700 W power limit (scan kernel
     * alone, CUDA events, 64 KB P50 blocks, split against one thread per block, marks in 32-byte chunks): faster while the
     * batch is small (1.20 against 2.13 ms for 4096 blocks, 1.72 against 2.12 ms for 8192), slower beyond (2.51 against
     * 2.10 ms for 12288, 3.47 against 2.14 ms for 16384, 30.6 against 2.6 ms for 65536: the one-thread scan's time grows
     * little with the batch, the split scan's does).  The partial call has a one-thread scan only. */
    if (kind == kDecodePartial) p.scan = kScanThread;
    else if (p.wide || (!perBlockCaps && dstCap > 65536)) p.scan = kScanPar;
    else if (!perBlockCaps && dstCap >= 16384 && nBlocks <= kSplitMaxBlocks) p.scan = kScanSplit;
    else p.scan = kScanThread;
    return p;
}

struct WsHeader { uint32_t slowCount, pad[3]; };

struct WsView {                                    /* the workspace as the decode kernels see it (nullptr: no such region) */
    WsHeader* hdr; uint32_t* nSeq; uint32_t* slowList; uint32_t* marks;
    uint32_t* scratch;                             /* split scan: 2 x markStride words per block */
    uint32_t* used;                                /* partial call: input bytes each block's walk consumed */
    uint32_t* tileFirst; uint32_t* tileFlag;       /* wide batches: see lz4_expand_tiles_kernel */
    uint32_t markStride, tilesMax;
    bool wide;
};

DP_FN WsView ws_view(const DecodePlan& p, void* ws)
{
    auto at = [ws](size_t off) { return off ? reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(ws) + off) : nullptr; };
    return WsView{reinterpret_cast<WsHeader*>(ws), at(p.nSeq), at(p.slowList), at(p.marks), at(p.scratch), at(p.used),
                  at(p.tileFirst), at(p.tileFlag), p.markStride, p.tilesMax, p.wide};
}

/* where a scan leaves block b's marks (nullptr: none).  Narrow: the blocks the rows kernel may take (input and capacity
 * within its 64 KB windows); partial: the same whatever the input size (the rows kernel stages only the consumed prefix);
 * wide: every block, for the tiles kernel */
enum MarksKind { kMarksNarrow, kMarksPartial, kMarksWide };
DP_FN uint32_t* block_marks(const WsView& w, int64_t b, int n, int cap, MarksKind kind)
{
    const bool want = kind == kMarksWide ? n > 0
                    : n > 0 && (kind == kMarksPartial || n <= 65535) && cap > 0 && cap <= 65536 && w.markStride > 0;
    return want ? w.marks + (size_t)b * w.markStride : nullptr;
}

/* the sequences a block's marks hold: one word each, two in a wide batch */
DP_FN uint32_t mark_cap(const WsView& w) { return w.wide ? w.markStride / 2u : w.markStride; }

/* a block the rows kernel takes: input (the partial call: the consumed prefix) and output fit its 64 KB windows, marks
 * for every sequence */
DP_FN bool rows_eligible(int n, int cap, uint32_t nseq, uint32_t markStride)
{
    return n > 0 && n <= 65535 && cap > 0 && cap <= 65536 && nseq <= (uint32_t)kMaxSeqFast && nseq <= markStride;
}

/* a block of a wide batch the tiles kernel takes: its wide marks hold every sequence */
DP_FN bool tiles_eligible(const WsView& w, uint32_t nseq) { return nseq <= w.markStride / 2u; }

#endif
