/*
 * lz4_cfiles_plan.h -- the host side of LZ4B200_compress_frames_host and LZ4B200_compress_legacy_host: every file's
 * verdict, block size ID, header and blocks with the frame encode's own rules (lz4_frame_core.h: fc_cindex_frame_sums
 * or fc_lindex_file, fc_optimal_bsid, fc_frame_header_sums, fc_cfill_frame), and the cut of the blocks into groups.  The
 * calls' budget is unlimited, so no file is ever over it.  Host C (C99, and C++ for tests/emul); it reads no byte of a
 * file.
 */
#ifndef LZ4_CFILES_PLAN_H
#define LZ4_CFILES_PLAN_H

#include <stdlib.h>
#include <string.h>
#include "lz4_frame_core.h"

typedef struct {
    int64_t nFiles, nBlocks;
    int legacy, contentSizeFlag;
    fc_frame_rec* files;       /* pass 1's record of every file; r.base is its first block in the call's list */
    /* the blocks of every file that passed, in file order (fc_cfill_frame's table with no slots) */
    int64_t* srcOff;           /* absolute offset of the block's source bytes in the call's source */
    int32_t* size;
    int32_t* cap;              /* size - 1 for a frame block, LZ4_compressBound(size) for a legacy chunk */
    int64_t* file;
    int64_t* slotOff;          /* (fc_cfill_frame's slots: unused) */
} cp_plan;

static inline void cp_free(cp_plan* p)
{
    free(p->files); free(p->srcOff); free(p->size); free(p->cap); free(p->file); free(p->slotOff);
    memset(p, 0, sizeof *p);
}

/* Pass 1 and the block list of every file.  legacy: `lz4 -l` streams (bsid, contentSizeFlag and sums unused); else
 * frames at requested block size ID bsid (4 .. 7) with the checksums sums (FC_BLOCK_SUM | FC_CONTENT_SUM).  Returns 0
 * when memory runs out. */
static inline int cp_build(const int64_t* srcOff, const int64_t* srcSize, const int64_t* dstCap, int64_t nFiles,
                           int legacy, int bsid, int contentSizeFlag, int sums, cp_plan* p)
{
    int64_t f, n = 0;
    memset(p, 0, sizeof *p);
    p->nFiles = nFiles; p->legacy = legacy; p->contentSizeFlag = contentSizeFlag != 0;
    p->files = (fc_frame_rec*)calloc((size_t)(nFiles ? nFiles : 1), sizeof(fc_frame_rec));
    if (!p->files) return 0;
    for (f = 0; f < nFiles; f++) {
        fc_frame_rec* r = &p->files[f];
        if (legacy) fc_lindex_file(srcSize[f], dstCap[f], r);
        else fc_cindex_frame_sums(srcSize[f], dstCap[f], bsid, contentSizeFlag, sums, r);
        r->base = n;
        if (r->status == LZ4B200_OK) n += r->count;
    }
    p->nBlocks = n;
    n = n ? n : 1;
    p->srcOff = (int64_t*)malloc((size_t)n * sizeof(int64_t));
    p->size = (int32_t*)malloc((size_t)n * sizeof(int32_t));
    p->cap = (int32_t*)malloc((size_t)n * sizeof(int32_t));
    p->file = (int64_t*)malloc((size_t)n * sizeof(int64_t));
    p->slotOff = (int64_t*)malloc((size_t)n * sizeof(int64_t));
    if (!p->srcOff || !p->size || !p->cap || !p->file || !p->slotOff) return 0;
    for (f = 0; f < nFiles; f++) {
        const fc_frame_rec* r = &p->files[f];
        const fc_cblock_tab t = {p->srcOff, p->size, p->slotOff, p->cap};
        int64_t k;
        if (r->status != LZ4B200_OK) continue;
        fc_cfill_frame(r, srcOff[f], 0, 0, t);
        for (k = 0; k < r->count; k++) p->file[r->base + k] = f;
    }
    return 1;
}

/* File f's header (it passed): the frame header into h[0 .. 15), or the legacy magic.  Returns its length. */
static inline int cp_header(const cp_plan* p, int64_t f, uint8_t* h)
{
    const fc_frame_rec* r = &p->files[f];
    if (p->legacy) {
        h[0] = (uint8_t)FC_MAGIC_LEGACY; h[1] = (uint8_t)(FC_MAGIC_LEGACY >> 8);
        h[2] = (uint8_t)(FC_MAGIC_LEGACY >> 16); h[3] = (uint8_t)(FC_MAGIC_LEGACY >> 24);
        return 4;
    }
    return fc_frame_header_sums(h, r->cls + 4, p->contentSizeFlag ? r->contentSize : 0, r->sums);
}

/* The end of the group that starts at block `first`: the blocks after it while the group holds at most maxBytes source
 * bytes and maxBlocks blocks; at least one. */
static inline int64_t cp_group_end(const cp_plan* p, int64_t first, int64_t maxBytes, int64_t maxBlocks)
{
    int64_t end = first + 1, bytes = p->size[first];
    while (end < p->nBlocks && end - first < maxBlocks && bytes + p->size[end] <= maxBytes) bytes += p->size[end++];
    return end;
}

#endif /* LZ4_CFILES_PLAN_H */
