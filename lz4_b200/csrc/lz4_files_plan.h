/*
 * lz4_files_plan.h -- the host side of LZ4B200_decompress_files_host and LZ4B200_decompress_files_to_device: the walk of
 * every file into its units and their blocks with the frame core's own steps (lz4_frame_core.h), the cut of the blocks
 * into groups, the placement of each group's output in the files, and the fold of the per-block results into every
 * file's result, consumed and prefix with the verdicts of LZ4B200_decompress_files.  The
 * call's budget is unlimited, so no unit or block is ever over it.  Host C (C99, and C++ for tests/emul); it allocates
 * and hashes no byte of a file.
 */
#ifndef LZ4_FILES_PLAN_H
#define LZ4_FILES_PLAN_H

#include <stdlib.h>
#include <string.h>
#include "lz4_frame_core.h"

typedef struct {               /* one block of the call, in file order */
    int64_t srcOff;            /* absolute offset of its stored bytes in the call's source */
    int64_t unit;
    int32_t size;              /* stored bytes */
    int8_t cls;                /* its class: 0 .. 3 frame blocks of block size ID 4 + c, FC_LEGACY_CLASS */
    int8_t raw;                /* stored raw */
    int8_t sumBytes;           /* 4 when a block checksum follows it */
    int8_t verify;             /* the call compares that checksum */
} fp_block;

typedef struct {
    fc_frame_rec r;            /* the unit's record; r.base is its first block in the call's list, r.count its blocks */
    int64_t file;
    uint32_t contentSum;       /* the content checksum it carries, when the call compares it (fp_content) */
    int32_t pad;
} fp_unit;

typedef struct {
    int64_t nFiles, nUnits, nBlocks;
    fc_file_rec* files;        /* units, base (its first unit) and status of fc_index_file's walk */
    fp_unit* units;
    fp_block* blocks;
    int64_t* uOff;             /* [nUnits] the unit's offset in its file */
    /* the results, one per block, filled as the groups retire: the fold's fc_block_tab */
    int32_t* outSize;          /* the decode's return value */
    int32_t* rawLen;           /* a stored-raw block's size, -1 */
    int64_t* sumState;         /* FC_SUM_NONE or FC_SUM_BAD */
    uint8_t* contentBad;       /* [nUnits] its content checksum did not match */
} fp_plan;

/* the unit compares a content checksum */
static inline int fp_content(const fp_unit* u) { return (u->r.sums & FC_VERIFY) && (u->r.sums & FC_CONTENT_SUM); }

static inline int fp_grow(void** p, int64_t* cap, int64_t need, size_t elem)
{
    void* q;
    int64_t c = *cap;
    if (need <= c) return 1;
    while (c < need) c = c ? 2 * c : 1024;
    q = realloc(*p, (size_t)c * elem);
    if (!q) return 0;
    *p = q; *cap = c;
    return 1;
}

static inline void fp_free(fp_plan* p)
{
    free(p->files); free(p->units); free(p->blocks); free(p->uOff);
    free(p->outSize); free(p->rawLen); free(p->sumState); free(p->contentBad);
    memset(p, 0, sizeof *p);
}

/* The walk of every file (src: the call's source; dstCap NULL when it only sizes): fc_index_file's walk with no budget,
 * each unit recorded with its blocks (fc_next_class_block from the end of its header).  mode: FC_SUMS_SKIP or
 * FC_SUMS_VERIFY.  Returns 0 when memory runs out. */
static inline int fp_build(const uint8_t* src, const int64_t* srcOff, const int64_t* srcSize, const int64_t* dstCap,
                           int64_t nFiles, int mode, fp_plan* p)
{
    const int64_t unlimited[FC_CLASSES] = {INT64_MAX, INT64_MAX, INT64_MAX, INT64_MAX, INT64_MAX};
    int64_t capU = 0, capB = 0, capO = 0, f, b;
    memset(p, 0, sizeof *p);
    p->nFiles = nFiles;
    p->files = (fc_file_rec*)calloc((size_t)(nFiles ? nFiles : 1), sizeof(fc_file_rec));
    if (!p->files) return 0;
    for (f = 0; f < nFiles; f++) {
        fc_file_rec* fr = &p->files[f];
        const uint8_t* s = src + srcOff[f];
        int64_t at = 0;
        fr->base = p->nUnits;
        if (srcSize[f] < 0 || (dstCap && dstCap[f] < 0)) { fr->status = LZ4B200_ERR_ARG; continue; }
        while (at < srcSize[f]) {
            fp_unit* u;
            int64_t ip, bat, bsz;
            int raw;
            if (!fp_grow((void**)&p->units, &capU, p->nUnits + 1, sizeof(fp_unit)) ||
                !fp_grow((void**)&p->uOff, &capO, p->nUnits + 1, sizeof(int64_t)))
                return 0;
            u = &p->units[p->nUnits];
            fc_next_unit(s + at, srcSize[f] - at, unlimited, mode, &u->r);
            u->file = f; u->contentSum = 0; u->pad = 0;
            p->uOff[p->nUnits] = at;
            u->r.base = p->nBlocks;
            fr->units++;
            p->nUnits++;
            if (u->r.status != LZ4B200_OK || u->r.consumed == 0) { fr->status = u->r.status; break; }
            if (u->r.cls >= 0) {
                ip = u->r.hdrLen;
                while (fc_next_class_block(s + at, srcSize[f] - at, u->r.cls, u->r.sums, &ip, &bat, &bsz, &raw) == 1) {
                    fp_block* k;
                    if (!fp_grow((void**)&p->blocks, &capB, p->nBlocks + 1, sizeof(fp_block))) return 0;
                    k = &p->blocks[p->nBlocks++];
                    k->srcOff = srcOff[f] + at + bat; k->unit = p->nUnits - 1; k->size = (int32_t)bsz;
                    k->cls = (int8_t)u->r.cls; k->raw = (int8_t)raw;
                    k->sumBytes = (u->r.sums & FC_BLOCK_SUM) ? 4 : 0;
                    k->verify = (u->r.sums & FC_VERIFY) && (u->r.sums & FC_BLOCK_SUM);
                }
            }
            if (fp_content(u)) u->contentSum = fc_rd_le32(s + at + u->r.consumed - 4);
            at += u->r.consumed;
        }
    }
    b = p->nBlocks ? p->nBlocks : 1;
    p->outSize = (int32_t*)malloc((size_t)b * sizeof(int32_t));
    p->rawLen = (int32_t*)malloc((size_t)b * sizeof(int32_t));
    p->sumState = (int64_t*)calloc((size_t)b, sizeof(int64_t));                  /* FC_SUM_NONE */
    p->contentBad = (uint8_t*)calloc((size_t)(p->nUnits ? p->nUnits : 1), 1);
    if (!p->outSize || !p->rawLen || !p->sumState || !p->contentBad) return 0;
    for (b = 0; b < p->nBlocks; b++) { p->outSize[b] = -1; p->rawLen[b] = p->blocks[b].raw ? p->blocks[b].size : -1; }
    for (f = 0; f < p->nUnits; f++) {                /* a frame of no blocks: the content checksum of no bytes */
        const fp_unit* u = &p->units[f];
        if (u->r.status == LZ4B200_OK && u->r.count == 0 && fp_content(u)) {
            fc_xxh32_state st;
            fc_xxh32_init(&st);
            p->contentBad[f] = fc_xxh32_digest(&st) != u->contentSum;
        }
    }
    return 1;
}

/* The end of the group that starts at block `first`: the blocks after it while the decode capacities (fc_class_bytes)
 * of the group stay within capBytes; at least one. */
static inline int64_t fp_group_end(const fp_plan* p, int64_t first, int64_t capBytes)
{
    int64_t end = first + 1, bytes = fc_class_bytes(p->blocks[first].cls);
    while (end < p->nBlocks && bytes + fc_class_bytes(p->blocks[end].cls) <= capBytes) bytes += fc_class_bytes(p->blocks[end++].cls);
    return end;
}

typedef struct {               /* len bytes of a group's output, from byte `packed` of it, to byte fileOff of file's output */
    int64_t packed, file, fileOff, len;
} fp_run;

/* The placement of the output of the group of blocks [first, end), once their results are in the plan (outSize): the
 * blocks' bytes lie back to back in the group's packed output in file order (a stored-raw block's size, a decoded
 * block's result, 0 when it failed), and each goes to its file's running position filePos[f], clipped to the room
 * dstCap[f].  A file takes nothing from its first block that failed to decode or was clipped on (fileStop[f]).  Runs of
 * one file that are contiguous on both sides are merged.  Returns the number of runs written to runs (at most
 * end - first). */
static inline int64_t fp_place(const fp_plan* p, int64_t first, int64_t end, const int64_t* dstCap, int64_t* filePos,
                               uint8_t* fileStop, fp_run* runs)
{
    int64_t k, pos = 0, n = 0;
    for (k = first; k < end; k++) {
        const fp_block* b = &p->blocks[k];
        const int64_t f = p->units[b->unit].file;
        const int64_t sz = b->raw ? b->size : p->outSize[k] > 0 ? p->outSize[k] : 0;
        if (!fileStop[f]) {
            if (!b->raw && p->outSize[k] < 0) fileStop[f] = 1;
            else {
                const int64_t room = dstCap[f] - filePos[f], w = sz < room ? sz : room > 0 ? room : 0;
                if (w > 0) {
                    fp_run* r = n ? &runs[n - 1] : NULL;
                    if (r && r->file == f && r->packed + r->len == pos && r->fileOff + r->len == filePos[f]) r->len += w;
                    else { r = &runs[n++]; r->packed = pos; r->file = f; r->fileOff = filePos[f]; r->len = w; }
                }
                if (w < sz) fileStop[f] = 1;
                filePos[f] += sz;
            }
        }
        pos += sz;
    }
    return n;
}

/* The fold, once every block's results are in:LZ4B200_decompress_files's totals, then either the results at unlimited
 * room (dstCap NULL: the call only sizes) or the place of every file's units (fc_place_file), the verdict on each
 * (fc_verdict_frame) and its content checksum; then fc_fold_file.  consumed and prefix may be NULL.  Returns 0 when
 * memory runs out. */
static inline int fp_fold(fp_plan* p, const int64_t* srcSize, const int64_t* dstCap, int64_t* result, int64_t* consumed,
                          int64_t* prefix)
{
    const fc_block_tab t = {NULL, p->sumState, NULL, p->outSize, p->rawLen};
    const size_t n = (size_t)(p->nUnits ? p->nUnits : 1);
    int64_t* totals = (int64_t*)malloc(n * sizeof(int64_t));
    int64_t* uDstOff = (int64_t*)malloc(n * sizeof(int64_t));
    int64_t* uDstCap = (int64_t*)malloc(n * sizeof(int64_t));
    int64_t u, f;
    if (!totals || !uDstOff || !uDstCap) { free(totals); free(uDstOff); free(uDstCap); return 0; }
    for (u = 0; u < p->nUnits; u++) totals[u] = fc_totals_frame(&p->units[u].r, t);
    if (dstCap) {
        for (f = 0; f < p->nFiles; f++)
            fc_place_file(&p->files[f], 0, dstCap[f], p->nUnits, totals, uDstOff, uDstCap);
        for (u = 0; u < p->nUnits; u++) {                                    /* totals[u] becomes the unit's result */
            fc_verdict_frame(&p->units[u].r, uDstOff[u], uDstCap[u], t, &totals[u], NULL);
            if (totals[u] >= 0 && fp_content(&p->units[u]) && p->contentBad[u]) totals[u] = LZ4B200_ERR_CHECKSUM;
        }
    }
    for (f = 0; f < p->nFiles; f++)
        fc_fold_file(&p->files[f], 0, srcSize[f], p->nUnits, totals, p->uOff, &result[f], consumed ? &consumed[f] : NULL,
                     prefix ? &prefix[f] : NULL);
    free(totals); free(uDstOff); free(uDstCap);
    return 1;
}

#endif /* LZ4_FILES_PLAN_H */
