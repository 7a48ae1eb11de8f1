// Host build of LZ4B200_decompress_files_host's plan and fold (lz4_b200/csrc/lz4_files_plan.h): the walk of every file,
// the cut of its blocks into groups of at most groupBytes of decode capacity, the results of each group put in the
// plan as the call's retire puts them -- each block's decode from a callback (the test's oracle), its block checksum
// compared here with fc_xxh32 (what the block checksum kernel does), the content checksum outcome of every frame whose
// last block is in the group from a second callback (the test's model) -- and the fold.
#include "../../lz4_b200/csrc/lz4_files_plan.h"

extern "C" {

// decoded size of a block (absolute source offset, stored size) at capacity cap: LZ4_decompress_safe's return
typedef int (*plan_decode_fn)(long long srcOff, int srcSize, int cap);
// 1 when the frame at byte unitOff of file `file` does not match its content checksum
typedef int (*plan_content_fn)(long long file, long long unitOff);

// dstCap NULL: the size-only pass.  Returns the number of groups, -1 when memory runs out, -2 when a group breaks the
// cut's rules (empty, not contiguous, or over groupBytes with more than one block).
long long files_plan_host(const unsigned char* src, const int64_t* srcOff, const int64_t* srcSize, const int64_t* dstCap,
                          long long nFiles, int skip, long long groupBytes, plan_decode_fn decode, plan_content_fn content,
                          int64_t* result, int64_t* consumed, int64_t* prefix)
{
    fp_plan p;
    long long groups = 0;
    int64_t first = 0, k;
    if (!fp_build(src, srcOff, srcSize, dstCap, nFiles, skip ? FC_SUMS_SKIP : FC_SUMS_VERIFY, &p)) { fp_free(&p); return -1; }
    while (first < p.nBlocks) {
        const int64_t end = fp_group_end(&p, first, groupBytes);
        int64_t bytes = 0;
        if (end <= first || end > p.nBlocks) { fp_free(&p); return -2; }
        for (k = first; k < end; k++) {
            const fp_block* b = &p.blocks[k];
            bytes += fc_class_bytes(b->cls);
            if (!b->raw) p.outSize[k] = decode(b->srcOff, b->size, (int)fc_class_bytes(b->cls));
            if (!skip && b->verify)
                p.sumState[k] = fc_xxh32(src + b->srcOff, (uint64_t)b->size, 0) == fc_rd_le32(src + b->srcOff + b->size)
                                ? FC_SUM_NONE : FC_SUM_BAD;
            const fp_unit* u = &p.units[b->unit];
            if (!skip && fp_content(u) && k == u->r.base + u->r.count - 1 && dstCap)
                p.contentBad[b->unit] = (uint8_t)content(u->file, p.uOff[b->unit]);
        }
        if (end - first > 1 && bytes > groupBytes) { fp_free(&p); return -2; }
        groups++;
        first = end;
    }
    const int ok = fp_fold(&p, srcSize, dstCap, result, consumed, prefix);
    fp_free(&p);
    return ok ? groups : -1;
}

}
