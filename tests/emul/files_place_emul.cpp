// Host build of the placement of LZ4B200_decompress_files_host's and LZ4B200_decompress_files_to_device's output
// (fp_place, lz4_b200/csrc/lz4_files_plan.h): the plan and groups of files_plan_emul.cpp, each group's packed output
// built here from the blocks in file order (a stored-raw block's bytes, a decoded block's bytes from the test's
// callback, nothing for a block that failed), and the runs fp_place emits copied from it into dst, as both calls' sinks
// copy them.  Then the fold.
#include <vector>

#include "../../lz4_b200/csrc/lz4_files_plan.h"

extern "C" {

// decoded size of a block (absolute source offset, stored size) at capacity cap, its bytes written to out
typedef int (*place_decode_fn)(long long srcOff, int srcSize, int cap, unsigned char* out);
typedef int (*place_content_fn)(long long file, long long unitOff);

// dst + dstOff[f] is file f's region.  Returns the number of runs, -1 when memory runs out, -2 when a run breaks its
// rules: outside its group's output or its file's room, or more runs than the group's blocks.
long long files_place_host(const unsigned char* src, const int64_t* srcOff, const int64_t* srcSize,
                           const int64_t* dstCap, long long nFiles, int skip, long long groupBytes,
                           place_decode_fn decode, place_content_fn content, unsigned char* dst, const int64_t* dstOff,
                           int64_t* result, int64_t* consumed, int64_t* prefix)
{
    fp_plan p;
    long long nRuns = 0;
    int64_t first = 0, k;
    if (!fp_build(src, srcOff, srcSize, dstCap, nFiles, skip ? FC_SUMS_SKIP : FC_SUMS_VERIFY, &p)) {
        fp_free(&p);
        return -1;
    }
    std::vector<int64_t> filePos(nFiles ? nFiles : 1, 0);
    std::vector<uint8_t> fileStop(nFiles ? nFiles : 1, 0);
    std::vector<fp_run> runs(p.nBlocks ? p.nBlocks : 1);
    std::vector<unsigned char> packed, one((size_t)fc_class_bytes(FC_LEGACY_CLASS) + 64);
    while (first < p.nBlocks) {
        const int64_t end = fp_group_end(&p, first, groupBytes);
        packed.clear();
        for (k = first; k < end; k++) {
            const fp_block* b = &p.blocks[k];
            if (b->raw) {
                packed.insert(packed.end(), src + b->srcOff, src + b->srcOff + b->size);
            } else {
                p.outSize[k] = decode(b->srcOff, b->size, (int)fc_class_bytes(b->cls), one.data());
                if (p.outSize[k] > 0) packed.insert(packed.end(), one.data(), one.data() + p.outSize[k]);
            }
            if (!skip && b->verify)
                p.sumState[k] = fc_xxh32(src + b->srcOff, (uint64_t)b->size, 0) == fc_rd_le32(src + b->srcOff + b->size)
                                ? FC_SUM_NONE : FC_SUM_BAD;
            const fp_unit* u = &p.units[b->unit];
            if (!skip && fp_content(u) && k == u->r.base + u->r.count - 1)
                p.contentBad[b->unit] = (uint8_t)content(u->file, p.uOff[b->unit]);
        }
        const int64_t n = fp_place(&p, first, end, dstCap, filePos.data(), fileStop.data(), runs.data());
        if (n > end - first) { fp_free(&p); return -2; }
        for (k = 0; k < n; k++) {
            const fp_run* r = &runs[k];
            if (r->len <= 0 || r->packed < 0 || r->packed + r->len > (int64_t)packed.size() || r->fileOff < 0 ||
                r->fileOff + r->len > dstCap[r->file]) { fp_free(&p); return -2; }
            memcpy(dst + dstOff[r->file] + r->fileOff, packed.data() + r->packed, (size_t)r->len);
        }
        nRuns += n;
        first = end;
    }
    const int ok = fp_fold(&p, srcSize, dstCap, result, consumed, prefix);
    fp_free(&p);
    return ok ? nRuns : -1;
}

}
