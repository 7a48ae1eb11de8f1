// Host build of the batched legacy encode's rules (lz4_b200/csrc/lz4_frame_core.h): the bound, and the index passes in
// the order the kernels run them -- pass 1 per file, the exclusive scan of the chunk counts in file order with the
// budget rule, the table cleared, pass 2 -- on a table of one class, FC_LEGACY_CLASS.
#include "../../lz4_b200/csrc/lz4_frame_core.h"

#include <vector>

extern "C" {

long long clegacy_bound_host(long long srcSize) { return fc_legacy_bound(srcSize); }

// n files of sizes srcSize[f] at source offsets srcOff[f], capacities dstCap[f], maxBlocks chunks.  Per file: status
// (after the budget rule), class (-1: none), chunk count, base in the table, header length.  The table (slots of
// LZ4_compressBound(8 MiB) rounded up to 16 from 0): source offset, size, slot offset, capacity.
void clegacy_index_host(const long long* srcOff, const long long* srcSize, const long long* dstCap, long long n,
                        long long maxBlocks, long long* status, long long* cls, long long* count, long long* base,
                        long long* hdrLen, long long* tabSrcOff, int* tabSrcSize, long long* tabSlotOff, int* tabCap)
{
    int64_t mb[FC_CLASSES] = {0, 0, 0, 0, 0};
    mb[FC_LEGACY_CLASS] = maxBlocks;
    const int64_t stride = (FC_LEGACY_BOUND + 15) & ~(int64_t)15;
    std::vector<fc_frame_rec> rec((size_t)n);
    for (long long f = 0; f < n; f++) fc_lindex_file(srcSize[f], dstCap[f], &rec[(size_t)f]);
    int64_t pre = 0;
    for (long long f = 0; f < n; f++) {
        fc_frame_rec* r = &rec[(size_t)f];
        if (r->cls < 0) continue;
        const int64_t k = fc_scan_count(r);
        fc_place_frame(r, pre, mb);
        pre += k;
    }
    std::vector<int64_t> so((size_t)maxBlocks, 0), sl((size_t)maxBlocks, 0);
    for (int64_t b = 0; b < maxBlocks; b++) { tabSrcSize[b] = 0; tabCap[b] = 0; }
    for (long long f = 0; f < n; f++) {
        const fc_frame_rec* r = &rec[(size_t)f];
        if (r->status != LZ4B200_OK) continue;
        fc_cblock_tab tab = {so.data(), tabSrcSize, sl.data(), tabCap};
        fc_cfill_frame(r, srcOff[f], 0, stride, tab);
    }
    for (int64_t b = 0; b < maxBlocks; b++) { tabSrcOff[b] = so[(size_t)b]; tabSlotOff[b] = sl[(size_t)b]; }
    for (long long f = 0; f < n; f++) {
        const fc_frame_rec& r = rec[(size_t)f];
        status[f] = r.status; cls[f] = r.cls; count[f] = r.count; base[f] = r.base; hdrLen[f] = r.hdrLen;
    }
}

}  // extern "C"
