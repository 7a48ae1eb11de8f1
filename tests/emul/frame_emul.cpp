// Host build of the batched frame decode's index passes (lz4_b200/csrc/lz4_frame_core.h), in the order the kernels run
// them: pass 1 per frame, the per-class exclusive scan in frame order with the budget rule, the table cleared, pass 2.
#include "../../lz4_b200/csrc/lz4_frame_core.h"

#include <vector>

extern "C" {

// n frames of src: frame f = src + srcOff[f], srcSize[f] bytes, capacity dstCap[f].  Per frame: status (after the budget
// rule), class (-1: none), block count, base in its class's table, consumed.  The table of all classes (class c's entries
// from tabBase[c] = sum of the earlier budgets): source offset, decode size, raw size.  Returns the table's entry count.
long long frames_index_host(const unsigned char* src, const long long* srcOff, const long long* srcSize,
                            const long long* dstCap, long long n, const long long* maxBlocks, long long* status,
                            long long* cls, long long* count, long long* base, long long* consumed, long long* tabSrcOff,
                            int* tabSrcSize, int* tabRawLen)
{
    int64_t mb[4], tb[4], entries = 0;
    for (int c = 0; c < 4; c++) { mb[c] = maxBlocks[c]; tb[c] = entries; entries += mb[c]; }
    std::vector<fc_frame_rec> rec((size_t)n);
    for (long long f = 0; f < n; f++) fc_index_frame(src + srcOff[f], srcSize[f], dstCap[f], mb, &rec[(size_t)f]);
    int64_t pre[4] = {0, 0, 0, 0};
    for (long long f = 0; f < n; f++) {
        fc_frame_rec* r = &rec[(size_t)f];
        if (r->cls < 0) continue;
        const int64_t k = fc_scan_count(r);
        fc_place_frame(r, pre[r->cls], mb);
        pre[r->cls] += k;
    }
    std::vector<int64_t> dstOff((size_t)entries), off((size_t)entries);
    std::vector<int32_t> outSize((size_t)entries);
    for (int64_t b = 0; b < entries; b++) { off[(size_t)b] = 0; tabSrcSize[b] = 0; tabRawLen[b] = -1; }
    for (long long f = 0; f < n; f++) {
        const fc_frame_rec* r = &rec[(size_t)f];
        if (r->status != LZ4B200_OK) continue;
        const int64_t t = tb[r->cls];
        fc_block_tab tab = {off.data() + t, dstOff.data() + t, tabSrcSize + t, outSize.data() + t, tabRawLen + t};
        fc_fill_frame(src + srcOff[f], srcOff[f], srcSize[f], r, tab);
    }
    for (int64_t b = 0; b < entries; b++) tabSrcOff[b] = off[(size_t)b];
    for (long long f = 0; f < n; f++) {
        const fc_frame_rec& r = rec[(size_t)f];
        status[f] = r.status; cls[f] = r.cls; count[f] = r.count; base[f] = r.base; consumed[f] = r.consumed;
    }
    return entries;
}

}  // extern "C"
