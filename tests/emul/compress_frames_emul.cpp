// Host build of the batched frame encode's frame rules (lz4_b200/csrc/lz4_frame_core.h): the header bytes, the bound,
// the optimal block size ID, and the index passes in the order the kernels run them -- pass 1 per frame, the per-class
// exclusive scan in frame order with the budget rule, the table cleared, pass 2.
#include "../../lz4_b200/csrc/lz4_frame_core.h"

#include <vector>

extern "C" {

int cframes_header_host(unsigned char* out, int bsid, long long contentSize)
{
    return fc_frame_header_bytes(out, bsid, contentSize);
}

long long cframes_bound_host(long long srcSize, int bsid) { return fc_frame_bound(srcSize, bsid); }

int cframes_optimal_bsid_host(int requested, long long srcSize) { return fc_optimal_bsid(requested, srcSize); }

// n frames of sizes srcSize[f] at source offsets srcOff[f], capacities dstCap[f].  Per frame: status (after the budget
// rule), class (-1: none), block count, base in its class's table, header length.  The table of all classes (class c's
// entries from tabBase[c] = sum of the earlier budgets, its slots from the sum of the earlier classes' slot bytes):
// source offset, size, slot offset, capacity.  Returns the table's entry count.
long long cframes_index_host(const long long* srcOff, const long long* srcSize, const long long* dstCap, long long n,
                             int bsid, int contentSizeFlag, const long long* maxBlocks, long long* status, long long* cls,
                             long long* count, long long* base, long long* hdrLen, long long* tabSrcOff,
                             int* tabSrcSize, long long* tabSlotOff, int* tabCap)
{
    int64_t mb[4], tb[4], sb[4], ss[4], entries = 0, slots = 0;
    for (int c = 0; c < 4; c++) {
        mb[c] = maxBlocks[c]; tb[c] = entries; entries += mb[c];
        ss[c] = (fc_block_bytes(4 + c) - 1 + 15) & ~(int64_t)15; sb[c] = slots; slots += mb[c] * ss[c];
    }
    std::vector<fc_frame_rec> rec((size_t)n);
    for (long long f = 0; f < n; f++) fc_cindex_frame(srcSize[f], dstCap[f], bsid, contentSizeFlag, &rec[(size_t)f]);
    int64_t pre[4] = {0, 0, 0, 0};
    for (long long f = 0; f < n; f++) {
        fc_frame_rec* r = &rec[(size_t)f];
        if (r->cls < 0) continue;
        const int64_t k = fc_scan_count(r);
        fc_place_frame(r, pre[r->cls], mb);
        pre[r->cls] += k;
    }
    std::vector<int64_t> so((size_t)entries, 0), sl((size_t)entries, 0);
    for (int64_t b = 0; b < entries; b++) { tabSrcSize[b] = 0; tabCap[b] = 0; }
    for (long long f = 0; f < n; f++) {
        const fc_frame_rec* r = &rec[(size_t)f];
        if (r->status != LZ4B200_OK) continue;
        const int64_t t = tb[r->cls];
        fc_cblock_tab tab = {so.data() + t, tabSrcSize + t, sl.data() + t, tabCap + t};
        fc_cfill_frame(r, srcOff[f], sb[r->cls], ss[r->cls], tab);
    }
    for (int64_t b = 0; b < entries; b++) { tabSrcOff[b] = so[(size_t)b]; tabSlotOff[b] = sl[(size_t)b]; }
    for (long long f = 0; f < n; f++) {
        const fc_frame_rec& r = rec[(size_t)f];
        status[f] = r.status; cls[f] = r.cls; count[f] = r.count; base[f] = r.base; hdrLen[f] = r.hdrLen;
    }
    return entries;
}

}  // extern "C"
