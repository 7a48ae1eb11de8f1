// Host build of the checksummed frame decode's rules (lz4_b200/csrc/lz4_frame_core.h): fc_xxh32, and the index passes in
// a checksum mode -- pass 1 per frame, the per-class exclusive scan in frame order with the budget rule, pass 2 -- as
// frames_index_host (frame_emul.cpp) runs them for the checksum-free call.
#include "../../lz4_b200/csrc/lz4_frame_core.h"

#include <vector>

extern "C" {

unsigned frames_xxh32_host(const unsigned char* p, unsigned long long len, unsigned seed)
{
    return fc_xxh32(p, len, seed);
}

// frames_index_host's arguments, with mode (FC_SUMS_REJECT 0, FC_SUMS_SKIP 1, FC_SUMS_VERIFY 2) after maxBlocks, and per
// frame the record's checksum bits (sums); tabMark: the entry's block checksum state after the fill (FC_SUM_*)
long long frames_index_mode_host(const unsigned char* src, const long long* srcOff, const long long* srcSize,
                                 const long long* dstCap, long long n, const long long* maxBlocks, int mode,
                                 long long* status, long long* cls, long long* count, long long* base, long long* consumed,
                                 long long* sums, long long* tabSrcOff, int* tabSrcSize, int* tabRawLen, long long* tabMark)
{
    int64_t mb[4], tb[4], entries = 0;
    for (int c = 0; c < 4; c++) { mb[c] = maxBlocks[c]; tb[c] = entries; entries += mb[c]; }
    std::vector<fc_frame_rec> rec((size_t)n);
    for (long long f = 0; f < n; f++) fc_index_frame_mode(src + srcOff[f], srcSize[f], dstCap[f], mb, mode, &rec[(size_t)f]);
    int64_t pre[4] = {0, 0, 0, 0};
    for (long long f = 0; f < n; f++) {
        fc_frame_rec* r = &rec[(size_t)f];
        if (r->cls < 0) continue;
        const int64_t k = fc_scan_count(r);
        fc_place_frame(r, pre[r->cls], mb);
        pre[r->cls] += k;
    }
    std::vector<int64_t> off((size_t)entries, 0), mark((size_t)entries, FC_SUM_NONE);
    std::vector<int32_t> outSize((size_t)entries);
    for (int64_t b = 0; b < entries; b++) { tabSrcSize[b] = 0; tabRawLen[b] = -1; }
    for (long long f = 0; f < n; f++) {
        const fc_frame_rec* r = &rec[(size_t)f];
        if (r->status != LZ4B200_OK) continue;
        const int64_t t = tb[r->cls];
        fc_block_tab tab = {off.data() + t, mark.data() + t, tabSrcSize + t, outSize.data() + t, tabRawLen + t};
        fc_fill_frame(src + srcOff[f], srcOff[f], srcSize[f], r, tab);
    }
    for (int64_t b = 0; b < entries; b++) { tabSrcOff[b] = off[(size_t)b]; tabMark[b] = mark[(size_t)b]; }
    for (long long f = 0; f < n; f++) {
        const fc_frame_rec& r = rec[(size_t)f];
        status[f] = r.status; cls[f] = r.cls; count[f] = r.count; base[f] = r.base; consumed[f] = r.consumed;
        sums[f] = r.sums;
    }
    return entries;
}

}  // extern "C"
