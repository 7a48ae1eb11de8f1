// Host build of the batched file decode's rules (lz4_b200/csrc/lz4_frame_core.h): the steps of LZ4B200_decompress_files in
// its order -- the walk of every file, the scan of the unit counts, the unit records, the frame decode's budget scan and
// table fill, the block checksums, the totals, the placement, the verdict and the fold -- with the decode of each table
// entry left to a callback (the test's oracle) and no bytes produced, so no content checksum is compared.
#include "../../lz4_b200/csrc/lz4_frame_core.h"

#include <vector>

extern "C" {

// decoded size of table entry (absolute source offset, compressed size) at capacity cap: LZ4_decompress_safe's return
typedef int (*files_decode_fn)(long long srcOff, int srcSize, int cap);

// sizeOnly != 0: unlimited room (dstCap unread).  Per file: result, consumed, prefix, and the walk's units, base and
// status.  Returns the number of unit records (at most maxUnits).
long long files_host(const unsigned char* src, const int64_t* srcOff, const int64_t* srcSize, const int64_t* dstCap,
                     long long nFiles, long long maxUnits, const int64_t* maxBlocks, int mode, int sizeOnly,
                     files_decode_fn decode, int64_t* result, int64_t* consumed, int64_t* prefix,
                     int64_t* units, int64_t* base, int64_t* status)
{
    int64_t mb[FC_CLASSES], tb[FC_CLASSES], entries = 0;
    for (int c = 0; c < FC_CLASSES; c++) { mb[c] = maxBlocks[c]; tb[c] = entries; entries += mb[c]; }
    std::vector<fc_file_rec> files((size_t)nFiles);
    for (long long f = 0; f < nFiles; f++)
        fc_index_file(src + srcOff[f], srcSize[f], sizeOnly ? 0 : dstCap[f], maxUnits, mb, mode, &files[(size_t)f]);
    int64_t pre = 0;
    for (auto& fr : files) { fr.base = pre; pre += fr.units; }
    std::vector<fc_frame_rec> rec((size_t)maxUnits);
    for (auto& r : rec) { fc_clear_rec(&r); r.status = -1; }      // the device's 0xFF records: passed over
    std::vector<int64_t> uSrcOff((size_t)maxUnits), uSrcSize((size_t)maxUnits), uDstOff((size_t)maxUnits, 0),
        uDstCap((size_t)maxUnits, 0), uResult((size_t)maxUnits, 0);
    for (long long f = 0; f < nFiles; f++)
        fc_fill_file(src + srcOff[f], srcOff[f], srcSize[f], maxUnits, mb, mode, &files[(size_t)f], rec.data(),
                     uSrcOff.data(), uSrcSize.data());
    int64_t cpre[FC_CLASSES] = {0, 0, 0, 0, 0};
    for (auto& r : rec) {
        if (r.cls < 0) continue;
        const int64_t k = fc_scan_count(&r);
        fc_place_frame(&r, cpre[r.cls], mb);
        cpre[r.cls] += k;
    }
    std::vector<int64_t> tSrcOff((size_t)entries, 0), tDstOff((size_t)entries, FC_SUM_NONE);
    std::vector<int32_t> tSrcSize((size_t)entries, 0), tOutSize((size_t)entries, -1), tRawLen((size_t)entries, -1);
    auto tab = [&](int cls) {
        const int64_t t = cls >= 0 ? tb[cls] : 0;
        return fc_block_tab{tSrcOff.data() + t, tDstOff.data() + t, tSrcSize.data() + t, tOutSize.data() + t, tRawLen.data() + t};
    };
    for (int64_t u = 0; u < maxUnits; u++)
        if (rec[(size_t)u].status == LZ4B200_OK)
            fc_fill_frame(src + uSrcOff[(size_t)u], uSrcOff[(size_t)u], uSrcSize[(size_t)u], &rec[(size_t)u], tab(rec[(size_t)u].cls));
    for (int c = 0; c < FC_CLASSES; c++)                           // the scans of every class's table
        for (int64_t b = tb[c]; b < tb[c] + mb[c]; b++)
            tOutSize[(size_t)b] = decode(tSrcOff[(size_t)b], tSrcSize[(size_t)b], (int)fc_class_bytes(c));
    if (mode == FC_SUMS_VERIFY)                                    // the block checksums
        for (int64_t b = 0; b < entries; b++)
            if (tDstOff[(size_t)b] == FC_SUM_PENDING) {
                const int64_t n = tRawLen[(size_t)b] >= 0 ? tRawLen[(size_t)b] : tSrcSize[(size_t)b];
                const uint8_t* p = src + tSrcOff[(size_t)b];
                tDstOff[(size_t)b] = fc_xxh32(p, (uint64_t)n, 0) == fc_rd_le32(p + n) ? FC_SUM_NONE : FC_SUM_BAD;
            }
    for (int64_t u = 0; u < maxUnits; u++) uResult[(size_t)u] = fc_totals_frame(&rec[(size_t)u], tab(rec[(size_t)u].cls));
    if (!sizeOnly) {
        for (long long f = 0; f < nFiles; f++)
            fc_place_file(&files[(size_t)f], 0, dstCap[f], maxUnits, uResult.data(), uDstOff.data(), uDstCap.data());
        for (int64_t u = 0; u < maxUnits; u++)
            fc_verdict_frame(&rec[(size_t)u], uDstOff[(size_t)u], uDstCap[(size_t)u], tab(rec[(size_t)u].cls),
                             &uResult[(size_t)u], nullptr);
    }
    for (long long f = 0; f < nFiles; f++) {
        fc_fold_file(&files[(size_t)f], srcOff[f], srcSize[f], maxUnits, uResult.data(), uSrcOff.data(), result + f,
                     consumed + f, prefix + f);
        units[f] = files[(size_t)f].units; base[f] = files[(size_t)f].base; status[f] = files[(size_t)f].status;
    }
    return pre < maxUnits ? pre : maxUnits;
}

}  // extern "C"
