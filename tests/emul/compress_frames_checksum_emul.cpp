// Host build of the checksummed frame encode's rules (lz4_b200/csrc/lz4_frame_core.h): the header bytes and the bound
// with the checksum flags, and pass 1's verdict on one frame.
#include "../../lz4_b200/csrc/lz4_frame_core.h"

extern "C" {

int cframes_header_sums_host(unsigned char* out, int bsid, long long contentSize, int sums)
{
    return fc_frame_header_sums(out, bsid, contentSize, sums);
}

long long cframes_bound_sums_host(long long srcSize, int bsid, int sums) { return fc_frame_bound_sums(srcSize, bsid, sums); }

// pass 1 on one frame: its status, and through the pointers its class, block count, header length and checksums
int cframes_index_sums_host(long long srcSize, long long dstCap, int bsid, int contentSizeFlag, int sums, int* cls,
                            long long* count, int* hdrLen, int* recSums)
{
    fc_frame_rec r;
    fc_cindex_frame_sums(srcSize, dstCap, bsid, contentSizeFlag, sums, &r);
    *cls = r.cls; *count = r.count; *hdrLen = r.hdrLen; *recSums = r.sums;
    return r.status;
}

}  // extern "C"
