// Host build of the decoder's scan (lz4_b200/csrc/lz4_scan_core.h): TEST INFRASTRUCTURE.
// The same text the scan kernel compiles for the device, compiled by g++ so that its logic -- the
// exact return value of LZ4_decompress_safe and the per-sequence marks -- can be checked against the
// oracle and the golden vectors without a GPU (tests/test_scan_core_host.py).
#include <stdint.h>
#include "../../lz4_b200/csrc/lz4_scan_core.h"

// src must be readable from the 4-byte aligned address at or below src up to the aligned word that
// holds src[n-1] (the device reads whole aligned words too).  A mark table of markCap words: the scan kernel hands every
// block `marks + b * markStride` and markCap = markStride, so the table of a block starts at any word of a 32-byte chunk;
// tests/test_scan_marks_host.py and tests/test_gpu_scan_marks.py place it the same way.
extern "C" int scan_host_cap(const uint8_t* src, int n, int cap, uint32_t* nSeqOut, uint32_t* marks, uint32_t markCap)
{
    *nSeqOut = 0;
    MemPtr<true> mem{src};
    return scan_block(mem, n, cap, nSeqOut, marks, markCap);
}

// A mark table of kMaxSeqFast words
extern "C" int scan_host(const uint8_t* src, int n, int cap, uint32_t* nSeqOut, uint32_t* marks)
{
    return scan_host_cap(src, n, cap, nSeqOut, marks, (uint32_t)kMaxSeqFast);
}

extern "C" int scan_host_max_seq(void) { return kMaxSeqFast; }
