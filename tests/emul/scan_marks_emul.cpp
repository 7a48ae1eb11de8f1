// Host build of the one-thread scan (lz4_b200/csrc/lz4_scan_core.h) with the caller's mark table: TEST INFRASTRUCTURE.
// The scan kernel hands every block `marks + b * markStride` and markCap = markStride, so the table of a block starts at
// any word of a 32-byte chunk; tests/test_scan_marks_host.py and tests/test_gpu_scan_marks.py place it the same way.
#include <stdint.h>
#include "../../lz4_b200/csrc/lz4_scan_core.h"

extern "C" int scan_host_cap(const uint8_t* src, int n, int cap, uint32_t* nSeqOut, uint32_t* marks, uint32_t markCap)
{
    *nSeqOut = 0;
    MemPtr<true> mem{src};
    return scan_block(mem, n, cap, nSeqOut, marks, markCap);
}
