// Host build of the decode call's plan (lz4_b200/csrc/lz4_decode_plan.h): TEST INFRASTRUCTURE.
// tests/test_decode_plan.py checks the layout and the route choice against the library's size functions, the sizes of the
// parent layout and the Python readers of the GPU tests.
#include <stdint.h>
#include "../../lz4_b200/csrc/lz4_decode_plan.h"

// out[12]: wide, markStride, tilesMax, scan, then the byte offsets nSeq, slowList, marks, scratch, used, tileFirst,
// tileFlag (0: absent) and the total bytes
extern "C" void plan_host(int64_t nBlocks, int perBlockCaps, int32_t dstCap, uint64_t workspaceBytes, int partial, uint64_t* out)
{
    const DecodePlan p = plan_decode(nBlocks, perBlockCaps != 0, dstCap, (size_t)workspaceBytes,
                                     partial ? kDecodePartial : kDecodeFull);
    const uint64_t v[12] = {p.wide, p.markStride, p.tilesMax, (uint64_t)p.scan, p.nSeq, p.slowList, p.marks,
                            p.scratch, p.used, p.tileFirst, p.tileFlag, p.bytes};
    for (int i = 0; i < 12; i++) out[i] = v[i];
}
