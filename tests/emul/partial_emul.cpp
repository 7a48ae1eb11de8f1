// Host build of the partial decode's device text: TEST INFRASTRUCTURE.
// The one-thread scan with PARTIAL = true (lz4_b200/csrc/lz4_scan_core.h) and the rows kernel's rebuild of every sequence
// from its mark (rw_parse<true>, lz4_rows_core.h).  The bytes are rebuilt run by run, in sequence order, from the clipped
// runs alone (literal runs from the consumed input prefix, match runs through rw_match_runs' pieces), the way the rows
// kernel's tables describe them.  tests/test_partial_emul.py checks the result against the reference's vectors.
#include <stdint.h>
#include "../../lz4_b200/csrc/lz4_scan_core.h"
#include "../../lz4_b200/csrc/lz4_rows_core.h"

// Returns the scan's result.  With marks and a block the rows kernel may take (cap <= 65536, consumed <= 65535,
// every mark kept) `out` receives the rebuilt bytes; -1000001 if a run starts or ends at or past the return value.
extern "C" int partial_emulate(const uint8_t* src, int n, int cap, uint32_t* nSeqOut, uint32_t* usedOut, uint32_t* marks,
                               uint32_t markCap, uint8_t* out)
{
    *nSeqOut = 0;
    *usedOut = 0;
    MemPtr<true> mem{src};
    const int r = scan_block<MemPtr<true>, true>(mem, n, cap, nSeqOut, marks, markCap, usedOut);
    const int ns = (int)*nSeqOut;
    if (!marks || r <= 0 || cap > 65536 || *usedOut > 65535u || (uint32_t)ns > markCap) return r;
    const uint8_t* in = src;                       // only [0, consumed) is read: the staged prefix
    for (int k = 0; k < ns; k++) {
        const RwSeq s = rw_parse<true>(in, marks[k], k, k + 1 == ns, r);
        if (s.ls + s.ll > (int)*usedOut) return -1000002;
        bool bad = (s.ll > 0 && s.op + s.ll > r) || (s.mlen > 0 && s.m + s.mlen > r);
        rw_seq_runs(s, 0, 0, [&](int st, int) { if (st >= r) bad = true; });
        if (bad) return -1000001;
        for (int i = 0; i < s.ll; i++) out[s.op + i] = in[s.ls + i];
        for (int i = 0; i < s.mlen; i++) out[s.m + i] = s.off ? out[s.m + i - s.off] : 0;
    }
    return r;
}
