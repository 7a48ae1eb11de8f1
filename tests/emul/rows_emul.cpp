// CPU emulator of the rows expand kernel (lz4_b200/csrc/lz4_kernels.cu: lz4_expand_rows_kernel): TEST INFRASTRUCTURE.
// Runs the kernel's phases -- scan marks, runs pass 1, rank, runs pass 2, waves -- with the arithmetic of
// lz4_b200/csrc/lz4_rows_core.h (the same text the device compiles), one "thread" after the other, and
// checks the property the kernel relies on: a byte read from the output window during a wave was written
// in an EARLIER wave.  Checked by tests/test_rows_emul.py.
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../lz4_b200/csrc/lz4_scan_core.h"
#include "../../lz4_b200/csrc/lz4_rows_core.h"

namespace {
constexpr int kThreads = 1024;
constexpr uint32_t kZeroA = 0, kInA = 16, kInBytes = 65536 + 64, kOutA = kInA + kInBytes;   // window layout: zero | in | out
}

// returns LZ4_decompress_safe's value; out (cap bytes) receives the decoded bytes when it is > 0.
// stats: [0] runs, [1] hops, [2] longest hop chain, [3] reads of a byte that was not final (must be 0), [4] sequences
extern "C" int rows_emulate(const uint8_t* comp, int n, int cap, uint8_t* out, int head, int rpt, long long* stats)
{
    for (int i = 0; i < 5; i++) stats[i] = 0;
    if (n <= 0 || n > 65535 || cap <= 0 || cap > 65536 || head < 0 || head > 15 || rpt < 1) return -1000000;
    std::vector<uint32_t> marks(kMaxSeqFast, 0);
    uint32_t nseqU = 0;
    MemPtr<true> mem{comp};
    const int total = scan_block(mem, n, cap, &nseqU, marks.data(), (uint32_t)kMaxSeqFast);
    if (total <= 0) return total;
    const int nseq = (int)nseqU;
    stats[4] = nseq;
    if (nseq > kMaxSeqFast) return -1000001;

    std::vector<uint8_t> win(kOutA + 65536, 0xEE);
    memset(win.data() + kZeroA, 0, 16);
    memcpy(win.data() + kInA + head, comp, (size_t)n);
    const uint8_t* in = win.data() + kInA + head;
    const uint32_t inA = kInA + (uint32_t)head, outA = kOutA;
    const int zeroDelta0 = (int)kZeroA - (int)kOutA;
    std::vector<uint2> rows(2048, uint2{0u, 0u});
    std::vector<uint32_t> tab(kRowsMaxRuns, 0xDEADBEEFu);

    const int litDelta = (int)(inA - outA);
    auto seq = [&](int k) {
        return rw_parse(in, marks[k], k, k + 1 == nseq);
    };
    // pass 1
    for (int tid = 0; tid < kThreads; tid++)
        for (int k = tid; k < nseq; k += kThreads)
            rw_seq_runs(seq(k), litDelta, zeroDelta0, [&](int p, int) { rows[p >> 5].x |= 1u << (p & 31); });
    // rank
    uint32_t run = 0;
    for (int r = 0; r < 2048; r++) { rows[r].y = run - 1u; run += (uint32_t)__builtin_popcount(rows[r].x); }
    stats[0] = run;
    if (run > (uint32_t)kRowsMaxRuns) return -1000002;           // the kernel hands such a block to the generic kernel
    // pass 2
    for (int tid = 0; tid < kThreads; tid++)
        for (int k = tid; k < nseq; k += kThreads) {
            const RwSeq s = seq(k);
            rw_put_deltas(rows.data(), tab.data(), rw_seq_first(s), [&](auto f) { rw_seq_runs(s, litDelta, zeroDelta0, f); });
        }
    // waves
    const int wave = kThreads * rpt;
    std::vector<uint8_t> stage((size_t)wave);
    for (int w0 = 0; w0 < total; w0 += wave) {
        const uint32_t waveA = outA + (uint32_t)w0;
        for (int p = w0; p < w0 + wave && p < total; p++) {
            uint32_t a = outA + (uint32_t)p + tab[rw_rank(rows.data(), (uint32_t)p)];
            long long chain = 0;
            while (a >= waveA) {
                if (a >= outA + (uint32_t)p) return -1000003;    // a hop must move strictly backwards
                a += tab[rw_rank(rows.data(), a - outA)];
                chain++;
            }
            stats[1] += chain;
            if (chain > stats[2]) stats[2] = chain;
            if (a >= outA + (uint32_t)total) return -1000004;
            if (a < kZeroA + 16 && a != kZeroA) stats[3]++;       // only the first zero byte is a legal source below `in`
            if (a >= kInA && a < outA && (a < inA || a >= inA + (uint32_t)n)) stats[3]++;   // outside the staged block
            stage[(size_t)(p - w0)] = win[a];                      // everything below waveA is final (earlier waves)
        }
        for (int p = w0; p < w0 + wave && p < total; p++) win[outA + (uint32_t)p] = stage[(size_t)(p - w0)];
    }
    memcpy(out, win.data() + outA, (size_t)total);
    return total;
}
