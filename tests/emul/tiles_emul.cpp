// CPU emulator of the tiles expand kernel (lz4_b200/csrc/lz4_kernels.cu: lz4_expand_tiles_kernel): TEST INFRASTRUCTURE.
// A block above 64 KB is decoded tile by tile with the device's text (lz4_rows_core.h: rw_parse_wide, rw_tile_runs,
// rw_put_deltas; lz4_decode_plan.h: tile_index_seq): wide marks from the scan, the tile index (first sequence per tile),
// per tile runs pass 1, rank, runs pass 2, waves with the kernel's three kinds of source -- compressed byte (virtual
// range), byte of this tile (window), byte of an earlier tile (destination).  Checks what the kernel relies on: every
// source read from the window was written in an earlier wave, every history read lies in an earlier tile.  Checked by
// tests/test_tiles_emul.py.
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../lz4_b200/csrc/lz4_scan_core.h"
#include "../../lz4_b200/csrc/lz4_rows_core.h"
#include "../../lz4_b200/csrc/lz4_decode_plan.h"

namespace {
constexpr int kThreads = 1024;
constexpr uint32_t kOutS = 65616 + 4096;              // any window address above 65535 (the device's is sBase + offsetof(out))
constexpr uint32_t kLitBase = 1u << 28, kZeroV = kLitBase + (1u << 27);
}

// returns LZ4_decompress_safe's value; out (cap bytes) receives the decoded bytes when it is > 0.
// stats: [0] tiles, [1] most runs in a tile, [2] hops, [3] illegal reads (must be 0), [4] sequences, [5] history reads
extern "C" int tiles_emulate(const uint8_t* comp, int n, int cap, uint8_t* out, int rpt, long long* stats)
{
    for (int i = 0; i < 6; i++) stats[i] = 0;
    if (n <= 0 || cap <= 65536 || rpt < 1) return -1000000;
    const uint32_t markCap = (uint32_t)cap / 4u + 2u;
    std::vector<uint32_t> marks(2 * (size_t)markCap, 0);
    uint32_t nseqU = 0;
    MemPtr<true, true> mem{comp};
    const int total = scan_block(mem, n, cap, &nseqU, marks.data(), markCap);
    if (total <= 0) return total;
    const int nseq = (int)nseqU;
    stats[4] = nseq;
    if (nseqU > markCap) return -1000001;
    // ---- lz4_tile_index_kernel ----
    const uint32_t nT = tiles_of(total);
    stats[0] = nT;
    std::vector<uint32_t> first(nT + 1, 0xFFFFFFFFu);
    for (uint32_t k = 0; k < nseqU; k++) tile_index_seq(first.data(), marks.data(), k, nseqU, nT);
    for (uint32_t t = 0; t <= nT; t++) if (first[t] == 0xFFFFFFFFu) return -1000005;
    // ---- tiles, in order ----
    std::vector<uint8_t> win(kOutS + 65536 + 16, 0xEE);
    std::vector<uint2> rows(2048);
    std::vector<uint32_t> tab(kRowsMaxRuns);
    memset(out, 0xEE, (size_t)cap);
    for (uint32_t t = 0; t < nT; t++) {
        const int os = (int)(t * (uint32_t)kTile), oe = os + kTile < total ? os + kTile : total, len = oe - os;
        const int k0 = first[t] ? (int)first[t] - 1 : 0, k1 = (int)(first[t + 1] + 1u < nseqU ? first[t + 1] + 1u : nseqU);
        const uint32_t litBase = kLitBase - kOutS + (uint32_t)os;
        const int zeroDelta0 = (int)(kZeroV - kOutS + (uint32_t)os);
        for (auto& r : rows) r = uint2{0u, 0u};
        for (auto& x : tab) x = 0xDEADBEEFu;
        auto seq = [&](int k) { return rw_parse_wide(comp, marks[2 * (size_t)k], marks[2 * (size_t)k + 1], k + 1 == nseq); };
        int covered = 0;
        for (int k = k0; k < k1; k++) {
            const RwSeq s = seq(k);
            int last = -1, firstSt = -1;
            rw_tile_runs(s, os, oe, litBase, zeroDelta0, [&](int st, int) {
                if (st < 0 || st >= len || st <= last) { stats[3]++; return; }
                if (last < 0) firstSt = st;
                last = st;
                rows[st >> 5].x |= 1u << (st & 31);
            });
            if (firstSt != rw_tile_first(s, os, oe)) stats[3]++;      // pass 2 looks up the rank of this run only
            const int a = s.op > os ? s.op : os, b = (s.mlen ? s.m + s.mlen : s.op + s.ll) < oe ? (s.mlen ? s.m + s.mlen : s.op + s.ll) : oe;
            if (b > a) covered += b - a;
        }
        if (covered != len) return -1000006;                      // the sequences [k0, k1) must tile the tile exactly
        uint32_t run = 0;
        for (int r = 0; r < 2048; r++) { rows[r].y = run - 1u; run += (uint32_t)__builtin_popcount(rows[r].x); }
        if ((long long)run > stats[1]) stats[1] = run;
        if (run > (uint32_t)kRowsMaxRuns) return -1000002;
        if (!(rows[0].x & 1u)) return -1000007;                   // byte 0 of a tile starts a run
        for (int k = k0; k < k1; k++) {
            const RwSeq s = seq(k);
            rw_put_deltas(rows.data(), tab.data(), rw_tile_first(s, os, oe), [&](auto f) { rw_tile_runs(s, os, oe, litBase, zeroDelta0, f); });
        }
        const int wave = kThreads * rpt;
        std::vector<uint8_t> stage((size_t)wave);
        for (int w0 = 0; w0 < len; w0 += wave) {
            const uint32_t waveS = kOutS + (uint32_t)w0;
            for (int p = w0; p < w0 + wave && p < len; p++) {
                uint32_t x = kOutS + (uint32_t)p + tab[rw_rank(rows.data(), (uint32_t)p)];
                while ((x - waveS) < (uint32_t)wave) {             // a source inside this wave: follow it
                    if (x >= kOutS + (uint32_t)p) return -1000003;   // a hop must move strictly backwards
                    x += tab[rw_rank(rows.data(), x - kOutS)];
                    stats[2]++;
                }
                uint8_t v;
                if (x >= kLitBase) {
                    if (x == kZeroV) v = 0;
                    else { const uint32_t c = x - kLitBase; if (c >= (uint32_t)n) { stats[3]++; v = 0; } else v = comp[c]; }
                } else if (x >= kOutS) {
                    if (x >= waveS) stats[3]++;                     // not final yet
                    v = win[x];
                } else {
                    const int64_t at = (int64_t)os - (int64_t)(kOutS - x);
                    stats[5]++;
                    if (at < 0 || at >= os) { stats[3]++; v = 0; } else v = out[at];
                }
                stage[(size_t)(p - w0)] = v;
            }
            for (int p = w0; p < w0 + wave && p < len; p++) win[kOutS + (uint32_t)p] = stage[(size_t)(p - w0)];
        }
        memcpy(out + os, win.data() + kOutS, (size_t)len);
    }
    return total;
}
