// CPU emulator of the intra-block parallel scan (lz4_b200/csrc/lz4_scan_par.h): TEST INFRASTRUCTURE.
// Runs the NL lanes of a CTA phase by phase (the device puts a CTA barrier between phases) on the
// host build of the same header and returns what the kernel would store for the block.
#include <stdint.h>
#include <string.h>
#include "../../lz4_b200/csrc/lz4_scan_par.h"

// nl lanes (at most kSpMaxLanes); stats[0] = fix-up rounds, stats[1] = lane walks in the fix-up rounds, stats[2] = lane
// that finished the block
template <class M>
static int run_par(M& mem, int n, int cap, uint32_t* nSeqOut, uint32_t* marks, uint32_t markCap, int* stats, int nl)
{
    *nSeqOut = 0;
    stats[0] = stats[1] = 0; stats[2] = -1;
    if (cap < 64 || n < kSpMinBytes) return scan_block(mem, n, cap, nSeqOut, marks, markCap);   // lane 0, one-thread scan
    static SpShared S;
    static SpLane L[kSpMaxLanes];
    memset(&S, 0, sizeof(S));
    for (int l = 0; l < nl; l++) sp_phase0(l, nl, L[l], S, mem, n, cap);
    for (;;) {
        for (int l = 0; l < nl; l++) sp_decide(l, L[l], S);
        S.changed = 0;
        for (int l = 0; l < nl; l++) { if (L[l].need && !L[l].newVoid) stats[1]++; sp_redo(l, L[l], S, mem, n, cap); }
        if (!S.changed) break;
        stats[0]++;
        if (stats[0] > 2 * nl) return -1000000;                // must converge within nl rounds
    }
    uint32_t cb = 0, ob = 0;
    int first = nl - 1;
    for (int l = 0; l < nl; l++) {
        sp_write(l, L[l], S, mem, n, cap, cb, ob, marks, markCap);
        cb += S.res[l].count; ob += S.res[l].olen;
    }
    for (int l = nl - 1; l >= 0; l--) if (S.end[l].kind != SP_RAN) first = l;
    S.ret = -2000000;
    for (int l = 0; l < nl; l++) sp_finish(l, first, S, mem, n, cap, marks, markCap);
    stats[2] = first;
    *nSeqOut = S.nseq;
    return S.ret;
}
extern "C" int scan_par_host(const uint8_t* src, int n, int cap, uint32_t* nSeqOut, uint32_t* marks, int* stats,
                             int nl)
{
    MemPtr<true> mem{src};
    return run_par(mem, n, cap, nSeqOut, marks, (uint32_t)kMaxSeqFast, stats, nl);
}
// blocks above 64 KB: wide marks (two words per sequence), parallel scan and one-thread scan
extern "C" int scan_par_host_wide(const uint8_t* src, int n, int cap, uint32_t* nSeqOut, uint32_t* marks, uint32_t markCap,
                                  int* stats, int nl)
{
    MemPtr<true, true> mem{src};
    return run_par(mem, n, cap, nSeqOut, marks, markCap, stats, nl);
}
extern "C" int scan_thread_host_wide(const uint8_t* src, int n, int cap, uint32_t* nSeqOut, uint32_t* marks, uint32_t markCap)
{
    MemPtr<true, true> mem{src};
    return scan_block(mem, n, cap, nSeqOut, marks, markCap);
}

// In-process differential fuzz: mutate a (valid) compressed block `iters` times, pick a capacity, and
// compare the parallel scan on nl lanes with the one-thread scan (return value, sequence count, marks).
// Returns the number of cases run, or -(1 + index) of the first mismatching case.
namespace {
struct FuzzRng { uint64_t s; uint32_t next() { s = s * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(s >> 33); } };
}
extern "C" long long scan_par_fuzz(const uint8_t* base, int n, int rawSize, int iters, uint64_t seed, long long* nErrors,
                                   int nl)
{
    FuzzRng r{seed * 0x9E3779B97F4A7C15ull + 1};
    uint8_t* buf = new uint8_t[(size_t)n + 64];
    uint32_t* m1 = new uint32_t[kMaxSeqFast];
    uint32_t* m2 = new uint32_t[kMaxSeqFast];
    long long cases = 0, errors = 0, bad = 0;
    for (int it = 0; it < iters && !bad; it++) {
        memset(buf, 0xEE, (size_t)n + 64);
        uint8_t* p = buf + 16 + (r.next() & 3);
        while (((uintptr_t)p & 3) != (uintptr_t)(it & 3)) p++;
        memcpy(p, base, (size_t)n);
        size_t len = (size_t)n;
        const int nm = it == 0 ? 0 : (int)(r.next() % 4);
        for (int k = 0; k < nm; k++) {
            const uint32_t mode = r.next() % 5;
            const size_t pos = r.next() % (len ? len : 1);
            if (mode == 0) p[pos] = (uint8_t)r.next();
            else if (mode == 1) { static const uint8_t v[6] = {0, 0xFF, 0xF0, 0x0F, 0x10, 0x1F}; p[pos] = v[r.next() % 6]; }
            else if (mode == 2 && len > 8) { const size_t d = 1 + r.next() % 3; if (pos + d < len) { memmove(p + pos, p + pos + d, len - pos - d); len -= d; } }
            else if (mode == 3 && len > 30) len = len - 1 - r.next() % 26;
            else p[pos] ^= (uint8_t)(1u << (r.next() & 7));
        }
        const int caps[6] = {rawSize, rawSize + 64, rawSize - 1, (int)(r.next() % (uint32_t)(rawSize + 5000)), rawSize + 1000, rawSize - 64};
        const int cap = caps[r.next() % 6];
        const bool wm = (len <= 65535 && cap <= 65536 && cap > 0);
        uint32_t ns1 = 0, ns2 = 0;
        int st[3];
        for (int i = 0; i < kMaxSeqFast; i++) { m1[i] = 0xABABABABu; m2[i] = 0xABABABABu; }
        MemPtr<true> memP{p};
        const int r1 = scan_block(memP, (int)len, cap, &ns1, wm ? m1 : nullptr, (uint32_t)kMaxSeqFast);
        const int r2 = scan_par_host(p, (int)len, cap, &ns2, wm ? m2 : nullptr, st, nl);
        const uint32_t k = ns1 < (uint32_t)kMaxSeqFast ? ns1 : (uint32_t)kMaxSeqFast;
        if (r1 != r2 || (r1 > 0 && ns1 != ns2) || (r1 > 0 && wm && memcmp(m1, m2, sizeof(uint32_t) * k) != 0)) bad = -(1 + (long long)it);
        cases++;
        errors += r1 < 0;
    }
    delete[] buf; delete[] m1; delete[] m2;
    *nErrors = errors;
    return bad ? bad : cases;
}
