// CPU emulator of the split scan (lz4_b200/csrc/lz4_scan_split.h): TEST INFRASTRUCTURE.
// Runs the lanes of a block phase by phase (the device puts a __syncwarp between phases) on the host build of the same
// header and returns what the kernel would store for the block.
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../lz4_b200/csrc/lz4_scan_split.h"

// stats[0] = 1 if the block fell back to the one-thread scan, [1] = steps walked in P2 (all lanes), [2] = lanes in the chain
extern "C" int scan_split_host(const uint8_t* src, int n, int cap, uint32_t* nSeqOut, uint32_t* marks, uint32_t markCap, int* stats)
{
    *nSeqOut = 0;
    stats[0] = stats[1] = stats[2] = 0;
    MemPtr<true> mem{src};
    if (!marks || cap < 64 || n < kSsMinBytes) return scan_block(mem, n, cap, nSeqOut, marks, markCap);
    const uint32_t R = markCap / kSsLanes;
    std::vector<uint32_t> A((size_t)kSsLanes * R + 1), B((size_t)kSsLanes * R + 1);
    static SsBlock S;
    memset(&S, 0, sizeof(S));
    for (int l = 0; l < kSsLanes; l++) ss_p1(l, S, mem, n, A.data() + (size_t)l * R, B.data() + (size_t)l * R, R);
    uint32_t before = 0;
    for (int l = 0; l < kSsLanes; l++) before += S.lane[l].cnt;
    for (int l = 0; l < kSsLanes; l++)
        ss_p2(l, S, mem, n, A.data() + (size_t)l * R, B.data() + (size_t)l * R, R, [&](int t) { return B.data() + (size_t)t * R; });
    uint32_t after = 0;
    for (int l = 0; l < kSsLanes; l++) after += S.lane[l].cnt;
    stats[1] = (int)(after - before);
    ss_p3(S, [&](int t) { return A.data() + (size_t)t * R; });
    if (S.fallback) { stats[0] = 1; return scan_block(mem, n, cap, nSeqOut, marks, markCap); }
    for (int l = 0; l < kSsLanes; l++) {
        uint32_t e, c, co;
        ss_p4(l, S, cap, A.data() + (size_t)l * R, B.data() + (size_t)l * R, marks, markCap, e, c, co);
        if (e < S.errIdx) S.errIdx = e;
        if (c < S.capIdx) { S.capIdx = c; S.capOpn = co; }
        stats[2] += S.lane[l].inChain;
    }
    return ss_p5(S, mem, n, cap, nSeqOut, marks, markCap);
}

// In-process differential fuzz: mutate a (valid) compressed block `iters` times, pick a capacity, and compare the split
// scan with the one-thread scan (return value, sequence count, marks).  Returns the number of cases run, or -(1 + index)
// of the first mismatching case.
namespace {
struct FuzzRng { uint64_t s; uint32_t next() { s = s * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(s >> 33); } };
}
extern "C" long long scan_split_fuzz(const uint8_t* base, int n, int rawSize, int iters, uint64_t seed, long long* nErrors, long long* nFallbacks)
{
    FuzzRng r{seed * 0x9E3779B97F4A7C15ull + 1};
    uint8_t* buf = new uint8_t[(size_t)n + 64];
    uint32_t* m1 = new uint32_t[kMaxSeqFast];
    uint32_t* m2 = new uint32_t[kMaxSeqFast];
    long long cases = 0, errors = 0, bad = 0, fb = 0;
    for (int it = 0; it < iters && !bad; it++) {
        memset(buf, 0xEE, (size_t)n + 64);
        uint8_t* p = buf + 16 + (r.next() & 3);
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
        const int caps[7] = {rawSize, rawSize + 64, rawSize - 1, (int)(r.next() % (uint32_t)(rawSize + 5000)), rawSize + 1000, rawSize - 64, 65536};
        int cap = caps[r.next() % 7];
        if (len > 65535 || cap > 65536 || cap <= 0) cap = rawSize <= 65536 ? rawSize : 65536;
        if (len > 65535) len = 65535;
        const uint32_t markCap = (uint32_t)cap / 4u + 2u < (uint32_t)kMaxSeqFast ? (uint32_t)cap / 4u + 2u : (uint32_t)kMaxSeqFast;
        uint32_t ns1 = 0, ns2 = 0;
        int st[3];
        for (int i = 0; i < kMaxSeqFast; i++) { m1[i] = 0xABABABABu; m2[i] = 0xABABABABu; }
        MemPtr<true> memP{p};
        const int r1 = scan_block(memP, (int)len, cap, &ns1, m1, markCap);
        const int r2 = scan_split_host(p, (int)len, cap, &ns2, m2, markCap, st);
        const uint32_t k = ns1 < markCap ? ns1 : markCap;
        if (r1 != r2 || (r1 > 0 && ns1 != ns2) || (r1 > 0 && memcmp(m1, m2, sizeof(uint32_t) * k) != 0)) bad = -(1 + (long long)it);
        cases++;
        errors += r1 < 0;
        fb += st[0];
    }
    delete[] buf; delete[] m1; delete[] m2;
    *nErrors = errors; *nFallbacks = fb;
    return bad ? bad : cases;
}
