/*
 * lz4_encode_par.cuh -- the PARALLEL-PARSE compressor: one CTA per block, every phase data-parallel.
 *
 * Included by lz4_kernels.cu.  Replaces, for throughput, the role of LZ4_compress_generic_validated
 * (lz4.c:930-1338) -- 4-byte hash table match finder + greedy parse -- with a formulation that has no
 * sequential walk over the block.  The output is a valid LZ4 block that round-trips exactly, it is
 * deterministic (no result depends on scheduling), but it is NOT byte-identical to the reference's output:
 * the parse differs (every position is a candidate, no skipping); the ratio is within 2 % of the
 * reference's at acceleration 1, usually above it (tests/test_gpu_parallel_compress.py; DESIGN.md 3.5).  The
 * byte-identical encoder (lz4_encode_kernel) remains behind LZ4_compress_default / LZ4_compress_fast and
 * LZ4B200_compress_blocks.
 *
 * A block of n <= 65 536 bytes is staged in shared memory by one TMA bulk load, then processed in WINDOWS
 * of 8192 positions; thread t of 512 owns the 16 consecutive positions 16t .. 16t+15 of the window (two CTAs share an
 * SM: 110 KB of shared memory each -- the block, one 8192-word table, the window's output -- so that one CTA's
 * barrier waits are the other's issue slots):
 *
 *   find    every position hashes its 4 bytes (Fibonacci hash, 13 bits: lz4.c:779).  The table word of a hash holds
 *           the LATEST position of an EARLIER window (low half) and the EARLIEST position of THIS window (high half,
 *           atomicMax on the complement of its index): both are scheduling-independent.  A position's
 *           candidate is, in this order: p-d if the 5 bytes at p repeat at distance d <= 4 (RLE-like data,
 *           where one table slot per hash cannot serve every position), this window's earliest position if it lies
 *           before p and its 4 bytes match, the earlier windows' latest.  One bit per position says "has a candidate".
 *   select  the reference's greedy rule -- the first position at or after the end of the previous match that
 *           has a candidate is taken, with its longest match (lz4.c:1014-1100, 1182) -- evaluated by all lanes at
 *           once: every lane walks its 16 positions as if the chain entered at its first position, a CTA-wide
 *           "last valid value" scan hands every lane the end of the last match selected before it, lanes whose
 *           search would start elsewhere walk again, until nothing changes.  Only SELECTED positions extend their
 *           match (4 bytes per step, by the lane alone), so the total comparison work is O(block size).
 *   emit    backward extension (lz4.c:1107-1109), sizes, CTA-wide exclusive sum; every lane writes the headers of its
 *           sequences, the literals are copied position-parallel (every lane stores those of its 16 positions that are
 *           literals); a window's output is assembled in shared memory and written out in aligned 16-byte pieces
 *           (scattered byte stores to HBM cost a transaction each).
 *   insert  the window's positions enter the low halves (atomicMax, after the high halves are cleared).
 *
 * The end-of-block rules of the format are the reference's: no match starts after n-12, the last 5 bytes
 * are literals (lz4.c:963-964, 1233); output that does not fit dstCapacity makes the call return 0.
 * `acceleration` > 4 thins the candidate positions (every `step`-th position is hashed / inserted).
 */
#pragma once

constexpr int kEpThreads = 512;                      /* two CTAs per SM: one CTA's barrier waits are the other's issue slots */
constexpr int kEpWarps = kEpThreads / 32;
constexpr int kEpPer = 16;                           /* positions per thread and window */
constexpr int kEpWin = kEpThreads * kEpPer;          /* 8192 positions per window */
constexpr int kEpHashLog = 13;
constexpr int kEpMaxSel = kEpPer / 4;                /* matches are >= 4 long: at most 4 selections per lane */
constexpr int kEpSolo = 32;                          /* a match at least this long (> kEpPer: it ends its lane's walk) is remembered across walks */
constexpr int kEpStage = kEpWin + 512;               /* a window's output is assembled here when it fits (it does unless literals of earlier windows come with it) */

struct EncParSmem {
    alignas(16) uint8_t pad[16];                     /* the 4 bytes "before" position 0 are read (never used) */
    alignas(16) uint8_t src[65536 + 64];             /* staged block (keeps the source's 16-byte phase) */
    /* per hash, one word: low half = latest position + 1 of an EARLIER window (0: none); high half = 0xFFFF - index in
     * window of the EARLIEST position of THIS window (0: none; cleared after every window).  Both are maxima, so one native
     * atomicMax serves each: the high half is raised with the low half carried along unchanged (it is stable while
     * positions are being published), the low half while every high half is zero. */
    alignas(16) uint32_t TT[1 << kEpHashLog];
    alignas(16) uint8_t stage[kEpStage];
    uint32_t carry[3];                               /* literals of EARLIER windows that the window's first sequence carries: {source position, output offset, length} */
    int warpFirst[kEpWarps][2];                      /* emit: {start, output offset - position of its literals (relative to the warp's output)} of the warp's first sequence */
    int warpLast[kEpWarps];                          /* chain scan: end of the last match selected in each warp, or -1 */
    uint32_t warpSum[kEpWarps];
    uint32_t E, O, fail;
    alignas(8) uint64_t mbar;
};
static_assert(sizeof(EncParSmem) <= (232448 - 2048) / 2, "two CTAs of the parallel compressor must fit one SM");

__device__ __forceinline__ uint32_t ep_ld32(const uint8_t* base, uint32_t i)      /* unaligned 4 bytes at base + i (base 4-aligned) */
{
    const uint32_t* w = reinterpret_cast<const uint32_t*>(base) + (i >> 2);
    const uint32_t sh = (i & 3u) * 8u;
    return __funnelshift_r(w[0], sh ? w[1] : 0u, sh);
}
__device__ __forceinline__ uint32_t ep_hash(uint32_t v) { return (v * 2654435761u) >> (32 - kEpHashLog); }
__device__ __forceinline__ uint32_t ep_runlen_bytes(uint32_t x) { return x >= 15u ? 1u + (x - 15u) / 255u : 0u; }

/* the 16 + 4 + 4 bytes around a lane's positions as 4-byte values: val(i) = the 4 bytes at position p0 + i, i in [-4, 16] */
struct EpBytes {
    uint32_t B[7];                                   /* B[j] = bytes p0 - 4 + 4j .. +3 */
    __device__ __forceinline__ void load(const uint8_t* ptr)          /* ptr = address of byte p0 - 4 */
    {
        const uintptr_t u = reinterpret_cast<uintptr_t>(ptr);
        const uint32_t* wp = reinterpret_cast<const uint32_t*>(u & ~uintptr_t(3));
        const uint32_t sh = (uint32_t)(u & 3u) * 8u;
        uint32_t W[8];
        #pragma unroll
        for (int j = 0; j < 8; j++) W[j] = wp[j];
        #pragma unroll
        for (int j = 0; j < 7; j++) B[j] = __funnelshift_r(W[j], W[j + 1], sh);
    }
    __device__ __forceinline__ uint32_t val(int i) const          /* i in [-4, 15], compile-time after unrolling */
    {
        const int o = i + 4;
        return __funnelshift_r(B[o >> 2], B[(o >> 2) + 1], (uint32_t)((o & 3) * 8));
    }
};

/* Where a position's candidate comes from, 4 bits per position (0: none): 1..4 = p - d (short-period rule), kEpKindWin = this
 * window's earliest position with the hash, kEpKindOld = the earlier windows' latest.  find 2 verifies and records the kind;
 * select turns the kind of the few SELECTED positions back into a position (the table does not change in between). */
constexpr uint32_t kEpKindWin = 5, kEpKindOld = 6;
__device__ __forceinline__ uint32_t ep_table_kind(const EncParSmem& S, const uint8_t* src, int head, int p, int c0, uint32_t v)
{
    const uint32_t tt = S.TT[ep_hash(v)];
    const uint32_t e = tt >> 16;
    const int q = c0 + (0xFFFF - (int)e);                                          /* earliest position of this window with this hash */
    if (e && q < p && ep_ld32(src, (uint32_t)(head + q)) == v) return kEpKindWin;
    const uint32_t o = tt & 0xFFFFu;
    if (o && ep_ld32(src, (uint32_t)head + o - 1u) == v) return kEpKindOld;
    return 0u;
}
__device__ __forceinline__ uint32_t ep_candidate_of_kind(const EncParSmem& S, const uint8_t* src, int head, int p, int c0, uint32_t kind)
{
    if (kind <= 4u) return (uint32_t)p - kind;
    const uint32_t tt = S.TT[ep_hash(ep_ld32(src, (uint32_t)(head + p)))];
    return kind == kEpKindWin ? (uint32_t)(c0 + 0xFFFF) - (tt >> 16) : (tt & 0xFFFFu) - 1u;
}

/* length of the match (p, c), both block positions, at most `limit` (>= 4): two word streams, 4 bytes per step.
 * A lane extends its match ALONE, however long.  A warp-cooperative finish of long matches (128 bytes per step through
 * ballots) is faster, but under compute-sanitizer the instrumented loads inside its loop split the warp while the
 * compiler, having proved the warp converged, emits bare VOTE / SHFL and a loop counter in a uniform register: the
 * ballots see partial warps and matches come out too long.  A kernel the sanitizer cannot check is not kept. */
__device__ __forceinline__ int ep_extend(const uint8_t* src, int head, int p, uint32_t c, int limit)
{
    const uint32_t pa = (uint32_t)(head + p) + 4u, ca = (uint32_t)head + c + 4u;
    const uint32_t* wa = reinterpret_cast<const uint32_t*>(src) + (pa >> 2);
    const uint32_t* wb = reinterpret_cast<const uint32_t*>(src) + (ca >> 2);
    const uint32_t sa = (pa & 3u) * 8u, sb = (ca & 3u) * 8u;
    uint32_t a0 = wa[0], b0 = wb[0];
    int L = 4;
    while (L < limit) {
        const uint32_t a1 = wa[1], b1 = wb[1];
        const uint32_t x = __funnelshift_r(a0, a1, sa) ^ __funnelshift_r(b0, b1, sb);
        if (x) { L += (__ffs(x) - 1) >> 3; break; }
        a0 = a1; b0 = b1; wa++; wb++; L += 4;
    }
    return L > limit ? limit : L;
}

__global__ void __launch_bounds__(kEpThreads, 2) lz4_encode_par_kernel(lz4k_encode_args a)
{
    extern __shared__ __align__(16) uint8_t smemRaw[];
    EncParSmem& S = *reinterpret_cast<EncParSmem*>(smemRaw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t parity = 0;
    const int accel = a.acceleration < 1 ? 1 : (a.acceleration > kAccelMax ? kAccelMax : a.acceleration);
    const int step = accel <= 4 ? 1 : 1 + (accel + 3) / 8;       /* every position for acceleration 1..4, then every 2nd (5..12), 3rd (13..20), ... */
    if (tid == 0) mbar_init(&S.mbar, 1);
    __syncthreads();
#ifdef LZ4K_PHASE_TIMING
    long long tPhase = clock64();
#endif

    for (int64_t b = blockIdx.x; b < a.nBlocks; b += gridDim.x) {
        const int n = a.srcSizeArr ? a.srcSizeArr[b] : a.srcSize;
        if (n < a.minSize || n > a.maxSize) continue;                 /* another launch's block */
        const uint8_t* gsrc = enc_src(a, b);
        uint8_t* dst = enc_dst(a, b);
        const int64_t cap = enc_cap(a, b);
        if (n <= 0 || n > 65536) {                                    /* n == 0: one token byte (lz4.c:1361-1371); larger blocks are not this kernel's */
            if (tid == 0) { int r = 0; if (n == 0 && cap >= 1) { dst[0] = 0; r = 1; } a.outSize[b] = r; }
            continue;
        }
        const int head = tma_stage(S.src, gsrc, n, &S.mbar, tid == 0);
        if (tid == 0) { S.E = 0; S.O = 0; S.fail = 0; S.carry[2] = 0; }
        for (int k = tid; k < (1 << kEpHashLog) / 4; k += kEpThreads) reinterpret_cast<uint4*>(S.TT)[k] = make_uint4(0, 0, 0, 0);
        __syncthreads();
        mbar_wait(&S.mbar, parity);
        parity ^= 1;
        const uint8_t* src = S.src;                                   /* byte i of the block = src[head + i] */
        const int mflimit = n - kMfLimit, matchlimit = n - kLastLiterals;
        const int nWin = (n >= kMinLength) ? (mflimit + kEpWin) / kEpWin : 0;      /* windows that hold positions <= mflimit */
        PHASE_MARK(6);                                     // load + tables

        for (int w = 0; w < nWin; w++) {
            const int c0 = w * kEpWin, i0 = kEpPer * tid, p0 = c0 + i0;
            const int cnt = min(kEpPer, mflimit + 1 - p0);               /* this lane's positions: p0 .. p0 + cnt - 1 (cnt may be <= 0) */
            EpBytes by;
            if (cnt > 0) by.load(src + head + p0 - 4);
            /* ---------------- find 1: publish the earliest position of this window per hash ---------------- */
            #pragma unroll
            for (int i = 0; i < kEpPer; i++)
                if (i < cnt && (step == 1 || (p0 + i) % step == 0))
                {
                    uint32_t* cell = &S.TT[ep_hash(by.val(i))];
                    atomicMax(cell, ((uint32_t)(0xFFFF - (i0 + i)) << 16) | (*cell & 0xFFFFu));
                }
            __syncthreads();
            PHASE_MARK(0);                                     // find 1
            /* ---------------- find 2: which positions have a candidate ---------------- */
            uint32_t has = 0;
            uint64_t kinds = 0;
            #pragma unroll
            for (int i = 0; i < kEpPer; i++) {
                if (i < cnt && (step == 1 || (p0 + i) % step == 0)) {
                    const int p = p0 + i;
                    const uint32_t v = by.val(i);
                    uint32_t kind = 0;
                    #pragma unroll
                    for (int d = 1; d <= 4; d++)                     /* a run of period d <= 4: the 5 bytes at p repeat at p - d */
                        if (!kind && p >= d && by.val(i - d) == v && ((by.val(i + 1) ^ by.val(i + 1 - d)) >> 24) == 0u) kind = (uint32_t)d;
                    if (!kind) kind = ep_table_kind(S, src, head, p, c0, v);
                    if (kind) { has |= 1u << i; kinds |= (uint64_t)kind << (4 * i); }
                }
            }
            PHASE_MARK(1);                                     // find 2
            /* ---------------- select: the greedy chain through this window, all lanes ---------------- */
            const int Ein = (int)S.E;
            int eCur = Ein, exitE = Ein, nSel = 0;
            int sPos[kEpMaxSel], sLen[kEpMaxSel], sLit[kEpMaxSel];
            uint32_t sCand[kEpMaxSel];
            int cacheP = -1, cacheL = 0;                               /* the last long match this lane extended (walks repeat) */
            uint32_t cacheC = 0;
            /* One walk of every lane that `go`es: the lane's positions from the chain position e.  A match of kEpSolo bytes or more
             * covers the rest of the lane's 16 positions (it is the lane's LAST selection); its length is remembered, because the
             * lane may walk again from another entry and meet it again. */
            auto walk = [&](bool go, int e) {
                if (go) {
                    nSel = 0;
                    int rel = max(e - p0, 0);
                    #pragma unroll
                    for (int k = 0; k < kEpMaxSel; k++) {
                        const uint32_t m = rel < kEpPer ? (has >> rel) : 0u;
                        if (m != 0u) {
                            rel += __ffs(m) - 1;
                            const int p = p0 + rel;
                            uint32_t c; int L;
                            if (p == cacheP) { c = cacheC; L = cacheL; }
                            else {
                                const int limit = matchlimit - p;
                                c = ep_candidate_of_kind(S, src, head, p, c0, (uint32_t)(kinds >> (4 * rel)) & 15u);
                                L = ep_extend(src, head, p, c, limit);           /* alone, whatever the length: see ep_extend */
                                if (L >= kEpSolo) { cacheP = p; cacheC = c; cacheL = L; }      /* a long one is remembered */
                            }
                            sPos[k] = p; sCand[k] = c; sLen[k] = L; sLit[k] = e;
                            nSel = k + 1;
                            e = p + L;
                            rel = e - p0;
                        }
                    }
                    exitE = e;
                }
            };
            walk(true, eCur);
#ifdef LZ4K_PHASE_TIMING
            unsigned statRounds = 0, statWalks = 1;
#endif
            /* Two levels of rounds.  Inside a warp the chain is settled with shuffles alone (no CTA barrier): given the position the
             * chain enters the WARP at, every lane takes the end of the last match selected before it and walks again if its search
             * would start elsewhere.  Across warps one barrier per round hands every warp the end of the last match selected in the
             * warps before it; a warp whose entry moved settles again.  The chain usually re-synchronises within a warp's 512
             * positions, so two CTA rounds are the rule. */
            int warpEntry = Ein;
            for (;;) {
                int val;
                for (;;) {
                    /* end of the last match selected at or before this lane (lanes that select nothing pass the chain through) */
                    val = nSel ? exitE : -1;
                    #pragma unroll
                    for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(kFull, val, d); if (lane >= d && val < 0) val = y; }
                    int prev = __shfl_up_sync(kFull, val, 1);            /* ... at or before the previous lane */
                    if (lane == 0) prev = -1;
                    const int eNew = prev < 0 ? warpEntry : prev;
                    const bool need = max(eNew - p0, 0) != max(eCur - p0, 0);      /* the search would start elsewhere */
                    eCur = eNew;
                    if (!__any_sync(kFull, need)) break;
#ifdef LZ4K_PHASE_TIMING
                    statWalks += need ? 1u : 0u;
#endif
                    walk(need, eNew);
                }
                if (lane == 31) S.warpLast[warp] = val;
                __syncthreads();
                int carry = -1;                                         /* ... in the warps before this one */
                for (int q = warp - 1; q >= 0; q--) { const int x = S.warpLast[q]; if (x >= 0) { carry = x; break; } }
                const int entry = carry < 0 ? Ein : carry;
                const int w0 = c0 + kEpPer * 32 * warp;                  /* the warp's first position */
                const bool moved = max(entry - w0, 0) != max(warpEntry - w0, 0);
                warpEntry = entry;
                if (!__syncthreads_or(moved ? 1 : 0)) break;
#ifdef LZ4K_PHASE_TIMING
                statRounds++;
#endif
            }
            {
                /* the true position the chain enters this lane at (an entry below the lane's first position was not propagated) */
                int val = nSel ? exitE : -1;
                #pragma unroll
                for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(kFull, val, d); if (lane >= d && val < 0) val = y; }
                int prev = __shfl_up_sync(kFull, val, 1);
                if (lane == 0) prev = -1;
                eCur = prev < 0 ? warpEntry : prev;
            }
#ifdef LZ4K_PHASE_TIMING
            if (tid == 0) atomicAdd(&g_loopStats[0], (unsigned long long)statRounds);
            atomicAdd(&g_loopStats[1], (unsigned long long)statWalks);
            if (tid == 0) atomicAdd(&g_loopStats[3], 1ull);
#endif
            if (nSel) sLit[0] = eCur;                                     /* the first one's literals start at the true entry */
            if (tid == kEpThreads - 1) {                                 /* the chain's position after this window */
                int last = nSel ? exitE : -1;
                for (int q = kEpWarps - 1; q >= 0 && last < 0; q--) last = S.warpLast[q];
                S.E = (uint32_t)(last < 0 ? Ein : last);
            }
            PHASE_MARK(4);                                     // select
            /* ---------------- emit ----------------
             * Every selection's sequence header (token, length bytes, offset, length bytes) is written by its lane; the LITERALS are
             * copied position-parallel: every lane stores those of its own 16 positions that are literals, at (position + D) where D
             * is constant per literal run -- the run belongs to the next sequence at or after the position, which a suffix scan
             * ("first sequence to the right") hands to the lanes that select nothing.  Only the literals that the window's first
             * sequence brings along from EARLIER windows have no owner lane: the whole CTA copies them. */
            {
                uint32_t size = 0, hdr0 = 0;
                #pragma unroll
                for (int k = 0; k < kEpMaxSel; k++) {
                    if (k < nSel) {
                        int p = sPos[k], L = sLen[k];
                        const int A = sLit[k];
                        uint32_t c = sCand[k];
                        while (p > A && c > 0u && src[head + p - 1] == src[head + c - 1u]) { p--; c--; L++; }      /* lz4.c:1107-1109 */
                        sPos[k] = p; sLen[k] = L; sCand[k] = c;
                        const uint32_t h = 1u + ep_runlen_bytes((uint32_t)(p - A));
                        if (k == 0) hdr0 = h;
                        size += h + (uint32_t)(p - A) + 2u + ep_runlen_bytes((uint32_t)(L - kMinMatch));
                    }
                }
                uint32_t incl = size;
                #pragma unroll
                for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(kFull, incl, d); if (lane >= d) incl += y; }
                /* first sequence at or after this lane: {start, D relative to the warp's first output byte} */
                int nStart = nSel ? sPos[0] : -1;
                int nD = nSel ? (int)(incl - size + hdr0) - sLit[0] : 0;
                #pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const int y = __shfl_down_sync(kFull, nStart, d), z = __shfl_down_sync(kFull, nD, d);
                    if (lane + d < 32 && nStart < 0) { nStart = y; nD = z; }
                }
                if (lane == 31) S.warpSum[warp] = incl;
                if (lane == 0) { S.warpFirst[warp][0] = nStart; S.warpFirst[warp][1] = nD; }
                int xStart = __shfl_down_sync(kFull, nStart, 1), xD = __shfl_down_sync(kFull, nD, 1);     /* ... strictly after this lane */
                if (lane == 31) xStart = -1;
                __syncthreads();
                const uint32_t O0 = S.O;
                uint32_t base = O0, winTotal = 0;
                for (int q = 0; q < kEpWarps; q++) { const uint32_t x = S.warpSum[q]; winTotal += x; if (q < warp) base += x; }
                if (xStart >= 0) xD += (int)base;
                else {
                    uint32_t bq = base + S.warpSum[warp];
                    for (int q = warp + 1; q < kEpWarps; q++) {
                        const int st = S.warpFirst[q][0];
                        if (st >= 0) { xStart = st; xD = S.warpFirst[q][1] + (int)bq; break; }
                        bq += S.warpSum[q];
                    }
                }
                /* (a window's output can exceed its 8192 positions: its first sequence carries the literals of earlier windows) */
                const bool staged = winTotal + 16u <= (uint32_t)kEpStage;
                const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(dst + O0) & 15u);   /* stage keeps the 16-byte phase of the destination */
                uint8_t* const obase = staged ? S.stage + mis - O0 : dst;       /* output offset o lives at obase + o */
                const int64_t lim = staged ? (int64_t)1 << 40 : cap;            /* direct stores must stay below the capacity */
                int64_t o = (int64_t)base + incl - size;
                uint32_t lm[kEpMaxSel + 1];                                      /* literal positions of this lane, per run: bit i = position p0 + i */
                int lD[kEpMaxSel + 1];
                auto range = [&](int from, int to) -> uint32_t {                 /* bits of the own positions in [from, to) */
                    const int lo = min(max(from - p0, 0), kEpPer), hi = min(max(to - p0, 0), kEpPer);
                    return hi > lo ? ((1u << hi) - 1u) & ~((1u << lo) - 1u) : 0u;
                };
                const bool fits = o + size <= cap;
                if (size && !fits) S.fail = 1;
                #pragma unroll
                for (int k = 0; k < kEpMaxSel; k++) {
                    lm[k] = 0; lD[k] = 0;
                    if (k < nSel && fits) {
                        uint8_t* d = obase + o;
                        const int ll = sPos[k] - sLit[k];
                        const uint32_t ml = (uint32_t)(sLen[k] - kMinMatch);
                        *d++ = (uint8_t)((min((uint32_t)ll, 15u) << 4) | min(ml, 15u));
                        if (ll >= 15) { uint32_t r = (uint32_t)ll - 15u; while (r >= 255u) { *d++ = 255; r -= 255u; } *d++ = (uint8_t)r; }
                        const uint32_t litDst = (uint32_t)(d - obase);
                        lD[k] = (int)litDst - sLit[k];
                        lm[k] = range(sLit[k], sPos[k]);
                        if (sLit[k] < c0) { S.carry[0] = (uint32_t)sLit[k]; S.carry[1] = litDst; S.carry[2] = (uint32_t)(min(c0, sPos[k]) - sLit[k]); }
                        d += ll;
                        const uint32_t off = (uint32_t)sPos[k] - sCand[k];
                        *d++ = (uint8_t)off; *d++ = (uint8_t)(off >> 8);
                        if (ml >= 15u) { uint32_t r = ml - 15u; while (r >= 255u) { *d++ = 255; r -= 255u; } *d++ = (uint8_t)r; }
                        o = d - obase;
                    }
                }
                /* the positions after this lane's last match (or after the match that covers its start) up to the next sequence */
                lm[kEpMaxSel] = xStart >= 0 ? range(nSel ? exitE : eCur, xStart) : 0u;
                lD[kEpMaxSel] = xD;
                {
                    uint32_t any = lm[kEpMaxSel];
                    #pragma unroll
                    for (int k = 0; k < kEpMaxSel; k++) any |= lm[k];
                    #pragma unroll
                    for (int i = 0; i < kEpPer; i++) {
                        if ((any >> i) & 1u) {
                            int D = lD[kEpMaxSel];
                            #pragma unroll
                            for (int k = kEpMaxSel - 1; k >= 0; k--) if ((lm[k] >> i) & 1u) D = lD[k];
                            const int64_t at = (int64_t)(p0 + i) + D;
                            if (at < lim) obase[at] = (uint8_t)by.val(i);
                        }
                    }
                }
                __syncthreads();
                if (tid == 0) S.O = O0 + winTotal;
                {
                    const uint32_t from = S.carry[0], to = S.carry[1], cntL = S.carry[2];
                    for (uint32_t i = tid; i < cntL; i += kEpThreads) if ((int64_t)to + i < lim) obase[to + i] = src[head + from + i];
                }
                /* this window's "earliest position" halves are done with */
                for (int k = tid; k < (1 << kEpHashLog) / 4; k += kEpThreads) {
                    uint4 t = reinterpret_cast<uint4*>(S.TT)[k];
                    t.x &= 0xFFFFu; t.y &= 0xFFFFu; t.z &= 0xFFFFu; t.w &= 0xFFFFu;
                    reinterpret_cast<uint4*>(S.TT)[k] = t;
                }
                __syncthreads();
                /* ---------------- insert: this window's positions enter the low halves ---------------- */
                #pragma unroll
                for (int i = 0; i < kEpPer; i++)
                    if (i < cnt && (step == 1 || (p0 + i) % step == 0))
                        atomicMax(&S.TT[ep_hash(by.val(i))], (uint32_t)(p0 + i) + 1u);
                /* write the window out in aligned 16-byte pieces */
                {
                    const bool put = staged && !S.fail;
                    uint8_t* const gbase = dst + O0 - mis;                        /* 16-byte aligned; stage byte i belongs at gbase + i */
                    const uint32_t nChunk = put ? (mis + winTotal + 15u) / 16u : 0u;
                    for (uint32_t c = tid; c < nChunk; c += kEpThreads) {
                        const uint4 v = reinterpret_cast<const uint4*>(S.stage)[c];
                        const uint32_t lo = c * 16u;
                        if (lo + 16u > mis) {
                            if (lo >= mis && lo + 16u <= mis + winTotal) *reinterpret_cast<uint4*>(gbase + lo) = v;
                            else {
                                const uint32_t wv[4] = {v.x, v.y, v.z, v.w};
                                #pragma unroll
                                for (uint32_t i = 0; i < 16u; i++)
                                    if (lo + i >= mis && lo + i < mis + winTotal) gbase[lo + i] = (uint8_t)(wv[i >> 2] >> ((i & 3u) * 8u));
                            }
                        }
                    }
                }
                if (tid == 0) S.carry[2] = 0;
                __syncthreads();
                PHASE_MARK(5);                                 // emit + insert
            }
        }
        /* ---------------- last literals (lz4.c:1302-1329) ---------------- */
        {
            const uint32_t E = S.E, O = S.O;
            const uint32_t last = (uint32_t)n - E;
            const int64_t total = (int64_t)O + 1 + ep_runlen_bytes(last) + last;
            const bool ok = !S.fail && total <= cap;
            if (ok) {
                uint8_t* d = dst + O;
                const uint32_t skip = 1u + ep_runlen_bytes(last);
                if (tid == 0) {
                    *d++ = (uint8_t)(min(last, 15u) << 4);
                    if (last >= 15u) { uint32_t r = last - 15u; while (r >= 255u) { *d++ = 255; r -= 255u; } *d++ = (uint8_t)r; }
                }
                for (uint32_t i = tid; i < last; i += kEpThreads) dst[O + skip + i] = src[head + E + i];
            }
            if (tid == 0) a.outSize[b] = ok ? (int32_t)total : 0;
        }
        __syncthreads();                                               /* S is reused by the next block */
        PHASE_MARK(2);                                     // last literals
    }
}
