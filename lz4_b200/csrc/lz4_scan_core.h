/*
 * lz4_scan_core.h -- the per-block scan of the decoder (acceptance + return value of
 * LZ4_decompress_safe, lz4.c:2022-2445) as plain C++ on plain pointers.
 *
 * Included by lz4_kernels.cu (inside its anonymous namespace), where it compiles for the device:
 * byte reads go through the read-only data cache (__ldg), the prefetch is a PTX prefetch.global.L1.
 * The same text also compiles for the host, which is how tests/ checks the scan's logic without a
 * GPU (tests/emul/): reads become plain loads, the prefetch disappears.  It is NOT a CPU path of
 * the product: nothing in the library calls it on the host.
 */
#ifndef LZ4_SCAN_CORE_H
#define LZ4_SCAN_CORE_H

#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define SC_FN __device__ __forceinline__
#define SC_MFN __device__ __forceinline__     /* member functions */
#define SC_MFN_COLD __device__ __noinline__     /* rare paths: kept out of the loops */
#define SC_DEV __device__
#define SC_LDG(p) __ldg(p)
#define SC_FUNNEL_R(lo, hi, s) __funnelshift_r((lo), (hi), (s))
#define SC_PREFETCH_L1(p) asm volatile("prefetch.global.L1 [%0];" ::"l"(p))
#else
#define SC_FN static inline
#define SC_MFN inline
#define SC_MFN_COLD inline
#define SC_DEV static inline
#define SC_LDG(p) (*(p))
static inline uint32_t sc_funnel_r_host(uint32_t lo, uint32_t hi, uint32_t s)
{
    s &= 31u;
    return s ? (lo >> s) | (hi << (32u - s)) : lo;
}
#define SC_FUNNEL_R(lo, hi, s) sc_funnel_r_host((lo), (hi), (s))
#define SC_PREFETCH_L1(p) ((void)(p))
#endif

#ifndef LZ4_SCAN_CORE_CONSTANTS
constexpr int kMinMatch = 4;
constexpr int kLastLiterals = 5;
constexpr int kMfLimit = 12;
#endif

/* ---------------------------------------------------------------------------------------------
 * How the scan reads the compressed block.  Every read goes through a "memory" object:
 *   MemPtr<true>   the block lies in GLOBAL memory (read-only data cache loads, L1 prefetch hints)
 *   MemPtr<false>  the block is staged in SHARED memory (plain loads through the generic address space)
 * b(i) / u16(i) / u32(i) read bytes [i, i+1/2/4) of the block.
 * ------------------------------------------------------------------------------------------- */
template <bool G> SC_FN uint32_t ldb(const uint8_t* p) { return G ? (uint32_t)SC_LDG(p) : (uint32_t)*p; }
template <bool G> SC_FN uint32_t ldw(const uint32_t* p) { return G ? SC_LDG(p) : *p; }
template <bool G> SC_FN uint32_t ld16(const uint8_t* p) { return ldb<G>(p) | (ldb<G>(p + 1) << 8); }

/* unaligned little-endian 32-bit read through two aligned words (never touches a word that holds
 * no requested byte) */
template <bool G> SC_FN uint32_t ld32u(const uint8_t* p)
{
    uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
    uint32_t sh = (uint32_t)(a & 3) * 8;
    uint32_t lo = ldw<G>(w);
    uint32_t hi = sh ? ldw<G>(w + 1) : 0u;
    return SC_FUNNEL_R(lo, hi, sh);
}

template <bool G, bool W = false> struct MemPtr {
    const uint8_t* p;
    SC_MFN uint32_t b(int64_t i) const { return ldb<G>(p + i); }
    SC_MFN uint32_t u16(int64_t i) const { return ld16<G>(p + i); }
    SC_MFN uint32_t u32(int64_t i) const { return ld32u<G>(p + i); }
    SC_MFN void prefetch(int64_t i) const { if (G) SC_PREFETCH_L1(p + i); }
    static constexpr bool kPrefetch = G;
    static constexpr bool kWide = W;            /* marks are two words per sequence (blocks above 64 KB): see mark_commit */
};

/* =============================================================================================
 * scan: exact acceptance + return value of LZ4_decompress_safe, one thread per block
 * ============================================================================================= */

/* lz4.c:1978-2014.  ip advances exactly like the reference's pointer so that the error code
 * -(ip)-1 (lz4.c:2443) is reproduced. */
template <class M> SC_FN bool read_runlength(M& mem, int64_t& ip, int64_t ilimit, bool initialCheck, int64_t& total)
{
    total = 0;
    if (initialCheck && ip >= ilimit) return false;
    uint32_t b;
    do {
        b = mem.b(ip);
        ip++;
        total += b;
        if (ip > ilimit) return false;
    } while (b == 255);
    return true;
}

/* Mark = (token position | output position of the sequence's MATCH << 16) of one sequence (for the last sequence,
 * which has no match: the end of its literals = the decoded size), written by the scan for every committed
 * sequence of a block that may go to the shared-memory expand kernel.  With the marks the expand kernel rebuilds
 * all sequence records of a block in parallel (one lane per sequence re-reads only its own token: literal
 * length, offset, match length) instead of re-walking the token chain.  16-bit fields: a value of 65 536 wraps
 * to 0, which only the last sequence of a 64 KB block can have. */
constexpr int kMaxSeqFast = 8192;              // most sequences a block of the shared-memory expand kernel may have
/* `markCap` = number of mark slots the caller reserved for this block (<= kMaxSeqFast); a block that can be
 * expanded from shared memory has at most capacity/4 + 1 sequences (every sequence but the last makes >= 4 bytes) */
/* Blocks above 64 KB (decoded in 60 KB output tiles by lz4_expand_tiles_kernel) get WIDE marks: two words per sequence,
 * {token position, match start}; the memory class of the walk says which (M::kWide). */
template <class M> SC_FN void mark_commit(uint32_t* marks, uint32_t markCap, uint32_t nseq, uint32_t tok, uint32_t matchStart)
{
    if (!marks || nseq >= markCap) return;
    if (M::kWide) { marks[2 * (size_t)nseq] = tok; marks[2 * (size_t)nseq + 1] = matchStart; }
    else marks[nseq] = tok | (matchStart << 16);
}

/* where the walk of one block stands between its two loops */
struct ScanState {
    int64_t ip, op, nextPrefetch;
    uint32_t nseq;
    bool fast;
};

/* ---- front loop: the fast-loop iterations of lz4.c:2083-2209 that stay in the fast loop ----
 * Same decisions as the byte-wise code of scan_tail, but kept to ~60 instructions per sequence: a
 * thread's time is the latency of its dependent instruction chain (32 threads = 32 different
 * blocks share a warp, a few warps per SM), so the chain is what is minimised: 32-bit state, two
 * dependent 4-byte reads per sequence (token + first length byte; offset + first match-length
 * byte).  Anything that would leave the fast loop (either end of the block getting close, an
 * error, absurd lengths) exits WITHOUT committing; the exact byte-wise code replays it.
 *
 * front_step parses the sequence whose token is at fip and applies the rules that depend on input positions only;
 * the three scans (scan_front here, the split and the parallel scan) add the rules that depend on the output position.
 * The lanes of a warp walk unrelated positions, so every data-dependent branch splits the warp and a walk's time is
 * (instructions issued per step, all paths of all lanes) x (latency of a dependent instruction).  The step is therefore
 * straight-line code for every sequence whose lengths need at most two extension bytes (literal runs < 525 bytes,
 * matches < 529); longer ones go round the reference's loops, which are skipped (condition false for every lane)
 * otherwise. */
struct FrontSeq {
    int ipn;                                    /* the next token's position */
    int lit, mlen;                              /* literal length, match length (kMinMatch included) */
    uint32_t off16;                             /* match offset */
    bool stop;                                  /* the front loop ends at fip (the other fields are then meaningless) */
};

/* `stop` is set for a reason that depends on input positions only, unless the caller passes `litCap`: then also when
 * the literal run ends past it (fop + lit > litCap: the output half of lz4.c:2104).  The capacity rule lz4.c:2137/2142,
 * which every scan applies, implies that rule, so only scan_front passes it: there the early exit skips the offset read
 * and the match-length loop, which keeps the one-thread scan kernel at fewer registers. */
template <class M> SC_FN FrontSeq front_step(M& mem, int nI, int fip, uint32_t fop = 0u, uint32_t litCap = 0xFFFFFFFFu)
{
    FrontSeq s = {fip, 0, 0, 0u, true};
    if (fip > nI - 26) return s;                               // lz4.c:2083 (the reads below stay inside the block)
    const uint32_t v = mem.u32(fip);                           // token, then the 3 bytes that follow it
    const int mcode = (int)(v & 15u), lit4 = (int)((v >> 4) & 15u);
    /* read_variable_length (lz4.c:2093), limit n-15: the first two extension bytes come with the token */
    const bool e1 = (lit4 == 15);
    const uint32_t l1 = (v >> 8) & 0xFFu, l2 = (v >> 16) & 0xFFu;
    const bool e2 = e1 && l1 == 255u;                          // (fip + 2 <= nI - 15 holds: fip <= nI - 26)
    int lit = lit4 + (e1 ? (int)l1 : 0) + (e2 ? (int)l2 : 0);
    int q = 1 + (e1 ? 1 : 0) + (e2 ? 1 : 0);
    uint32_t b = e2 ? l2 : l1;
    while (e1 && b == 255u && fip + q <= nI - 15 && lit < (1 << 28)) { b = mem.b(fip + q); q++; lit += (int)b; }
    /* read limit / absurd run, or literals ending within 32 bytes of the input end (lz4.c:2104 -> safe_literal_copy) */
    const bool stopL = e1 && (b == 255u || fip + q > nI - 15 || fop + (uint32_t)lit > litCap ||
                              (uint32_t)(fip + q) + (uint32_t)lit + 32u > (uint32_t)nI);   // (unsigned: sums may pass 2^31)
    const int offPos = fip + q + lit;
    const uint32_t v3 = mem.u32(stopL ? fip : offPos);         // offset (LE16), then the first two match-length bytes;
                                                               // a stopping step must not read at a wild position
    /* read_variable_length (lz4.c:2128), limit n-4 */
    const bool m1 = (mcode == 15);
    const uint32_t x1 = (v3 >> 16) & 0xFFu, x2 = v3 >> 24;
    const bool m2 = m1 && x1 == 255u && offPos + 3 <= nI - 4;
    int mlen = mcode + kMinMatch + (m1 ? (int)x1 : 0) + (m2 ? (int)x2 : 0);
    int ipn = offPos + 2 + (m1 ? 1 : 0) + (m2 ? 1 : 0);
    b = m2 ? x2 : x1;
    while (!stopL && m1 && b == 255u && ipn <= nI - 4 && mlen < (1 << 28)) { b = mem.b(ipn); ipn++; mlen += (int)b; }
    s.ipn = ipn; s.lit = lit; s.mlen = mlen; s.off16 = v3 & 0xFFFFu;
    s.stop = stopL || (m1 && (b == 255u || ipn > nI - 4));
    return s;
}

/* L1 prefetch hint, once per 128 input bytes of a walk over global memory */
template <class M> SC_FN void front_prefetch(M& mem, int nI, int fip, int& nextEvt)
{
    if (M::kPrefetch && fip >= nextEvt) {
        if (fip + 128 < nI) mem.prefetch(fip + 128);
        nextEvt = ((fip >> 7) + 1) << 7;
    }
}

/* Returns false for the one error it decides itself (offset before the start of the output, lz4.c:2161), with st.ip at
 * the reference's error position.  The exits are collected and taken once, in the reference's order. */
template <class M> SC_FN bool scan_front(M& mem, int nIn, int capIn, ScanState& st, uint32_t* marks, uint32_t markCap)
{
    uint32_t nseq = st.nseq;
    int fip = 0, fop = 0, nextEvt = 0;
    while (fip <= nIn - 26) {                                  // front_step tests it too; testing it first here, before
        front_prefetch(mem, nIn, fip, nextEvt);                // the prefetch, compiles to fewer registers
        const FrontSeq s = front_step(mem, nIn, fip, (uint32_t)fop, (uint32_t)(capIn - 32));
        const int opn = fop + s.lit;
        if (s.stop || (uint32_t)opn + (uint32_t)s.mlen >= (uint32_t)(capIn - 64)) break;   // lz4.c:2137/2142 -> safe_match_copy
        if ((int)s.off16 > opn) { st.ip = s.ipn; st.nseq = nseq; return false; }            // lz4.c:2161
        mark_commit<M>(marks, markCap, nseq, (uint32_t)fip, (uint32_t)opn);
        fip = s.ipn; fop = opn + s.mlen; nseq++;
    }
    st.ip = fip; st.op = fop; st.nseq = nseq;
    if (nextEvt > 0) st.nextPrefetch = (int64_t)nextEvt + 128;
    return true;
}

/* ---- the exact byte-wise walk (lz4.c:2083-2435) from the state `st` to the end of the block ---- */
template <class M> SC_FN int scan_tail(M& mem, int nIn, int capIn, const ScanState& st, uint32_t* nSeqOut, uint32_t* marks, uint32_t markCap)
{
    int64_t nextPrefetch = st.nextPrefetch;
    int64_t n = nIn, cap = capIn, ip = st.ip, op = st.op, ll = 0, ml = 0, add = 0, tokPos = 0, mop = 0;
    uint32_t token = 0, offset = 0, nseq = st.nseq;
    bool fast = st.fast;

    for (;;) {
        tokPos = ip;                                                   /* this sequence's token; mop = where its match starts */
        if (ip + 128 >= nextPrefetch) {                               // keep the input one 128-byte line ahead in L1
            if (ip + 128 < n) mem.prefetch(ip + 128);
            nextPrefetch = ip + 256;
        }
        token = mem.b(ip); ip++;
        ll = token >> 4;
        ml = token & 15;

        if (fast) {                                                    // lz4.c:2083-2209
            if (ll == 15) {
                if (!read_runlength(mem, ip, n - 15, true, add)) goto bad;
                ll += add;
                if (op + ll > cap - 32 || ip + ll > n - 32) { fast = false; goto safe_literals; }
            } else if (ip > n - 17) {
                fast = false; goto safe_literals;
            }
            ip += ll; op += ll; mop = op;
            offset = mem.u16(ip); ip += 2;
            if (ml == 15) {
                if (!read_runlength(mem, ip, n - 4, false, add)) goto bad;
                ml += add;
            }
            ml += kMinMatch;
            if (op + ml >= cap - 64) { fast = false; goto safe_match; }
            if ((int64_t)offset > op) goto bad;                        // lz4.c:2161
            mark_commit<M>(marks, markCap, nseq, (uint32_t)tokPos, (uint32_t)mop);
            op += ml; nseq++;
            continue;
        }

        /* safe loop, lz4.c:2215-2435 */
        if (ll != 15 && ip < n - 16 && op <= cap - 32) {               // two-stage shortcut :2230-2261
            op += ll; ip += ll; mop = op;
            offset = mem.u16(ip); ip += 2;
            if (ml != 15 && offset >= 8 && (int64_t)offset <= op) {
                mark_commit<M>(marks, markCap, nseq, (uint32_t)tokPos, (uint32_t)mop);
                op += ml + kMinMatch; nseq++;
                continue;
            }
            goto match_length;
        }
        if (ll == 15) {
            if (!read_runlength(mem, ip, n - 15, true, add)) goto bad;
            ll += add;
        }
safe_literals:
        if (op + ll > cap - kMfLimit || ip + ll > n - (2 + 1 + kLastLiterals)) {   // lz4.c:2279
            if (ip + ll != n || op + ll > cap) goto bad;               // lz4.c:2312
            op += ll;
            mark_commit<M>(marks, markCap, nseq, (uint32_t)tokPos, (uint32_t)op);   /* last sequence: the end of its literals */
            nseq++;
            *nSeqOut = nseq;
            return (int)op;                                            // lz4.c:2439
        }
        ip += ll; op += ll; mop = op;
        offset = mem.u16(ip); ip += 2;
match_length:
        if (ml == 15) {
            if (!read_runlength(mem, ip, n - 4, false, add)) goto bad;
            ml += add;
        }
        ml += kMinMatch;
safe_match:
        if ((int64_t)offset > op) goto bad;                            // lz4.c:2356
        if (op + ml > cap - kLastLiterals) goto bad;                   // lz4.c:2421-2423
        mark_commit<M>(marks, markCap, nseq, (uint32_t)tokPos, (uint32_t)mop);
        op += ml; nseq++;
    }
bad:
    *nSeqOut = 0;
    return (int)(-ip) - 1;                                             // lz4.c:2443
}

template <class M> SC_DEV int scan_block(M& mem, int nIn, int capIn, uint32_t* nSeqOut, uint32_t* marks, uint32_t markCap)
{
    ScanState st;
    st.ip = 0; st.op = 0; st.nextPrefetch = 128; st.nseq = 0;

    if (capIn < 0) return -1;                                          // lz4.c:2036
    if (capIn == 0) { if (nIn != 1) return -1; return mem.b(0) == 0 ? 0 : -1; }   // lz4.c:2064-2068
    if (nIn <= 0) return -1;                                           // lz4.c:2069
    st.fast = (capIn >= 64);                                           // lz4.c:2076

    if (st.fast && !scan_front(mem, nIn, capIn, st, marks, markCap)) {
        *nSeqOut = 0;
        return (int)(-st.ip) - 1;                                      // lz4.c:2443
    }
    return scan_tail(mem, nIn, capIn, st, nSeqOut, marks, markCap);
}

#endif /* LZ4_SCAN_CORE_H */
