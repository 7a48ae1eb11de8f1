/*
 * lz4_rows_core.h -- the arithmetic of the "rows" expand kernel (lz4_kernels.cu: lz4_expand_rows_kernel)
 * as plain C++ on plain arrays, so that the same text runs on the device and, for tests/, on the host
 * (tests/emul/rows_emul.cpp replays the kernel phase by phase, one "thread" after the other).
 * It is NOT a CPU path of the product: nothing in the library calls it on the host.
 *
 * Formulation (DESIGN.md section 3.2).  A decoded block is a concatenation of RUNS: the literal run
 * and the match run of every sequence (lz4.c:2083-2435 produces them one after the other).  Inside one
 * run every output byte p comes from the byte at a constant distance:
 *
 *        out[p] = window[A_out + p + delta(run)]
 *
 * where `window` is the CTA's shared memory seen as one byte array that holds the staged compressed
 * block (`in`) BELOW the output window (`out`), so that a literal run is just a run with a large
 * negative delta (into `in`) and a match run has delta = -offset (into `out`).  One bit per run start
 * in a 64 Kbit map indexed by output position plus one running count per 32-byte ROW turn "which run
 * covers byte p" into   j = rows[p/32].base + popc(rows[p/32].bits & lanemask_le)   -- for the 32
 * lanes of a warp working on the 32 bytes of one row the two loads are uniform.  The output is
 * produced one byte per thread, in WAVES of kWave consecutive bytes separated by a CTA barrier: a
 * source below the current wave is final; a source inside the current wave is not read but FOLLOWED
 * (the source byte's own run and delta are looked up, "hop"), which terminates because every hop moves
 * strictly backwards and literal runs end the chain.  There are no done flags, no spinning and no
 * per-piece control flow: every lane of every warp executes the same ~14 instructions per byte row.
 *
 * Self-overlapping matches (offset < length, lz4.c:2379-2420) are cut into pieces at
 * m + offset*2^t whose deltas are multiples of the offset (bytes of such a match are periodic), so a
 * byte of an RLE-style match reaches a byte before the match start in O(log(length/offset)) hops.
 * Offset 0 (which the reference decodes to zero bytes, lz4.c:2407,:500) becomes one byte read from an
 * always-zero cell followed by an offset-1 periodic run.
 */
#ifndef LZ4_ROWS_CORE_H
#define LZ4_ROWS_CORE_H

#include <stdint.h>

#if defined(__CUDACC__)
#define RW_FN __device__ __forceinline__
#define RW_POPC(x) __popc(x)
#else
#define RW_FN static inline
#define RW_POPC(x) __builtin_popcount(x)
struct uint2 { uint32_t x, y; };
#endif

constexpr int kRowsMaxRuns = 20480;            /* run table of the rows kernel (u32 per run) */

/* one sequence as the rows kernel sees it */
struct RwSeq {
    int op;        /* first output byte of the sequence (= start of its literal run) */
    int ll;        /* literal length */
    int ls;        /* position of the first literal byte in the compressed block */
    int m;         /* first output byte of the match run */
    int mlen;      /* match length (0: the last sequence has no match) */
    int off;       /* match offset */
};

/* Sequence k from the scan's mark (token position | match start << 16, lz4_scan_core.h): the lane re-reads only its
 * own token -- literal length incl. extension bytes (lz4.c:1978-2014), the offset and the match length; the last
 * sequence has no match and its mark holds the end of its literals.
 * PARTIAL (LZ4_decompress_safe_partial, lz4_scan_core.h: scan_tail): the last sequence's mark holds the START of its
 * literals and the decode ended at `total`, so its literal run is min(token's length, total - start) bytes and, if the
 * token's literals end before `total`, a match at their end fills the rest.  The match length comes from `total`, not
 * from the token: the only input bytes read are the ones the scan read. */
template <bool PARTIAL = false>
RW_FN RwSeq rw_parse(const uint8_t* in, uint32_t mk, int k, bool last, int total = 0)
{
    RwSeq s;
    if (PARTIAL && last) {
        const int tok = (int)(mk & 0xFFFFu);
        int st = (int)(mk >> 16);
        if (k != 0 && st == 0) st = 65536;             /* 16-bit wrap: a final token without bytes at 65536 */
        const uint32_t t = in[tok];
        int pp = tok + 1;
        int ll = (int)(t >> 4);
        if (ll == 15) { uint32_t x; do { x = in[pp++]; ll += (int)x; } while (x == 255); }
        s.ls = pp; s.op = st;
        s.ll = ll < total - st ? ll : total - st;
        s.m = st + s.ll;
        s.off = 0; s.mlen = 0;
        if (s.ll == ll && s.m < total) {
            pp += ll;
            s.off = (int)((uint32_t)in[pp] | ((uint32_t)in[pp + 1] << 8));
            s.mlen = total - s.m;
        }
        return s;
    }
    const int tok = (int)(mk & 0xFFFFu);
    int m = (int)(mk >> 16);
    if (k != 0 && m == 0) m = 65536;                   /* 16-bit wrap: only the last sequence of a 64 KB block ends at 65536 */
    const uint32_t t = in[tok];
    int pp = tok + 1;
    int ll = (int)(t >> 4);
    if (ll == 15) { uint32_t x; do { x = in[pp++]; ll += (int)x; } while (x == 255); }
    s.ll = ll; s.ls = pp; s.m = m; s.op = m - ll;
    s.off = 0; s.mlen = 0;
    if (!last) {
        pp += ll;
        s.off = (int)((uint32_t)in[pp] | ((uint32_t)in[pp + 1] << 8));
        pp += 2;
        int ml = (int)(t & 15u);
        if (ml == 15) { uint32_t x; do { x = in[pp++]; ml += (int)x; } while (x == 255); }
        s.mlen = ml + 4;
    }
    return s;
}

/* The same from a WIDE mark (blocks above 64 KB: {token position, match start} as two words); `in` may be global memory */
RW_FN RwSeq rw_parse_wide(const uint8_t* in, uint32_t tok, uint32_t mstart, bool last)
{
    RwSeq s;
    const uint32_t t = in[tok];
    int64_t pp = (int64_t)tok + 1;
    int ll = (int)(t >> 4);
    if (ll == 15) { uint32_t x; do { x = in[pp++]; ll += (int)x; } while (x == 255); }
    s.ll = ll; s.ls = (int)pp; s.m = (int)mstart; s.op = (int)mstart - ll;
    s.off = 0; s.mlen = 0;
    if (!last) {
        pp += ll;
        s.off = (int)((uint32_t)in[pp] | ((uint32_t)in[pp + 1] << 8));
        pp += 2;
        int ml = (int)(t & 15u);
        if (ml == 15) { uint32_t x; do { x = in[pp++]; ml += (int)x; } while (x == 255); }
        s.mlen = ml + 4;
    }
    return s;
}

/* The runs of one match (m, off, len): calls f(start, delta) for each, in increasing start order.
 * delta is relative to the output position (source = p + delta); `zeroDelta0` is the delta that maps
 * output position 0 onto the always-zero cell (so position p needs zeroDelta0 - p). */
template <class F>
RW_FN void rw_match_runs(int m, int off, int len, int zeroDelta0, F f)
{
    if (off >= len) { f(m, -off); return; }            /* the common case: no self-overlap */
    int base = m, period = off, rem = len;
    if (off == 0) {                                     /* zero byte, then an offset-1 run that repeats it */
        f(m, zeroDelta0 - m);
        base = m + 1; period = 1; rem = len - 1;
        if (rem <= 0) return;
    }
    /* [base, base + 2*period) reads `period` back; then pieces [base + period*2^t, base + period*2^(t+1))
     * read period*2^t back: always a multiple of the period and never before base - period */
    f(base, -period);
    /* (no piece reads more than 65 535 back -- only matches of blocks above 64 KB get that far: the last piece then
     * runs to the end of the match, still a multiple of the period back) */
    for (long long step = 2LL * period; step < rem && step <= 65535; step *= 2) f(base + (int)step, -(int)step);
}

/* The runs of one sequence CLIPPED to the output tile [os, oe) of a block above 64 KB, as f(start - os, delta), in
 * increasing start order.  Deltas keep the meaning "source = position + delta" in the tile's window (position counted
 * from the tile start): a match run's delta is the same number as in block coordinates (a source before the tile start
 * lies in an earlier tile = global memory); a literal run's delta is litBase + (ls - op), with litBase chosen by the
 * caller so that the sum lands in a virtual range that means "byte ls + (p - op) of the compressed block";
 * zeroDelta0 = what rw_match_runs needs for the always-zero cell, in the same convention. */
template <class F>
RW_FN void rw_tile_runs(const RwSeq& s, int os, int oe, uint32_t litBase, int zeroDelta0, F f)
{
    const int lo = s.op > os ? s.op : os, hi = (s.op + s.ll) < oe ? (s.op + s.ll) : oe;
    if (hi > lo) f(lo - os, (int)(litBase + (uint32_t)(s.ls - s.op)));
    if (s.mlen > 0 && s.m + s.mlen > os && s.m < oe) {
        bool pend = false;                              /* the last piece that starts at or before the tile start covers it */
        int pd = 0;
        rw_match_runs(s.m, s.off, s.mlen, zeroDelta0, [&](int st, int d) {
            if (st <= os) { pend = true; pd = d; return; }
            if (pend) { f(0, pd); pend = false; }
            if (st < oe) f(st - os, d);
        });
        if (pend) f(0, pd);
    }
}

/* run index of output byte q: rows[r] = {bits of row r, (run starts before row r) - 1} */
RW_FN uint32_t rw_rank(const uint2* rows, uint32_t q)
{
    const uint2 r = rows[q >> 5];
    return r.y + (uint32_t)RW_POPC(r.x & (0xFFFFFFFFu >> (31u - (q & 31u))));
}

/* Source byte index (into `window`) of output byte p, given that everything below window index
 * `waveA` is final: follow sources that lie inside the current wave. */
RW_FN uint32_t rw_resolve(const uint2* rows, const uint32_t* tab, uint32_t outA, uint32_t waveA, uint32_t p, uint32_t j)
{
    uint32_t a = outA + p + tab[j];
    while (a >= waveA) {
        const uint32_t q = a - outA;
        a += tab[rw_rank(rows, q)];
    }
    return a;
}

#endif /* LZ4_ROWS_CORE_H */
