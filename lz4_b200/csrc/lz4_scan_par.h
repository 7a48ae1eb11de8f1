/*
 * lz4_scan_par.h -- intra-block PARALLEL scan: NL lanes per block instead of one thread.
 *
 * Same result as scan_block() of lz4_scan_core.h, bit for bit: LZ4_decompress_safe's return value
 * (lz4.c:2022-2445, incl. the negative error position), the sequence count and one mark per sequence.
 * The one-thread scan walks ~2 400 dependent sequences per 64 KB block (its time hardly depends on the batch size);
 * here a block's token chain is cut in NL segments that are walked at the same time.
 *
 * A token chain started at an ARBITRARY byte of LZ4 data falls back onto the true chain quickly
 * (tests/perf/sync_study.py: 74 bytes median on P50 data), which allows a speculative split:
 *
 *   1. COUNT: the input range of the front loop (token positions <= n-26, lz4.c:2083-2209) is cut in NL
 *      segments; lane l parses from the first byte of segment l as if it were a token, up to the first
 *      token at or past the next segment (exit position, #sequences, #output bytes; only the rules that
 *      depend on input positions apply);
 *   2. FIX-UP: lane l's true entry is lane l-1's exit.  Lanes whose entry differs from what they parsed
 *      from parse again; repeated until nothing changes (lane 0 starts at 0, so by induction every lane
 *      ends up parsing from its true entry; most speculative walks have merged with the true chain
 *      before their segment ends, so their exit does not move and the rounds die out quickly);
 *   3. exclusive sums give every lane its first sequence index and output position (done by the caller:
 *      shuffles on the device, a loop in the CPU emulator);
 *   4. WRITE: every lane re-walks its segment with absolute positions, writes the marks and applies the
 *      output-dependent rules of scan_front (capacity, offset before the start);
 *   5. the first lane (in order) whose walk ends -- leaving the front region, a rule that hands over to
 *      the byte-wise code, or the offset error -- owns the rest: it returns the error or runs scan_tail
 *      from exactly the state the one-thread front loop would have reached.
 *
 * Plain C++ on plain pointers: lz4_kernels.cu compiles it for the device (G = false: the block is staged
 * in shared memory by a TMA bulk load; a CTA barrier separates the phases), tests/emul/scan_par_emul.cpp
 * compiles the same text for the host and runs the lanes of a phase one after the other
 * (tests/test_scan_par_emul.py: identical to the one-thread scan on valid, corrupted and capacity-limited
 * blocks from 2 KB to 4 MB, for 32 / 128 / 256 lanes).
 */
#ifndef LZ4_SCAN_PAR_H
#define LZ4_SCAN_PAR_H

#include "lz4_scan_core.h"

enum { SP_RAN = 0, SP_END = 1, SP_ERR = 2 };
constexpr int kSpMaxLanes = 256;
constexpr int kSpMinBytes = 2048;          /* smaller inputs: lane 0 runs the one-thread scan */

struct SpRes {                             /* COUNT pass of one lane */
    int exitPos;                           /* first token position at or past the segment end (or where the walk stopped) */
    int stop;                              /* 1: the front region ends at exitPos (later lanes have nothing) */
    uint32_t count, olen;                  /* sequences committed, output bytes they produce */
};
struct SpEnd {                             /* WRITE pass of one lane */
    int kind;                              /* SP_RAN: ran into the next segment; SP_END: front loop ends here; SP_ERR */
    int ip;                                /* SP_END: token position to resume at; SP_ERR: error position */
    uint32_t op, nseq;                     /* SP_END: output position / sequence index at ip */
    int nextEvt;
};
struct SpShared {
    SpRes res[kSpMaxLanes];
    SpEnd end[kSpMaxLanes];
    int changed;
    int ret;
    uint32_t nseq;
};
struct SpLane {                            /* registers of one lane */
    int segStart, segEnd, from, isVoid;
    int newFrom, newVoid, need;
};

/* One walk over [from, segEnd) with front_step (lz4_scan_core.h), the output position relative (COUNT) or
 * absolute (WRITE).  Position-only rules apply in both passes, output-dependent rules in WRITE only. */
template <class M, bool WRITE>
SC_FN void sp_walk(M& mem, int nI, int capI, int from, int segEnd,
                   uint32_t opBase, uint32_t seqBase, uint32_t* marks, uint32_t markCap, SpRes& R, SpEnd& E)
{
    int fip = from, nextEvt = 0, stop = 0, kind = SP_RAN, errIp = 0;
    uint32_t fop = opBase, cnt = 0;
    while (fip < segEnd) {
        front_prefetch(mem, nI, fip, nextEvt);
        const FrontSeq s = front_step(mem, nI, fip);
        if (s.stop) { stop = 1; kind = SP_END; break; }
        const uint32_t opn = fop + (uint32_t)s.lit;
        if (WRITE) {
            if (opn + (uint32_t)s.mlen >= (uint32_t)(capI - 64)) { kind = SP_END; break; }   // lz4.c:2137/2142
            if (s.off16 > opn) { kind = SP_ERR; errIp = s.ipn; break; }                        // lz4.c:2161
            mark_commit<M>(marks, markCap, seqBase + cnt, (uint32_t)fip, opn);
        }
        fip = s.ipn; fop = opn + (uint32_t)s.mlen; cnt++;
    }
    if (WRITE) {
        E.kind = kind; E.ip = (kind == SP_ERR) ? errIp : fip; E.op = fop; E.nseq = seqBase + cnt; E.nextEvt = nextEvt;
    } else {
        R.exitPos = fip; R.stop = stop; R.count = cnt; R.olen = fop - opBase;
    }
}

/* ---- phase 0: segments + first speculative walk ---- */
template <class M>
SC_FN void sp_phase0(int lane, int nl, SpLane& L, SpShared& S, M& mem, int nI, int capI)
{
    const int lim = nI - 26;                                   /* last token position of the front region */
    int seg = (lim + nl) / nl;
    if (seg < 64) seg = 64;
    L.segStart = lane * seg;
    L.segEnd = (lane == nl - 1) ? 0x7FFFFFFF : (lane + 1) * seg;
    L.from = L.segStart;
    L.isVoid = 0;
    SpEnd unused;
    sp_walk<M, false>(mem, nI, capI, L.from, L.segEnd, 0u, 0u, nullptr, 0u, S.res[lane], unused);
    if (lane == 0) S.changed = 0;
}

/* ---- fix-up round, part 1 (read): where does my segment really start? ---- */
SC_FN void sp_decide(int lane, SpLane& L, const SpShared& S)
{
    L.need = 0;
    if (lane == 0) { L.newFrom = 0; L.newVoid = 0; return; }     /* (the caller resets S.changed between rounds) */
    const SpRes prev = S.res[lane - 1];
    L.newVoid = prev.stop;
    L.newFrom = prev.exitPos;
    L.need = (L.newVoid != L.isVoid) || (L.newFrom != L.from);
}

/* ---- fix-up round, part 2 (write): walk again from the new entry ---- */
template <class M>
SC_FN void sp_redo(int lane, SpLane& L, SpShared& S, M& mem, int nI, int capI)
{
    if (!L.need) return;
    L.from = L.newFrom;
    L.isVoid = L.newVoid;
    if (L.isVoid) {                                            /* the front region ended in an earlier lane */
        S.res[lane].exitPos = L.from; S.res[lane].stop = 1; S.res[lane].count = 0; S.res[lane].olen = 0;
    } else {
        SpEnd unused;
        sp_walk<M, false>(mem, nI, capI, L.from, L.segEnd, 0u, 0u, nullptr, 0u, S.res[lane], unused);
    }
    S.changed = 1;
}

/* ---- WRITE pass; seqBase / outBase = exclusive sums of res[].count / res[].olen over the lanes before this one ---- */
template <class M>
SC_FN void sp_write(int lane, const SpLane& L, SpShared& S, M& mem, int nI, int capI,
                    uint32_t seqBase, uint32_t outBase, uint32_t* marks, uint32_t markCap)
{
    if (L.isVoid) { S.end[lane].kind = SP_RAN; return; }
    SpRes unused;
    sp_walk<M, true>(mem, nI, capI, L.from, L.segEnd, outBase, seqBase, marks, markCap, unused, S.end[lane]);
}

/* ---- the first lane whose walk ended (`first` = smallest lane with end[].kind != SP_RAN, or nl - 1) finishes the block ---- */
template <class M>
SC_FN void sp_finish(int lane, int first, SpShared& S, M& mem, int nI, int capI, uint32_t* marks, uint32_t markCap)
{
    if (lane != first) return;
    const SpEnd e = S.end[first];
    if (e.kind == SP_ERR) { S.ret = (int)(-(int64_t)e.ip) - 1; S.nseq = 0; return; }   /* lz4.c:2443 */
    ScanState st;
    st.ip = e.ip; st.op = (int64_t)e.op; st.nseq = e.nseq; st.fast = true;
    st.nextPrefetch = (e.nextEvt > 0) ? (int64_t)e.nextEvt + 128 : 128;
    uint32_t ns = 0;
    S.ret = scan_tail(mem, nI, capI, st, &ns, marks, markCap);
    S.nseq = ns;
}

#endif /* LZ4_SCAN_PAR_H */
