/*
 * lz4_scan_split.h -- the scan of one block split over kSsLanes lanes that MERGE (no re-walking).
 *
 * Same result as scan_block() of lz4_scan_core.h, bit for bit: LZ4_decompress_safe's return value
 * (lz4.c:2022-2445, incl. the negative error position), the sequence count and one mark per sequence.
 *
 * The one-thread scan is a chain of ~2 400 dependent steps per 64 KB block and its duration is the latency of that
 * chain, whatever the batch size.  Here the input of the front loop (lz4.c:2083-2209) is cut in kSsLanes
 * segments and every lane walks its own segment, lane 0 from the first token, the others from the first BYTE of
 * their segment as if it were a token.  Such a speculative chain falls onto the true chain after a few dozen bytes
 * (tests/perf/sync_study.py), so instead of re-walking:
 *
 *   P1  every lane walks its segment with front_step (lz4_scan_core.h) and LISTS what it commits: (token position,
 *       offset, match start relative to an output position 0 at its own start) -- only the rules that depend on input
 *       positions apply;
 *   P2  a lane that reaches the end of its segment keeps walking until it stands on a token of the next lane's
 *       list: from there on the two chains are the same chain, so the rest of the next lane's list is TRUE, up to a
 *       constant shift of its output positions (a next lane that never meets the chain is void and skipped);
 *   P3  one lane follows the merges from lane 0, giving every lane of the chain the first valid index of its list,
 *       its output shift and its place in the final order;
 *   P4  every lane copies its valid entries to the final marks (absolute output positions) and applies the
 *       OUTPUT-dependent rules of the front loop entry by entry: offset before the start of the output (error,
 *       lz4.c:2161) and the capacity rules that hand over to the safe loop (lz4.c:2104, 2137, 2142);
 *   P5  one lane takes the FIRST such event in sequence order -- exactly where the one-thread front loop would have
 *       stopped -- and returns the error or runs the byte-wise scan_tail from that state.
 *
 * No sequence is walked twice (apart from the few steps of P2), so the instruction count stays that of the
 * one-thread scan while the dependent chain is kSsLanes times shorter.  A lane whose list does not fit its share of
 * the scratch space makes the block fall back to the one-thread scan (pathological inputs only).
 *
 * Plain C++ on plain pointers and a small per-block record shared by the lanes: lz4_kernels.cu compiles it for the
 * device (the lanes of a block sit in one warp, __syncwarp between the phases), tests/emul/scan_split_emul.cpp for
 * the host (the lanes of a phase run one after the other); tests/test_scan_split_emul.py checks it against the
 * one-thread scan on valid, corrupted and capacity-limited blocks, incl. an in-process differential fuzz.
 */
#ifndef LZ4_SCAN_SPLIT_H
#define LZ4_SCAN_SPLIT_H

#include "lz4_scan_core.h"

constexpr int kSsLanes = 4;
constexpr int kSsMinBytes = 4096;           /* smaller inputs: the one-thread scan */
enum { SS_RUN = 0, SS_STOP = 1, SS_FULL = 2, SS_MERGED = 3 };

struct SsPub {                              /* one lane's public state */
    int fip;                                /* input position its walk stands at */
    uint32_t fop;                           /* output position there, relative to the lane's own origin */
    uint32_t cnt, cntP1;                    /* entries in its list now / at the end of P1 */
    int fipP1;                              /* where it stood at the end of P1 */
    int stateP1;                            /* its state at the end of P1 (other lanes read this one during P2) */
    int state;
    int target;                             /* SS_MERGED: the lane it merged into ... */
    uint32_t mergeIdx;                      /* ... at this index of that lane's list ... */
    uint32_t mergeOpn;                      /* ... where the sequence's match starts at this output position (own origin) */
    /* filled by P3 for the lanes of the chain */
    int inChain;
    uint32_t first;                         /* first valid index of its list */
    uint32_t base;                          /* add to its relative output positions (mod 2^32) */
    uint32_t place;                         /* final index of its first valid entry */
};
struct SsBlock {
    SsPub lane[kSsLanes];
    int fallback;                           /* 1: some list overflowed -> one-thread scan */
    int endLane;                            /* the lane whose walk ended the front loop */
    uint32_t nFront;                        /* committed sequences of the front loop before any output-dependent event */
    uint32_t errIdx, capIdx;                /* P4: first sequence with the offset error / with match start >= capacity - 64 */
    uint32_t capOpn;                        /* ... and that match start in full (it may not fit the 16 bits of a mark) */
};

/* literal length of the sequence whose token sits at `tok` (a committed sequence: the reads are in range) */
template <class M>
SC_FN int ss_lit_at(M& mem, int tok)
{
    const uint32_t t = mem.b(tok);
    int ll = (int)(t >> 4), p = tok + 1;
    if (ll == 15) { uint32_t x; do { x = mem.b(p++); ll += (int)x; } while (x == 255u); }
    return ll;
}

SC_FN int ss_seg_start(int lane, int nI)
{
    int seg = (nI - 26 + kSsLanes) / kSsLanes;
    return lane * seg;
}

/* commit one step of `me` into its list; false when the list is full */
SC_FN bool ss_push(SsPub& me, uint32_t* A, uint32_t* B, uint32_t R, int tok, uint32_t off16, uint32_t opn)
{
    if (me.cnt >= R) { me.state = SS_FULL; return false; }
    A[me.cnt] = opn;
    B[me.cnt] = (uint32_t)tok | (off16 << 16);
    me.cnt++;
    return true;
}

/* ---- P1: walk the own segment.  A/B = this lane's part of the scratch (R entries each) ---- */
template <class M>
SC_FN void ss_p1(int lane, SsBlock& S, M& mem, int nI, uint32_t* A, uint32_t* B, uint32_t R)
{
    SsPub& me = S.lane[lane];
    const int segEnd = (lane == kSsLanes - 1) ? 0x7FFFFFFF : ss_seg_start(lane + 1, nI);
    int fip = ss_seg_start(lane, nI);
    uint32_t fop = 0;
    me.cnt = 0; me.state = SS_RUN; me.inChain = 0; me.target = -1;
    int nextEvt = 0;
    while (fip < segEnd) {
        front_prefetch(mem, nI, fip, nextEvt);
        const FrontSeq s = front_step(mem, nI, fip);
        if (s.stop) { me.state = SS_STOP; break; }
        if (!ss_push(me, A, B, R, fip, s.off16, fop + (uint32_t)s.lit)) break;
        fip = s.ipn; fop += (uint32_t)s.lit + (uint32_t)s.mlen;
    }
    me.fip = fip; me.fop = fop; me.cntP1 = me.cnt; me.fipP1 = fip; me.stateP1 = me.state;
    if (lane == 0) { S.fallback = 0; S.errIdx = 0xFFFFFFFFu; S.capIdx = 0xFFFFFFFFu; }
}

/* ---- P2: keep walking until the chain stands on a token of a later lane's P1 list (or the front loop ends) ----
 * scratchB(t) = list B of lane t */
template <class M, class ListB>
SC_FN void ss_p2(int lane, SsBlock& S, M& mem, int nI, uint32_t* A, uint32_t* B, uint32_t R, ListB scratchB)
{
    SsPub& me = S.lane[lane];
    if (me.state != SS_RUN) return;                                 /* stopped or full in P1 (the last lane always is) */
    int fip = me.fip;
    uint32_t fop = me.fop;
    int t = lane + 1;
    uint32_t cur = 0;
    for (;;) {
        /* the next token of lane t's P1 chain at or after... : its committed entries, then the position it stopped at */
        const SsPub& T = S.lane[t];
        const int tk = (cur < T.cntP1) ? (int)(scratchB(t)[cur] & 0xFFFFu) : T.fipP1;
        if (fip > tk) {
            if (cur < T.cntP1) { cur++; continue; }
            if (t + 1 < kSsLanes) { t++; cur = 0; continue; }          /* lane t never met the chain: void */
            /* no lane left: walk to the end of the front loop (lane t = last lane stopped before this position) */
        } else if (fip == tk) {
            if (cur == T.cntP1 && T.stateP1 == SS_STOP) { me.state = SS_STOP; break; }   /* the front loop ends here for everybody */
            if (cur == T.cntP1 && T.stateP1 == SS_FULL) { me.state = SS_FULL; break; }
            const FrontSeq s = front_step(mem, nI, fip);
            if (s.stop) { me.state = SS_STOP; break; }                   /* (cannot happen for a committed entry) */
            me.state = SS_MERGED; me.target = t; me.mergeIdx = cur; me.mergeOpn = fop + (uint32_t)s.lit;
            break;
        }
        const FrontSeq s = front_step(mem, nI, fip);
        if (s.stop) { me.state = SS_STOP; break; }
        if (!ss_push(me, A, B, R, fip, s.off16, fop + (uint32_t)s.lit)) break;
        fip = s.ipn; fop += (uint32_t)s.lit + (uint32_t)s.mlen;
    }
    me.fip = fip; me.fop = fop;
}

/* ---- P3 (one lane): follow the merges from lane 0 ---- listA(t) = list A of lane t */
template <class ListA>
SC_FN void ss_p3(SsBlock& S, ListA scratchA)
{
    int j = 0;
    uint32_t first = 0, base = 0, place = 0;
    for (;;) {
        SsPub& L = S.lane[j];
        L.inChain = 1; L.first = first; L.base = base; L.place = place;
        if (L.state == SS_FULL) { S.fallback = 1; return; }
        place += L.cnt - first;
        if (L.state != SS_MERGED) { S.endLane = j; S.nFront = place; return; }     /* SS_STOP: the front loop ends in this lane */
        const SsPub& T = S.lane[L.target];
        const uint32_t trueOpn = base + L.mergeOpn;                                  /* absolute match start of the sequence both stand on */
        first = L.mergeIdx;
        /* lane T's relative match start of the same sequence: its entry, or -- when it committed nothing from there on --
         * what it computed for its own merge at this very token */
        const uint32_t rel = (T.cnt > first) ? scratchA(L.target)[first] : T.mergeOpn;
        base = trueOpn - rel;
        j = L.target;
    }
}

/* ---- P4: every lane of the chain writes its valid entries to the final marks and reports output-dependent events ---- */
SC_FN void ss_p4(int lane, SsBlock& S, int capI, const uint32_t* A, const uint32_t* B, uint32_t* marks, uint32_t markCap,
                 uint32_t& errIdx, uint32_t& capIdx, uint32_t& capOpn)
{
    const SsPub& me = S.lane[lane];
    errIdx = 0xFFFFFFFFu; capIdx = 0xFFFFFFFFu; capOpn = 0;
    if (!me.inChain) return;
    for (uint32_t k = me.first; k < me.cnt; k++) {
        const uint32_t g = me.place + (k - me.first);
        const uint32_t opn = A[k] + me.base, tb = B[k];
        if ((tb >> 16) > opn && errIdx == 0xFFFFFFFFu) errIdx = g;                               /* lz4.c:2161 */
        if ((int64_t)opn >= (int64_t)capI - 64 && capIdx == 0xFFFFFFFFu) { capIdx = g; capOpn = opn; }
        if (marks && g < markCap) marks[g] = (tb & 0xFFFFu) | (opn << 16);
    }
}

/* ---- P5 (one lane): the first event in sequence order decides ---- */
template <class M>
SC_FN int ss_p5(SsBlock& S, M& mem, int nIn, int capIn, uint32_t* nSeqOut, uint32_t* marks, uint32_t markCap)
{
    const SsPub& E = S.lane[S.endLane];
    const uint32_t K = S.nFront;
    const int fipEnd = E.fip;
    const uint32_t fopEnd = E.fop + E.base;
    /* token position / output start of front-loop sequence g (g <= K; g == K: where the walk ended) */
    auto tokOf = [&](uint32_t g) -> int { return g < K ? (int)(marks[g] & 0xFFFFu) : fipEnd; };
    auto startOf = [&](uint32_t g) -> uint32_t {
        if (g >= K) return fopEnd;
        uint32_t opn = (g == S.capIdx) ? S.capOpn : (marks[g] >> 16);      /* (before capIdx every match start is below the capacity: 16 bits) */
        return opn - (uint32_t)ss_lit_at(mem, tokOf(g));
    };
    /* capacity rule (lz4.c:2137/2142; lz4.c:2104 implies it): the front loop stops at the first sequence that ENDS at or past
     * capacity - 64.  The first one whose match STARTS there is capIdx; the one before it may already end there. */
    uint32_t kx = K;
    {
        const uint32_t k1 = S.capIdx < K ? S.capIdx : K;
        if (k1 > 0 && (int)startOf(k1) >= capIn - 64) kx = k1 - 1;
        else if (k1 < K) kx = k1;
    }
    if (S.errIdx < kx) {                                       /* offset before the start of the output: lz4.c:2161, :2443 */
        *nSeqOut = 0;
        return (int)(-(int64_t)tokOf(S.errIdx + 1)) - 1;
    }
    ScanState st;
    st.ip = tokOf(kx); st.op = (int64_t)startOf(kx); st.nseq = kx; st.fast = true;
    st.nextPrefetch = st.ip + 128;
    MarkSink<M> ms(marks, markCap, kx);
    const int r = scan_tail(mem, nIn, capIn, st, nSeqOut, ms);
    ms.flush();
    return r;
}

#endif /* LZ4_SCAN_SPLIT_H */
