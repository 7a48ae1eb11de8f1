/*
 * lz4_hc_core.h -- the parses of LZ4_compress_HC (lz4hc.c, v1.10.0) at every level, for host and device.
 *
 * One call compresses one block from a freshly initialised state, exactly as LZ4_compress_HC does with no dictionary
 * and favorDecSpeed off (lz4hc.c:1500-1510): the same output bytes and the same return value.
 *   levels 1 .. 2 (and the lz4mid entries of the level table): LZ4MID_compress, lz4hc.c:522-773
 *   levels 3 .. 9 (and < 1 -> 9):                             LZ4HC_compress_hashChain, lz4hc.c:1121-1362
 *   levels 10 .. 12 (and > 12 -> 12):                         LZ4HC_compress_optimal, lz4hc.c:1823-2123
 * hc_compress_block serves levels up to 9 and returns kHcNoLevel above; hc_compress_block_opt serves 10 and above and
 * returns kHcNoLevel below.  Every parse takes the reference's fillOutput directive as the template flag FILL:
 * hc_compress_block_dest and hc_compress_block_opt_dest are LZ4_compress_HC_destSize (lz4hc.c:1538-1545), which
 * compresses as much input as fits a fixed-size output.
 *
 * Positions are byte offsets into the block.  The reference's indices are position + kHcStart (LZ4HC_init_internal,
 * lz4hc.c:242-259, starts a fresh state at 64 KB), so a zero hash entry is never a candidate.
 *
 * The parse reaches its input, its tables and its output through an accessor `A` with
 *   uint32_t in8(uint32_t p), in32(uint32_t p)      byte / little-endian 32-bit word of the input at p
 *   uint64_t in64(uint32_t p)                       little-endian 64-bit word of the input at p
 *   uint32_t hash(uint32_t h); void set_hash(uint32_t h, uint32_t v)      2^15 entries, all 0 at the start of a block
 *   uint32_t chain(uint32_t i); void set_chain(uint32_t i, uint32_t v)    2^16 16-bit entries, any content at the start
 *   void out(int64_t o, uint32_t v); void copy(int64_t o, uint32_t p, uint32_t len)    output byte / literal copy
 *   Opt& opt(int r)                                 the optimal parser's table, kOptEntries entries, any content at the
 *                                                   start (only hc_compress_block_opt* call it)
 * The chain table needs no initial value: the hash-chain walk only reads the entry of an index in
 * [ipIndex - 65535, ipIndex), and LZ4HC_Insert has written every such index before the walk, the entry of index i last.
 * The chain swap reads the entries of [matchIndex, matchIndex + longest - 4], and only when matchIndex + longest <=
 * ipIndex: with matchIndex >= lowest they all lie in [lowest, ipIndex), which the walk's rule covers.
 * The optimal parser's table needs none either: a step writes entries 0 .. last + 3 before it reads any, and every
 * later write that moves `last` writes the positions it newly covers (a match reaching past last + 3 is always
 * stored), so no read in [0, last + 3] finds an entry from an earlier step or from before the block.
 * Nothing is written at or past the capacity: every output byte is written after the check that covers it (the fill
 * parse's unchecked last sequence after its room test against oend - 3).
 */
#ifndef LZ4_HC_CORE_H
#define LZ4_HC_CORE_H

#include <stdint.h>

#if defined(__CUDACC__)
#define HC_FN __host__ __device__ __forceinline__
#else
#define HC_FN static inline
#endif

namespace hc {

constexpr int kMinMatch = 4;
constexpr int kLastLiterals = 5;
constexpr int kMfLimit = 12;
constexpr int kMinLength = kMfLimit + 1;
constexpr int kOptimalMl = 18;                    /* (ML_MASK - 1) + MINMATCH, lz4hc.c:76 */
constexpr uint32_t kMaxDistance = 65535;          /* LZ4_DISTANCE_MAX */
constexpr uint32_t kHcStart = 65536;              /* index of a fresh state's first byte, lz4hc.c:252 */
constexpr uint32_t kMaxInput = 0x7E000000u;       /* LZ4_MAX_INPUT_SIZE */
constexpr int kHashLog = 15;                      /* LZ4HC_HASH_LOG */
constexpr int kMidHashLog = kHashLog - 1;         /* LZ4MID_HASHLOG: hash4 table, then hash8 table */
constexpr uint32_t kMidHash8 = 1u << kMidHashLog;
constexpr int kHashEntries = 1 << kHashLog;
constexpr int kChainEntries = 1 << 16;
constexpr int kMaxLevel = 9;                      /* above: the optimal parser */
constexpr int kMinOptLevel = 10;                  /* LZ4HC_CLEVEL_OPT_MIN */
constexpr int kHcNoLevel = -1;
constexpr int kOptNum = 4096;                     /* LZ4_OPT_NUM */
constexpr int kTrailingLiterals = 3;
constexpr int kOptEntries = kOptNum + kTrailingLiterals;

/* LZ4HC_optimal_t: one position of the optimal parser's price table */
struct Opt { int price, off, mlen, litlen; };

struct Level { bool mid; int nbSearches; };

/* LZ4HC_getCLevelParams (lz4hc.c:92-116) below the optimal parser */
HC_FN Level level_params(int level)
{
    if (level < 1) level = 9;                     /* LZ4HC_CLEVEL_DEFAULT */
    Level l;
    l.mid = level <= 2;                           /* lz4mid, 2 searches (unused by the mid parse) */
    l.nbSearches = l.mid ? 2 : 1 << (level - 1);  /* 3 -> 4, 4 -> 8, ..., 9 -> 256 */
    return l;
}

HC_FN uint32_t hash4(uint32_t v) { return (v * 2654435761u) >> (32 - kHashLog); }
HC_FN uint32_t mid_hash4(uint32_t v) { return (v * 2654435761u) >> (32 - kMidHashLog); }
HC_FN uint32_t mid_hash8(uint64_t v) { return (uint32_t)(((v << 8) * 58295818150454627ull) >> (64 - kMidHashLog)); }

HC_FN int ctz32(uint32_t x)
{
#if defined(__CUDA_ARCH__)
    return __ffs((int)x) - 1;
#else
    return __builtin_ctz(x);
#endif
}

/* LZ4_count: the common prefix of p and m, not reaching `limit` */
template <class A> HC_FN uint32_t count(A& a, uint32_t p, uint32_t m, uint32_t limit)
{
    const uint32_t p0 = p;
    while (p + 4 <= limit) {
        const uint32_t x = a.in32(p) ^ a.in32(m);
        if (x) return p - p0 + (uint32_t)(ctz32(x) >> 3);
        p += 4; m += 4;
    }
    while (p < limit && a.in8(p) == a.in8(m)) { p++; m++; }
    return p - p0;
}

/* LZ4HC_countBack: minus the common bytes before p and m, at most `most` of them */
template <class A> HC_FN int count_back(A& a, uint32_t p, uint32_t m, uint32_t most)
{
    uint32_t k = 0;
    while (k < most && a.in8(p - 1 - k) == a.in8(m - 1 - k)) k++;
    return -(int)k;
}

/* LZ4HC_countPattern: bytes from p, before `end`, that continue the 4-byte pattern from its byte 0 */
template <class A> HC_FN uint32_t count_pattern(A& a, uint32_t p, uint32_t end, uint32_t pattern)
{
    uint32_t k = 0;
    while (p + k + 4 <= end && a.in32(p + k) == pattern) k += 4;
    while (p + k < end && a.in8(p + k) == ((pattern >> ((k & 3) * 8)) & 0xFF)) k++;
    return k;
}

/* LZ4HC_reverseCountPattern with iLow = the block start: bytes before p that continue the pattern backwards from its
 * byte 3 */
template <class A> HC_FN uint32_t reverse_count_pattern(A& a, uint32_t p, uint32_t pattern)
{
    uint32_t k = 0;
    while (k + 4 <= p && a.in32(p - k - 4) == pattern) k += 4;
    while (k < p && a.in8(p - 1 - k) == ((pattern >> ((3 - (k & 3)) * 8)) & 0xFF)) k++;
    return k;
}

/* Offsets are signed: the fill parse's end lies LASTLITERALS before the target while it parses, before dst for targets
 * below 8, and every comparison with it must then come out "does not fit". */
struct Out {
    int64_t op;           /* bytes written */
    int64_t cap;          /* dstCapacity; oend - LASTLITERALS while the fill parse runs (lz4hc.c:565, 1154) */
    bool limited;         /* limitedOutput (fillOutput included) */
    uint32_t consumed;    /* the fill parse: the input bytes the output holds */
};

/* the length bytes after a 15 in a token nibble */
template <class A> HC_FN void put_length(A& a, Out& o, uint32_t len)
{
    for (; len >= 255; len -= 255) a.out(o.op++, 255);
    a.out(o.op++, len);
}

/* LZ4HC_encodeSequence (lz4hc.c:268-354): literals [anchor, ip), then the match.  false when the output limit is hit
 * (the caller's block then returns 0); on success ip and anchor move past the match. */
template <class A> HC_FN bool encode_sequence(A& a, Out& o, uint32_t& ip, uint32_t& anchor, uint32_t mlen, uint32_t off)
{
    const int64_t token = o.op++;
    const uint32_t ll = ip - anchor;
    if (o.limited && o.op + ll / 255 + ll + (2 + 1 + kLastLiterals) > o.cap) return false;
    uint32_t t;
    if (ll >= 15) { t = 15u << 4; put_length(a, o, ll - 15); }
    else t = ll << 4;
    a.copy(o.op, anchor, ll);
    o.op += ll;
    a.out(o.op++, off & 0xFF);
    a.out(o.op++, off >> 8);
    uint32_t ml = mlen - kMinMatch;
    if (o.limited && o.op + ml / 255 + (1 + kLastLiterals) > o.cap) return false;
    if (ml >= 15) {
        t += 15;
        ml -= 15;
        for (; ml >= 510; ml -= 510) { a.out(o.op++, 255); a.out(o.op++, 255); }
        if (ml >= 255) { ml -= 255; a.out(o.op++, 255); }
        a.out(o.op++, ml);
    } else {
        t += ml;
    }
    a.out(token, t);
    ip += mlen;
    anchor = ip;
    return true;
}

/* the last literals (lz4hc.c:1308-1337, 707-741): the block's size, or 0 when they do not fit a limited output.  The
 * fill parse restores its end and takes as many literals as fit there. */
template <bool FILL, class A> HC_FN int last_literals(A& a, Out& o, uint32_t anchor, uint32_t n)
{
    uint32_t run = n - anchor;
    const int64_t total = 1 + (int64_t)(run + 255 - 15) / 255 + run;
    if (FILL) {
        o.cap += kLastLiterals;
        if (o.op + total > o.cap) {
            const int64_t room = o.cap - o.op - 1;                     /* >= 0: the parse leaves a byte for the token */
            run = (uint32_t)(room - (room + 256 - 15) / 256);
        }
        o.consumed = anchor + run;
    } else if (o.limited && o.op + total > o.cap) {
        return 0;
    }
    if (run >= 15) { a.out(o.op++, 15u << 4); put_length(a, o, run - 15); }
    else a.out(o.op++, run << 4);
    a.copy(o.op, anchor, run);
    o.op += run;
    return (int)o.op;
}

/* The fill parse's end after a sequence that does not fit (lz4hc.c:747-769, 1340-1358): the output goes back to `saved`,
 * before the sequence.  When its literals fit below maxLitPos = oend - 3, the match is clamped to the room left and
 * the sequence goes out unchecked if the MFLIMIT test holds; the last literals follow. */
template <class A> HC_FN int fill_overflow(A& a, Out& o, int64_t saved, uint32_t ip, uint32_t anchor, uint32_t mlen,
                                           uint32_t off, uint32_t n)
{
    o.op = saved;
    const int64_t ll = ip - anchor;
    const int64_t llTotal = 1 + (ll + 240) / 255 + ll;
    const int64_t maxLitPos = o.cap - 3;
    if (o.op + llTotal <= maxLitPos) {
        const int64_t maxMl = kMinMatch + 14 + (maxLitPos - (o.op + llTotal)) * 255;
        if ((int64_t)mlen > maxMl) mlen = (uint32_t)maxMl;
        if ((o.cap + kLastLiterals) - (o.op + llTotal + 2) - 1 + (int64_t)mlen >= kMfLimit) {
            o.limited = false;
            encode_sequence(a, o, ip, anchor, mlen, off);
            o.limited = true;
        }
    }
    return last_literals<true>(a, o, anchor, n);
}

/* LZ4MID_compress (lz4hc.c:522-773) without a dictionary.  Note that ipIndex keeps the search position's index when the
 * catch-back or the ip + 1 match moves ip: the reference adds the next positions with it. */
template <bool FILL, class A> HC_FN int mid_compress(A& a, Out& o, uint32_t n)
{
    uint32_t ip = 0, anchor = 0;
    if (n < (uint32_t)kMinLength) return last_literals<FILL>(a, o, anchor, n);
    const uint32_t mflimit = n - kMfLimit, matchlimit = n - kLastLiterals;
    const uint32_t ilimitIdx = n - 8 + kHcStart;                    /* LZ4MID_HASHSIZE */
    while (ip <= mflimit) {
        const uint32_t ipIndex = ip + kHcStart;
        uint32_t mlen = 0, dist = 0;
        bool found = false;
        {   /* long match */
            const uint32_t h8 = kMidHash8 + mid_hash8(a.in64(ip));
            const uint32_t pos8 = a.hash(h8);
            a.set_hash(h8, ipIndex);
            if (ipIndex - pos8 <= kMaxDistance && pos8 >= kHcStart) {
                mlen = count(a, ip, pos8 - kHcStart, matchlimit);
                if (mlen >= (uint32_t)kMinMatch) { dist = ipIndex - pos8; found = true; }
            }
        }
        if (!found) {   /* short match, then a longer one at ip + 1 */
            const uint32_t h4 = mid_hash4(a.in32(ip));
            const uint32_t pos4 = a.hash(h4);
            a.set_hash(h4, ipIndex);
            if (ipIndex - pos4 <= kMaxDistance && pos4 >= kHcStart) {
                mlen = count(a, ip, pos4 - kHcStart, matchlimit);
                if (mlen >= (uint32_t)kMinMatch) {
                    const uint32_t h8 = kMidHash8 + mid_hash8(a.in64(ip + 1));
                    const uint32_t pos8 = a.hash(h8);
                    const uint32_t d2 = ipIndex + 1 - pos8;
                    dist = ipIndex - pos4;
                    found = true;
                    if (d2 <= kMaxDistance && pos8 >= kHcStart && ip < mflimit) {
                        const uint32_t ml2 = count(a, ip + 1, pos8 - kHcStart, matchlimit);
                        if (ml2 > mlen) {
                            a.set_hash(h8, ipIndex + 1);
                            ip++;
                            mlen = ml2;
                            dist = d2;
                        }
                    }
                }
            }
        }
        if (!found) {
            ip += 1 + ((ip - anchor) >> 9);
            continue;
        }
        while (ip > anchor && ip > dist && a.in8(ip - 1) == a.in8(ip - 1 - dist)) { ip--; mlen++; }
        a.set_hash(kMidHash8 + mid_hash8(a.in64(ip + 1)), ipIndex + 1);
        a.set_hash(kMidHash8 + mid_hash8(a.in64(ip + 2)), ipIndex + 2);
        a.set_hash(mid_hash4(a.in32(ip + 1)), ipIndex + 1);
        const int64_t saved = o.op;
        if (!encode_sequence(a, o, ip, anchor, mlen, dist))
            return FILL ? fill_overflow(a, o, saved, ip, anchor, mlen, dist, n) : 0;
        const uint32_t end = ip + kHcStart;
        if (end - 2 < ilimitIdx) {
            if (ip > 5) a.set_hash(kMidHash8 + mid_hash8(a.in64(ip - 5)), end - 5);
            a.set_hash(kMidHash8 + mid_hash8(a.in64(ip - 3)), end - 3);
            a.set_hash(kMidHash8 + mid_hash8(a.in64(ip - 2)), end - 2);
            a.set_hash(mid_hash4(a.in32(ip - 2)), end - 2);
            a.set_hash(mid_hash4(a.in32(ip - 1)), end - 1);
        }
    }
    return last_literals<FILL>(a, o, anchor, n);
}

struct Match { int len, off, back; };

struct ChainState {
    uint32_t nextToUpdate;    /* index */
    int nbSearches;
    bool patternAnalysis;
};

/* LZ4HC_Insert (lz4hc.c:781-802): every index before `target` joins its hash chain */
template <class A> HC_FN void insert(A& a, ChainState& s, uint32_t target)
{
    for (uint32_t idx = s.nextToUpdate; idx < target; idx++) {
        const uint32_t h = hash4(a.in32(idx - kHcStart));
        uint32_t delta = idx - a.hash(h);
        if (delta > kMaxDistance) delta = kMaxDistance;
        a.set_chain(idx & 0xFFFF, delta);
        a.set_hash(h, idx);
    }
    s.nextToUpdate = target;
}

/* LZ4HC_InsertAndGetWiderMatch (lz4hc.c:884-1104) for one prefix, no favorDecSpeed: the longest match through ip that
 * starts no earlier than iLow, is longer than `longest` and ends by iHigh.  The candidates are taken in the chain's
 * order, and the 2-byte quick reject at longest - 1 comes first: it decides which later candidates count.
 * SWAP is the chain swap of the optimal parser (lz4hc.c:964-985, called with iLow == ip): a candidate whose length ties
 * or sets the best so far moves the walk to the chain, among the best match's positions, that reaches farthest back.
 * chainPos (matchChainPos) is never reset: once set it shuts the repeat-pattern branch and shifts every later step. */
template <bool SWAP = false, class A>
HC_FN Match wider_match(A& a, ChainState& s, uint32_t ip, uint32_t iLow, uint32_t iHigh, int longest)
{
    const uint32_t ipIndex = ip + kHcStart;
    const uint32_t lowest = (kHcStart + kMaxDistance + 1 > ipIndex) ? kHcStart : ipIndex - kMaxDistance;
    const uint32_t lookBack = ip - iLow;
    const uint32_t pattern = a.in32(ip);
    int nb = s.nbSearches;
    int repeat = 0;                       /* 0 untested, 1 not a repeat, 2 confirmed */
    uint32_t srcPatternLength = 0;
    uint32_t chainPos = 0;
    Match r; r.len = longest; r.off = 0; r.back = 0;
    insert(a, s, ipIndex);
    uint32_t matchIndex = a.hash(hash4(pattern));
    while (matchIndex >= lowest && nb > 0) {
        nb--;
        const uint32_t m = matchIndex - kHcStart;
        const uint32_t q = (uint32_t)r.len - 1;
        if (a.in8(iLow + q) == a.in8(m - lookBack + q) && a.in8(iLow + q + 1) == a.in8(m - lookBack + q + 1)
            && a.in32(m) == pattern) {
            const uint32_t most = lookBack < m ? lookBack : m;
            const int back = lookBack ? count_back(a, ip, m, most) : 0;
            const int len = kMinMatch + (int)count(a, ip + kMinMatch, m + kMinMatch, iHigh) - back;
            if (len > r.len) { r.len = len; r.off = (int)(ipIndex - matchIndex); r.back = back; }
            /* the swap fires on matchLength == longest after the update, ties included; a rejected candidate's
             * matchLength is 0 and never does */
            if constexpr (SWAP) {
                if (len == r.len && matchIndex + (uint32_t)r.len <= ipIndex) {
                    /* the entries of [matchIndex, matchIndex + longest - 4], with a stride that grows while none is
                     * larger */
                    uint32_t farthest = 1;
                    const int end = r.len - kMinMatch + 1;
                    int step = 1, accel = 1 << 4;
                    for (int pos = 0; pos < end; pos += step) {
                        const uint32_t d = a.chain((matchIndex + (uint32_t)pos) & 0xFFFF);
                        step = accel++ >> 4;
                        if (d > farthest) { farthest = d; chainPos = (uint32_t)pos; accel = 1 << 4; }
                    }
                    if (farthest > 1) {
                        if (farthest > matchIndex) break;
                        matchIndex -= farthest;
                        continue;
                    }
                }
            }
        }
        const uint32_t next = a.chain(matchIndex & 0xFFFF);
        if (s.patternAnalysis && next == 1 && (!SWAP || chainPos == 0)) {
            const uint32_t cand = matchIndex - 1;
            if (repeat == 0) {
                if ((pattern & 0xFFFF) == (pattern >> 16) && (pattern & 0xFF) == (pattern >> 24)) {
                    repeat = 2;
                    srcPatternLength = count_pattern(a, ip + 4, iHigh, pattern) + 4;
                } else {
                    repeat = 1;
                }
            }
            if (repeat == 2 && cand >= lowest) {
                const uint32_t mp = cand - kHcStart;
                if (a.in32(mp) == pattern) {
                    const uint32_t fwd = count_pattern(a, mp + 4, iHigh, pattern) + 4;
                    uint32_t backLength = reverse_count_pattern(a, mp, pattern);
                    const uint32_t from = cand - backLength > lowest ? cand - backLength : lowest;
                    backLength = cand - from;
                    const uint32_t segment = backLength + fwd;
                    if (segment >= srcPatternLength && fwd <= srcPatternLength) {
                        matchIndex = cand + fwd - srcPatternLength;        /* the whole source pattern fits */
                    } else {
                        matchIndex = cand - backLength;                    /* the segment's farthest position */
                        if (lookBack == 0) {
                            const uint32_t maxML = segment < srcPatternLength ? segment : srcPatternLength;
                            if ((uint32_t)r.len < maxML) {
                                if (ipIndex - matchIndex > kMaxDistance) break;
                                r.len = (int)maxML;
                                r.off = (int)(ipIndex - matchIndex);
                            }
                            const uint32_t d = a.chain(matchIndex & 0xFFFF);
                            if (d > matchIndex) break;
                            matchIndex -= d;
                        }
                    }
                    continue;
                }
            }
        }
        if constexpr (SWAP) matchIndex -= a.chain((matchIndex + chainPos) & 0xFFFF);
        else matchIndex -= next;
    }
    return r;
}

/* LZ4HC_compress_hashChain (lz4hc.c:1121-1362) without a dictionary: the _Search2 / _Search3 state machine.  The fill
 * parse restores the output to optr, before the sequence that overflows: for the second of the ML1 and ML2 pair that
 * is m2 at start2 (lz4hc.c:1231-1237). */
template <bool FILL, class A> HC_FN int chain_compress(A& a, Out& o, uint32_t n, int nbSearches)
{
    uint32_t anchor = 0;
    if (n < (uint32_t)kMinLength) return last_literals<FILL>(a, o, anchor, n);
    ChainState s;
    s.nextToUpdate = kHcStart;
    s.nbSearches = nbSearches;
    s.patternAnalysis = nbSearches > 128;
    const int mflimit = (int)n - kMfLimit;
    const uint32_t matchlimit = n - kLastLiterals;
    int ip = 0, start0 = 0, start2 = 0, start3 = 0;
    Match m0, m1, m2, m3;
    const Match none = {0, 0, 0};
    while (ip <= mflimit) {
        m1 = wider_match(a, s, (uint32_t)ip, (uint32_t)ip, matchlimit, kMinMatch - 1);
        if (m1.len < kMinMatch) { ip++; continue; }
        start0 = ip; m0 = m1;
        int state = 2;                        /* 2: _Search2, 3: _Search3, 0: back to the main loop */
        while (state) {
            if (state == 2) {
                if (ip + m1.len <= mflimit) {
                    start2 = ip + m1.len - 2;
                    m2 = wider_match(a, s, (uint32_t)start2, (uint32_t)ip, matchlimit, m1.len);
                    start2 += m2.back;
                } else {
                    m2 = none;
                }
                if (m2.len <= m1.len) {       /* no better match: ML1 goes out */
                    uint32_t u = (uint32_t)ip, an = anchor;
                    const int64_t optr = o.op;
                    if (!encode_sequence(a, o, u, an, (uint32_t)m1.len, (uint32_t)m1.off))
                        return FILL ? fill_overflow(a, o, optr, u, an, (uint32_t)m1.len, (uint32_t)m1.off, n) : 0;
                    ip = (int)u; anchor = an;
                    state = 0;
                    continue;
                }
                if (start0 < ip && start2 < ip + m0.len) { ip = start0; m1 = m0; }
                if (start2 - ip < 3) { ip = start2; m1 = m2; continue; }     /* first match too short: dropped */
                state = 3;
            }
            /* _Search3 */
            if (start2 - ip < kOptimalMl) {
                int newMl = m1.len > kOptimalMl ? kOptimalMl : m1.len;
                if (ip + newMl > start2 + m2.len - kMinMatch) newMl = start2 - ip + m2.len - kMinMatch;
                const int corr = newMl - (start2 - ip);
                if (corr > 0) { start2 += corr; m2.len -= corr; }
            }
            if (start2 + m2.len <= mflimit) {
                start3 = start2 + m2.len - 3;
                m3 = wider_match(a, s, (uint32_t)start3, (uint32_t)start2, matchlimit, m2.len);
                start3 += m3.back;
            } else {
                m3 = none;
            }
            if (m3.len <= m2.len) {           /* no better match: ML1 and ML2 go out */
                if (start2 < ip + m1.len) m1.len = start2 - ip;
                uint32_t u = (uint32_t)ip, an = anchor;
                int64_t optr = o.op;
                if (!encode_sequence(a, o, u, an, (uint32_t)m1.len, (uint32_t)m1.off))
                    return FILL ? fill_overflow(a, o, optr, u, an, (uint32_t)m1.len, (uint32_t)m1.off, n) : 0;
                u = (uint32_t)start2;
                optr = o.op;
                if (!encode_sequence(a, o, u, an, (uint32_t)m2.len, (uint32_t)m2.off))
                    return FILL ? fill_overflow(a, o, optr, u, an, (uint32_t)m2.len, (uint32_t)m2.off, n) : 0;
                ip = (int)u; anchor = an;
                state = 0;
                continue;
            }
            if (start3 < ip + m1.len + 3) {   /* no room for ML2 */
                if (start3 >= ip + m1.len) {  /* ML1 goes out, ML3 becomes ML1 */
                    if (start2 < ip + m1.len) {
                        const int corr = ip + m1.len - start2;
                        start2 += corr;
                        m2.len -= corr;
                        if (m2.len < kMinMatch) { start2 = start3; m2 = m3; }
                    }
                    uint32_t u = (uint32_t)ip, an = anchor;
                    const int64_t optr = o.op;
                    if (!encode_sequence(a, o, u, an, (uint32_t)m1.len, (uint32_t)m1.off))
                        return FILL ? fill_overflow(a, o, optr, u, an, (uint32_t)m1.len, (uint32_t)m1.off, n) : 0;
                    anchor = an;
                    ip = start3; m1 = m3;
                    start0 = start2; m0 = m2;
                    state = 2;
                    continue;
                }
                start2 = start3; m2 = m3;
                continue;                     /* _Search3 */
            }
            /* three ascending matches: ML1 goes out, shortened to meet ML2 */
            if (start2 < ip + m1.len) {
                if (start2 - ip < kOptimalMl) {
                    if (m1.len > kOptimalMl) m1.len = kOptimalMl;
                    if (ip + m1.len > start2 + m2.len - kMinMatch) m1.len = start2 - ip + m2.len - kMinMatch;
                    const int corr = m1.len - (start2 - ip);
                    if (corr > 0) { start2 += corr; m2.len -= corr; }
                } else {
                    m1.len = start2 - ip;
                }
            }
            uint32_t u = (uint32_t)ip, an = anchor;
            const int64_t optr = o.op;
            if (!encode_sequence(a, o, u, an, (uint32_t)m1.len, (uint32_t)m1.off))
                return FILL ? fill_overflow(a, o, optr, u, an, (uint32_t)m1.len, (uint32_t)m1.off, n) : 0;
            anchor = an;
            ip = start2; m1 = m2;
            start2 = start3; m2 = m3;
        }
    }
    return last_literals<FILL>(a, o, anchor, n);
}

/* LZ4HC_literalsPrice / LZ4HC_sequencePrice (lz4hc.c:1778-1800): bytes of a literal run, and of a sequence (mlen >= 4) */
HC_FN int literals_price(int litlen) { return litlen >= 15 ? litlen + 1 + (litlen - 15) / 255 : litlen; }
HC_FN int sequence_price(int litlen, int mlen)
{
    return 3 + literals_price(litlen) + (mlen >= 15 + kMinMatch ? 1 + (mlen - 15 - kMinMatch) / 255 : 0);
}

/* LZ4HC_FindLongerMatch (lz4hc.c:1802-1820) without favorDecSpeed: a match at ip longer than minLen (pattern analysis
 * and the chain swap on), else {0, 0, 0} */
template <class A> HC_FN Match longer_match(A& a, ChainState& s, uint32_t ip, uint32_t iHigh, int minLen)
{
    Match m = wider_match<true>(a, s, ip, ip, iHigh, minLen);
    if (m.len <= minLen) { m.len = 0; m.off = 0; }
    return m;
}

struct OptLevel { int nbSearches, sufficient; bool fullUpdate; };

/* the level table for 10 .. 12 (lz4hc.c:103-105; above 12 reads as 12), targetLength clamped to LZ4_OPT_NUM - 1
 * (lz4hc.c:1861), and ultra mode from the level as given (lz4hc.c:1409) */
HC_FN OptLevel opt_level_params(int level)
{
    OptLevel l;
    l.nbSearches = level == 10 ? 96 : level == 11 ? 512 : 16384;
    l.sufficient = level == 10 ? 64 : level == 11 ? 128 : kOptNum - 1;
    l.fullUpdate = level >= 12;
    return l;
}

/* LZ4HC_compress_optimal (lz4hc.c:1823-2123) without a dictionary or favorDecSpeed.  Each step prices every position up
 * to the end of the matches found so far (a.opt(r) for r = 0 .. last + 3), walks the cheapest path back and encodes it.
 * Literal runs and prices grow with ip - anchor, so they stay 32-bit.  The fill parse restores the output to `saved`,
 * before the sequence that overflows. */
template <bool FILL, class A> HC_FN int opt_compress(A& a, Out& o, uint32_t n, const OptLevel l)
{
    uint32_t ip = 0, anchor = 0;
    /* below 13 bytes the reference's loop runs at most one search, at position 0 of an empty table, and finds nothing */
    if (n < (uint32_t)kMinLength) return last_literals<FILL>(a, o, anchor, n);
    ChainState s;
    s.nextToUpdate = kHcStart;
    s.nbSearches = l.nbSearches;
    s.patternAnalysis = true;
    const uint32_t mflimit = n - kMfLimit, matchlimit = n - kLastLiterals;
    while (ip <= mflimit) {
        const int llen = (int)(ip - anchor);
        const Match first = longer_match(a, s, ip, matchlimit, kMinMatch - 1);
        if (first.len == 0) { ip++; continue; }
        if (first.len > l.sufficient) {                              /* good enough: encoded at once */
            const int64_t saved = o.op;
            if (!encode_sequence(a, o, ip, anchor, (uint32_t)first.len, (uint32_t)first.off))
                return FILL ? fill_overflow(a, o, saved, ip, anchor, (uint32_t)first.len, (uint32_t)first.off, n) : 0;
            continue;
        }
        for (int r = 0; r < kMinMatch; r++) {
            Opt& e = a.opt(r);
            e.mlen = 1; e.off = 0; e.litlen = llen + r; e.price = literals_price(llen + r);
        }
        for (int ml = kMinMatch; ml <= first.len; ml++) {
            Opt& e = a.opt(ml);
            e.mlen = ml; e.off = first.off; e.litlen = llen; e.price = sequence_price(llen, ml);
        }
        int last = first.len;
        for (int k = 1; k <= kTrailingLiterals; k++) {
            Opt& e = a.opt(last + k);
            e.mlen = 1; e.off = 0; e.litlen = k; e.price = a.opt(last).price + literals_price(k);
        }
        int cur, bestLen = 0, bestOff = 0;
        bool now = false;                                            /* a match at cur is encoded at once */
        for (cur = 1; cur < last; cur++) {
            if (ip + cur > mflimit) break;
            const int pc = a.opt(cur).price;
            if (a.opt(cur + 1).price <= pc && (!l.fullUpdate || a.opt(cur + kMinMatch).price < pc + 3)) continue;
            const Match m = longer_match(a, s, ip + cur, matchlimit, l.fullUpdate ? kMinMatch - 1 : last - cur);
            if (m.len == 0) continue;
            if (m.len > l.sufficient || m.len + cur >= kOptNum) {
                bestLen = m.len; bestOff = m.off; last = cur + 1; now = true;
                break;
            }
            const int baseLit = a.opt(cur).litlen;
            for (int lit = 1; lit < kMinMatch; lit++) {                  /* literals before the match: strictly cheaper */
                const int price = pc - literals_price(baseLit) + literals_price(baseLit + lit);
                Opt& e = a.opt(cur + lit);
                if (price < e.price) { e.mlen = 1; e.off = 0; e.litlen = baseLit + lit; e.price = price; }
            }
            const bool afterLit = a.opt(cur).mlen == 1;
            const int ll = afterLit ? baseLit : 0;
            const int base = afterLit ? (cur > ll ? a.opt(cur - ll).price : 0) : pc;
            for (int ml = kMinMatch; ml <= m.len; ml++) {                /* the match: ties win, and so does past last + 3 */
                const int pos = cur + ml;
                const int price = base + sequence_price(ll, ml);
                if (pos > last + kTrailingLiterals || price <= a.opt(pos).price) {
                    if (ml == m.len && last < pos) last = pos;
                    Opt& e = a.opt(pos);
                    e.mlen = ml; e.off = m.off; e.litlen = ll; e.price = price;
                }
            }
            for (int k = 1; k <= kTrailingLiterals; k++) {
                Opt& e = a.opt(last + k);
                e.mlen = 1; e.off = 0; e.litlen = k; e.price = a.opt(last).price + literals_price(k);
            }
        }
        if (!now) {
            bestLen = a.opt(last).mlen;
            bestOff = a.opt(last).off;
            cur = last - bestLen;
        }
        {   /* the path back from cur: each position takes the step that leaves it */
            int pos = cur, ml = bestLen, off = bestOff;
            for (;;) {
                Opt& e = a.opt(pos);
                const int nml = e.mlen, noff = e.off;
                e.mlen = ml; e.off = off;
                ml = nml; off = noff;
                if (nml > pos) break;
                pos -= nml;
            }
        }
        for (int r = 0; r < last;) {
            const int ml = a.opt(r).mlen, off = a.opt(r).off;
            if (ml == 1) { ip++; r++; continue; }
            r += ml;
            const int64_t saved = o.op;
            if (!encode_sequence(a, o, ip, anchor, (uint32_t)ml, (uint32_t)off))
                return FILL ? fill_overflow(a, o, saved, ip, anchor, (uint32_t)ml, (uint32_t)off, n) : 0;
        }
    }
    return last_literals<FILL>(a, o, anchor, n);
}

/* LZ4_compress_HC(src, dst, n, cap, level) for level <= 9 from a fresh state; kHcNoLevel for levels above 9 */
template <class A> HC_FN int hc_compress_block(A& a, int n, int cap, int level)
{
    if (level > kMaxLevel) return kHcNoLevel;
    if ((uint32_t)n > kMaxInput) return 0;                                      /* lz4hc.c:1389 */
    Out o;
    o.op = 0;
    o.cap = cap;
    o.limited = cap < n + n / 255 + 16;                                         /* LZ4_compressBound, lz4hc.c:1506 */
    const Level l = level_params(level);
    return l.mid ? mid_compress<false>(a, o, (uint32_t)n) : chain_compress<false>(a, o, (uint32_t)n, l.nbSearches);
}

/* LZ4_compress_HC_destSize(state, src, dst, &n, target, level) for level <= 9 from a fresh state, kHcNoLevel for levels
 * above 9.  `consumed` is what the reference leaves in *srcSizePtr: the input bytes the output holds, or n where it
 * leaves it alone (lz4hc.c:1388-1389).  The fill parse runs at every target from 1 up, the bound and above included. */
template <class A> HC_FN int hc_compress_block_dest(A& a, int n, int target, int level, int& consumed)
{
    consumed = n;
    if (level > kMaxLevel) return kHcNoLevel;
    if (target < 1) return 0;                                                   /* lz4hc.c:1388 */
    if ((uint32_t)n > kMaxInput) return 0;                                      /* lz4hc.c:1389 */
    Out o;
    o.op = 0;
    o.cap = (int64_t)target - kLastLiterals;
    o.limited = true;
    o.consumed = 0;
    const Level l = level_params(level);
    const int r = l.mid ? mid_compress<true>(a, o, (uint32_t)n) : chain_compress<true>(a, o, (uint32_t)n, l.nbSearches);
    consumed = (int)o.consumed;
    return r;
}

/* LZ4_compress_HC(src, dst, n, cap, level) for level >= 10 from a fresh state (above 12 reads as 12); kHcNoLevel for
 * levels below 10, which belong to hc_compress_block */
template <class A> HC_FN int hc_compress_block_opt(A& a, int n, int cap, int level)
{
    if (level < kMinOptLevel) return kHcNoLevel;
    if ((uint32_t)n > kMaxInput) return 0;                                      /* lz4hc.c:1389 */
    Out o;
    o.op = 0;
    o.cap = cap;
    o.limited = cap < n + n / 255 + 16;                                         /* LZ4_compressBound, lz4hc.c:1506 */
    return opt_compress<false>(a, o, (uint32_t)n, opt_level_params(level));
}

/* LZ4_compress_HC_destSize(state, src, dst, &n, target, level) for level >= 10 from a fresh state, kHcNoLevel below;
 * `consumed` as for hc_compress_block_dest */
template <class A> HC_FN int hc_compress_block_opt_dest(A& a, int n, int target, int level, int& consumed)
{
    consumed = n;
    if (level < kMinOptLevel) return kHcNoLevel;
    if (target < 1) return 0;                                                   /* lz4hc.c:1388 */
    if ((uint32_t)n > kMaxInput) return 0;                                      /* lz4hc.c:1389 */
    Out o;
    o.op = 0;
    o.cap = (int64_t)target - kLastLiterals;
    o.limited = true;
    o.consumed = 0;
    const int r = opt_compress<true>(a, o, (uint32_t)n, opt_level_params(level));
    consumed = (int)o.consumed;
    return r;
}

}  // namespace hc

#undef HC_FN
#endif
