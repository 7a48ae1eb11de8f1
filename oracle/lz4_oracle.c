/*
 * oracle/lz4_oracle.c -- TEST INFRASTRUCTURE ONLY (see lz4_oracle.h).
 *
 * Plain-C restatement of the reference LZ4 block codec, written from the algorithm (index based,
 * byte-exact copies, no wild copies) rather than from the reference's pointer code.  Each
 * function cites the reference lines (lib/lz4.c of lz4 v1.10.0) whose behaviour it reproduces.
 * One parse (compress_generic) serves LZ4_compress_fast and LZ4_compress_destSize, one decoder
 * (decompress_generic) LZ4_decompress_safe and LZ4_decompress_safe_partial.  The route functions
 * hold the entry rules and pass the output directive and `partial` as constants, so the compiler
 * may specialise the shared text per route.
 * Pinned against the compiled reference (oracle/_ref) by tests/test_oracle_vs_ref.py,
 * tests/test_destsize_oracle.py and tests/test_partial_oracle.py, and against tests/golden/
 * fixtures by those files and tests/test_oracle_golden.py.
 */
#include "lz4_oracle.h"
#include <string.h>

/* constants: lz4.c:242-249 (MINMATCH, LASTLITERALS, MFLIMIT, FASTLOOP_SAFE_DISTANCE),
 * lz4.c:710-711 (64K limit, skip trigger), lz4.c:52-58 (acceleration clamp), lz4.h:214 */
enum {
    K_MINMATCH = 4,
    K_LASTLITERALS = 5,
    K_MFLIMIT = 12,
    K_MINLENGTH = 13,
    K_MAXDIST = 65535,
    K_SMALL_LIMIT = 65536 + 11,
    K_SKIP_TRIGGER = 6,
    K_ACCEL_MAX = 65537,
    K_FAST_DISTANCE = 64,
    K_MATCH_SAFEGUARD = 12
};
#define K_MAX_INPUT 0x7E000000
#define K_FILL_ACCEL_MAX ((1 << 25) - 1)

static uint32_t load32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
static uint64_t load64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }

int oracle_lz4_compress_bound(int srcSize)
{
    if ((uint32_t)srcSize > (uint32_t)K_MAX_INPUT) return 0;
    return srcSize + srcSize / 255 + 16;
}

/* ------------------------------------------------------------------------------------------
 * Compressor
 * ------------------------------------------------------------------------------------------ */

/* lz4.c:777-783: 4-byte multiplicative hash, 13 bits for the u16 table */
static uint32_t hash_small(const uint8_t* p) { return (load32(p) * 2654435761u) >> 19; }
/* lz4.c:785-791 + :799: on 64-bit LE hosts every non-u16 table hashes the low 5 bytes, 12 bits */
static uint32_t hash_large(const uint8_t* p) { return (uint32_t)(((load64(p) << 24) * 889523592379ull) >> 52); }

typedef struct {
    uint32_t slot[8192];   /* u16 semantics when small (values < 65536), u32[4096] otherwise */
    int small;
} match_table;

static uint32_t tbl_hash(const match_table* t, const uint8_t* p) { return t->small ? hash_small(p) : hash_large(p); }

/* lz4.c:679-703 LZ4_count: length of the common prefix of a[..alimit) and b */
static uint32_t common_prefix(const uint8_t* a, const uint8_t* b, const uint8_t* alimit)
{
    uint32_t n = 0;
    while (a + n < alimit && a[n] == b[n]) n++;
    return n;
}

/* Emit `len` as a run of 255s plus a remainder byte (lz4.c:1123-1128, :1318-1323) */
static int64_t put_runlength(uint8_t* dst, int64_t op, size_t len)
{
    while (len >= 255) { dst[op++] = 255; len -= 255; }
    dst[op++] = (uint8_t)len;
    return op;
}

/* lz4.c:328-332: what the parse does at the end of dst */
typedef enum { NOT_LIMITED, LIMITED_OUTPUT, FILL_OUTPUT } output_directive;

/* lz4.c:930-1335 for 1 <= n <= LZ4_MAX_INPUT_SIZE, noDict / noDictIssue, 64-bit little-endian host.
 * LIMITED_OUTPUT returns 0 where the output would pass dstCapacity; FILL_OUTPUT stops there instead,
 * leaves the input it consumed in *consumed and the first output limit it met in *path. */
static int compress_generic(const uint8_t* src, uint8_t* dst, int n, int dstCapacity, int acceleration,
                            output_directive dir, int* consumed, int* path)
{
    match_table T;
    const int64_t olimit = dstCapacity;   /* signed: a negative dstCapacity must compare like the reference's pointer */
    size_t ip, anchor, filled = 0;
    int64_t op;
    size_t mflimit1, matchlimit;
    uint32_t fwdHash;
    int first = ORACLE_DS_PATH_FILLED;    /* FILL_OUTPUT: the first output limit the parse meets */

    /* lz4.c:1389-1393, :1489-1494 table choice; lz4.c:1558, :1483 zeroed table */
    memset(T.slot, 0, sizeof(T.slot));
    T.small = (n < K_SMALL_LIMIT);

    ip = 0; anchor = 0; op = 0;
    mflimit1 = (size_t)n - K_MFLIMIT + 1;      /* lz4.c:963, only meaningful when n >= 13 */
    matchlimit = (size_t)n - K_LASTLITERALS;   /* lz4.c:964 */

    if (n < K_MINLENGTH) goto tail;            /* lz4.c:1002 */

    T.slot[tbl_hash(&T, src)] = 0;             /* lz4.c:1005-1010 */
    ip = 1;
    fwdHash = tbl_hash(&T, src + 1);           /* lz4.c:1011 */

    for (;;) {
        size_t cand;
        int64_t tokenPos;

        /* --- search (lz4.c:1042-1101) --- */
        {
            size_t fwd = ip;
            uint32_t step = 1;
            uint32_t attempts = (uint32_t)acceleration << K_SKIP_TRIGGER;
            for (;;) {
                uint32_t h = fwdHash;
                size_t cur = fwd;
                cand = T.slot[h];
                ip = cur;
                fwd += step;
                step = attempts++ >> K_SKIP_TRIGGER;
                if (fwd > mflimit1) goto tail;                     /* lz4.c:1055 */
                fwdHash = tbl_hash(&T, src + fwd);
                T.slot[h] = (uint32_t)cur;
                if (!T.small && cand + K_MAXDIST < cur) continue;  /* lz4.c:1090-1093 */
                if (load32(src + cand) == load32(src + cur)) break;/* lz4.c:1096 */
            }
        }
        if (dir == FILL_OUTPUT) filled = ip;                       /* lz4.c:1105 */

        /* --- backward extension (lz4.c:1107-1109) --- */
        while (ip > anchor && cand > 0 && src[ip - 1] == src[cand - 1]) { ip--; cand--; }

        /* --- literals (lz4.c:1112-1136) --- */
        {
            size_t lit = ip - anchor;
            tokenPos = op++;
            if (dir == LIMITED_OUTPUT && op + (int64_t)lit + (2 + 1 + K_LASTLITERALS) + (int64_t)(lit / 255) > olimit)
                return 0;
            /* lz4.c:1118-1122: no room for these literals, a match and the last literals: drop the token */
            if (dir == FILL_OUTPUT
                && op + (int64_t)((lit + 240) / 255) + (int64_t)lit + 2 + 1 + K_MFLIMIT - K_MINMATCH > olimit) {
                op--;
                if (first == ORACLE_DS_PATH_FILLED) first = ORACLE_DS_PATH_LITERALS;
                goto tail;
            }
            if (lit >= 15) {
                dst[tokenPos] = 0xF0;
                op = put_runlength(dst, op, lit - 15);
            } else {
                dst[tokenPos] = (uint8_t)(lit << 4);
            }
            memcpy(dst + op, src + anchor, lit);
            op += (int64_t)lit;
        }

        for (;;) {   /* the "_next_match" chain: lz4.c:1138-1294 */
            uint32_t mcode;
            size_t off;
            /* lz4.c:1147-1152: the match would end too close to olimit: rewind to the token */
            if (dir == FILL_OUTPUT && op + 2 + 1 + K_MFLIMIT - K_MINMATCH > olimit) {
                op = tokenPos;
                if (first == ORACLE_DS_PATH_FILLED) first = ORACLE_DS_PATH_NEXT_MATCH;
                goto tail;
            }
            off = ip - cand;
            dst[op++] = (uint8_t)off;                              /* lz4.c:1162 LE16 */
            dst[op++] = (uint8_t)(off >> 8);

            mcode = common_prefix(src + ip + K_MINMATCH, src + cand + K_MINMATCH, src + matchlimit);  /* lz4.c:1182 */
            ip += (size_t)mcode + K_MINMATCH;

            if (dir != NOT_LIMITED && op + (1 + K_LASTLITERALS) + (mcode + 240) / 255 > olimit) {  /* lz4.c:1187-1211 */
                uint32_t shorter;
                if (dir == LIMITED_OUTPUT) return 0;
                /* lz4.c:1189-1207: shorten the match to what fits, forget the positions hashed beyond it */
                shorter = 15 - 1 + ((uint32_t)(olimit - op) - 1 - K_LASTLITERALS) * 255;
                ip -= mcode - shorter;
                mcode = shorter;
                if (first == ORACLE_DS_PATH_FILLED) first = ORACLE_DS_PATH_REDUCED;
                if (ip <= filled) {
                    size_t p;
                    for (p = ip; p <= filled; p++) T.slot[tbl_hash(&T, src + p)] = 0;
                }
            }
            if (mcode >= 15) {                                     /* lz4.c:1213-1225 */
                dst[tokenPos] += 15;
                op = put_runlength(dst, op, mcode - 15);
            } else {
                dst[tokenPos] += (uint8_t)mcode;
            }

            anchor = ip;
            if (ip >= mflimit1) goto tail;                         /* lz4.c:1233 */

            T.slot[tbl_hash(&T, src + ip - 2)] = (uint32_t)(ip - 2);   /* lz4.c:1236-1242 */

            {   /* immediate re-test at ip: lz4.c:1255-1294 */
                uint32_t h = tbl_hash(&T, src + ip);
                cand = T.slot[h];
                T.slot[h] = (uint32_t)ip;
                if ((T.small || cand + K_MAXDIST >= ip) && load32(src + cand) == load32(src + ip)) {
                    tokenPos = op++;
                    dst[tokenPos] = 0;
                    continue;
                }
            }
            break;
        }

        ip++;                                                      /* lz4.c:1298 */
        fwdHash = tbl_hash(&T, src + ip);
    }

tail:   /* lz4.c:1302-1333 */
    {
        size_t last = (size_t)n - anchor;
        if (dir != NOT_LIMITED && op + (int64_t)last + 1 + (int64_t)((last + 255 - 15) / 255) > olimit) {
            if (dir == LIMITED_OUTPUT) return 0;
            /* lz4.c:1307-1311: as many literals as fit */
            last = (size_t)(olimit - op) - 1;
            last -= (last + 256 - 15) / 256;
            if (first == ORACLE_DS_PATH_FILLED) first = ORACLE_DS_PATH_LAST_LITERALS;
        }
        if (last >= 15) {
            dst[op++] = 0xF0;
            op = put_runlength(dst, op, last - 15);
        } else {
            dst[op++] = (uint8_t)(last << 4);
        }
        memcpy(dst + op, src + anchor, last);
        op += (int64_t)last;
        if (dir == FILL_OUTPUT) {
            *consumed = (int)(anchor + last);                       /* lz4.c:1327, 1332 */
            *path = first;
        }
    }
    return (int)op;
}

int oracle_lz4_compress_fast(const uint8_t* src, uint8_t* dst, int srcSize, int dstCapacity, int acceleration)
{
    const int limited = !(dstCapacity >= oracle_lz4_compress_bound(srcSize));

    /* lz4.c:1386-1388 */
    if (acceleration < 1) acceleration = 1;
    if (acceleration > K_ACCEL_MAX) acceleration = K_ACCEL_MAX;

    /* lz4.c:1360-1372 */
    if ((uint32_t)srcSize > (uint32_t)K_MAX_INPUT) return 0;
    if (srcSize == 0) {
        if (limited && dstCapacity <= 0) return 0;
        dst[0] = 0;
        return 1;
    }
    /* lz4.c:1389-1401 */
    if (limited) return compress_generic(src, dst, srcSize, dstCapacity, acceleration, LIMITED_OUTPUT, NULL, NULL);
    return compress_generic(src, dst, srcSize, dstCapacity, acceleration, NOT_LIMITED, NULL, NULL);
}

int oracle_lz4_compress_destSize_extState(const uint8_t* src, uint8_t* dst, int* srcSizePtr, int targetDstSize,
                                          int acceleration, int* path)
{
    const int n = *srcSizePtr;
    int unused;
    if (path == NULL) path = &unused;

    /* lz4.c:1486-1487: success is guaranteed, LZ4_compress_fast_extState (which clamps the acceleration) */
    if (targetDstSize >= oracle_lz4_compress_bound(n)) {
        *path = ORACLE_DS_PATH_FAST;
        return oracle_lz4_compress_fast(src, dst, n, targetDstSize, acceleration);
    }
    /* lz4.c:1360-1372 with fillOutput */
    if ((uint32_t)n > (uint32_t)K_MAX_INPUT) { *path = ORACLE_DS_PATH_BAD_SIZE; return 0; }
    if (n == 0) {
        *path = ORACLE_DS_PATH_EMPTY;
        if (targetDstSize <= 0) return 0;
        dst[0] = 0;
        *srcSizePtr = 0;
        return 1;
    }
    /* lz4.c:985 */
    if (targetDstSize < 1) { *path = ORACLE_DS_PATH_NO_ROOM; return 0; }
    /* lz4.c:1490-1493 pass the acceleration unclamped; the two ends are brought into range (see lz4_oracle.h) */
    if (acceleration < 1) acceleration = 1;
    if (acceleration > K_FILL_ACCEL_MAX) acceleration = K_FILL_ACCEL_MAX;
    return compress_generic(src, dst, n, targetDstSize, acceleration, FILL_OUTPUT, srcSizePtr, path);
}

/* ------------------------------------------------------------------------------------------
 * Decoder
 * ------------------------------------------------------------------------------------------ */

/* lz4.c:1978-2014 read_variable_length.  *pip advances exactly as the reference's ip does, so
 * that the error code -(ip)-1 matches.  Returns -1 on error. */
static int64_t read_runlength(const uint8_t* src, int64_t* pip, int64_t ilimit, int initial_check)
{
    int64_t total = 0;
    uint32_t b;
    if (initial_check && *pip >= ilimit) return -1;
    do {
        b = src[*pip];
        (*pip)++;
        total += b;
        if (*pip > ilimit) return -1;
    } while (b == 255);
    return total;
}

/* LZ77 copy with the reference's observable semantics: byte-serial self-overlap; offset 0
 * yields zero bytes (lz4.c:2407 / :500 zero-fill then self-copy). */
static void copy_match(uint8_t* dst, int64_t op, int64_t offset, int64_t len)
{
    int64_t i;
    if (offset == 0) { memset(dst + op, 0, (size_t)len); return; }
    for (i = 0; i < len; i++) dst[op + i] = dst[op + i - offset];
}

/* lz4.c:2071-2445, LZ4_decompress_generic after its entry checks (noDict, x86-64 build with
 * LZ4_FAST_DEC_LOOP=1), for srcSize >= 1 and outputSize >= 1.  It follows the reference's control
 * flow decision by decision, because the error value -(ip)-1 depends on which loop reads which
 * byte, but copies bytes one at a time.  `partial` is partialDecoding: stop at outputSize instead
 * of failing there; *lastPath then records how the decode stopped (see lz4_oracle.h). */
static int decompress_generic(const uint8_t* src, uint8_t* dst, int srcSize, int outputSize, int partial,
                              int* lastPath)
{
    const int64_t n = srcSize, cap = outputSize;
    int64_t ip = 0, op = 0;
    int64_t ll, ml, offset;
    uint32_t token;

    /* ---- fast loop region (lz4.c:2076-2209) ---- */
    if (cap - op >= K_FAST_DISTANCE) {
        for (;;) {
            token = src[ip++];
            ll = token >> 4;
            if (ll == 15) {                                        /* lz4.c:2092-2106 */
                int64_t add = read_runlength(src, &ip, n - 15, 1);
                if (add < 0) goto error;
                ll += add;
                if (op + ll > cap - 32 || ip + ll > n - 32) goto safe_literals;
            } else if (!(ip <= n - 17)) {                          /* lz4.c:2107-2115 */
                goto safe_literals;
            }
            memcpy(dst + op, src + ip, (size_t)ll);
            ip += ll; op += ll;

            offset = src[ip] | (src[ip + 1] << 8); ip += 2;        /* lz4.c:2118 */
            ml = token & 15;
            if (ml == 15) {                                        /* lz4.c:2127-2139 */
                int64_t add = read_runlength(src, &ip, n - 4, 0);
                if (add < 0) goto error;
                ml += add;
            }
            /* lz4.c:2148-2159: the 18-byte shortcut performs no offset check of its own, but is only
             * entered when the match source is inside dst */
            ml += K_MINMATCH;
            if (op + ml >= cap - K_FAST_DISTANCE) goto safe_match;
            if (offset > op) goto error;                           /* lz4.c:2161 */
            copy_match(dst, op, offset, ml);                       /* lz4.c:2199-2208 */
            op += ml;
        }
    }

    /* ---- safe loop (lz4.c:2215-2435) ---- */
    for (;;) {
        token = src[ip++];
        ll = token >> 4;

        /* two-stage shortcut, lz4.c:2230-2261 */
        if (ll != 15 && ip < n - 16 && op <= cap - 32) {
            memcpy(dst + op, src + ip, (size_t)ll);
            op += ll; ip += ll;
            ml = token & 15;
            offset = src[ip] | (src[ip + 1] << 8); ip += 2;
            if (ml != 15 && offset >= 8 && offset <= op) {
                copy_match(dst, op, offset, ml + K_MINMATCH);
                op += ml + K_MINMATCH;
                continue;
            }
            goto match_length;
        }

        if (ll == 15) {                                            /* lz4.c:2264-2270 */
            int64_t add = read_runlength(src, &ip, n - 15, 1);
            if (add < 0) goto error;
            ll += add;
        }

safe_literals:                                                     /* lz4.c:2273-2334 */
        if (op + ll > cap - K_MFLIMIT || ip + ll > n - (2 + 1 + K_LASTLITERALS)) {
            if (partial) {
                if (ip + ll > n) ll = n - ip;                      /* lz4.c:2295-2298 */
                if (op + ll > cap) ll = cap - op;                  /* lz4.c:2301-2305 */
            } else if (ip + ll != n || op + ll > cap) {
                goto error;                                        /* lz4.c:2312 */
            }
            memmove(dst + op, src + ip, (size_t)ll);
            ip += ll; op += ll;
            if (!partial) break;                                   /* end of block */
            if (op == cap || ip >= n - 2) { *lastPath |= 1; break; }   /* lz4.c:2328 */
        } else {
            memcpy(dst + op, src + ip, (size_t)ll);
            ip += ll; op += ll;
        }

        offset = src[ip] | (src[ip + 1] << 8); ip += 2;            /* lz4.c:2337 */
        ml = token & 15;

match_length:                                                      /* lz4.c:2344-2351 */
        if (ml == 15) {
            int64_t add = read_runlength(src, &ip, n - 4, 0);
            if (add < 0) goto error;
            ml += add;
        }
        ml += K_MINMATCH;

safe_match:                                                        /* lz4.c:2354-2434 */
        if (offset > op) goto error;                               /* lz4.c:2356 */
        if (op + ml > cap - K_MATCH_SAFEGUARD) {
            if (partial) {                                         /* lz4.c:2392-2404 */
                const int64_t m = ml < cap - op ? ml : cap - op;
                copy_match(dst, op, offset, m);
                if (offset == 0 && m > 0) *lastPath |= 4;
                op += m;
                if (op == cap) { *lastPath |= 2; break; }
                continue;
            }
            if (op + ml > cap - K_LASTLITERALS) goto error;        /* lz4.c:2423 */
        }
        copy_match(dst, op, offset, ml);
        op += ml;
    }
    return (int)op;                                                /* lz4.c:2439 */

error:
    return (int)(-ip) - 1;                                         /* lz4.c:2443 */
}

int oracle_lz4_decompress_safe(const uint8_t* src, uint8_t* dst, int compressedSize, int dstCapacity)
{
    if (src == NULL || dstCapacity < 0) return -1;                 /* lz4.c:2036 */
    if (dstCapacity == 0) return (compressedSize == 1 && src[0] == 0) ? 0 : -1;   /* lz4.c:2064-2068 */
    if (compressedSize == 0) return -1;                            /* lz4.c:2069 */
    return decompress_generic(src, dst, compressedSize, dstCapacity, 0, NULL);
}

int oracle_lz4_decompress_safe_partial(const uint8_t* src, uint8_t* dst, int srcSize, int targetOutputSize,
                                       int dstCapacity, int* lastPath)
{
    const int outputSize = targetOutputSize < dstCapacity ? targetOutputSize : dstCapacity;   /* lz4.c:2461 */
    *lastPath = 0;
    if (src == NULL || outputSize < 0) return -1;                  /* lz4.c:2036 */
    if (outputSize == 0) return 0;                                 /* lz4.c:2066 */
    if (srcSize <= 0) return -1;                                   /* lz4.c:2069, and a negative size */
    return decompress_generic(src, dst, srcSize, outputSize, 1, lastPath);
}

/* Token walk over a VALID block (no bounds checking beyond the input length). */
int oracle_lz4_block_stats(const uint8_t* src, int compressedSize, oracle_block_stats* st)
{
    int64_t ip = 0, n = compressedSize;
    memset(st, 0, sizeof(*st));
    while (ip < n) {
        uint32_t token = src[ip++];
        int64_t ll = token >> 4, ml = token & 15, off;
        if (ll == 15) { uint32_t b; do { if (ip >= n) return -1; b = src[ip++]; ll += b; } while (b == 255); }
        st->n_sequences++;
        st->literal_bytes += (uint32_t)ll;
        ip += ll;
        if (ip >= n) return (ip == n) ? 0 : -1;
        if (ip + 2 > n) return -1;
        off = src[ip] | (src[ip + 1] << 8); ip += 2;
        if (ml == 15) { uint32_t b; do { if (ip >= n) return -1; b = src[ip++]; ml += b; } while (b == 255); }
        ml += K_MINMATCH;
        st->match_bytes += (uint32_t)ml;
        if (off < ml) st->overlap_matches++;
    }
    return -1;
}
