/*
 * tests/destsize_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C restatement of the reference's LZ4_compress_destSize / LZ4_compress_destSize_extState
 * (lib/lz4.c of lz4 v1.10.0: lz4.c:1481-1503 -> :1344 / :930 with fillOutput), index based like the
 * compressor of oracle/lz4_oracle.c, which this file is compiled with (tests/destsize_oracle.py builds
 * both into one library): the route where success is guaranteed is that file's oracle_lz4_compress_fast.
 * 64-bit little-endian host.  Byte-identical output, return value and *srcSizePtr.  The acceleration reaches
 * the fill parse unclamped (lz4.c:1490-1493); values below 1 (the reference asserts) are taken as 1 and values
 * of 2^25 and above (where the reference's `acceleration << 6` overflows int) as 2^25 - 1.  Pinned against the
 * compiled reference by tests/test_destsize_oracle.py and tests/golden/kat_destsize.json.
 */
#include "lz4_oracle.h"
#include <string.h>

/* *path receives the route taken and, in the fill parse, the first output limit met */
enum {
    ORACLE_DS_FAST = 0,          /* target >= LZ4_compressBound(n): LZ4_compress_fast_extState (lz4.c:1486-1487) */
    ORACLE_DS_EMPTY = 1,         /* n == 0 (lz4.c:1361-1371) */
    ORACLE_DS_NO_ROOM = 2,       /* target < 1 (lz4.c:985) */
    ORACLE_DS_LITERALS = 3,      /* the literal check dropped a token (lz4.c:1118-1122) */
    ORACLE_DS_NEXT_MATCH = 4,    /* the _next_match check rewound to a token (lz4.c:1147-1152) */
    ORACLE_DS_REDUCED = 5,       /* a match was shortened (lz4.c:1187-1207) */
    ORACLE_DS_LAST_LITERALS = 6, /* the last literal run was cut (lz4.c:1305-1311) */
    ORACLE_DS_FILLED = 7,        /* the whole input fit without meeting a limit */
    ORACLE_DS_BAD_SIZE = 8       /* n outside 0 .. LZ4_MAX_INPUT_SIZE below the bound (lz4.c:1360) */
};

/* constants: lz4.c:242-249, lz4.c:710-711, lz4.h:214 */
enum {
    K_MINMATCH = 4,
    K_LASTLITERALS = 5,
    K_MFLIMIT = 12,
    K_MINLENGTH = 13,
    K_MAXDIST = 65535,
    K_SMALL_LIMIT = 65536 + 11,
    K_SKIP_TRIGGER = 6
};
#define K_MAX_INPUT 0x7E000000

static uint32_t load32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
static uint64_t load64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }

/* lz4.c:777-783: 4-byte multiplicative hash, 13 bits for the u16 table */
static uint32_t hash_small(const uint8_t* p) { return (load32(p) * 2654435761u) >> 19; }
/* lz4.c:785-791 + :799: on 64-bit LE hosts the u32 table hashes the low 5 bytes, 12 bits */
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

int oracle_lz4_compress_destSize(const uint8_t* src, uint8_t* dst, int* srcSizePtr, int targetDstSize, int acceleration,
                                 int* path);

#define K_FILL_ACCEL_MAX ((1 << 25) - 1)

int oracle_lz4_compress_destSize(const uint8_t* src, uint8_t* dst, int* srcSizePtr, int targetDstSize, int acceleration,
                                 int* path)
{
    match_table T;
    const int n = *srcSizePtr;
    const int64_t olimit = targetDstSize;
    size_t ip, anchor, filled = 0;
    int64_t op;
    size_t mflimit1, matchlimit;
    uint32_t fwdHash;
    int first = ORACLE_DS_FILLED;   /* the first output limit the parse meets */
    int unused;
    if (path == NULL) path = &unused;

    /* lz4.c:1486-1487: success is guaranteed, LZ4_compress_fast_extState (which clamps the acceleration) */
    if (targetDstSize >= oracle_lz4_compress_bound(n)) {
        *path = ORACLE_DS_FAST;
        return oracle_lz4_compress_fast(src, dst, n, targetDstSize, acceleration);
    }
    /* lz4.c:1360-1372 with fillOutput */
    if ((uint32_t)n > (uint32_t)K_MAX_INPUT) { *path = ORACLE_DS_BAD_SIZE; return 0; }
    if (n == 0) {
        *path = ORACLE_DS_EMPTY;
        if (targetDstSize <= 0) return 0;
        dst[0] = 0;
        *srcSizePtr = 0;
        return 1;
    }
    /* lz4.c:985 */
    if (targetDstSize < 1) { *path = ORACLE_DS_NO_ROOM; return 0; }
    /* lz4.c:1490-1493 pass the acceleration unclamped; the two ends are brought into range (see the top) */
    if (acceleration < 1) acceleration = 1;
    if (acceleration > K_FILL_ACCEL_MAX) acceleration = K_FILL_ACCEL_MAX;

    /* lz4.c:1489-1494 table choice; lz4.c:1483 zeroed table */
    memset(T.slot, 0, sizeof(T.slot));
    T.small = (n < K_SMALL_LIMIT);

    ip = 0; anchor = 0; op = 0;
    mflimit1 = (size_t)n - K_MFLIMIT + 1;      /* lz4.c:963 */
    matchlimit = (size_t)n - K_LASTLITERALS;   /* lz4.c:964 */

    if (n < K_MINLENGTH) goto tail;            /* lz4.c:1002 */

    T.slot[tbl_hash(&T, src)] = 0;             /* lz4.c:1005-1010 */
    ip = 1;
    fwdHash = tbl_hash(&T, src + 1);

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
        filled = ip;                                               /* lz4.c:1105 */

        /* --- backward extension (lz4.c:1107-1109) --- */
        while (ip > anchor && cand > 0 && src[ip - 1] == src[cand - 1]) { ip--; cand--; }

        /* --- literals (lz4.c:1112-1136) --- */
        {
            size_t lit = ip - anchor;
            tokenPos = op++;
            /* lz4.c:1118-1122: no room for these literals, a match and the last literals: drop the token */
            if (op + (int64_t)((lit + 240) / 255) + (int64_t)lit + 2 + 1 + K_MFLIMIT - K_MINMATCH > olimit) {
                op--;
                if (first == ORACLE_DS_FILLED) first = ORACLE_DS_LITERALS;
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
            if (op + 2 + 1 + K_MFLIMIT - K_MINMATCH > olimit) {
                op = tokenPos;
                if (first == ORACLE_DS_FILLED) first = ORACLE_DS_NEXT_MATCH;
                goto tail;
            }
            off = ip - cand;
            dst[op++] = (uint8_t)off;                              /* lz4.c:1162 LE16 */
            dst[op++] = (uint8_t)(off >> 8);

            mcode = common_prefix(src + ip + K_MINMATCH, src + cand + K_MINMATCH, src + matchlimit);  /* lz4.c:1182 */
            ip += (size_t)mcode + K_MINMATCH;

            if (op + (1 + K_LASTLITERALS) + (mcode + 240) / 255 > olimit) {
                /* lz4.c:1189-1207: shorten the match to what fits, forget the positions hashed beyond it */
                uint32_t shorter = 15 - 1 + ((uint32_t)(olimit - op) - 1 - K_LASTLITERALS) * 255;
                ip -= mcode - shorter;
                mcode = shorter;
                if (first == ORACLE_DS_FILLED) first = ORACLE_DS_REDUCED;
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
        if (op + (int64_t)last + 1 + (int64_t)((last + 255 - 15) / 255) > olimit) {
            /* lz4.c:1307-1311: as many literals as fit */
            last = (size_t)(olimit - op) - 1;
            last -= (last + 256 - 15) / 256;
            if (first == ORACLE_DS_FILLED) first = ORACLE_DS_LAST_LITERALS;
        }
        if (last >= 15) {
            dst[op++] = 0xF0;
            op = put_runlength(dst, op, last - 15);
        } else {
            dst[op++] = (uint8_t)(last << 4);
        }
        memcpy(dst + op, src + anchor, last);
        op += (int64_t)last;
        *srcSizePtr = (int)(anchor + last);                         /* lz4.c:1327, 1332 */
    }
    *path = first;
    return (int)op;
}

