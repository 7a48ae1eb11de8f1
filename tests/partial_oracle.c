/*
 * partial_oracle.c -- LZ4_decompress_safe_partial on the CPU, written from the reference's rules -- TEST INFRASTRUCTURE.
 *
 * A restatement of the partial_decode instantiation of LZ4_decompress_generic (lz4 v1.10.0, lz4.c:2022-2445 with
 * partialDecoding = 1, noDict), called as LZ4_decompress_safe_partial does (lz4.c:2459-2465).  It follows the reference's
 * control flow decision by decision, because the error value -(ip)-1 depends on which loop reads which byte, but copies
 * bytes one at a time.  One documented deviation: an offset-0 match writes zeros everywhere (lz4.c:2407, :500), also on the
 * cut path of lz4.c:2392-2404, where the reference copies dst onto itself (bytes that depend on what dst held, including
 * what its own over-long copies left there); such a call sets bit 2 of *lastPath.
 * Built by tests/partial_oracle.py.
 */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#define MINMATCH 4
#define LASTLITERALS 5
#define MFLIMIT 12
#define MATCH_SAFEGUARD 12          /* MATCH_SAFEGUARD_DISTANCE, lz4.c:1838 */
#define FASTLOOP_SAFE 64            /* FASTLOOP_SAFE_DISTANCE, lz4.c:1837 */

/* lz4.c:1978-2014: returns 0 on a read past `ilimit` (positions are offsets into src) */
static int read_len(const uint8_t* src, int64_t* ip, int64_t ilimit, int initial, int64_t* out)
{
    uint32_t s;
    int64_t len = 0;
    if (initial && *ip >= ilimit) return 0;
    do {
        s = src[*ip];
        (*ip)++;
        len += s;
        if (*ip > ilimit) return 0;
    } while (s == 255);
    *out = len;
    return 1;
}

static void copy_match(uint8_t* dst, int64_t op, uint32_t offset, int64_t len)
{
    int64_t k;
    for (k = 0; k < len; k++) dst[op + k] = offset ? dst[op + k - offset] : 0;
}

/* Returns the reference's result; *lastPath: 1 = stopped after literals, 2 = stopped in a match, 0 = none; bit 2: see above */
int oracle_lz4_decompress_safe_partial(const uint8_t* src, uint8_t* dst, int srcSize, int targetOutputSize,
                                       int dstCapacity, int* lastPath)
{
    const int outputSize = targetOutputSize < dstCapacity ? targetOutputSize : dstCapacity;   /* lz4.c:2461 */
    const int64_t n = srcSize, oend = outputSize;
    int64_t ip = 0, op = 0, length = 0, add = 0;
    uint32_t token = 0, offset = 0;
    *lastPath = 0;
    if (src == NULL || outputSize < 0) return -1;                    /* lz4.c:2036 */
    if (outputSize == 0) return 0;                                   /* lz4.c:2066 */
    if (srcSize <= 0) return -1;                                     /* lz4.c:2069 (a negative size: rejected here too) */

    if (oend - op >= FASTLOOP_SAFE) {                                /* lz4.c:2076-2209 */
        for (;;) {
            token = src[ip++];
            length = token >> 4;
            if (length == 15) {
                if (!read_len(src, &ip, n - 15, 1, &add)) goto error;
                length += add;
                if (op + length > oend - 32 || ip + length > n - 32) goto safe_literal_copy;
            } else if (ip > n - 17) {
                goto safe_literal_copy;
            }
            memcpy(dst + op, src + ip, (size_t)length);
            ip += length; op += length;
            offset = (uint32_t)src[ip] | ((uint32_t)src[ip + 1] << 8);
            ip += 2;
            length = token & 15;
            if (length == 15) {
                if (!read_len(src, &ip, n - LASTLITERALS + 1, 0, &add)) goto error;
                length += add;
            }
            length += MINMATCH;
            if (op + length >= oend - FASTLOOP_SAFE) goto safe_match_copy;
            if ((int64_t)offset > op) goto error;                    /* lz4.c:2161 */
            copy_match(dst, op, offset, length);
            op += length;
        }
    }

    for (;;) {                                                       /* lz4.c:2215-2435 */
        token = src[ip++];
        length = token >> 4;
        if (length != 15 && ip < n - 16 && op <= oend - 32) {        /* lz4.c:2230-2261 */
            memcpy(dst + op, src + ip, (size_t)length);
            op += length; ip += length;
            length = token & 15;
            offset = (uint32_t)src[ip] | ((uint32_t)src[ip + 1] << 8);
            ip += 2;
            if (length != 15 && offset >= 8 && (int64_t)offset <= op) {
                copy_match(dst, op, offset, length + MINMATCH);
                op += length + MINMATCH;
                continue;
            }
            goto copy_match_len;
        }
        if (length == 15) {
            if (!read_len(src, &ip, n - 15, 1, &add)) goto error;
            length += add;
        }
safe_literal_copy:
        if (op + length > oend - MFLIMIT || ip + length > n - (2 + 1 + LASTLITERALS)) {   /* lz4.c:2279 */
            if (ip + length > n) length = n - ip;                    /* lz4.c:2295-2298 */
            if (op + length > oend) length = oend - op;              /* lz4.c:2301-2305 */
            memmove(dst + op, src + ip, (size_t)length);
            ip += length; op += length;
            if (op == oend || ip >= n - 2) { *lastPath |= 1; break; }  /* lz4.c:2328 */
        } else {
            memcpy(dst + op, src + ip, (size_t)length);
            ip += length; op += length;
        }
        offset = (uint32_t)src[ip] | ((uint32_t)src[ip + 1] << 8);
        ip += 2;
        length = token & 15;
copy_match_len:
        if (length == 15) {                                          /* lz4.c:2342-2347 */
            if (!read_len(src, &ip, n - LASTLITERALS + 1, 0, &add)) goto error;
            length += add;
        }
        length += MINMATCH;
safe_match_copy:
        if ((int64_t)offset > op) goto error;                        /* lz4.c:2356 */
        if (op + length > oend - MATCH_SAFEGUARD) {                  /* lz4.c:2392-2404 */
            const int64_t m = length < oend - op ? length : oend - op;
            copy_match(dst, op, offset, m);
            if (offset == 0 && m > 0) *lastPath |= 4;
            op += m;
            if (op == oend) { *lastPath |= 2; break; }
            continue;
        }
        copy_match(dst, op, offset, length);
        op += length;
    }
    return (int)op;                                                  /* lz4.c:2439 */
error:
    return (int)(-ip) - 1;                                           /* lz4.c:2443 */
}
