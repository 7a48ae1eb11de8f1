"""A host model of the parallel-parse compressor (LZ4B200_compress_blocks_parallel, lz4_encode_par.cuh).

The parse is fully specified and does not depend on scheduling (DESIGN.md 3.5), so every input has exactly one correct
output.  This module computes it from the documented rules, not from the kernel's code:

  * n == 0 gives the single token 0x00 (if cap >= 1); n < 13 is the last literals alone; n > 65 536 is not the parallel
    parse's (those blocks are LZ4_compress_fast's, i.e. the oracle's).  The output is all or nothing: 0 if it does not
    fit `cap`.
  * acceleration a is clamped to [1, 65537]; step = 1 for a <= 4, else 1 + (a + 3) // 8.  Only the positions
    p % step == 0 are hashed, inserted and may start a match, and only p <= mflimit = n - 12.  Windows are 8192
    positions long.
  * hash(p) = (le32(p) * 2654435761 mod 2^32) >> 19.
  * A position's candidate is the first that applies of: p - d for the first d in 1..4 with p >= d,
    le32(p - d) == le32(p) and byte[p + 4] == byte[p + 4 - d]; the earliest eligible position q of p's window with
    the same hash, if q < p and le32(q) == le32(p); the latest eligible position of an earlier window with that hash,
    if its 4 bytes equal le32(p).  (Positions enter the table after their window is done, so the candidates do not
    depend on the parse.)
  * Greedy chain from E = 0: take the first position >= E that has a candidate, extend its match 4 bytes at a time up
    to n - 5 - p bytes, E = p + L; across window seams alike.  Backward extension (lz4.c:1107-1109) runs down to the
    previous E.  Sequences are emitted in the usual format; the last literals are [E, n).

Per window the model also reports what the kernel's emit phase sees: the output bytes of the sequences selected in the
window (their literals included, also those carried from earlier windows), whether that exceeds the shared-memory stage
(kEpStage = 8704 bytes; such a window stores directly to global memory), and whether a match or a backward extension
crossed a window seam.
"""
import bisect

import numpy as np

WIN = 8192                 # kEpWin: positions per window
STAGE = WIN + 512          # kEpStage: a window's output is staged in shared memory when out + 16 <= STAGE
ACCEL_MAX = 65537          # lz4.c:58
HASH_MUL = 2654435761      # lz4.c:779
MFLIMIT, LAST_LITERALS, MIN_MATCH, MIN_LENGTH = 12, 5, 4, 13


def step_of(acceleration):
    a = min(max(int(acceleration), 1), ACCEL_MAX)
    return 1 if a <= 4 else 1 + (a + 3) // 8


def _rl(x):
    """bytes of the length extension of a 4-bit field holding x"""
    return 1 + (x - 15) // 255 if x >= 15 else 0


def _ext(x):
    if x < 15:
        return b""
    r = x - 15
    return b"\xff" * (r // 255) + bytes([r % 255])


def candidates(b, step):
    """candidate source position of every position 0 .. n - 12 (-1: none), and the rule that gave it
    (1..4: the short period d, 5: this window's earliest, 6: an earlier window's latest, 0: none)"""
    n = len(b)
    mflimit = n - MFLIMIT
    cand = np.full(mflimit + 1, -1, dtype=np.int64)
    kind = np.zeros(mflimit + 1, dtype=np.int8)
    w = b.astype(np.uint32)
    v = w[0:n - 3] | (w[1:n - 2] << 8) | (w[2:n - 1] << 16) | (w[3:n] << 24)     # le32 of positions 0 .. n - 4
    P = np.arange(0, mflimit + 1, step, dtype=np.int64)                         # the eligible positions
    vp = v[P]
    h = ((vp.astype(np.uint64) * HASH_MUL) & 0xFFFFFFFF) >> 19
    ck = np.full(len(P), -1, dtype=np.int64)
    kk = np.zeros(len(P), dtype=np.int8)
    for d in range(1, 5):
        src = np.maximum(P - d, 0)
        ok = (kk == 0) & (P >= d) & (v[src] == vp) & (b[P + 4] == b[np.maximum(P + 4 - d, 0)])
        ck[ok] = P[ok] - d
        kk[ok] = d
    old = np.full(1 << 13, -1, dtype=np.int64)          # latest eligible position of the earlier windows, per hash
    first = np.zeros(1 << 13, dtype=np.int64)           # earliest eligible position of this window, per hash
    for c0 in range(0, mflimit + 1, WIN):
        lo, hi = np.searchsorted(P, [c0, c0 + WIN])
        Pw, vw, hw = P[lo:hi], vp[lo:hi], h[lo:hi]
        uniq, at = np.unique(hw, return_index=True)
        first[uniq] = Pw[at]
        q = first[hw]
        win_ok = (q < Pw) & (v[q] == vw)
        o = old[hw]
        old_ok = (o >= 0) & (v[np.maximum(o, 0)] == vw)
        free = kk[lo:hi] == 0
        sel_w, sel_o = free & win_ok, free & ~win_ok & old_ok
        ck[lo:hi][sel_w] = q[sel_w]
        kk[lo:hi][sel_w] = 5
        ck[lo:hi][sel_o] = o[sel_o]
        kk[lo:hi][sel_o] = 6
        np.maximum.at(old, hw, Pw)                       # insert: this window's positions, after it is done
    cand[P] = ck
    kind[P] = kk
    return cand, kind


def _lcp(b, i, j, m):
    """common prefix length of b[i:] and b[j:], at most m"""
    k, chunk = 0, 16
    while k < m:
        t = min(chunk, m - k)
        ne = np.flatnonzero(b[i + k:i + k + t] != b[j + k:j + k + t])
        if ne.size:
            return k + int(ne[0])
        k += t
        chunk *= 4
    return m


def parse(data, acceleration=1):
    """The sequences of a block of 13 .. 65 536 bytes: [(literal start, match start, match source, match length,
    selected position)] after backward extension, and the final chain position E (start of the last literals)."""
    b = np.frombuffer(bytes(data), dtype=np.uint8)
    raw = bytes(data)
    n = len(b)
    assert MIN_LENGTH <= n <= 65536
    cand, kind = candidates(b, step_of(acceleration))
    idx = np.flatnonzero(cand >= 0).tolist()
    matchlimit = n - LAST_LITERALS
    seqs, E, k = [], 0, 0
    while True:
        k = bisect.bisect_left(idx, E, k)
        if k == len(idx):
            break
        p = idx[k]
        c = int(cand[p])
        L = MIN_MATCH + _lcp(b, p + MIN_MATCH, c + MIN_MATCH, matchlimit - p - MIN_MATCH)
        s, sc = p, c
        while s > E and sc > 0 and raw[s - 1] == raw[sc - 1]:
            s -= 1
            sc -= 1
        seqs.append((E, s, sc, p + L - s, p))
        E = p + L
    return seqs, E


class Result:
    """ret: the call's return value (0: did not fit); out: the block (bytes of the whole output, whatever cap was);
    windows: per window, [output bytes, staged, a match crossed its end seam, a backward extension crossed its start seam,
    first sequence carries literals of earlier windows]; win_off: output offset where each window's bytes start;
    body: output bytes before the last literals; last: number of last literals; step: positions probed."""


def compress(data, acceleration=1, cap=None, oracle=None):
    """What LZ4B200_compress_blocks_parallel returns for one block and capacity cap (default: compressBound)."""
    raw = bytes(data)
    n = len(raw)
    r = Result()
    r.step, r.windows, r.win_off, r.seqs = step_of(acceleration), [], [], []
    if cap is None:
        cap = n + n // 255 + 16
    if n > 65536:
        assert oracle is not None, "blocks above 64 KB are LZ4_compress_fast's: pass the oracle"
        r.ret, r.out = oracle.compress(raw, acceleration, cap)
        r.body, r.last = None, None
        return r
    if n == 0:
        r.out, r.body, r.last = b"\x00", 0, 0
        r.ret = 1 if cap >= 1 else 0
        return r
    seqs, E = parse(raw, acceleration) if n >= MIN_LENGTH else ([], 0)
    n_win = (n - MFLIMIT + WIN) // WIN if n >= MIN_LENGTH else 0
    wins = [[0, True, False, False, False] for _ in range(n_win)]
    out = bytearray()
    for A, s, c, L, p in seqs:
        w = p // WIN
        ll, ml = s - A, L - MIN_MATCH
        wins[w][0] += 1 + _rl(ll) + ll + 2 + _rl(ml)
        wins[w][2] |= (s + L - 1) // WIN > w                 # the match reaches into a later window
        wins[w][3] |= s // WIN < w                           # the backward extension reaches into an earlier one
        wins[w][4] |= A < w * WIN
        out += bytes([(min(ll, 15) << 4) | min(ml, 15)]) + _ext(ll) + raw[A:s]
        out += bytes([(s - c) & 255, (s - c) >> 8]) + _ext(ml)
    r.body = len(out)
    off = 0
    for wv in wins:
        wv[1] = wv[0] + 16 <= STAGE
        r.win_off.append(off)
        off += wv[0]
    assert off == r.body
    r.last = n - E
    out += bytes([min(r.last, 15) << 4]) + _ext(r.last) + raw[E:]
    r.out = bytes(out)
    r.windows, r.seqs = wins, seqs
    r.ret = len(out) if len(out) <= cap else 0
    return r


# ------------------------------------------------------------------------------------------
# inputs built to reach the parse's edges
# ------------------------------------------------------------------------------------------
def hash_of(word):
    return ((int(word) * HASH_MUL) & 0xFFFFFFFF) >> 19


def colliding_words(rng, target, k):
    """k distinct 32-bit words whose hash is `target`"""
    out = set()
    while len(out) < k:
        v = rng.integers(0, 1 << 32, 1 << 20, dtype=np.uint64)
        h = ((v * HASH_MUL) & 0xFFFFFFFF) >> 19
        out.update(v[h == target].tolist())
    return np.array(sorted(out)[:k], dtype=np.uint32)


def _le32(b, p):
    return int(b[p]) | int(b[p + 1]) << 8 | int(b[p + 2]) << 16 | int(b[p + 3]) << 24


def rle_block(period, seed, n=65536, interleaved=False):
    """period-d data: one run over the whole block after 7 random bytes, or runs of 50 .. 400 bytes between 20 random ones"""
    rng = np.random.default_rng(seed)
    pat = bytes(rng.integers(0, 256, period, dtype=np.uint8))
    if not interleaved:
        return (bytes(rng.integers(0, 256, 7, dtype=np.uint8)) + pat * (n // period + 1))[:n]
    out = bytearray()
    while len(out) < n:
        out += bytes(rng.integers(0, 256, 20, dtype=np.uint8))
        out += (pat * 400)[:int(rng.integers(50, 401))]
    return bytes(out[:n])


def collision_block(k, seed, n=65536, shift_every=0):
    """words drawn from k distinct words of one 13-bit hash; every aligned position shares that hash.  shift_every > 0:
    a random byte after every shift_every words moves the alignment"""
    rng = np.random.default_rng(seed)
    words = colliding_words(rng, int(rng.integers(0, 1 << 13)), k)
    out = bytearray()
    cnt = 0
    while len(out) < n:
        out += int(words[int(rng.integers(0, k))]).to_bytes(4, "little")
        cnt += 1
        if shift_every and cnt % shift_every == 0:
            out.append(int(rng.integers(0, 256)))
    return bytes(out[:n])


def seam_block(seed, n=65536):
    """Random bytes with:
      - a 300-byte copy at 8 092 of the bytes at 1 000: a match that runs over the seam at 8 192;
      - a 300-byte copy at 16 382 of the bytes at 10 000 whose first two positions find no candidate (an earlier word of
        window 1 with the same hash shadows each), so the match is found in window 2 and extended backward over the
        seam at 16 384."""
    rng = np.random.default_rng(seed)
    b = rng.integers(0, 256, n, dtype=np.uint8)
    b[8092:8392] = b[1000:1300]
    src, at = 10000, 16382
    b[at:at + 300] = b[src:src + 300]
    b[at - 1] = b[src - 1] ^ 0x5A
    for k, where in ((0, 9000), (1, 9100)):
        w = colliding_words(rng, hash_of(_le32(b, src + k)), 2)
        w = w[0] if int(w[0]) != _le32(b, src + k) else w[1]
        b[where:where + 4] = np.frombuffer(int(w).to_bytes(4, "little"), dtype=np.uint8)
    return b.tobytes()


def prefix_block(k_bytes, seed, n=65536):
    """k_bytes of random bytes, then 1 000-byte copies of random pieces of them with 10 random bytes between: the first
    sequence carries k_bytes of literals, so its window's output exceeds the shared-memory stage"""
    rng = np.random.default_rng(seed)
    out = bytearray(rng.integers(0, 256, k_bytes, dtype=np.uint8).tobytes())
    while len(out) < n:
        s = int(rng.integers(0, k_bytes - 1000))
        out += out[s:s + 1000] + bytes(rng.integers(0, 256, 10, dtype=np.uint8))
    return bytes(out[:n])


def special_blocks():
    """[(name, block, claim)]: claim is what the block reaches at acceleration 1 ("nonstaged", "seam" -- a match and a
    backward extension over a window seam -- or None)"""
    out = []
    for d in range(1, 9):
        out.append(("rle%d" % d, rle_block(d, d), None))
        out.append(("rle%d-runs" % d, rle_block(d, 100 + d, interleaved=True), None))
    for k, shift in ((2, 0), (8, 0), (64, 0), (64, 37)):
        out.append(("collide%d/%d" % (k, shift), collision_block(k, 7 + k + shift, shift_every=shift), None))
    out.append(("seam", seam_block(11), "seam"))
    for kb in (10, 20, 40):
        out.append(("prefix%dk" % kb, prefix_block(kb * 1024, kb), "nonstaged"))
    return out


def reaches(r, claim):
    """does the model Result r reach `claim` (see special_blocks)"""
    if claim == "nonstaged":
        return any(not w[1] for w in r.windows)
    if claim == "seam":
        return any(w[2] for w in r.windows) and any(w[3] for w in r.windows)
    return True
