"""Blocks above 64 KB for the parallel scan (lz4_scan_par.h), the tile index and the tiles expand kernel, and a
plain-Python restatement of what the scan and the tile index leave in the workspace for a valid block.

Pinned on the CPU by tests/test_big_corpus_emul.py, used on the GPU by tests/test_gpu_big_routes.py."""
import numpy as np

from gpu_util import corrupt, lz4_seq, run_block

TILE = 61440                       # output bytes per tile (kTile, lz4_kernels.cu)
LANES = 128                        # lanes of the parallel scan (kScanLanes)
SP_MIN_BYTES = 2048                # smaller inputs: lane 0 runs the one-thread scan (kSpMinBytes)
TILE_MAX_CAP = 64 << 20            # larger capacities take the generic kernel (kTileMaxCap)


def tiles_of(nbytes):
    return (nbytes + TILE - 1) // TILE


def seg_len(n):
    """input bytes per lane of the parallel scan for an n-byte block (sp_phase0)"""
    return max((n - 26 + LANES) // LANES, 64)


def lane_of(pos, n):
    """the lane whose segment holds token position pos"""
    return min(pos // seg_len(n), LANES - 1)


def ext_len(v):
    """extension bytes of a length field of value v (literal count, or match length - 4)"""
    return 0 if v < 15 else (v - 15) // 255 + 1


# ------------------------------------------------------------------------------------------
# restatement of the scan's sequence list and of the tile index, for a valid block
# ------------------------------------------------------------------------------------------
def seq_list(blk):
    """(token position, match start, offset, match length) of every sequence of a block LZ4_decompress_safe accepts;
    the last sequence has no match: its match start is the decoded size, its offset and length are 0"""
    out, ip, op, n = [], 0, 0, len(blk)
    while True:
        tok = ip
        t = blk[ip]
        ip += 1
        ll = t >> 4
        if ll == 15:
            while True:
                b = blk[ip]
                ip += 1
                ll += b
                if b != 255:
                    break
        ip += ll
        op += ll
        if ip >= n:
            out.append((tok, op, 0, 0))
            return out
        off = blk[ip] | blk[ip + 1] << 8
        ip += 2
        ml = t & 15
        if ml == 15:
            while True:
                b = blk[ip]
                ip += 1
                ml += b
                if b != 255:
                    break
        ml += 4
        out.append((tok, op, off, ml))
        op += ml


def wide_marks(seqs):
    """the wide marks mark_commit stores: {token position, match start} per sequence (uint32 pairs, flattened)"""
    return np.array([(tok, ms) for tok, ms, _, _ in seqs], dtype=np.uint32).reshape(-1)


def tile_first(seqs):
    """tileFirst[t] = min{k : matchStart(k) >= t * TILE} for t = 0 .. tiles(decoded size); nseq where there is none"""
    starts = np.array([ms for _, ms, _, _ in seqs], dtype=np.int64)
    t = np.arange(tiles_of(int(starts[-1])) + 1, dtype=np.int64) * TILE
    return np.searchsorted(starts, t, side="left").astype(np.uint32)


# ------------------------------------------------------------------------------------------
# hand-made blocks
# ------------------------------------------------------------------------------------------
class Stream:
    """an LZ4 block under construction: tokens are put at chosen input positions and matches end at chosen output
    positions; the filler is valid sequences of 8..24 literals and a match of 4..12 bytes 8..200 back"""

    def __init__(self, rng):
        self.b, self.op, self.rng = bytearray(), 0, rng

    def seq(self, lits, off, ml=0):
        pos = len(self.b)
        self.b += lz4_seq(lits, off, ml)
        self.op += len(lits) + ml
        return pos

    def lits(self, k):
        return bytes(self.rng.integers(1, 256, k, dtype=np.uint8))

    def filler(self):
        ll, ml = int(self.rng.integers(8, 25)), int(self.rng.integers(4, 13))
        self.seq(self.lits(ll), min(self.op + ll, int(self.rng.integers(8, 201))), ml)

    def fill_to(self, pos):
        """filler, then one bridge sequence, so that the next token lies at input position pos"""
        if pos == len(self.b):
            return
        while len(self.b) < pos - 64:
            self.filler()
        gap = pos - len(self.b)
        assert gap >= 19, (pos, len(self.b))
        self.seq(self.lits(gap - 4), min(self.op + gap - 4, 8), 4)     # token, 1 length byte, literals, offset
        assert len(self.b) == pos

    def end(self, n):
        """filler and 29 last literals (31 bytes) so that the block has exactly n bytes"""
        self.fill_to(n - 31)
        self.seq(self.lits(29), None)
        assert len(self.b) == n
        return bytes(self.b)


def offset_event(s, valid):
    """3 literals and a match whose offset reaches exactly the output start (valid) or one byte before it; returns the
    token position"""
    opn = s.op + 3
    assert opn + 1 <= 65535
    return s.seq(b"abc", opn if valid else opn + 1, 4)


def capacity_event(s, end):
    """3 literals and an offset-1 match that ends at output position `end`; returns the token position"""
    assert end - s.op - 3 >= 4, (end, s.op)
    return s.seq(b"abc", 1, end - s.op - 3)


def lane_event_blocks(cap, seed):
    """[(name, block, finishing lane)] of blocks whose events sit in chosen lanes of the parallel scan.  The lane that
    finishes a block is the first lane whose walk ends (lz4_scan_par.h sp_finish): the lane of the first offset error
    (offset > output position, lz4.c:2161) or capacity event (match end >= cap - 64, lz4.c:2137/2142), or the lane of the
    front region's end (lane 127 here) when there is neither."""
    rng = np.random.default_rng(seed)
    out = []
    # staged: <= 65 535 input bytes, in shared memory; global: walked in global memory.  The filler makes about 1.2 output
    # bytes per input byte: up to cap - 64 before a capacity event, below 65 535 before an offset error
    n_st = min(48000, cap // 2)
    shapes = [("staged", n_st)] + ([("global", min(200000, int(cap * 0.7)))] if int(cap * 0.7) > 65535 else [])
    lanes = (0, 1, 31, 32, 63, 64, 126, 127)
    for where, n in shapes:
        seg = seg_len(n)
        for lane in lanes:
            for delta in ((0,) if lane == 0 else (-1, 0, 1)):       # tokens at l * seg - 1, l * seg and l * seg + 1
                pos = max(lane * seg + delta, 0) if lane else seg // 2
                if pos < 64 and pos:
                    continue
                want = lane_of(pos, n)
                for valid in (True, False):
                    s = Stream(rng)
                    s.fill_to(pos)
                    if s.op + 4 > 65535:                           # an offset cannot reach before the output start
                        break
                    offset_event(s, valid)
                    out.append(("%s offset%s lane %d%+d" % (where, "-ok" if valid else "", lane, delta), s.end(n),
                                LANES - 1 if valid else want))
                for d in (-1, 0, 1):                               # match end at cap - 65 (no event), cap - 64, cap - 63
                    s = Stream(rng)
                    if pos > 0.3 * n:                              # a long run first, so that the event's match is short
                        s.seq(s.lits(1), 1, max(int(cap - 64 - 1.6 * pos - 2000), 4))
                    s.fill_to(pos)
                    capacity_event(s, cap - 64 + d)
                    nxt = len(s.b)                                 # d = -1: the next sequence has the event
                    if nxt > n - 120:
                        continue
                    out.append(("%s capacity%+d lane %d%+d" % (where, d, lane, delta), s.end(n),
                                want if d >= 0 else lane_of(nxt, n)))
        # two events: the first in stream order wins
        if where == "staged":
            for j, k in ((1, 100), (31, 32), (0, 127)):            # two offset errors
                s = Stream(rng)
                s.fill_to(j * seg + 7 if j else 0)
                offset_event(s, False)
                s.fill_to(k * seg + 7)
                offset_event(s, False)
                out.append(("staged offset lanes %d, %d" % (j, k), s.end(n), j))
            for j, k in ((1, 64), (31, 63)):                       # an offset error, then a capacity event
                s = Stream(rng)
                s.fill_to(j * seg + 3)
                offset_event(s, False)
                s.fill_to(k * seg + 3)
                capacity_event(s, cap - 64)
                if len(s.b) < n - 120:
                    out.append(("staged offset lane %d, capacity lane %d" % (j, k), s.end(n), j))
            if cap - 64 + 60 < 65535:                              # a capacity event, then an offset error in the next lane
                for j in (5, 63):
                    guess = 0
                    for _ in range(6):
                        s = Stream(np.random.default_rng(seed + j))
                        s.fill_to((j + 1) * seg - 36 - 6 - guess)
                        ext = ext_len(cap - 64 - s.op - 3 - 4)
                        p = capacity_event(s, cap - 64)
                        gap = (j + 1) * seg - len(s.b)
                        if 19 <= gap <= 40:
                            s.fill_to((j + 1) * seg)
                            s.seq(b"abc", 65535, 4)
                            out.append(("staged capacity lane %d, offset lane %d" % (lane_of(p, n), j + 1), s.end(n),
                                        lane_of(p, n)))
                            break
                        guess = ext
            # an offset error in the last 26 input bytes (lane 127 finishes the front region; the tail walk finds it)
            s = Stream(rng)
            s.fill_to(n - 20)
            offset_event(s, False)
            s.seq(s.lits(13), None)
            out.append(("staged offset in the tail", bytes(s.b), LANES - 1))
        # a capacity hand-over whose block is accepted: the match ends at cap - 64, then the last literals
        s = Stream(rng)
        s.seq(s.lits(1), 1, max(int(cap - 64 - 1.6 * (n - 400) - 2000), 4))
        s.fill_to(n - 400)
        p = capacity_event(s, cap - 64)
        s.seq(s.lits(29), None)
        out.append(("%s capacity accepted" % where, bytes(s.b), lane_of(p, len(s.b))))
    return out


def sized_block(rng, size, decoded):
    """a valid block of exactly `size` bytes: literals, one offset-1 match, 16 last literals, `decoded` bytes in all (or
    literals alone, when `decoded` is too small for the match)"""
    for last in (16, 17):
        for a in range(15, size):
            ml = decoded - a - last
            if ml >= 4 and 1 + ext_len(a) + a + 2 + ext_len(ml - 4) + 1 + ext_len(last) + last == size:
                lits = bytes(rng.integers(1, 256, a, dtype=np.uint8))
                return lz4_seq(lits, 1, ml) + lz4_seq(bytes(range(1, last + 1)), None)
    for a in range(size - 300, size):
        if 1 + ext_len(a) + a == size and a <= decoded:
            return lz4_seq(bytes(rng.integers(1, 256, a, dtype=np.uint8)), None)
    raise AssertionError((size, decoded))


def threshold_blocks(cap, seed):
    """[(name, block)]: compressed sizes 2 047 / 2 048 (one lane / all lanes) and 65 535 / 65 536 (staged / global walk);
    where the capacity allows, a block of at most 65 535 bytes that decodes to 15 MB and more (staged, many tiles)"""
    rng = np.random.default_rng(seed)
    out = []
    for size in (2047, 2048, 65535, 65536):
        decoded = min(cap - 100, 3 * size + 70000)
        out.append(("size %d" % size, sized_block(rng, size, decoded)))
    if cap >= (15 << 20) + 100000:
        out.append(("size 65535 to 15 MB", sized_block(rng, 65535, (15 << 20) + 4321)))
    return out


def two_back_block(rng, total):
    """at the start of every tile t >= 2, a match whose source lies in tile t - 2 (offset 61 441 .. 65 535)"""
    s = Stream(rng)
    s.seq(s.lits(65535), 65535, 4)                                 # history to point into
    t = 2
    while (t + 1) * TILE < total:
        d = (t * 37) % 1000
        target = t * TILE + d
        while s.op < target - 60:
            s.filler()
        off = 61441 + d + (t * 997) % (65535 - 61441 - d)
        assert target - off < (t - 1) * TILE
        s.seq(s.lits(target - s.op), off, 4 + (t % 40))
        t += 1
    while s.op < total - 60:
        s.filler()
    s.seq(s.lits(total - s.op), None)
    return bytes(s.b)


def dense_tile_block(rng, dense_seqs):
    """filler, with `dense_seqs` run_block sequences (1 literal + an offset-1 match of 5 bytes: 4 runs per 6 output bytes)
    from the start of tile 1 on, then filler to 4 tiles"""
    s = Stream(rng)
    while s.op < TILE - 60:
        s.filler()
    s.seq(s.lits(TILE - s.op), 100, 5)
    s.b += run_block(dense_seqs)[:-31]                             # (without its last literals)
    s.op += 6 * dense_seqs
    while s.op < 4 * TILE - 60:
        s.filler()
    s.seq(s.lits(4 * TILE - s.op), None)
    return bytes(s.b)


def tile_edge_blocks(oracle, cap, seed):
    """[(kind, name, block)]: decoded sizes 61 440 k - 1, k, k + 1; literal runs over several tiles with the next match
    on a tile edge; offset 0 and short-offset matches across a tile edge; sources two tiles back; one run-dense tile"""
    rng = np.random.default_rng(seed)
    lit = lambda k: bytes(rng.integers(1, 256, k, dtype=np.uint8))
    out = []
    for k in (1, 2, 68):
        for d in (-1, 0, 1):
            size = TILE * k + d
            if size <= cap:
                _, c = oracle.compress(oracle.datagen(size, 0.5, 7 * k + d + 2), 1)
                out.append(("tile", "size %d tiles %+d" % (k, d), c))
    for t, d in ((1, 0), (2, 0), (3, 0), (2, -1), (2, 1)):
        if t * TILE + d + 10100 < cap - 64:
            blk = lz4_seq(lit(t * TILE + d), 100, 1000) + lz4_seq(lit(5), 3, 9000) + lz4_seq(lit(20), None)
            out.append(("tile", "literals to tile %d %+d" % (t, d), blk))
    if 4 * TILE + 200 < cap:
        for off in (0, 1, 2, 3, 7, 15):
            blk = lz4_seq(lit(TILE - 10), off, 100) + lz4_seq(lit(TILE), off, 2 * TILE) + lz4_seq(lit(20), None)
            out.append(("tile", "offset %d across edges" % off, blk))
    if 4 * TILE + 100 < cap:
        total = min(cap - 100, 40 * TILE + 777)
        out.append(("two-back", "sources two tiles back", two_back_block(rng, total)))
        out.append(("runs-over", "one run-dense tile", dense_tile_block(rng, 10500)))
        out.append(("runs-fit", "one half-dense tile", dense_tile_block(rng, 3500)))
    return out


DEGENERATE = [("degenerate", b"\x00"), ("degenerate", b"\x10a"), ("degenerate", b"\xc0" + bytes(range(1, 13))),
              ("degenerate", b"")]


def big_corpus(oracle, cap, seed=0):
    """[(kind, block)] for a batch of one capacity cap > 64 KB:
      datagen    P0 / P0.2 / P0.5 / P0.9 / P1 blocks of cap, cap -/+ 1, cap -/+ 64 bytes
      broken     each truncated by one byte, halved, with one byte appended, and corrupted copies
      lane       lane_event_blocks (offset errors and capacity events in chosen lanes of the parallel scan)
      threshold  threshold_blocks
      tile, two-back, runs-over, runs-fit    tile_edge_blocks
      degenerate a 1-byte empty block, 1 literal, 13 literals, no input at all"""
    rng = np.random.default_rng(seed)
    out = []
    n_corrupt = 1 if cap > (1 << 20) else 3
    for p in (0.0, 0.2, 0.5, 0.9, 1.0):
        for n in (cap, cap - 1, cap - 64, cap + 1, cap + 64):
            _, c = oracle.compress(oracle.datagen(n, p, 1000 * seed + int(100 * p) + n % 97), 1)
            out.append(("datagen", c))
            out += [("broken", c[:-1]), ("broken", c[:len(c) // 2]), ("broken", c + b"\x00")]
            out += [("broken", corrupt(rng, c)) for _ in range(n_corrupt)]
    out += [("lane", b) for _, b, _ in lane_event_blocks(cap, seed + 1)]
    out += [("threshold", b) for _, b in threshold_blocks(cap, seed + 2)]
    out += [(k, b) for k, _, b in tile_edge_blocks(oracle, cap, seed + 3)]
    return out + DEGENERATE
