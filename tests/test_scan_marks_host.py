"""Where the scans leave their marks (lz4_b200/csrc/lz4_scan_core.h, MarkSink), on the host build of the same text.

The scans write a block's marks in whole 32-byte chunks; the words of a chunk the walk does not own are written one
by one.  A block's table starts at `marks + b * markStride` words and markStride = capacity / 4 + 2 is rarely a
multiple of 8, so the table starts at any word of a chunk.  Here every table is placed at each of the 8 word phases
of a chunk inside a buffer of sentinel words, and the words the scan leaves must be the same at every phase: the
true marks of an accepted block, nothing outside [0, min(sequences, markCap)) of the table, and for a rejected or
capacity-limited block the same words whatever the phase.  The split and the parallel scan (whose lanes share
chunks at the edges of their parts) must leave the one-thread scan's marks."""
import ctypes as C
import os

import numpy as np
import pytest

import big_corpus as bc
import host_build
from gpu_util import corrupt, lz4_seq, seq_count_block
from oracle.pyoracle import Oracle
from test_scan_core_host import true_marks

HERE = os.path.dirname(os.path.abspath(__file__))
SENT = 0xEEEEEEEE
GUARD = 16                      # sentinel words on either side of a table


@pytest.fixture(scope="module")
def lib():
    return host_build.require()


def place_block(block, shift):
    """the block at byte `shift` of a 16-byte granule, 16 readable bytes on either side"""
    n = len(block)
    buf = np.full(n + 64, 0xEE, dtype=np.uint8)
    pad = (-buf.ctypes.data) % 16 + 16 + shift
    buf[pad:pad + n] = np.frombuffer(bytes(block), dtype=np.uint8)
    return buf, buf.ctypes.data + pad


def run(lib, which, block, cap, mark_cap, phase, shift=0):
    """-> (ret, nseq, the words of a table of mark_cap words at word `phase` of a 32-byte chunk, with GUARD sentinel
    words before and after it)"""
    buf, src = place_block(block, shift)
    words = np.full(mark_cap + 2 * GUARD + 16, SENT, dtype=np.uint32)
    first = ((-words.ctypes.data) % 32) // 4 + GUARD + phase     # word `phase` of a chunk, GUARD words in
    table = words.ctypes.data + 4 * first
    ns = C.c_uint32(0)
    st = (C.c_int * 3)()
    n = len(block)
    if which == "thread":
        r = lib.scan_host_cap(src, n, cap, C.byref(ns), table, mark_cap)
    elif which == "split":
        r = lib.scan_split_host(src, n, cap, C.byref(ns), table, mark_cap, st)
    elif which == "par":
        assert mark_cap == 8192
        r = lib.scan_par_host(src, n, cap, C.byref(ns), table, st, bc.LANES)
    elif which == "thread-wide":
        r = lib.scan_thread_host_wide(src, n, cap, C.byref(ns), table, mark_cap // 2)
    else:
        r = lib.scan_par_host_wide(src, n, cap, C.byref(ns), table, mark_cap // 2, st, bc.LANES)
    del buf
    return r, ns.value, words[first - GUARD:first + mark_cap + GUARD].copy()


def check_block(lib, block, cap, mark_cap, shifts=(0,), scans=("thread",), orc=None):
    """every scan at every phase and source shift leaves the same words; an accepted block's are its true marks"""
    want = None
    for which in scans:
        for shift in shifts:
            for phase in range(8):
                r, ns, w = run(lib, which, block, cap, mark_cap, phase, shift)
                assert (w[:GUARD] == SENT).all() and (w[GUARD + mark_cap:] == SENT).all(), \
                    (which, phase, shift, "wrote outside the block's table")
                table = w[GUARD:GUARD + mark_cap]
                if want is None:
                    want = (r, ns, table)
                    if orc is not None:
                        assert r == orc.decompress(bytes(block), cap)[0], (which, cap, r)
                    if r > 0 and mark_cap and not which.endswith("wide"):
                        tm = [m & 0xFFFFFFFF for m in true_marks(block)]
                        k = min(len(tm), mark_cap)
                        assert ns == len(tm)
                        assert table[:k].tolist() == tm[:k], (which, phase, shift)
                        assert (table[k:] == SENT).all(), (which, phase, shift, "marks past the last sequence")
                    continue
                assert (r, ns) == want[:2], (which, phase, shift, r, ns, want[:2])
                if which == scans[0]:                          # the same scan at another phase or shift: every word
                    assert table.tolist() == want[2].tolist(), (which, phase, shift)
                elif r > 0:
                    # another scan: the marks of an accepted block (the split scan's lanes may leave words past the end of
                    # the front loop that the one-thread scan never writes, as they always did)
                    k = min(ns * (2 if which.endswith("wide") else 1), mark_cap)
                    assert table[:k].tolist() == want[2][:k].tolist(), (which, phase, shift, k)
    return want


def test_fixture_block_every_phase_and_shift(lib):
    blk = open(os.path.join(HERE, "golden", "p50_seed0_64k.lz4block"), "rb").read()
    r, ns, _ = check_block(lib, blk, 65536, 8192, shifts=range(16), scans=("thread", "split", "par"))
    assert r == 65536 and ns > 2000


@pytest.mark.parametrize("cap", [1000, 16383, 20000, 65536])
def test_capacities_with_odd_mark_strides(lib, cap):
    """markStride = cap / 4 + 2 (252, 4 097, 5 002, 16 386 -> 8 192): a block's table starts mid-chunk"""
    orc = Oracle()
    mark_cap = min(cap // 4 + 2, 8192)
    rng = np.random.default_rng(cap)
    scans = ("thread", "split") if cap >= 16384 else ("thread",)
    for p in (0.0, 0.5, 1.0):
        raw = orc.datagen(cap, p, int(rng.integers(0, 1 << 30)))
        _, c = orc.compress(raw, 1)
        c = bytes(c)
        check_block(lib, c, cap, mark_cap, shifts=(0, 5, 15), scans=scans, orc=orc)
        for k in range(6):                                     # rejected and capacity-limited blocks
            check_block(lib, corrupt(rng, c), cap, mark_cap, shifts=(k,), orc=orc)
        for c2 in (cap - 1, cap - 70, cap // 2):
            check_block(lib, c, c2, mark_cap, shifts=(3,), orc=orc)


def test_last_byte_at_every_granule_offset(lib):
    """source shifts 0..15 put a block's last byte at every offset of its granule"""
    orc = Oracle()
    for size in (777, 4096, 30001):
        raw = orc.datagen(size, 0.5, size)
        _, c = orc.compress(raw, 1)
        check_block(lib, bytes(c), size, size // 4 + 2, shifts=range(16), orc=orc)


def test_long_runs_and_extension_bytes(lib):
    """literal runs and matches of 1 .. 3 extension bytes, their lengths and offsets at every position of a granule"""
    orc = Oracle()
    rng = np.random.default_rng(7)
    lit = lambda k: bytes(rng.integers(1, 256, k, dtype=np.uint8))
    for lead in range(16):
        seqs = [lz4_seq(lit(1 + lead), 1, 4)]
        for ll, ml in ((14, 18), (15, 19), (16, 270), (269, 4), (270, 523), (530, 600), (40, 70000)):
            seqs.append(lz4_seq(lit(ll), 1 + int(rng.integers(0, 15)), ml))
            seqs += [lz4_seq(lit(int(rng.integers(0, 9))), 1 + int(rng.integers(0, 30)), 4 + int(rng.integers(0, 12)))
                     for _ in range(int(rng.integers(1, 9)))]
        blk = b"".join(seqs) + lz4_seq(lit(20), None)
        size = orc.decompress(blk, 1 << 20)[0]
        assert size > 0
        cap = min(size, 65536)
        check_block(lib, blk, cap, min(cap // 4 + 2, 8192), shifts=(lead, 15 - lead), orc=orc)


def test_blocks_at_the_mark_cap(lib):
    """8 191 .. 8 200 sequences against the 8 192-word table: the table fills, nothing is written past it"""
    for ns in (8191, 8192, 8193, 8200):
        r, got, table = check_block(lib, seq_count_block(ns), 65536, 8192, shifts=(0, 9), scans=("thread", "split", "par"))
        assert r == 4 * ns + 13 and got == ns


def test_wide_marks(lib):
    """two words per sequence (blocks above 64 KB): the one-thread and the parallel scan leave the same words"""
    orc = Oracle()
    raw = orc.datagen(300000, 0.5, 3)
    _, c = orc.compress(raw, 1)
    mark_cap = 2 * (300000 // 4 + 2)
    r, ns, table = check_block(lib, bytes(c), 300000, mark_cap, shifts=(0, 7), scans=("thread-wide", "par-wide"))
    assert r == 300000
    assert table[:2 * ns].tolist() == bc.wide_marks(bc.seq_list(bytes(c))).tolist()
    assert (table[2 * ns:] == SENT).all()
