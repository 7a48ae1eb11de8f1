"""CPU pin of the corpus of blocks above 64 KB (tests/big_corpus.py, used by tests/test_gpu_big_routes.py).

The GPU tests of routes R5 / R6 rely on these blocks sitting exactly where the corpus says: an event in a chosen lane of
the parallel scan, a compressed size on a threshold of the scan kernel, a tile edge of the tiles kernel.  The emulators
compile the device's own text (tests/emul/), so if a constant or a rule moves, this fails here instead of the GPU corpus
silently losing its edge cases:
  - every lane-event block is finished by the lane the corpus claims (scan_par_host_wide, 128 lanes: stats[2]), with the
    oracle's return value, and the one-thread scan agrees;
  - the threshold blocks have the exact compressed sizes, and the 2 047-byte block is the one the lanes leave to lane 0;
  - the tile-edge blocks decode to the sizes and matches they claim; the tiles emulator hands the run-dense tile to the
    generic kernel and takes the half-dense one; the two-tiles-back blocks read tile t - 2 at the start of every tile;
  - the Python restatement of the wide marks and the tile index (big_corpus.seq_list / wide_marks / tile_first) equals
    the emulators' marks, and the tile index kernel's neighbour rule, on every accepted block.
"""
import ctypes as C
import re

import numpy as np
import pytest

from oracle.pyoracle import Oracle
import big_corpus as bc
import host_build

HANDOFF = -1000002                   # the emulators' code for "more runs than the table holds: generic kernel"
ROWS_MAX_RUNS = 20480
CAPS = (65537, 122880, 300000, 4 << 20)


@pytest.fixture(scope="module")
def scans():
    """(par, thread): scan_par_host_wide with 128 lanes / scan_thread_host_wide -> (return value, nseq, marks, lane)"""
    lib = host_build.require()

    def run(par, blk, cap):
        mcap = cap // 4 + 2
        buf = np.frombuffer(bytes(blk) + b"\xEE" * 64, dtype=np.uint8).copy()
        marks = np.full(2 * mcap, 0xABABABAB, dtype=np.uint32)
        ns = C.c_uint32(0)
        st = (C.c_int * 3)(0, 0, -7)
        if par:
            r = lib.scan_par_host_wide(buf.ctypes.data, len(blk), cap, C.byref(ns), marks.ctypes.data, mcap, st,
                                       bc.LANES)
        else:
            r = lib.scan_thread_host_wide(buf.ctypes.data, len(blk), cap, C.byref(ns), marks.ctypes.data, mcap)
        return r, ns.value, marks[:2 * min(ns.value, mcap)], st[2]
    return run


@pytest.fixture(scope="module")
def tiles():
    lib = host_build.require()

    def run(comp, cap):
        out = C.create_string_buffer(cap)
        stats = (C.c_longlong * 6)()
        r = lib.tiles_emulate(bytes(comp), len(comp), cap, out, 4, stats)
        return r, out.raw[:max(r, 0)], list(stats)
    return run


@pytest.mark.parametrize("cap", CAPS)
def test_lane_events_finish_in_the_claimed_lane(scans, cap):
    orc = Oracle()
    blocks = bc.lane_event_blocks(cap, seed=cap % 1009 + 1)
    lanes, rejected = set(), 0
    for name, blk, lane in blocks:
        want = orc.decompress(blk, cap)[0]
        r, ns, _, got = scans(True, blk, cap)
        assert (r, got) == (want, lane), (cap, name, len(blk), r, want, got, lane)
        assert scans(False, blk, cap)[:2] == (r, ns), (cap, name)
        assert (len(blk) <= 65535) == name.startswith("staged"), (cap, name, len(blk))
        if re.search(r"offset lane|offset in", name):
            assert r < 0, (cap, name)
        if "offset-ok" in name or "capacity accepted" in name:
            assert r > 0, (cap, name)
        lanes.add(lane)
        rejected += r < 0
    assert {0, 1, 31, 32, 63, 64, 126, 127} <= lanes, sorted(lanes)
    assert rejected >= 60 and len(blocks) - rejected >= 20, (len(blocks), rejected)
    names = " | ".join(n for n, _, _ in blocks)
    for part in ("offset lanes", "offset in the tail", "capacity accepted", "capacity-1 lane 127", "capacity+0 lane 64-1"):
        assert part in names, part
    if cap == 65537:
        assert "offset lane 6 |" in names and ", offset lane 64" in names
    else:
        assert "global offset lane 31" in names and "global capacity+1 lane 127+1" in names


@pytest.mark.parametrize("cap", CAPS + (64 << 20,))
def test_threshold_blocks_have_exact_sizes(scans, cap):
    orc = Oracle()
    blocks = bc.threshold_blocks(cap, seed=5)
    sizes = [len(b) for _, b in blocks]
    assert sizes[:4] == [2047, 2048, 65535, 65536]
    for name, blk in blocks:
        want = orc.decompress(blk, cap)[0]
        assert 0 < want <= cap, (cap, name, want)
        r, _, _, lane = scans(True, blk, cap)
        assert r == want
        assert (lane == -1) == (len(blk) < bc.SP_MIN_BYTES), (name, lane)     # -1: lane 0 alone (one-thread scan)
    if cap == 64 << 20:
        assert sizes[4] <= 65535 and orc.decompress(blocks[4][1], cap)[0] >= 15 << 20


def test_tile_edge_blocks(oracle, scans, tiles):
    cap = 4 << 20
    seen = set()
    for kind, name, blk in bc.tile_edge_blocks(oracle, cap, seed=11):
        want, data = oracle.decompress(blk, cap)
        assert want > 0, name
        seqs = bc.seq_list(blk)
        m = re.match(r"size (\d+) tiles ([-+]\d+)", name)
        if m:
            assert want == bc.TILE * int(m.group(1)) + int(m.group(2)), name
        m = re.match(r"literals to tile (\d+) ([-+]\d+)", name)
        if m:
            assert seqs[0][1] == bc.TILE * int(m.group(1)) + int(m.group(2)), name
        r, got, st = tiles(blk, cap)
        if kind == "runs-over":                      # the dense tile has more runs than the table: generic kernel
            assert r == HANDOFF and st[1] > ROWS_MAX_RUNS, (name, st)
        else:
            assert (r, got) == (want, data) and st[3] == 0, (name, r, st)
            if kind == "runs-fit":                   # its neighbour with fewer dense sequences stays in the tiles kernel
                assert 0.75 * ROWS_MAX_RUNS < st[1] <= ROWS_MAX_RUNS, (name, st)
        if kind == "two-back":                       # every tile t >= 2 starts with a match whose source is in tile t - 2
            starts = {}
            for _, ms, off, ml in seqs:
                if ml and ms % bc.TILE < 4096:
                    starts.setdefault(ms // bc.TILE, set()).add((ms - off) // bc.TILE - ms // bc.TILE)
            tl = bc.tiles_of(want)
            assert all(-2 in starts.get(t, ()) for t in range(2, tl - 1)), starts
            assert tl >= 5 and st[5] > 0
        if "offset" in name:
            assert any(off == int(name.split()[1]) and ms // bc.TILE != (ms + ml - 1) // bc.TILE for _, ms, off, ml in seqs)
        seen.add(kind)
    assert seen == {"tile", "two-back", "runs-over", "runs-fit"}


def kernel_tile_index(marks, ns, total):
    """lz4_tile_index_kernel's rule: sequence k serves the tiles between its predecessor's match start and its own"""
    nt = bc.tiles_of(total)
    first = np.full(nt + 1, 0xFFFFFFFF, dtype=np.uint32)
    for k in range(ns):
        t1 = min(int(marks[2 * k + 1]) // bc.TILE, nt)
        t0 = min(int(marks[2 * k - 1]) // bc.TILE, nt) + 1 if k else 0
        first[t0:t1 + 1] = k
        if k + 1 == ns:
            first[t1 + 1:] = ns
    return first


@pytest.mark.parametrize("cap", CAPS)
def test_restatement_equals_the_emulated_marks(oracle, scans, tiles, cap):
    """on every accepted block of the corpus: nseq, the wide marks and tileFirst of the Python restatement equal the
    parallel scan's, the one-thread scan's and the tile index rule's; the tiles emulator hands exactly the run-dense
    blocks to the generic kernel (the slow list the GPU test expects)"""
    checked = tiles_compared = 0
    for kind, blk in bc.big_corpus(oracle, cap, seed=cap % 1009):
        want = oracle.decompress(blk, cap)[0]
        if want <= 0:
            continue
        seqs = bc.seq_list(blk)
        marks = bc.wide_marks(seqs)
        assert seqs[-1][1] == want
        for par in (True, False):
            r, ns, got, _ = scans(par, blk, cap)
            assert (r, ns) == (want, len(seqs)), (cap, kind, par, r, ns, want, len(seqs))
            assert np.array_equal(got, marks), (cap, kind, par)
        first = bc.tile_first(seqs)
        assert np.array_equal(kernel_tile_index(marks, len(seqs), want), first), (cap, kind)
        r, _, st = tiles(blk, cap)
        assert r == (HANDOFF if kind == "runs-over" else want), (cap, kind, r, st)
        checked += 1
        tiles_compared += len(first)
    assert checked >= 40 and tiles_compared >= 60, (checked, tiles_compared)
