"""CPU pin of the hand-made blocks of the hostile decode corpus (tests/gpu_util.py, used by tests/test_gpu_decode_routes.py).

The GPU route tests rely on these blocks sitting exactly on a kernel's edge.  The emulators compile the device's own text
(tests/emul/), so if a constant or a kernel rule moves, this fails here instead of the GPU corpus silently losing its
edge cases:
  - the run-overflow blocks give 20 477 / 20 481 runs and the rows kernel hands the second one to the generic kernel;
  - the sequence-count blocks have 8 191, 8 192 and 8 193 sequences for the one-thread scan;
  - the tiles kernel hands the 200 KB block of run-dense sequences to the generic kernel;
  - the event blocks are rejected by the oracle where the corpus says they are.
"""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle.pyoracle import Oracle
from gpu_util import (RUNS_ABOVE, RUNS_BELOW, event_block, hostile_corpus, run_block, seq_count_block)

HERE = os.path.dirname(os.path.abspath(__file__))
ROWS_MAX_RUNS = 20480
HANDOFF = -1000002                   # the emulators' code for "more runs than the table holds: generic kernel"


def _build(tmp_path_factory, name):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp(name) / ("lib%s.so" % name))
    subprocess.run([gxx, "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-o", so,
                    os.path.join(HERE, "emul", name + ".cpp")], check=True)
    return C.CDLL(so)


@pytest.fixture(scope="module")
def rows(tmp_path_factory):
    lib = _build(tmp_path_factory, "rows_emul")
    lib.rows_emulate.restype = C.c_int
    lib.rows_emulate.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_char_p, C.c_int, C.c_int, C.POINTER(C.c_longlong)]

    def run(comp, cap):
        out = C.create_string_buffer(cap)
        stats = (C.c_longlong * 5)()
        r = lib.rows_emulate(comp, len(comp), cap, out, 0, 4, stats)
        return r, out.raw[:max(r, 0)], list(stats)
    return run


@pytest.fixture(scope="module")
def scan(tmp_path_factory):
    lib = _build(tmp_path_factory, "scan_emul")
    lib.scan_host.restype = C.c_int
    lib.scan_host.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_uint32), C.c_void_p]

    def run(comp, cap):
        buf = np.zeros(len(comp) + 64, dtype=np.uint8)
        buf[:len(comp)] = np.frombuffer(comp, dtype=np.uint8)
        marks = np.zeros(lib.scan_host_max_seq(), dtype=np.uint32)
        ns = C.c_uint32(0)
        r = lib.scan_host(buf.ctypes.data, len(comp), cap, C.byref(ns), marks.ctypes.data)
        return r, ns.value
    return run


@pytest.fixture(scope="module")
def tiles(tmp_path_factory):
    lib = _build(tmp_path_factory, "tiles_emul")
    lib.tiles_emulate.restype = C.c_int
    lib.tiles_emulate.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_char_p, C.c_int, C.POINTER(C.c_longlong)]

    def run(comp, cap):
        out = C.create_string_buffer(cap)
        stats = (C.c_longlong * 6)()
        r = lib.tiles_emulate(comp, len(comp), cap, out, 4, stats)
        return r, list(stats)
    return run


def test_run_overflow_blocks_hand_off_from_the_rows_kernel(rows):
    orc = Oracle()
    below, above = run_block(RUNS_BELOW), run_block(RUNS_ABOVE)
    for cap in (32768, 65535, 65536):
        want = orc.decompress(below, cap)
        assert want[0] == 6 * RUNS_BELOW + 29
        r, data, st = rows(below, cap)
        assert (r, data) == want and st[0] == 4 * RUNS_BELOW + 1 <= ROWS_MAX_RUNS
        r, _, st = rows(above, cap)
        assert orc.decompress(above, cap)[0] == 6 * RUNS_ABOVE + 29
        assert r == HANDOFF and st[0] == 4 * RUNS_ABOVE + 1 > ROWS_MAX_RUNS
    for k, ml in ((7277, 8), (6549, 9)):                # the denser blocks of offset-1 matches of 8 and 9 bytes
        blk = run_block(k, ml)
        assert orc.decompress(blk, 65536)[0] == k * (ml + 1) + 29
        assert rows(blk, 65536)[0] == HANDOFF


def test_sequence_count_blocks_straddle_the_mark_table(scan, rows):
    orc = Oracle()
    for k in (8191, 8192, 8193):
        blk = seq_count_block(k)
        want = orc.decompress(blk, 65536)
        assert want[0] == 4 * k + 13
        assert scan(blk, 65536) == (want[0], k)
        if k <= 8192:                                    # the rows kernel takes it
            r, data, _ = rows(blk, 65536)
            assert (r, data) == want
        else:                                            # one sequence more than the mark table: generic kernel
            assert rows(blk, 65536)[0] == -1000001


def test_big_run_dense_block_hands_off_from_the_tiles_kernel(tiles):
    blk = run_block(33333)
    want = Oracle().decompress(blk, 300000)[0]
    assert want == 6 * 33333 + 29
    r, st = tiles(blk, 300000)
    assert r == HANDOFF and st[1] > ROWS_MAX_RUNS


def test_event_blocks_fail_where_the_corpus_says(scan):
    orc = Oracle()
    rng = np.random.default_rng(4)
    for cap in (16384, 20000, 32768, 65535, 65536):
        for q in range(4):
            for kind in ("offset", "capacity"):
                blk = event_block(rng, cap, q, kind)
                assert 4096 <= len(blk) <= 65535
                r = orc.decompress(blk, cap)[0]
                assert r < 0, (cap, q, kind)
                assert scan(blk, cap)[0] == r
                if kind == "offset":                     # the error position lies in the quarter it was put in
                    assert q * len(blk) // 4 < -r - 1 < (q + 1) * len(blk) // 4, (cap, q, -r - 1, len(blk))


def test_corpus_has_accepted_and_rejected_blocks():
    orc = Oracle()
    for cap in (64, 16384, 65536):
        corpus = hostile_corpus(orc, cap)
        rets = [orc.decompress(b, cap)[0] for _, b in corpus]
        assert sum(r > 0 for r in rets) >= 20 and sum(r < 0 for r in rets) >= 60, (cap, len(corpus))
