"""CPU check of the partial decode's device text (PARTIAL scan of lz4_scan_core.h, rw_parse<true> of lz4_rows_core.h).

tests/emul/partial_emul.cpp compiles the same text with g++.  On every case of kat_partial.json it must give the
reference's return value and, for every block the rows kernel may take, the checker's bytes rebuilt from the marks and
the clipped runs.  The marks of valid blocks are checked against their sequences: match starts, and the literal start of
the last sequence (16 bits).  4 MB blocks at targets up to 61 440 must fit the rows kernel's consumed-prefix window.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import host_build

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_golden_partial as mg  # noqa: E402


@pytest.fixture(scope="module")
def emul():
    return host_build.require()


def run(lib, src, cap):
    """(ret, nseq, consumed, marks, rebuilt bytes or None) with the mark table the kernel reserves (cap/4 + 2, <= 8192)"""
    mcap = min(cap // 4 + 2, 8192) if 0 < cap <= 65536 else 0
    marks = (C.c_uint32 * max(mcap, 1))()
    ns, used = C.c_uint32(0), C.c_uint32(0)
    out = C.create_string_buffer(max(cap, 1) if mcap else 1)
    r = lib.partial_emulate(bytes(src), len(src), cap, C.byref(ns), C.byref(used), marks if mcap else None, mcap, out)
    ok = mcap and r > 0 and used.value <= 65535 and ns.value <= mcap
    return r, ns.value, used.value, list(marks)[:min(ns.value, mcap)], out.raw[:r] if ok else None


def test_emulated_partial_decode_matches_the_reference(emul, oracle):
    _, groups = mg.golden()
    rebuilt = 0
    for name, cases, rets, _ in groups:
        for (src, t, c), want in zip(cases, rets):
            r, _, used, _, out = run(emul, src, min(t, c))
            assert r == want, (name, t, c)
            if out is not None:
                assert out == oracle.decompress_partial(src, t, c)[1] and used <= len(src), (name, t, c)
                rebuilt += 1
    assert rebuilt > 10000


def test_marks_and_last_sequence_encoding(emul, oracle):
    checked = 0
    for (bid, size, kind, seed) in mg.blocks():
        if not 0 < size <= 65536:
            continue
        raw, comp = mg.make_block(oracle, size, kind, seed)
        seqs = mg.sequences(comp)
        starts = [s[0] for s in seqs] + [seqs[-1][2] if seqs else 0]     # the final literal run starts after the last match
        for t in sorted(x for x in {1, 4, 5, 17, 64, 65, 1000, 4096, 65535, size} if x <= size):
            r, ns, used, marks, out = run(emul, comp, t)
            assert r == t and out in (None, raw[:t]), (bid, t)
            if out is None:                    # consumed > 65 535: the generic kernel's block, no marks needed
                continue
            assert [m >> 16 for m in marks[:ns - 1]] == [s[1] % 65536 for s in seqs[:ns - 1]], (bid, t)
            assert marks[ns - 1] >> 16 == starts[ns - 1] % 65536, (bid, t)
            checked += 1
    assert checked > 100


def test_zero_byte_final_token_at_64k(emul):
    """A block of exactly 65 536 bytes whose last token adds nothing: its start wraps to 0 and every byte is rebuilt"""
    rng = np.random.default_rng(3)
    lit0 = rng.integers(0, 256, 65000, dtype=np.uint8).tobytes()
    lit1 = rng.integers(0, 256, 14, dtype=np.uint8).tobytes()
    # 65 000 literals + an offset-1 match of 504 (op = 65 536 - 32); then the safe loop's shortcut (lz4.c:2230), which has
    # no stop test, takes 14 literals + an 18-byte match up to exactly 65 536; the next token (0x00) stops at once
    blk = bytes([0xFF]) + b"\xff" * 254 + bytes([215]) + lit0 + b"\x01\x00" + bytes([255, 230])
    blk += bytes([0xEE]) + lit1 + b"\x64\x00" + b"\x00"
    want = bytearray(lit0 + lit0[-1:] * 504 + lit1)
    for _ in range(18):
        want.append(want[len(want) - 100])
    r, ns, used, marks, out = run(emul, blk, 65536)
    assert r == 65536 and out == bytes(want)
    assert ns == 3 and used == len(blk) and marks[2] >> 16 == 0 and marks[2] & 0xFFFF == len(blk) - 1


def test_big_blocks_take_the_rows_window_at_61440(emul, oracle):
    n = 0
    for (bid, size, kind, seed) in mg.blocks():
        if size != 4 << 20:
            continue
        raw, comp = mg.make_block(oracle, size, kind, seed)
        for t in (4096, 30000, 61440):
            r, ns, used, _, out = run(emul, comp, t)
            assert r == t and (out is None or out == raw[:t])
            n += out is not None
    assert n >= 12
