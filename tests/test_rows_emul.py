"""CPU check of the rows expand kernel's arithmetic (lz4_b200/csrc/lz4_rows_core.h).

The header is plain C++: the device kernel (lz4_kernels.cu: lz4_expand_rows_kernel) and the emulator
(tests/emul/rows_emul.cpp, built here with g++) compile the same text.  The emulator replays the
kernel's phases thread by thread on reference-compressed and hand-made blocks and the result is
compared with the oracle's LZ4_decompress_safe: return value and bytes.  This pins run splitting
(self-overlapping matches, offset 0), ranks and the wave / hop logic before the kernel runs on a GPU.
"""
import ctypes as C
import os

import numpy as np
import pytest

import host_build
from oracle.pyoracle import Oracle, Reference, have_reference

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emul():
    return host_build.require()


def run(lib, comp, cap, head=0, rpt=4):
    out = C.create_string_buffer(max(cap, 1))
    stats = (C.c_longlong * 5)()
    r = lib.rows_emulate(bytes(comp), len(comp), cap, out, head, rpt, stats)
    return r, out.raw[:max(r, 0)], list(stats)


def raw_blocks():
    codec = Reference() if have_reference() else Oracle()
    out = []
    for proba, seed in ((0.5, 0), (0.9, 1), (0.2, 2), (0.99, 3), (1.0, 4), (0.0, 5)):
        data = codec.datagen(2 * 65536, proba, seed)
        for k in range(2):
            out.append(("P%g/%d" % (proba, k), bytes(data[k * 65536:(k + 1) * 65536])))
    rng = np.random.default_rng(11)
    for period in list(range(1, 20)) + [31, 32, 33, 255, 1000, 4095, 4096, 4097]:
        seedb = bytes(rng.integers(0, 256, period, dtype=np.uint8))
        body = (seedb * (70000 // period + 1))[:int(rng.integers(3000, 65536))]
        out.append(("period%d" % period, body))
    out.append(("zeros64k", b"\x00" * 65536))
    out.append(("zeros_ragged", b"\x00" * 40001))
    words = [bytes(rng.integers(97, 123, int(rng.integers(2, 9)), dtype=np.uint8)) for _ in range(300)]
    text = b" ".join(words[int(i)] for i in rng.integers(0, 300, 14000))[:65536]
    out += [("text", text), ("text24k", text[:24000]), ("tiny", b"abcabcabcabcabcabcabcabcabc" * 3), ("13", b"0123456789abc"),
            ("mixed", bytes(rng.integers(0, 256, 5000, dtype=np.uint8)) + b"\x00" * 20000 + text[:20000] + b"ab" * 5000)]
    return out


def test_rows_kernel_arithmetic_on_compressed_blocks(emul):
    oracle = Oracle()
    n_hops = 0
    for name, raw in raw_blocks():
        r, comp = oracle.compress(raw)
        assert r > 0
        if len(comp) > 65535 or run(emul, comp, len(raw))[0] == -1000001:
            continue                                    # incompressible, or > 8192 sequences: not a block of the smem kernel
        for rpt in (1, 4, 64):                          # wave = 1 KB, 4 KB, the whole block
            for head in (0, 7, 15):
                got, data, st = run(emul, comp, len(raw), head, rpt)
                assert got == len(raw), (name, rpt, head, got)
                assert data == raw, (name, rpt, head)
                assert st[3] == 0, (name, "read of a byte outside the staged block / the final window")
                n_hops += st[1]
        # larger capacity than needed, and capacity exactly as needed + the reference's error when it is too small
        for cap in (min(65536, len(raw) + 100), len(raw)):
            got, data, st = run(emul, comp, cap)
            want, wdata = oracle.decompress(comp, cap)
            assert (got, data) == (want, wdata), (name, cap)
        if len(raw) > 100:
            got, _, _ = run(emul, comp, len(raw) - 1)
            want, _ = oracle.decompress(comp, len(raw) - 1)
            assert got == want and got < 0
    assert n_hops > 0


def _seq(lits, off, mlen):
    """one LZ4 sequence: literals, then a match (offset, length >= 4); off=None: last sequence"""
    ll = len(lits)
    ml = 0 if off is None else mlen - 4
    tok = (min(ll, 15) << 4) | min(ml, 15)
    out = bytearray([tok])
    if ll >= 15:
        x = ll - 15
        while x >= 255:
            out.append(255); x -= 255
        out.append(x)
    out += lits
    if off is not None:
        out += bytes([off & 255, off >> 8])
        if ml >= 15:
            x = ml - 15
            while x >= 255:
                out.append(255); x -= 255
            out.append(x)
    return bytes(out)


def test_rows_kernel_hand_made_blocks(emul):
    """offset 0 (the reference zero-fills), chains of overlapping matches, matches that read matches of the same wave"""
    oracle = Oracle()
    rng = np.random.default_rng(5)
    cases = []
    lit = lambda k: bytes(rng.integers(1, 256, k, dtype=np.uint8))
    tail = lit(12)
    for off in (0, 1, 2, 3, 5, 8, 13):
        for mlen in (4, 5, 8, 19, 64, 300, 5000, 60000):
            if mlen + 40 > 65536:
                continue
            cases.append(_seq(lit(20), off, mlen) + _seq(lit(3), 7, 9) + _seq(tail, None, 0))
    # many short matches each reading the previous one (long hop chains inside a wave)
    blk = _seq(lit(16), 4, 4)
    for _ in range(1500):
        blk += _seq(b"", 4, 4) + _seq(lit(1), 3, 7)
    cases.append(blk + _seq(tail, None, 0))
    # alternating offset-0 runs and literal runs
    blk = b""
    for k in range(60):
        blk += _seq(lit(5 + k), 0, 4 + 7 * k)
    cases.append(blk + _seq(tail, None, 0))
    for comp in cases:
        for cap in (65536, 40000):
            want, wdata = oracle.decompress(comp, cap)
            for rpt in (1, 4, 64):
                got, data, st = run(emul, comp, cap, 3, rpt)
                assert (got, data) == (want, wdata), (comp[:16].hex(), cap, rpt, got, want)
                assert st[3] == 0


def test_rows_kernel_golden_decode_vectors(emul):
    """the reference-made known answers (tests/golden/kat_decode.json): return value and bytes"""
    import json
    cases = json.load(open(os.path.join(HERE, "golden", "kat_decode.json")))["cases"]
    n = 0
    for v in cases:
        comp = bytes.fromhex(v["block"])
        cap = int(v["cap"])
        if not (0 < len(comp) <= 65535 and 0 < cap <= 65536):
            continue
        got, data, st = run(emul, comp, cap)
        assert got not in (-1000001, -1000002, -1000003, -1000004)
        assert got == int(v["ret"]), (v["block"][:40], cap, got, v["ret"])
        if got > 0:
            assert data == bytes.fromhex(v["out"]) and st[3] == 0
        n += 1
    assert n > 100
