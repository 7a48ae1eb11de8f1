"""The decoder's scan (lz4_b200/csrc/lz4_scan_core.h -- the text the scan kernel compiles for the device),
compiled for the host by g++ and checked against the golden known-answer vectors and the oracle:
return value of LZ4_decompress_safe for valid, corrupted and capacity-limited blocks, number of
sequences and the per-sequence marks.  Test infrastructure only: the library never runs this on the host.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest

import host_build
from oracle.pyoracle import Oracle, Reference, have_reference

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def scan():
    lib = host_build.require()
    entry = lib.scan_host
    max_seq = lib.scan_host_max_seq()

    def run(block, cap, shift=0, want_marks=True):
        """-> (ret, nseq, marks[:min(nseq, max)])  block placed at byte offset 16+shift of a 16-byte aligned buffer"""
        n = len(block)
        buf = np.full(n + 80, 0xEE, dtype=np.uint8)
        base = buf.ctypes.data
        pad = (-base) % 16 + 16 + shift
        buf[pad:pad + n] = np.frombuffer(bytes(block), dtype=np.uint8)
        marks = np.zeros(max_seq, dtype=np.uint32)
        ns = C.c_uint32(0)
        r = entry(base + pad, n, cap, C.byref(ns), marks.ctypes.data if want_marks else None)
        return r, ns.value, marks[:min(ns.value, max_seq)].copy()
    run.max_seq = max_seq
    return run


def true_marks(block):
    """(token position | match start << 16) of every sequence of a VALID block (last sequence: the end of its
    literals), by a plain walk."""
    b, n, p, o, out = bytes(block), len(block), 0, 0, []
    while True:
        tokpos = p
        tok = b[p]
        p += 1
        ll = tok >> 4
        if ll == 15:
            while True:
                s = b[p]
                p += 1
                ll += s
                if s != 255:
                    break
        p += ll
        o += ll
        out.append((tokpos & 0xFFFFFFFF) | ((o << 16) & 0xFFFFFFFF))
        if p >= n:
            return out
        p += 2
        ml = (tok & 15) + 4
        if (tok & 15) == 15:
            while True:
                s = b[p]
                p += 1
                ml += s
                if s != 255:
                    break
        o += ml


def test_golden_decode_vectors(scan):
    cases = json.load(open(os.path.join(HERE, "golden", "kat_decode.json")))["cases"]
    assert len(cases) > 1000
    for i, c in enumerate(cases):
        blk = bytes.fromhex(c["block"])
        r, ns, _ = scan(blk, c["cap"], shift=i % 16)
        assert r == c["ret"], (i, c["cap"], r, c["ret"])
        if r <= 0:
            assert ns == 0 or r == 0


def test_fixture_block_marks(scan):
    blk = open(os.path.join(HERE, "golden", "p50_seed0_64k.lz4block"), "rb").read()
    for shift in range(16):
        r, ns, marks = scan(blk, 65536, shift)
        want = true_marks(blk)
        assert r == 65536 and ns == len(want)
        assert marks.tolist() == [m & 0xFFFFFFFF for m in want[:scan.max_seq]]
    # a larger capacity keeps the walk in the fast loop to the end; a smaller one fails like the reference
    orc = Oracle()
    for cap in (65536 + 64, 65536 + 1000, 65535, 65000, 64, 63, 1):
        assert scan(blk, cap)[0] == orc.decompress(blk, cap)[0]


def test_valid_and_corrupted_blocks_vs_oracle(scan):
    orc = Oracle()
    gen = Reference() if have_reference() else orc
    rng = np.random.default_rng(20260923)
    checked = bad = 0
    for proba in (0.0, 0.2, 0.5, 0.9, 1.0):
        for size in (0, 1, 12, 13, 64, 100, 1000, 4096, 65536, 70000, 200000):
            raw = bytes(gen.datagen(size, proba, int(rng.integers(0, 1 << 30)))) if size else b""
            _, comp = orc.compress(raw, 1)
            comp = bytes(comp)
            for cap in {size, size + 1, size + 64, size + 100, max(size - 1, 0), max(size - 70, 0), size // 2}:
                r, ns, marks = scan(comp, cap, shift=int(rng.integers(0, 16)))
                want, _ = orc.decompress(comp, cap)
                assert r == want, (proba, size, cap, r, want)
                if r > 0:
                    tm = true_marks(comp)
                    assert ns == len(tm)
                    if len(comp) <= 65535 and cap <= 65536:
                        assert marks.tolist() == [m & 0xFFFFFFFF for m in tm[:scan.max_seq]]
                checked += 1
            # corruptions
            for _ in range(60 if size <= 4096 else 12):
                b = bytearray(comp)
                for _ in range(int(rng.integers(1, 4))):
                    mode = int(rng.integers(0, 4))
                    pos = int(rng.integers(0, max(len(b), 1)))
                    if mode == 0 and b:
                        b[pos] = int(rng.integers(0, 256))
                    elif mode == 1 and b:
                        b[pos] = int(rng.choice([0, 0xFF, 0xF0, 0x0F, 0x10, 0x1F]))
                    elif mode == 2 and len(b) > 4:
                        del b[pos:pos + int(rng.integers(1, 4))]
                    else:
                        b[pos:pos] = bytes(rng.integers(0, 256, int(rng.integers(1, 4)), dtype=np.uint8))
                cap = int(rng.choice([size, size + 64, size + 1000, max(size - 5, 0)]))
                r, ns, _ = scan(bytes(b), cap, shift=int(rng.integers(0, 16)))
                want, _ = orc.decompress(bytes(b), cap)
                assert r == want, (proba, size, cap, r, want)
                bad += want < 0
                checked += 1
    assert checked > 2500 and bad > 500, (checked, bad)
