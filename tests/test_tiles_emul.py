"""CPU check of the tiles expand kernel's arithmetic (blocks above 64 KB: lz4_kernels.cu lz4_expand_tiles_kernel).

tests/emul/tiles_emul.cpp compiles the same text as the device (lz4_scan_core.h wide marks, lz4_rows_core.h
rw_parse_wide / rw_tile_runs) and replays scan, tile index, and every tile's passes and waves on reference-compressed
and hand-made big blocks; the result is compared with the oracle's LZ4_decompress_safe: return value and bytes.  This pins
the clipping of sequences at tile edges, the first-sequence index and the three kinds of wave source (compressed byte,
byte of this tile, byte of an earlier tile) before the kernel runs on a GPU.
"""
import ctypes as C
import os

import numpy as np
import pytest

import host_build
from oracle.pyoracle import Oracle, Reference, have_reference

HERE = os.path.dirname(os.path.abspath(__file__))
TILE = 61440


@pytest.fixture(scope="module")
def emul():
    return host_build.require()


def run(lib, comp, cap, rpt=4):
    out = C.create_string_buffer(cap)
    stats = (C.c_longlong * 6)()
    r = lib.tiles_emulate(bytes(comp), len(comp), cap, out, rpt, stats)
    return r, out.raw[:max(r, 0)], list(stats)


def big_inputs():
    codec = Reference() if have_reference() else Oracle()
    rng = np.random.default_rng(5)
    out = []
    for proba, seed, size in ((0.5, 0, 4 << 20), (0.9, 1, 1 << 20), (0.2, 2, 300000), (0.99, 3, 700001), (0.0, 4, 200000)):
        out.append(("P%g/%d" % (proba, size), bytes(codec.datagen(size, proba, seed))))
    for period in (1, 2, 3, 4, 7, 8, 255, 4096, 61439, 61440, 61441, 65535):
        seedb = bytes(rng.integers(0, 256, period, dtype=np.uint8))
        out.append(("period%d" % period, (seedb * (400000 // period + 2))[:int(rng.integers(70000, 400000))]))
    out.append(("zeros1m", b"\x00" * (1 << 20)))
    words = [bytes(rng.integers(97, 123, int(rng.integers(2, 9)), dtype=np.uint8)) for _ in range(300)]
    text = b" ".join(words[int(i)] for i in rng.integers(0, 300, 60000))
    out.append(("text", text[:250000]))
    # long literal stretches and long matches that straddle several tile boundaries
    noise = bytes(rng.integers(0, 256, 200000, dtype=np.uint8))
    out.append(("noise+copy", noise + noise[:150000] + b"\x00" * 130000 + noise[100:90000]))
    out.append(("tile-exact", (text * 3)[:2 * TILE]))
    out.append(("tile+1", (text * 3)[:2 * TILE + 1]))
    out.append(("tile-1", (text * 3)[:2 * TILE - 1]))
    return codec, out


def test_tiles_emulator_matches_the_oracle_on_big_blocks(emul):
    codec, inputs = big_inputs()
    orc = Oracle()
    hist = 0
    for name, raw in inputs:
        ret, comp = codec.compress(np.frombuffer(raw, dtype=np.uint8), 1)
        assert ret > 0, name
        for cap in (len(raw), len(raw) + 777):
            if cap <= 65536:
                continue
            r, got, st = run(emul, comp, cap)
            assert r == len(raw), (name, cap, r, st)
            assert st[3] == 0, (name, "illegal reads", st)
            assert got == raw, (name, "bytes differ", st)
            hist += st[5]
        er, eo = orc.decompress(comp, len(raw))
        assert er == len(raw) and eo == raw
    assert hist > 0                                   # matches that reach into an earlier tile were exercised


def test_tiles_emulator_hand_made_sequences(emul):
    """offset 0 and self-overlapping matches that start in one tile and end in another; matches whose source is the very first byte"""
    def block(seqs, last_lits):
        out = bytearray()
        for lits, off, mlen in seqs:
            ll, ml = len(lits), mlen - 4
            out.append((min(ll, 15) << 4) | min(ml, 15))
            if ll >= 15:
                r = ll - 15
                while r >= 255: out.append(255); r -= 255
                out.append(r)
            out += lits
            out += bytes([off & 255, off >> 8])
            if ml >= 15:
                r = ml - 15
                while r >= 255: out.append(255); r -= 255
                out.append(r)
        ll = len(last_lits)
        out.append(min(ll, 15) << 4)
        if ll >= 15:
            r = ll - 15
            while r >= 255: out.append(255); r -= 255
            out.append(r)
        out += last_lits
        return bytes(out)
    orc = Oracle()
    rng = np.random.default_rng(9)
    lit = lambda k: bytes(rng.integers(1, 256, k, dtype=np.uint8))
    cases = {
        "rle across two tile edges": [(lit(1000), 1, 150000), (lit(10), 3, 70000)],
        "offset 0 across a tile edge": [(lit(TILE - 10), 0, 100), (lit(5), 2, 9000)],
        "period = tile": [(lit(TILE), TILE, 3 * TILE + 17)],
        "far sources": [(lit(65535), 65535, 65535), (lit(3), 65535, 65535), (lit(0), 65535, 200000)],
        "short matches at every edge": [(lit(TILE - 2), 5, 4)] + [(lit(TILE - 4), 7, 4) for _ in range(4)],
    }
    for name, seqs in cases.items():
        comp = block(seqs, lit(5))
        er, eo = orc.decompress(comp, 1 << 20)
        assert er > 65536, (name, er)
        r, got, st = run(emul, comp, 1 << 20)
        assert r == er and got == eo and st[3] == 0, (name, r, er, st)
        er2, eo2 = orc.decompress(comp, er)               # exact capacity: the end-of-block rules may reject a hand-made block
        r, got, st = run(emul, comp, er)
        assert r == er2 and (r <= 0 or got == eo2) and st[3] == 0, (name, "exact capacity", r, er2, st)


def test_tiles_emulator_random_sequence_structures(emul):
    """Randomly structured big blocks: literal runs from 0 to 70 000 bytes, matches from 4 to 150 000 bytes at offsets from 1 to
    65 535 (self-overlapping ones included), so that runs start, end and straddle tile edges in every way."""
    orc = Oracle()
    rng = np.random.default_rng(2026)

    def ext(v, out):
        if v >= 15:
            r = v - 15
            while r >= 255:
                out.append(255)
                r -= 255
            out.append(r)

    for case in range(150):
        out = bytearray()
        produced = 0
        target = int(rng.integers(70_000, 500_000))
        while produced < target:
            kind = rng.integers(0, 10)
            ll = int(rng.choice([0, 1, 3, 14, 15, 16, 300, int(rng.integers(0, 70_000))], p=[.2, .15, .15, .1, .1, .1, .1, .1])) if kind else int(rng.integers(60_000, 70_000))
            if produced == 0 and ll == 0:
                ll = 1
            mlen = int(rng.choice([4, 5, 18, 19, 20, 270, int(rng.integers(4, 150_000))], p=[.25, .15, .1, .1, .1, .1, .2]))
            off = int(rng.choice([1, 2, 3, 4, 7, 8, 255, 4096, 61439, 61440, 61441, 65535, int(rng.integers(1, 65536))]))
            off = max(1, min(off, produced + ll))
            out.append((min(ll, 15) << 4) | min(mlen - 4, 15))
            ext(ll, out)
            out += bytes(rng.integers(0, 256, ll, dtype=np.uint8))
            out += bytes([off & 255, off >> 8])
            ext(mlen - 4, out)
            produced += ll + mlen
        last = bytes(rng.integers(0, 256, int(rng.integers(5, 40)), dtype=np.uint8))
        out.append(min(len(last), 15) << 4)
        ext(len(last), out)
        out += last
        comp = bytes(out)
        er, eo = orc.decompress(comp, 1 << 20)
        assert er > 65536, (case, er)
        for cap in (er + 100, er):
            er2, eo2 = orc.decompress(comp, cap)
            r, got, st = run(emul, comp, cap)
            assert r == er2 and (r <= 0 or got == eo2) and st[3] == 0, (case, cap, r, er2, st)
