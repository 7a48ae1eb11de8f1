"""CPU check of the intra-block parallel scan (lz4_b200/csrc/lz4_scan_par.h; device: lz4_scan_par_kernel).

The header is compiled for the host and its lanes are run phase by phase (tests/emul/scan_par_emul.cpp)
for 32, 128 and 256 lanes per block;
for every block -- valid, corrupted, capacity-limited, 64 KB to 4 MB -- the result must be IDENTICAL to
the one-thread scan of lz4_scan_core.h (itself pinned to the golden vectors and the oracle by
tests/test_scan_core_host.py): return value, sequence count, and the marks of every sequence.
"""
import ctypes as C
import os

import numpy as np
import pytest

import host_build
from oracle.pyoracle import Oracle, Reference, have_reference

HERE = os.path.dirname(os.path.abspath(__file__))
MAX_SEQ = 8192


@pytest.fixture(scope="module")
def lib():
    return host_build.require()


@pytest.fixture(params=[32, 128, 256])
def lanes(request):
    return request.param


def both(lib, lanes, block, cap, shift=0, with_marks=True):
    n = len(block)
    buf = np.full(n + 32, 0xEE, dtype=np.uint8)
    base = buf.ctypes.data
    pad = (-base) % 8 + 8 + shift
    buf[pad:pad + n] = np.frombuffer(bytes(block), dtype=np.uint8)
    m1 = np.full(MAX_SEQ, 0xABABABAB, dtype=np.uint32)
    m2 = np.full(MAX_SEQ, 0xABABABAB, dtype=np.uint32)
    n1, n2 = C.c_uint32(0), C.c_uint32(0)
    stats = (C.c_int * 3)()
    r1 = lib.scan_host(base + pad, n, cap, C.byref(n1), m1.ctypes.data if with_marks else None)
    r2 = lib.scan_par_host(base + pad, n, cap, C.byref(n2), m2.ctypes.data if with_marks else None, stats, lanes)
    k = min(n1.value, MAX_SEQ)
    return (r1, n1.value, m1[:k]), (r2, n2.value, m2[:k]), list(stats)


def corrupt(rng, comp):
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
    return bytes(b)


def test_parallel_scan_equals_one_thread_scan(lib, lanes):
    orc = Oracle()
    gen = Reference() if have_reference() else orc
    rng = np.random.default_rng(20260924)
    checked = errors = rounds = 0
    for proba in (0.0, 0.2, 0.5, 0.9, 0.99, 1.0):
        for size in ((2000, 4096, 10000, 65536, 65536, 70000, 300000, 1 << 20, 4 << 20) if lanes == 128 else (4096, 65536, 70000, 1 << 20)):
            raw = bytes(gen.datagen(size, proba, int(rng.integers(0, 1 << 30))))
            _, comp = orc.compress(raw, 1)
            comp = bytes(comp)
            caps = {size, size + 1, size + 64, size + 1000, size - 1, size - 70, size // 2, 64, 63}
            for cap in caps:
                a, b, st = both(lib, lanes, comp, cap, shift=int(rng.integers(0, 4)), with_marks=(len(comp) <= 65535 and cap <= 65536))
                assert a[0] == b[0] and a[1] == b[1], (proba, size, cap, a[:2], b[:2], st)
                assert np.array_equal(a[2], b[2]), (proba, size, cap, st)
                if cap == size:
                    assert a[0] == size
                    assert st[0] <= lanes                  # the fix-up converges within one round per lane
                    if proba == 0.5 and size >= 65536:
                        rounds = max(rounds, st[0])
                checked += 1
            for _ in range(10 if size <= 70000 else 3):
                bad = corrupt(rng, comp)
                cap = int(rng.choice([size, size + 64, size + 1000, max(size - 5, 0)]))
                a, b, st = both(lib, lanes, bad, cap, shift=int(rng.integers(0, 4)), with_marks=(len(bad) <= 65535 and cap <= 65536))
                assert a[0] == b[0] and a[1] == b[1], (proba, size, cap, a[:2], b[:2], st)
                assert np.array_equal(a[2], b[2])
                errors += a[0] < 0
                checked += 1
    assert checked > 300 and errors > 40
    assert rounds <= {32: 4, 128: 16, 256: 32}[lanes]   # P50: the re-walks die out after a few rounds (longest run of unsynchronised lanes)


def test_fixture_block_and_special_shapes(lib, lanes):
    blk = open(os.path.join(HERE, "golden", "p50_seed0_64k.lz4block"), "rb").read()
    for cap in (65536, 65536 + 64, 65535, 65536 - 64, 70000, 100, 64, 0, -1):
        for shift in range(4):
            a, b, st = both(lib, lanes, blk, cap, shift)
            assert a[0] == b[0] and a[1] == b[1] and np.array_equal(a[2], b[2]), (cap, shift, a[:2], b[:2], st)
    # long literal runs (chains jump over whole segments), long matches, RLE, text
    rng = np.random.default_rng(5)
    orc = Oracle()
    shapes = [bytes(rng.integers(0, 256, 30000, dtype=np.uint8)) + b"\x00" * 30000,
              b"\x00" * 65536, b"ab" * 32768, bytes(rng.integers(0, 256, 65536 - 300, dtype=np.uint8)),
              (bytes(rng.integers(0, 256, 3000, dtype=np.uint8)) + b"x" * 500) * 18,
              b" ".join(bytes(rng.integers(97, 123, int(rng.integers(2, 9)), dtype=np.uint8)) for _ in range(9000))[:65536]]
    for raw in shapes:
        _, comp = orc.compress(raw, 1)
        for cap in (len(raw), len(raw) + 64, len(raw) + 5000, len(raw) - 1):
            a, b, st = both(lib, lanes, bytes(comp), cap, 1, with_marks=(len(comp) <= 65535 and cap <= 65536))
            assert a[0] == b[0] and a[1] == b[1] and np.array_equal(a[2], b[2]), (len(raw), cap, a[:2], b[:2], st)


def test_differential_fuzz_in_process(lib, lanes):
    """Tens of thousands of mutated blocks, compared inside the emulator library (fast): the warp scan
    must agree with the one-thread scan on the return value (incl. every error code), count and marks."""
    gen = Reference() if have_reference() else Oracle()
    total = errors = 0
    k = 1 if lanes == 128 else 4
    for seed, (proba, size, iters) in enumerate(((0.5, 65536, 12000 // k), (0.9, 65536, 8000 // k), (0.2, 65536, 4000 // k), (0.0, 60000, 1500 // k),
                                                 (1.0, 65536, 1500 // k), (0.5, 3000, 6000 // k), (0.5, 4 << 20, 150 // k), (0.9, 1 << 20, 300 // k))):
        raw = bytes(gen.datagen(size, proba, seed))
        _, comp = gen.compress(raw, 1)
        ne = C.c_longlong(0)
        n = lib.scan_par_fuzz(bytes(comp), len(comp), size, iters, seed, C.byref(ne), lanes)
        assert n == iters, (proba, size, "first mismatch at case %d" % (-n - 1))
        total += n
        errors += ne.value
    assert total > 30000 // k and errors > 10000 // k


def test_wide_marks_of_big_blocks(lib, lanes):
    """Blocks above 64 KB get two-word marks {token position, match start} for the tiles kernel: the parallel scan and the
    one-thread scan must write the same ones, on valid, truncated and corrupted blocks."""
    gen = Reference() if have_reference() else Oracle()
    rng = np.random.default_rng(lanes)
    for proba, size, seed in ((0.5, 1 << 20, 1), (0.9, 300000, 2), (0.0, 150000, 3), (0.5, 4 << 20, 4)):
        raw = bytes(gen.datagen(size, proba, seed))
        _, comp = gen.compress(raw, 1)
        variants = [(bytes(comp), size), (bytes(comp), size + 100), (bytes(comp), size - 1), (bytes(comp[:len(comp) // 2]), size)]
        bad = bytearray(comp)
        for pos in rng.integers(0, len(bad), 3):
            bad[int(pos)] ^= 0x5A
        variants.append((bytes(bad), size))
        for blk, cap in variants:
            mcap = cap // 4 + 2
            buf = np.frombuffer(blk + b"\xEE" * 32, dtype=np.uint8).copy()
            m1 = np.full(2 * mcap, 0xABABABAB, dtype=np.uint32)
            m2 = np.full(2 * mcap, 0xABABABAB, dtype=np.uint32)
            n1, n2 = C.c_uint32(0), C.c_uint32(0)
            st = (C.c_int * 3)()
            r1 = lib.scan_thread_host_wide(buf.ctypes.data, len(blk), cap, C.byref(n1), m1.ctypes.data, mcap)
            r2 = lib.scan_par_host_wide(buf.ctypes.data, len(blk), cap, C.byref(n2), m2.ctypes.data, mcap, st, lanes)
            assert r1 == r2 and n1.value == n2.value, (proba, size, cap, r1, r2, n1.value, n2.value)
            if r1 > 0:
                k = min(n1.value, mcap)
                assert np.array_equal(m1[:2 * k], m2[:2 * k]), (proba, size, cap)
                assert int(m1[2 * k - 1]) == r1                     # the last mark's second word = decoded size
