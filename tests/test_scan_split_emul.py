"""CPU check of the split scan (lz4_b200/csrc/lz4_scan_split.h; device: lz4_scan_split_kernel).

The header is compiled for the host and the lanes of a block are run phase by phase (tests/emul/scan_split_emul.cpp);
for every block -- valid, corrupted, capacity-limited -- the result must be IDENTICAL to the one-thread scan of
lz4_scan_core.h (itself pinned to the golden vectors and the oracle by tests/test_scan_core_host.py): return value,
sequence count, and the marks of every sequence.
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


def both(lib, block, cap, shift=0):
    n = len(block)
    buf = np.full(n + 80, 0xEE, dtype=np.uint8)
    base = buf.ctypes.data
    pad = (-base) % 16 + 16 + shift
    buf[pad:pad + n] = np.frombuffer(bytes(block), dtype=np.uint8)
    m1 = np.full(MAX_SEQ, 0xABABABAB, dtype=np.uint32)
    m2 = np.full(MAX_SEQ, 0xABABABAB, dtype=np.uint32)
    n1, n2 = C.c_uint32(0), C.c_uint32(0)
    stats = (C.c_int * 3)()
    r1 = lib.scan_host(base + pad, n, cap, C.byref(n1), m1.ctypes.data)
    r2 = lib.scan_split_host(base + pad, n, cap, C.byref(n2), m2.ctypes.data, MAX_SEQ, stats)
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
    return bytes(b)[:65535]


def test_split_scan_equals_one_thread_scan(lib):
    orc = Oracle()
    gen = Reference() if have_reference() else orc
    rng = np.random.default_rng(20260925)
    checked = errors = fallbacks = p2 = 0
    for proba in (0.0, 0.2, 0.5, 0.9, 0.99, 1.0):
        for size in (2000, 4200, 10000, 40000, 65536, 65536, 65536):
            raw = bytes(gen.datagen(size, proba, int(rng.integers(0, 1 << 30))))
            _, comp = orc.compress(raw, 1)
            comp = bytes(comp)
            if len(comp) > 65535:
                continue
            for cap in {size, size + 1, size + 64, min(size + 1000, 65536), size - 1, size - 70, size // 2, 64, 63, 65536}:
                if cap > 65536:
                    continue
                a, b, st = both(lib, comp, cap, shift=int(rng.integers(0, 16)))
                assert a[0] == b[0] and a[1] == b[1], (proba, size, cap, a[:2], b[:2], st)
                assert np.array_equal(a[2], b[2]), (proba, size, cap, st)
                if cap == size:
                    assert a[0] == size
                    fallbacks += st[0]
                    p2 += st[1]
                checked += 1
            for _ in range(12):
                bad = corrupt(rng, comp)
                cap = int(rng.choice([size, min(size + 64, 65536), min(size + 1000, 65536), max(size - 5, 1)]))
                a, b, st = both(lib, bad, cap, shift=int(rng.integers(0, 16)))
                assert a[0] == b[0] and a[1] == b[1], (proba, size, cap, a[:2], b[:2], st)
                assert np.array_equal(a[2], b[2])
                errors += a[0] < 0
                checked += 1
    assert checked > 600 and errors > 100
    assert fallbacks == 0                                  # well-formed data never needs the one-thread scan


def test_fixture_block_and_special_shapes(lib):
    blk = open(os.path.join(HERE, "golden", "p50_seed0_64k.lz4block"), "rb").read()
    for cap in (65536, 65535, 65536 - 64, 65536 - 65, 40000, 100, 64):
        for shift in range(4):
            a, b, st = both(lib, blk, cap, shift)
            assert a[0] == b[0] and a[1] == b[1] and np.array_equal(a[2], b[2]), (cap, shift, a[:2], b[:2], st)
    rng = np.random.default_rng(5)
    orc = Oracle()
    shapes = [bytes(rng.integers(0, 256, 30000, dtype=np.uint8)) + b"\x00" * 30000,
              b"\x00" * 65536, b"ab" * 32768, bytes(rng.integers(0, 256, 60000, dtype=np.uint8)),
              (bytes(rng.integers(0, 256, 3000, dtype=np.uint8)) + b"x" * 500) * 18,
              b" ".join(bytes(rng.integers(97, 123, int(rng.integers(2, 9)), dtype=np.uint8)) for _ in range(9000))[:65536]]
    for raw in shapes:
        _, comp = orc.compress(raw, 1)
        if len(comp) > 65535:
            continue
        for cap in (len(raw), min(len(raw) + 64, 65536), len(raw) - 1, len(raw) // 3):
            a, b, st = both(lib, bytes(comp), cap, 1)
            assert a[0] == b[0] and a[1] == b[1] and np.array_equal(a[2], b[2]), (len(raw), cap, a[:2], b[:2], st)


def test_differential_fuzz_in_process(lib):
    """Tens of thousands of mutated blocks, compared inside the emulator library (fast)."""
    gen = Reference() if have_reference() else Oracle()
    total = errors = 0
    for seed, (proba, size, iters) in enumerate(((0.5, 65536, 12000), (0.9, 65536, 8000), (0.2, 65536, 4000), (0.0, 60000, 1500),
                                                 (1.0, 65536, 1500), (0.5, 9000, 6000), (0.99, 65536, 3000))):
        raw = bytes(gen.datagen(size, proba, seed))
        _, comp = gen.compress(raw, 1)
        if len(comp) > 65535:
            continue
        ne, nf = C.c_longlong(0), C.c_longlong(0)
        n = lib.scan_split_fuzz(bytes(comp), len(comp), size, iters, seed, C.byref(ne), C.byref(nf))
        assert n == iters, (proba, size, "first mismatch at case %d" % (-n - 1))
        total += n
        errors += ne.value
    assert total > 25000 and errors > 8000
