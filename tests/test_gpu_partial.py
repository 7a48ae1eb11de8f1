"""LZ4_decompress_safe_partial and LZ4B200_decompress_blocks_partial on the GPU.

Every case of tests/golden/kat_partial.json (results of the compiled reference) goes through the drop-in call and
through batch calls, grouped by target and as one batch of per-block targets; the bytes are compared with the checker
(tests/partial_oracle.c), itself pinned to the reference's digests.  The cases include srcSize = exact .. exact + 9 at
target = decoded size (the reference's tests/decompress-partial.c) and the exhaustive target sweeps.  Also: routes P1 / P2 through the slow list, guard bytes at and
past every slot's return value, launch counts, argument errors, equality with the full decode, and a seeded fuzz loop.
"""
import os
import sys
from collections import defaultdict

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_golden_partial as mg  # noqa: E402
from lz4_b200 import _lib, batch, block  # noqa: E402
from oracle.pyoracle import Oracle  # noqa: E402
from partial_oracle import PartialOracle, golden  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GUARD = 0xA5


@pytest.fixture(scope="module")
def kat():
    return golden()


def pack(srcs):
    """blocks back to back with 16 bytes of slack at both ends (readable padding)"""
    offs, buf = [], bytearray(16)
    for s in srcs:
        offs.append(len(buf))
        buf += s
    buf += bytes(16)
    d = torch.from_numpy(np.frombuffer(bytes(buf), dtype=np.uint8).copy()).to(DEV)
    return (d, torch.tensor(offs, dtype=torch.int64, device=DEV),
            torch.tensor([len(s) for s in srcs], dtype=torch.int32, device=DEV))


def run_batch(srcs, targets, stride=None, shift=0, ws=None):
    """one partial batch call; per-block targets when `targets` is a list.  Returns (rets, slots, slowCount) after
    checking the guard bytes at and past every slot's return value."""
    lib = _lib.load()
    comp, offs, sizes = pack(srcs)
    n = len(srcs)
    per = isinstance(targets, list)
    tl = targets if per else [targets] * n
    stride = stride if stride is not None else max([max(t, 0) for t in tl] + [1])
    out = torch.full((n * stride + shift + 64,), GUARD, dtype=torch.uint8, device=DEV)
    rets = torch.empty(n, dtype=torch.int32, device=DEV)
    tt = torch.tensor(tl, dtype=torch.int32, device=DEV) if per else None
    wsb = int(lib.LZ4B200_decompress_workspace_bytes_for(n, int(per), 0 if per else int(targets)))
    wsb = ws if ws is not None else wsb
    w = torch.zeros(max(wsb, 256), dtype=torch.uint8, device=DEV)
    rc = lib.LZ4B200_decompress_blocks_partial(comp.data_ptr(), offs.data_ptr(), sizes.data_ptr(), out.data_ptr() + shift,
                                               None, stride, tt.data_ptr() if per else None, 0 if per else int(targets),
                                               rets.data_ptr(), n, w.data_ptr(), wsb, torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "LZ4B200_decompress_blocks_partial")
    torch.cuda.synchronize()
    r = rets.cpu().numpy()
    h = out.cpu().numpy()
    slots = []
    for i in range(n):
        base = shift + i * stride
        k = max(int(r[i]), 0)
        slots.append(h[base:base + k].tobytes())
        assert (h[base + k:base + stride] == GUARD).all(), "block %d wrote at or past its return value" % i
    assert (h[:shift] == GUARD).all() and (h[shift + n * stride:] == GUARD).all()
    slow = int(w[:4].view(torch.int32).cpu()[0])
    return r, slots, slow


def test_drop_in_matches_the_reference(kat):
    _, groups = kat
    po = PartialOracle()
    for name, cases, rets, digest in groups:
        res = []
        for src, t, c in cases:
            got = block.LZ4_decompress_safe_partial(src, t, c)
            assert got == po.decompress_partial(src, t, c), (name, t, c)
            res.append((got[0], None if po.dst_dependent else got[1]))
        assert [r for r, _ in res] == rets and mg.run_digest(res) == digest, name


def test_batches_by_target_and_per_block(kat):
    """every case with capacity = target: one batch per target, then one batch of per-block targets (the exhaustive
    sweeps included) at an odd stride and an unaligned base"""
    _, groups = kat
    po = PartialOracle()
    flat = [(src, t, r) for _, cases, rets, _ in groups for (src, t, c), r in zip(cases, rets) if t == c]
    by_t = defaultdict(list)
    for x in flat:
        by_t[x[1]].append(x)
    for t, xs in sorted(by_t.items()):
        rets, slots, _ = run_batch([x[0] for x in xs], t)
        for (src, _, want), r, s in zip(xs, rets, slots):
            assert r == want and (r, s) == po.decompress_partial(src, t), (t, want, r)
    small = [x for x in flat if x[1] <= 70000]
    rets, slots, _ = run_batch([x[0] for x in small], [x[1] for x in small], stride=70001, shift=3)
    for (src, t, want), r, s in zip(small, rets, slots):
        assert r == want and (r, s) == po.decompress_partial(src, t), (t, want, r)


def test_stops_in_every_run_class():
    """literal stops, match stops at 0..13 bytes from its end, offsets 0, 1 and < 8, and the last 5 bytes as a match
    (which LZ4_decompress_safe rejects)"""
    po = PartialOracle()
    rng = np.random.default_rng(5)
    lit = rng.integers(0, 256, 40, dtype=np.uint8).tobytes()
    cases = []
    for off in (0, 1, 2, 3, 7, 8, 40):
        ml = 30
        blk = bytes([0xFF, 40 - 15]) + lit + bytes([off, 0, ml - 19]) + bytes([0x50]) + lit[:5]
        full = 40 + ml + 5
        for t in list(range(36, full + 2)) + [40 + ml - d for d in range(14)]:
            cases.append((blk, t))
    # a block that ends in a match (the last 5 bytes are not literals): full decode rejects it, partial accepts it
    blk = bytes([0x5F]) + lit[:5] + b"\x01\x00" + bytes([255, 10]) + bytes(6)
    cases += [(blk, t) for t in (1, 5, 6, 100, 200, 289, 290)]
    rets, slots, _ = run_batch([c[0] for c in cases], [c[1] for c in cases], stride=400)
    for (b, t), r, s in zip(cases, rets, slots):
        assert (r, s) == po.decompress_partial(b, t), (b[:4].hex(), t)
    assert block.LZ4_decompress_safe(blk, 300)[0] < 0


def test_routes():
    orc = Oracle()
    raw, comp = mg.make_block(orc, 65536, "p50", 11)
    for t in (4096, 16384, 65536):
        rets, slots, slow = run_batch([comp] * 300, t)
        assert slow == 0 and all(s == raw[:t] for s in slots)                # P1
    big_raw, big = mg.make_block(orc, 4 << 20, "p50", 12)
    rets, slots, slow = run_batch([big] * 3, 61440)
    assert slow == 0 and all(s == big_raw[:61440] for s in slots)           # P1: 4 MB blocks, consumed prefix < 64 KB
    rets, slots, slow = run_batch([big] * 3, 300000)
    assert slow == 3 and all(s == big_raw[:300000] for s in slots)          # P2: target above 64 KB
    rraw, rcomp = mg.make_block(orc, 65536 + 100, "random", 13)
    rets, slots, slow = run_batch([rcomp], 65536)
    assert slow == 1 and slots[0] == rraw[:65536]                           # P2: consumed > 65 535
    # > 8 192 sequences: 4-byte matches between single literals
    seqs = b"".join(bytes([0x10, 0x41 + (k % 20), 1, 0]) for k in range(9000)) + bytes([0x50]) + b"ABCDE"
    rets, slots, slow = run_batch([seqs], 45000 + 5)
    assert slow == 1 and (rets[0], slots[0]) == PartialOracle().decompress_partial(seqs, 45005)
    # > 20 480 runs with <= 8 192 sequences: 1 literal + an offset-0 match of 4 (4 runs each)
    runs = b"".join(bytes([0x10, 0x30 + (k % 9), 0, 0]) for k in range(6000)) + bytes([0x50]) + b"ABCDE"
    rets, slots, slow = run_batch([runs], 30005)
    assert slow == 1 and (rets[0], slots[0]) == PartialOracle().decompress_partial(runs, 30005)


def test_launch_counts_and_argument_errors():
    lib = _lib.load()
    orc = Oracle()
    raw, comp = mg.make_block(orc, 4096, "p50", 14)
    run_batch([comp], 100)
    c0 = lib.LZ4B200_launch_count()
    run_batch([comp] * 5, 100)
    assert lib.LZ4B200_launch_count() - c0 == 3
    c0 = lib.LZ4B200_launch_count()
    st = torch.cuda.current_stream().cuda_stream
    assert lib.LZ4B200_decompress_blocks_partial(None, None, None, None, None, 0, None, 100, None, 0, None, 0, st) == 0
    assert lib.LZ4B200_launch_count() == c0
    d, offs, sizes = pack([comp])
    out = torch.empty(256, dtype=torch.uint8, device=DEV)
    rets = torch.empty(1, dtype=torch.int32, device=DEV)
    need = int(lib.LZ4B200_decompress_workspace_bytes_for(1, 0, 100))
    w = torch.empty(need, dtype=torch.uint8, device=DEV)
    args = [d.data_ptr(), offs.data_ptr(), sizes.data_ptr(), out.data_ptr(), None, 128, None, 100, rets.data_ptr(), 1,
            w.data_ptr(), need, st]
    assert lib.LZ4B200_decompress_blocks_partial(*args) == 0
    for i in (0, 1, 2, 3, 8, 10):
        bad = list(args); bad[i] = None
        assert lib.LZ4B200_decompress_blocks_partial(*bad) == -1
    bad = list(args); bad[9] = -1
    assert lib.LZ4B200_decompress_blocks_partial(*bad) == -1
    bad = list(args); bad[11] = need - 1
    assert lib.LZ4B200_decompress_blocks_partial(*bad) == -1
    assert lib.LZ4B200_launch_count() == c0 + 3
    # drop-in argument rules (lz4.c:2036, :2066, :2069) and the documented deviations
    assert block.LZ4_decompress_safe_partial(comp, -1) == (-1, b"")
    assert block.LZ4_decompress_safe_partial(b"\xff\xff", 0) == (0, b"")
    assert block.LZ4_decompress_safe_partial(b"", 10) == (-1, b"")
    assert lib.LZ4_decompress_safe_partial(None, None, 5, 10, 10) == -1
    src = np.frombuffer(comp, dtype=np.uint8)
    assert lib.LZ4_decompress_safe_partial(src.ctypes.data, None, len(comp), 10, 10) == -1
    assert lib.LZ4_decompress_safe_partial(src.ctypes.data, None, len(comp), 10, 0) == 0
    dst = np.full(64, 7, dtype=np.uint8)
    assert lib.LZ4_decompress_safe_partial(src.ctypes.data, dst.ctypes.data, -3, 10, 10) == -1
    assert lib.LZ4_decompress_safe_partial(b"\xf0" * 3, dst.ctypes.data, 3, 10, 10) < 0 and (dst == 7).all()


def test_equals_full_decode_when_target_covers_the_block():
    orc = Oracle()
    srcs, raws = [], []
    for k in range(40):
        raw, comp = mg.make_block(orc, 65536, mg.KINDS[k % 7], 500 + k)
        srcs.append(comp); raws.append(raw)
    comp, offs, sizes = pack(srcs)
    full, frets = batch.decompress_blocks(comp, offs, sizes, 65536)
    part, prets = batch.decompress_blocks_partial(comp, offs, sizes, 65536)
    torch.cuda.synchronize()
    assert torch.equal(frets, prets) and torch.equal(full, part)
    t = torch.full((40,), 70000, dtype=torch.int32, device=DEV)
    part2, prets2 = batch.decompress_blocks_partial(comp, offs, sizes, t, out_stride=65536)
    torch.cuda.synchronize()
    assert torch.equal(frets, prets2) and torch.equal(full, part2)


@pytest.mark.parametrize("seed", [1, 2, 2026])
def test_fuzz_like_reference_fuzzer(seed):
    """fuzzer.c:641-652: partial decode of a random prefix: ret == target, dst[target] untouched, prefix correct"""
    orc = Oracle()
    rng = np.random.default_rng(seed)
    srcs, ts, raws = [], [], []
    for k in range(200):
        size = int(rng.integers(1, 70000))
        raw = orc.datagen(size, float(rng.random()), int(rng.integers(0, 1 << 30))).tobytes()
        r, comp = orc.compress(raw, 1)
        t = int(rng.integers(0, size + 1))
        srcs.append(comp); ts.append(t); raws.append(raw)
        got, out = block.LZ4_decompress_safe_partial(comp, t, size)
        assert got == t and out == raw[:t]
    rets, slots, _ = run_batch(srcs, ts, stride=70001)       # the guard at dst[target] is checked there
    for t, raw, r, s in zip(ts, raws, rets, slots):
        assert r == t and s == raw[:t]
