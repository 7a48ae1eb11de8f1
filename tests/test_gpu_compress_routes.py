"""GPU tests of the batch compress and pack calls at every stride, size and capacity.

- The parallel-parse compressor (LZ4B200_compress_blocks_parallel) against its host model (tests/encpar_model.py),
  byte for byte: return value, bytes, and the 0 verdict, for datagen, boundary-size, short-period, hash-colliding,
  window-seam and incompressible-prefix blocks, at every acceleration class and at capacities that run out in every
  part of the output.
- Both compressors with unaligned and odd source and destination strides, and with per-block sizes on both sides of
  64 KB in one batch: the byte-identical encoder (LZ4B200_compress_blocks) against the oracle, the parallel call against
  the model (blocks up to 64 KB) and the oracle (larger blocks).
- LZ4B200_pack_blocks and LZ4B200_pack_frame_blocks against a restatement, at odd strides and offsets.

Every compress call checks that nothing outside a slot's first `cap` bytes is written (gpu_util.compress_call)."""
import collections

import numpy as np
import pytest
import torch

import encpar_model as M
from gpu_util import compress_call, odd_stride, pack_call

pytestmark = pytest.mark.gpu
BS = 65536
ACCELS = (0, 1, 4, 5, 12, 13, 20, 21, 1000, 65537, 1 << 30, -3)
BOUNDARY_SIZES = (1, 4, 11, 12, 13, 14, 15, 16, 17, 31, 64, 100, 255, 4095, 4096, 4097, 4107, 4108, 4109, 8191, 8192,
                  8193, 8200, 16383, 16384, 16385, 20000, 65523, 65524, 65525, 65535, 65536)
STATS = collections.Counter()


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    assert lib.LZ4B200_device_count() > 0, "GPU tests need a CUDA device"
    return lib


_model_cache = {}


def model(raw, accel, oracle=None):
    key = (raw, M.step_of(accel) if len(raw) <= BS else accel)
    if key not in _model_cache:
        _model_cache[key] = M.compress(raw, accel, oracle=oracle)
    return _model_cache[key]


@pytest.fixture(scope="module")
def corpus(oracle):
    """[(name, block, claim)] of blocks of at most 64 KB"""
    out = []
    for p in (0.0, 0.2, 0.5, 0.9, 1.0):
        for seed in (1, 2):
            out.append(("P%d/%d" % (100 * p, seed), oracle.datagen(BS, p, 10 * seed + int(10 * p)).tobytes(), None))
    rng = np.random.default_rng(3)
    words = [bytes(rng.integers(97, 123, int(rng.integers(2, 9)), dtype=np.uint8)) for _ in range(200)]
    text = b" ".join(words[int(i)] for i in rng.integers(0, 200, 14000))
    for n in BOUNDARY_SIZES:
        out += [("dg%d" % n, oracle.datagen(n, 0.5, n).tobytes(), None), ("text%d" % n, text[:n], None),
                ("zero%d" % n, b"\0" * n, None), ("rand%d" % n, bytes(rng.integers(0, 256, n, dtype=np.uint8)), None),
                ("abc%d" % n, (b"abcdefg" * 10000)[:n], None)]
    out += M.special_blocks()
    return out


def check_vs_model(name, raw, accel, cap, ret, got):
    r = model(raw, accel)
    want = r.out if len(r.out) <= cap else None
    assert int(ret) == (len(want) if want is not None else 0), (name, len(raw), accel, cap, int(ret), len(r.out))
    if want is not None:
        assert got == want, (name, len(raw), accel, cap, "bytes differ from the model at %d" %
                             next(i for i in range(len(want)) if i >= len(got) or got[i] != want[i]))
    STATS["model blocks"] += 1
    STATS["model zero verdicts"] += want is None
    STATS["step %d" % r.step] += 1
    STATS["non-staged windows"] += sum(not w[1] for w in r.windows)
    return r


def test_parallel_equals_model_at_every_acceleration(lib, oracle, corpus):
    """One batch of the whole corpus per acceleration; odd strides, a source phase and a destination phase that change
    from block to block (srcStride = 16 k + 7, dstStride odd, d_dst 1 .. 15 bytes past alignment)."""
    blocks = [b for _, b, _ in corpus]
    cap = oracle.compress_bound(BS)
    src_stride, dst_stride = BS + 16 * 3 + 7, odd_stride(cap)
    phases = collections.Counter()
    for k, accel in enumerate(ACCELS):
        ret, got = compress_call(True, blocks, cap, accel, src_stride=src_stride, src_phase=k % 16,
                                 dst_stride=dst_stride, dst_mis=1 + k % 15, seed=k)
        for i, ((name, raw, claim), r, g) in enumerate(zip(corpus, ret, got)):
            m = check_vs_model(name, raw, accel, cap, r, g)
            if M.step_of(accel) == 1:
                assert M.reaches(m, claim), (name, claim)
            phases["src %d" % ((k % 16 + i * src_stride) % 16)] += 1       # (torch allocations are 512-byte aligned)
            phases["dst %d" % ((1 + k % 15 + i * dst_stride) % 16)] += 1
    assert len(phases) == 32
    print("\nSTATS parallel==model:", dict(STATS), dict(phases))


def _caps(r, n):
    """capacities that end in every part of the model's output r of an n-byte block"""
    caps = {len(r.out), len(r.out) - 1, 1, n + n // 255 + 16}
    staged = [w for w, x in enumerate(r.windows) if x[1] and x[0] > 32]
    if staged:
        caps.add(r.win_off[staged[0]] + r.windows[staged[0]][0] // 2)
    for w, x in enumerate(r.windows):
        if not x[1]:
            caps.add(r.win_off[w] + x[0] // 2)
            caps.add(r.win_off[w] + x[0] - 1)
    if r.last and r.last > 2:
        caps.add(r.body + (len(r.out) - r.body) // 2)
    return sorted(c for c in caps if c >= 1)


def test_parallel_capacity_rule_vs_model(lib, oracle, corpus):
    """All or nothing: every block of the set at every capacity one of them needs -- its exact size, one byte less, a
    capacity that runs out inside a staged window, inside a window that stores directly to global memory, inside the
    last literals, 1 and compressBound -- and never a byte past the capacity."""
    names = ("P20/1", "P50/1", "P90/1", "seam", "prefix10k", "prefix20k", "prefix40k", "rle1", "rle5-runs",
             "collide64/37", "dg13", "dg17", "dg4108", "text8193", "zero16385", "rand65536", "abc65524")
    pick = [c for c in corpus if c[0] in names]
    assert len(pick) == len(names)
    blocks = [b for _, b, _ in pick]
    for accel in (1, 21):
        caps = set()
        for _, raw, _ in pick:
            caps.update(_caps(model(raw, accel), len(raw)))
        for cap in sorted(caps):
            ret, got = compress_call(True, blocks, cap, accel, src_stride=BS + 9, dst_mis=cap % 16, seed=cap)
            for (name, raw, _), r, g in zip(pick, ret, got):
                check_vs_model(name, raw, accel, cap, r, g)
            STATS["capacities"] += 1
    print("\nSTATS capacities:", dict(STATS))


MIXED = (0, 1, 12, 13, 14, 4096, 65535, 65536, 65537, 200000, 4 << 20)


def mixed_blocks(oracle):
    return [oracle.datagen(n, 0.5, 1000 + n).tobytes() for n in MIXED]


@pytest.mark.parametrize("scalar", [0, 65536, 4 << 20])
def test_mixed_sizes_route_each_block_by_its_own_size(lib, oracle, scalar):
    """d_srcSize with sizes on both sides of 64 KB: the scalar srcSize is not used.  The byte-identical encoder gives the
    oracle's bytes for every block; the parallel call gives the model's for blocks up to 64 KB and the oracle's above."""
    blocks = mixed_blocks(oracle)
    cap = oracle.compress_bound(4 << 20)
    src_stride = (4 << 20) + 16 * 5 + 3
    for parallel in (False, True):
        ret, got = compress_call(parallel, blocks, cap, 1, src_stride=src_stride, src_phase=5, dst_mis=11,
                                 scalar=scalar, seed=scalar)
        for raw, r, g in zip(blocks, ret, got):
            if parallel and len(raw) <= BS:
                check_vs_model("mixed", raw, 1, cap, r, g)
            else:
                assert (int(r), g) == oracle.compress(raw, 1, cap), (parallel, len(raw), int(r))
                STATS["oracle blocks"] += 1
    print("\nSTATS mixed:", dict(STATS))


def test_exact_encoder_limited_capacity_vs_oracle(lib, oracle):
    """The byte-identical encoder at capacities around every block's size, block by block against the oracle (the
    drop-in host calls stage into a private buffer, so only a device call shows a write past dstCapacity)."""
    blocks = mixed_blocks(oracle)[:10] + [oracle.datagen(BS, p, 7).tobytes() for p in (0.0, 0.5, 1.0)]
    caps = set()
    for raw in blocks:
        r = oracle.compress(raw, 1)[0]
        caps.update({r, r - 1, r // 2, len(raw) - 1, 16, 15, 1})
    for accel in (1, 9):
        for cap in sorted(c for c in caps if c >= 1):
            ret, got = compress_call(False, blocks, cap, accel, src_stride=200000 + 16 * 2 + 13, src_phase=cap % 16,
                                     dst_mis=(cap + 7) % 16, seed=cap)
            for raw, r, g in zip(blocks, ret, got):
                assert (int(r), g) == oracle.compress(raw, accel, cap), (len(raw), accel, cap, int(r))
                STATS["oracle blocks"] += 1
    print("\nSTATS exact limited:", dict(STATS))


def test_layouts_both_compressors(lib, oracle):
    """Uniform 64 KB batches with and without d_srcSize, at every destination phase 0 .. 15 and odd strides."""
    blocks = [oracle.datagen(BS, 0.5, 200 + i).tobytes() for i in range(18)]
    cap = oracle.compress_bound(BS)
    for mis in range(16):
        for parallel in (False, True):
            ret, got = compress_call(parallel, blocks, cap, 1, src_stride=BS + 16 * 7 + 1 + 2 * mis, src_phase=mis,
                                     dst_stride=odd_stride(cap) + 2 * mis, dst_mis=mis, per_block_sizes=mis % 2 == 0,
                                     seed=mis)
            for raw, r, g in zip(blocks, ret, got):
                if parallel:
                    check_vs_model("layout", raw, 1, cap, r, g)
                else:
                    assert (int(r), g) == oracle.compress(raw, 1, cap)
                    STATS["oracle blocks"] += 1


def test_warps_reuse_tables_across_small_and_large_blocks(lib, oracle):
    """More blocks than the byte-identical encoder has warps (13 per SM): the warp of block b also compresses block
    b + grid.  Blocks 0 .. 31 and grid + 32 .. grid + 63 take the large table (65 547 bytes or more, lz4.c:1389),
    blocks 32 .. 63 and grid .. grid + 31 the small one; every block must start from a clean table.  The parallel call
    sends the large blocks to the same encoder and the others to the parallel kernel, whose CTAs also take several
    blocks each."""
    grid = torch.cuda.get_device_properties(0).multi_processor_count * 13
    n = grid + 64
    sizes = [100 + (i % 50) for i in range(n)]
    for i in range(32):
        sizes[i] = sizes[grid + 32 + i] = 65547 + 97 * i
        sizes[32 + i] = sizes[grid + i] = 4096 + 1931 * i
    d = oracle.datagen_mt(n * 70000, 1 << 20, 0.5, 9)
    blocks = [d[i * 70000:i * 70000 + s].tobytes() for i, s in enumerate(sizes)]
    cap = oracle.compress_bound(70000)
    for parallel in (False, True):
        ret, got = compress_call(parallel, blocks, cap, 1, src_stride=70000 + 5, src_phase=3, dst_mis=9)
        for raw, r, g in zip(blocks, ret, got):
            if parallel and len(raw) <= BS:
                check_vs_model("reuse", raw, 1, cap, r, g)
            else:
                assert (int(r), g) == oracle.compress(raw, 1, cap), (parallel, len(raw))
                STATS["oracle blocks"] += 1
    print("\nSTATS reuse:", dict(STATS))


def test_launch_count_per_route(lib, oracle):
    """A batch without d_srcSize is one launch of one kernel; with d_srcSize the parallel call launches the parallel
    kernel and then the byte-identical encoder, each for its own blocks."""
    blocks = [oracle.datagen(BS, 0.5, 300 + i).tobytes() for i in range(4)]
    cap = oracle.compress_bound(BS)
    for per_block, want in ((False, 1), (True, 2)):
        before = lib.LZ4B200_launch_count()
        compress_call(True, blocks, cap, 1, per_block_sizes=per_block)
        assert lib.LZ4B200_launch_count() - before == want
    big = [oracle.datagen(70000, 0.5, 5).tobytes()] * 2
    before = lib.LZ4B200_launch_count()
    ret, got = compress_call(True, big, oracle.compress_bound(70000), 1, per_block_sizes=False)
    assert lib.LZ4B200_launch_count() - before == 1
    assert (int(ret[0]), got[0]) == oracle.compress(big[0], 1)


# ------------------------------------------------------------------------------------------
# pack
# ------------------------------------------------------------------------------------------
def _slots(rng, n, stride):
    return rng.integers(0, 256, n * stride, dtype=np.uint8).tobytes()


def test_pack_blocks_odd_strides_and_offsets(lib):
    """sizes 0, negative (error codes count as 0), 1 .. 17 and 65 535; slot strides and stream offsets of every phase"""
    rng = np.random.default_rng(5)
    small = [0, -1, -65536] + list(range(1, 18))
    for stride in (17, 19, 33, 64, 101):
        n = 3 * len(small)
        sizes = np.array([small[(i * 7) % len(small)] for i in range(n)], dtype=np.int32)
        sizes = np.minimum(sizes, stride)
        slots = _slots(rng, n, stride)
        for hdr in (0, 4):
            for mis in range(16):
                pack_call(slots, stride, sizes, hdr, packed_mis=mis, slot_phase=(mis * 3 + stride) % 16)
                STATS["pack calls"] += 1
    stride = 65537
    sizes = np.array([65535, 3, 65535, 0, 65535, 17, -3, 65535], dtype=np.int32)
    slots = _slots(rng, len(sizes), stride)
    for hdr in (0, 4):
        for mis in (0, 1, 6, 15):
            pack_call(slots, stride, sizes, hdr, packed_mis=mis, slot_phase=mis)


def test_pack_blocks_many_blocks_cross_the_scan_carry(lib):
    rng = np.random.default_rng(6)
    for n in (1023, 1024, 1025, 3000):
        stride = 301
        sizes = rng.integers(-2, 302, n).astype(np.int32)
        sizes[rng.integers(0, n, n // 7)] = 0
        slots = _slots(rng, n, stride)
        for hdr in (0, 4):
            off = pack_call(slots, stride, sizes, hdr, packed_mis=n % 16, slot_phase=3)
            assert off[n] == int(np.maximum(sizes, 0).sum()) + hdr * n


def test_pack_frame_blocks_stored_raw_rule(lib):
    """lz4frame.c:896-899: a block whose size is 0 (or an error) or not below its source size is stored raw, with bit
    31 of its header set; the last block has lastSize source bytes"""
    rng = np.random.default_rng(7)
    for bsz, last in ((300, 0), (300, 17), (4097, 1), (4097, 4096)):
        n = 1100
        sizes = []
        for i in range(n):
            sz = last if (i == n - 1 and last > 0) else bsz
            sizes.append([0, sz - 1, sz, sz + 5, -4, 1 + i % (sz - 1 or 1)][i % 6])
        sizes = np.array(sizes, dtype=np.int32)
        stride = odd_stride(bsz)
        slots = _slots(rng, n, stride)
        fstride = bsz + 16 * 2 + 5
        fsrc = _slots(rng, n, fstride)
        for mis in (0, 5, 15):
            off = pack_call(slots, stride, sizes, 4, packed_mis=mis, slot_phase=mis, frame=(fsrc, fstride, bsz, last))
            STATS["frame calls"] += 1
        assert off[n] > 0
