"""LZ4_compress_destSize on the GPU: the drop-in calls and LZ4B200_compress_blocks_destSize against the reference's
results (tests/golden/kat_destsize.json) and the oracle's fill parse, with guard bytes, round trips through the GPU
decoder, odd strides and phases, and warps that compress many blocks."""
import collections
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_golden
from golden.make_golden_destsize import ACCELS, HEX_MAX, inputs, make_input, sha
from oracle.pyoracle import PATHS

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
UNWRITTEN = -123456789
DEV = "cuda:0"


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    if lib.LZ4B200_device_count() <= 0:
        pytest.skip("no CUDA device")
    return lib


def bound(n):
    return n + n // 255 + 16 if 0 <= n <= 0x7E000000 else 0


def room(n, target):
    """bytes of block n's slot the call may write: below the target, and below the bound on the compress_fast route"""
    return bound(n) if target >= bound(n) else max(target, 0)


def dest_batch(lib, blocks, target, acc, src_phase=0, dst_phase=0, src_pad=0, dst_pad=16):
    """One LZ4B200_compress_blocks_destSize call over `blocks` (numpy u8 arrays, per-block sizes) with the source at
    base + src_phase + i * src_stride and slot i at base + dst_phase + i * dst_stride.  Every slot is pre-filled with
    SENTINEL and checked to be unchanged at and past what the call may write.  Returns [(ret, consumed, bytes)]."""
    nb = len(blocks)
    sizes = [len(b) for b in blocks]
    src_stride = max(max(sizes), 1) + src_pad
    dst_stride = max(max(room(n, target) for n in sizes), 1) + dst_pad
    src_h = np.zeros(src_phase + nb * src_stride + 16, dtype=np.uint8)
    for i, b in enumerate(blocks):
        src_h[src_phase + i * src_stride:src_phase + i * src_stride + len(b)] = b
    src = torch.from_numpy(src_h).to(DEV)
    dst = torch.full((dst_phase + nb * dst_stride + 16,), SENTINEL, dtype=torch.uint8, device=DEV)
    szs = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    outs = torch.full((nb,), UNWRITTEN, dtype=torch.int32, device=DEV)
    cons = torch.full((nb,), UNWRITTEN, dtype=torch.int32, device=DEV)
    l0 = lib.LZ4B200_launch_count()
    rc = lib.LZ4B200_compress_blocks_destSize(src.data_ptr() + src_phase, src_stride, szs.data_ptr(), 0,
                                              dst.data_ptr() + dst_phase, dst_stride, int(target),
                                              1 if acc is None else int(acc), outs.data_ptr(), cons.data_ptr(), nb,
                                              torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert lib.LZ4B200_launch_count() == l0 + 1
    d = dst.cpu().numpy()
    rets, cs = outs.cpu().numpy(), cons.cpu().numpy()
    assert (d[:dst_phase] == SENTINEL).all() and (d[dst_phase + nb * dst_stride:] == SENTINEL).all()
    res = []
    for i in range(nb):
        slot = d[dst_phase + i * dst_stride:dst_phase + (i + 1) * dst_stride]
        lim = room(sizes[i], target)
        assert (slot[lim:] == SENTINEL).all(), ("write at or past the target", i, sizes[i], target, acc)
        assert rets[i] != UNWRITTEN and cs[i] != UNWRITTEN, i
        res.append((int(rets[i]), int(cs[i]), slot[:max(int(rets[i]), 0)].tobytes()))
    return res


def check_against_oracle(oracle, blocks, target, acc, res):
    paths = collections.Counter()
    for i, (b, got) in enumerate(zip(blocks, res)):
        r, c, o, p = oracle.compress_dest_size(b, target, acc)
        assert got == (r, c, o), (i, len(b), target, acc, got[:2], (r, c))
        paths[p] += 1
    return paths


def gpu_round_trip(lib, res):
    """LZ4B200_decompress_blocks with per-block capacities = consumed: returns consumed and the consumed prefix"""
    ok = [(i, r, c, o) for i, (r, c, o) in enumerate(res) if r > 0]
    if not ok:
        return {}
    offs, buf = [], bytearray(16)
    for _, _, _, o in ok:
        offs.append(len(buf))
        buf += o
    buf += b"\0" * 16
    n = len(ok)
    comp = torch.from_numpy(np.frombuffer(bytes(buf), dtype=np.uint8).copy()).to(DEV)
    d_off = torch.tensor(offs, dtype=torch.int64, device=DEV)
    d_sz = torch.tensor([r for _, r, _, _ in ok], dtype=torch.int32, device=DEV)
    caps = [c for _, _, c, _ in ok]
    d_cap = torch.tensor(caps, dtype=torch.int32, device=DEV)
    stride = max(max(caps), 1)
    out = torch.zeros(n * stride, dtype=torch.uint8, device=DEV)
    rets = torch.empty(n, dtype=torch.int32, device=DEV)
    ws = torch.empty(int(lib.LZ4B200_decompress_workspace_bytes_for(n, 1, 0)), dtype=torch.uint8, device=DEV)
    rc = lib.LZ4B200_decompress_blocks(comp.data_ptr(), d_off.data_ptr(), d_sz.data_ptr(), out.data_ptr(), None, stride,
                                       d_cap.data_ptr(), 0, rets.data_ptr(), n, ws.data_ptr(), ws.numel(),
                                       torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    h, rr = out.cpu().numpy(), rets.cpu().numpy()
    return {i: (int(rr[k]), h[k * stride:k * stride + max(int(rr[k]), 0)].tobytes()) for k, (i, _, _, _) in enumerate(ok)}


def assert_round_trip(lib, blocks, res):
    for i, (r, data) in gpu_round_trip(lib, res).items():
        c = res[i][1]
        assert (r, data) == (c, blocks[i][:c].tobytes()), (i, len(blocks[i]), r, c)


# ---- 1. golden vectors: both drop-in entry points and batch calls grouped by (target, acceleration) ----

@pytest.fixture(scope="module")
def kat(oracle):
    doc = load_golden("kat_destsize.json")
    data = {}
    for (iid, size, kind, seed), row in zip(inputs(), doc["inputs"]):
        data[iid] = make_input(oracle, size, kind, seed)
        assert sha(data[iid]) == row["sha256"]
    return data, doc["vectors"]


def _key(out):
    return out.hex() if len(out) <= HEX_MAX else sha(out)


def test_golden_vectors_drop_in(lib, kat):
    from lz4_b200 import block
    data, vecs = kat
    for iid, target, acc, ret, consumed, out in vecs:
        d = data[iid]
        calls = [acc] if acc is not None else [None, 1]
        for a in calls:
            r, c, o = block.LZ4_compress_destSize(d, target, a)
            assert (r, c, _key(o)) == (ret, consumed, out), (iid, len(d), target, a)


def test_golden_vectors_batch(lib, kat):
    data, vecs = kat
    groups = collections.defaultdict(list)
    for v in vecs:
        groups[(v[1], v[2])].append(v)
    for (target, acc), vs in groups.items():
        blocks = [data[v[0]] for v in vs]
        res = dest_batch(lib, blocks, target, acc)
        for v, (r, c, o) in zip(vs, res):
            assert (r, c, _key(o)) == (v[3], v[4], v[5]), (v[0], len(data[v[0]]), target, acc)


# ---- 2. 64 KB datagen blocks x targets x accelerations against the oracle, every path ----

TARGETS_64K = [-1, 0] + list(range(1, 21)) + [64, 100, 4096, 16384, 32768, 65535, bound(65536) - 1, bound(65536)]


def test_64k_datagen_blocks_every_target_and_acceleration(lib, oracle):
    blocks = [oracle.datagen(65536, p, 100 * k + s) for k, p in enumerate([0.0, 0.5, 0.9, 0.99]) for s in range(4)]
    paths = collections.Counter()
    for target in TARGETS_64K:
        for acc in (1, 2, 8, 65537, 65538, 1 << 20):
            res = dest_batch(lib, blocks, target, acc)
            paths += check_against_oracle(oracle, blocks, target, acc, res)
            if target in (100, 4096, 32768):
                assert_round_trip(lib, blocks, res)
    assert {PATHS[p] for p in paths} == {"fast", "no_room", "literals", "next_match", "reduced",
                                                    "last_literals", "filled"}, paths


# ---- 3 + 4 + 5. per-block sizes 0 .. 4 MiB, unaligned phases, odd strides, guard bytes, GPU round trip ----

MIXED_SIZES = [0, 1, 12, 13, 14, 100, 4095, 65535, 65546, 65547, 65548, 200000, 1 << 20, 4 << 20, 777, 31]


@pytest.mark.parametrize("target,acc", [(1, 1), (20, 8), (4096, 1), (30000, 2), (65537, 65538), (1 << 20, 1),
                                        (bound(4 << 20), 1 << 20), (bound(4 << 20) - 1, (1 << 25) - 1)])
def test_mixed_sizes_odd_strides_and_phases(lib, oracle, target, acc):
    kinds = ["p50", "p90", "random", "period", "zero", "p0", "p99"]
    blocks = [make_input(oracle, n, kinds[i % len(kinds)], 300 + i) for i, n in enumerate(MIXED_SIZES)]
    res = dest_batch(lib, blocks, target, acc, src_phase=3, dst_phase=5, src_pad=7, dst_pad=9)
    check_against_oracle(oracle, blocks, target, acc, res)
    assert_round_trip(lib, blocks, res)


# ---- 6. warps that compress many blocks of both table types, fill exits in between ----

def test_warps_rezero_the_table_between_blocks(lib, oracle):
    nb = 3600                                       # above the grid (13 warps per SM): every warp takes 2-3 blocks
    big = oracle.datagen_mt(nb * 66000, 66000, 0.6, 11)
    sizes = [66000 if i % 3 == 0 else (100 if i % 4 == 3 else 20000) for i in range(nb)]
    blocks = [big[i * 66000:i * 66000 + sizes[i]] for i in range(nb)]
    res = dest_batch(lib, blocks, 5000, 1)
    paths = check_against_oracle(oracle, blocks, 5000, 1, res)
    assert paths[0] > 0 and sum(paths.values()) - paths[0] > 1000


# ---- 7. one launch per call, none for nBlocks == 0, argument errors ----

def test_launch_count_and_argument_errors(lib):
    src = torch.zeros(4096, dtype=torch.uint8, device=DEV)
    dst = torch.zeros(4096, dtype=torch.uint8, device=DEV)
    outs = torch.zeros(4, dtype=torch.int32, device=DEV)
    cons = torch.zeros(4, dtype=torch.int32, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    f = lib.LZ4B200_compress_blocks_destSize
    l0 = lib.LZ4B200_launch_count()
    assert f(src.data_ptr(), 1024, None, 1024, dst.data_ptr(), 1024, 500, 1, outs.data_ptr(), cons.data_ptr(), 4, st) == 0
    torch.cuda.synchronize()
    assert lib.LZ4B200_launch_count() == l0 + 1
    assert f(src.data_ptr(), 1024, None, 1024, dst.data_ptr(), 1024, 500, 1, outs.data_ptr(), cons.data_ptr(), 0, st) == 0
    assert f(None, 1024, None, 1024, dst.data_ptr(), 1024, 500, 1, outs.data_ptr(), cons.data_ptr(), 0, st) == 0
    assert lib.LZ4B200_launch_count() == l0 + 1
    bad = [
        (src.data_ptr(), dst.data_ptr(), outs.data_ptr(), cons.data_ptr(), -1),
        (None, dst.data_ptr(), outs.data_ptr(), cons.data_ptr(), 4),
        (src.data_ptr(), None, outs.data_ptr(), cons.data_ptr(), 4),
        (src.data_ptr(), dst.data_ptr(), None, cons.data_ptr(), 4),
        (src.data_ptr(), dst.data_ptr(), outs.data_ptr(), None, 4),
    ]
    for s, d, o, c, n in bad:
        assert f(s, 1024, None, 1024, d, 1024, 500, 1, o, c, n, st) == -1
    assert lib.LZ4B200_launch_count() == l0 + 1
    # drop-in deviations: NULL srcSizePtr / dst, invalid state
    n = C.c_int(100)
    buf = np.zeros(200, dtype=np.uint8)
    assert lib.LZ4_compress_destSize(buf.ctypes.data, buf.ctypes.data, None, 50) == 0
    assert lib.LZ4_compress_destSize(buf.ctypes.data, None, C.byref(n), 50) == 0 and n.value == 100
    assert lib.LZ4_compress_destSize_extState(buf.ctypes.data + 4, buf.ctypes.data, buf.ctypes.data, C.byref(n), 50, 1) == 0
    assert n.value == 100


# ---- 8. seeded fuzz loop through the drop-in entry points (fuzzer.c:399-420, 488-492, 1694-1704) ----

@pytest.mark.parametrize("seed", [1, 2, 2026])
def test_fuzz_drop_in(lib, oracle, seed):
    from lz4_b200 import block
    rng = np.random.default_rng(seed)
    state = np.zeros(2052, dtype=np.uint64)
    for it in range(120):
        n = int(rng.integers(1, 1 << int(rng.integers(4, 18))))
        d = make_input(oracle, n, ["p50", "p90", "random", "period", "zero"][it % 5], seed * 1000 + it)
        if it % 3 == 0:                                              # fuzzer.c:399-420: target = n * k / 128
            target, acc = n * int(rng.integers(1, 129)) >> 7, None
        elif it % 3 == 1:                                            # fuzzer.c:488-492: one byte short of compress_fast
            r, _ = block.LZ4_compress_fast(d, None, 8)
            target, acc = r - 1, 8
        else:                                                        # fuzzer.c:1694-1704: one-byte payload, small dst
            d = np.full(n, int(rng.integers(0, 256)), dtype=np.uint8)
            target, acc = int(rng.integers(1, 64)), None
        end = int(rng.integers(0, 256))
        dst = np.full(max(target, 0) + 8, end, dtype=np.uint8)
        cnt = C.c_int(n)
        if acc is None:
            r = lib.LZ4_compress_destSize(d.ctypes.data, dst.ctypes.data, C.byref(cnt), target)
        else:
            r = lib.LZ4_compress_destSize_extState(state.ctypes.data, d.ctypes.data, dst.ctypes.data, C.byref(cnt), target, acc)
        assert (dst[max(target, 0):] == end).all(), "wrote past the target"
        assert 0 <= r <= max(target, 0) and cnt.value <= n
        if target > 0:
            assert r > 0
            assert oracle.decompress(dst[:r].tobytes(), cnt.value) == (cnt.value, d[:cnt.value].tobytes())
        if it % 3 == 1 and target > 0:
            assert cnt.value < n                                    # fuzzer.c:490: consumes less than the input
        assert (r, cnt.value, dst[:r].tobytes()) == oracle.compress_dest_size(d, target, acc)[:3], (seed, it, n, target, acc)
