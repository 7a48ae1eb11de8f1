"""LZ4B200_compress_blocks_hc on the GPU through the C ABI: the reference's results (tests/golden/kat_hc.json) and the
host build of the same parse (tests/hc_emul.py), with mixed sizes, odd strides, capacities at and below the returned
size, guard bytes, workspace sizes, round trips through the GPU decoder, argument errors, launch counts and a fuzz loop."""
import numpy as np
import pytest
import torch

import hc_emul as he
from hc_emul import host_hc, mg

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
UNWRITTEN = -123456789
DEV = "cuda:0"
ERR_ARG = -1


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    if lib.LZ4B200_device_count() <= 0:
        pytest.skip("no CUDA device")
    return lib


def hc_batch(lib, blocks, cap, level, src_phase=0, dst_phase=0, src_pad=0, dst_pad=16, ws_extra=0):
    """One LZ4B200_compress_blocks_hc call over `blocks` (per-block sizes through d_srcSize).  Every slot is pre-filled
    with SENTINEL and checked unchanged at and past the capacity (and between slots).  Returns [(ret, bytes)]."""
    nb = len(blocks)
    sizes = [len(b) for b in blocks]
    src_stride = max(max(sizes), 1) + src_pad
    room = [max(min(cap, mg.compress_bound(n)), 0) for n in sizes]
    dst_stride = max(max(room), 1) + dst_pad
    src_h = np.zeros(src_phase + nb * src_stride + 16, dtype=np.uint8)
    for i, b in enumerate(blocks):
        src_h[src_phase + i * src_stride:src_phase + i * src_stride + len(b)] = np.frombuffer(bytes(b), dtype=np.uint8)
    src = torch.from_numpy(src_h).to(DEV)
    dst = torch.full((dst_phase + nb * dst_stride + 16,), SENTINEL, dtype=torch.uint8, device=DEV)
    szs = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    outs = torch.full((nb,), UNWRITTEN, dtype=torch.int32, device=DEV)
    wsb = int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(nb)) + ws_extra
    ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=DEV)
    l0 = lib.LZ4B200_launch_count()
    rc = lib.LZ4B200_compress_blocks_hc(src.data_ptr() + src_phase, src_stride, szs.data_ptr(), 0,
                                        dst.data_ptr() + dst_phase, dst_stride, int(cap), int(level), outs.data_ptr(), nb,
                                        ws.data_ptr(), wsb, torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert lib.LZ4B200_launch_count() == l0 + 1
    d = dst.cpu().numpy()
    rets = outs.cpu().numpy()
    assert (d[:dst_phase] == SENTINEL).all() and (d[dst_phase + nb * dst_stride:] == SENTINEL).all()
    res = []
    for i in range(nb):
        slot = d[dst_phase + i * dst_stride:dst_phase + (i + 1) * dst_stride]
        assert (slot[room[i]:] == SENTINEL).all(), ("write at or past the capacity", i, sizes[i], cap, level)
        assert rets[i] != UNWRITTEN
        res.append((int(rets[i]), slot[:max(int(rets[i]), 0)].tobytes()))
    return res


def test_golden_vectors(lib, oracle):
    """Every capacity of every vector up to 256 KB.  A block is compressed by one thread, so the 1 MB and 4 MB inputs
    are checked at the bound only, all in one call per level (their other capacities are the CPU suite's)."""
    doc, ins = he.golden("kat_hc.json")
    by_level, big = {}, {}
    for iid, lv, rb, rets, dig in doc["vectors"]:
        (big if ins[iid]["size"] > (256 << 10) else by_level).setdefault(lv, []).append((iid, rb, rets, dig))
    for lv, vecs in sorted(big.items()):
        data = [mg.make_input(oracle, ins[v[0]]["size"], ins[v[0]]["kind"], ins[v[0]]["seed"]) for v in vecs]
        got = hc_batch(lib, data, mg.compress_bound(4 << 20), lv)
        for d, v, g in zip(data, vecs, got):
            assert g[0] == v[1] and g == host_hc(d, mg.compress_bound(len(d)), lv), (ins[v[0]], lv)
    for lv, vecs in sorted(by_level.items()):
        data = [mg.make_input(oracle, ins[v[0]]["size"], ins[v[0]]["kind"], ins[v[0]]["seed"]) for v in vecs]
        ncaps = max(len(mg.capacities(len(d), v[1])) for d, v in zip(data, vecs))
        got = [[] for _ in vecs]
        # one call per capacity position k: block j gets its own k-th capacity through a call per distinct capacity
        caps = [mg.capacities(len(d), v[1]) for d, v in zip(data, vecs)]
        for k in range(ncaps):
            groups = {}
            for j, c in enumerate(caps):
                if k < len(c):
                    groups.setdefault(c[k], []).append(j)
            for cap, js in groups.items():
                for j, r in zip(js, hc_batch(lib, [data[j] for j in js], cap, lv)):
                    got[j].append(r)
        for (iid, rb, rets, dig), g in zip(vecs, got):
            assert [r for r, _ in g] == rets and mg.run_digest(g) == dig, (ins[iid], lv)


def test_run_digests(lib, oracle):
    doc, _ = he.golden("kat_hc.json")
    cases = list(mg.random_cases(oracle, doc["run_cases"]))
    got = [None] * len(cases)
    groups = {}
    for j, (d, cap, lv) in enumerate(cases):
        groups.setdefault((cap, lv), []).append(j)
    for (cap, lv), js in groups.items():
        for j, r in zip(js, hc_batch(lib, [cases[j][0] for j in js], cap, lv)):
            got[j] = r
    chunk = doc["run_chunk"]
    assert [mg.run_digest(got[k:k + chunk]) for k in range(0, len(got), chunk)] == doc["run_digests"]


@pytest.mark.parametrize("level", [-1, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9])
def test_seeded_batches_match_the_host_build(lib, oracle, level):
    rng = np.random.default_rng(500 + level)
    blocks = [mg.make_input(oracle, int(rng.choice([13, 100, 4096, 30000, 65536])),
                            mg.KINDS[int(rng.integers(0, len(mg.KINDS)))], 7000 + k) for k in range(48)]
    for cap in (1 << 30, 40000):
        got = hc_batch(lib, blocks, cap, level, src_phase=3, dst_phase=5, src_pad=7, dst_pad=3)
        assert got == [host_hc(b, cap, level) for b in blocks]


def test_mixed_sizes_in_one_call(lib, oracle):
    blocks = [mg.make_input(oracle, n, "p50", 11 + n) for n in range(14)]
    blocks += [mg.make_input(oracle, 65536, "p50", 3), mg.make_input(oracle, 4 << 20, "p90l60", 4)]
    got = hc_batch(lib, blocks, 1 << 30, 9)
    assert got == [host_hc(b, 1 << 30, 9) for b in blocks]
    assert got[0] == (1, b"\x00")


def test_capacities_at_the_bound_ret_and_below(lib, oracle):
    blocks = [mg.make_input(oracle, 20000, k, 40 + i) for i, k in enumerate(["p50", "per1", "random", "p90"])]
    for lv in (2, 6, 9):
        full = hc_batch(lib, blocks, mg.compress_bound(20000), lv)
        for b, (r, out) in zip(blocks, full):
            assert hc_batch(lib, [b], r, lv) == [(r, out)]
            assert hc_batch(lib, [b], r - 1, lv)[0][0] == 0


def test_output_independent_of_calls_and_workspace(lib, oracle):
    blocks = [mg.make_input(oracle, 65536, mg.KINDS[k % len(mg.KINDS)], 900 + k) for k in range(40)]
    a = hc_batch(lib, blocks, 1 << 30, 9)
    assert hc_batch(lib, blocks, 1 << 30, 9) == a
    assert hc_batch(lib, blocks, 1 << 30, 9, ws_extra=(1 << 20) * 5 + 123) == a


def test_round_trip_through_the_gpu_decoder(lib, oracle):
    from lz4_b200 import batch
    data = oracle.datagen(64 * 65536, 0.5, 5)
    src = torch.from_numpy(data).to(DEV)
    for lv in (2, 3, 9):
        slots, sizes, stride = batch.compress_blocks_hc(src, 65536, lv)
        packed, offs = batch.pack_blocks(slots, stride, sizes)
        out, rets = batch.decompress_blocks(packed, offs[:-1].contiguous(), sizes, 65536)
        torch.cuda.synchronize()
        assert bool((rets == 65536).all()) and torch.equal(out, src), lv
        h = slots.cpu().numpy()
        for i in (0, 17, 63):
            assert (int(sizes[i]), h[i * stride:i * stride + int(sizes[i])].tobytes()) == \
                host_hc(data[i * 65536:(i + 1) * 65536], mg.compress_bound(65536), lv)


def test_argument_errors_and_launch_counts(lib):
    src = torch.zeros(1024, dtype=torch.uint8, device=DEV)
    dst = torch.zeros(4096, dtype=torch.uint8, device=DEV)
    outs = torch.zeros(4, dtype=torch.int32, device=DEV)
    wsb = int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(4))
    assert wsb == 4 * 256 * 1024 and lib.LZ4B200_compress_blocks_hc_workspace_bytes(0) == 0
    assert lib.LZ4B200_compress_blocks_hc_workspace_bytes(1 << 20) == 16384 * 256 * 1024
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    s = torch.cuda.current_stream().cuda_stream

    def call(src_p=src.data_ptr(), dst_p=dst.data_ptr(), out_p=outs.data_ptr(), ws_p=ws.data_ptr(), n=4, level=9,
             wsbytes=wsb):
        return lib.LZ4B200_compress_blocks_hc(src_p, 256, None, 256, dst_p, 1024, 1024, level, out_p, n, ws_p, wsbytes, s)

    l0 = lib.LZ4B200_launch_count()
    for lv in (10, 11, 12, 100):
        assert call(level=lv) == ERR_ARG
    assert call(n=-1) == ERR_ARG
    assert call(dst_p=None) == ERR_ARG and call(out_p=None) == ERR_ARG and call(ws_p=None) == ERR_ARG
    assert call(src_p=None) == ERR_ARG and call(wsbytes=wsb - 1) == ERR_ARG
    assert call(n=0, wsbytes=0) == 0 and call(src_p=None, n=0) == 0
    assert lib.LZ4B200_launch_count() == l0
    assert call() == 0
    torch.cuda.synchronize()
    assert lib.LZ4B200_launch_count() == l0 + 1


def test_fuzz(lib, oracle):
    rng = np.random.default_rng(4242)
    for it in range(12):
        lv = int(rng.integers(-1, 10))
        blocks = []
        for k in range(int(rng.integers(1, 40))):
            n = int(rng.choice([0, 5, 13, 14, 200, 3000, 65536, 100000]))
            blocks.append(mg.make_input(oracle, n, mg.KINDS[int(rng.integers(0, len(mg.KINDS)))], it * 100 + k))
        cap = int(rng.choice([1 << 30, int(rng.integers(0, 3000)), 65536]))
        got = hc_batch(lib, blocks, cap, lv, src_phase=int(rng.integers(0, 4)), dst_phase=int(rng.integers(0, 4)),
                       src_pad=int(rng.integers(0, 9)), dst_pad=int(rng.integers(0, 9)))
        assert got == [host_hc(b, cap, lv) for b in blocks], (it, lv, cap)
