"""LZ4B200_compress_blocks_hc_destSize on the GPU through the C ABI: the reference's results
(tests/golden/kat_hc_destsize.json) and the host build of the same parse (tests/hc_emul.py), with mixed sizes, odd
strides and phases, guard bytes at and past every slot's limit, targets at and below zero, workspace sizes, two calls on
one workspace, round trips through the GPU decoder, argument errors, launch counts, the Python wrapper and a fuzz loop."""
import numpy as np
import pytest
import torch

import hc_emul as he
from hc_emul import host_hc_dest, mg, mgd

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


def hcd_batch(lib, blocks, target, level, src_phase=0, dst_phase=0, src_pad=0, dst_pad=16, ws=None):
    """One LZ4B200_compress_blocks_hc_destSize call over `blocks` (per-block sizes through d_srcSize), on the minimum
    workspace unless `ws` is given.  Every slot is pre-filled with SENTINEL and checked unchanged at and past
    min(target, bound) (and between slots).  Returns [(ret, consumed, bytes)]."""
    nb = len(blocks)
    sizes = [len(b) for b in blocks]
    src_stride = max(max(sizes), 1) + src_pad
    room = [he.room(n, target) for n in sizes]
    dst_stride = max(max(room), 1) + dst_pad
    src_h = np.zeros(src_phase + nb * src_stride + 16, dtype=np.uint8)
    for i, b in enumerate(blocks):
        src_h[src_phase + i * src_stride:src_phase + i * src_stride + len(b)] = np.frombuffer(bytes(b), dtype=np.uint8)
    src = torch.from_numpy(src_h).to(DEV)
    dst = torch.full((dst_phase + nb * dst_stride + 16,), SENTINEL, dtype=torch.uint8, device=DEV)
    szs = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    outs = torch.full((nb,), UNWRITTEN, dtype=torch.int32, device=DEV)
    cons = torch.full((nb,), UNWRITTEN, dtype=torch.int32, device=DEV)
    if ws is None:
        ws = torch.empty(max(int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(nb)), 1), dtype=torch.uint8, device=DEV)
    l0 = lib.LZ4B200_launch_count()
    rc = lib.LZ4B200_compress_blocks_hc_destSize(src.data_ptr() + src_phase, src_stride, szs.data_ptr(), 0,
                                                 dst.data_ptr() + dst_phase, dst_stride, int(target), int(level),
                                                 outs.data_ptr(), cons.data_ptr(), nb, ws.data_ptr(), ws.numel(),
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
        assert (slot[room[i]:] == SENTINEL).all(), ("write at or past min(target, bound)", i, sizes[i], target, level)
        assert rets[i] != UNWRITTEN and cs[i] != UNWRITTEN
        res.append((int(rets[i]), int(cs[i]), slot[:max(int(rets[i]), 0)].tobytes()))
    return res


def grouped(lib, cases):
    """[(data, target, level)] through one call per distinct (target, level); results in the cases' order"""
    got, groups = [None] * len(cases), {}
    for j, (_, t, lv) in enumerate(cases):
        groups.setdefault((t, lv), []).append(j)
    for (t, lv), js in groups.items():
        for j, r in zip(js, hcd_batch(lib, [cases[j][0] for j in js], t, lv)):
            got[j] = r
    return got


def test_golden_vectors(lib, oracle):
    """Every target of every vector up to 64 KB.  A block is compressed by one thread, so the larger inputs are checked
    at the targets up to 65 536, where the parse stops early, and at 2^30 (their other targets are the CPU suite's)."""
    doc, ins = he.golden("kat_hc_destsize.json")
    data = {iid: mg.make_input(oracle, i["size"], i["kind"], i["seed"]) for iid, i in ins.items()}
    cases, want = [], []
    for iid, lv, rb, rets, cons, dig in doc["vectors"]:
        n = ins[iid]["size"]
        ts = mgd.targets(n, rb)
        keep = [k for k, t in enumerate(ts) if n <= 65536 or t <= 65536 or t == 1 << 30]
        want.append((iid, lv, [ts[k] for k in keep], [rets[k] for k in keep], [cons[k] for k in keep],
                     dig if len(keep) == len(ts) else None))
        cases += [(data[iid], ts[k], lv) for k in keep]
    got = grouped(lib, cases)
    pos = 0
    for iid, lv, ts, rets, cons, dig in want:
        g = got[pos:pos + len(ts)]
        pos += len(ts)
        assert [r for r, _, _ in g] == rets and [c for _, c, _ in g] == cons, (ins[iid], lv)
        if dig is not None:
            assert mgd.run_digest(g) == dig, (ins[iid], lv)
        else:
            assert g == [host_hc_dest(data[iid], t, lv) for t in ts], (ins[iid], lv)
    assert pos == len(got)


def test_run_digests(lib, oracle):
    doc, _ = he.golden("kat_hc_destsize.json")
    got = grouped(lib, list(mgd.random_cases(oracle, doc["run_cases"])))
    chunk = doc["run_chunk"]
    assert [mgd.run_digest(got[k:k + chunk]) for k in range(0, len(got), chunk)] == doc["run_digests"]


@pytest.mark.parametrize("level", [-1, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9])
def test_seeded_batches_match_the_host_build(lib, oracle, level):
    rng = np.random.default_rng(600 + level)
    blocks = [mg.make_input(oracle, int(rng.choice([0, 12, 13, 100, 4096, 30000, 65536])),
                            mg.KINDS[int(rng.integers(0, len(mg.KINDS)))], 8000 + k) for k in range(40)]
    for target in (1 << 30, 16384, 777, 7):
        got = hcd_batch(lib, blocks, target, level, src_phase=3, dst_phase=5, src_pad=7, dst_pad=3)
        assert got == [host_hc_dest(b, target, level) for b in blocks], target


def test_mixed_sizes_in_one_call(lib, oracle):
    blocks = [mg.make_input(oracle, n, "p50", 21 + n) for n in (0, 12, 13, 65536)]
    blocks.append(mg.make_input(oracle, 4 << 20, "p90l60", 5))
    for target, lv in ((1, 9), (13, 2), (4096, 9), (65536, 3), (1 << 30, 3)):
        got = hcd_batch(lib, blocks, target, lv, src_phase=1, dst_phase=2, src_pad=5, dst_pad=1)
        assert got == [host_hc_dest(b, target, lv) for b in blocks], (target, lv)
        assert got[0] == (1, 0, b"\x00")
        if target == 1:
            assert all(g == (1, 0, b"\x00") for g in got)


def test_targets_at_or_below_zero(lib, oracle):
    blocks = [mg.make_input(oracle, n, "p50", 31 + n) for n in (0, 5, 13, 65536)]
    for target in (0, -1, -100000):
        for lv in (1, 9):
            assert hcd_batch(lib, blocks, target, lv) == [(0, len(b), b"") for b in blocks]


def test_minimum_workspace_with_more_blocks_than_slots(lib, oracle):
    """16 384 + 300 blocks on the minimum workspace (16 384 slots, threads take several blocks) against one slot per
    block."""
    nb = 16384 + 300
    data = oracle.datagen(nb * 1000, 0.5, 9)
    blocks = [data[i * 1000:(i + 1) * 1000] for i in range(nb)]
    assert int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(nb)) == 16384 * 256 * 1024
    small = hcd_batch(lib, blocks, 300, 4)
    torch.cuda.empty_cache()
    big_ws = torch.empty(nb * 256 * 1024, dtype=torch.uint8, device=DEV)
    assert hcd_batch(lib, blocks, 300, 4, ws=big_ws) == small
    del big_ws
    torch.cuda.empty_cache()
    for i in (0, 1, 16383, 16384, nb - 1):
        assert small[i] == host_hc_dest(blocks[i], 300, 4), i


def test_two_calls_in_a_row_on_one_workspace(lib, oracle):
    blocks = [mg.make_input(oracle, 65536, mg.KINDS[k % len(mg.KINDS)], 950 + k) for k in range(24)]
    ws = torch.empty(int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(len(blocks))), dtype=torch.uint8, device=DEV)
    for target in (16384, 4096):
        assert hcd_batch(lib, blocks, target, 9, ws=ws) == [host_hc_dest(b, target, 9) for b in blocks], target


def test_round_trip_through_the_gpu_decoder(lib, oracle):
    """The Python wrapper's slots, packed, decode through LZ4B200_decompress_blocks at capacity consumed[i] to exactly
    each block's first consumed[i] bytes."""
    from lz4_b200 import batch
    data = oracle.datagen(64 * 65536 + 1000, 0.5, 6)
    src = torch.from_numpy(data).to(DEV)
    for lv, target in ((2, 4096), (3, 16384), (9, 16384), (9, 1 << 30)):
        slots, sizes, consumed, stride = batch.compress_blocks_hc_dest_size(src, 65536, target, lv)
        n = int(sizes.numel())
        assert n == 65 and int(consumed.numel()) == n
        packed, offs = batch.pack_blocks(slots, stride, sizes)
        cap = int(consumed.max())
        out = torch.full((n * cap + 16,), SENTINEL, dtype=torch.uint8, device=DEV)
        rets = torch.full((n,), UNWRITTEN, dtype=torch.int32, device=DEV)
        wsb = int(lib.LZ4B200_decompress_workspace_bytes_for(n, 1, 0))
        ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=DEV)
        rc = lib.LZ4B200_decompress_blocks(packed.data_ptr(), offs[:-1].contiguous().data_ptr(), sizes.data_ptr(),
                                           out.data_ptr(), None, cap, consumed.data_ptr(), 0, rets.data_ptr(), n,
                                           ws.data_ptr(), wsb, torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        torch.cuda.synchronize()
        assert torch.equal(rets, consumed), (lv, target)
        o, c, h = out.cpu().numpy(), consumed.cpu().numpy(), slots.cpu().numpy()
        for i in range(n):
            blk = data[i * 65536:(i + 1) * 65536]
            assert (o[i * cap:i * cap + c[i]] == blk[:c[i]]).all(), (lv, target, i)
            if i in (0, 17, 64):
                assert (int(sizes[i]), int(c[i]), h[i * stride:i * stride + int(sizes[i])].tobytes()) == \
                    host_hc_dest(blk, target, lv), (lv, target, i)
    with pytest.raises(Exception):
        batch.compress_blocks_hc_dest_size(src, 65536, 4096, 10)


def test_argument_errors_and_launch_counts(lib):
    src = torch.zeros(1024, dtype=torch.uint8, device=DEV)
    dst = torch.zeros(4096, dtype=torch.uint8, device=DEV)
    outs = torch.zeros(4, dtype=torch.int32, device=DEV)
    cons = torch.zeros(4, dtype=torch.int32, device=DEV)
    wsb = int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(4))
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    s = torch.cuda.current_stream().cuda_stream

    def call(src_p=src.data_ptr(), dst_p=dst.data_ptr(), out_p=outs.data_ptr(), cons_p=cons.data_ptr(),
             ws_p=ws.data_ptr(), n=4, level=9, wsbytes=wsb):
        return lib.LZ4B200_compress_blocks_hc_destSize(src_p, 256, None, 256, dst_p, 1024, 1024, level, out_p, cons_p, n,
                                                       ws_p, wsbytes, s)

    l0 = lib.LZ4B200_launch_count()
    for lv in (10, 11, 12, 100):
        assert call(level=lv) == ERR_ARG
    assert call(n=-1) == ERR_ARG
    assert call(dst_p=None) == ERR_ARG and call(out_p=None) == ERR_ARG and call(cons_p=None) == ERR_ARG
    assert call(ws_p=None) == ERR_ARG
    assert call(src_p=None) == ERR_ARG and call(wsbytes=wsb - 1) == ERR_ARG
    assert call(n=0, wsbytes=0) == 0 and call(src_p=None, n=0) == 0
    assert lib.LZ4B200_launch_count() == l0
    assert call() == 0
    torch.cuda.synchronize()
    assert lib.LZ4B200_launch_count() == l0 + 1


def test_fuzz(lib, oracle):
    rng = np.random.default_rng(4343)
    for it in range(12):
        lv = int(rng.integers(-1, 10))
        blocks = []
        for k in range(int(rng.integers(1, 40))):
            n = int(rng.choice([0, 5, 13, 14, 200, 3000, 65536, 100000]))
            blocks.append(mg.make_input(oracle, n, mg.KINDS[int(rng.integers(0, len(mg.KINDS)))], it * 100 + k))
        target = int(rng.choice([1 << 30, int(rng.integers(-2, 40)), int(rng.integers(1, 3000)), 65536]))
        got = hcd_batch(lib, blocks, target, lv, src_phase=int(rng.integers(0, 4)), dst_phase=int(rng.integers(0, 4)),
                        src_pad=int(rng.integers(0, 9)), dst_pad=int(rng.integers(0, 9)))
        assert got == [host_hc_dest(b, target, lv) for b in blocks], (it, lv, target)
