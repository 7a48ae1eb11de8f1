"""LZ4B200_compress_blocks_hc_opt and LZ4B200_compress_blocks_hc_opt_destSize (LZ4HC levels 10 .. 12) on the GPU through
the C ABI: the reference's results (tests/golden/kat_hc_opt.json) and the host build of the same parse
(tests/hc_emul.py), with mixed sizes, odd strides and phases, guard bytes at and past every slot's limit, poisoned
and small workspaces, two calls on one workspace, round trips through the GPU decoder, side streams and graph capture,
argument errors, launch counts and the Python wrappers.

One thread parses a block, so a call takes as long as its slowest block (about 1 s for a 64 KB P50 block at level 12 on
an H100): no block above 256 KB goes through levels 11 and 12 here, and the calls are grouped.  The CPU suite checks
every vector of the golden file in full."""
import numpy as np
import pytest
import torch

import hc_emul as he
from hc_emul import host_hc_opt, host_hc_opt_dest, mg, mgd, mgo

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
UNWRITTEN = -123456789
DEV = "cuda:0"
ERR_ARG = -1
SLOT = 262144 + 4099 * 16
SHARED_TARGETS = [1, 7, 16, 100, 4096, 16384, 65536, 1 << 30]


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    if lib.LZ4B200_device_count() <= 0:
        pytest.skip("no CUDA device")
    yield lib
    # the file allocates workspaces of several GB and captures a graph: hand their cached memory back, so that the
    # files after this one allocate on the device as they would without it
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def limit_of(n, limit):
    return max(min(limit, mg.compress_bound(n)), 0)


def opt_batch(lib, blocks, limit, level, fill, src_phase=0, dst_phase=0, src_pad=0, dst_pad=16, ws=None, stream=None,
              launches=1):
    """One LZ4B200_compress_blocks_hc_opt (fill: _destSize) call over `blocks` (per-block sizes through d_srcSize) with
    dstCap / targetDstSize = limit, on the minimum workspace unless `ws` is given.  Every slot is pre-filled with
    SENTINEL and checked unchanged at and past min(limit, bound) and between slots.  Returns [(ret, bytes)], or
    [(ret, consumed, bytes)] in fill mode."""
    nb = len(blocks)
    sizes = [len(b) for b in blocks]
    src_stride = max(max(sizes), 1) + src_pad
    room = [limit_of(n, limit) for n in sizes]
    dst_stride = max(max(room), 1) + dst_pad
    src_h = np.zeros(src_phase + nb * src_stride + 16, dtype=np.uint8)
    for i, b in enumerate(blocks):
        src_h[src_phase + i * src_stride:src_phase + i * src_stride + len(b)] = np.frombuffer(bytes(b), dtype=np.uint8)
    st = stream or torch.cuda.current_stream()
    with torch.cuda.stream(st):
        src = torch.from_numpy(src_h).to(DEV)
        dst = torch.full((dst_phase + nb * dst_stride + 16,), SENTINEL, dtype=torch.uint8, device=DEV)
        szs = torch.tensor(sizes, dtype=torch.int32, device=DEV)
        outs = torch.full((nb,), UNWRITTEN, dtype=torch.int32, device=DEV)
        cons = torch.full((nb,), UNWRITTEN, dtype=torch.int32, device=DEV)
        if ws is None:
            ws = torch.empty(max(int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(nb)), 1), dtype=torch.uint8,
                             device=DEV)
    l0 = lib.LZ4B200_launch_count()
    if fill:
        rc = lib.LZ4B200_compress_blocks_hc_opt_destSize(src.data_ptr() + src_phase, src_stride, szs.data_ptr(), 0,
                                                         dst.data_ptr() + dst_phase, dst_stride, int(limit), int(level),
                                                         outs.data_ptr(), cons.data_ptr(), nb, ws.data_ptr(), ws.numel(),
                                                         st.cuda_stream)
    else:
        rc = lib.LZ4B200_compress_blocks_hc_opt(src.data_ptr() + src_phase, src_stride, szs.data_ptr(), 0,
                                                dst.data_ptr() + dst_phase, dst_stride, int(limit), int(level),
                                                outs.data_ptr(), nb, ws.data_ptr(), ws.numel(), st.cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert lib.LZ4B200_launch_count() == l0 + launches
    d = dst.cpu().numpy()
    rets, cs = outs.cpu().numpy(), cons.cpu().numpy()
    assert (d[:dst_phase] == SENTINEL).all() and (d[dst_phase + nb * dst_stride:] == SENTINEL).all()
    res = []
    for i in range(nb):
        slot = d[dst_phase + i * dst_stride:dst_phase + (i + 1) * dst_stride]
        assert (slot[room[i]:] == SENTINEL).all(), ("write at or past the limit", i, sizes[i], limit, level)
        assert rets[i] != UNWRITTEN
        out = slot[:max(int(rets[i]), 0)].tobytes()
        if fill:
            assert cs[i] != UNWRITTEN
            res.append((int(rets[i]), int(cs[i]), out))
        else:
            assert cs[i] == UNWRITTEN
            res.append((int(rets[i]), out))
    return res


def grouped(lib, cases, fill):
    """[(data, limit, level)] through one call per distinct (limit, level); results in the cases' order"""
    got, groups = [None] * len(cases), {}
    for j, (_, t, lv) in enumerate(cases):
        groups.setdefault((t, lv), []).append(j)
    for (t, lv), js in groups.items():
        for j, r in zip(js, opt_batch(lib, [cases[j][0] for j in js], t, lv, fill)):
            got[j] = r
    return got


def host(data, limit, level, fill):
    return host_hc_opt_dest(data, limit, level) if fill else host_hc_opt(data, limit, level)


@pytest.fixture(scope="module")
def golden(oracle):
    doc, ins = he.golden("kat_hc_opt.json")
    return doc, ins, {iid: mg.make_input(oracle, i["size"], i["kind"], i["seed"]) for iid, i in ins.items()}


def test_golden_vectors_plain(lib, golden):
    """Every input up to 256 KB at the bound, one call per level: the capacity is the largest bound, which routes every
    block as its own bound does (unlimited)."""
    doc, ins, data = golden
    by_level = {}
    for iid, lv, rb, rets, dig in doc["vectors"]:
        if ins[iid]["size"] <= 256 << 10:
            by_level.setdefault(lv, []).append((iid, rb))
    for lv, vs in sorted(by_level.items()):
        cap = max(mg.compress_bound(ins[iid]["size"]) for iid, _ in vs)
        got = opt_batch(lib, [data[iid] for iid, _ in vs], cap, lv, False)
        for (iid, rb), (r, out) in zip(vs, got):
            assert r == rb and (r, out) == host_hc_opt(data[iid], cap, lv), (ins[iid], lv)


def test_golden_vectors_fill(lib, golden):
    """The shared targets, one call per (target, level); inputs above 256 KB only at level 10 and targets up to 65 536,
    where the parse stops early; levels 13 and 100 at three of the targets."""
    doc, ins, data = golden
    cases, want = [], []
    for iid, lv, rb, rets, cons, dig in doc["dest_vectors"]:
        n = ins[iid]["size"]
        ts = mgd.targets(n, rb)
        for t in SHARED_TARGETS:
            if (n > 256 << 10 and (t > 65536 or lv > 10)) or (lv > 12 and t not in (16, 4096, 1 << 30)):
                continue
            k = ts.index(t)
            cases.append((data[iid], t, lv))
            want.append((iid, lv, t, rets[k], cons[k]))
    got = grouped(lib, cases, True)
    for (iid, lv, t, r, c), g, (d, _, _) in zip(want, got, cases):
        assert g[:2] == (r, c) and g == host_hc_opt_dest(d, t, lv), (ins[iid], lv, t)
    assert len({(t, lv) for _, t, lv in cases}) <= 32


def test_run_digests(lib, oracle):
    doc, _ = he.golden("kat_hc_opt.json")
    chunk = doc["run_chunk"]
    got = grouped(lib, list(mgo.random_cases(oracle, doc["run_cases"], mgo.PLAIN_SEED)), False)
    assert [mg.run_digest(got[k:k + chunk]) for k in range(0, len(got), chunk)] == doc["run_digests"]
    got = grouped(lib, list(mgo.random_cases(oracle, doc["run_cases"], mgo.DEST_SEED)), True)
    assert [mgd.run_digest(got[k:k + chunk]) for k in range(0, len(got), chunk)] == doc["dest_run_digests"]


def seeded_blocks(oracle, seed, count=24):
    rng = np.random.default_rng(seed)
    return [mg.make_input(oracle, int(rng.choice([0, 12, 13, 100, 4096, 30000, 65536])),
                          mg.KINDS[int(rng.integers(0, len(mg.KINDS)))], seed * 100 + k) for k in range(count)]


@pytest.mark.parametrize("level", [10, 11, 12, 13])
def test_seeded_batches_match_the_host_build(lib, oracle, level):
    blocks = seeded_blocks(oracle, 700 + level)
    for fill, limit in ((False, 1 << 30), (False, 777), (True, 16384), (True, 7)):
        got = opt_batch(lib, blocks, limit, level, fill, src_phase=3, dst_phase=5, src_pad=7, dst_pad=3)
        assert got == [host(b, limit, level, fill) for b in blocks], (fill, limit)


def test_poisoned_workspace(lib, oracle):
    """A workspace of 0xFF bytes, and one of random bytes, give what a fresh one gives."""
    blocks = seeded_blocks(oracle, 41, 16)
    nbytes = int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(len(blocks)))
    assert nbytes == len(blocks) * SLOT
    fresh = opt_batch(lib, blocks, 1 << 30, 12, False)
    ff = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)
    assert opt_batch(lib, blocks, 1 << 30, 12, False, ws=ff) == fresh
    rnd = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device=DEV,
                        generator=torch.Generator(device=DEV).manual_seed(5))
    assert opt_batch(lib, blocks, 4096, 12, True, ws=rnd) == [host_hc_opt_dest(b, 4096, 12) for b in blocks]
    assert fresh == [host_hc_opt(b, 1 << 30, 12) for b in blocks]


def test_minimum_workspace_with_more_blocks_than_slots(lib, oracle):
    """16 384 + 300 blocks on the minimum workspace (16 384 slots, threads take several blocks) against one slot per
    block."""
    nb = 16384 + 300
    data = oracle.datagen(nb * 1000, 0.5, 19)
    blocks = [data[i * 1000:(i + 1) * 1000] for i in range(nb)]
    assert int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(nb)) == 16384 * SLOT
    small = opt_batch(lib, blocks, 300, 11, True)
    torch.cuda.empty_cache()
    big_ws = torch.empty(nb * SLOT, dtype=torch.uint8, device=DEV)
    assert opt_batch(lib, blocks, 300, 11, True, ws=big_ws) == small
    del big_ws
    torch.cuda.empty_cache()
    for i in (0, 1, 16383, 16384, nb - 1):
        assert small[i] == host_hc_opt_dest(blocks[i], 300, 11), i


def test_two_calls_in_a_row_on_one_workspace(lib, oracle):
    blocks = [mg.make_input(oracle, 65536, mg.KINDS[k % len(mg.KINDS)], 960 + k) for k in range(14)]
    ws = torch.empty(int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(len(blocks))), dtype=torch.uint8,
                     device=DEV)
    assert opt_batch(lib, blocks, 1 << 30, 10, False, ws=ws) == [host_hc_opt(b, 1 << 30, 10) for b in blocks]
    assert opt_batch(lib, blocks, 4096, 12, True, ws=ws) == [host_hc_opt_dest(b, 4096, 12) for b in blocks]


def test_round_trip_through_the_gpu_decoder_and_the_python_wrappers(lib, oracle):
    """Both wrappers' slots, packed, decode through LZ4B200_decompress_blocks: the plain mode at the block size to the
    input, the fill mode at capacity consumed[i] to each block's first consumed[i] bytes."""
    from lz4_b200 import batch
    data = oracle.datagen(24 * 65536 + 1000, 0.5, 16)
    src = torch.from_numpy(data).to(DEV)

    def decode(slots, stride, sizes, cap, caps=None):
        n = int(sizes.numel())
        packed, offs = batch.pack_blocks(slots, stride, sizes)
        out = torch.full((n * cap + 16,), SENTINEL, dtype=torch.uint8, device=DEV)
        rets = torch.full((n,), UNWRITTEN, dtype=torch.int32, device=DEV)
        wsb = int(lib.LZ4B200_decompress_workspace_bytes_for(n, caps is not None, 0 if caps is not None else cap))
        ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=DEV)
        rc = lib.LZ4B200_decompress_blocks(packed.data_ptr(), offs[:-1].contiguous().data_ptr(), sizes.data_ptr(),
                                           out.data_ptr(), None, cap, caps.data_ptr() if caps is not None else None,
                                           0 if caps is not None else cap, rets.data_ptr(), n, ws.data_ptr(), wsb,
                                           torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        torch.cuda.synchronize()
        return out.cpu().numpy(), rets

    slots, sizes, stride = batch.compress_blocks_hc_opt(src, 65536, 11)
    n = int(sizes.numel())
    assert n == 25
    o, rets = decode(slots, stride, sizes, 65536)
    want = [min(65536, len(data) - i * 65536) for i in range(n)]
    assert rets.cpu().tolist() == want
    h = slots.cpu().numpy()
    for i in range(n):
        assert (o[i * 65536:i * 65536 + want[i]] == data[i * 65536:i * 65536 + want[i]]).all(), i
    for i in (0, 24):
        blk = data[i * 65536:(i + 1) * 65536]
        assert (int(sizes[i]), h[i * stride:i * stride + int(sizes[i])].tobytes()) == \
            host_hc_opt(blk, mg.compress_bound(65536), 11), i

    slots, sizes, consumed, stride = batch.compress_blocks_hc_opt_dest_size(src, 65536, 16384)
    cap = int(consumed.max())
    o, rets = decode(slots, stride, sizes, cap, consumed)
    assert torch.equal(rets, consumed)
    c, h = consumed.cpu().numpy(), slots.cpu().numpy()
    for i in range(n):
        blk = data[i * 65536:(i + 1) * 65536]
        assert (o[i * cap:i * cap + c[i]] == blk[:c[i]]).all(), i
        if i in (0, 13, 24):
            assert (int(sizes[i]), int(c[i]), h[i * stride:i * stride + int(sizes[i])].tobytes()) == \
                host_hc_opt_dest(blk, 16384, 12), i
    for lv in (9, 1, 0, -1):
        with pytest.raises(Exception):
            batch.compress_blocks_hc_opt(src, 65536, lv)
        with pytest.raises(Exception):
            batch.compress_blocks_hc_opt_dest_size(src, 65536, 4096, lv)


def test_side_stream_and_graph_capture(lib, oracle):
    """A call on a non-blocking side stream, queued behind a sleep, and one captured into a CUDA graph and replayed,
    give the default stream's results."""
    from lz4_b200 import batch
    blocks = seeded_blocks(oracle, 77, 12)
    want = opt_batch(lib, blocks, 2000, 10, True)
    # PyTorch creates its pool streams non-blocking.  A high-priority one comes from its own round robin, so the
    # default-priority streams that later test files take stay the ones they take without this file.
    side = torch.cuda.Stream(priority=-1)
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
    assert opt_batch(lib, blocks, 2000, 10, True, stream=side) == want

    data = oracle.datagen(6 * 65536, 0.5, 23)
    src = torch.from_numpy(data).to(DEV)
    ref_slots, ref_sizes, stride = batch.compress_blocks_hc_opt(src, 65536, 10)
    ws = torch.empty(int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(6)), dtype=torch.uint8, device=DEV)
    slots = torch.full_like(ref_slots, SENTINEL)
    sizes = torch.full_like(ref_sizes, UNWRITTEN)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            batch.compress_blocks_hc_opt(src, 65536, 10, slots=slots, slot_stride=stride, out_sizes=sizes, workspace=ws)
    torch.cuda.synchronize()
    assert bool((sizes == UNWRITTEN).all())
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(sizes, ref_sizes)
    for i in range(6):
        k = int(ref_sizes[i])
        assert torch.equal(slots[i * stride:i * stride + k], ref_slots[i * stride:i * stride + k]), i


def test_argument_errors_and_launch_counts(lib):
    src = torch.zeros(1024, dtype=torch.uint8, device=DEV)
    dst = torch.zeros(4096, dtype=torch.uint8, device=DEV)
    outs = torch.zeros(4, dtype=torch.int32, device=DEV)
    cons = torch.zeros(4, dtype=torch.int32, device=DEV)
    wsb = int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(4))
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    s = torch.cuda.current_stream().cuda_stream

    def plain(src_p=src.data_ptr(), dst_p=dst.data_ptr(), out_p=outs.data_ptr(), ws_p=ws.data_ptr(), n=4, level=12,
              wsbytes=wsb):
        return lib.LZ4B200_compress_blocks_hc_opt(src_p, 256, None, 256, dst_p, 1024, 1024, level, out_p, n, ws_p,
                                                  wsbytes, s)

    def dest(src_p=src.data_ptr(), dst_p=dst.data_ptr(), out_p=outs.data_ptr(), cons_p=cons.data_ptr(),
             ws_p=ws.data_ptr(), n=4, level=12, wsbytes=wsb):
        return lib.LZ4B200_compress_blocks_hc_opt_destSize(src_p, 256, None, 256, dst_p, 1024, 1024, level, out_p,
                                                           cons_p, n, ws_p, wsbytes, s)

    l0 = lib.LZ4B200_launch_count()
    for call in (plain, dest):
        for lv in (9, 1, 0, -1):
            assert call(level=lv) == ERR_ARG
        assert call(n=-1) == ERR_ARG
        assert call(dst_p=None) == ERR_ARG and call(out_p=None) == ERR_ARG and call(ws_p=None) == ERR_ARG
        assert call(src_p=None) == ERR_ARG and call(wsbytes=wsb - 1) == ERR_ARG
        assert call(n=0, wsbytes=0) == 0 and call(src_p=None, n=0, level=100) == 0
    assert dest(cons_p=None) == ERR_ARG
    assert lib.LZ4B200_launch_count() == l0
    for k, call in enumerate((plain, dest)):
        assert call(level=13) == 0
        torch.cuda.synchronize()
        assert lib.LZ4B200_launch_count() == l0 + k + 1
