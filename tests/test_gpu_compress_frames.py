"""LZ4B200_compress_frames and batch.compress_frames on the GPU.

Every frame must be the reference's LZ4F_compressFrame output (tests/golden/compress_frames.json) or, for batches the
fixture does not hold, the host model's (tests/compress_frames_model.py: the oracle's LZ4_compress_fast below level 2,
the host build of the HC parses from level 2).  Sources sit at shuffled offsets of every 16-byte phase; outputs abut at
odd offsets between guard bytes, so that a byte written outside [dst_f, dst_f + result_f) shows.

HC blocks stay at or below 256 KB except one 1 MB frame at level 3: one thread parses a block.
"""
import hashlib
import json
import os
import struct

import numpy as np
import pytest
import torch

import compress_frames_model as M
from conftest import GOLDEN
from frame_oracle import decompress_frame
from gpu_util import Recorder

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
GUARD = 0xA5
L31, L32 = 1 << 31, 1 << 32


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    assert lib.LZ4B200_device_count() > 0, "GPU tests need a CUDA device"
    yield lib
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def release_workspaces():
    """frees the workspaces batch keeps per stream after every test: a frames call's workspace holds a slot per
    budgeted block (4 GiB for the frame over 4 GiB), which would otherwise stay allocated for the rest of the session"""
    yield
    from lz4_b200 import batch
    torch.cuda.synchronize()
    batch._workspaces.clear()
    torch.cuda.empty_cache()


def t(a):
    return torch.from_numpy(np.array(a)).to(DEV)                   # a writable copy: the sources may be read-only bytes


def place(datas, seed, gap=64):
    """an arena holding every source at a shuffled offset of every 16-byte phase, 16 readable bytes around each"""
    rng = np.random.default_rng(seed)
    order = rng.permutation(len(datas))
    offs = [0] * len(datas)
    at = 16
    for k, i in enumerate(order):
        at += k % 16                                    # every phase
        offs[i] = at
        at += len(datas[i]) + gap
    arena = np.full(at + 16, 0x3C, dtype=np.uint8)
    for i, d in enumerate(datas):
        arena[offs[i]:offs[i] + len(d)] = np.frombuffer(bytes(d), dtype=np.uint8)
    return arena, np.array(offs, dtype=np.int64)


def run(datas, bsid, level, cs=False, parallel=False, caps=None, budget=None, seed=0, sizes=None):
    """one call over abutting outputs at an odd base between guards: (results, out bytes, out offsets, caps)"""
    from lz4_b200 import batch
    arena, soff = place(datas, seed)
    sizes = np.array([len(d) for d in datas] if sizes is None else sizes, dtype=np.int64)
    if caps is None:
        caps = [M.bound(max(int(n), 0), bsid) for n in sizes]
    caps = np.array(caps, dtype=np.int64)
    room = np.maximum(caps, 0)
    doff = 7 + np.concatenate([[0], np.cumsum(room)[:-1]]).astype(np.int64)
    out = torch.full((int(room.sum()) + 7 + 64,), GUARD, dtype=torch.uint8, device=DEV)
    if budget is None:
        budget = M.budget([int(n) if c >= M.bound(max(int(n), 0), bsid) else -1 for n, c in zip(sizes, caps)], bsid)
    _, res = batch.compress_frames(t(arena), t(soff), t(sizes), max_blocks=budget, block_size_id=bsid, level=level,
                                   content_size=cs, parallel=parallel, out=out, out_offsets=t(doff), capacities=t(caps))
    torch.cuda.synchronize()
    return res.cpu().numpy(), out.cpu().numpy(), doff, caps


def check_written(out, doff, res):
    """every byte outside the frames' [dst_f, dst_f + result_f) is still a guard"""
    mask = np.ones(len(out), dtype=bool)
    for o, r in zip(doff, res):
        if r > 0:
            mask[o:o + r] = False
    bad = np.nonzero(out[mask] != GUARD)[0]
    assert len(bad) == 0, "wrote outside the frames (%d bytes)" % len(bad)


def check_model(datas, bsid, level, cs, res, out, doff, oracle, want=None):
    codec = M.block_codec(oracle, level)
    for f, d in enumerate(datas):
        w = want[f] if want is not None else None
        if w is not None and w < 0:
            assert res[f] == w, (f, res[f], w)
            continue
        fr = M.frame(d, bsid, cs, codec)
        assert res[f] == len(fr), (f, len(d), res[f], len(fr))
        assert out[doff[f]:doff[f] + len(fr)].tobytes() == fr, (f, len(d))
    check_written(out, doff, res)


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLDEN, "compress_frames.json")) as f:
        return json.load(f)["frames"]


# ------------------------------------------------------------------------------------------
# 1. the reference's frames
# ------------------------------------------------------------------------------------------
def test_golden_frames(lib, oracle, golden):
    """every golden frame byte for byte: one call per (level, block size ID, content size), every size of the group in
    it, each output at the reference's exact bound"""
    groups = {}
    for g in golden:
        groups.setdefault((g["level"], g["bsid"], g["content_size"]), []).append(g)
    for (level, bsid, cs), gs in groups.items():
        datas = [M.corpus_data(oracle, g["kind"], g["size"], g["seed"]) for g in gs]
        res, out, doff, caps = run(datas, bsid, level, cs, caps=[g["bound"] for g in gs], seed=level & 0xFF)
        for g, r, o in zip(gs, res, doff):
            assert r == g["length"], (g["id"], r)
            assert hashlib.sha256(out[o:o + r].tobytes()).hexdigest() == g["sha256"], g["id"]
        check_written(out, doff, res)


# ------------------------------------------------------------------------------------------
# 2. random batches, mixed classes, budgets, argument errors
# ------------------------------------------------------------------------------------------
def _random_datas(oracle, rng, n, big=8):
    sizes = list(rng.integers(0, 200000, n - big - 8)) + [0, 1, 15, 16, 65536, 65537, 300000, 1 << 20] + \
        list(rng.integers(1 << 20, 6 << 20, big))
    rng.shuffle(sizes)
    return [oracle.datagen(int(s), 0.5, 1000 + i) if i % 3 else rng.integers(0, 256, int(s), dtype=np.uint8).tobytes()
            for i, s in enumerate(sizes)]


@pytest.mark.parametrize("bsid,level,cs", [(7, 0, True), (5, -5, False), (0, 1, True)])
def test_random_batches_at_the_bound_and_one_below(lib, oracle, bsid, level, cs):
    rng = np.random.default_rng(bsid * 10 + level)
    datas = _random_datas(oracle, rng, 3000 if bsid == 7 else 1200)
    short = rng.random(len(datas)) < 0.2
    caps = [M.bound(len(d), bsid) - int(s) for d, s in zip(datas, short)]
    want = [M.ERR_DSTSIZE if s else None for s in short]
    res, out, doff, _ = run(datas, bsid, level, cs, caps=caps, seed=bsid)
    check_model(datas, bsid, level, cs, res, out, doff, oracle, want)
    if bsid == 7:
        assert len({M.frame_bsid(7, len(d)) for d in datas}) == 4      # every class in one call


def test_budget_rule(lib, oracle):
    """LZ4B200_ERR_LIMIT from the first frame past its class's budget, frames after it included; the other classes and
    the frames before it are unaffected"""
    rng = np.random.default_rng(4)
    datas = _random_datas(oracle, rng, 300, big=6)
    need = M.budget([len(d) for d in datas], 7)
    for budget in (need, [need[0] - 1, need[1], 0, need[3]], [need[0] // 2, need[1] - 1, need[2], 1], [0, 0, 0, 0]):
        res, out, doff, caps = run(datas, 7, 0, True, budget=budget, seed=5)
        v = M.verdicts([len(d) for d in datas], caps, 7, budget)
        check_model(datas, 7, 0, True, res, out, doff, oracle, [r for r, *_ in v])
        assert (budget == need) == all(r is None for r, *_ in v)


def test_per_frame_argument_errors(lib, oracle):
    datas = [oracle.datagen(n, 0.5, n).tobytes() for n in (1000, 70000, 5, 0, 300)]
    sizes = [1000, -1, 5, 0, 300]
    caps = [M.bound(1000, 4), M.bound(70000, 4), -3, 23, M.bound(300, 4)]
    res, out, doff, _ = run(datas, 4, 0, False, caps=caps, sizes=sizes, budget=[4, 0, 0, 0])
    check_model([datas[0], b"", b"", b"", datas[4]], 4, 0, False, res, out, doff, oracle,
                [None, M.ERR_ARG, M.ERR_ARG, None, None])


# ------------------------------------------------------------------------------------------
# 3. the parallel parse, HC levels, the round trip
# ------------------------------------------------------------------------------------------
def test_parallel_parse(lib, oracle):
    """payloads equal compress_buffers(parse="parallel") on the same blocks at capacity size - 1; header, block headers,
    raw rule and EndMark as the model; the frames decode to their sources"""
    from lz4_b200 import batch
    rng = np.random.default_rng(12)
    datas = _random_datas(oracle, rng, 400, big=4)
    res, out, doff, caps = run(datas, 6, 0, True, parallel=True, seed=12)
    blocks = []
    for d in datas:
        bs = M.block_bytes(M.frame_bsid(6, len(d)))
        blocks += [d[i:i + bs] for i in range(0, len(d), bs)]
    arena, boff = place(blocks, 13)
    bsz = np.array([len(b) for b in blocks], dtype=np.int32)
    pout, psz, poff, _ = batch.compress_buffers(t(arena), t(boff), t(bsz), parse="parallel", capacities=t(bsz - 1))
    psz, poff, pout = psz.cpu().numpy(), poff.cpu().numpy(), pout.cpu().numpy()
    k = 0
    for f, d in enumerate(datas):
        n = len(M.blocks(M.frame(d, 6, True, None, payload=lambda i, b: (0, b""))))
        base = k
        fr = M.frame(d, 6, True, None,
                     payload=lambda i, b: (int(psz[base + i]), pout[poff[base + i]:poff[base + i] + max(psz[base + i], 0)].tobytes()))
        k += n
        assert res[f] == len(fr) and out[doff[f]:doff[f] + len(fr)].tobytes() == fr, f
        assert decompress_frame(oracle, fr)[0] == bytes(d), f
    check_written(out, doff, res)


@pytest.mark.parametrize("level", [2, 9, 10, 12])
def test_hc_levels(lib, oracle, level):
    rng = np.random.default_rng(level)
    for bsid in (4, 5):
        sizes = [0, 1, 15, 5000, 65535, 65536, 65537, int(rng.integers(70000, 260000)), 262145][: 9 if bsid == 5 else 8]
        datas = [oracle.datagen(s, 0.5, level * 100 + i).tobytes() if i % 2 else
                 rng.integers(0, 256, s, dtype=np.uint8).tobytes() for i, s in enumerate(sizes)]
        res, out, doff, _ = run(datas, bsid, level, bool(bsid == 5), seed=level)
        check_model(datas, bsid, level, bsid == 5, res, out, doff, oracle)


def test_hc_level_3_one_mb_block(lib, oracle):
    datas = [oracle.datagen((1 << 20) - 5, 0.5, 77).tobytes(), oracle.datagen(3000, 0.5, 78).tobytes()]
    res, out, doff, _ = run(datas, 6, 3, True, seed=3)
    check_model(datas, 6, 3, True, res, out, doff, oracle)


@pytest.mark.parametrize("level,parallel", [(-70000, False), (-5, False), (0, False), (1, True), (3, False), (11, False),
                                            (13, False)])
def test_round_trip(lib, oracle, level, parallel):
    """the frames decode through decompress_frames and through the host model's decoder to their sources"""
    from lz4_b200 import batch
    rng = np.random.default_rng(abs(level))
    sizes = [0, 1, 70000, 65536, 300000] + ([3 << 20] if level < 2 else [])
    datas = [oracle.datagen(s, 0.4, i).tobytes() for i, s in enumerate(sizes)]
    res, out, doff, _ = run(datas, 5, level, bool(rng.integers(2)), parallel=parallel)
    assert (res > 0).all()
    offs = torch.tensor(doff + 64, dtype=torch.int64, device=DEV)        # 16 readable bytes around every frame
    dec, dres, _ = batch.decompress_frames(t(np.concatenate([np.zeros(64, np.uint8), out])), offs, t(res.astype(np.int64)),
                                           torch.tensor([max(s, 1) for s in sizes], dtype=torch.int64, device=DEV),
                                           M.budget(sizes, 5))
    dec, dres = dec.cpu().numpy(), dres.cpu().numpy()
    at = 0
    for f, d in enumerate(datas):
        assert dres[f] == len(d), f
        assert dec[at:at + len(d)].tobytes() == d, f
        assert decompress_frame(oracle, out[doff[f]:doff[f] + res[f]].tobytes())[0] == d, f
        at += max(len(d), 1)


# ------------------------------------------------------------------------------------------
# 4. launches, streams, graphs, far offsets, a frame over 4 GiB
# ------------------------------------------------------------------------------------------
def test_launch_count(lib, oracle):
    datas = [oracle.datagen(n, 0.5, n).tobytes() for n in (100, 70000, 0)]
    for level, parallel, budget, want in ((0, False, None, 7), (9, False, None, 7), (12, False, None, 7),
                                          (1, True, None, 8), (0, False, [0, 0, 0, 0], 5), (1, True, [0, 0, 0, 0], 5)):
        before = lib.LZ4B200_launch_count()
        run(datas, 4, level, parallel=parallel, budget=budget)
        assert lib.LZ4B200_launch_count() - before == want, (level, parallel, budget)


def test_side_stream_and_graph_replay(lib, oracle):
    from lz4_b200 import batch
    datas = [oracle.datagen(n, 0.5, 40 + i).tobytes() for i, n in enumerate([0, 999, 65536, 70001, 300000, 5 << 20])]
    arena, soff = place(datas, 21)
    sizes = np.array([len(d) for d in datas], dtype=np.int64)
    caps = np.array([M.bound(len(d), 7) for d in datas], dtype=np.int64)
    doff = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64) + 3
    budget = M.budget(sizes, 7)
    src, offs, sz, cp, do = t(arena), t(soff), t(sizes), t(caps), t(doff)
    ws = torch.empty(batch.compress_frames_workspace_bytes(len(datas), budget, 0), dtype=torch.uint8, device=DEV)
    out = torch.full((int(caps.sum()) + 64,), GUARD, dtype=torch.uint8, device=DEV)
    res = torch.empty(len(datas), dtype=torch.int64, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.cuda.stream(side):
            batch.compress_frames(src, offs, sz, max_blocks=budget, block_size_id=7, out=out, out_offsets=do,
                                  capacities=cp, results=res, workspace=ws, stream=side)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    side.synchronize()
    check_model(datas, 7, 0, False, res.cpu().numpy(), out.cpu().numpy(), doff, oracle)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        batch.compress_frames(src, offs, sz, max_blocks=budget, block_size_id=7, out=out, out_offsets=do, capacities=cp,
                              results=res, workspace=ws, stream=s)
    for seed in (1, 2):
        new = [oracle.datagen(len(d), 0.3 * seed, 500 + seed * 10 + i).tobytes() for i, d in enumerate(datas)]
        host = arena.copy()
        for i, d in enumerate(new):
            host[soff[i]:soff[i] + len(d)] = np.frombuffer(d, dtype=np.uint8)
        src.copy_(t(host))
        out.fill_(GUARD)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        check_model(new, 7, 0, False, res.cpu().numpy(), out.cpu().numpy(), doff, oracle)


def test_far_offsets(lib, oracle):
    """sources and frames at and across 2^31 and 2^32 in one arena; the guard bytes around every frame hold"""
    from lz4_b200 import batch
    datas = [oracle.datagen(n, 0.5, 60 + i).tobytes() for i, n in enumerate([70000, 300000, 5000, 65536, 200001])]
    lines = [L31 - 1, L31 + 400000, L32 - 3, L32 + 400017, L32 - 400000]     # across 2^31 and 2^32, and past 2^32
    arena = torch.full((L32 + (16 << 20),), GUARD, dtype=torch.uint8, device=DEV)
    caps = [M.bound(len(d), 5) for d in datas]
    for role in ("src", "dst"):
        soff = list(lines) if role == "src" else [1000 + 400000 * i for i in range(5)]
        doff = list(lines) if role == "dst" else [(1 << 30) + 400000 * i for i in range(5)]
        for o, d in zip(soff, datas):
            arena[o:o + len(d)] = t(np.frombuffer(d, dtype=np.uint8))
        _, res = batch.compress_frames(arena, t(np.array(soff)), t(np.array([len(d) for d in datas])),
                                       max_blocks=M.budget([len(d) for d in datas], 5), block_size_id=5,
                                       out=arena, out_offsets=t(np.array(doff)), capacities=t(np.array(caps)))
        torch.cuda.synchronize()
        res = res.cpu().numpy()
        for f, d in enumerate(datas):
            fr = M.frame(d, 5, False, M.block_codec(oracle, 0))
            assert res[f] == len(fr), (role, f)
            win = arena[doff[f] - 64:doff[f] + len(fr) + 64].cpu().numpy()
            assert win[64:64 + len(fr)].tobytes() == fr, (role, f)
            assert (win[:64] == GUARD).all() and (win[64 + len(fr):] == GUARD).all(), (role, f)
        arena.fill_(GUARD)
    del arena
    torch.cuda.empty_cache()


def test_frame_over_4_gib(lib, oracle):
    """one FAST frame of 2^32 + 19 bytes at block size ID 7, against the model's digest: the source repeats a 64 MB
    period, so the model compresses 16 distinct 4 MB blocks and a 19-byte tail"""
    from lz4_b200 import batch
    period, n = 64 << 20, L32 + 19
    unit = oracle.datagen(period, 0.5, 7)
    src = t(unit).repeat(n // period + 1)[:n]
    bs = 4 << 20
    h = hashlib.sha256(M.header(7, n))
    comp = {}
    length = 15
    for at in range(0, n, bs):
        blk = unit[at % period:at % period + min(bs, n - at)].tobytes() if n - at >= bs else \
            np.asarray(src[at:].cpu()).tobytes()
        key = (at % period, len(blk))
        if key not in comp:
            r, c = oracle.compress(blk, 1, len(blk) - 1)
            comp[key] = struct.pack("<I", r) + c[:r] if 0 < r < len(blk) else struct.pack("<I", len(blk) | 1 << 31) + blk
        h.update(comp[key])
        length += len(comp[key])
    h.update(b"\0\0\0\0")
    length += 4
    cap = M.bound(n, 7)
    out = torch.full((cap + 32,), GUARD, dtype=torch.uint8, device=DEV)
    _, res = batch.compress_frames(src, torch.zeros(1, dtype=torch.int64, device=DEV),
                                   torch.tensor([n], dtype=torch.int64, device=DEV), max_blocks=[0, 0, 0, 1025],
                                   block_size_id=7, content_size=True, out=out,
                                   out_offsets=torch.zeros(1, dtype=torch.int64, device=DEV),
                                   capacities=torch.tensor([cap], dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    assert int(res[0]) == length
    host = out.cpu().numpy()
    assert hashlib.sha256(memoryview(host[:length])).hexdigest() == h.hexdigest()
    assert (host[length:] == GUARD).all()
    del src, out
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------
# 5. the wrapper's checks, through the recording stand-in
# ------------------------------------------------------------------------------------------
class FramesRecorder(Recorder):
    SIZES = Recorder.SIZES + ("LZ4B200_compress_frames_workspace_bytes", "LZ4B200_compressFrameBound")


@pytest.fixture
def rec(monkeypatch):
    from lz4_b200 import _lib, batch
    r = FramesRecorder(_lib.load())
    monkeypatch.setattr(_lib, "load", lambda: r)
    monkeypatch.setattr(batch, "_workspaces", {})
    return r


N = 4


def _z(n, dtype=torch.uint8, dev=DEV):
    return torch.zeros(n, dtype=dtype, device=dev)


def _good():
    return dict(src=_z(4096), offsets=_z(N, torch.int64), sizes=torch.full((N,), 100, dtype=torch.int64, device=DEV),
                max_blocks=[N, 0, 0, 0], out=_z(4096), out_offsets=_z(N, torch.int64),
                capacities=torch.full((N,), 200, dtype=torch.int64, device=DEV), results=_z(N, torch.int64))


def test_compress_frames_wrapper(rec):
    from lz4_b200 import batch
    batch.compress_frames(**_good())
    assert [c[0] for c in rec.calls] == ["LZ4B200_compress_frames"]
    args = rec.calls[0][1]
    assert args[7] == N and args[8:12] == (4, 0, 0, 0) and list(args[12]) == [N, 0, 0, 0]
    rec.calls.clear()
    batch.compress_frames(**dict(_good(), max_blocks=None, capacities=None, out=None, out_offsets=None, results=None),
                          block_size_id=7, level=9, content_size=True)
    args = rec.calls[0][1]
    assert args[8:12] == (7, 9, 1, 0) and list(args[12]) == [N, 0, 0, 0]
    bad = [("src", _z(16, torch.int8)), ("offsets", _z(N, torch.int32)), ("offsets", _z(N - 1, torch.int64)),
           ("sizes", _z(N, torch.int32)), ("capacities", _z(N - 1, torch.int64)), ("capacities", _z(N, torch.int32)),
           ("results", _z(N - 1, torch.int64)), ("out_offsets", _z(N, torch.int64, "cpu")), ("out", _z(64, dev="cpu")),
           ("max_blocks", [1, 2, 3]), ("max_blocks", [-1, 0, 0, 0]), ("max_blocks", [0, 0, 0, 2 ** 31]),
           ("block_size_id", 3), ("block_size_id", 8), ("level", 2 ** 31), ("workspace", _z(8))]
    for arg, v in bad:
        kw = _good()
        kw[arg] = v
        rec.calls.clear()
        with pytest.raises(ValueError):
            batch.compress_frames(**kw)
        assert not rec.calls, arg
    rec.calls.clear()
    with pytest.raises(ValueError):
        batch.compress_frames(**_good(), parallel=True, level=2)
    s = torch.cuda.Stream()
    ws = _z(1 << 20)
    for drop in ("max_blocks", "out", "capacities"):
        kw = _good()
        kw[drop] = None
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
            with pytest.raises(ValueError):
                batch.compress_frames(stream=s, workspace=ws, **kw)
    assert not rec.calls
    torch.cuda.synchronize()
