"""LZ4B200_compress_legacy and batch.compress_legacy on the GPU.

Every stream must be what the reference tool's `lz4 -l` writes (tests/golden/compress_legacy.json) or, for batches the
fixture does not hold, the host model's (tests/compress_legacy_model.py: the oracle's LZ4_compress_fast below level 3,
the host build of the HC parses from level 3).  Sources sit at shuffled offsets of every 16-byte phase; outputs abut at
odd offsets between guard bytes, so that a byte written outside [dst_f, dst_f + result_f) shows.

HC sources stay at or below 1 MB except one 8 MiB chunk of random bytes at levels 3 and 10: one thread parses a chunk.
"""
import hashlib
import json
import os
import struct
import time

import numpy as np
import pytest
import torch

import compress_legacy_model as M
from conftest import GOLDEN
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
    """frees the workspaces batch keeps per stream after every test: the call's workspace holds a slot of 8 MiB per
    budgeted chunk (4 GiB for the file over 4 GiB), which would otherwise stay allocated for the rest of the session"""
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
        at += k % 16
        offs[i] = at
        at += len(datas[i]) + gap
    arena = np.full(at + 16, 0x3C, dtype=np.uint8)
    for i, d in enumerate(datas):
        arena[offs[i]:offs[i] + len(d)] = np.frombuffer(bytes(d), dtype=np.uint8)
    return arena, np.array(offs, dtype=np.int64)


def run(datas, level, caps=None, budget=None, seed=0, sizes=None):
    """one call over abutting outputs at an odd base between guards: (results, out bytes, out offsets, caps)"""
    from lz4_b200 import batch
    arena, soff = place(datas, seed)
    sizes = np.array([len(d) for d in datas] if sizes is None else sizes, dtype=np.int64)
    if caps is None:
        caps = [M.bound(max(int(n), 0)) for n in sizes]
    caps = np.array(caps, dtype=np.int64)
    room = np.maximum(caps, 0)
    doff = 7 + np.concatenate([[0], np.cumsum(room)[:-1]]).astype(np.int64)
    out = torch.full((int(room.sum()) + 7 + 64,), GUARD, dtype=torch.uint8, device=DEV)
    if budget is None:
        budget = sum(M.n_chunks(int(n)) for n, c in zip(sizes, caps) if n >= 0 and c >= M.bound(int(n)))
    _, res = batch.compress_legacy(t(arena), t(soff), t(sizes), max_blocks=budget, level=level, out=out,
                                   out_offsets=t(doff), capacities=t(caps))
    torch.cuda.synchronize()
    return res.cpu().numpy(), out.cpu().numpy(), doff, caps


def check_written(out, doff, res):
    """every byte outside the streams' [dst_f, dst_f + result_f) is still a guard"""
    mask = np.ones(len(out), dtype=bool)
    for o, r in zip(doff, res):
        if r > 0:
            mask[o:o + r] = False
    bad = np.nonzero(out[mask] != GUARD)[0]
    assert len(bad) == 0, "wrote outside the streams (%d bytes)" % len(bad)


def check_model(datas, level, res, out, doff, oracle, want=None):
    codec = M.block_codec(oracle, level)
    for f, d in enumerate(datas):
        if want is not None and want[f] is not None:
            assert res[f] == want[f], (f, res[f], want[f])
            continue
        st = M.stream(d, codec)
        assert res[f] == len(st), (f, len(d), res[f], len(st))
        assert out[doff[f]:doff[f] + len(st)].tobytes() == st, (f, len(d))
    check_written(out, doff, res)


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLDEN, "compress_legacy.json")) as f:
        return json.load(f)["streams"]


# ------------------------------------------------------------------------------------------
# 1. the reference tool's streams
# ------------------------------------------------------------------------------------------
def test_golden_streams(lib, oracle, golden):
    """every golden stream byte for byte, one call per level, each output at the bound; then the same call one byte
    below it: LZ4B200_ERR_DSTSIZE, with every byte of the output still a guard"""
    groups = {}
    for g in golden:
        groups.setdefault(g["level"], []).append(g)
    for level, gs in groups.items():
        datas = [M.corpus_data(oracle, g["kind"], g["size"], g["seed"]) for g in gs]
        t0 = time.perf_counter()
        res, out, doff, caps = run(datas, level, caps=[g["bound"] for g in gs], seed=abs(level) & 0xFF)
        elapsed = time.perf_counter() - t0
        if any(g["kind"] == "split" for g in gs):
            print("level %d call with an 8 MiB random chunk: %.2f s" % (level, elapsed))
        for g, r, o in zip(gs, res, doff):
            assert r == g["length"], (g["id"], r)
            assert hashlib.sha256(out[o:o + r].tobytes()).hexdigest() == g["sha256"], g["id"]
        check_written(out, doff, res)
        if level >= 3:
            continue                                    # the capacity rule is decided before the encode
        res, out, doff, caps = run(datas, level, caps=[g["bound"] - 1 for g in gs], seed=7)
        assert (res == M.ERR_DSTSIZE).all(), level
        assert (out == GUARD).all()


# ------------------------------------------------------------------------------------------
# 2. many files, budgets, argument errors, the level routing
# ------------------------------------------------------------------------------------------
def _random_datas(oracle, rng, n):
    sizes = np.where(rng.random(n) < 0.005, rng.integers(M.CHUNK - 3, 20 * M.MIB, n),
                     np.where(rng.random(n) < 0.2, 0, rng.integers(0, 200000, n)))
    return [oracle.datagen(int(s), float(rng.choice([0.2, 0.5, 0.9])), int(rng.integers(1 << 30))).tobytes()
            for s in sizes]


@pytest.mark.parametrize("level", [1, -17])
def test_thousands_of_files(lib, oracle, level):
    """3000 files of 0 B to 20 MiB at shuffled source offsets, abutting outputs, against the model"""
    rng = np.random.default_rng(level & 0xFFFF)
    datas = _random_datas(oracle, rng, 3000)
    assert max(len(d) for d in datas) > M.CHUNK and min(len(d) for d in datas) == 0
    res, out, doff, caps = run(datas, level, seed=5)
    check_model(datas, level, res, out, doff, oracle)


def test_budget_rule(lib, oracle):
    """exact fit, one chunk short (the first file over the budget and every later one with chunks fail; empty files
    after it fail too), and 0"""
    datas = [oracle.datagen(n, 0.5, 30 + i).tobytes() for i, n in enumerate([M.CHUNK + 1, 0, 5000, M.CHUNK, 0, 17])]
    need = sum(M.n_chunks(len(d)) for d in datas)
    for budget in (need, need - 1, 2, 0):
        res, out, doff, caps = run(datas, 1, budget=budget, seed=budget)
        want = [None if v[0] is None else v[0] for v in M.verdicts([len(d) for d in datas], caps, budget)]
        check_model(datas, 1, res, out, doff, oracle, want)


def test_per_file_argument_errors(lib, oracle):
    datas = [oracle.datagen(n, 0.5, 50 + i).tobytes() for i, n in enumerate([1000, 2000, 3000, 4000, 5000])]
    sizes = [1000, -1, 3000, 4000, 5000]
    caps = [M.bound(1000), 100, -1, M.bound(4000) - 1, M.bound(5000)]
    res, out, doff, _ = run(datas, 1, caps=caps, sizes=sizes, budget=3)
    check_model(datas, 1, res, out, doff, oracle, [None, M.ERR_ARG, M.ERR_ARG, M.ERR_DSTSIZE, None])


def test_level_routing(lib, oracle):
    """--fast=N is acceleration N (not the frame writer's N + 1), level 2 the fast parse, level 13 level 12"""
    d = oracle.datagen(300000, 0.5, 99).tobytes()
    outs = {}
    for level in (-17, 2, 12, 13):
        res, out, doff, _ = run([d], level)
        outs[level] = out[doff[0]:doff[0] + res[0]].tobytes()
    fast = lambda a: M.stream(d, lambda b, cap: oracle.compress(b, a, cap))
    assert outs[-17] == fast(17) != fast(18)
    assert outs[2] == fast(1)
    assert outs[13] == outs[12] == M.stream(d, M.block_codec(oracle, 12))


# ------------------------------------------------------------------------------------------
# 3. the round trip through decompress_files
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", [-5, 1, 3, 10])
def test_round_trip(lib, oracle, level):
    """every stream decodes to its source through decompress_files, and a legacy stream followed by a checksummed
    frame (what `cat a.lz4 b.lz4` gives) decodes as one file to both sources"""
    from lz4_b200 import batch
    big = M.CHUNK + 12345 if level < 3 else 300000
    datas = [oracle.datagen(n, 0.5, 70 + i).tobytes() for i, n in enumerate([0, 1, 4096, big])]
    res, out, doff, _ = run(datas, level)
    tail = oracle.datagen(200000, 0.5, 80).tobytes()
    fr_out, fr_res = batch.compress_frames_checksummed(t(np.frombuffer(tail, dtype=np.uint8)), t([0]), t([len(tail)]))
    frame = fr_out.cpu().numpy()[:int(fr_res[0])].tobytes()
    files = [out[o:o + r].tobytes() for o, r in zip(doff, res)]
    files.append(files[-1] + frame)
    want = datas + [datas[-1] + tail]
    pad = np.zeros(16, np.uint8)                                    # 16 readable bytes around every file
    comp = np.concatenate([pad] + [np.frombuffer(f, dtype=np.uint8) for f in files] + [pad])
    offs = 16 + np.concatenate([[0], np.cumsum([len(f) for f in files])[:-1]]).astype(np.int64)
    caps = np.array([len(w) for w in want], dtype=np.int64)
    legacy_blocks = sum(M.n_chunks(len(w)) for w in datas) + M.n_chunks(len(datas[-1]))
    dec, results, _, _ = batch.decompress_files(t(comp), t(offs), t([len(f) for f in files]), t(caps),
                                                max_units=len(files) + 1, max_blocks=[4, 0, 0, 0, legacy_blocks])
    torch.cuda.synchronize()
    assert list(results.cpu().numpy()) == list(caps)
    dec = dec.cpu().numpy()
    at = 0
    for w in want:
        assert dec[at:at + len(w)].tobytes() == w
        at += len(w)


# ------------------------------------------------------------------------------------------
# 4. launches, streams, graphs, far offsets, a file over 4 GiB
# ------------------------------------------------------------------------------------------
def test_launch_count(lib, oracle):
    datas = [oracle.datagen(n, 0.5, n).tobytes() for n in (100, 70000, 0)]
    for level, budget, want in ((1, None, 7), (9, None, 7), (12, None, 7), (1, 0, 5), (12, 0, 5)):
        before = lib.LZ4B200_launch_count()
        run(datas, level, budget=budget)
        assert lib.LZ4B200_launch_count() - before == want, (level, budget)


def test_side_stream_and_graph_replay(lib, oracle):
    from lz4_b200 import batch
    datas = [oracle.datagen(n, 0.5, 40 + i).tobytes() for i, n in enumerate([0, 999, 65536, 300000, M.CHUNK + 5])]
    arena, soff = place(datas, 21)
    sizes = np.array([len(d) for d in datas], dtype=np.int64)
    caps = np.array([M.bound(len(d)) for d in datas], dtype=np.int64)
    doff = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64) + 3
    budget = sum(M.n_chunks(len(d)) for d in datas)
    src, offs, sz, cp, do = t(arena), t(soff), t(sizes), t(caps), t(doff)
    ws = torch.empty(batch.compress_legacy_workspace_bytes(len(datas), budget, 1), dtype=torch.uint8, device=DEV)
    out = torch.full((int(caps.sum()) + 64,), GUARD, dtype=torch.uint8, device=DEV)
    res = torch.empty(len(datas), dtype=torch.int64, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.cuda.stream(side):
            batch.compress_legacy(src, offs, sz, max_blocks=budget, out=out, out_offsets=do, capacities=cp,
                                  results=res, workspace=ws, stream=side)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    side.synchronize()
    check_model(datas, 1, res.cpu().numpy(), out.cpu().numpy(), doff, oracle)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        batch.compress_legacy(src, offs, sz, max_blocks=budget, out=out, out_offsets=do, capacities=cp, results=res,
                              workspace=ws, stream=s)
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
        check_model(new, 1, res.cpu().numpy(), out.cpu().numpy(), doff, oracle)


def test_far_offsets(lib, oracle):
    """sources and streams at and across 2^31 and 2^32 in one arena; the guard bytes around every stream hold"""
    from lz4_b200 import batch
    datas = [oracle.datagen(n, 0.5, 60 + i).tobytes() for i, n in enumerate([70000, M.CHUNK + 3, 5000, 65536, 200001])]
    lines = [L31 - 1, L31 + 400000, L32 - 3, L32 + 9000017, L32 - 9000000]     # across 2^31 and 2^32, and past 2^32
    arena = torch.full((L32 + (32 << 20),), GUARD, dtype=torch.uint8, device=DEV)
    caps = [M.bound(len(d)) for d in datas]
    for role in ("src", "dst"):
        soff = list(lines) if role == "src" else [1000 + 9000000 * i for i in range(5)]
        doff = list(lines) if role == "dst" else [(1 << 30) + 9000000 * i for i in range(5)]
        for o, d in zip(soff, datas):
            arena[o:o + len(d)] = t(np.frombuffer(d, dtype=np.uint8))
        _, res = batch.compress_legacy(arena, t(np.array(soff)), t(np.array([len(d) for d in datas])), out=arena,
                                       out_offsets=t(np.array(doff)), capacities=t(np.array(caps)))
        torch.cuda.synchronize()
        res = res.cpu().numpy()
        for f, d in enumerate(datas):
            st = M.stream(d, M.block_codec(oracle, 1))
            assert res[f] == len(st), (role, f)
            win = arena[doff[f] - 64:doff[f] + len(st) + 64].cpu().numpy()
            assert win[64:64 + len(st)].tobytes() == st, (role, f)
            assert (win[:64] == GUARD).all() and (win[64 + len(st):] == GUARD).all(), (role, f)
        arena.fill_(GUARD)
    del arena
    torch.cuda.empty_cache()


def test_file_over_4_gib(lib, oracle):
    """one level-1 stream of 2^32 + 19 bytes against the model's digest: the source repeats a 64 MiB period, so the
    model compresses 8 distinct 8 MiB chunks and a 19-byte tail"""
    from lz4_b200 import batch
    period, n = 64 << 20, L32 + 19
    unit = oracle.datagen(period, 0.5, 7)
    src = t(unit).repeat(n // period + 1)[:n]
    h = hashlib.sha256(struct.pack("<I", M.MAGIC))
    comp = {}
    length = 4
    for at in range(0, n, M.CHUNK):
        key = (at % period, min(M.CHUNK, n - at))
        if key not in comp:
            blk = unit[key[0]:key[0] + key[1]].tobytes()
            r, c = oracle.compress(blk, 1, M.compress_bound(len(blk)))
            comp[key] = struct.pack("<I", r) + c[:r]
        h.update(comp[key])
        length += len(comp[key])
    cap = M.bound(n)
    out = torch.full((cap + 32,), GUARD, dtype=torch.uint8, device=DEV)
    _, res = batch.compress_legacy(src, torch.zeros(1, dtype=torch.int64, device=DEV),
                                   torch.tensor([n], dtype=torch.int64, device=DEV), max_blocks=M.n_chunks(n), out=out,
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
class LegacyRecorder(Recorder):
    SIZES = Recorder.SIZES + ("LZ4B200_compress_legacy_workspace_bytes", "LZ4B200_compressLegacyBound")


@pytest.fixture
def rec(monkeypatch):
    from lz4_b200 import _lib, batch
    r = LegacyRecorder(_lib.load())
    monkeypatch.setattr(_lib, "load", lambda: r)
    monkeypatch.setattr(batch, "_workspaces", {})
    return r


N = 4


def _z(n, dtype=torch.uint8, dev=DEV):
    return torch.zeros(n, dtype=dtype, device=dev)


def _good():
    return dict(src=_z(4096), offsets=_z(N, torch.int64), sizes=torch.full((N,), 100, dtype=torch.int64, device=DEV),
                max_blocks=N, out=_z(4096), out_offsets=_z(N, torch.int64),
                capacities=torch.full((N,), 200, dtype=torch.int64, device=DEV), results=_z(N, torch.int64))


def test_compress_legacy_wrapper(rec):
    from lz4_b200 import batch
    batch.compress_legacy(**_good())
    assert [c[0] for c in rec.calls] == ["LZ4B200_compress_legacy"]
    args = rec.calls[0][1]
    assert args[7:10] == (N, 1, N)
    rec.calls.clear()
    sizes = torch.tensor([0, M.CHUNK, M.CHUNK + 1, 5], dtype=torch.int64, device=DEV)
    out, _ = batch.compress_legacy(**dict(_good(), sizes=sizes, max_blocks=None, capacities=None, out=None,
                                          out_offsets=None, results=None), level=-3)
    args = rec.calls[0][1]
    assert args[7:10] == (N, -3, 4)                                  # 0 + 1 + 2 + 1 chunks
    assert out.numel() == sum(M.bound(n) for n in (0, M.CHUNK, M.CHUNK + 1, 5))
    bad = [("src", _z(16, torch.int8)), ("offsets", _z(N, torch.int32)), ("offsets", _z(N - 1, torch.int64)),
           ("sizes", _z(N, torch.int32)), ("capacities", _z(N - 1, torch.int64)), ("capacities", _z(N, torch.int32)),
           ("results", _z(N - 1, torch.int64)), ("out_offsets", _z(N, torch.int64, "cpu")), ("out", _z(64, dev="cpu")),
           ("max_blocks", -1), ("max_blocks", 2 ** 31), ("level", 2 ** 31), ("workspace", _z(8))]
    for arg, v in bad:
        kw = _good()
        kw[arg] = v
        rec.calls.clear()
        with pytest.raises(ValueError):
            batch.compress_legacy(**kw)
        assert not rec.calls, arg
    s = torch.cuda.Stream()
    ws = _z(1 << 20)
    for drop in ("max_blocks", "out", "capacities"):
        kw = _good()
        kw[drop] = None
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
            with pytest.raises(ValueError):
                batch.compress_legacy(stream=s, workspace=ws, **kw)
    assert not rec.calls
    torch.cuda.synchronize()
