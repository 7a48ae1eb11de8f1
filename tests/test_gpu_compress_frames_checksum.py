"""LZ4B200_compress_frames_checksummed and batch.compress_frames_checksummed on the GPU.

Every frame must be the reference's LZ4F_compressFrame output with the given checksum flags
(tests/golden/compress_frames_checksum.json), the `lz4` tool's file for the same input, or, for batches the fixture
does not hold, the host model's (tests/compress_frames_checksum_model.py).  Sources sit at shuffled
offsets of every 16-byte phase; outputs abut at odd offsets between guard bytes, so that a byte written outside
[dst_f, dst_f + result_f) shows.  The content hash is checked on both sides of the length at which a warp takes over
from one thread (256 KiB), at every source alignment, in the writer and in LZ4B200_decompress_frames_checksummed.
"""
import ctypes as C
import hashlib
import json
import os
import struct

import numpy as np
import pytest
import torch

import compress_frames_checksum_model as M
import host_build
from conftest import GOLDEN
from frame_checksum_model import xxh32
from gpu_util import Recorder

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
GUARD = 0xA5
STAGED_MIN = 256 << 10                                 # the content hash's warp path takes messages from here on


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
    """frees the workspaces batch keeps per stream after every test (a frames call's workspace holds a slot per block)"""
    yield
    from lz4_b200 import batch
    torch.cuda.synchronize()
    batch._workspaces.clear()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "compress_frames_checksum.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def xxh():
    """XXH32 of bytes: the host build of fc_xxh32 (fast), else the Python XXH32"""
    h = host_build.load()
    if h is None:
        return xxh32
    h.frames_xxh32_host.restype = C.c_uint
    h.frames_xxh32_host.argtypes = [C.c_void_p, C.c_ulonglong, C.c_uint]

    def f(b):
        a = np.frombuffer(bytes(b), dtype=np.uint8)
        return int(h.frames_xxh32_host(a.ctypes.data if len(a) else None, len(a), 0))
    return f


def t(a):
    return torch.from_numpy(np.array(a)).to(DEV)


def place(datas, seed, gap=64, phases=None):
    """an arena holding every source at a shuffled offset, 16 readable bytes around each; source i starts at 16-byte
    phase phases[i] (default: every phase in turn)"""
    rng = np.random.default_rng(seed)
    order = rng.permutation(len(datas))
    offs = [0] * len(datas)
    at = 16
    for k, i in enumerate(order):
        at = (at + 15) // 16 * 16 + (phases[i] if phases is not None else k % 16)
        offs[i] = at
        at += len(datas[i]) + gap
    arena = np.full(at + 16, 0x3C, dtype=np.uint8)
    for i, d in enumerate(datas):
        arena[offs[i]:offs[i] + len(d)] = np.frombuffer(bytes(d), dtype=np.uint8)
    return arena, np.array(offs, dtype=np.int64)


def run(datas, bsid, level, bsum, csum, cs=False, parallel=False, caps=None, budget=None, seed=0, phases=None):
    """one call over abutting outputs at an odd base between guards: (results, out bytes, out offsets, caps)"""
    from lz4_b200 import batch
    arena, soff = place(datas, seed, phases=phases)
    sizes = np.array([len(d) for d in datas], dtype=np.int64)
    if caps is None:
        caps = [M.bound(int(n), bsid, bsum, csum) for n in sizes]
    caps = np.array(caps, dtype=np.int64)
    room = np.maximum(caps, 0)
    doff = 7 + np.concatenate([[0], np.cumsum(room)[:-1]]).astype(np.int64)
    out = torch.full((int(room.sum()) + 7 + 64,), GUARD, dtype=torch.uint8, device=DEV)
    if budget is None:
        budget = M.budget([int(n) if c >= M.bound(int(n), bsid, bsum, csum) else -1 for n, c in zip(sizes, caps)], bsid)
    _, res = batch.compress_frames_checksummed(t(arena), t(soff), t(sizes), max_blocks=budget, block_size_id=bsid,
                                               level=level, content_size=cs, parallel=parallel, block_checksum=bsum,
                                               content_checksum=csum, out=out, out_offsets=t(doff), capacities=t(caps))
    torch.cuda.synchronize()
    return res.cpu().numpy(), out.cpu().numpy(), doff, caps


def check_written(out, doff, res):
    mask = np.ones(len(out), dtype=bool)
    for o, r in zip(doff, res):
        if r > 0:
            mask[o:o + r] = False
    bad = np.nonzero(out[mask] != GUARD)[0]
    assert len(bad) == 0, "wrote outside the frames (%d bytes)" % len(bad)


def check_model(datas, bsid, level, bsum, csum, res, out, doff, oracle, xxh, want=None, cs=False):
    codec = M.block_codec(oracle, level)
    for f, d in enumerate(datas):
        w = want[f] if want is not None else None
        if w is not None and w < 0:
            assert res[f] == w, (f, res[f], w)
            continue
        fr = M.frame(d, bsid, cs, codec, block_sum=bsum, content_sum=csum, xxh=xxh)
        assert res[f] == len(fr), (f, len(d), res[f], len(fr))
        assert out[doff[f]:doff[f] + len(fr)].tobytes() == fr, (f, len(d))
    check_written(out, doff, res)


# ------------------------------------------------------------------------------------------
# 1. the reference's frames and the `lz4` tool's files
# ------------------------------------------------------------------------------------------
def test_golden_frames(lib, oracle, fixture):
    """every golden frame byte for byte: one call per (level, block size ID, content size, flags), every size of the
    group in it, each output at the reference's exact bound"""
    groups = {}
    for g in fixture["frames"]:
        groups.setdefault((g["level"], g["bsid"], g["content_size"]), []).append(g)
    for (level, bsid, cs), gs in groups.items():
        datas = [M.corpus_data(oracle, g["kind"], g["size"], g["seed"]) for g in gs]
        for name, (bsum, csum) in M.SUM_FLAGS.items():
            res, out, doff, _ = run(datas, bsid, level, bsum, csum, cs, caps=[g["sums"][name]["bound"] for g in gs],
                                    seed=level & 0xFF)
            for g, r, o in zip(gs, res, doff):
                w = g["sums"][name]
                assert r == w["length"], (g["id"], name, r)
                assert hashlib.sha256(out[o:o + r].tobytes()).hexdigest() == w["sha256"], (g["id"], name)
            check_written(out, doff, res)


def test_cli_frames(lib, oracle, fixture):
    """the `lz4` tool's files for an input of more than 8 MB, byte for byte, through the wrapper's default capacities"""
    from lz4_b200 import batch
    data = M.cli_data(oracle)
    src = t(np.frombuffer(data, dtype=np.uint8))
    for c in fixture["cli"]:
        out, res = batch.compress_frames_checksummed(src, t([0]), t([len(data)]), block_size_id=c["bsid"],
                                                     level=c["level"], block_checksum=c["block_sum"],
                                                     content_checksum=c["content_sum"])
        r = int(res[0])
        assert r == c["length"], c["args"]
        assert hashlib.sha256(out[:r].cpu().numpy().tobytes()).hexdigest() == c["sha256"], c["args"]


# ------------------------------------------------------------------------------------------
# 2. both flags off; launches; capacities; budgets
# ------------------------------------------------------------------------------------------
def _mixed(oracle, seed):
    rng = np.random.default_rng(seed)
    sizes = [0, 1, 15, 16, 17, 65535, 65536, 65537, 300001, 1 << 20, (1 << 20) + 3, 5 << 20]
    sizes += [int(x) for x in rng.integers(0, 200000, 20)]
    return [oracle.datagen(n, 0.5, seed + i).tobytes() if i % 3 else
            np.random.default_rng(seed + i).integers(0, 256, n, dtype=np.uint8).tobytes() for i, n in enumerate(sizes)]


def _call_pair(lib, datas, bsid, level, parallel, flags):
    """(results, out, launches) of LZ4B200_compress_frames (flags None) or the checksummed call, on one layout"""
    from lz4_b200 import batch
    arena, soff = place(datas, 3)
    sizes = np.array([len(d) for d in datas], dtype=np.int64)
    caps = np.array([M.bound(int(n), bsid, True, True) for n in sizes], dtype=np.int64)
    doff = 5 + np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64)
    out = torch.full((int(caps.sum()) + 64,), GUARD, dtype=torch.uint8, device=DEV)
    budget = M.budget(sizes.tolist(), bsid)
    ws = torch.empty(batch.compress_frames_workspace_bytes(len(datas), budget, level), dtype=torch.uint8, device=DEV)
    args = (t(arena), t(soff), t(sizes))
    kw = dict(max_blocks=budget, block_size_id=bsid, level=level, parallel=parallel, out=out, out_offsets=t(doff),
              capacities=t(caps), workspace=ws)
    torch.cuda.synchronize()
    before = lib.LZ4B200_launch_count()
    if flags is None:
        _, res = batch.compress_frames(*args, **kw)
    else:
        _, res = batch.compress_frames_checksummed(*args, block_checksum=flags[0], content_checksum=flags[1], **kw)
    torch.cuda.synchronize()
    return res.cpu().numpy(), out.cpu().numpy(), lib.LZ4B200_launch_count() - before, doff


def test_no_flags_is_compress_frames(lib, oracle):
    """with both flags 0 the call gives LZ4B200_compress_frames's results, bytes and launch count"""
    datas = _mixed(oracle, 100)
    for bsid, level, par in ((4, 1, False), (7, 0, False), (5, -5, True), (0, 1, True), (4, 9, False)):
        base = _call_pair(lib, datas, bsid, level, par, None)
        got = _call_pair(lib, datas, bsid, level, par, (False, False))
        assert np.array_equal(got[0], base[0]), (bsid, level, par)
        assert np.array_equal(got[1], base[1]), (bsid, level, par)
        assert got[2] == base[2] == (8 if par else 7), (bsid, level, par)


def test_launch_counts(lib, oracle):
    """LZ4B200_compress_frames's launches, plus one per flag that is set (5 with every budget 0)"""
    datas = _mixed(oracle, 200)[:8]
    for par in (False, True):
        for b, c in ((True, False), (False, True), (True, True)):
            *_, n, _ = _call_pair(lib, datas, 4, 0, par, (b, c))
            assert n == 7 + par + b + c, (par, b, c)
    from lz4_b200 import batch
    out = torch.zeros(64, dtype=torch.uint8, device=DEV)
    for b, c in ((False, False), (True, False), (False, True), (True, True)):
        before = lib.LZ4B200_launch_count()
        _, res = batch.compress_frames_checksummed(out, t([0]), t([10]), max_blocks=[0, 0, 0, 0], block_checksum=b,
                                                   content_checksum=c, out=out, capacities=t([64]))
        torch.cuda.synchronize()
        assert lib.LZ4B200_launch_count() - before == 5 + b + c and int(res[0]) == M.ERR_LIMIT


def test_capacity_at_the_bound_and_one_below(lib, oracle, xxh):
    """each frame at its checksummed bound, and every other one a byte below it (LZ4B200_ERR_DSTSIZE, nothing
    written), outputs abutting between guard bytes"""
    datas = _mixed(oracle, 300)
    for bsid in (4, 6):
        for b, c in ((True, False), (False, True), (True, True)):
            exact = [M.bound(len(d), bsid, b, c) for d in datas]
            caps = [e - (i % 2) for i, e in enumerate(exact)]
            want = [None if i % 2 == 0 else M.ERR_DSTSIZE for i in range(len(datas))]
            res, out, doff, _ = run(datas, bsid, 1, b, c, caps=caps, seed=bsid)
            check_model(datas, bsid, 1, b, c, res, out, doff, oracle, xxh, want)


def test_budget_overruns(lib, oracle, xxh):
    """a mixed batch past its budget: the frames the rule fails get LZ4B200_ERR_LIMIT and no bytes; the others are
    written with their checksums"""
    datas = _mixed(oracle, 400)
    sizes = [len(d) for d in datas]
    need = M.budget(sizes, 5)
    budget = [max(need[0] - 7, 0), max(need[1] - 1, 0), 0, 0]
    caps = [M.bound(n, 5, True, True) for n in sizes]
    want = [v[0] for v in M.verdicts(sizes, caps, 5, budget, True, True)]
    assert M.ERR_LIMIT in want and None in want
    res, out, doff, _ = run(datas, 5, 0, True, True, caps=caps, budget=budget, seed=9)
    check_model(datas, 5, 0, True, True, res, out, doff, oracle, xxh, want)


# ------------------------------------------------------------------------------------------
# 3. the round trip; the content hash's two paths
# ------------------------------------------------------------------------------------------
def _decode_verify(out, doff, res, datas, bsid):
    from lz4_b200 import batch
    n = len(datas)
    src = t(out)
    lens = np.array([len(d) for d in datas], dtype=np.int64)
    budget = M.budget(lens.tolist(), bsid)
    dec, r, cons = batch.decompress_frames_checksummed(src, t(doff), t(res), t(lens), budget)
    torch.cuda.synchronize()
    assert np.array_equal(r.cpu().numpy(), lens) and np.array_equal(cons.cpu().numpy(), res)
    dec = dec.cpu().numpy()
    at = np.concatenate([[0], np.cumsum(lens)[:-1]])
    for f in range(n):
        assert dec[at[f]:at[f] + lens[f]].tobytes() == bytes(datas[f]), f


def test_round_trip_verifies(lib, oracle):
    """frames of every level route and of the parallel parse, both checksums on, decode and verify"""
    datas = _mixed(oracle, 500)
    for bsid, level, par in ((4, -5, False), (7, 1, False), (5, 0, True), (4, 2, False), (4, 10, False)):
        ds = datas if level < 2 else [d[:150000] for d in datas]
        res, out, doff, _ = run(ds, bsid, level, True, True, parallel=par, seed=level & 7)
        assert (res > 0).all(), (bsid, level, par)
        _decode_verify(out, doff, res, ds, bsid)


def test_content_hash_on_both_sides_of_the_warp_path(lib, oracle, xxh):
    """content lengths below, at and above the length from which a warp hashes a frame, at all 16 source phases, in
    one call; the frames' content checksums against XXH32, then verified by the decoder, whose outputs sit at other
    phases"""
    lens = [STAGED_MIN + d for d in (-17, -16, -1, 0, 1, 15, 16, 1 << 16)] + [17, 4096, 65537, (1 << 20) + 3]
    datas, phases = [], []
    for i, n in enumerate(lens):
        for ph in range(16):
            datas.append(oracle.datagen(n, 0.5, 7000 + 16 * i + ph).tobytes() if ph % 4 else
                         np.random.default_rng(ph + i).integers(0, 256, n, dtype=np.uint8).tobytes())
            phases.append(ph)
    res, out, doff, _ = run(datas, 7, 1, False, True, phases=phases, seed=11)
    for f, d in enumerate(datas):
        assert res[f] > 0
        assert struct.unpack_from("<I", out, doff[f] + res[f] - 4)[0] == xxh(d), (f, len(d), phases[f])
    check_model(datas, 7, 1, False, True, res, out, doff, oracle, xxh)
    _decode_verify(out, doff, res, datas, 7)


def test_content_over_4_gib(lib):
    """one frame whose content is 2^32 + 3 x 65 536 + 19 bytes (the far content of tests/test_frames_scale_rules.py,
    built on the device) written with a content checksum: the reference's XXH32 of it (tests/golden/frames_scale.json)"""
    from lz4_b200 import batch
    with open(os.path.join(GOLDEN, "frames_scale.json")) as f:
        g = json.load(f)
    n, bs = g["content_size"], 65536
    full = n // bs
    src = torch.empty(n, dtype=torch.uint8, device=DEV)
    step = 4096
    for a in range(0, full + 1, step):
        k = min(step, full + 1 - a)
        idx = torch.arange(a, a + k, dtype=torch.int64, device=DEV)
        rows = torch.empty((k, bs), dtype=torch.uint8, device=DEV)
        rows[:, 8:] = ((idx * 37 + 11) & 0xFF).to(torch.uint8)[:, None]
        rows[:, :8] = idx.view(torch.uint8).view(k, 8)
        end = min((a + k) * bs, n)
        src[a * bs:end] = rows.view(-1)[:end - a * bs]
        del rows
    blocks = (n + bs - 1) // bs
    cap = M.bound(n, 4, False, True)
    out = torch.full((cap + 32,), GUARD, dtype=torch.uint8, device=DEV)
    _, res = batch.compress_frames_checksummed(src, t([0]), t([n]), max_blocks=[blocks, 0, 0, 0], block_size_id=4,
                                               content_size=True, out=out, out_offsets=t([16]), capacities=t([cap]))
    torch.cuda.synchronize()
    r = int(res[0])
    assert 0 < r < cap
    tail = out[16 + r - 8:16 + r].cpu().numpy().tobytes()
    assert tail == struct.pack("<II", 0, g["xxh32"])
    assert bool((out[:16] == GUARD).all()) and bool((out[16 + r:] == GUARD).all())
    del src, out
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------
# 4. streams, capture, the wrapper
# ------------------------------------------------------------------------------------------
def test_side_stream_and_graph_replay(lib, oracle, xxh):
    from lz4_b200 import batch
    datas = [oracle.datagen(n, 0.5, 800 + i).tobytes() for i, n in enumerate([0, 5, 70000, 1 << 20, (1 << 20) + 9,
                                                                              3 << 20])]
    arena, soff = place(datas, 12)
    sizes = [len(d) for d in datas]
    caps = np.array([M.bound(n, 7, True, True) for n in sizes], dtype=np.int64)
    doff = 3 + np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64)
    budget = M.budget(sizes, 7)
    src, offs, sz, do, cp = t(arena), t(soff), t(sizes), t(doff), t(caps)
    out = torch.full((int(caps.sum()) + 64,), GUARD, dtype=torch.uint8, device=DEV)
    res = torch.empty(len(datas), dtype=torch.int64, device=DEV)
    ws = torch.empty(batch.compress_frames_workspace_bytes(len(datas), budget, 0), dtype=torch.uint8, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.cuda.stream(side):
            batch.compress_frames_checksummed(src, offs, sz, max_blocks=budget, block_size_id=7, block_checksum=True,
                                              out=out, out_offsets=do, capacities=cp, results=res, workspace=ws,
                                              stream=side)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    side.synchronize()
    check_model(datas, 7, 0, True, True, res.cpu().numpy(), out.cpu().numpy(), doff, oracle, xxh)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        batch.compress_frames_checksummed(src, offs, sz, max_blocks=budget, block_size_id=7, block_checksum=True,
                                          out=out, out_offsets=do, capacities=cp, results=res, workspace=ws, stream=s)
    for seed in (1, 2):
        new = [oracle.datagen(len(d), 0.3 * seed, 900 + seed * 10 + i).tobytes() for i, d in enumerate(datas)]
        host = arena.copy()
        for i, d in enumerate(new):
            host[soff[i]:soff[i] + len(d)] = np.frombuffer(d, dtype=np.uint8)
        src.copy_(t(host))
        out.fill_(GUARD)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        check_model(new, 7, 0, True, True, res.cpu().numpy(), out.cpu().numpy(), doff, oracle, xxh)


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


def test_compress_frames_checksummed_wrapper(rec, lib):
    from lz4_b200 import batch
    batch.compress_frames_checksummed(**_good())
    assert [c[0] for c in rec.calls] == ["LZ4B200_compress_frames_checksummed"]
    args = rec.calls[0][1]
    assert args[7] == N and args[8:14] == (4, 0, 0, 0, 0, 1) and list(args[14]) == [N, 0, 0, 0]   # the tool's default
    rec.calls.clear()
    batch.compress_frames_checksummed(**dict(_good(), max_blocks=None, capacities=None, out=None, out_offsets=None,
                                             results=None), block_size_id=5, level=9, content_size=True,
                                      block_checksum=True, content_checksum=False)
    args = rec.calls[0][1]
    assert args[8:14] == (5, 9, 1, 0, 1, 0) and list(args[14]) == [N, 0, 0, 0]
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
            batch.compress_frames_checksummed(**kw)
        assert not rec.calls, arg
    with pytest.raises(ValueError):
        batch.compress_frames_checksummed(**_good(), parallel=True, level=2)
    s = torch.cuda.Stream()
    ws = _z(1 << 20)
    for drop in ("max_blocks", "out", "capacities"):
        kw = _good()
        kw[drop] = None
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
            with pytest.raises(ValueError):
                batch.compress_frames_checksummed(stream=s, workspace=ws, **kw)
    assert not rec.calls
    torch.cuda.synchronize()
