"""LZ4B200_compress_legacy on the CPU: the host model of its streams against the reference tool's (tests/golden/
compress_legacy.json), the legacy rules of lz4_frame_core.h built for the host against the model at every budget edge,
and the call's argument rules and workspace size, which are decided on the host: no row launches anything."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import compress_legacy_model as M
import host_build
from conftest import GOLDEN

OK, ARG = 0, -1
_ll, _llp, _ip = C.c_longlong, C.POINTER(C.c_longlong), C.POINTER(C.c_int)
STRIDE = (M.compress_bound(M.CHUNK) + 15) // 16 * 16


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLDEN, "compress_legacy.json")) as f:
        return json.load(f)["streams"]


@pytest.fixture(scope="module")
def emul():
    lib = host_build.require()
    lib.clegacy_bound_host.restype = _ll
    lib.clegacy_bound_host.argtypes = [_ll]
    lib.clegacy_index_host.restype = None
    lib.clegacy_index_host.argtypes = [_llp, _llp, _llp, _ll, _ll] + [_llp] * 5 + [_llp, _ip, _llp, _ip]
    return lib


def test_golden_corpus_is_the_model_corpus(golden):
    """the fixture holds every case the corpus defines, and the corpus covers the levels, sizes and data it promises"""
    assert [g["id"] for g in golden] == [c[0] for c in M.corpus_cases()]
    assert {g["level"] for g in golden} == set(M.FAST_LEVELS + M.HC_LEVELS)
    assert set(M.FAST_SIZES + [20 * M.MIB]) <= {g["size"] for g in golden}
    assert {g["kind"] for g in golden} == set(M.KINDS + ["split"])
    assert all(g["size"] <= M.MIB for g in golden if g["level"] >= 3 and g["kind"] != "split")


def test_model_reproduces_every_golden_stream(oracle, golden):
    grown = 0
    for g in golden:
        data = M.corpus_data(oracle, g["kind"], g["size"], g["seed"])
        st = M.stream(data, M.block_codec(oracle, g["level"]))
        assert (len(st), M.sha(st)) == (g["length"], g["sha256"]), g["id"]
        assert M.bound(g["size"]) == g["bound"] and len(st) <= g["bound"], g["id"]
        assert len(M.chunks(st)) == M.n_chunks(g["size"]), g["id"]
        grown += any(k > M.CHUNK for k in M.chunks(st))
    assert grown > 0                # incompressible chunks are written compressed, larger than they are


def test_bound_matches_the_model(emul, golden):
    sizes = {g["size"] for g in golden} | {2, 254, 255, 256, M.CHUNK - 255, 3 * M.CHUNK, 5 * M.CHUNK + 7, 1 << 40}
    for n in sorted(sizes):
        assert emul.clegacy_bound_host(n) == M.bound(n), n
    assert emul.clegacy_bound_host(2 ** 63 - 8) == 2 ** 63 - 1           # saturates


def _index(emul, sizes, caps, budget, src_off):
    n = len(sizes)
    arr = lambda v: np.ascontiguousarray(v, dtype=np.int64)
    sizes, caps, src_off = arr(sizes), arr(caps), arr(src_off)
    outs = [np.zeros(max(n, 1), dtype=np.int64) for _ in range(5)]
    t_off, t_slot = np.zeros(max(budget, 1), np.int64), np.zeros(max(budget, 1), np.int64)
    t_size, t_cap = np.zeros(max(budget, 1), np.int32), np.zeros(max(budget, 1), np.int32)
    p = lambda a: a.ctypes.data_as(_llp)
    q = lambda a: a.ctypes.data_as(_ip)
    emul.clegacy_index_host(p(src_off), p(sizes), p(caps), n, budget, *[p(o) for o in outs], p(t_off), q(t_size),
                            p(t_slot), q(t_cap))
    return [o[:n] for o in outs], (t_off[:budget], t_size[:budget], t_slot[:budget], t_cap[:budget])


def _check_batch(emul, sizes, caps, budget, rng):
    src_off = rng.integers(0, 1 << 40, len(sizes))
    (status, cls, count, base, hdr), (t_off, t_size, t_slot, t_cap) = _index(emul, sizes, caps, budget, src_off)
    used = np.zeros(len(t_size), dtype=bool)
    for f, (res, k, b) in enumerate(M.verdicts(sizes, caps, budget)):
        assert status[f] == (res if res is not None else OK), f
        if res in (M.ERR_ARG, M.ERR_DSTSIZE):
            assert cls[f] == -1
            continue
        assert (cls[f], count[f], base[f], hdr[f]) == (4, k, b, 4), f
        if res is not None:
            continue
        for j in range(k):
            sz = min(M.CHUNK, sizes[f] - j * M.CHUNK)
            assert (t_off[b + j], t_size[b + j], t_slot[b + j], t_cap[b + j]) == (
                src_off[f] + j * M.CHUNK, sz, (b + j) * STRIDE, M.compress_bound(sz)), (f, j)
            used[b + j] = True
    assert (t_size[~used] == 0).all() and (t_cap[~used] == 0).all()       # unused entries compress nothing


def test_index_passes_match_the_model(emul):
    rng = np.random.default_rng(11)
    for trial in range(40):
        n = int(rng.integers(1, 200))
        pick = rng.integers(0, 5, n)
        sizes = np.select([pick == 0, pick == 1, pick == 2, pick == 3],
                          [0, rng.integers(1, M.CHUNK + 2, n), rng.integers(M.CHUNK, 5 * M.CHUNK, n),
                           -rng.integers(1, 5, n)], rng.integers(0, 300000, n)).astype(np.int64)
        caps = np.array([M.bound(max(s, 0)) for s in sizes], dtype=np.int64)
        caps -= (rng.random(n) < 0.15).astype(np.int64)                  # one byte short: LZ4B200_ERR_DSTSIZE
        caps[rng.random(n) < 0.03] = -1                                   # LZ4B200_ERR_ARG
        need = sum(M.n_chunks(s) for s, c in zip(sizes, caps) if s >= 0 and c >= M.bound(s))
        for budget in (need, max(need - 1, 0), 0, int(rng.integers(0, need + 2))):
            _check_batch(emul, sizes, caps, budget, rng)


def test_index_budget_edges(emul):
    """exact fit, one short (the first over-budget file and every later one fail), budget 0 with empty files (no
    chunks: they pass), and empty files after an over-budget file (they fail: the earlier chunks exceed)"""
    rng = np.random.default_rng(13)
    sizes = [M.CHUNK + 1, 0, M.CHUNK, 3 * M.CHUNK, 0, 1, 0]
    caps = [M.bound(s) for s in sizes]
    need = sum(M.n_chunks(s) for s in sizes)
    for budget in (need, need - 1, 0, 2, 3):
        _check_batch(emul, sizes, caps, budget, rng)
    (status, *_), _ = _index(emul, [0, 0], [4, 3], 0, [0, 0])
    assert list(status) == [OK, M.ERR_DSTSIZE]                           # an empty file needs its 4-byte magic
    (status, *_), _ = _index(emul, [M.CHUNK + 1, 0, 5], [M.bound(M.CHUNK + 1), 4, M.bound(5)], 1, [0, 0, 0])
    assert list(status) == [M.ERR_LIMIT, M.ERR_LIMIT, M.ERR_LIMIT]


# ------------------------------------------------------------------------------------------
# the call's argument rules and workspace size, decided on the host
# ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import build, _lib
    build.build()
    return _lib.load()


_keep = np.zeros(1 << 16, dtype=np.uint8)
P = _keep.ctypes.data


def _call(lib, n=3, level=1, mb=4, ws=P, wb=None, **ptrs):
    a = dict(src=P, soff=P, ssz=P, dst=P, doff=P, cap=P, res=P)
    a.update(ptrs)
    if wb is None:
        wb = int(lib.LZ4B200_compress_legacy_workspace_bytes(max(n, 0), mb, level))
    return lib.LZ4B200_compress_legacy(a["src"], a["soff"], a["ssz"], a["dst"], a["doff"], a["cap"], a["res"], n,
                                       level, mb, ws, wb, None)


def test_argument_rules_launch_nothing(lib):
    rows = [
        ("nFiles < 0", lambda: _call(lib, n=-1), ARG),
        ("nFiles == 0", lambda: _call(lib, n=0, src=None, dst=None, ws=None, wb=0), OK),
        ("nFiles == 0, level 12", lambda: _call(lib, n=0, level=12, ws=None, wb=0), OK),
        ("maxBlocks < 0", lambda: _call(lib, mb=-1, wb=1 << 20), ARG),
        ("maxBlocks = 2^31", lambda: _call(lib, mb=2 ** 31, wb=1 << 62), ARG),
        ("maxBlocks = 2^31, no files", lambda: _call(lib, n=0, mb=2 ** 31, wb=0), ARG),
        ("NULL d_src", lambda: _call(lib, src=None), ARG),
        ("NULL d_srcOff", lambda: _call(lib, soff=None), ARG),
        ("NULL d_srcSize", lambda: _call(lib, ssz=None), ARG),
        ("NULL d_dst", lambda: _call(lib, dst=None), ARG),
        ("NULL d_dstOff", lambda: _call(lib, doff=None), ARG),
        ("NULL d_dstCap", lambda: _call(lib, cap=None), ARG),
        ("NULL d_result", lambda: _call(lib, res=None), ARG),
        ("NULL d_workspace", lambda: _call(lib, ws=None), ARG),
    ]
    for level in (-70000, -1, 0, 2, 3, 9, 10, 12, 13):
        rows.append(("level %d workspace one byte short" % level,
                     lambda level=level: _call(lib, level=level, mb=3, wb=int(
                         lib.LZ4B200_compress_legacy_workspace_bytes(3, 3, level)) - 1), ARG))
    before = lib.LZ4B200_launch_count()
    for name, call, want in rows:
        assert call() == want, name
    assert lib.LZ4B200_launch_count() == before


def test_workspace_size(lib):
    ws = lambda n, mb, level: int(lib.LZ4B200_compress_legacy_workspace_bytes(n, mb, level))
    assert ws(-1, 1, 1) == ws(1, -1, 1) == ws(1, 2 ** 31, 1) == 0
    base = ws(0, 0, 1)
    assert 0 < base <= 4096
    got = ws(0, 100, 1)
    assert 100 * (STRIDE + 40) <= got - base <= 100 * (STRIDE + 48) + 8 * 256           # slot + table entry
    hc, opt = int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(100)), int(
        lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(100))
    fast = ws(50, 100, 1)
    assert ws(50, 100, -70000) == ws(50, 100, 0) == ws(50, 100, 2) == fast           # level 2 is the fast parse
    assert ws(50, 100, 3) == ws(50, 100, 9) and fast + hc <= ws(50, 100, 3) <= fast + hc + 256
    assert ws(50, 100, 10) == ws(50, 100, 13) and fast + opt <= ws(50, 100, 12) <= fast + opt + 256
    assert ws(10 ** 6, 0, 1) - base >= 48 * 10 ** 6                                    # one record per file


def test_frames_workspace_is_unchanged(lib):
    """the frame-encode plan gained the legacy class; the frames calls give it no budget, so their workspace is the
    parent's formula: records, 48 bytes per budgeted block, a slot of blockSize - 1 rounded up to 16, the HC workspace"""
    up = lambda x: (x + 255) // 256 * 256
    rng = np.random.default_rng(3)
    for trial in range(60):
        n = int(rng.integers(0, 5000))
        mb = [int(x) for x in rng.integers(0, 3000, 4) * (rng.random(4) < 0.7)]
        level = int(rng.choice([-9, 0, 1, 2, 9, 10, 12]))
        e = sum(mb)
        at = up(n * 48)
        for width in (8, 4, 8, 4, 4):
            at = up(at + e * width)
        at = up(at + (e + 1) * 8)
        at = up(at + e * 8)
        at = up(at + sum(m * (((1 << (8 + 2 * (4 + c))) - 1 + 15) // 16 * 16) for c, m in enumerate(mb)))
        hcb = 0 if level < 2 else int((lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes if level >= 10
                                       else lib.LZ4B200_compress_blocks_hc_workspace_bytes)(e))
        want = up(at + hcb) + 256
        got = int(lib.LZ4B200_compress_frames_workspace_bytes(n, (C.c_int64 * 4)(*mb), level))
        assert got == want, (n, mb, level)


def test_legacy_bound_entry(lib):
    for n in [0, 1, 13, 4096, M.CHUNK - 1, M.CHUNK, M.CHUNK + 1, 20 * M.MIB, 1 << 33]:
        assert int(lib.LZ4B200_compressLegacyBound(n)) == M.bound(n), n
    assert int(lib.LZ4B200_compressLegacyBound(-1)) == ARG
