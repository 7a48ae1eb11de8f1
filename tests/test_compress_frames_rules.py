"""LZ4B200_compress_frames on the CPU: the host model of its frames against the reference's (tests/golden/
compress_frames.json), the frame rules of lz4_frame_core.h built for the host against the fixture and the model, the index
passes against the model's verdicts on random batches, and the call's argument rules and workspace size, which are
decided on the host: no row launches anything."""
import ctypes as C
import json
import os
import struct

import numpy as np
import pytest

import compress_frames_model as M
import host_build
from conftest import GOLDEN

OK, ARG = 0, -1
_ll, _llp, _ip = C.c_longlong, C.POINTER(C.c_longlong), C.POINTER(C.c_int)


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLDEN, "compress_frames.json")) as f:
        return json.load(f)["frames"]


@pytest.fixture(scope="module")
def emul():
    lib = host_build.require()
    lib.cframes_header_host.restype = C.c_int
    lib.cframes_header_host.argtypes = [C.c_void_p, C.c_int, _ll]
    lib.cframes_bound_host.restype = _ll
    lib.cframes_bound_host.argtypes = [_ll, C.c_int]
    lib.cframes_optimal_bsid_host.restype = C.c_int
    lib.cframes_optimal_bsid_host.argtypes = [C.c_int, _ll]
    lib.cframes_index_host.restype = _ll
    lib.cframes_index_host.argtypes = [_llp, _llp, _llp, _ll, C.c_int, C.c_int, _llp] + [_llp] * 6 + [_ip, _llp, _ip]
    return lib


def _data(oracle, rec):
    return M.corpus_data(oracle, rec["kind"], rec["size"], rec["seed"])


def test_golden_corpus_is_the_model_corpus(golden):
    """the fixture holds every case the corpus defines, and the corpus covers the levels, sizes and flags it promises"""
    assert [g["id"] for g in golden] == [c[0] for c in M.corpus_cases()]
    assert {g["level"] for g in golden} == set(M.FAST_LEVELS + M.HC_LEVELS)
    assert {g["bsid"] for g in golden} == {0, 4, 5, 6, 7}
    assert {g["content_size"] for g in golden} == {False, True}
    assert {0, 1, 15, 16, 65535, 65536, 65537, 4 << 20, (4 << 20) + 1, 8 << 20} <= {g["size"] for g in golden}


def test_model_reproduces_every_golden_frame(oracle, golden):
    raw_blocks = one_byte_tails = 0
    for g in golden:
        data = _data(oracle, g)
        fr = M.frame(data, g["bsid"], g["content_size"], M.block_codec(oracle, g["level"]))
        assert (len(fr), M.sha(fr)) == (g["length"], g["sha256"]), g["id"]
        assert M.bound(g["size"], g["bsid"]) == g["bound"], g["id"]
        if "hex" in g:
            assert fr.hex() == g["hex"], g["id"]
        raw_blocks += sum(raw for raw, _ in M.blocks(fr))
        one_byte_tails += g["size"] % M.block_bytes(M.frame_bsid(g["bsid"], g["size"])) == 1
    assert raw_blocks > 0 and one_byte_tails > 0        # the corpus has stored-raw blocks and 1-byte last blocks


def test_frame_core_header_and_bound_match_the_fixture(emul, golden):
    buf = np.zeros(16, dtype=np.uint8)
    for g in golden:
        b = emul.cframes_optimal_bsid_host(g["bsid"] or 4, g["size"])
        assert b == M.frame_bsid(g["bsid"], g["size"]), g["id"]
        assert emul.cframes_bound_host(g["size"], b) == g["bound"], g["id"]
        hl = emul.cframes_header_host(buf.ctypes.data, b, g["size"] if g["content_size"] else 0)
        hdr = buf[:hl].tobytes()
        assert hdr == M.header(b, g["size"] if g["content_size"] else 0), g["id"]
        if "hex" in g:
            assert bytes.fromhex(g["hex"])[:hl] == hdr, g["id"]
    assert emul.cframes_bound_host(2 ** 63 - 8, 4) == 2 ** 63 - 1            # saturates


def _index(emul, sizes, caps, bsid, budget, src_off=None, cs=0):
    n = len(sizes)
    arr = lambda v: np.ascontiguousarray(v, dtype=np.int64)
    sizes, caps = arr(sizes), arr(caps)
    src_off = arr(src_off if src_off is not None else np.zeros(n))
    mb = arr(budget)
    outs = [np.zeros(max(n, 1), dtype=np.int64) for _ in range(5)]
    e = int(sum(budget))
    t_off, t_slot = np.zeros(max(e, 1), np.int64), np.zeros(max(e, 1), np.int64)
    t_size, t_cap = np.zeros(max(e, 1), np.int32), np.zeros(max(e, 1), np.int32)
    p = lambda a: a.ctypes.data_as(_llp)
    q = lambda a: a.ctypes.data_as(_ip)
    got = emul.cframes_index_host(p(src_off), p(sizes), p(caps), n, bsid or 4, cs, p(mb), *[p(o) for o in outs],
                                  p(t_off), q(t_size), p(t_slot), q(t_cap))
    assert got == e
    return [o[:n] for o in outs], (t_off[:e], t_size[:e], t_slot[:e], t_cap[:e])


def _check_batch(emul, sizes, caps, bsid, budget, rng):
    src_off = rng.integers(0, 1 << 40, len(sizes))
    (status, cls, count, base, hdr), (t_off, t_size, t_slot, t_cap) = _index(emul, sizes, caps, bsid, budget, src_off,
                                                                             cs=1)
    want = M.verdicts(sizes, caps, bsid, budget)
    tab_base = np.concatenate([[0], np.cumsum(budget)])[:4]
    stride = [((M.block_bytes(4 + c) - 1 + 15) // 16) * 16 for c in range(4)]
    slot_base = np.concatenate([[0], np.cumsum([budget[c] * stride[c] for c in range(4)])])[:4]
    used = np.zeros(len(t_size), dtype=bool)
    for f, (res, c, k, b) in enumerate(want):
        assert status[f] == (res if res is not None else OK), f
        if res in (M.ERR_ARG, M.ERR_DSTSIZE):
            assert cls[f] == -1
            continue
        assert (cls[f], count[f], base[f]) == (c, k, b), f
        assert hdr[f] == (15 if sizes[f] > 0 else 7)
        if res is not None:
            continue
        bs = M.block_bytes(4 + c)
        for j in range(k):
            e = tab_base[c] + b + j
            sz = min(bs, sizes[f] - j * bs)
            assert (t_off[e], t_size[e], t_slot[e], t_cap[e]) == (src_off[f] + j * bs, sz, slot_base[c] + (b + j) * stride[c],
                                                                  sz - 1), (f, j)
            used[e] = True
    assert (t_size[~used] == 0).all() and (t_cap[~used] == 0).all()       # unused entries compress nothing


def test_index_passes_match_the_model(emul):
    rng = np.random.default_rng(5)
    for trial in range(40):
        n = int(rng.integers(1, 300))
        bsid = int(rng.choice([0, 4, 5, 6, 7]))
        pick = rng.integers(0, 6, n)
        sizes = np.select([pick == 0, pick == 1, pick == 2, pick == 3, pick == 4],
                          [0, rng.integers(1, 70000, n), rng.integers(65537, 1 << 20, n), rng.integers(1 << 20, 9 << 20, n),
                           -rng.integers(1, 5, n)], rng.integers(0, 300000, n)).astype(np.int64)
        caps = np.array([M.bound(max(s, 0), bsid) for s in sizes], dtype=np.int64)
        caps -= (rng.random(n) < 0.15).astype(np.int64)                  # one byte short: LZ4B200_ERR_DSTSIZE
        caps[rng.random(n) < 0.03] = -1                                   # LZ4B200_ERR_ARG
        need = M.budget([s if c >= M.bound(max(s, 0), bsid) else -1 for s, c in zip(sizes, caps)], bsid)
        for budget in (need, [max(x - 1, 0) for x in need], [0, 0, 0, 0],
                       [int(rng.integers(0, x + 2)) for x in need]):
            _check_batch(emul, sizes, caps, bsid, budget, rng)


def test_index_budget_edges(emul):
    """exact fit, one short (the first over-budget frame and every later one of its class fail), budget 0 with empty
    frames (no blocks: they pass), and empty frames after an over-budget frame (they fail: the earlier blocks exceed)"""
    rng = np.random.default_rng(9)
    sizes = [70000, 0, 65536, 200000, 0, 1, 0]
    caps = [M.bound(s, 4) for s in sizes]
    for budget in ([M.budget(sizes, 4)[0], 0, 0, 0], [M.budget(sizes, 4)[0] - 1, 0, 0, 0], [0, 0, 0, 0], [2, 0, 0, 0]):
        _check_batch(emul, sizes, caps, 4, budget, rng)
    (status, *_), _ = _index(emul, [0, 0], [23, 22], 7, [0, 0, 0, 0])
    assert list(status) == [OK, M.ERR_DSTSIZE]                           # an empty frame needs 23 bytes of room
    (status, *_), _ = _index(emul, [65537, 0, 5], [M.bound(65537, 4), 23, M.bound(5, 4)], 4, [1, 0, 0, 0])
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


def _budget(v):
    return (C.c_int64 * 4)(*v) if v is not None else None


def _call(lib, n=3, bsid=4, level=0, cs=0, par=0, mb=(4, 0, 0, 0), ws=P, wb=None, **ptrs):
    a = dict(src=P, soff=P, ssz=P, dst=P, doff=P, cap=P, res=P)
    a.update(ptrs)
    b = _budget(mb)
    if wb is None:
        wb = int(lib.LZ4B200_compress_frames_workspace_bytes(max(n, 0), b, level)) if mb is not None else 0
    return lib.LZ4B200_compress_frames(a["src"], a["soff"], a["ssz"], a["dst"], a["doff"], a["cap"], a["res"], n, bsid,
                                       level, cs, par, b, ws, wb, None)


def _rows(lib):
    rows = [
        ("nFrames < 0", lambda: _call(lib, n=-1), ARG),
        ("nFrames == 0", lambda: _call(lib, n=0, src=None, dst=None, ws=None, wb=0), OK),
        ("nFrames == 0, level 12, parallel 0", lambda: _call(lib, n=0, level=12, ws=None, wb=0), OK),
        ("NULL maxBlocks", lambda: _call(lib, mb=None), ARG),
        ("NULL maxBlocks, no frames", lambda: _call(lib, n=0, mb=None), ARG),
        ("maxBlocks[0] < 0", lambda: _call(lib, mb=(-1, 0, 0, 0)), ARG),
        ("maxBlocks[3] = 2^31", lambda: _call(lib, mb=(0, 0, 0, 2 ** 31), wb=1 << 40), ARG),
        ("maxBlocks[2] = 2^31, no frames", lambda: _call(lib, n=0, mb=(0, 0, 2 ** 31, 0), wb=0), ARG),
        ("parallel at level 2", lambda: _call(lib, level=2, par=1), ARG),
        ("parallel at level 12", lambda: _call(lib, level=12, par=1), ARG),
        ("parallel at level 2, no frames", lambda: _call(lib, n=0, level=2, par=1), ARG),
        ("NULL d_src", lambda: _call(lib, src=None), ARG),
        ("NULL d_srcOff", lambda: _call(lib, soff=None), ARG),
        ("NULL d_srcSize", lambda: _call(lib, ssz=None), ARG),
        ("NULL d_dst", lambda: _call(lib, dst=None), ARG),
        ("NULL d_dstOff", lambda: _call(lib, doff=None), ARG),
        ("NULL d_dstCap", lambda: _call(lib, cap=None), ARG),
        ("NULL d_result", lambda: _call(lib, res=None), ARG),
        ("NULL d_workspace", lambda: _call(lib, ws=None), ARG),
    ]
    for bsid in (-1, 1, 2, 3, 8, 100):
        rows.append(("blockSizeID %d" % bsid, lambda bsid=bsid: _call(lib, bsid=bsid), ARG))
        rows.append(("blockSizeID %d, no frames" % bsid, lambda bsid=bsid: _call(lib, n=0, bsid=bsid), ARG))
    for level in (-70000, 0, 1, 2, 9, 10, 12, 13):
        rows.append(("level %d workspace one byte short" % level,
                     lambda level=level: _call(lib, level=level, mb=(3, 2, 1, 1),
                                               wb=int(lib.LZ4B200_compress_frames_workspace_bytes(
                                                   3, _budget((3, 2, 1, 1)), level)) - 1), ARG))
    return rows


def test_argument_rules_launch_nothing(lib):
    before = lib.LZ4B200_launch_count()
    for name, call, want in _rows(lib):
        assert call() == want, name
    assert lib.LZ4B200_launch_count() == before


def test_workspace_size(lib):
    ws = lambda n, mb, level: int(lib.LZ4B200_compress_frames_workspace_bytes(n, _budget(mb), level))
    assert ws(-1, (1, 0, 0, 0), 0) == 0
    assert ws(1, (-1, 0, 0, 0), 0) == 0
    assert ws(1, (0, 0, 0, 2 ** 31), 0) == 0
    assert int(lib.LZ4B200_compress_frames_workspace_bytes(1, None, 0)) == 0
    base = ws(0, (0, 0, 0, 0), 0)
    assert 0 < base <= 4096
    slots = [65536, 262144, 1 << 20, 4 << 20]                  # blockSize - 1 rounded up to 16
    for c in range(4):
        mb = [0, 0, 0, 0]
        mb[c] = 1000
        got = ws(0, mb, 0)
        assert 1000 * (slots[c] + 40) <= got - base <= 1000 * (slots[c] + 48) + 8 * 256, c   # slot + table entry
    hc, opt = int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(1111)), int(
        lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(1111))
    mb = (1000, 100, 10, 1)
    fast = ws(50, mb, 1)
    assert ws(50, mb, -5) == fast == ws(50, mb, 0)
    assert ws(50, mb, 2) == ws(50, mb, 9) and fast + hc <= ws(50, mb, 9) <= fast + hc + 256
    assert ws(50, mb, 10) == ws(50, mb, 13) and fast + opt <= ws(50, mb, 12) <= fast + opt + 256
    assert ws(10 ** 6, (0, 0, 0, 0), 0) - base >= 48 * 10 ** 6             # one record per frame
