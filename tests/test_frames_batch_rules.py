"""LZ4B200_decompress_frames without a GPU: its argument rules and workspace size, and its index passes -- pass 1, the
per-class scan with the budget rule, pass 2 -- built on the host from lz4_b200/csrc/lz4_frame_core.h
(tests/emul/frame_emul.cpp), against a Python walk of the chain and LZ4B200_decompressFrame_host's verdicts."""
import ctypes as C

import numpy as np
import pytest

import frame_corpus as fc
import host_build


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import build, _lib
    build.build()
    return _lib.load()


_ll, _llp = C.c_longlong, C.POINTER(C.c_longlong)
_ip = C.POINTER(C.c_int)


def frames_emul():
    """host_build's library (every tests/emul/*.cpp, frame_emul.cpp included) with frames_index_host's prototype"""
    fn = host_build.require().frames_index_host
    fn.restype = _ll
    fn.argtypes = [C.c_void_p, _llp, _llp, _llp, _ll, _llp, _llp, _llp, _llp, _llp, _llp, _llp, _ip, _ip]
    return fn


def budget(*mb):
    return (C.c_int64 * 4)(*mb)


def test_workspace_size_function(lib):
    ws = lib.LZ4B200_decompress_frames_workspace_bytes
    assert ws(-1, budget(1, 0, 0, 0)) == 0
    assert ws(4, None) == 0
    assert ws(4, budget(0, -1, 0, 0)) == 0
    assert ws(4, budget(0, 0, 0, 1 << 31)) == 0
    assert ws(4, budget(0, 0, 0, (1 << 31) - 1)) > 0
    base = ws(0, budget(0, 0, 0, 0))
    assert 0 < base <= 4096
    assert ws(1000, budget(0, 0, 0, 0)) >= base + 48 * 1000
    for c in range(4):
        mb = [0, 0, 0, 0]
        mb[c] = 37
        dec = lib.LZ4B200_decompress_workspace_bytes_for(37, 0, 1 << (16 + 2 * c))
        grow = ws(10, budget(*mb)) - ws(10, budget(0, 0, 0, 0))
        assert dec + 37 * 28 <= grow <= dec + 37 * 28 + 6 * 256, c     # the class's decode workspace and table
    assert ws(10, budget(1, 2, 3, 4)) >= ws(10, budget(1, 2, 3, 3))


def test_argument_rules(lib):
    ws = lib.LZ4B200_decompress_frames_workspace_bytes
    f = lib.LZ4B200_decompress_frames
    p = 4096                                        # non-NULL stand-ins: every call below is refused before a launch
    mb = budget(2, 1, 0, 0)
    need = ws(3, mb)
    args = [p, p, p, p, p, p, p, p, 3, mb, p, need, None]
    assert f(*args[:8], -1, *args[9:]) == fc.ERR_ARG
    assert f(*args[:9], None, *args[10:]) == fc.ERR_ARG
    assert f(*args[:9], budget(2, -1, 0, 0), *args[10:]) == fc.ERR_ARG
    assert f(*args[:9], budget(2, 1 << 31, 0, 0), *args[10:]) == fc.ERR_ARG
    for i in (0, 1, 2, 3, 4, 5, 6, 10):            # every pointer but d_consumed (7)
        bad = list(args)
        bad[i] = None
        assert f(*bad) == fc.ERR_ARG, i
    bad = list(args)
    bad[11] = need - 1
    assert f(*bad) == fc.ERR_ARG
    bad[7] = None
    assert f(*bad) == fc.ERR_ARG
    assert f(None, None, None, None, None, None, None, None, 0, mb, None, 0, None) == fc.OK   # no frames: no launch
    assert lib.LZ4B200_launch_count() == 0 or lib.LZ4B200_device_count() > 0


def index_host(frames, caps, mb, sizes=None, seed=0):
    """run the index passes of the host build on frames; returns per-frame arrays and the table"""
    index = frames_emul()
    buf, offs = fc.layout(frames, seed=seed)
    n = len(frames)
    src = np.frombuffer(buf, dtype=np.uint8)
    off = np.array(offs, dtype=np.int64)
    size = np.array(sizes if sizes is not None else [len(x) for x in frames], dtype=np.int64)
    cap = np.array(caps, dtype=np.int64)
    mba = np.array(mb, dtype=np.int64)
    outs = [np.zeros(max(n, 1), dtype=np.int64) for _ in range(5)]
    ent = int(sum(mb))
    tso, tsz, trl = np.zeros(max(ent, 1), np.int64), np.zeros(max(ent, 1), np.int32), np.zeros(max(ent, 1), np.int32)
    P = lambda a, t: a.ctypes.data_as(C.POINTER(t))                                    # noqa: E731
    got = index(src.ctypes.data, P(off, C.c_longlong), P(size, C.c_longlong), P(cap, C.c_longlong), n,
                P(mba, C.c_longlong), *[P(o, C.c_longlong) for o in outs], P(tso, C.c_longlong),
                P(tsz, C.c_int), P(trl, C.c_int))
    assert got == ent
    status, cls, count, base, consumed = (o[:n].tolist() for o in outs)
    return dict(src=buf, off=offs, status=status, cls=cls, count=count, base=base, consumed=consumed,
                tab=list(zip(tso[:ent].tolist(), tsz[:ent].tolist(), trl[:ent].tolist())))


def host_verdict(lib, frame, cap):
    src = np.frombuffer(frame + b"\0" * 16, dtype=np.uint8)
    dst = np.zeros(max(cap, 1), dtype=np.uint8)
    used = C.c_int64(0)
    r = int(lib.LZ4B200_decompressFrame_host(src.ctypes.data, len(frame), dst.ctypes.data, cap, C.byref(used)))
    return r, used.value


def corpus(oracle):
    good = [f for f, _ in fc.good_frames(oracle, big=False)]
    frames = list(good)
    for g in (good[4], good[9], good[-1]):
        frames += [m for _, m in fc.mutations(g)]
    return frames


def check_tables(r, frames, mb):
    """every frame that passed: its entries equal the Python walk; every other entry is cleared"""
    tab_base = [sum(mb[:c]) for c in range(4)]
    used = set()
    for f, fr in enumerate(frames):
        if r["status"][f] != fc.OK:
            continue
        blocks, consumed = fc.walk(fr)
        assert r["count"][f] == len(blocks) and r["consumed"][f] == consumed, f
        for k, (o, sz, raw) in enumerate(blocks):
            e = tab_base[r["cls"][f]] + r["base"][f] + k
            used.add(e)
            assert r["tab"][e] == (r["off"][f] + o, 0 if raw else sz, sz if raw else -1), (f, k)
    for e, t in enumerate(r["tab"]):
        if e not in used:
            assert t[1:] == (0, -1), e


def need_of(r):
    need = [0, 0, 0, 0]
    for st, c, n in zip(r["status"], r["cls"], r["count"]):
        if st == fc.OK:
            need[c] += n
    return need


def test_index_passes_match_the_chain_walk_and_the_host_verdicts(lib, oracle):
    frames = corpus(oracle)
    rng = np.random.default_rng(3)
    caps = [int(rng.choice([0, 1, 1 << 20, 1 << 24])) for _ in frames]
    big = [1 << 16] * 4
    r = index_host(frames, caps, big)
    assert fc.ERR_LIMIT not in r["status"]
    check_tables(r, frames, big)
    seen = set()
    for f, fr in enumerate(frames):
        want, used = host_verdict(lib, fr, caps[f])
        st = r["status"][f]
        seen.add(st)
        if st != fc.OK:                             # decided by the header or the chain: the host call's result, no decode
            assert st == want and r["consumed"][f] == 0, (f, st, want)
        else:                                       # the chain is valid: the host call walked it to the same length
            assert used == r["consumed"][f] == fc.walk(fr)[1], f
            assert want not in (fc.ERR_UNSUPPORTED, fc.ERR_ARG)
            if r["count"][f] == 0:                  # decided without a decode: 0, or the content size's verdict
                assert want in (0, fc.ERR_FRAME)
    assert {fc.OK, fc.ERR_FRAME, fc.ERR_UNSUPPORTED} <= seen


def test_argument_verdicts_per_frame(lib, oracle):
    fr = fc.good_frames(oracle, big=False)[5][0]
    r = index_host([fr, fr, fr, fr], [10, -1, 10, 0], [8, 8, 8, 8], sizes=[-1, len(fr), len(fr), len(fr)])
    assert r["status"][:3] == [fc.ERR_ARG, fc.ERR_ARG, fc.OK]
    assert r["base"][3] == r["count"][2]            # frame 3 comes after frame 2 in its class's table


@pytest.mark.parametrize("which", ["need", "one_less", "zero"])
def test_budget_rule_places_limit_on_the_right_frame(oracle, which):
    frames = corpus(oracle)
    order = np.random.default_rng(11).permutation(len(frames))
    frames = [frames[i] for i in order]
    caps = [1 << 24] * len(frames)
    free = index_host(frames, caps, [1 << 16] * 4)
    need = need_of(free)
    assert all(need)
    for c in range(4):
        mb = list(need)
        mb[c] = {"need": need[c], "one_less": need[c] - 1, "zero": 0}[which]
        r = index_host(frames, caps, mb)
        want = fc.budget_rule(frames, free["status"], free["cls"], mb)
        assert r["status"] == want, c
        limited = [f for f, s in enumerate(r["status"]) if s == fc.ERR_LIMIT and free["status"][f] == fc.OK]
        with_blocks = [f for f in range(len(frames)) if free["status"][f] == fc.OK and free["cls"][f] == c and free["count"][f]]
        if which == "need":
            assert not limited
        elif which == "one_less":                   # the last frame of the class with blocks, and every frame of the class after it
            assert limited[0] == with_blocks[-1] and all(free["cls"][f] == c for f in limited)
        else:
            assert set(with_blocks) <= set(limited)
        assert all(r["consumed"][f] == 0 for f in limited)
        check_tables(r, frames, mb)


def test_walk_stops_after_budget_plus_one_blocks(oracle):
    """a frame of many empty-ish blocks whose chain breaks late: over the budget it is LZ4B200_ERR_LIMIT, not a chain
    error, and the walk does not read past block budget + 1"""
    blk = fc.header((1 << 6) | (1 << 5), 4 << 4)
    body = b"".join(b"\x01\x00\x00\x00\x00" for _ in range(40))      # 40 one-byte blocks (token 0x00: 0 bytes)
    broken = blk + body + b"\x09\x00"                                  # then a truncated block header
    r = index_host([broken], [1 << 20], [39, 0, 0, 0])
    assert r["status"] == [fc.ERR_LIMIT] and r["count"] == [40]
    r = index_host([broken], [1 << 20], [40, 0, 0, 0])
    assert r["status"] == [fc.ERR_FRAME]
