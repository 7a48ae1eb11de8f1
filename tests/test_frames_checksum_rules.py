"""LZ4B200_decompress_frames_checksummed without a GPU: its argument rules and workspace, XXH32 (the Python model's and
the device header's fc_xxh32) against the reference's digests, the index passes in checksum mode against a Python walk
of chains with checksum fields, and the Python model of the call against every outcome of the reference in
tests/golden/frames_checksum.json."""
import ctypes as C
import hashlib

import numpy as np
import pytest

import frame_checksum_model as fm
import frame_corpus as fc
import host_build
from conftest import load_golden

REJECT, SKIP, VERIFY = 0, 1, 2                      # FC_SUMS_* (lz4_frame_core.h)
SUM_NONE, SUM_PENDING = 0, 1                        # FC_SUM_*
BLOCK_SUM, CONTENT_SUM, VERIFY_BIT = 1, 2, 4        # fc_frame_rec.sums


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import build, _lib
    build.build()
    return _lib.load()


@pytest.fixture(scope="module")
def golden():
    return load_golden("frames_checksum.json")


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


_ll, _llp, _ip = C.c_longlong, C.POINTER(C.c_longlong), C.POINTER(C.c_int)


def emul():
    """host_build's library with the prototypes of tests/emul/frame_checksum_emul.cpp"""
    h = host_build.require()
    h.frames_xxh32_host.restype = C.c_uint
    h.frames_xxh32_host.argtypes = [C.c_void_p, C.c_ulonglong, C.c_uint]
    fn = h.frames_index_mode_host
    fn.restype = _ll
    fn.argtypes = [C.c_void_p, _llp, _llp, _llp, _ll, _llp, C.c_int] + [_llp] * 7 + [_ip, _ip, _llp]
    return h


def budget(*mb):
    return (C.c_int64 * 4)(*mb)


def test_workspace_is_the_checksum_free_calls(lib):
    """the same workspace function, and the call refuses one byte less"""
    ws = lib.LZ4B200_decompress_frames_workspace_bytes
    f = lib.LZ4B200_decompress_frames_checksummed
    p = 4096
    for mb in (budget(2, 1, 0, 0), budget(0, 0, 0, 5), budget(7, 7, 7, 7)):
        need = ws(3, mb)
        for skip in (0, 1):
            assert f(p, p, p, p, p, p, p, p, 3, mb, skip, p, need - 1, None) == fc.ERR_ARG


@pytest.mark.parametrize("skip", [0, 1, 7])
def test_argument_rules(lib, skip):
    ws = lib.LZ4B200_decompress_frames_workspace_bytes
    f = lib.LZ4B200_decompress_frames_checksummed
    p = 4096                                        # non-NULL stand-ins: every call below is refused before a launch
    mb = budget(2, 1, 0, 0)
    need = ws(3, mb)
    args = [p, p, p, p, p, p, p, p, 3, mb, skip, p, need, None]
    assert f(*args[:8], -1, *args[9:]) == fc.ERR_ARG
    assert f(*args[:9], None, *args[10:]) == fc.ERR_ARG
    assert f(*args[:9], budget(2, -1, 0, 0), *args[10:]) == fc.ERR_ARG
    assert f(*args[:9], budget(2, 1 << 31, 0, 0), *args[10:]) == fc.ERR_ARG
    for i in (0, 1, 2, 3, 4, 5, 6, 11):             # every pointer but d_consumed (7)
        bad = list(args)
        bad[i] = None
        assert f(*bad) == fc.ERR_ARG, i
    bad = list(args)
    bad[12] = need - 1
    assert f(*bad) == fc.ERR_ARG
    assert f(None, None, None, None, None, None, None, None, 0, mb, skip, None, 0, None) == fc.OK   # no frames, no launch


def test_xxh32_against_the_reference(oracle, golden):
    data = oracle.datagen(*golden["xxh32_data"]).tobytes()
    h = emul()
    assert len(golden["xxh32"]) >= 200
    for row in golden["xxh32"]:
        n, seed = row["len"], row["seed"]
        assert fm.xxh32(data[:n], seed) == row["xxh32"], (n, seed)
        assert h.frames_xxh32_host(data, n, seed) == row["xxh32"], (n, seed)


def index_mode(frames, caps, mb, mode, seed=0):
    h = emul()
    buf, offs = fc.layout(frames, seed=seed)
    n = len(frames)
    src = np.frombuffer(buf, dtype=np.uint8)
    off = np.array(offs, dtype=np.int64)
    size = np.array([len(x) for x in frames], dtype=np.int64)
    cap = np.array(caps, dtype=np.int64)
    mba = np.array(mb, dtype=np.int64)
    outs = [np.zeros(max(n, 1), dtype=np.int64) for _ in range(6)]
    ent = max(int(sum(mb)), 1)
    tso, tsz, trl, tmk = np.zeros(ent, np.int64), np.zeros(ent, np.int32), np.zeros(ent, np.int32), np.zeros(ent, np.int64)
    P = lambda a, t: a.ctypes.data_as(C.POINTER(t))                                    # noqa: E731
    got = h.frames_index_mode_host(src.ctypes.data, P(off, _ll), P(size, _ll), P(cap, _ll), n, P(mba, _ll), mode,
                                   *[P(o, _ll) for o in outs], P(tso, _ll), P(tsz, C.c_int), P(trl, C.c_int), P(tmk, _ll))
    assert got == sum(mb)
    status, cls, count, base, consumed, sums = (o[:n].tolist() for o in outs)
    return dict(off=offs, status=status, cls=cls, count=count, base=base, consumed=consumed, sums=sums,
                tab=list(zip(tso.tolist(), tsz.tolist(), trl.tolist(), tmk.tolist())))


def sum_corpus(oracle):
    """checksummed frames of every flag combination and block size, with raw blocks, and every truncation of their tails"""
    d = oracle.datagen(150000, 0.5, 3).tobytes()
    noise = np.random.default_rng(1).integers(0, 256, 70000, dtype=np.uint8).tobytes()
    frames = []
    for bsid in (4, 5, 6, 7):
        for bsum, csum in ((0, 0), (1, 0), (0, 1), (1, 1)):
            pieces = [d[:65536], noise[:65536], d[65536:70000], b"x"]
            frames.append(fm.frame_of_blocks(oracle, pieces, bsid, raw=(1, 3), block_sum=bsum, content_sum=csum,
                                             content_size=sum(map(len, pieces)) if bsid % 2 else None))
    cuts = []
    for f in frames[4:8]:                           # bsid 4, every flag combination: each cut inside the last 14 bytes
        cuts += [f[:len(f) - k] for k in range(1, 15)]
        blocks, _ = fm.walk(f)
        o, sz, _ = blocks[0]
        cuts += [f[:o + sz + k] for k in range(0, 4)]   # inside the first block's checksum (or the next header)
    return frames + cuts


@pytest.mark.parametrize("mode", [SKIP, VERIFY])
def test_index_passes_walk_the_checksum_fields(oracle, mode):
    frames = sum_corpus(oracle)
    mb = [1 << 12] * 4
    r = index_mode(frames, [1 << 24] * len(frames), mb, mode)
    tab_base = [sum(mb[:c]) for c in range(4)]
    seen = set()
    for f, fr in enumerate(frames):
        w = fm.walk(fr)
        bsum, csum = fm.sums_of(fr)
        if w is None:
            assert r["status"][f] == fc.ERR_FRAME and r["consumed"][f] == 0, f
            seen.add("cut")
            continue
        blocks, consumed = w
        assert r["status"][f] == fc.OK, f
        assert r["count"][f] == len(blocks) and r["consumed"][f] == consumed, f
        want_sums = (BLOCK_SUM if bsum else 0) | (CONTENT_SUM if csum else 0)
        assert r["sums"][f] == want_sums | (VERIFY_BIT if want_sums and mode == VERIFY else 0), f
        for k, (o, sz, raw) in enumerate(blocks):
            e = tab_base[r["cls"][f]] + r["base"][f] + k
            mark = SUM_PENDING if (bsum and mode == VERIFY) else SUM_NONE
            assert r["tab"][e] == (r["off"][f] + o, 0 if raw else sz, sz if raw else -1, mark), (f, k)
        seen.add((bsum, csum))
    assert seen == {"cut", (0, 0), (0, 1), (1, 0), (1, 1)}


def test_reject_mode_is_the_checksum_free_calls(oracle):
    """FC_SUMS_REJECT: a checksum flag is LZ4B200_ERR_UNSUPPORTED, a frame without one indexes as in the other modes"""
    frames = sum_corpus(oracle)[:16]
    mb = [1 << 12] * 4
    rej = index_mode(frames, [1 << 24] * len(frames), mb, REJECT)
    ver = index_mode(frames, [1 << 24] * len(frames), mb, VERIFY)
    for f, fr in enumerate(frames):
        if any(fm.sums_of(fr)):
            assert rej["status"][f] == fc.ERR_UNSUPPORTED and rej["consumed"][f] == 0
        else:
            assert (rej["status"][f], rej["count"][f], rej["consumed"][f], rej["sums"][f]) == \
                (ver["status"][f], ver["count"][f], ver["consumed"][f], 0)


def golden_frames(oracle, golden):
    """(frame, content) of every golden row, rebuilt by the model and checked against the reference's digest"""
    out = []
    for row in golden["frames"]:
        data = fm.content(oracle.datagen, row["spec"])
        f = fm.compress_frame(oracle, data, row["bsid"], row["content_size"], row["block_sum"], row["content_sum"])
        assert len(f) == row["frame_size"] and sha(f) == row["frame_sha256"] and sha(data) == row["src_sha256"]
        if "frame_hex" in row:
            assert f.hex() == row["frame_hex"]
        out.append((f, data))
    return out


def test_model_decodes_every_golden_frame(oracle, golden):
    frames = golden_frames(oracle, golden)
    assert {(r["block_sum"], r["content_sum"]) for r in golden["frames"]} == {(0, 0), (0, 1), (1, 0), (1, 1)}
    assert {fm.optimal_bsid(r["bsid"], r["spec"][0]) for r in golden["frames"]} == {4, 5, 6, 7}
    assert any(raw for f, _ in frames for _, _, raw in fm.walk(f)[0])
    cli = bytes.fromhex(golden["cli"]["frame_hex"])
    data = fm.content(oracle.datagen, golden["cli"]["spec"])
    assert sha(data) == golden["cli"]["src_sha256"] and fm.sums_of(cli) == (False, True)
    for f, d in frames + [(cli, data)]:
        for skip in (0, 1):
            assert fm.decode(oracle, f, len(d), skip) == (len(d), d, len(f))


def test_model_against_every_corrupted_outcome(oracle, golden):
    frames = golden_frames(oracle, golden)
    names = set()
    for row in golden["corrupted"]:
        f = frames[row["frame"]][0]
        m = dict(fm.mutations(f))[row["mutation"]]
        names.add(row["mutation"])
        for mode in ("verify", "skip"):
            ref = row[mode]
            got, data, _ = fm.decode(oracle, m, row["cap"], mode == "skip")
            if mode == "skip" and ref["error"] == "blockChecksum_invalid":
                # lz4frame.c:1871-1883 compares a compressed block's checksum even under skipChecksums; the call
                # compares none, so the block decodes as it is
                assert row["mutation"] in ("compressedPayload", "compressedBlockSum"), row
                if row["mutation"] == "compressedBlockSum":
                    assert got == len(frames[row["frame"]][1])
                continue
            want = fm.ref_class(ref)
            assert got == want, (row, got)
            if ref["error"] is None:
                assert sha(data) == ref["sha"], row
            if got == fm.ERR_CHECKSUM:
                assert mode == "verify"
    assert names == {"compressedPayload", "rawPayload", "compressedBlockSum", "rawBlockSum", "truncBlockSum",
                     "contentSum", "truncContentSum", "contentSize+1", "contentSize-1"}
