"""LZ4B200_compress_frames_host and LZ4B200_compress_legacy_host without a GPU: the plan, the cut into groups and the
placement of runs, headers and trailers (lz4_cfiles_plan.h, through tests/emul/compress_files_host_emul.cpp) with the
blocks compressed by the oracle, against the golden corpus and the models of the device calls, at group sizes from one
block up, with the XXH32 state carried across every cut; the argument rules and nFiles == 0, which return before any
device use; LZ4B200_compressFrameBound_checksummed against the model; and the Python wrappers' checks."""
import ctypes as C
import hashlib
import random

import numpy as np
import pytest

import compress_frames_checksum_model as M
import compress_legacy_model as LM
import host_build
from conftest import load_golden
from frame_checksum_model import xxh32
from lz4_b200 import frame

ERR_ARG, ERR_DSTSIZE = -1, -5
MIB = 1 << 20

_ll, _llp = C.c_longlong, C.POINTER(C.c_longlong)
# (block index, source offset, size, capacity, out buffer) -> compressed size
ENCODE = C.CFUNCTYPE(C.c_int, C.c_longlong, C.c_longlong, C.c_int, C.c_int, C.c_void_p)
SHIM = [("compress_files_host_emul", _ll, [C.c_void_p, _llp, _llp, C.c_void_p, _llp, _llp, _llp, _ll, C.c_int,
                                           C.c_int, C.c_int, C.c_int, _ll, _ll, ENCODE])]


@pytest.fixture(scope="module")
def emu():
    lib = host_build.require()
    for name, res, args in SHIM:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import build, _lib
    build.build()
    return _lib.load()


@pytest.fixture(scope="module")
def oracle():
    from oracle.pyoracle import Oracle
    return Oracle()


def i64(a):
    return np.ascontiguousarray(np.array(a, dtype=np.int64))


def run_emul(emu, datas, caps, codec, legacy=False, bsid=7, cs=False, sums=0, group_bytes=1 << 30,
             group_blocks=1 << 20):
    """the shim over the files laid out back to back: (results, outputs, groups)"""
    src = np.frombuffer(b"".join(datas) + b"\0", dtype=np.uint8)
    n = len(datas)
    sizes = i64([len(d) for d in datas])
    offs = i64(np.concatenate([[0], np.cumsum(sizes)[:-1]]) if n else [])
    caps = i64(caps)
    room = np.maximum(caps, 0)
    doff = i64(np.concatenate([[0], np.cumsum(room)[:-1]]) if n else [])
    out = np.full(int(room.sum()) + 1, 0xA5, dtype=np.uint8)
    res = np.zeros(n, dtype=np.int64)

    def enc(b, off, size, cap, to):
        r, c = codec(src[off:off + size].tobytes(), cap)
        r = max(int(r), 0)
        C.memmove(to, bytes(c[:r]), r)
        return r

    cb = ENCODE(lambda b, off, size, cap, to: enc(b, off, size, cap, to))
    p = lambda a: a.ctypes.data_as(_llp)
    groups = emu.compress_files_host_emul(src.ctypes.data, p(offs), p(sizes), out.ctypes.data, p(doff), p(caps), p(res),
                                          n, int(legacy), bsid, int(cs), sums, group_bytes, group_blocks, cb)
    assert groups >= 0
    return res.tolist(), [out[o:o + r].tobytes() if r > 0 else b"" for o, r in zip(doff, res)], groups


def sha(b):
    return hashlib.sha256(b).hexdigest()


FLAGS = {"B": (True, False), "C": (False, True), "BC": (True, True)}


@pytest.mark.parametrize("group_bytes", [1, 200000, 1 << 30])
def test_golden_frames(emu, oracle, group_bytes):
    """every fast-level case of the checksummed corpus in all three flag combinations, one call per level, block size ID
    and content-size flag"""
    cases = [c for c in load_golden("compress_frames_checksum.json")["frames"] if c["level"] < 2]
    calls = {}
    for c in cases:
        calls.setdefault((c["level"], c["bsid"], c["content_size"]), []).append(c)
    for (level, bsid, cs), cs_cases in sorted(calls.items()):
        datas = [M.corpus_data(oracle, c["kind"], c["size"], c["seed"]) for c in cs_cases]
        codec = M.block_codec(oracle, level)
        for flags, (b, s) in FLAGS.items():
            sums = (1 if b else 0) | (2 if s else 0)
            caps = [c["sums"][flags]["bound"] for c in cs_cases]
            res, outs, _ = run_emul(emu, datas, caps, codec, bsid=bsid or 4, cs=cs, sums=sums, group_bytes=group_bytes)
            for c, r, o in zip(cs_cases, res, outs):
                g = c["sums"][flags]
                assert (r, sha(o)) == (g["length"], g["sha256"]), (c["id"], flags, group_bytes)


def test_golden_legacy(emu, oracle):
    """every fast-level stream of the legacy corpus, in groups of one chunk and in one group"""
    streams = [c for c in load_golden("compress_legacy.json")["streams"] if c["level"] < 3]
    calls = {}
    for c in streams:
        calls.setdefault(c["level"], []).append(c)
    for level, cases in sorted(calls.items()):
        datas = [LM.corpus_data(oracle, c["kind"], c["size"], c["seed"]) for c in cases]
        for group_bytes in (1, 1 << 30):
            res, outs, _ = run_emul(emu, datas, [c["bound"] for c in cases], LM.block_codec(oracle, level), legacy=True,
                                    group_bytes=group_bytes)
            assert [(r, sha(o)) for r, o in zip(res, outs)] == [(c["length"], c["sha256"]) for c in cases], level


def test_random_batches_against_the_model(emu, oracle):
    """seeded batches with failing files (a negative size is not laid out: capacities short by one), at random group
    sizes and block limits: every file equals the model of the device call, and the XXH32 state crosses every cut"""
    rng = random.Random(5)
    codec = M.block_codec(oracle, 1)
    for trial in range(12):
        n = rng.randint(1, 12)
        datas = [oracle.datagen(rng.choice([0, 1, 100, 65535, 65536, 65537, 300000, 1100000]), 0.5,
                                rng.randint(0, 999)).tobytes() for _ in range(n)]
        bsid, cs = rng.choice([4, 5, 6, 7]), rng.random() < 0.5
        b, s = rng.random() < 0.5, rng.random() < 0.5
        sums = (1 if b else 0) | (2 if s else 0)
        caps = [M.bound(len(d), bsid, b, s) - (1 if rng.random() < 0.2 else 0) for d in datas]
        res, outs, groups = run_emul(emu, datas, caps, codec, bsid=bsid, cs=cs, sums=sums,
                                     group_bytes=rng.choice([1, 70000, 1 << 20, 1 << 30]),
                                     group_blocks=rng.choice([1, 2, 3, 1 << 20]))
        for d, cap, r, o in zip(datas, caps, res, outs):
            if cap < M.bound(len(d), bsid, b, s):
                assert (r, o) == (ERR_DSTSIZE, b""), trial
            else:
                want = M.frame(d, bsid, cs, codec, block_sum=b, content_sum=s, xxh=xxh32)
                assert (r, o) == (len(want), want), trial
    # legacy streams of several chunks, one chunk per group
    datas = [oracle.datagen(n, 0.5, 3).tobytes() for n in (0, 8 * MIB, 8 * MIB + 1, 17 * MIB + 5)]
    lcodec = LM.block_codec(oracle, 1)
    res, outs, groups = run_emul(emu, datas, [LM.bound(len(d)) for d in datas], lcodec, legacy=True, group_bytes=1)
    assert groups == 6 and outs == [LM.stream(d, lcodec) for d in datas] and res == [len(o) for o in outs]


# ------------------------------------------------------------------------------------------
# without a device
# ------------------------------------------------------------------------------------------
def test_bound_against_the_model(lib):
    for n in [0, 1, 65535, 65536, 65537, 262144, 262145, 4 * MIB, 4 * MIB + 1, 10 ** 9, 5 * 10 ** 9]:
        for bsid in (0, 4, 5, 6, 7):
            for b in (0, 1):
                for c in (0, 1):
                    assert lib.LZ4B200_compressFrameBound_checksummed(n, bsid, b, c) == M.bound(n, bsid or 4, b, c)
    assert lib.LZ4B200_compressFrameBound_checksummed(-1, 7, 0, 1) == ERR_ARG
    for bsid in (1, 3, 8, -1):
        assert lib.LZ4B200_compressFrameBound_checksummed(10, bsid, 0, 1) == ERR_ARG


def test_argument_rules_without_a_device(lib):
    z = np.zeros(4, dtype=np.int64)
    p = z.ctypes.data
    f = lib.LZ4B200_compress_frames_host
    assert f(None, None, None, None, None, None, None, 0, 7, 1, 0, 0, 0, 1) == 0
    assert f(p, p, p, p, p, p, p, -1, 7, 1, 0, 0, 0, 1) == ERR_ARG
    for bsid in (1, 3, 8):
        assert f(p, p, p, p, p, p, p, 1, bsid, 1, 0, 0, 0, 1) == ERR_ARG
        assert f(None, None, None, None, None, None, None, 0, bsid, 1, 0, 0, 0, 1) == ERR_ARG
    assert f(p, p, p, p, p, p, p, 1, 7, 2, 0, 1, 0, 1) == ERR_ARG
    for k in range(7):
        args = [p] * 7
        args[k] = None
        assert f(*args, 1, 7, 1, 0, 0, 0, 1) == ERR_ARG
    g = lib.LZ4B200_compress_legacy_host
    assert g(None, None, None, None, None, None, None, 0, 1) == 0
    assert g(p, p, p, p, p, p, p, -1, 1) == ERR_ARG
    for k in range(7):
        args = [p] * 7
        args[k] = None
        assert g(*args, 1, 1) == ERR_ARG


def test_python_wrapper_checks():
    assert frame.compress_files([]) == []
    for kw in (dict(block_size_id=4), dict(content_size=True), dict(block_checksum=True), dict(content_checksum=False),
               dict(parallel=True)):
        with pytest.raises(ValueError):
            frame.compress_files([b"x"], legacy=True, **kw)
    with pytest.raises(ValueError):
        frame.compress_file(b"x", level=2 ** 31)
    with pytest.raises(ValueError):
        frame.compress_file(np.zeros(4, dtype=np.int32))
    with pytest.raises(frame.Lz4FrameError) as e:
        frame.compress_file(b"x", block_size_id=3)
    assert e.value.code == ERR_ARG
