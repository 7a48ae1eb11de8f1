"""LZ4B200_compress_frames_checksummed on the CPU: the host model of its frames
(tests/compress_frames_checksum_model.py) against the reference's (tests/golden/compress_frames_checksum.json: LZ4F_compressFrame with
every nonzero flag combination, and the `lz4` tool's files), the header and bound of lz4_frame_core.h built for the host
for every flag combination, pass 1's capacity verdict against the checksummed bound, the call's argument rules, which
are decided on the host (no row launches anything), and the default capacities of batch.compress_frames_checksummed."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import compress_frames_checksum_model as M
import host_build
from conftest import GOLDEN
from frame_checksum_model import xxh32

OK, ARG = 0, -1
_ll = C.c_longlong
FLAGS = [(b, c) for b in (False, True) for c in (False, True)]


def _sums(b, c):
    return (1 if b else 0) | (2 if c else 0)


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "compress_frames_checksum.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def emul():
    lib = host_build.require()
    lib.cframes_header_sums_host.restype = C.c_int
    lib.cframes_header_sums_host.argtypes = [C.c_void_p, C.c_int, _ll, C.c_int]
    lib.cframes_bound_sums_host.restype = _ll
    lib.cframes_bound_sums_host.argtypes = [_ll, C.c_int, C.c_int]
    lib.cframes_index_sums_host.restype = C.c_int
    lib.cframes_index_sums_host.argtypes = [_ll, _ll, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(_ll),
                                            C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.cframes_header_host.restype = C.c_int
    lib.cframes_header_host.argtypes = [C.c_void_p, C.c_int, _ll]
    lib.cframes_bound_host.restype = _ll
    lib.cframes_bound_host.argtypes = [_ll, C.c_int]
    lib.frames_xxh32_host.restype = C.c_uint
    lib.frames_xxh32_host.argtypes = [C.c_void_p, C.c_ulonglong, C.c_uint]
    return lib


@pytest.fixture(scope="module")
def fast_xxh(emul):
    """XXH32 by the host build of fc_xxh32, for the megabytes of the large rows (pinned to the Python XXH32 below)"""
    def h(b):
        a = np.frombuffer(bytes(b), dtype=np.uint8)
        return int(emul.frames_xxh32_host(a.ctypes.data if len(a) else None, len(a), 0))
    return h


def test_fixture_covers_the_corpus(fixture):
    frames = fixture["frames"]
    assert [g["id"] for g in frames] == [c[0] for c in M.checksum_cases()]
    assert {g["level"] for g in frames} == {-5, 0, 1, 2, 9, 10, 12}
    assert {g["bsid"] for g in frames} == {0, 4, 5, 6, 7}
    assert {g["content_size"] for g in frames} == {False, True}
    assert {g["kind"] for g in frames} == {"p50", "rand"}
    assert all(set(g["sums"]) == {"B", "C", "BC"} for g in frames)
    assert {0, 1, 65535, 65536, 65537, 131073, (4 << 20) - 1, 4 << 20, (4 << 20) + 1, (8 << 20) + 1} <= \
        {g["size"] for g in frames}
    assert [(c["args"], c["bsid"], c["level"], c["block_sum"], c["content_sum"]) for c in fixture["cli"]] == \
        [tuple(r) for r in M.CLI_RUNS]
    assert fixture["cli_input"]["size"] == M.CLI_SIZE > 8 << 20 and fixture["cli_input"]["seed"] == M.CLI_SEED


def test_python_xxh32_is_the_host_xxh32(oracle, fast_xxh):
    for n in (0, 1, 15, 16, 17, 100, 65536, 200001):
        d = oracle.datagen(n, 0.5, n).tobytes()
        assert xxh32(d) == fast_xxh(d), n


def test_model_reproduces_every_golden_frame(oracle, fixture, fast_xxh):
    raw_blocks = 0
    for g in fixture["frames"]:
        data = M.corpus_data(oracle, g["kind"], g["size"], g["seed"])
        memo = {}
        codec = M.block_codec(oracle, g["level"])

        def cached(blk, cap):
            key = (len(blk), hash(blk))
            if key not in memo:
                memo[key] = codec(blk, cap)
            return memo[key]
        for name, (bsum, csum) in M.SUM_FLAGS.items():
            want = g["sums"][name]
            fr = M.frame(data, g["bsid"], g["content_size"], cached, block_sum=bsum, content_sum=csum,
                         xxh=xxh32 if g["size"] <= 70000 else fast_xxh)
            assert (len(fr), M.sha(fr)) == (want["length"], want["sha256"]), (g["id"], name)
            assert M.bound(g["size"], g["bsid"], bsum, csum) == want["bound"], (g["id"], name)
            if "hex" in want:
                assert fr.hex() == want["hex"], (g["id"], name)
            raw_blocks += sum(r for r, _ in M.blocks(fr))
    assert raw_blocks > 0                                    # stored-raw blocks carry checksums too


def test_model_reproduces_the_cli_frames(oracle, fixture, fast_xxh):
    data = M.cli_data(oracle)
    for c in fixture["cli"]:
        fr = M.frame(data, c["bsid"], False, M.block_codec(oracle, c["level"]), block_sum=c["block_sum"],
                     content_sum=c["content_sum"], xxh=fast_xxh)
        assert (len(fr), M.sha(fr)) == (c["length"], c["sha256"]), c["args"]
        assert len(M.blocks(fr)) > 1


def test_header_and_bound_on_the_host(emul, fixture):
    """fc_frame_header_sums and fc_frame_bound_sums for every flag combination, against the model and the fixture's
    verbatim frames and bounds; with no flags they are the functions LZ4B200_compress_frames uses"""
    buf = (C.c_ubyte * 16)()
    for bsid in (4, 5, 6, 7):
        for cs in (0, 1, 65536, (1 << 32) + 5):
            for b, c in FLAGS:
                n = emul.cframes_header_sums_host(buf, bsid, cs, _sums(b, c))
                assert bytes(buf[:n]) == M.header(bsid, cs, b, c), (bsid, cs, b, c)
                if not (b or c):
                    assert n == emul.cframes_header_host(buf, bsid, cs) and bytes(buf[:n]) == M.header(bsid, cs)
            for n in (0, 1, 65535, 65536, 65537, 5 << 20, 1 << 40):
                for b, c in FLAGS:
                    got = emul.cframes_bound_sums_host(n, bsid, _sums(b, c))
                    assert got == 19 + (8 if b else 4) * M.n_blocks(n, bsid) + n + 4 + (4 if c else 0)
                assert emul.cframes_bound_sums_host(n, bsid, 0) == emul.cframes_bound_host(n, bsid)
    assert emul.cframes_bound_sums_host(2 ** 63 - 30, 7, 3) == 2 ** 63 - 1             # saturates
    for g in fixture["frames"]:
        b = M.frame_bsid(g["bsid"], g["size"])
        for name, (bsum, csum) in M.SUM_FLAGS.items():
            want = g["sums"][name]
            assert emul.cframes_bound_sums_host(g["size"], b, _sums(bsum, csum)) == want["bound"], (g["id"], name)
            if "hex" in want:
                h = M.header(b, g["size"] if g["content_size"] else 0, bsum, csum)
                assert bytes.fromhex(want["hex"])[:len(h)] == h, (g["id"], name)


def test_index_pass_judges_the_checksummed_bound(emul):
    cls, hdr, sums = C.c_int(), C.c_int(), C.c_int()
    count = _ll()
    for n in (0, 1, 65536, 65537, 300000, 9 << 20):
        for bsid in (4, 5, 7):
            for b, c in FLAGS:
                s = _sums(b, c)
                bound = M.bound(n, bsid, b, c)
                for cap, want in ((bound, OK), (bound - 1, M.ERR_DSTSIZE), (-1, ARG)):
                    st = emul.cframes_index_sums_host(n, cap, bsid, 1, s, C.byref(cls), C.byref(count), C.byref(hdr),
                                                      C.byref(sums))
                    assert st == want, (n, bsid, b, c, cap)
                    if want == OK:
                        fb = M.frame_bsid(bsid, n)
                        assert (cls.value, count.value, hdr.value, sums.value) == \
                            (fb - 4, M.n_blocks(n, fb), 15 if n else 7, s)
    assert emul.cframes_index_sums_host(-1, 100, 4, 0, 3, C.byref(cls), C.byref(count), C.byref(hdr),
                                        C.byref(sums)) == ARG


# ------------------------------------------------------------------------------------------
# the call's argument rules, decided on the host
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


def _call(lib, n=3, bsid=4, level=0, cs=0, par=0, bsum=1, csum=1, mb=(4, 0, 0, 0), ws=P, wb=None, **ptrs):
    a = dict(src=P, soff=P, ssz=P, dst=P, doff=P, cap=P, res=P)
    a.update(ptrs)
    b = _budget(mb)
    if wb is None:
        wb = int(lib.LZ4B200_compress_frames_workspace_bytes(max(n, 0), b, level)) if mb is not None else 0
    return lib.LZ4B200_compress_frames_checksummed(a["src"], a["soff"], a["ssz"], a["dst"], a["doff"], a["cap"],
                                                   a["res"], n, bsid, level, cs, par, bsum, csum, b, ws, wb, None)


def _rows(lib):
    rows = []
    for bsum, csum in ((1, 1), (1, 0), (0, 1), (0, 0), (7, -3)):
        f = dict(bsum=bsum, csum=csum)
        tag = " (flags %d, %d)" % (bsum, csum)
        rows += [
            ("nFrames < 0" + tag, lambda f=f: _call(lib, n=-1, **f), ARG),
            ("nFrames == 0" + tag, lambda f=f: _call(lib, n=0, src=None, dst=None, ws=None, wb=0, **f), OK),
            ("NULL maxBlocks" + tag, lambda f=f: _call(lib, mb=None, **f), ARG),
            ("maxBlocks[0] < 0" + tag, lambda f=f: _call(lib, mb=(-1, 0, 0, 0), **f), ARG),
            ("maxBlocks[3] = 2^31" + tag, lambda f=f: _call(lib, mb=(0, 0, 0, 2 ** 31), wb=1 << 40, **f), ARG),
            ("parallel at level 2" + tag, lambda f=f: _call(lib, level=2, par=1, **f), ARG),
            ("parallel at level 12, no frames" + tag, lambda f=f: _call(lib, n=0, level=12, par=1, **f), ARG),
            ("NULL d_src" + tag, lambda f=f: _call(lib, src=None, **f), ARG),
            ("NULL d_srcOff" + tag, lambda f=f: _call(lib, soff=None, **f), ARG),
            ("NULL d_srcSize" + tag, lambda f=f: _call(lib, ssz=None, **f), ARG),
            ("NULL d_dst" + tag, lambda f=f: _call(lib, dst=None, **f), ARG),
            ("NULL d_dstOff" + tag, lambda f=f: _call(lib, doff=None, **f), ARG),
            ("NULL d_dstCap" + tag, lambda f=f: _call(lib, cap=None, **f), ARG),
            ("NULL d_result" + tag, lambda f=f: _call(lib, res=None, **f), ARG),
            ("NULL d_workspace" + tag, lambda f=f: _call(lib, ws=None, **f), ARG),
        ]
        for bsid in (-1, 1, 3, 8):
            rows.append(("blockSizeID %d" % bsid + tag, lambda bsid=bsid, f=f: _call(lib, bsid=bsid, **f), ARG))
        for level in (-5, 1, 2, 10, 13):
            rows.append(("level %d workspace one byte short" % level + tag,
                         lambda level=level, f=f: _call(lib, level=level, mb=(3, 2, 1, 1),
                                                        wb=int(lib.LZ4B200_compress_frames_workspace_bytes(
                                                            3, _budget((3, 2, 1, 1)), level)) - 1, **f), ARG))
    return rows


def test_argument_rules_launch_nothing(lib):
    """the rules of LZ4B200_compress_frames, whatever the checksum flags, decided before any launch"""
    before = lib.LZ4B200_launch_count()
    for name, call, want in _rows(lib):
        assert call() == want, name
    assert lib.LZ4B200_launch_count() == before


def test_default_capacities(lib):
    """batch's plan: the budget of compress_frames, and its capacities (LZ4B200_compressFrameBound, at least the
    reference's bound) plus 4 per block with block checksums and 4 per frame with a content checksum -- at least the
    reference's bound for those flags"""
    import torch
    from lz4_b200 import batch
    sizes = torch.tensor([0, 1, 65536, 65537, 300000, 9 << 20, -1], dtype=torch.int64)
    for bsid in (0, 4, 5, 7):
        base = batch._frame_plan(sizes, bsid)
        for b, c in FLAGS:
            budget, caps = batch._frame_plan(sizes, bsid, b, c)
            assert budget == base[0] == M.budget([int(n) for n in sizes], bsid)
            for n, cap, cap0 in zip(sizes.tolist(), caps, base[1]):
                if n < 0:
                    assert cap == (4 if c else 0) + cap0
                    continue
                assert cap == cap0 + (4 * M.n_blocks(n, M.frame_bsid(bsid, n)) if b else 0) + (4 if c else 0)
                assert cap >= M.bound(n, bsid, b, c), (bsid, n, b, c)
