"""LZ4B200_decompress_files without a GPU: the Python model of the call against every outcome of the reference `lz4`
tool in tests/golden/decompress_files.json (its deviations listed), the host build of the frame core's file steps
(tests/emul/decompress_files_emul.cpp) against the model on random files and at every budget edge, and the argument
rules and workspace size, checked without a launch."""
import ctypes as C
import hashlib
import random

import numpy as np
import pytest

import decompress_files_model as dm
import host_build
from conftest import load_golden

VERIFY, SKIP = 2, 1                                 # FC_SUMS_* (lz4_frame_core.h)

# Where the call and `lz4 -d` (v1.10.0) part, on purpose:
#   linked blocks are LZ4B200_ERR_UNSUPPORTED here and decoded by the tool;
DEV_LINKED = {"cli-BD-multi"}
#   under skipChecksums a compressed block's checksum is not compared (the tool still compares it);
DEV_SKIPPED_BLOCK_SUM = {("corrupt_blocksum", "skip"), ("corrupt_payload", "skip")}
#   the tool's multithreaded frame reader takes its input in 4 MB chunks and loses what follows a frame's end inside
#   the chunk, then reports "Stream followed by undecodable data"; the call follows the grammar, so the tool's output
#   is a prefix of the call's.
DEV_TOOL_CHUNKS = {"concat8", "concat13", "concat21", "concat40"}


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


@pytest.fixture(scope="module")
def oracle():
    from oracle.pyoracle import Oracle
    return Oracle()


@pytest.fixture(scope="module")
def corpus(oracle):
    g = load_golden("decompress_files.json")["files"]
    files = [dm.build_file(oracle, c) for c in g]
    return g, files


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import build, _lib
    build.build()
    return _lib.load()


def test_corpus_rebuilds(corpus):
    g, files = corpus
    assert len(g) >= 100
    for c, f in zip(g, files):
        assert len(f) == c["size"] and sha(f) == c["sha256"], c["name"]


@pytest.mark.parametrize("mode", ["verify", "skip"])
def test_model_matches_tool(corpus, oracle, mode):
    g, files = corpus
    units, blocks = dm.budget_needed(files, mode == "skip")
    res = dm.decompress_files(oracle, files, [1 << 40] * len(files), units, blocks, skip=mode == "skip")
    for c, (r, at, pre, out) in zip(g, res):
        ref = c[mode]
        if c["name"] in DEV_LINKED:
            assert r == dm.ERR_UNSUPPORTED and ref["exit"] == 0, c["name"]
        elif (c["name"], mode) in DEV_SKIPPED_BLOCK_SUM or c["name"] in DEV_TOOL_CHUNKS:
            assert r >= 0 and ref["exit"] != 0 and sha(out[:ref["size"]]) == ref["sha256"], c["name"]
        elif ref["exit"] == 0:
            assert (r, at, pre) == (ref["size"], c["size"], ref["size"]) and sha(out) == ref["sha256"], c["name"]
        else:
            assert r < 0 and pre <= ref["size"] and at < c["size"] or c["size"] == 0, c["name"]
            assert len(out) == pre


# ------------------------------------------------------------------------------------------------------------------
# the host build of the file steps
# ------------------------------------------------------------------------------------------------------------------
_ll, _llp = C.c_longlong, C.POINTER(C.c_longlong)
DECODE = C.CFUNCTYPE(C.c_int, C.c_longlong, C.c_int, C.c_int)


def emul():
    h = host_build.require()
    fn = h.files_host
    fn.restype = _ll
    fn.argtypes = [C.c_void_p, _llp, _llp, _llp, _ll, _ll, _llp, C.c_int, C.c_int, DECODE] + [_llp] * 6
    return h


def run_emul(oracle, files, caps, max_units, max_blocks, skip, size_only):
    """files_host on the batch laid out back to back: [(result, consumed, prefix)]"""
    h = emul()
    buf = np.frombuffer(b"".join(bytes(f) for f in files) + b"\0" * 16, dtype=np.uint8)
    sizes = [len(f) for f in files]
    offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64) if files else np.zeros(0, np.int64)
    arr = lambda v: np.ascontiguousarray(np.array(v, dtype=np.int64))   # noqa: E731
    so, ss, cp, mb = arr(offs), arr(sizes), arr(caps), arr(max_blocks)
    n = len(files)
    out = [np.zeros(n, np.int64) for _ in range(6)]

    def dec(off, size, cap):
        return oracle.decompress(buf[off:off + size].tobytes(), cap)[0] if size > 0 else -1

    p = lambda a: a.ctypes.data_as(_llp)                                 # noqa: E731
    h.files_host(buf.ctypes.data, p(so), p(ss), p(cp), n, max_units, p(mb), SKIP if skip else VERIFY,
                 1 if size_only else 0, DECODE(dec), *[p(o) for o in out])
    return list(zip(*[o.tolist() for o in out[:3]]))


def _batch(corpus, seed, k):
    g, files = corpus
    rng = random.Random(seed)
    pick = [i for i, c in enumerate(g) if c["size"] < (2 << 20)]
    return [files[rng.choice(pick)] for _ in range(k)]


def _check(oracle, files, caps, mu, mb, skip, size_only):
    want = [r[:3] for r in dm.decompress_files(oracle, files, caps, mu, mb, skip, size_only, content=False)]
    assert run_emul(oracle, files, caps, mu, mb, skip, size_only) == want, (mu, mb, skip, size_only)


@pytest.mark.parametrize("seed", range(4))
def test_emul_matches_model_random(corpus, oracle, seed):
    files = _batch(corpus, seed, 24)
    skip = bool(seed & 1)
    mu, mb = dm.budget_needed(files, skip)
    rng = random.Random(seed)
    caps = []
    for f in files:
        need = dm.decompress_files(oracle, [f], [1 << 40], mu, mb, skip, content=False)[0][0]
        caps.append(max(need, 0) + rng.choice([0, -1, 5, -3]) if need > 0 else rng.choice([0, 10]))
    caps[0] = -1                                          # ERR_ARG
    for size_only in (False, True):
        _check(oracle, files, caps, mu, mb, skip, size_only)


def test_emul_matches_model_budget_edges(corpus, oracle):
    files = _batch(corpus, 99, 16) + [dm.build_file(oracle, {"parts": [["legacy", [9 << 20, 0.5, 3, 0]]]})]
    mu, mb = dm.budget_needed(files)
    caps = [1 << 40] * len(files)
    edges = [(mu, mb), (mu - 1, mb), (0, mb), (1, mb)]
    for c in range(dm.CLASSES):
        if mb[c]:
            edges.append((mu, mb[:c] + [mb[c] - 1] + mb[c + 1:]))
            edges.append((mu, mb[:c] + [0] + mb[c + 1:]))
    for u, b in edges:
        for size_only in (False, True):
            _check(oracle, files, caps, max(u, 0), b, False, size_only)


def test_emul_hostile_skippable(oracle):
    f = b"".join(dm.skippable(b"", k % 16) for k in range(500))
    for mu in (499, 500, 501, 1000):
        _check(oracle, [f, f], [0, 0], mu, [0] * 5, False, False)


# ------------------------------------------------------------------------------------------------------------------
# argument rules, without a launch
# ------------------------------------------------------------------------------------------------------------------
def _budget(v):
    return (C.c_int64 * 5)(*v)


def test_workspace_bytes(lib):
    ws = lib.LZ4B200_decompress_files_workspace_bytes
    ok = _budget([1, 2, 3, 4, 5])
    assert ws(-1, 1, ok) == 0 and ws(1, -1, ok) == 0 and ws(1, 1 << 31, ok) == 0 and ws(1, 1, None) == 0
    for c in range(5):
        for bad in (-1, 1 << 31):
            v = [1] * 5
            v[c] = bad
            assert ws(1, 1, _budget(v)) == 0
    assert ws(0, 0, _budget([0] * 5)) > 0
    # the frames workspace for maxUnits frames, plus 40 bytes per unit and 32 per file (each region on 256 bytes)
    frames = lib.LZ4B200_decompress_frames_workspace_bytes
    base = frames(1000, (C.c_int64 * 4)(1, 2, 3, 4))
    assert ws(0, 1000, _budget([1, 2, 3, 4, 0])) == base + 5 * 8192
    assert ws(256, 1000, _budget([1, 2, 3, 4, 0])) == base + 5 * 8192 + 8192
    # a legacy block: about 2 x 8 MiB of the tiles kernel's marks
    extra = ws(0, 1, _budget([0, 0, 0, 0, 1])) - ws(0, 1, _budget([0] * 5))
    assert 2 * (8 << 20) < extra < 2 * (8 << 20) + (1 << 16)
    assert ws(0, 1, _budget([0, 0, 0, 0, 2])) - ws(0, 1, _budget([0] * 5)) > 2 * extra - 4096


def test_argument_errors(lib):
    f = lib.LZ4B200_decompress_files
    n0 = lib.LZ4B200_launch_count()
    ok = _budget([1] * 5)
    need = lib.LZ4B200_decompress_files_workspace_bytes(1, 1, ok)
    p = 4096                                                 # never dereferenced: every call below fails first
    a = [p, p, p, p, p, p, p, p, p]
    assert f(*a, 0, 1, ok, 0, 0, p, need, None) == 0
    assert f(*a, 0, 1, ok, 0, 1, None, 0, None) == 0          # nFiles == 0: OK, whatever the rest
    assert f(*a, -1, 1, ok, 0, 0, p, need, None) == -1
    assert f(*a, 1, 1, None, 0, 0, p, need, None) == -1
    assert f(*a, 1, -1, ok, 0, 0, p, need, None) == -1
    assert f(*a, 1, 1 << 31, ok, 0, 0, p, need, None) == -1
    assert f(*a, 1, 1, _budget([1, 1, 1, 1, -1]), 0, 0, p, need, None) == -1
    assert f(*a, 1, 1, ok, 0, 0, p, need - 1, None) == -1
    assert f(*a, 1, 1, ok, 0, 0, None, need, None) == -1
    for i in (0, 1, 2, 3, 4, 5, 6):                           # d_src .. d_result; d_consumed and d_prefix may be NULL
        b = list(a)
        b[i] = None
        assert f(*b, 1, 1, ok, 0, 0, p, need, None) == -1, i
        if i in (3, 4, 5):                                    # d_dst, d_dstOff, d_dstCap: not needed when sizing
            continue
        assert f(*b, 1, 1, ok, 0, 1, p, need, None) == -1, i
    assert lib.LZ4B200_launch_count() == n0


def test_size_only_block_checksum_without_content_checksum(oracle):
    """a frame with block checksums and no content checksum, one block checksum wrong: the size-only pass verifies block
    checksums, so the file fails with LZ4B200_ERR_CHECKSUM there too (the model once rewrote the EndMark as a content
    checksum and said LZ4B200_ERR_FRAME)"""
    import frame_checksum_model as fm
    pieces = [oracle.datagen(65536, 0.5, 3).tobytes(), oracle.datagen(1000, 0.5, 4).tobytes()]
    fr = bytearray(fm.frame_of_blocks(oracle, pieces, 4, block_sum=True, content_size=66536))
    blocks, _ = fm.walk(bytes(fr))
    o, sz, _ = blocks[1]
    fr[o + sz] ^= 1
    files = [bytes(fr)]
    for size_only in (False, True):
        r = dm.decompress_files(oracle, files, [1 << 20], 1, [2, 0, 0, 0, 0], size_only=size_only, content=False)
        assert r[0][:3] == (dm.ERR_CHECKSUM, 0, 0), size_only
        _check(oracle, files, [1 << 20], 1, [2, 0, 0, 0, 0], False, size_only)
