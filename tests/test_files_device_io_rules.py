"""LZ4B200_decompress_files_to_device, LZ4B200_compress_frames_from_device and LZ4B200_compress_legacy_from_device
without a GPU: the placement both file readers share (fp_place in lz4_files_plan.h, through
tests/emul/files_place_emul.cpp) puts every file's bytes where the model of LZ4B200_decompress_files puts them, and stops
and clips where it stops, on the golden corpus and on seeded random batches at group sizes from one block up, with rooms
at the exact size, one byte less and 0; the three calls' argument rules and their order, which need no device; and the
Python wrappers' own checks."""
import ctypes as C
import random

import numpy as np
import pytest

import decompress_files_model as dm
import host_build
import test_decompress_files_host_rules as R
from conftest import load_golden
from lz4_b200 import frame

ERR_ARG, ERR_CUDA = -1, -2
MIB = 1 << 20
GUARD, GAP = 0xA5, 24

_ll, _llp = C.c_longlong, C.POINTER(C.c_longlong)
DECODE = C.CFUNCTYPE(C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_void_p)
CONTENT = R.CONTENT
SHIM = [("files_place_host", _ll, [C.c_void_p, _llp, _llp, _llp, _ll, C.c_int, _ll, DECODE, CONTENT, C.c_void_p, _llp,
                                   _llp, _llp, _llp])]


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


@pytest.fixture(scope="module")
def corpus(oracle):
    return [dm.build_file(oracle, c) for c in load_golden("decompress_files.json")["files"]]


def run_place(emu, oracle, files, caps, skip, group_bytes):
    """files_place_host on the files laid out back to back, into regions GAP guard bytes apart: [(result, consumed,
    prefix)], each region's bytes, whether every guard is intact, and the number of runs"""
    buf = np.frombuffer(b"".join(files) + b"\0" * 16, dtype=np.uint8)
    n = len(files)
    sizes = np.array([len(f) for f in files], dtype=np.int64)
    offs = np.zeros(n, dtype=np.int64)
    offs[1:] = np.cumsum(sizes)[:-1]
    capa = np.array(caps, dtype=np.int64)
    room = np.maximum(capa, 0)
    oo = GAP + np.concatenate([[0], np.cumsum(room + GAP)[:-1]]).astype(np.int64)
    dst = np.full(int((room + GAP).sum()) + GAP, GUARD, dtype=np.uint8)
    out = [np.zeros(n, dtype=np.int64) for _ in range(3)]

    def dec(off, size, cap, at):
        if size <= 0:
            return -1
        r, b = oracle.decompress(buf[off:off + size].tobytes(), cap)
        C.memmove(at, b, len(b))
        return r

    def content(f, off):
        d = files[f]
        u = next(u for u in dm.walk_file(d, 1 << 40, [1 << 40] * 5, skip) if u["off"] == off)
        fr = d[off:off + u["length"]]
        with_sum = dm._frame_decode(oracle, fr, 1 << 62, skip, True)[0]
        without = dm._frame_decode(oracle, fr, 1 << 62, skip, False)[0]
        return int(without >= 0 and with_sum == dm.ERR_CHECKSUM)

    p = lambda a: a.ctypes.data_as(_llp)                                 # noqa: E731
    runs = emu.files_place_host(buf.ctypes.data, p(offs), p(sizes), p(capa), n, 1 if skip else 0, group_bytes,
                                DECODE(dec), CONTENT(content), dst.ctypes.data, p(oo), *[p(o) for o in out])
    assert runs >= 0, runs
    regions = [dst[o:o + c].tobytes() for o, c in zip(oo, room)]
    mask = np.ones(len(dst), dtype=bool)
    for o, c in zip(oo, room):
        mask[o:o + c] = False
    return list(zip(*[o.tolist() for o in out])), regions, bool((dst[mask] == GUARD).all()), runs


def check_place(emu, oracle, files, caps, skip, group_bytes):
    """the results are the model's, and each region begins with the model's bytes of the file: its output, or the
    prefix's on failure"""
    mu, mb = dm.budget_needed(files, skip)
    want = dm.decompress_files(oracle, files, caps, mu, mb, skip)
    got, regions, guards, runs = run_place(emu, oracle, files, caps, skip, group_bytes)
    assert got == [w[:3] for w in want], (skip, group_bytes)
    assert guards, (skip, group_bytes)
    for k, (w, reg) in enumerate(zip(want, regions)):
        assert reg[:len(w[3])] == w[3], (k, skip, group_bytes)
    return runs


@pytest.mark.parametrize("skip", [False, True])
def test_placement_on_the_corpus(emu, oracle, corpus, skip):
    mu, mb = dm.budget_needed(corpus, skip)
    sized = dm.decompress_files(oracle, corpus, [1 << 40] * len(corpus), mu, mb, skip)
    exact = [r if r >= 0 else p for r, _, p, _ in sized]
    for group_bytes in (1, 300 << 10, MIB, 64 * MIB):
        for caps in (exact, [e - 1 if e > 0 else 0 for e in exact], [0] * len(exact)):
            runs = check_place(emu, oracle, corpus, caps, skip, group_bytes)
            if not any(caps):
                assert runs == 0


@pytest.mark.parametrize("seed", range(4))
def test_placement_on_random_batches(emu, oracle, corpus, seed):
    rng = random.Random(seed)
    small = [f for f in corpus if len(f) < 2 * MIB]
    files = [R.random_file(oracle, rng) if rng.random() < 0.6 else rng.choice(small) for _ in range(30)]
    skip = bool(seed & 1)
    mu, mb = dm.budget_needed(files, skip)
    need = [w[0] if w[0] >= 0 else w[2] for w in dm.decompress_files(oracle, files, [1 << 40] * len(files), mu, mb,
                                                                        skip)]
    for group_bytes in (1, 64 << 10, 300 << 10, 4 * MIB, 64 * MIB):
        caps = [max(r, 0) + rng.choice([0, 0, -1, 7, -r]) for r in need]
        caps[rng.randrange(len(caps))] = -1               # ERR_ARG
        check_place(emu, oracle, files, caps, skip, group_bytes)


def test_one_run_per_file_of_one_group(emu, oracle):
    """the blocks of one file that lie together in a group merge into one run"""
    d = oracle.datagen(3 * MIB + 5, 0.5, 2).tobytes()
    f = dm.fm.compress_frame(oracle, d, 4, False, 1, 1)
    files = [f, f, f]
    assert check_place(emu, oracle, files, [len(d)] * 3, False, 64 * MIB) == 3
    assert check_place(emu, oracle, files, [len(d)] * 3, False, 1) == 3 * 49


# ------------------------------------------------------------------------------------------
# argument rules, with no device
# ------------------------------------------------------------------------------------------
def arrays():
    i64 = lambda *v: np.array(v, dtype=np.int64)              # noqa: E731
    return np.zeros(64, dtype=np.uint8), i64(0), i64(7), i64(100), i64(0), np.zeros(100, dtype=np.uint8)


def test_reader_argument_rules(lib):
    call = lib.LZ4B200_decompress_files_to_device
    src, off, size, cap, res, dst = arrays()
    p = lambda a: a.ctypes.data                                # noqa: E731
    launches = lib.LZ4B200_launch_count()
    assert call(None, None, None, None, None, None, None, None, None, -1, 0, None) == ERR_ARG
    assert call(None, None, None, None, None, None, None, None, None, 0, 0, None) == 0
    assert call(p(src), p(off), p(size), p(dst), p(off), p(cap), p(res), None, None, -1, 0, None) == ERR_ARG
    assert call(p(src), p(off), p(size), p(dst), p(off), p(cap), p(res), None, None, 0, 1, None) == 0
    assert lib.LZ4B200_launch_count() == launches
    full = [p(src), p(off), p(size), p(dst), p(off), p(cap), p(res), None, None, 1, 0, None]
    for k in range(7):                                    # every required pointer, one at a time
        args = list(full)
        args[k] = None
        assert call(*args) == ERR_ARG, k
    if lib.LZ4B200_device_count() == 0:
        assert call(*full) == ERR_CUDA and b"no CUDA device" in lib.LZ4B200_last_cuda_error()


@pytest.mark.parametrize("legacy", [False, True])
def test_writer_argument_rules(lib, legacy):
    src, off, size, cap, res, dst = arrays()
    p = lambda a: a.ctypes.data                                # noqa: E731
    if legacy:
        call = lambda s, o, z, d, do, c, r, n, bsid=7, par=0: lib.LZ4B200_compress_legacy_from_device(  # noqa: E731
            s, o, z, d, do, c, r, n, 1, None)
    else:
        call = lambda s, o, z, d, do, c, r, n, bsid=7, par=0: lib.LZ4B200_compress_frames_from_device(  # noqa: E731
            s, o, z, d, do, c, r, n, bsid, 1, 0, par, 0, 1, None)
    launches = lib.LZ4B200_launch_count()
    assert call(None, None, None, None, None, None, None, -1) == ERR_ARG
    assert call(None, None, None, None, None, None, None, 0) == 0
    assert call(None, None, None, None, None, None, None, 0, bsid=3, par=1) == 0      # nFiles == 0 comes first
    assert lib.LZ4B200_launch_count() == launches
    full = [p(src), p(off), p(size), p(dst), p(off), p(cap), p(res), 1]
    for k in range(7):
        args = list(full)
        args[k] = None
        assert call(*args) == ERR_ARG, k
    if not legacy:
        for bsid in (1, 3, 8, -1):
            assert call(*full, bsid=bsid) == ERR_ARG, bsid
        assert lib.LZ4B200_compress_frames_from_device(*full, 7, 2, 0, 1, 0, 1, None) == ERR_ARG   # parallel, HC
    if lib.LZ4B200_device_count() == 0:
        assert call(*full) == ERR_CUDA and b"no CUDA device" in lib.LZ4B200_last_cuda_error()
        if not legacy:
            assert call(*full, bsid=0) == ERR_CUDA                     # 0 means 4
            assert call(*full, par=1) == ERR_CUDA                      # parallel at level 1


class Recorder:
    def __init__(self):
        self.calls = 0

    def __getattr__(self, name):
        if not name.startswith("LZ4B200_"):
            raise AttributeError(name)

        def rec(*args):
            self.calls += 1
            return 0
        return rec


def test_wrapper_checks(monkeypatch):
    torch = pytest.importorskip("torch")
    rec = Recorder()
    monkeypatch.setattr(frame._lib, "load", lambda: rec)
    with pytest.raises(ValueError, match="int64"):
        frame.decompress_files_to_device([b"x"], [2 ** 63])
    with pytest.raises(ValueError, match="capacities has"):
        frame.decompress_files_to_device([b"x", b"y"], [1])
    with pytest.raises(ValueError, match="uint8"):
        frame.decompress_file_to_device(np.zeros(4, dtype=np.int16))
    assert frame.decompress_files_to_device([]) == []
    with pytest.raises(ValueError, match="CPU"):
        frame.compress_files_from_device([torch.zeros(4)])
    with pytest.raises(ValueError, match="CPU"):
        frame.compress_file_from_device(torch.zeros(4, 4).t())
    with pytest.raises(ValueError, match="not a tensor"):
        frame.compress_file_from_device(b"abc")
    for kw in (dict(block_size_id=4), dict(content_size=True), dict(block_checksum=True), dict(content_checksum=False),
               dict(parallel=True)):
        with pytest.raises(ValueError, match="legacy"):
            frame.compress_files_from_device([torch.zeros(4)], legacy=True, **kw)
    assert rec.calls == 0
