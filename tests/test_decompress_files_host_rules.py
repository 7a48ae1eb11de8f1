"""LZ4B200_decompress_files_host without a GPU: its plan and fold (lz4_files_plan.h, through
tests/emul/files_plan_emul.cpp) against the model of LZ4B200_decompress_files with a budget that covers every file, on
the golden corpus and on seeded random batches at group sizes from one block up, with the blocks decoded by the oracle;
its argument rules and nFiles == 0, which return before any device use; the Python wrappers' checks; and the carried
XXH32 state of lz4_frame_core.h (tests/emul/xxh32_state_emul.cpp), which the call's carry kernel runs across groups,
against the one-shot fc_xxh32 and the model's xxh32 at every split of short messages and at random splits of long
ones."""
import ctypes as C
import random

import numpy as np
import pytest

import decompress_files_model as dm
import frame_checksum_model as fm
import host_build
from conftest import load_golden
from lz4_b200 import frame

ERR_ARG = -1

# the shim's functions, attached here so that host_build.PROTOTYPES stays the table of the shared emulators
_ll, _llp = C.c_longlong, C.POINTER(C.c_longlong)
DECODE = C.CFUNCTYPE(C.c_int, C.c_longlong, C.c_int, C.c_int)
CONTENT = C.CFUNCTYPE(C.c_int, C.c_longlong, C.c_longlong)
SHIM = [
    ("xxh32_state_pieces", C.c_uint, [C.c_void_p, _ll, _llp, C.c_int]),
    ("xxh32_state_oneshot", C.c_uint, [C.c_void_p, _ll]),
    ("files_plan_host", _ll, [C.c_void_p, _llp, _llp, _llp, _ll, C.c_int, _ll, DECODE, CONTENT, _llp, _llp, _llp]),
    # the host build of LZ4B200_decompress_files's own steps (tests/emul/decompress_files_emul.cpp)
    ("files_host", _ll, [C.c_void_p, _llp, _llp, _llp, _ll, _ll, _llp, C.c_int, C.c_int, DECODE] + [_llp] * 6),
]
MIB = 1 << 20


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


def run_plan(emu, oracle, files, caps, skip, group_bytes):
    """files_plan_host on the files laid out back to back (caps None: the size-only pass): [(result, consumed, prefix)]
    and the number of groups"""
    buf = np.frombuffer(b"".join(files) + b"\0" * 16, dtype=np.uint8)
    n = len(files)
    sizes = np.array([len(f) for f in files], dtype=np.int64)
    offs = np.zeros(n, dtype=np.int64)
    offs[1:] = np.cumsum(sizes)[:-1]
    capa = None if caps is None else np.array(caps, dtype=np.int64)
    out = [np.zeros(n, dtype=np.int64) for _ in range(3)]

    def dec(off, size, cap):
        return oracle.decompress(buf[off:off + size].tobytes(), cap)[0] if size > 0 else -1

    def content(f, off):                                   # the model's verdict on the frame's content checksum
        d = files[f]
        u = next(u for u in dm.walk_file(d, 1 << 40, [1 << 40] * 5, skip) if u["off"] == off)
        fr = d[off:off + u["length"]]
        with_sum = dm._frame_decode(oracle, fr, 1 << 62, skip, True)[0]
        without = dm._frame_decode(oracle, fr, 1 << 62, skip, False)[0]
        return int(without >= 0 and with_sum == dm.ERR_CHECKSUM)

    p = lambda a: None if a is None else a.ctypes.data_as(_llp)          # noqa: E731
    groups = emu.files_plan_host(buf.ctypes.data, p(offs), p(sizes), p(capa), n, 1 if skip else 0, group_bytes,
                                 DECODE(dec), CONTENT(content), *[p(o) for o in out])
    assert groups >= 0, groups
    return list(zip(*[o.tolist() for o in out])), groups


def device_sizes(emu, oracle, files, skip):
    """the size-only pass of LZ4B200_decompress_files's host build with the budget that covers every file.  (The model's
    size-only path, which re-decodes a frame that failed a checksum with its last four bytes made to match its content,
    reads those bytes as a content checksum even in a frame that has none; the device call's own steps are the
    reference here.)"""
    mu, mb = dm.budget_needed(files, skip)
    buf = np.frombuffer(b"".join(files) + b"\0" * 16, dtype=np.uint8)
    n = len(files)
    arr = lambda v: np.ascontiguousarray(np.array(v, dtype=np.int64))   # noqa: E731
    sizes = arr([len(f) for f in files])
    offs = np.zeros(n, dtype=np.int64)
    offs[1:] = np.cumsum(sizes)[:-1]
    out = [np.zeros(n, np.int64) for _ in range(6)]

    def dec(off, size, cap):
        return oracle.decompress(buf[off:off + size].tobytes(), cap)[0] if size > 0 else -1

    p = lambda a: a.ctypes.data_as(_llp)                                 # noqa: E731
    emu.files_host(buf.ctypes.data, p(offs), p(sizes), p(arr([0] * n)), n, mu, p(arr(mb)), 1 if skip else 2, 1,
                   DECODE(dec), *[p(o) for o in out])
    return list(zip(*[o.tolist() for o in out[:3]]))


def check_plan(emu, oracle, files, caps, skip, group_bytes, sized):
    """the decoding fold against the model, the size-only fold against `sized`"""
    mu, mb = dm.budget_needed(files, skip)
    want = [w[:3] for w in dm.decompress_files(oracle, files, caps, mu, mb, skip)]
    got, groups = run_plan(emu, oracle, files, caps, skip, group_bytes)
    assert got == want, (skip, group_bytes)
    assert run_plan(emu, oracle, files, None, skip, group_bytes)[0] == sized, (skip, group_bytes)
    return groups


@pytest.mark.parametrize("skip", [False, True])
def test_plan_and_fold_on_the_corpus(emu, oracle, corpus, skip):
    mu, mb = dm.budget_needed(corpus, skip)
    sized = dm.decompress_files(oracle, corpus, [1 << 40] * len(corpus), mu, mb, skip)
    exact = [r if r >= 0 else p + (1 << 16) for r, _, p, _ in sized]
    short = [e - 1 if e > 0 else 0 for e in exact]
    sized = device_sizes(emu, oracle, corpus, skip)
    assert sized == [w[:3] for w in dm.decompress_files(oracle, corpus, exact, mu, mb, skip, size_only=True)]
    for group_bytes in (1, MIB, 64 * MIB):
        for caps in (exact, short):
            groups = check_plan(emu, oracle, corpus, caps, skip, group_bytes, sized)
        if group_bytes == 1:                              # one block per group
            assert groups == sum(sum(u["count"] for u in dm.walk_file(f, 1 << 40, [1 << 40] * 5, skip)
                                     if u["status"] == dm.OK) for f in corpus)


def random_file(oracle, rng):
    """a file of 1 .. 5 units: frames at every block size with random checksum flags (some corrupted), skippable
    frames, legacy streams; sometimes cut short"""
    out = bytearray()
    for _ in range(rng.randint(1, 5)):
        kind = rng.random()
        n = rng.choice([0, 1, 100, 5000, 70000, 300000, 1100000])
        data = oracle.datagen(n, rng.choice([0.2, 0.5, 0.9]), rng.randrange(1000)).tobytes() if n else b""
        if kind < 0.65:
            f = bytearray(fm.compress_frame(oracle, data, rng.randint(4, 7), rng.random() < 0.5, rng.random() < 0.5,
                                            rng.random() < 0.6))
            if len(f) > 20 and rng.random() < 0.2:
                f[rng.randrange(7, len(f))] ^= 0x20
            out += f
        elif kind < 0.8:
            out += dm.skippable(bytes(rng.randrange(50)), rng.randrange(16))
        else:
            out += dm.legacy(lambda b: oracle.compress(b, 1)[1], data)
    if rng.random() < 0.1:
        out = out[:rng.randrange(len(out) + 1)]
    return bytes(out)


@pytest.mark.parametrize("seed", range(4))
def test_plan_and_fold_on_random_batches(emu, oracle, corpus, seed):
    rng = random.Random(seed)
    small = [f for f in corpus if len(f) < 2 * MIB]
    files = [random_file(oracle, rng) if rng.random() < 0.6 else rng.choice(small) for _ in range(30)]
    skip = bool(seed & 1)
    mu, mb = dm.budget_needed(files, skip)
    need = [w[0] for w in dm.decompress_files(oracle, files, [1 << 40] * len(files), mu, mb, skip)]
    caps = [max(r, 0) + rng.choice([0, 0, -1, 7]) for r in need]
    caps[rng.randrange(len(caps))] = -1                   # ERR_ARG
    sized = device_sizes(emu, oracle, files, skip)
    for group_bytes in (1, 64 << 10, 300 << 10, 4 * MIB, 64 * MIB):
        check_plan(emu, oracle, files, caps, skip, group_bytes, sized)


def pieces(emu, buf, cuts):
    arr = (_ll * max(len(cuts), 1))(*cuts)
    return emu.xxh32_state_pieces(buf.ctypes.data, len(buf), arr, len(cuts))


def test_short_messages_split_at_every_point(emu):
    rng = np.random.default_rng(1)
    for n in range(101):
        buf = rng.integers(0, 256, max(n, 1), dtype=np.uint8)[:n].copy()
        want = fm.xxh32(buf.tobytes())
        assert emu.xxh32_state_oneshot(buf.ctypes.data, n) == want, n
        assert pieces(emu, buf, []) == want and pieces(emu, buf, [n]) == want, n
        for a in range(n + 1):
            assert pieces(emu, buf, [a, n]) == want, (n, a)
        for a in range(0, n + 1, 7):                      # three pieces, empty ones included
            for b in range(a, n + 1, 5):
                assert pieces(emu, buf, [a, b, n]) == want, (n, a, b)


def test_long_messages_in_random_pieces(emu):
    rng = np.random.default_rng(2)
    r = random.Random(3)
    big = rng.integers(0, 256, 20 << 20, dtype=np.uint8)
    for trial in range(24):
        n = r.randint(1 << 20, 20 << 20)
        buf = big[:n]
        want = emu.xxh32_state_oneshot(buf.ctypes.data, n)
        k = r.randint(1, 64)
        cuts = sorted(r.sample(range(1, n), k - 1)) + [n]
        if trial % 4 == 0:                                # pieces that end on and next to stripe edges
            cuts = sorted({min(n, max(1, c - c % 16 + r.choice([-1, 0, 1]))) for c in cuts} | {n})
        assert pieces(emu, buf, cuts) == want, (n, k)
    small = big[:100000]
    assert emu.xxh32_state_oneshot(small.ctypes.data, len(small)) == fm.xxh32(small.tobytes())
    assert pieces(emu, small, [1, 17, 50000, 99999, 100000]) == fm.xxh32(small.tobytes())


def test_argument_rules_before_any_device_use(lib):
    """ERR_ARG and nFiles == 0 are decided on the arguments alone: no device is needed for them"""
    call = lib.LZ4B200_decompress_files_host
    src = np.zeros(16, dtype=np.uint8)
    i64 = lambda *v: np.array(v, dtype=np.int64)
    off, size, cap, res, dst = i64(0), i64(7), i64(100), i64(0), np.zeros(100, dtype=np.uint8)
    p = lambda a: a.ctypes.data
    assert call(None, None, None, None, None, None, None, None, None, 0, 0, 0) == 0
    assert call(None, None, None, None, None, None, None, None, None, 0, 1, 1) == 0
    assert call(p(src), p(off), p(size), p(dst), p(off), p(cap), p(res), None, None, -1, 0, 0) == ERR_ARG
    full = [p(src), p(off), p(size), p(dst), p(off), p(cap), p(res), None, None, 1, 0, 0]
    for k in (0, 1, 2, 3, 4, 5, 6):                       # every required pointer, one at a time
        args = list(full)
        args[k] = None
        assert call(*args) == ERR_ARG, k
    for k in (0, 1, 2, 6):                                # sizeOnly still needs the source and the results
        args = list(full)
        args[k] = None
        args[11] = 1
        assert call(*args) == ERR_ARG, k


class Recorder:
    def __init__(self):
        self.calls = 0

    def LZ4B200_decompress_files_host(self, *args):
        self.calls += 1
        return 0


def test_wrapper_checks(monkeypatch):
    rec = Recorder()
    monkeypatch.setattr(frame._lib, "load", lambda: rec)
    with pytest.raises(ValueError, match="int64"):
        frame.decompress_files([b"x"], [2 ** 63])
    with pytest.raises(ValueError, match="int64"):
        frame.decompress_file(b"x", -2 ** 63 - 1)
    with pytest.raises(ValueError, match="capacities has"):
        frame.decompress_files([b"x", b"y"], [1])
    with pytest.raises(ValueError, match="uint8"):
        frame.decompress_files([np.zeros(4, dtype=np.int16)])
    assert rec.calls == 0
    assert frame.decompress_files([]) == []
    assert frame.decompress_files([], size_only=True) == []


def test_error_names():
    assert "budget" in str(frame.Lz4FrameError(-6, "x")) and "checksum" in str(frame.Lz4FrameError(-7, "x"))
