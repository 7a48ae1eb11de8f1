"""The host wrappers (lz4_b200.block, lz4_b200.frame) hand the library every byte of what they are given, and refuse what
the C call would misread.

A uint8 ndarray of any shape or layout is passed as its bytes in C order: a (4, 100) array is 400 bytes, not 4 rows.
Another dtype, and a length, capacity, target, level or acceleration outside the C int the call takes, raise ValueError
before the library is called (ctypes would cut 2^32 + 5 to 5).  The CPU tests run against a stand-in of the library
that records what each call received; the GPU test runs a 2-D array through the real calls against the oracle."""
import ctypes as C

import numpy as np
import pytest

from lz4_b200 import _lib, block, frame

INT_MAX = 2 ** 31 - 1


class HostRecorder:
    """liblz4_b200's host calls as block.py and frame.py see them: each call records (name, the bytes at its source
    pointer, its source length) and returns 0; the bound and state-size functions compute what the library returns."""

    def __init__(self):
        self.calls = []

    def LZ4_compressBound(self, n):
        return n + n // 255 + 16 if 0 <= n <= 0x7E000000 else 0

    def LZ4_sizeofStateHC(self):
        return 262200

    def LZ4B200_compressFrameBound(self, n, bsid):
        return n + n // 255 + 4096

    def __getattr__(self, name):
        if not name.startswith("LZ4"):
            raise AttributeError(name)
        # where the source pointer and its length are in each prototype (a length given by pointer is read through it)
        at = {"LZ4_compress_fast": (0, 2), "LZ4_compress_default": (0, 2), "LZ4_compress_HC": (0, 2),
              "LZ4_decompress_safe": (0, 2), "LZ4_decompress_safe_partial": (0, 2), "LZ4_compress_destSize": (0, 2),
              "LZ4_compress_destSize_extState": (1, 3), "LZ4_compress_HC_destSize": (1, 3),
              "LZ4B200_compressFrame_host": (0, 1), "LZ4B200_decompressFrame_host": (0, 1)}[name]

        def call(*args):
            ptr, n = args[at[0]], args[at[1]]
            n = n._obj.value if isinstance(n, type(C.byref(C.c_int()))) else int(n)
            self.calls.append((name, C.string_at(ptr, n) if ptr else b"", n))
            return 0
        return call


@pytest.fixture
def rec(monkeypatch):
    r = HostRecorder()
    monkeypatch.setattr(_lib, "load", lambda: r)
    return r


# every host call as f(data): its C entry point, and the call with valid sizes
CALLS = {
    "LZ4_compress_fast": ("LZ4_compress_fast", lambda d: block.LZ4_compress_fast(d)),
    "LZ4_compress_default": ("LZ4_compress_default", lambda d: block.LZ4_compress_default(d, 1000)),
    "LZ4_compress_destSize": ("LZ4_compress_destSize", lambda d: block.LZ4_compress_destSize(d, 300)),
    "LZ4_compress_destSize accel": ("LZ4_compress_destSize_extState",
                                    lambda d: block.LZ4_compress_destSize(d, 300, acceleration=2)),
    "LZ4_compress_HC": ("LZ4_compress_HC", lambda d: block.LZ4_compress_HC(d, 9)),
    "LZ4_compress_HC_destSize": ("LZ4_compress_HC_destSize", lambda d: block.LZ4_compress_HC_destSize(d, 300, 9)),
    "LZ4_decompress_safe": ("LZ4_decompress_safe", lambda d: block.LZ4_decompress_safe(d, 5000)),
    "LZ4_decompress_safe_partial": ("LZ4_decompress_safe_partial", lambda d: block.LZ4_decompress_safe_partial(d, 99)),
    "compress_frame": ("LZ4B200_compressFrame_host", lambda d: frame.compress_frame(d)),
    "decompress_frame": ("LZ4B200_decompressFrame_host", lambda d: frame.decompress_frame(d, 5000)),
}
BLOCK_CALLS = [k for k, (entry, _) in CALLS.items() if entry.startswith("LZ4_")]


def layouts():
    """(name, array, its bytes in C order): 2-D, 3-D, non-contiguous and transposed uint8 arrays"""
    a = np.arange(1200, dtype=np.uint64).astype(np.uint8).reshape(4, 300)
    yield "2-D", a[:, :100].copy(), a[:, :100].tobytes()
    yield "3-D", a.reshape(4, 3, 100), a.tobytes()
    yield "strided columns", a[:, ::3], a[:, ::3].tobytes()
    yield "transposed", a[:, :7].T, np.ascontiguousarray(a[:, :7].T).tobytes()
    yield "every other row", a[::2], a[::2].tobytes()


@pytest.mark.parametrize("call", list(CALLS))
@pytest.mark.parametrize("layout", [name for name, _, _ in layouts()])
def test_an_array_passes_all_its_bytes(rec, call, layout):
    entry, fn = CALLS[call]
    _, arr, want = next(x for x in layouts() if x[0] == layout)
    fn(arr)
    (name, got, n), = rec.calls
    assert name == entry and n == len(want) and got == want, (name, n, len(want))


@pytest.mark.parametrize("call", list(CALLS))
@pytest.mark.parametrize("dtype", [np.int8, np.uint16, np.float32, np.int64])
def test_an_array_of_another_dtype_raises_before_any_call(rec, call, dtype):
    _, fn = CALLS[call]
    with pytest.raises(ValueError):
        fn(np.zeros(64, dtype=dtype))
    assert rec.calls == []


# the sizes each block call takes as a C int, with a value just past INT_MAX and one that ctypes would cut to a small one
TOO_BIG = [INT_MAX + 1, 2 ** 32 + 5, -2 ** 31 - 1]
SIZE_ARGS = [
    ("LZ4_compress_fast", lambda v, d: block.LZ4_compress_fast(d, v)),
    ("LZ4_compress_fast", lambda v, d: block.LZ4_compress_fast(d, 100, acceleration=v)),
    ("LZ4_compress_default", lambda v, d: block.LZ4_compress_default(d, v)),
    ("LZ4_compress_destSize", lambda v, d: block.LZ4_compress_destSize(d, v)),
    ("LZ4_compress_destSize", lambda v, d: block.LZ4_compress_destSize(d, 100, acceleration=v)),
    ("LZ4_compress_HC", lambda v, d: block.LZ4_compress_HC(d, 9, v)),
    ("LZ4_compress_HC", lambda v, d: block.LZ4_compress_HC(d, v)),
    ("LZ4_compress_HC_destSize", lambda v, d: block.LZ4_compress_HC_destSize(d, v)),
    ("LZ4_compress_HC_destSize", lambda v, d: block.LZ4_compress_HC_destSize(d, 100, v)),
    ("LZ4_decompress_safe", lambda v, d: block.LZ4_decompress_safe(d, v)),
    ("LZ4_decompress_safe_partial", lambda v, d: block.LZ4_decompress_safe_partial(d, v)),
    ("LZ4_decompress_safe_partial", lambda v, d: block.LZ4_decompress_safe_partial(d, 10, v)),
    ("LZ4_compressBound", lambda v, d: block.LZ4_compressBound(v)),
]


@pytest.mark.parametrize("k", range(len(SIZE_ARGS)), ids=["%s-%d" % (a[0], i) for i, a in enumerate(SIZE_ARGS)])
@pytest.mark.parametrize("value", TOO_BIG)
def test_a_size_past_the_c_int_raises_before_any_call(rec, k, value):
    _, fn = SIZE_ARGS[k]
    with pytest.raises(ValueError):
        fn(value, b"\x01" * 64)
    assert rec.calls == []


def test_sizes_at_the_c_int_limits_go_through(rec):
    """INT_MAX and INT_MIN themselves fit: they reach the call unchanged"""
    block.LZ4_decompress_safe(b"\x10\x41", INT_MAX)
    block.LZ4_decompress_safe_partial(b"\x10\x41", 5, -2 ** 31)
    assert [n for _, _, n in rec.calls] == [2, 2]


@pytest.mark.parametrize("call", BLOCK_CALLS)
def test_a_source_past_int_max_never_reaches_the_library(rec, call):
    """2^31 + 5 bytes (never touched: numpy maps them lazily) are refused, not cut to their first 5"""
    _, fn = CALLS[call]
    with pytest.raises(ValueError):
        fn(np.empty(2 ** 31 + 5, dtype=np.uint8))
    with pytest.raises(ValueError, match="C int"):
        fn(np.empty((2, 2 ** 30 + 3), dtype=np.uint8))      # 2^31 + 6 bytes in 2 rows: a row count would have passed
    assert rec.calls == []


@pytest.mark.gpu
def test_a_2d_array_gives_the_oracles_result_on_its_bytes(oracle):
    """through the real library: a (64, 1024) array compresses and decodes as its 65 536 bytes, in blocks and frames"""
    import frame_oracle as fo
    data = oracle.datagen(68 * 1024, 0.5, 7)
    arr = data[:65536].reshape(64, 1024)
    flat = arr.tobytes()
    assert block.LZ4_compress_fast(arr) == oracle.compress(flat, 1)
    _, comp = oracle.compress(flat, 1)
    c2d = np.frombuffer(comp, dtype=np.uint8).reshape(1, -1)
    assert block.LZ4_decompress_safe(c2d, 65536) == oracle.decompress(comp, 65536) == (65536, flat)
    cols = data.reshape(68, 1024)[:, ::2]                       # non-contiguous: its bytes in C order
    assert block.LZ4_compress_fast(cols) == oracle.compress(cols.tobytes(), 1)
    f = frame.compress_frame(arr)
    assert f == fo.compress_frame(oracle, flat)
    assert frame.decompress_frame(np.frombuffer(f, dtype=np.uint8).reshape(2, -1) if len(f) % 2 == 0 else
                                  np.frombuffer(f, dtype=np.uint8).reshape(1, -1), 65536) == flat
