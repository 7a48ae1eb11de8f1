"""The host-buffer pipeline under the compress calls, on the GPU: LZ4B200_compress_blocks_host over more chunks than it
has pipeline slots, and LZ4B200_compressFrame_host over more than one 256 MiB group.

The host compress runs in a child process with 1 MiB chunks (LZ4B200_HOST_CHUNK_MB is read once per process), so that
every slot is reused and the short last block is in the last of many chunks.  The frame compress is checked byte for
byte against the Python frame restatement (tests/frame_oracle.py) into a destination of exactly
LZ4B200_compressFrameBound bytes, and decoded back by LZ4B200_decompressFrame_host.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import frame_oracle as fo

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
MiB = 1 << 20

# 1 MiB chunks of 65 600-byte source strides hold 15 blocks: 150 blocks are 10 chunks through the 4 slots
BS, SRC_STRIDE, N_BLOCKS, LAST = 65536, 65600, 150, 12345


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    assert lib.LZ4B200_device_count() > 0, "GPU tests need a CUDA device"
    return lib


def _host_compress_input(oracle):
    """N_BLOCKS blocks at SRC_STRIDE: datagen of three ratios, every 11th block incompressible"""
    src = np.zeros(N_BLOCKS * SRC_STRIDE, dtype=np.uint8)
    rng = np.random.default_rng(7)
    for i in range(N_BLOCKS):
        n = LAST if i == N_BLOCKS - 1 else BS
        blk = rng.integers(0, 256, n, dtype=np.uint8) if i % 11 == 3 else oracle.datagen(n, (0.2, 0.5, 0.9)[i % 3], 500 + i)
        src[i * SRC_STRIDE:i * SRC_STRIDE + n] = blk
    return src


def _host_compress(lib, src, cap):
    stride = (cap + 15) // 16 * 16
    slots = np.zeros(N_BLOCKS * stride, dtype=np.uint8)
    sizes = np.full(N_BLOCKS, -7, dtype=np.int32)
    rc = lib.LZ4B200_compress_blocks_host(src.ctypes.data, SRC_STRIDE, BS, LAST, slots.ctypes.data, stride, cap, 1,
                                          sizes.ctypes.data, N_BLOCKS)
    assert rc == 0, lib.LZ4B200_last_cuda_error()
    return sizes, [slots[i * stride:i * stride + max(int(r), 0)].tobytes() for i, r in enumerate(sizes)]


@pytest.mark.parametrize("cap", [65809, 40000])
def test_host_compress_over_many_chunks(lib, oracle, tmp_path, cap):
    """every return value and every block against the oracle, with 1 MiB chunks in a child process and with the default
    64 MiB chunk (one chunk) here; at the bound every block fits, at 40 000 bytes the incompressible ones return 0"""
    src = _host_compress_input(oracle)
    want = [oracle.compress(src[i * SRC_STRIDE:i * SRC_STRIDE + (LAST if i == N_BLOCKS - 1 else BS)], 1, cap)
            for i in range(N_BLOCKS)]
    assert (cap < 65809) == any(r == 0 for r, _ in want)
    env = dict(os.environ, LZ4B200_HOST_CHUNK_MB="1")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path), str(cap)], env=env, timeout=600,
                       capture_output=True, text=True)
    assert p.returncode == 0, (p.stdout[-2000:], p.stderr[-4000:])
    chunked = np.load(str(tmp_path / "sizes.npy")), np.load(str(tmp_path / "blocks.npy"), allow_pickle=True).tolist()
    for sizes, blocks in (chunked, _host_compress(lib, src, cap)):
        assert sizes.tolist() == [r for r, _ in want]
        for i, ((_, eout), out) in enumerate(zip(want, blocks)):
            assert out == eout, i


def _frame_input(oracle, n):
    """n bytes of datagen with incompressible stretches in the second 256 MiB group: every block of 64 KB and three of
    4 MB in them are stored raw"""
    d = oracle.datagen_mt(n, 4 * MiB, 0.5, 300)
    rng = np.random.default_rng(3)
    for lo, hi in ((264 * MiB, 276 * MiB), (280 * MiB + 1000, 280 * MiB + 300000)):
        d[lo:hi] = rng.integers(0, 256, hi - lo, dtype=np.uint8)
    return d


@pytest.mark.parametrize("bsid", [4, 7])
def test_frame_compress_over_several_groups(lib, oracle, bsid):
    n = 300 * 1000 * 1000 + 3
    bs = 1 << (8 + 2 * bsid)
    assert -(-n // bs) > (256 * MiB) // bs                 # more blocks than one group holds
    d = _frame_input(oracle, n)
    want = fo.compress_frame(oracle, d, bsid, 0, True)
    cap = int(lib.LZ4B200_compressFrameBound(n, bsid))
    dst = np.zeros(cap, dtype=np.uint8)
    r = int(lib.LZ4B200_compressFrame_host(d.ctypes.data, n, dst.ctypes.data, cap, bsid, 0, 1))
    assert r == len(want), (r, len(want), lib.LZ4B200_last_cuda_error())
    assert dst[:r].tobytes() == want
    raw = sum(1 for _ in _raw_blocks(want))
    assert raw >= (3 if bsid == 7 else 192), raw
    back = np.zeros(n, dtype=np.uint8)
    used = C.c_int64(-1)
    assert int(lib.LZ4B200_decompressFrame_host(dst.ctypes.data, r, back.ctypes.data, n, C.byref(used))) == n
    assert used.value == r and np.array_equal(back, d)


def _raw_blocks(frame):
    """offsets of the stored-raw blocks of a frame with a content-size field"""
    ip = 15
    while True:
        h = int.from_bytes(frame[ip:ip + 4], "little")
        if h == 0:
            return
        if h >> 31:
            yield ip
        ip += 4 + (h & 0x7FFFFFFF)


def child_main(d, cap):
    sys.path[:0] = [os.path.dirname(HERE), HERE]
    from lz4_b200 import _lib
    from oracle.pyoracle import Oracle
    sizes, blocks = _host_compress(_lib.load(), _host_compress_input(Oracle()), cap)
    np.save(os.path.join(d, "sizes.npy"), sizes)
    np.save(os.path.join(d, "blocks.npy"), np.array(blocks, dtype=object), allow_pickle=True)


if __name__ == "__main__":
    child_main(sys.argv[1], int(sys.argv[2]))
