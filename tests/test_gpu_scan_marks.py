"""The marks the scan kernels leave in the workspace, on the GPU, word for word against the host build of the same scan.

The scans write a block's marks in whole 32-byte chunks and the words of a chunk they do not own one by one
(MarkSink, lz4_scan_core.h).  A lost or misplaced word only shows when the rows kernel expands that block, and not at
all when the block goes to the generic kernel; so these tests read the narrow marks table back from the workspace:
  R3  > 8 192 blocks of one capacity in [16 KB, 64 KB]: one-thread scan; every word of every block's table
      (markStride words, sentinels included) equals what the host scan leaves, for rejected blocks too;
  R2  <= 8 192 blocks: split scan; accepted blocks' marks equal the host scan's;
  R4  capacities below 16 KB (markStride = cap / 4 + 2: tables start at every word of a chunk): as R3.
Blocks sit at all 16 source phases; the corpus is gpu_util.hostile_corpus plus datagen blocks.  Return values and
bytes are checked against the oracle, the sequence counts against the host scan."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from gpu_util import dev, hostile_corpus, to_dev

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SENT = 0xEEEEEEEE


@pytest.fixture(scope="module")
def host_scan(tmp_path_factory):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("scanmarks") / "libscanmarks.so")
    subprocess.run([gxx, "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-o", so,
                    os.path.join(HERE, "emul", "scan_marks_emul.cpp")], check=True)
    lib = C.CDLL(so)
    lib.scan_host_cap.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_uint32), C.c_void_p, C.c_uint32]
    memo = {}

    def run(block, cap, stride):
        """-> (ret, nseq, the block's table of `stride` words as the host scan leaves it in a table of sentinels)"""
        key = (block, cap, stride)
        if key not in memo:
            n = len(block)
            buf = np.full(n + 64, 0xEE, dtype=np.uint8)
            pad = (-buf.ctypes.data) % 16 + 16
            buf[pad:pad + n] = np.frombuffer(block, dtype=np.uint8)
            table = np.full(stride + 8, SENT, dtype=np.uint32)
            has_marks = 0 < n <= 65535 and 0 < cap <= 65536          # block_marks (lz4_decode_plan.h)
            ns = C.c_uint32(0)
            r = lib.scan_host_cap(buf.ctypes.data + pad, n, cap, C.byref(ns), table.ctypes.data if has_marks else None, stride)
            memo[key] = (r, ns.value, table[:stride].copy())
        return memo[key]
    return run


def narrow_workspace(ws, n, stride):
    """nSeq[n] and the narrow marks tables (n x stride words) of a workspace (plan_layout, lz4_decode_plan.h): a 256-byte
    header, nSeq[n], slowList[n] (each rounded up to 256 bytes), then the marks"""
    r256 = lambda x: (x + 255) // 256 * 256
    w = ws.cpu().numpy().view(np.uint32)
    lst = r256(n * 4)
    m0 = (256 + 2 * lst) // 4
    return w[64:64 + n].copy(), w[m0:m0 + n * stride].reshape(n, stride)


def decode_phases(blocks, cap):
    """Scan, then expand, a batch of one capacity with block i at byte i % 16 of a 16-byte granule.  The workspace
    starts as sentinel words and is read back between the two phases.  -> (rets, outputs, nSeq, marks tables)"""
    from lz4_b200 import _lib
    lib = _lib.load()
    n = len(blocks)
    offs = np.zeros(n, dtype=np.int64)
    pos = 16
    for i, b in enumerate(blocks):
        pos += (i % 16 - pos) % 16
        offs[i] = pos
        pos += len(b)
    src = np.zeros(pos + 32, dtype=np.uint8)
    for o, b in zip(offs, blocks):
        src[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    sizes = np.array([len(b) for b in blocks], dtype=np.int32)
    stride = (cap + 64 + 15) // 16 * 16
    d_src, d_offs, d_sizes = to_dev(src), to_dev(offs), to_dev(sizes)
    d_out = torch.zeros(n * stride, dtype=torch.uint8, device=dev())
    d_ret = torch.zeros(n, dtype=torch.int32, device=dev())
    ws_bytes = int(lib.LZ4B200_decompress_workspace_bytes_for(n, 0, cap))
    ws = torch.full((ws_bytes,), 0xEE, dtype=torch.uint8, device=dev())
    args = (d_src.data_ptr(), d_offs.data_ptr(), d_sizes.data_ptr(), d_out.data_ptr(), None, stride, None, cap,
            d_ret.data_ptr(), n, ws.data_ptr(), ws_bytes)
    s = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.LZ4B200_decompress_blocks_phased(*args, 1, s), "scan")
    torch.cuda.synchronize()
    mark_stride = min(cap // 4 + 2, 8192)
    nseq, marks = narrow_workspace(ws, n, mark_stride)
    _lib.check(lib.LZ4B200_decompress_blocks_phased(*args, 2, s), "expand")
    torch.cuda.synchronize()
    out = d_out.cpu().numpy().reshape(n, stride)
    return d_ret.cpu().numpy(), out, nseq, marks, mark_stride


def corpus(oracle, cap, n, seed):
    """hostile_corpus(cap) and datagen blocks of cap bytes, repeated to n blocks"""
    blocks = [bytes(b) for _, b in hostile_corpus(oracle, cap, seed=seed, n_corrupt=2)]
    for k in range(24):
        _, c = oracle.compress(oracle.datagen(cap, (0.3, 0.5, 0.7)[k % 3], 100 + k + seed), 1)
        blocks.append(bytes(c))
    rng = np.random.default_rng(seed)
    return [blocks[i] for i in np.resize(rng.permutation(len(blocks)), n)]


def check(oracle, host_scan, blocks, cap, whole_table):
    rets, out, nseq, marks, mark_stride = decode_phases(blocks, cap)
    memo = {}
    accepted = rejected = 0
    for i, b in enumerate(blocks):
        if (b, cap) not in memo:
            memo[(b, cap)] = oracle.decompress(b, cap)
        eret, eout = memo[(b, cap)]
        assert rets[i] == eret, (i, len(b), cap, int(rets[i]), eret)
        hr, hns, htable = host_scan(b, cap, mark_stride)
        assert hr == eret
        assert nseq[i] == hns, (i, int(nseq[i]), hns)
        if eret > 0:
            accepted += 1
            assert out[i, :eret].tobytes() == eout, (i, len(b), cap)
        else:
            rejected += 1
        if whole_table:
            assert (marks[i] == htable).all(), (i, len(b), cap, eret, int(np.argmax(marks[i] != htable)))
        elif eret > 0:
            k = min(hns, mark_stride) if 0 < len(b) <= 65535 else 0
            assert (marks[i, :k] == htable[:k]).all(), (i, len(b), cap, int(np.argmax(marks[i, :k] != htable[:k])))
    assert accepted > 0 and rejected > 0


def test_one_thread_scan_large_batch(oracle, host_scan):
    """R3: 8 200 blocks of 64 KB capacity (markStride 8 192)"""
    check(oracle, host_scan, corpus(oracle, 65536, 8200, 1), 65536, whole_table=True)


def test_one_thread_scan_odd_stride(oracle, host_scan):
    """R3 with a capacity of 20 000 (markStride 5 002: tables start at every other word of a chunk)"""
    check(oracle, host_scan, corpus(oracle, 20000, 8300, 2), 20000, whole_table=True)


def test_split_scan(oracle, host_scan):
    """R2: the split scan's lanes share chunks at the edges of their parts"""
    for cap, seed in ((65536, 3), (16384, 4), (20000, 5)):
        check(oracle, host_scan, corpus(oracle, cap, 1500, seed), cap, whole_table=False)


@pytest.mark.parametrize("cap", [1000, 4097, 16383])
def test_small_capacities(oracle, host_scan, cap):
    """R4: markStride = cap / 4 + 2 = 252, 1 026, 4 097"""
    check(oracle, host_scan, corpus(oracle, cap, 2000, cap), cap, whole_table=True)
