"""LZ4B200_decompress_files_host on the GPU: every file of tests/golden/decompress_files.json in both checksum modes and
the size-only pass against LZ4B200_decompress_files (with a budget that covers them all) and the Python model, with guard
bytes around every output region at exact capacity and one byte less; the same corpus and long frames, a legacy stream,
late corruptions and a frame of blocks just short of 64 KB in a child process with 1 MiB groups, so that every pipeline
slot is reused, frame, unit and file boundaries fall on group edges and a carried content hash has a partial stripe; at the default group size a 1 GiB frame of 4 MB blocks and one of 64 KB blocks,
20 000 small files in one call and outputs past 2^32 in one buffer; the single-frame files against
LZ4B200_decompressFrame_host; device memory over repeated calls; four threads beside LZ4B200_decompress_blocks_host;
and the Python wrappers."""
import ctypes as C
import hashlib
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if __name__ == "__main__":
    sys.path[:0] = [os.path.dirname(HERE), HERE]

import decompress_files_model as dm                      # noqa: E402
from lz4_b200 import batch, frame                        # noqa: E402

pytestmark = pytest.mark.gpu

GUARD, GAP = 0xA5, 40
MIB = 1 << 20
ERR_CHECKSUM, ERR_DSTSIZE = -7, -5


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def oracle():
    from oracle.pyoracle import Oracle
    return Oracle()


def golden_files(oracle):
    import json
    with open(os.path.join(HERE, "golden", "decompress_files.json")) as f:
        g = json.load(f)["files"]
    return g, [dm.build_file(oracle, c) for c in g]


@pytest.fixture(scope="module")
def corpus(oracle):
    return golden_files(oracle)


def host_call(lib, files, caps, skip=False, size_only=False, out=None, oo=None):
    """the call on files packed in one host buffer, outputs GAP guard bytes apart: (results, consumed, prefixes, out,
    output offsets); out and oo may be given (a caller's buffer and offsets)"""
    sizes = np.array([len(f) for f in files], dtype=np.int64)
    offs = np.zeros(len(files), dtype=np.int64)
    offs[1:] = np.cumsum(sizes)[:-1]
    src = np.frombuffer(b"".join(files) or b"\0", dtype=np.uint8)
    n = len(files)
    res, con, pre = (np.full(n, -99, dtype=np.int64) for _ in range(3))
    capa = np.array(caps, dtype=np.int64)
    if out is None and not size_only:
        oo = np.zeros(n, dtype=np.int64)
        at = GAP
        for k, c in enumerate(caps):
            oo[k] = at
            at += max(c, 0) + GAP
        out = np.full(at, GUARD, dtype=np.uint8)
    p = lambda a: None if a is None else a.ctypes.data
    rc = lib.LZ4B200_decompress_files_host(src.ctypes.data, offs.ctypes.data, sizes.ctypes.data,
                                           None if size_only else p(out), None if size_only else p(oo),
                                           None if size_only else p(capa), res.ctypes.data, con.ctypes.data,
                                           pre.ctypes.data, n, 1 if skip else 0, 1 if size_only else 0)
    assert rc == 0, (rc, lib.LZ4B200_last_cuda_error())
    return res.tolist(), con.tolist(), pre.tolist(), out, oo


def device_call(files, caps, skip=False, size_only=False):
    """LZ4B200_decompress_files on the same files with the budget that covers them all: results, consumed, prefixes and
    each file's output bytes up to its prefix"""
    buf, offs = bytearray(), []
    for f in files:
        buf += b"\0" * ((-len(buf)) % 16)
        offs.append(len(buf))
        buf += f
    buf += b"\0" * 16
    comp = torch.frombuffer(buf, dtype=torch.uint8).cuda()
    d = lambda a: torch.tensor(list(a), dtype=torch.int64, device="cuda")
    mu, mb = dm.budget_needed(files, skip)
    if size_only:
        res, con, pre = batch.decompressed_file_sizes(comp, d(offs), d(len(f) for f in files), mu, mb, skip)
        return res.tolist(), con.tolist(), pre.tolist(), None
    oo, at = [], 0
    for c in caps:
        oo.append(at)
        at += max(c, 0)
    out = torch.zeros(max(at, 1), dtype=torch.uint8, device="cuda")
    _, res, con, pre = batch.decompress_files(comp, d(offs), d(len(f) for f in files), d(caps), mu, mb, skip, out=out,
                                              out_offsets=d(oo))
    h = out.cpu().numpy()
    pre = pre.tolist()
    return res.tolist(), con.tolist(), pre, [h[o:o + p].tobytes() for o, p in zip(oo, pre)]


def sized_caps(files, skip=False):
    """each file's room: its decoded size from the device call's size-only pass, or its prefix + 64 KiB when it fails"""
    res, _, pre, _ = device_call(files, None, skip, size_only=True)
    return [r if r >= 0 else p + (1 << 16) for r, p in zip(res, pre)]


def check_against_device(lib, files, caps, skip, size_only=False):
    """the host call equals the device call; guard bytes outside every region untouched.  Returns the host results."""
    res, con, pre, out, oo = host_call(lib, files, caps, skip, size_only)
    dres, dcon, dpre, dbytes = device_call(files, caps, skip, size_only)
    assert (res, con, pre) == (dres, dcon, dpre)
    if not size_only:
        for k, c in enumerate(caps):
            o, c = int(oo[k]), max(c, 0)
            assert out[o:o + pre[k]].tobytes() == dbytes[k], k
            assert (out[o - GAP:o] == GUARD).all() and (out[o + c:o + c + GAP] == GUARD).all(), k
    return res, con, pre, out, oo


@pytest.mark.parametrize("mode", ["verify", "skip"])
def test_golden_files(lib, corpus, oracle, mode):
    g, files = corpus
    skip = mode == "skip"
    mu, mb = dm.budget_needed(files, skip)
    sized = dm.decompress_files(oracle, files, [1 << 40] * len(files), mu, mb, skip)
    exact = [r if r >= 0 else p + (1 << 16) for r, _, p, _ in sized]
    for caps in (exact, [e - 1 if e > 0 else 0 for e in exact]):
        res, con, pre, out, oo = check_against_device(lib, files, caps, skip)
        want = dm.decompress_files(oracle, files, caps, mu, mb, skip)
        for k, (r, at, p, b) in enumerate(want):
            assert (res[k], con[k], pre[k]) == (r, at, p), (g[k]["name"], (res[k], con[k], pre[k]), (r, at, p))
            assert out[int(oo[k]):int(oo[k]) + p].tobytes() == b, g[k]["name"]
    for c, (r, _, p, b) in zip(g, sized):                 # the tool's bytes, where the model has no deviation
        if c[mode]["exit"] == 0 and r >= 0:
            assert sha(b) == c[mode]["sha256"], c["name"]
    res, con, pre, _ = host_call(lib, files, exact, skip, size_only=True)[:4]
    nocontent = dm.decompress_files(oracle, files, exact, mu, mb, skip, size_only=True)
    assert (res, con, pre) == tuple([w[i] for w in nocontent] for i in range(3))
    assert (res, con, pre) == tuple(device_call(files, exact, skip, size_only=True)[:3])


def late_corruptions(frame):
    """the 40 MiB frame (64 KB blocks, block and content checksums) with its last block's checksum, a byte of its
    payload, and its content checksum flipped: [payload][block sum][EndMark][content sum] end the frame"""
    out = []
    for at in (len(frame) - 10, len(frame) - 20, len(frame) - 1):
        b = bytearray(frame)
        b[at] ^= 0x20
        out.append(bytes(b))
    return out


SHORT_BLOCKS = [65536 - 1 - k % 15 for k in range(40)]


def short_blocks_frames(oracle, data):
    """a frame with block and content checksums of blocks of SHORT_BLOCKS bytes, three stored raw, so that the group
    edges inside it fall after content that is not a multiple of 16 bytes; then the same frame with its content
    checksum flipped"""
    ends = np.cumsum(SHORT_BLOCKS)
    pieces = [data[e - n:e] for e, n in zip(ends, SHORT_BLOCKS)]
    frame = dm.fm.frame_of_blocks(oracle, pieces, 4, raw=(3, 17, 30), block_sum=True, content_sum=True)
    bad = bytearray(frame)
    bad[-1] ^= 1
    return [frame, bytes(bad)]


def chunked_files(oracle):
    """the corpus, then files whose frames, units and blocks cross 1 MiB group edges"""
    _, files = golden_files(oracle)
    data = oracle.datagen(40 * MIB, 0.5, 21).tobytes()
    big = dm.fm.compress_frame(oracle, data, 4, False, 1, 1)
    leg = dm.legacy(lambda b: oracle.compress(b, 1)[1], data[:20 * MIB + 1]) + \
        dm.fm.compress_frame(oracle, data[:300000], 5, True, 1, 1)
    mixed = b"".join(dm.fm.compress_frame(oracle, data[k * 70000:(k + 1) * 70000 + k], 4 + k % 4, k % 2 == 0, k % 3 == 0,
                                          k % 2 == 1) + dm.skippable(b"s" * k, k % 16) for k in range(40))
    return files + [big, leg, mixed] + late_corruptions(big) + short_blocks_frames(oracle, data) + files[:20]


def chunked_results(lib, files):
    got = []
    for skip in (False, True):
        caps = sized_caps(files, skip)
        res, con, pre, out, oo = host_call(lib, files, caps, skip)
        got.append([res, con, pre, [sha(out[int(o):int(o) + p]) for o, p in zip(oo, pre)]])
        got.append(list(host_call(lib, files, caps, skip, size_only=True)[:3]))
    return got


def child_main(d):
    from lz4_b200 import _lib
    from oracle.pyoracle import Oracle
    import json
    with open(os.path.join(d, "chunked.json"), "w") as f:
        json.dump(chunked_results(_lib.load(), chunked_files(Oracle())), f)


def test_one_mib_groups_in_a_child(lib, oracle, tmp_path):
    import json
    env = dict(os.environ, LZ4B200_HOST_CHUNK_MB="1")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path)], env=env, timeout=1200,
                       capture_output=True, text=True)
    assert p.returncode == 0, (p.stdout[-2000:], p.stderr[-4000:])
    with open(str(tmp_path / "chunked.json")) as f:
        got = json.load(f)
    files = chunked_files(oracle)
    k = 0
    for skip in (False, True):
        caps = sized_caps(files, skip)
        dres, dcon, dpre, dbytes = device_call(files, caps, skip)
        assert got[k][:3] == [dres, dcon, dpre]
        assert got[k][3] == [sha(b) for b in dbytes]
        assert got[k + 1] == list(device_call(files, caps, skip, size_only=True)[:3])
        k += 2
        n = len(files) - 20 - 5
        if not skip:                                      # the late corruptions fail with a checksum error: the
            sres = got[k - 1][0]                          # block ones in the size-only pass, the content ones decoding
            assert dres[n - 3:n] == [40 * MIB, 20 * MIB + 1 + 300000, dres[n - 1]] and dres[n - 1] > 0
            assert sres[n:n + 2] == [ERR_CHECKSUM] * 2 and dres[n + 2] == ERR_CHECKSUM, (sres[n:n + 3], dres[n:n + 3])
            assert dres[n + 3:n + 5] == [sum(SHORT_BLOCKS), ERR_CHECKSUM], dres[n + 3:n + 5]


def gpu_frame(data, bsid):
    """one frame of data with block and content checksums, written by compress_frames_checksummed"""
    src = torch.from_numpy(data).cuda()
    z = torch.zeros(1, dtype=torch.int64, device="cuda")
    out, res = batch.compress_frames_checksummed(src, z, z + len(data), block_size_id=bsid, block_checksum=True,
                                                 content_checksum=True)
    torch.cuda.synchronize()
    f = out[:int(res[0])].cpu().numpy().tobytes()
    del src, out
    return f


@pytest.mark.parametrize("bsid", [7, 4])
def test_one_gib_frame(lib, oracle, bsid):
    data = oracle.datagen_mt(1 << 30, 1 << 20, 0.5, 30 + bsid)
    f = gpu_frame(data, bsid)
    assert f[4] & 0x14 == 0x14                           # block and content checksums
    for skip in (False, True):
        res, con, pre, out, oo = host_call(lib, [f], [1 << 30], skip)
        assert (res, con, pre) == ([1 << 30], [len(f)], [1 << 30])
        assert np.array_equal(out[GAP:GAP + (1 << 30)], data)
        assert (out[:GAP] == GUARD).all() and (out[GAP + (1 << 30):] == GUARD).all()
    bad = bytearray(f)
    bad[-1] ^= 1
    assert host_call(lib, [bytes(bad)], [1 << 30])[0] == [ERR_CHECKSUM]
    assert host_call(lib, [bytes(bad)], [1 << 30], skip=True)[0] == [1 << 30]


def test_many_small_files(lib, oracle):
    n = 20000
    data = oracle.datagen(3 * MIB, 0.5, 4).tobytes()
    files, want = [], []
    for k in range(n):
        w = data[k * 97:k * 97 + 100 + k % 3000]
        want.append(w)
        files.append(dm.fm.compress_frame(oracle, w, 4 + k % 4, k % 2 == 0, k % 3 == 0, k % 5 != 0))
    res, con, pre, out, oo = host_call(lib, files, [len(w) for w in want])
    assert res == [len(w) for w in want] and con == [len(f) for f in files]
    for k in range(0, n, 7):
        assert out[int(oo[k]):int(oo[k]) + len(want[k])].tobytes() == want[k], k
    assert all((out[int(o) - GAP:int(o)] == GUARD).all() for o in oo[::101])
    res2 = frame.decompress_files(files[:300])
    assert [r for r, _, _, _ in res2] == [len(w) for w in want[:300]] and [b for _, _, _, b in res2] == want[:300]


def test_outputs_past_4gib(lib, oracle):
    d = oracle.datagen(300000, 0.5, 5).tobytes()
    files = [dm.fm.compress_frame(oracle, d, 5, True, 1, 1), dm.legacy(lambda b: oracle.compress(b, 1)[1], d),
             dm.skippable(b"abc") + dm.fm.compress_frame(oracle, d[:1000], 4, False, 0, 1)]
    total = (1 << 32) + (1 << 20)
    out = np.full(total, GUARD, dtype=np.uint8)
    oo = np.array([(1 << 32) - 7, (1 << 31) + 3, (1 << 32) + 500000], dtype=np.int64)
    caps = [300000, 300000, 1000]
    res, con, pre, out, _ = host_call(lib, files, caps, out=out, oo=oo)
    assert res == [300000, 300000, 1000] and con == [len(f) for f in files]
    for o, c, want in zip(oo, caps, [d, d, d[:1000]]):
        assert out[o:o + c].tobytes() == want
        assert out[o - 1] == GUARD and out[o + c] == GUARD


def test_single_frames_match_the_frame_host_call(lib, corpus):
    g, files = corpus
    n = 0
    for c, f in zip(g, files):
        src = np.frombuffer(f or b"\0", dtype=np.uint8)
        cap = sized_caps([f])[0] + 1000
        dst = np.zeros(cap, dtype=np.uint8)
        used = C.c_int64(-1)
        r = int(lib.LZ4B200_decompressFrame_host(src.ctypes.data, len(f), dst.ctypes.data, cap, C.byref(used)))
        if r < 0 or used.value != len(f):
            continue
        res, con, pre, out, oo = host_call(lib, [f], [cap])
        assert res == [r] and out[GAP:GAP + r].tobytes() == dst[:r].tobytes(), c["name"]
        n += 1
    assert n >= 5


def test_device_memory_does_not_grow(lib, corpus):
    _, files = corpus
    caps = sized_caps(files)
    host_call(lib, files, caps)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(5):
        host_call(lib, files, caps)
        host_call(lib, files, caps, size_only=True)
    assert torch.cuda.mem_get_info()[0] >= free0


def test_threads_beside_the_blocks_call(lib, corpus, oracle):
    _, files = corpus
    caps = sized_caps(files)
    serial = host_call(lib, files, caps)[:3]
    blocks = [oracle.compress(oracle.datagen(65536, 0.5, k).tobytes(), 1)[1] for k in range(64)]
    sizes = np.array([len(b) for b in blocks], dtype=np.int32)
    offs = np.zeros(64, dtype=np.int64)
    offs[1:] = np.cumsum(sizes)[:-1]
    src = np.frombuffer(b"".join(blocks) + b"\0" * 16, dtype=np.uint8)
    errors = []

    def files_worker():
        for _ in range(3):
            if host_call(lib, files, caps)[:3] != serial:
                errors.append("files")

    def blocks_worker():
        for _ in range(3):
            out = np.zeros(64 * 65536, dtype=np.uint8)
            rets = np.zeros(64, dtype=np.int32)
            rc = lib.LZ4B200_decompress_blocks_host(src.ctypes.data, offs.ctypes.data, sizes.ctypes.data, out.ctypes.data,
                                                    65536, 65536, rets.ctypes.data, 64)
            if rc != 0 or (rets != 65536).any():
                errors.append("blocks")

    ts = [threading.Thread(target=files_worker) for _ in range(4)] + [threading.Thread(target=blocks_worker) for _ in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert errors == []


def test_python_wrappers(lib, oracle):
    d = oracle.datagen(500000, 0.5, 8).tobytes()
    f = dm.fm.compress_frame(oracle, d, 5, False, 1, 1)
    assert frame.decompress_file(f) == d
    assert frame.decompress_file(np.frombuffer(f, dtype=np.uint8).reshape(1, -1), len(d)) == d
    with pytest.raises(frame.Lz4FrameError) as e:
        frame.decompress_file(f, len(d) - 1)
    assert e.value.code == ERR_DSTSIZE
    bad = bytearray(f)
    bad[-1] ^= 1
    with pytest.raises(frame.Lz4FrameError) as e:
        frame.decompress_file(bytes(bad))
    assert e.value.code == ERR_CHECKSUM
    assert frame.decompress_file(bytes(bad), skip_checksums=True) == d
    two = f + dm.skippable(b"zz") + dm.legacy(lambda b: oracle.compress(b, 1)[1], d[:1000])
    assert frame.decompress_files([two, b""], size_only=True) == [(len(d) + 1000, len(two), len(d) + 1000, None),
                                                                  (0, 0, 0, None)]
    # a file whose first frame fails its content checksum and whose second frame is cut short: at unlimited room the
    # content checksum comes first
    cut = bytes(bad) + f[:-30]
    (r, c, p, b), = frame.decompress_files([cut])
    assert (r, c, p, b) == (ERR_CHECKSUM, 0, 0, b"")
    (r, c, p, b), = frame.decompress_files([f + f[:-30]])
    assert (r, c, p) == (-3, len(f), len(d)) and b == d


if __name__ == "__main__":
    child_main(sys.argv[1])
