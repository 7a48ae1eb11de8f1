"""LZ4B200_compress_blocks_indexed, LZ4B200_pack_blocks_indexed and their Python wrappers on the GPU.

Every block of an indexed call must come out as the matching one-block call makes it: LZ4_compress_fast (the oracle),
the parallel parse (tests/encpar_model.py, LZ4_compress_fast above 64 KB) or LZ4_compress_HC (the host build of the HC
parses, tests/hc_emul.py).  Sources sit in one arena at shuffled offsets of every 16-byte phase; outputs are packed
back to back, each region exactly its capacity, with guard bytes before the first and after the last, so that a byte
written outside [dst_i, dst_i + cap_i) lands in a neighbour or a guard and shows.

HC blocks stop at 200 000 bytes: one thread parses a block, so a 4 MB block takes tens of seconds at any level
(DESIGN section 5).  The 4 MB blocks run through PARSE_FAST and PARSE_PARALLEL.
"""
import numpy as np
import pytest
import torch

import encpar_model as M
from gpu_util import Recorder, pack_model
from hc_emul import host_hc, host_hc_opt

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
FAST, PARALLEL, HC = 0, 1, 2
PARSE_NAME = {FAST: "fast", PARALLEL: "parallel", HC: "hc"}
GUARD = 0xA5
MiB, GiB = 1 << 20, 1 << 30
L31, L32 = 1 << 31, 1 << 32
MAX_INPUT = 0x7E000000
SIZES = [0, 1, 12, 13, 14, 4096, 65535, 65536, 65537, 65546, 65547, 200000, 4 << 20]
HC_SIZES = [s for s in SIZES if s <= 200000]
CASES = [(FAST, 1), (FAST, 9), (FAST, 65537), (PARALLEL, 1), (PARALLEL, 5), (PARALLEL, 13),
         (HC, 1), (HC, 2), (HC, 3), (HC, 9), (HC, 10), (HC, 12)]


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    assert lib.LZ4B200_device_count() > 0, "GPU tests need a CUDA device"
    yield lib
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def bound(n):
    return n + n // 255 + 16 if 0 <= n <= MAX_INPUT else 0


def expected(oracle, parse, param, data, cap):
    """(return value, bytes) of the one-block call block i must match"""
    data = bytes(data)
    if parse == FAST:
        return oracle.compress(data, param, cap)
    if parse == PARALLEL:
        r = M.compress(data, param, cap, oracle)
        return r.ret, (bytes(r.out[:r.ret]) if r.ret > 0 else b"")
    return (host_hc_opt if param >= 10 else host_hc)(data, cap, param)


def payloads(oracle, sizes, seed):
    """per size one datagen P50 block and one of random bytes (the second does not fit below its bound)"""
    rng = np.random.default_rng(seed)
    out = []
    for k, n in enumerate(sizes):
        out.append(oracle.datagen(n, 0.5, seed + k) if n else np.zeros(0, np.uint8))
        out.append(rng.integers(0, 256, n, dtype=np.uint8))
    return out


def place_sources(datas, seed, pad=64):
    """datas in one arena at shuffled, non-monotone offsets; the k-th placed block has phase k mod 16.  Returns
    (host arena, offsets)"""
    rng = np.random.default_rng(seed)
    offs = np.zeros(len(datas), np.int64)
    pos = pad
    for k, i in enumerate(rng.permutation(len(datas))):
        pos = (pos + 15) // 16 * 16 + k % 16
        offs[i] = pos
        pos += len(datas[i]) + int(rng.integers(1, 40))
    arena = np.full(pos + pad, 0x3C, np.uint8)
    for i, d in enumerate(datas):
        arena[offs[i]:offs[i] + len(d)] = d
    return arena, offs


def abutting(caps, head=37, tail=61):
    """output offsets packed back to back (dstOff[i+1] = dstOff[i] + cap_i, a capacity below 0 taking no room) after
    `head` guard bytes; returns (offsets, bytes of the output buffer with `tail` guard bytes after the last)"""
    room = np.maximum(np.asarray(caps, np.int64), 0)
    offs = head + np.concatenate([[0], np.cumsum(room)[:-1]]).astype(np.int64)
    return offs, int(head + room.sum() + tail)


def t(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to(DEV)


def run_indexed(lib, src, soff, sizes, dst, doff, caps, parse, param, ws=None):
    """one LZ4B200_compress_blocks_indexed on the current stream (src, dst: u8 tensors or device pointers; the tables
    host arrays); returns the out sizes (a device tensor)"""
    n = len(sizes)
    soff_t, size_t, doff_t, cap_t = t(soff, np.int64), t(sizes, np.int32), t(doff, np.int64), t(caps, np.int32)
    out = torch.full((max(n, 1),), -99, dtype=torch.int32, device=DEV)
    if parse == HC and ws is None:
        ws = torch.empty(max(int(lib.LZ4B200_compress_blocks_indexed_workspace_bytes(n, parse, param)), 1),
                         dtype=torch.uint8, device=DEV)
    sp = src.data_ptr() if isinstance(src, torch.Tensor) else src
    dp = dst.data_ptr() if isinstance(dst, torch.Tensor) else dst
    rc = lib.LZ4B200_compress_blocks_indexed(sp, soff_t.data_ptr(), size_t.data_ptr(), dp, doff_t.data_ptr(),
                                             cap_t.data_ptr(), out.data_ptr(), n, parse, param,
                                             ws.data_ptr() if ws is not None else None,
                                             ws.numel() if ws is not None else 0, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rc
    return out[:n]


def check_outputs(out_h, doff, caps, got, want, what=""):
    """block i's return value and bytes; every byte outside the blocks' results is the guard -- except the rest of the
    region of a block that returned 0, which the call may have written"""
    ref = np.full(len(out_h), GUARD, np.uint8)
    care = np.ones(len(out_h), bool)
    for i, (r, b) in enumerate(want):
        assert int(got[i]) == r, "%sblock %d: returned %d, expected %d" % (what, i, int(got[i]), r)
        o = int(doff[i])
        ref[o:o + len(b)] = np.frombuffer(b, np.uint8)
        if r <= 0:
            care[o:o + max(int(caps[i]), 0)] = False
    bad = np.flatnonzero((out_h != ref) & care)
    if len(bad):
        at = int(bad[0])
        owner = [i for i in range(len(doff)) if doff[i] <= at < doff[i] + max(int(caps[i]), 0)]
        raise AssertionError("%sbyte %d is %d, want %d (%d bytes differ; region of block %s)" % (
            what, at, out_h[at], ref[at], len(bad), owner or "none: a guard"))


def run_layout(lib, oracle, parse, param, datas, caps, seed, sizes=None):
    """the whole check of one indexed call: sources placed by place_sources, outputs abutting"""
    arena, soff = place_sources(datas, seed)
    sizes = [len(d) for d in datas] if sizes is None else sizes
    doff, total = abutting(caps)
    src = t(arena)
    dst = torch.full((total,), GUARD, dtype=torch.uint8, device=DEV)
    got = run_indexed(lib, src, soff, sizes, dst, doff, caps, parse, param).cpu().numpy()
    want = [expected(oracle, parse, param, d, c) if 0 <= s <= MAX_INPUT else (0, b"")
            for d, c, s in zip(datas, caps, sizes)]
    check_outputs(dst.cpu().numpy(), doff, caps, got, want, "%s %d: " % (PARSE_NAME[parse], param))


# ------------------------------------------------------------------------------------------
# 1, 2. every parse at mixed sizes and capacities
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("parse,param", CASES, ids=["%s-%d" % (PARSE_NAME[p], q) for p, q in CASES])
def test_mixed_sizes_at_the_bound(lib, oracle, parse, param):
    """every size of SIZES twice (P50 and random bytes), each at its bound, plus a size of -1 and one past
    LZ4_MAX_INPUT_SIZE (both return 0 without reading their source)"""
    datas = payloads(oracle, HC_SIZES if parse == HC else SIZES, 11 * param + parse)
    caps = [bound(len(d)) for d in datas]
    sizes = [len(d) for d in datas] + [-1, MAX_INPUT + 1]
    datas += [np.zeros(0, np.uint8)] * 2
    caps += [40, 17]
    run_layout(lib, oracle, parse, param, datas, caps, seed=param, sizes=sizes)


CAP_SIZES = [0, 1, 13, 14, 4096, 65536, 65537, 65547, 200000]


@pytest.mark.parametrize("parse,param", CASES, ids=["%s-%d" % (PARSE_NAME[p], q) for p, q in CASES])
def test_capacities_around_the_result(lib, oracle, parse, param):
    """each block at {bound, r, r - 1, len - 1, 16, 15, 1, 0, -1} around its result r at the bound, mixed in one batch:
    limited and unlimited blocks side by side, outputs that fill their region exactly next to failed ones"""
    sizes = [s for s in CAP_SIZES if parse != HC or s <= 65547]
    base = payloads(oracle, sizes, 7 + param)
    datas, caps = [], []
    for d in base:
        n = len(d)
        r = expected(oracle, parse, param, d, bound(n))[0]
        for c in (bound(n), r, r - 1, n - 1, 16, 15, 1, 0, -1):
            datas.append(d)
            caps.append(c)
    order = np.random.default_rng(param).permutation(len(datas))
    run_layout(lib, oracle, parse, param, [datas[i] for i in order], [caps[i] for i in order], seed=3 + param)


# ------------------------------------------------------------------------------------------
# 3. a strided layout given as offsets is the strided call
# ------------------------------------------------------------------------------------------
STRIDED = {"compress_blocks": (FAST, 1), "parallel": (PARALLEL, 1), "hc": (HC, 9), "hc_opt": (HC, 10)}


@pytest.mark.parametrize("call", list(STRIDED))
@pytest.mark.parametrize("block", [4096, 65536, 100000])
def test_strided_layout_as_offsets(lib, oracle, call, block):
    """n blocks at srcStride / dstStride with one capacity and a short last block: same bytes, sizes and launch count as
    the strided call"""
    parse, param = STRIDED[call]
    n = 24 if parse != HC else 8
    total = n * block - block // 3
    data = oracle.datagen(total, 0.5, block)
    src_stride, dst_stride = block + 16 * 3 + 5, bound(block) + 29
    cap = bound(block) if block != 4096 else 2000          # 4 KB blocks at a capacity that fails some of them
    srch = np.full(n * src_stride + 64, 0x11, np.uint8)
    sizes = np.array([min(block, total - i * block) for i in range(n)], np.int32)
    for i in range(n):
        srch[16 + i * src_stride:16 + i * src_stride + sizes[i]] = data[i * block:i * block + sizes[i]]
    src = t(srch)
    sz = t(sizes)
    res = []
    for indexed in (False, True):
        dst = torch.full((n * dst_stride,), GUARD, dtype=torch.uint8, device=DEV)
        out = torch.full((n,), -99, dtype=torch.int32, device=DEV)
        ws = None
        if parse == HC:
            ws = torch.empty(int(lib.LZ4B200_compress_blocks_indexed_workspace_bytes(n, HC, param)), dtype=torch.uint8,
                             device=DEV)
        l0 = lib.LZ4B200_launch_count()
        st = torch.cuda.current_stream().cuda_stream
        if indexed:
            out = run_indexed(lib, src.data_ptr() + 16, np.arange(n) * src_stride, sizes, dst,
                              np.arange(n) * dst_stride, [cap] * n, parse, param, ws=ws)
        else:
            args = (src.data_ptr() + 16, src_stride, sz.data_ptr(), block, dst.data_ptr(), dst_stride, cap, param,
                    out.data_ptr(), n)
            if parse == HC:
                fn = lib.LZ4B200_compress_blocks_hc_opt if param >= 10 else lib.LZ4B200_compress_blocks_hc
                rc = fn(*args, ws.data_ptr(), ws.numel(), st)
            else:
                fn = lib.LZ4B200_compress_blocks if parse == FAST else lib.LZ4B200_compress_blocks_parallel
                rc = fn(*args, st)
            assert rc == 0
        launches = lib.LZ4B200_launch_count() - l0
        res.append((out.cpu().numpy().copy(), dst.cpu().numpy(), launches))
    assert np.array_equal(res[0][0], res[1][0])
    assert np.array_equal(res[0][1], res[1][1])
    assert res[0][2] == res[1][2] == (2 if parse == PARALLEL else 1)
    if parse == FAST:                                   # and both are the oracle's
        for i in range(n):
            r, b = oracle.compress(data[i * block:i * block + sizes[i]], 1, cap)
            assert res[1][0][i] == r and res[1][1][i * dst_stride:i * dst_stride + r].tobytes() == b


# ------------------------------------------------------------------------------------------
# 4. scale: more blocks than resident warps, CTAs and HC slots
# ------------------------------------------------------------------------------------------
SMALL_MAX, SMALL_CAP, LIMITED_CAP = 3000, bound(3000), 600


@pytest.mark.parametrize("parse,param", [(FAST, 1), (PARALLEL, 1), (HC, 9)], ids=["fast", "parallel", "hc-9"])
def test_scale_with_big_blocks_at_both_ends(lib, oracle, parse, param):
    """40 000 small blocks with a big block first and last (4 MB; 200 000 bytes for HC), the HC workspace at its
    minimum (16 384 slots): tables and slots reused across very different sizes.  Every 7th small block is limited to
    600 bytes.  The parallel parse's small blocks are checked against the strided parallel call on a copy of the same
    blocks at other addresses (one call per capacity), its big ones against the oracle."""
    rng = np.random.default_rng(40)
    n_small = 40000
    big = (4 << 20) if parse != HC else 200000
    sizes = np.concatenate([[big], rng.integers(0, SMALL_MAX + 1, n_small), [big + 7]]).astype(np.int32)
    pool = oracle.datagen(int(sizes.sum()) + 1, 0.5, 5)
    starts = np.concatenate([[0], np.cumsum(sizes[:-1].astype(np.int64))])
    datas = [pool[s:s + n] for s, n in zip(starts, sizes)]
    caps = np.array([bound(int(sizes[0]))] + [SMALL_CAP] * n_small + [bound(int(sizes[-1]))], np.int64)
    caps[1:-1:7] = LIMITED_CAP
    arena, soff = place_sources(datas, 41)
    doff, total = abutting(caps)
    dst = torch.full((total,), GUARD, dtype=torch.uint8, device=DEV)
    ws = None
    if parse == HC:
        need = int(lib.LZ4B200_compress_blocks_indexed_workspace_bytes(len(sizes), HC, param))
        assert need == 16384 * 256 * 1024
        ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    got = run_indexed(lib, t(arena), soff, sizes, dst, doff, caps, parse, param, ws=ws).cpu().numpy()
    out_h = dst.cpu().numpy()
    del ws, dst
    if parse == FAST:
        want = [oracle.compress(d, param, int(c)) for d, c in zip(datas, caps)]
    elif parse == HC:
        want = [host_hc(d, int(c), param) for d, c in zip(datas, caps)]
    else:
        want = [oracle.compress(datas[0], param, int(caps[0]))] + [None] * n_small + \
               [oracle.compress(datas[-1], param, int(caps[-1]))]
        stride = SMALL_MAX + 16 + 3
        sh = np.zeros(n_small * stride + 64, np.uint8)
        for i in range(n_small):
            sh[16 + i * stride:16 + i * stride + sizes[i + 1]] = datas[i + 1]
        ssrc, ssz = t(sh), t(sizes[1:-1])
        for cap in (SMALL_CAP, LIMITED_CAP):
            odst = torch.full((n_small * SMALL_CAP,), GUARD, dtype=torch.uint8, device=DEV)
            out = torch.zeros(n_small, dtype=torch.int32, device=DEV)
            rc = lib.LZ4B200_compress_blocks_parallel(ssrc.data_ptr() + 16, stride, ssz.data_ptr(), 0, odst.data_ptr(),
                                                      SMALL_CAP, cap, param, out.data_ptr(), n_small,
                                                      torch.cuda.current_stream().cuda_stream)
            assert rc == 0
            oh, dh = out.cpu().numpy(), odst.cpu().numpy()
            for j in np.flatnonzero(caps[1:-1] == cap):
                r = int(oh[j])
                want[j + 1] = (r, dh[j * SMALL_CAP:j * SMALL_CAP + max(r, 0)].tobytes())
    check_outputs(out_h, doff, caps, got, want, "%s scale: " % PARSE_NAME[parse])


# ------------------------------------------------------------------------------------------
# 5. far offsets
# ------------------------------------------------------------------------------------------
SENT = 0x5A
LOW = L31                       # arena bytes below the base pointers: where an offset cut to a signed 32-bit int lands
ABOVE = L32 + 64 * MiB
LINES = [L31 - 1, L31, L32 - 3, L32 + 17, L32 - 30000]             # the last one: blocks across 2^32
NEAR_SRC = [1 * MiB + 5, 2 * MiB + 9, 3 * MiB + 1]
NEAR_DST = [5 * MiB + 3, 6 * MiB + 11, 7 * MiB]


@pytest.fixture(scope="module")
def far_arena():
    """one allocation of 2 GiB + 4 GiB + 64 MiB filled with a sentinel; the call's base pointers sit 2 GiB in, so that an
    offset cut to 32 bits, unsigned or signed, lands inside the arena and shows as a written sentinel"""
    free, _ = torch.cuda.mem_get_info()
    if free < LOW + ABOVE + 512 * MiB:
        pytest.skip("needs %.1f GiB of free device memory" % ((LOW + ABOVE) / GiB))
    a = torch.full((LOW + ABOVE,), SENT, dtype=torch.uint8, device=DEV)
    yield a
    del a
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def cuts(off, n):
    """the offsets an n-byte range at off lands on when off is cut to 32 bits: unsigned, and signed at or above 2^31"""
    u = off & (L32 - 1)
    out = [u] if u != off else []
    if u + n > L31 and u - L32 != off:
        out.append(u - L32)
    return out


@pytest.mark.parametrize("parse,param", [(FAST, 1), (PARALLEL, 1), (HC, 9)], ids=["fast", "parallel", "hc-9"])
def test_far_offsets(lib, oracle, far_arena, parse, param):
    """one block's source, then its output, at 2^31 - 1, 2^31, 2^32 - 3, 2^32 + 17 and across 2^32, next to two blocks
    near the base: results, the bytes around every output, and the windows at the far offset cut to 32 bits"""
    sizes = [65536, 70000, 4096]
    datas = [oracle.datagen(n, 0.5, 90 + k) for k, n in enumerate(sizes)]
    caps = [bound(n) for n in sizes]
    caps[2] = 1000                                      # a limited block
    want = [expected(oracle, parse, param, d, c) for d, c in zip(datas, caps)]
    a = far_arena
    a.fill_(SENT)
    W = 4096
    view = lambda off, n: a[LOW + off:LOW + off + n]
    for line in LINES:
        for role in ("src", "dst"):
            soff = [line if role == "src" else NEAR_SRC[0]] + NEAR_SRC[1:]
            doff = [line if role == "dst" else NEAR_DST[0]] + NEAR_DST[1:]
            for o, d in zip(soff, datas):
                view(o, len(d)).copy_(t(d))
            torch.cuda.synchronize()
            got = run_indexed(lib, a.data_ptr() + LOW, soff, sizes, a.data_ptr() + LOW, doff, caps, parse,
                              param).cpu().numpy()
            for i, (o, c, (r, b)) in enumerate(zip(doff, caps, want)):
                what = "%s at %d, block %d: " % (role, line, i)
                assert int(got[i]) == r, what + "returned %d, expected %d" % (int(got[i]), r)
                win = view(o - W, c + 2 * W).cpu().numpy()
                assert (win[:W] == SENT).all() and (win[W + c:] == SENT).all(), what + "wrote outside its region"
                assert win[W:W + r].tobytes() == b, what + "bytes"
                if r > 0:                               # (a block that returned 0 may have written its region)
                    assert (win[W + r:W + c] == SENT).all(), what + "wrote past its result"
            far = (line, sizes[0]) if role == "src" else (line, caps[0])
            for cut in cuts(*far):
                lo = max(cut - W, -LOW)
                assert bool((view(lo, cut + far[1] + W - lo) == SENT).all()), \
                    "%s at %d: the window at its offset cut to 32 bits (%d) was written" % (role, line, cut)
            for o, d in zip(soff, datas):
                assert view(o, len(d)).cpu().numpy().tobytes() == d.tobytes(), "a source changed"
                view(o, len(d)).fill_(SENT)
            for o, c in zip(doff, caps):
                view(o, c).fill_(SENT)


# ------------------------------------------------------------------------------------------
# 6. streams and graphs
# ------------------------------------------------------------------------------------------
def _buffers(oracle, seed, n=64):
    rng = np.random.default_rng(seed)
    sizes = rng.integers(0, 70000, n).astype(np.int32)
    datas = [oracle.datagen(int(s), 0.5, seed * 1000 + i) for i, s in enumerate(sizes)]
    arena, soff = place_sources(datas, seed)
    return datas, arena, soff, sizes


@pytest.mark.parametrize("parse", ["fast", "parallel", "hc"])
def test_side_stream_and_graph_replay(oracle, parse):
    """compress_buffers on a side stream equals the call on the default stream; captured into a CUDA graph and replayed
    on two new payloads of the same sizes, it gives each payload's result"""
    from lz4_b200 import batch
    datas, arena, soff, sizes = _buffers(oracle, 3)
    src, offs, sz = t(arena), t(soff), t(sizes)
    out0, s0, oo0, caps0 = batch.compress_buffers(src, offs, sz, parse=parse)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        out1, s1, oo1, caps1 = batch.compress_buffers(src, offs, sz, parse=parse, stream=side)
    side.synchronize()
    torch.cuda.synchronize()
    assert torch.equal(s0, s1) and torch.equal(oo0, oo1) and torch.equal(caps0, caps1)
    for i in range(len(sizes)):
        o, r = int(oo0[i]), int(s0[i])
        assert torch.equal(out0[o:o + r], out1[o:o + r])
    # graph: static inputs and outputs
    out = torch.full_like(out0, GUARD)
    outs = torch.empty(len(sizes), dtype=torch.int32, device=DEV)
    ws = None
    if parse == "hc":
        ws = torch.empty(int(batch._lib.load().LZ4B200_compress_blocks_indexed_workspace_bytes(len(sizes), 2, 9)),
                         dtype=torch.uint8, device=DEV)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.graph(g, stream=s):
        batch.compress_buffers(src, offs, sz, parse=parse, out=out, out_offsets=oo0, capacities=caps0, out_sizes=outs,
                               workspace=ws, stream=s)
    for seed in (8, 9):
        rng = np.random.default_rng(seed)
        new = [oracle.datagen(len(d), 0.3 + 0.1 * (seed - 8), seed * 77 + i) if i % 2 else
               rng.integers(0, 256, len(d), dtype=np.uint8) for i, d in enumerate(datas)]
        host = arena.copy()
        for i, d in enumerate(new):
            host[soff[i]:soff[i] + len(d)] = d
        src.copy_(t(host))
        out.fill_(GUARD)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        code = {"fast": FAST, "parallel": PARALLEL, "hc": HC}[parse]
        want = [expected(oracle, code, 1 if code != HC else 9, d, int(c)) for d, c in zip(new, caps0.cpu().numpy())]
        check_outputs(out.cpu().numpy(), oo0.cpu().numpy(), caps0.cpu().numpy(), outs.cpu().numpy(), want,
                      "replay %d: " % seed)


# ------------------------------------------------------------------------------------------
# 7. round trip through the wrappers
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("parse", ["fast", "parallel", "hc"])
@pytest.mark.parametrize("header", [0, 4])
def test_round_trip_through_pack_and_decode(oracle, parse, header):
    """compress_buffers -> pack_blocks(slot_offsets=) -> decompress_blocks with offsets gives the inputs back; the packed
    stream is the pack model's"""
    from lz4_b200 import batch
    datas, arena, soff, sizes = _buffers(oracle, 5 + header)
    out, osz, ooff, caps = batch.compress_buffers(t(arena), t(soff), t(sizes), parse=parse, level=3)
    packed, poff = batch.pack_blocks(out, None, osz, header_bytes=header, slot_offsets=ooff)
    n = len(sizes)
    cap = int(max(sizes.max(), 1))
    dec, rets = batch.decompress_blocks(packed, (poff[:-1] + header).contiguous(), osz, cap)
    torch.cuda.synchronize()
    assert (rets.cpu().numpy() == sizes).all()
    dh = dec.cpu().numpy()
    for i, d in enumerate(datas):
        assert dh[i * cap:i * cap + len(d)].tobytes() == d.tobytes(), i
    # the pack model over the same slots laid out at a stride
    oh, ooh, szh = out.cpu().numpy(), ooff.cpu().numpy(), osz.cpu().numpy()
    S = int(caps.max())
    slots = np.zeros(n * S, np.uint8)
    for i in range(n):
        slots[i * S:i * S + max(int(szh[i]), 0)] = oh[ooh[i]:ooh[i] + max(int(szh[i]), 0)]
    want_off, want = pack_model(slots, S, szh, header)
    assert np.array_equal(poff.cpu().numpy(), want_off)
    assert packed[:len(want)].cpu().numpy().tobytes() == want
    # with slot_stride given as the bound of every size, the same
    packed2, poff2 = batch.pack_blocks(out, S, osz, header_bytes=header, slot_offsets=ooff)
    assert torch.equal(poff2, poff) and torch.equal(packed2[:len(want)], packed[:len(want)])


def test_pack_indexed_is_pack_at_strided_offsets(lib):
    """LZ4B200_pack_blocks_indexed with slotOff = i * slotStride is LZ4B200_pack_blocks: offsets, bytes and launches"""
    rng = np.random.default_rng(1)
    n, stride = 3000, 777
    sizes = rng.integers(-3, stride + 1, n).astype(np.int32)
    slots = t(rng.integers(0, 256, n * stride + 16, dtype=np.uint8))
    sz = t(sizes)
    offs = t(np.arange(n, dtype=np.int64) * stride)
    st = torch.cuda.current_stream().cuda_stream
    res = []
    for hdr in (0, 4):
        for indexed in (False, True):
            packed = torch.full((n * (stride + 4) + 16,), GUARD, dtype=torch.uint8, device=DEV)
            oo = torch.empty(n + 1, dtype=torch.int64, device=DEV)
            l0 = lib.LZ4B200_launch_count()
            if indexed:
                rc = lib.LZ4B200_pack_blocks_indexed(slots.data_ptr(), offs.data_ptr(), sz.data_ptr(), n,
                                                     packed.data_ptr(), oo.data_ptr(), hdr, st)
            else:
                rc = lib.LZ4B200_pack_blocks(slots.data_ptr(), stride, sz.data_ptr(), n, packed.data_ptr(),
                                             oo.data_ptr(), hdr, st)
            assert rc == 0
            res.append((packed.cpu().numpy(), oo.cpu().numpy(), lib.LZ4B200_launch_count() - l0))
        assert np.array_equal(res[-1][0], res[-2][0]) and np.array_equal(res[-1][1], res[-2][1])
        assert res[-1][2] == res[-2][2] == 2


# ------------------------------------------------------------------------------------------
# 8. the wrappers reject what the kernels would misread
# ------------------------------------------------------------------------------------------
class _Rec(Recorder):
    SIZES = Recorder.SIZES + ("LZ4B200_compress_blocks_indexed_workspace_bytes",)


@pytest.fixture
def rec(monkeypatch):
    from lz4_b200 import _lib, batch
    r = _Rec(_lib.load())
    monkeypatch.setattr(_lib, "load", lambda: r)
    monkeypatch.setattr(batch, "_workspaces", {})
    return r


N = 3


def _z(n, dtype=torch.uint8, dev=DEV):
    return torch.zeros(n, dtype=dtype, device=dev)


def _good(parse):
    from lz4_b200 import _lib
    kw = dict(src=_z(256), offsets=_z(N, torch.int64), sizes=torch.full((N,), 16, dtype=torch.int32, device=DEV),
              parse=parse, out=_z(128), out_offsets=_z(N, torch.int64),
              capacities=torch.full((N,), 32, dtype=torch.int32, device=DEV), out_sizes=_z(N, torch.int32))
    if parse == "hc":
        kw["workspace"] = _z(int(_lib.load().LZ4B200_compress_blocks_indexed_workspace_bytes(N, 2, 9)))
    return kw


def _noncontig(x):
    return torch.stack([x, x], 1)[:, 0]


DEFECTS = [
    ("src", lambda kw: _z(256, torch.float32)), ("src", lambda kw: _z(256, dev="cpu")),
    ("src", lambda kw: _noncontig(kw["src"])),
    ("offsets", lambda kw: _z(N, torch.int32)), ("offsets", lambda kw: _z(N - 1, torch.int64)),
    ("offsets", lambda kw: _z(N, torch.int64, "cpu")), ("offsets", lambda kw: _noncontig(kw["offsets"])),
    ("sizes", lambda kw: _z(N, torch.int64)), ("sizes", lambda kw: _z(N, torch.int32, "cpu")),
    ("sizes", lambda kw: _noncontig(kw["sizes"])),
    ("out", lambda kw: _z(128, torch.int8)), ("out", lambda kw: _z(128, dev="cpu")),
    ("out", lambda kw: _noncontig(kw["out"])),
    ("out_offsets", lambda kw: _z(N, torch.int32)), ("out_offsets", lambda kw: _z(N - 1, torch.int64)),
    ("out_offsets", lambda kw: _noncontig(kw["out_offsets"])),
    ("capacities", lambda kw: _z(N, torch.int64)), ("capacities", lambda kw: _z(N - 1, torch.int32)),
    ("capacities", lambda kw: _z(N + 1, torch.int32)), ("capacities", lambda kw: _noncontig(kw["capacities"])),
    ("out_sizes", lambda kw: _z(N, torch.int64)), ("out_sizes", lambda kw: _z(N - 1, torch.int32)),
    ("out_sizes", lambda kw: _z(N, torch.int32, "cpu")),
    ("acceleration", lambda kw: 2 ** 31), ("level", lambda kw: -2 ** 31 - 1), ("parse", lambda kw: "exact"),
]


@pytest.mark.parametrize("parse", ["fast", "parallel", "hc"])
def test_compress_buffers_rejects(rec, parse):
    from lz4_b200 import batch
    batch.compress_buffers(**_good(parse))
    assert len(rec.calls) == 1 and rec.calls[0][0] == "LZ4B200_compress_blocks_indexed"
    rows = list(DEFECTS)
    if parse == "hc":
        rows += [("workspace", lambda kw: kw["workspace"][:-1]), ("workspace", lambda kw: _z(kw["workspace"].numel() // 4,
                                                                                             torch.int32))]
    for arg, make in rows:
        kw = _good(parse)
        kw[arg] = make(kw)
        rec.calls.clear()
        with pytest.raises(ValueError):
            batch.compress_buffers(**kw)
        assert not rec.calls, (arg, "reached the library")


def test_compress_buffers_needs_out_and_workspace_under_capture(rec):
    from lz4_b200 import batch
    s = torch.cuda.Stream()
    for parse, drop in (("fast", "out"), ("parallel", "out"), ("hc", "out"), ("hc", "workspace")):
        kw = _good(parse)
        del kw[drop]
        del kw["out_offsets"]                           # computed inside the capture
        rec.calls.clear()
        with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
            with pytest.raises(ValueError):
                batch.compress_buffers(stream=s, **kw)
        assert not rec.calls, (parse, drop)
    torch.cuda.synchronize()


def test_pack_blocks_slot_offsets_rejects(rec):
    from lz4_b200 import batch
    good = dict(slots=_z(256), slot_stride=None, sizes=torch.full((N,), 16, dtype=torch.int32, device=DEV),
                packed=_z(64), slot_offsets=_z(N, torch.int64))
    batch.pack_blocks(**good)
    assert rec.calls[-1][0] == "LZ4B200_pack_blocks_indexed"
    for arg, bad in (("slot_offsets", _z(N, torch.int32)), ("slot_offsets", _z(N - 1, torch.int64)),
                     ("slot_offsets", _z(N, torch.int64, "cpu")), ("slot_offsets", _noncontig(_z(N, torch.int64))),
                     ("slots", _z(256, torch.int32)), ("sizes", _z(N, torch.int64)), ("packed", _z(64, dev="cpu")),
                     ("slot_stride", -1), ("header_bytes", 2 ** 31)):
        kw = dict(good)
        kw[arg] = bad
        rec.calls.clear()
        with pytest.raises(ValueError):
            batch.pack_blocks(**kw)
        assert not rec.calls, arg
    kw = dict(good, slot_stride=100)                    # with slot_stride, packed must hold n * (stride + header)
    kw["packed"] = _z(3 * 100 - 1)
    with pytest.raises(ValueError):
        batch.pack_blocks(**kw)
    s = torch.cuda.Stream()
    kw = dict(good)
    del kw["packed"]
    rec.calls.clear()
    with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
        with pytest.raises(ValueError):
            batch.pack_blocks(stream=s, **kw)
    assert not rec.calls
    torch.cuda.synchronize()
