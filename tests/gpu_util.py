"""Helpers shared by the GPU parity tests: a stand-in of the library that records the batch wrappers' calls, device-API
decode calls that check what they may not touch, the decode route a call takes, and the hostile block corpus of the route
tests."""
import hashlib

import numpy as np
import torch


def dev():
    return torch.device("cuda:0")


def to_dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


def pack_host_blocks(blocks):
    """list of bytes -> (u8 array, int64 offsets, int32 sizes)"""
    sizes = np.array([len(b) for b in blocks], dtype=np.int32)
    offs = np.zeros(len(blocks), dtype=np.int64)
    if len(blocks) > 1:
        offs[1:] = np.cumsum(sizes[:-1].astype(np.int64))
    buf = np.frombuffer(b"".join(blocks) + b"\x00" * 16, dtype=np.uint8).copy()
    return buf, offs, sizes


class Recorder:
    """liblz4_b200 as the lz4_b200.batch wrappers see it: the size functions are the library's own, every batch call is
    recorded as (name, arguments), with the device current at the call in .devices, and returns 0 without touching the
    device."""
    SIZES = ("LZ4_compressBound", "LZ4B200_decompress_workspace_bytes_for", "LZ4B200_compress_blocks_hc_workspace_bytes",
             "LZ4B200_compress_blocks_hc_opt_workspace_bytes", "LZ4B200_decompress_frames_workspace_bytes",
             "LZ4B200_last_cuda_error")

    def __init__(self, real):
        self.real, self.calls, self.devices = real, [], []

    def __getattr__(self, name):
        if name in self.SIZES:
            return getattr(self.real, name)
        if not name.startswith("LZ4B200_"):
            raise AttributeError(name)

        def call(*args):
            self.calls.append((name, args))
            self.devices.append(torch.cuda.current_device())
            return 0
        return call


# ------------------------------------------------------------------------------------------
# decode calls
# ------------------------------------------------------------------------------------------
def ws_lists(ws, n):
    """(nSeq[n], slow list) left in a decode workspace.  Layout (plan_layout, lz4_decode_plan.h): a 256-byte header
    whose first word is the slow-list count, then nSeq[n] and slowList[n], each rounded up to 256 bytes."""
    lst = (n * 4 + 255) // 256 * 256
    w = ws[:256 + 2 * lst].cpu().numpy().view(np.uint32)
    count = int(w[0])
    assert count <= n, "slow list count %d > %d blocks" % (count, n)
    return w[64:64 + n].copy(), w[(256 + lst) // 4:(256 + lst) // 4 + count].copy()


def route(n_blocks, cap=None, per_block_caps=False, ws_bytes=0):
    """The decode route lz4k_launch_decode takes with LZ4K_SCAN_IMPL unset (plan_decode, lz4_decode_plan.h):
      R1 per-block capacities: one-thread scan -> rows / generic
      R2 one capacity in [16 KB, 64 KB], <= 8 192 blocks: split scan -> rows / generic
      R3 one capacity in [16 KB, 64 KB], > 8 192 blocks: one-thread scan -> rows / generic
      R4 one capacity below 16 KB: one-thread scan -> rows / generic
      R5 one capacity in (64 KB, 64 MB] and the workspace of LZ4B200_decompress_workspace_bytes_for (the
         plan's wide flag): parallel scan -> tile index -> tiles / generic
      R6 one capacity above 64 KB otherwise: parallel scan -> generic"""
    if per_block_caps:
        return "R1"
    if cap > 65536:
        from lz4_b200 import _lib
        wide = cap <= (64 << 20) and ws_bytes >= int(_lib.load().LZ4B200_decompress_workspace_bytes_for(n_blocks, 0, cap))
        return "R5" if wide else "R6"
    if cap >= 16384:
        return "R2" if n_blocks <= 8192 else "R3"
    return "R4"


class Decoded(list):
    """(return value, decoded bytes) per block.  .slow: the slow list (blocks the generic kernel decoded), .nseq: the
    scan's sequence count per block, .route: route(...) of the call, .ws: the workspace (device tensor)."""


def _decode(blocks, slot_off, slot_len, total, dst_off, stride, caps, cap, ws_bytes, phases, rt):
    from lz4_b200 import _lib
    lib = _lib.load()
    assert phases in ("one", "split")
    n = len(blocks)
    buf, offs, sizes = pack_host_blocks(blocks)
    d_buf, d_offs, d_sizes = to_dev(buf), to_dev(offs), to_dev(sizes)
    d_caps = to_dev(np.asarray(caps, dtype=np.int32)) if caps is not None else None
    d_dst_off = to_dev(dst_off) if dst_off is not None else None
    d_out = torch.full((total,), 0xA5, dtype=torch.uint8, device=dev())
    d_ret = torch.zeros(n, dtype=torch.int32, device=dev())
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev())
    args = (d_buf.data_ptr(), d_offs.data_ptr(), d_sizes.data_ptr(), d_out.data_ptr(),
            d_dst_off.data_ptr() if d_dst_off is not None else None, stride,
            d_caps.data_ptr() if d_caps is not None else None, cap, d_ret.data_ptr(), n, ws.data_ptr(), ws.numel())
    stream = torch.cuda.current_stream().cuda_stream
    scanned = None
    if phases == "split":                       # scan, read the sizes, then expand with the same workspace
        _lib.check(lib.LZ4B200_decompress_blocks_phased(*args, 1, stream), "decompress_blocks_phased(scan)")
        scanned = d_ret.cpu().numpy().copy()
        _lib.check(lib.LZ4B200_decompress_blocks_phased(*args, 2, stream), "decompress_blocks_phased(expand)")
    else:
        _lib.check(lib.LZ4B200_decompress_blocks(*args, stream), "decompress_blocks")
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    ret = d_ret.cpu().numpy()
    if scanned is not None:
        assert (scanned == ret).all(), "the expand phase changed the sizes the scan left"
    res = Decoded()
    res.nseq, res.slow = ws_lists(ws, n)
    res.route = rt
    res.ws = ws
    assert len(set(res.slow.tolist())) == len(res.slow), "a block is on the slow list twice"
    assert all(ret[b] > 0 for b in res.slow), "a rejected or empty block is on the slow list"
    for i in range(n):
        o, r = int(slot_off[i]), int(ret[i])
        keep = max(r, 0)
        # every expand kernel writes exactly [0, ret): a rejected block's slot, and the rest of an accepted one, stay as they were
        untouched = out[o + keep:o + int(slot_len[i])]
        assert (untouched == 0xA5).all(), "block %d (return value %d) wrote outside [0, %d) of its %d-byte slot" % (
            i, r, keep, int(slot_len[i]))
        res.append((r, out[o:o + keep].tobytes()))
    return res


def decode_batch(blocks, caps, phases="one"):
    """Run blocks through LZ4B200_decompress_blocks with per-block capacities (device API; route R1), each in a slot of
    its capacity + 64 bytes.  phases="split": the scan and the expand as two calls.  Returns a Decoded."""
    from lz4_b200 import _lib
    n = len(blocks)
    caps = np.asarray(caps, dtype=np.int32)
    slot = np.maximum(caps, 0).astype(np.int64) + 64
    dst_off = np.zeros(n, dtype=np.int64)
    dst_off[1:] = np.cumsum(slot[:-1])
    ws_bytes = int(_lib.load().LZ4B200_decompress_workspace_bytes(n))
    return _decode(blocks, dst_off, slot, int(slot.sum()), dst_off, 0, caps, 0, ws_bytes, phases,
                   route(n, per_block_caps=True))


def decode_batch_uniform(blocks, cap, wide=True, stride=None, phases="one", dst_off=None, ws_bytes=None):
    """Run blocks through LZ4B200_decompress_blocks with ONE capacity for all of them (device API).  wide=True gives the
    workspace LZ4B200_decompress_workspace_bytes_for asks for (blocks above 64 KB: the tiles kernel), wide=False the
    one for any capacities (blocks above 64 KB: the generic kernel); ws_bytes: this many bytes instead.  stride:
    destination stride (default: capacity + 64 rounded up to 16 bytes; an odd one leaves the destinations unaligned).
    dst_off: per-block destination offsets instead of the stride (slots of capacity bytes that must not overlap).
    Returns a Decoded."""
    from lz4_b200 import _lib
    lib = _lib.load()
    n = len(blocks)
    stride = (cap + 64 + 15) // 16 * 16 if stride is None else stride
    assert stride >= cap
    if ws_bytes is None:
        ws_bytes = int(lib.LZ4B200_decompress_workspace_bytes_for(n, 0, cap)) if wide else int(lib.LZ4B200_decompress_workspace_bytes(n))
    if dst_off is None:
        slot_off, slot_len, total = np.arange(n, dtype=np.int64) * stride, np.full(n, stride, dtype=np.int64), n * stride
    else:
        slot_off = np.asarray(dst_off, dtype=np.int64)
        order = np.argsort(slot_off)
        assert (np.diff(slot_off[order]) >= cap).all(), "destination slots overlap"
        slot_len = np.full(n, cap, dtype=np.int64)
        total, stride = int(slot_off.max()) + cap + 64, 0
    return _decode(blocks, slot_off, slot_len, total, None if dst_off is None else slot_off, stride, None, cap, ws_bytes,
                   phases, route(n, cap, ws_bytes=ws_bytes))


def wide_workspace(res, n, cap):
    """Readers of what the scan and the tile index left in an R5 call's workspace (plan_layout, lz4_decode_plan.h): header |
    nSeq | slowList | marks (2 * (cap / 4 + 2) words per block) | tileFirst (tiles_of(cap) + 1 words per block) |
    tileFlag.  Returns (marks(b, nseq): the first nseq wide marks of block b, flattened; tile_first(b, nt): its first
    nt + 1 tileFirst entries)."""
    r256 = lambda x: (x + 255) // 256 * 256
    stride = 2 * (cap // 4 + 2)
    tiles_max = (cap + 61439) // 61440
    marks0 = 256 + 2 * r256(n * 4)
    first0 = marks0 + r256(n * stride * 4)

    def words(at, k):
        return res.ws[at:at + 4 * k].cpu().numpy().view(np.uint32).copy()

    def marks(b, nseq):
        return words(marks0 + b * stride * 4, 2 * nseq)

    def tile_first(b, nt):
        return words(first0 + b * (tiles_max + 1) * 4, nt + 1)
    return marks, tile_first


# ------------------------------------------------------------------------------------------
# compress and pack calls
# ------------------------------------------------------------------------------------------
GUARD = 0xA5


def odd_stride(nbytes):
    """an odd slot stride with at least 16 guard bytes past nbytes"""
    return nbytes + 17 if nbytes % 2 == 0 else nbytes + 16


def compress_call(parallel, blocks, cap, accel, src_stride=None, src_phase=0, dst_stride=None, dst_mis=0,
                  scalar=None, per_block_sizes=True, seed=0):
    """One LZ4B200_compress_blocks(_parallel) call.  Block i is at d_src + src_phase + i * src_stride, between random
    bytes (16 readable bytes around every block: the header's readable padding); its slot is at
    d_dst + dst_mis + i * dst_stride (default: an odd stride), filled with GUARD bytes.  per_block_sizes=False passes no
    d_srcSize (all blocks then have the size `scalar`, default len(blocks[0])); scalar defaults to 0 otherwise.
    Checks that no byte outside the slots changed, nor any byte of a slot past `cap` -- or past the block's size when it
    fitted.  Returns (return values, [slot i's bytes [0, ret)])."""
    from lz4_b200 import _lib
    lib = _lib.load()
    n = len(blocks)
    sizes = np.array([len(b) for b in blocks], dtype=np.int32)
    src_stride = src_stride or int(sizes.max())
    dst_stride = dst_stride or odd_stride(cap)
    assert src_stride >= sizes.max() and dst_stride >= cap
    if scalar is None:
        scalar = 0 if per_block_sizes else int(sizes[0])
    if not per_block_sizes:
        assert (sizes == scalar).all()
    rng = np.random.default_rng(seed)
    src = rng.integers(0, 256, 16 + src_phase + n * src_stride + 16, dtype=np.uint8)
    for i, b in enumerate(blocks):
        o = 16 + src_phase + i * src_stride
        src[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    d_src = to_dev(src)
    d_sizes = to_dev(sizes)
    total = dst_mis + n * dst_stride + 64
    d_dst = torch.full((total,), GUARD, dtype=torch.uint8, device=dev())
    d_ret = torch.full((n,), -7, dtype=torch.int32, device=dev())
    fn = lib.LZ4B200_compress_blocks_parallel if parallel else lib.LZ4B200_compress_blocks
    rc = fn(d_src.data_ptr() + 16 + src_phase, src_stride, d_sizes.data_ptr() if per_block_sizes else None, scalar,
            d_dst.data_ptr() + dst_mis, dst_stride, cap, accel, d_ret.data_ptr(), n, torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "compress_blocks")
    torch.cuda.synchronize()
    out, ret = d_dst.cpu().numpy(), d_ret.cpu().numpy()
    assert (out[:dst_mis] == GUARD).all() and (out[dst_mis + n * dst_stride:] == GUARD).all(), "wrote outside the slots"
    res = []
    for i in range(n):
        r, o = int(ret[i]), dst_mis + i * dst_stride
        assert 0 <= r <= max(cap, 0), (i, r, cap)
        keep = r if r > 0 else max(cap, 0)
        assert (out[o + keep:o + dst_stride] == GUARD).all(), \
            "block %d (%d bytes, return value %d) wrote past %d bytes of its slot (capacity %d)" % (i, sizes[i], r, keep, cap)
        res.append(out[o:o + r].tobytes())
    return ret.copy(), res


def pack_model(slots, slot_stride, sizes, header_bytes, frame=None):
    """LZ4B200_pack_blocks / LZ4B200_pack_frame_blocks restated: (outOff[n + 1], packed bytes).  slots: host bytes of
    the slots (slot i at i * slot_stride); frame = (source bytes, source stride, blockSize, lastSize)."""
    n = len(sizes)
    offs, out = [0], bytearray()
    for i in range(n):
        c = int(sizes[i])
        raw = False
        if frame is None:
            pay = max(c, 0)
            body = slots[i * slot_stride:i * slot_stride + pay]
        else:
            fsrc, fstride, bsz, last = frame
            sz = last if (i == n - 1 and last > 0) else bsz
            raw = c <= 0 or c >= sz                                      # lz4frame.c:896-899
            pay = sz if raw else c
            body = fsrc[i * fstride:i * fstride + pay] if raw else slots[i * slot_stride:i * slot_stride + pay]
        if header_bytes:
            out += (pay | (0x80000000 if raw else 0)).to_bytes(4, "little")
        out += bytes(body)
        offs.append(len(out))
    return np.array(offs, dtype=np.int64), bytes(out)


def pack_call(slots, slot_stride, sizes, header_bytes, packed_mis=0, slot_phase=0, frame=None):
    """One LZ4B200_pack_blocks (frame=None) or LZ4B200_pack_frame_blocks call on host slots laid out at
    d_slots + slot_phase; the packed stream at d_packed + packed_mis in a buffer of GUARD bytes.  Checks outOff and the
    bytes against pack_model, and that nothing outside [0, outOff[n]) of the stream changed."""
    from lz4_b200 import _lib
    lib = _lib.load()
    n = len(sizes)
    want_off, want = pack_model(slots, slot_stride, sizes, header_bytes, frame)
    d_slots = to_dev(np.concatenate([np.zeros(slot_phase, np.uint8), np.frombuffer(bytes(slots), np.uint8),
                                     np.zeros(64, np.uint8)]))
    d_sizes = to_dev(np.asarray(sizes, dtype=np.int32))
    d_off = torch.full((n + 1,), -1, dtype=torch.int64, device=dev())
    cap = packed_mis + len(want) + 64
    d_packed = torch.full((cap,), GUARD, dtype=torch.uint8, device=dev())
    st = torch.cuda.current_stream().cuda_stream
    if frame is None:
        rc = lib.LZ4B200_pack_blocks(d_slots.data_ptr() + slot_phase, slot_stride, d_sizes.data_ptr(), n,
                                     d_packed.data_ptr() + packed_mis, d_off.data_ptr(), header_bytes, st)
    else:
        fsrc, fstride, bsz, last = frame
        d_fsrc = to_dev(np.concatenate([np.frombuffer(bytes(fsrc), np.uint8), np.zeros(64, np.uint8)]))
        rc = lib.LZ4B200_pack_frame_blocks(d_slots.data_ptr() + slot_phase, slot_stride, d_sizes.data_ptr(),
                                           d_fsrc.data_ptr(), fstride, bsz, last, n, d_packed.data_ptr() + packed_mis,
                                           d_off.data_ptr(), st)
    _lib.check(rc, "pack")
    torch.cuda.synchronize()
    off, out = d_off.cpu().numpy(), d_packed.cpu().numpy()
    assert (off == want_off).all(), "outOff differs at %d" % int(np.flatnonzero(off != want_off)[0])
    assert out[packed_mis:packed_mis + len(want)].tobytes() == want, "packed bytes differ"
    assert (out[:packed_mis] == GUARD).all() and (out[packed_mis + len(want):] == GUARD).all(), "wrote outside the stream"
    return off


# ------------------------------------------------------------------------------------------
# hostile corpus
# ------------------------------------------------------------------------------------------
def lz4_seq(lits, off, mlen=0):
    """one LZ4 sequence: literals, then a match of offset `off` and length mlen >= 4; off=None: the last sequence"""
    def ext(v):
        if v < 15:
            return b""
        r = v - 15
        return b"\xff" * (r // 255) + bytes([r % 255])
    ll, ml = len(lits), (0 if off is None else mlen - 4)
    out = bytes([(min(ll, 15) << 4) | min(ml, 15)]) + ext(ll) + lits
    return out if off is None else out + bytes([off & 255, off >> 8]) + ext(ml)


def seq_count_block(nseq):
    """a valid block of exactly nseq sequences (the last one literals only): 1 literal + an offset-1 match of 4, then
    empty-literal offset-1 matches of 4, then 16 literals; decodes to 4 * nseq + 13 bytes"""
    return lz4_seq(b"\x07", 1, 4) + lz4_seq(b"", 1, 4) * (nseq - 2) + lz4_seq(bytes(range(1, 17)), None)


# the rows kernel's run table holds kRowsMaxRuns = 20 480 runs (lz4_rows_core.h).  One literal + an offset-1 match of
# 5 bytes is 4 runs (the literal, and match pieces of 1, 2 and 2 bytes: rw_match_runs), so k such sequences and a
# literal tail make 4k + 1 runs: 20 477 for k = 5 119 and 20 481 for k = 5 120, in about 30 KB of output.
RUNS_BELOW, RUNS_ABOVE = 5119, 5120


def run_block(k, mlen=5, tail=29):
    """a valid block of k sequences of 1 literal + an offset-1 match of mlen bytes, then `tail` literals"""
    return b"".join(lz4_seq(bytes([1 + i % 251]), 1, mlen) for i in range(k)) + lz4_seq(bytes(range(1, tail + 1)), None)


def _filler(rng, out, op, until):
    """valid sequences (8..24 literals + a short match 8..200 back) appended to `out` until it holds `until` bytes"""
    while len(out) < until:
        lits = bytes(rng.integers(1, 256, int(rng.integers(8, 25)), dtype=np.uint8))
        ml = int(rng.integers(4, 13))
        off = min(op + len(lits), int(rng.integers(8, 201)))
        out += lz4_seq(lits, off, ml)
        op += len(lits) + ml
    return op


def event_block(rng, cap, quarter, kind):
    """A block of about 0.7 * cap input bytes (split scan: >= 4 096) whose first event lies in the middle of input
    quarter `quarter`: kind="offset", an offset that reaches before the output start (lz4.c:2161); kind="capacity", a
    match that ends at or beyond capacity - 64 (lz4.c:2137/2142), after which the output runs past the capacity."""
    n_in = min(int(cap * 0.7), 60000)
    out = bytearray()
    op = _filler(rng, out, 0, n_in * (2 * quarter + 1) // 8)
    if kind == "offset":
        out += lz4_seq(b"abc", min(op + 3 + int(rng.integers(1, 100)), 65535), 4)
    else:
        ml = cap - 64 - (op + 3) + int(rng.integers(0, 40))
        out += lz4_seq(b"abc", 1, ml)
        op += 3 + ml
    _filler(rng, out, op, n_in - 40)
    return bytes(out) + lz4_seq(bytes(rng.integers(1, 256, 29, dtype=np.uint8)), None)


def corrupt(rng, c):
    """1..5 random edits of the kinds of tests/fuzzer.c:588-622: set a byte, set a special value, flip a bit, delete,
    insert"""
    b = bytearray(c)
    for _ in range(int(rng.integers(1, 6))):
        if not b:
            break
        mode, pos = int(rng.integers(0, 5)), int(rng.integers(0, len(b)))
        if mode == 0:
            b[pos] = int(rng.integers(0, 256))
        elif mode == 1:
            b[pos] = int(rng.choice([0, 0xFF, 0xF0, 0x0F, 0x10, 0x1F]))
        elif mode == 2:
            b[pos] ^= 1 << int(rng.integers(0, 8))
        elif mode == 3:
            del b[pos:pos + int(rng.integers(1, 4))]
        else:
            b[pos:pos] = bytes(rng.integers(0, 256, int(rng.integers(1, 4)), dtype=np.uint8))
    return bytes(b) if b else b"\x00"


def hostile_corpus(oracle, cap, seed=0, n_corrupt=4):
    """[(kind, block)] for a batch of one capacity `cap`:
      datagen  P0 / P0.2 / P0.5 / P0.9 / P1 blocks of cap, cap -/+ 1, cap -/+ 64 and 2 * cap bytes (the capacity is
               exact, +1, +64, -1, -64 and half of what the block needs)
      broken   each of those truncated by one byte, cut in half, with one byte appended, and n_corrupt corrupted copies
      seqs-fit, seqs-over   exactly 8 191, 8 192 / 8 193 sequences (kMaxSeqFast: the mark table is full / one slot short)
      runs-fit, runs-over   4k + 1 runs just below (k = RUNS_BELOW) and just above (RUNS_ABOVE) the rows kernel's run table, and the
               denser blocks of offset-1 matches of 8 and 9 bytes (29 109 and 32 746 runs)
      offset   offset-0 and offset-1 runs of 4 .. 60 000 bytes
      event    (capacities >= 16 KB: the split scan) an offset error and a capacity event in each input quarter"""
    rng = np.random.default_rng(seed)
    out = []
    for p in (0.0, 0.2, 0.5, 0.9, 1.0):
        for n in (cap, cap - 1, cap - 64, cap + 1, cap + 64, 2 * cap):
            raw = oracle.datagen(max(n, 1), p, 1000 * seed + int(100 * p) + n % 97)
            _, c = oracle.compress(raw, 1)
            out.append(("datagen", c))
            out += [("broken", c[:-1]), ("broken", c[:len(c) // 2] or b"\x00"), ("broken", c + b"\x00")]
            out += [("broken", corrupt(rng, c)) for _ in range(n_corrupt)]
    out += [("seqs-fit", seq_count_block(8191)), ("seqs-fit", seq_count_block(8192)), ("seqs-over", seq_count_block(8193))]
    out += [("runs-fit", run_block(RUNS_BELOW)), ("runs-over", run_block(RUNS_ABOVE)),
            ("runs-over", run_block(7277, 8)), ("runs-over", run_block(6549, 9))]
    lit = lambda k: bytes(rng.integers(1, 256, k, dtype=np.uint8))
    for off in (0, 1):
        for ml in (4, 5, 19, 300, 5000, 60000):
            out.append(("offset", lz4_seq(lit(20), off, ml) + lz4_seq(lit(3), 7, 9) + lz4_seq(lit(12), None)))
        blk = b"".join(lz4_seq(lit(5 + k), off, 4 + 7 * k) for k in range(60))
        out.append(("offset", blk + lz4_seq(lit(12), None)))
    if cap >= 16384:
        for q in range(4):
            out += [("event", event_block(rng, cap, q, "offset")), ("event", event_block(rng, cap, q, "capacity"))]
    return out


def arrange(kinds, rets, n, ncta, seed=0):
    """Indices into a corpus for a batch of n blocks: the corpus in a shuffled cycle, and hostile blocks (rejected or run
    overflow) where the kernels' own structure puts blocks side by side:
      - in all 8 slots of a warp of the split scan (blocks 8 .. 15: the second warp of its first CTA) and as the last
        block (the last, partial group of lanes);
      - on CTA columns 0, 1 and ncta - 1 of the persistent expand kernels, which take blocks b, b + ncta, ...: run
        overflow, rejected and accepted blocks in turn, so that the block-ahead descriptor follows a skipped block."""
    rng = np.random.default_rng(seed)
    idx = np.resize(rng.permutation(len(kinds)), n)
    over = [i for i, k in enumerate(kinds) if k == "runs-over" and rets[i] > 0] or [i for i, r in enumerate(rets) if r < 0]
    rejected = [i for i, r in enumerate(rets) if r < 0]
    accepted = [i for i, r in enumerate(rets) if r > 0 and kinds[i] != "runs-over"]
    hostile = over + rejected
    pools = (over, rejected, accepted)
    for col in sorted({0, 1, ncta - 1}):
        for k, b in enumerate(range(col, n, ncta)):
            pool = pools[k % 3]
            idx[b] = pool[(b // 3) % len(pool)]
    for s in range(8, min(16, n)):
        idx[s] = hostile[(7 * s) % len(hostile)]
    if n < 8:
        idx[:] = [hostile[(5 * s) % len(hostile)] for s in range(n)]
    idx[n - 1] = rejected[len(rejected) // 2]
    return idx


def check_vs_oracle(oracle, blocks, caps, kinds, res, want_route):
    """Every block against oracle.decompress: return value (incl. the negative error position) and bytes.  Accepted
    run-overflow blocks and blocks of more sequences than the mark table must be on the slow list; accepted blocks the
    rows kernel must take (run and sequence counts just within its tables) must not.  Returns the counts of rejected and
    accepted blocks, of the slow list, and of the run-overflow blocks on it."""
    assert res.route == want_route, (res.route, want_route)
    slow = set(res.slow.tolist())
    memo = {}
    cnt = {"rejected": 0, "accepted": 0, "slow": len(slow), "overflow handed off": 0}
    for i, (blk, cap, kind, (ret, out)) in enumerate(zip(blocks, caps, kinds, res)):
        key = (blk, cap)
        if key not in memo:
            memo[key] = oracle.decompress(blk, cap)
        eret, eout = memo[key]
        assert ret == eret, (i, kind, len(blk), cap, ret, eret)
        if ret < 0:
            cnt["rejected"] += 1
            continue
        assert out == eout, (i, kind, len(blk), cap)
        cnt["accepted"] += 1
        if kind == "runs-over" or (kind == "seqs-over" and want_route != "R5"):   # (the tiles kernel has wide marks)
            assert i in slow, (i, kind, cap, "not handed to the generic kernel")
            cnt["overflow handed off"] += kind == "runs-over"
        elif kind in ("runs-fit", "seqs-fit") and cap <= 65536:
            assert i not in slow, (i, kind, cap, "the rows kernel must take it")
    return cnt
