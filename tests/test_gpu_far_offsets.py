"""Every batch call with bytes at and past 2^31 and 2^32 from its base pointers: decode routes R1 .. R6 and the partial
decode at far source and destination offsets and strides, a bench-shaped batch whose output passes 2^32, the wide
decode's workspace past 2^32, every compressor and the pack kernels at strides of about 2^31, the HC workspaces of a
full call (slots past 2^31 and 2^32), packed output past 4 GiB, and a decode into a pageable host buffer past 4 GiB.

The far layouts live in one arena (Arena) filled with a sentinel.  The call's base pointers sit 2 GiB into it, so that
an offset cut to 32 bits -- unsigned or signed -- still lands inside the arena, where it shows as wrong bytes rather than
a fault.  Every call is checked three ways: the results, the bytes around every block (the arena's model: sentinel
except where the test wrote input or expects output), and the alias windows at off mod 2^32 (and that minus 2^32 when it
is at or above 2^31), which must still hold the sentinel: they catch a truncated offset even when the far bytes happen
to be right.  Bulk output is compared on the device; only windows around blocks come back to the host.

Each test stays at or below 11 GiB of device memory (need() skips with the amount when the shared card lacks it) and
frees what it allocated; the module hands the cached memory back at the end."""
import numpy as np
import pytest
import torch

import encpar_model as M
import gpu_util as gu
from hc_emul import host_hc, host_hc_dest, host_hc_opt, host_hc_opt_dest, mg

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MiB, GiB = 1 << 20, 1 << 30
L31, L32 = 1 << 31, 1 << 32
SENT = 0x5A
W = 4096                               # sentinel window checked on both sides of every block and alias
LOW = L31                              # arena bytes below the base pointer: where a sign-extended 32-bit offset lands
SRC_ORG = GiB                          # the source pointer's offset from the base (the destination's is 0 or a phase)
ABOVE = L32 + GiB + 128 * MiB          # arena bytes at and above the base
UNWRITTEN = -123456789
PEAK = 11 * GiB


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    assert lib.LZ4B200_device_count() > 0, "GPU tests need a CUDA device"
    yield lib
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def memory_peak():
    """frees what the test left, and holds its peak to PEAK"""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    torch.cuda.empty_cache()
    print("peak device memory %.2f GiB" % (peak / GiB))
    assert peak <= PEAK, "peak device memory %.2f GiB" % (peak / GiB)


def need(nbytes):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + 256 * MiB:
        pytest.skip("needs %.1f GiB of free device memory, %.1f GiB free" % (nbytes / GiB, free / GiB))


def stream():
    return torch.cuda.current_stream().cuda_stream


def dev_u8(a):
    return torch.from_numpy(np.ascontiguousarray(np.frombuffer(bytes(a), np.uint8).copy() if isinstance(a, bytes) else a)).to(DEV)


def aliases(off, n):
    """[start] of the windows an n-byte range at off (>= 0) lands on when its offset is cut to 32 bits: off mod 2^32, and
    that minus 2^32 when a part of the range lies at or above 2^31 (a signed cut; a range across 2^32 lands across 0)"""
    a = off & (L32 - 1)
    out = []
    if a != off:
        out.append(a)
    if a + n > L31 and a - L32 != off:
        out.append(a - L32)
    return out


class Arena:
    """One uint8 allocation of LOW + ABOVE bytes filled with SENT; offsets are relative to the base, LOW bytes in.
    regions: (offset, bytes) the test wrote or expects after the call; ranges: (pointer offset from the base, offset from
    that pointer, length) of what the calls address, whose alias windows check() looks at."""

    def __init__(self, above=ABOVE):
        need(LOW + above)
        self.t = torch.full((LOW + above,), SENT, dtype=torch.uint8, device=DEV)
        self.base = self.t.data_ptr() + LOW
        self.regions = []
        self.ranges = []                      # (origin, offset from it, bytes): what aliases() is checked for

    def ptr(self, off):
        return self.base + off

    def put(self, off, data):
        """write data at off; the model keeps it there"""
        data = bytes(data)
        self.t[LOW + off:LOW + off + len(data)] = dev_u8(data)
        self.regions.append((off, data))

    def expect(self, off, data):
        """the call is to leave data at off"""
        self.regions.append((off, bytes(data)))

    def far(self, origin, off, n):
        """a range the call addresses as origin + off: its alias windows must stay sentinel"""
        self.ranges.append((origin, off, n))

    def view(self, off, n):
        return self.t[LOW + off:LOW + off + n]

    def _model(self, lo, hi):
        want = np.full(hi - lo, SENT, dtype=np.uint8)
        for off, data in self.regions:
            a, b = max(off, lo), min(off + len(data), hi)
            if a < b:
                want[a - lo:b - lo] = np.frombuffer(data, np.uint8)[a - off:b - off]
        return want

    def check(self, dont_care=()):
        """every region padded by W against the model (dont_care: (offset, length) ranges the call may have written), then
        every alias window against the sentinel"""
        spans = sorted([(off - W, off + len(d) + W) for off, d in self.regions] +
                       [(off - W, off + n + W) for off, n in dont_care])
        merged = []
        for a, b in spans:
            if merged and a <= merged[-1][1]:
                merged[-1][1] = max(merged[-1][1], b)
            else:
                merged.append([a, b])
        for lo, hi in merged:
            want = self._model(lo, hi)
            got = self.view(lo, hi - lo).cpu().numpy()
            for off, n in dont_care:
                a, b = max(off, lo), min(off + n, hi)
                if a < b:
                    got[a - lo:b - lo] = want[a - lo:b - lo]
            bad = np.flatnonzero(got != want)
            if len(bad):
                at = lo + int(bad[0])
                owner = [(off, len(d)) for off, d in self.regions if off <= at < off + len(d)]
                raise AssertionError("byte at base%+d is %d, want %d (%d bytes differ in [%d, %d); inside %s)" % (
                    at, got[bad[0]], want[bad[0]], len(bad), lo, hi, owner or "no region: the sentinel"))
        for origin, off, n in self.ranges:
            for a in aliases(off, n):
                lo, hi = max(origin + a - W, -LOW), origin + a + n + W     # (a signed alias may start below the arena)
                assert hi <= ABOVE
                assert not any(o < hi and lo < o + len(d) for o, d in self.regions), \
                    "layout: a region lies in the alias window of base%+d" % (origin + off)
                assert bool((self.view(lo, hi - lo) == SENT).all()), \
                    "the alias window at base%+d of the range at base%+d (%d bytes) was written" % (
                        origin + a, origin + off, n)


# ------------------------------------------------------------------------------------------
# decode at far offsets
# ------------------------------------------------------------------------------------------
ROUTES = {                   # route: (capacity, per-block capacities, wide workspace, partial: None / "one" / "per")
    "R1": (65536, True, False, None),
    "R2": (65536, False, False, None),
    "R3": (65536, False, False, None),
    "R4": (8192, False, False, None),
    "R5": (300000, False, True, None),
    "R6": (300000, False, False, None),
    "P-one": (40000, False, False, "one"),
    "P-per": (65536, False, False, "per"),
}
# far slot starts (offsets from the destination pointer), three sets: the lines themselves, one byte short, past them
FAR_DST = [
    lambda cap: [L31 - 1, L32 - 3, L32 + 2 * MiB + 1],
    lambda cap: [L31, L32, L32 - MiB],
    lambda cap: [L31 + 5, L32 + 17 - cap, L32 + 17],
]
STRIDES = [L31 + MiB + 9, L31 + MiB]
FILLERS = 8200


_corpora = {}


def corpus(oracle, cap):
    """(blocks, kinds) for a batch of capacity cap: P50 blocks that fill it, then the hostile corpus"""
    if cap not in _corpora:
        far = []
        for k in range(6):
            raw = oracle.datagen(cap - 7 * k, 0.5, 40 + k)
            far.append(("datagen", oracle.compress(raw, 1)[1]))
        hostile = gu.hostile_corpus(oracle, cap, seed=cap % 997, n_corrupt=1)
        _corpora[cap] = far + hostile
    return _corpora[cap]


def expected(oracle, blk, cap, target):
    if target is None:
        return oracle.decompress(blk, cap)
    return oracle.decompress_partial(blk, target)


def decode_far(lib, oracle, route, layout, phases):
    """One decode call of `route` with its blocks at far offsets.  layout: ("off", k) -- destination offsets of FAR_DST[k]
    for the P50 blocks and past 2^31 and 2^32 for the hostile ones, or ("stride", k): i * STRIDES[k].  Sources always at
    far srcOff: two runs of blocks, across 2^31 and across 2^32."""
    cap, per_block, wide, partial = ROUTES[route]
    items = corpus(oracle, cap)
    mode, k = layout
    if mode == "stride":                        # three blocks: P50, a generic-kernel (or, below 64 KB, rejected) block, P50
        mid = [it for it in items if it[0] == ("runs-over" if cap >= 65536 else "broken")][0]
        items = [items[0], mid, items[1]]
    n_real = len(items)
    fillers = FILLERS - n_real if route == "R3" else 0
    n = n_real + fillers
    blocks = [b for _, b in items] + [b"\x00"] * fillers
    kinds = [kk for kk, _ in items] + ["filler"] * fillers
    rng = np.random.default_rng(sum(map(ord, route)) + 7 * k)
    if partial == "per":
        targets = rng.integers(0, cap + 1, n).astype(np.int32)
        targets[:3] = (cap, cap // 2 + 1, 1)
    else:
        targets = np.full(n, cap, dtype=np.int32)
    caps = np.full(n, cap, dtype=np.int32)
    if per_block:
        caps[6:n_real] = [cap - (i % 3) * 997 for i in range(6, n_real)]

    ar = Arena()
    org_dst = 3 if (mode == "stride" and k == 0) else 0
    # sources: alternate between the run across 2^31 and the run across 2^32 (offsets from the source pointer)
    src_off = np.zeros(n, dtype=np.int64)
    heads = [L31 - len(blocks[0]) // 2, L32 - len(blocks[1]) // 2 - 1]
    for i in range(n_real):
        r = i % 2
        src_off[i] = heads[r]
        ar.put(SRC_ORG + heads[r], blocks[i])
        ar.far(SRC_ORG, heads[r], len(blocks[i]))
        heads[r] += len(blocks[i]) + (i % 5)
    if fillers:
        src_off[n_real:] = heads[0]
        ar.put(SRC_ORG + heads[0], b"\x00")
    sizes = np.array([len(b) for b in blocks], dtype=np.int32)
    # destinations
    slot = np.maximum(caps, 0).astype(np.int64)
    dst_off, stride = None, 0
    if mode == "off":
        dst_off = np.zeros(n, dtype=np.int64)
        far = FAR_DST[k](cap)
        pos = [L31 + 8 * MiB, L32 + 8 * MiB]
        for i in range(n_real):
            if i < len(far):
                dst_off[i] = far[i]
            else:
                r = i % 2
                dst_off[i] = pos[r] + (i % 3)
                pos[r] += int(slot[i]) + 16
        if fillers:
            dst_off[n_real:] = 160 * MiB + np.arange(fillers, dtype=np.int64) * cap
        order = np.argsort(dst_off)
        assert (np.diff(dst_off[order]) >= slot[order][:-1]).all(), "slots overlap"
    else:
        stride = STRIDES[k]
    slot_at = lambda i: int(dst_off[i]) if dst_off is not None else i * stride

    d_sizes, d_src_off = dev_u8(sizes.view(np.uint8)).view(torch.int32), dev_u8(src_off.view(np.uint8)).view(torch.int64)
    d_dst_off = dev_u8(dst_off.view(np.uint8)).view(torch.int64) if dst_off is not None else None
    d_caps = dev_u8(caps.view(np.uint8)).view(torch.int32) if per_block else None
    d_tgt = dev_u8(targets.view(np.uint8)).view(torch.int32) if partial == "per" else None
    d_ret = torch.full((n,), UNWRITTEN, dtype=torch.int32, device=DEV)
    if partial:
        wsb = int(lib.LZ4B200_decompress_workspace_bytes_for(n, partial == "per", 0 if partial == "per" else cap))
    elif wide or per_block:
        wsb = int(lib.LZ4B200_decompress_workspace_bytes_for(n, per_block, 0 if per_block else cap))
    else:
        wsb = int(lib.LZ4B200_decompress_workspace_bytes(n)) if route == "R6" else \
            int(lib.LZ4B200_decompress_workspace_bytes_for(n, 0, cap))
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    rt = "P" if partial else gu.route(n, cap, per_block, wsb)
    assert partial or rt == route, (rt, route)
    args = (ar.ptr(SRC_ORG), d_src_off.data_ptr(), d_sizes.data_ptr(), ar.ptr(org_dst),
            d_dst_off.data_ptr() if d_dst_off is not None else None, stride)
    if partial:
        rc = lib.LZ4B200_decompress_blocks_partial(*args, d_tgt.data_ptr() if d_tgt is not None else None, cap,
                                                   d_ret.data_ptr(), n, ws.data_ptr(), wsb, stream())
        assert rc == 0
    elif phases == "split":
        tail = (d_caps.data_ptr() if per_block else None, cap, d_ret.data_ptr(), n, ws.data_ptr(), wsb)
        assert lib.LZ4B200_decompress_blocks_phased(*args, *tail, 1, stream()) == 0
        scanned = d_ret.cpu().numpy().copy()
        assert lib.LZ4B200_decompress_blocks_phased(*args, *tail, 2, stream()) == 0
    else:
        rc = lib.LZ4B200_decompress_blocks(*args, d_caps.data_ptr() if per_block else None, cap, d_ret.data_ptr(), n,
                                           ws.data_ptr(), wsb, stream())
        assert rc == 0
    torch.cuda.synchronize()
    ret = d_ret.cpu().numpy()
    if phases == "split" and not partial:
        assert (scanned == ret).all(), "the expand phase changed the sizes the scan left"

    res = gu.Decoded()
    res.route = rt
    memo = {}
    for i in range(n_real):
        key = (blocks[i], int(caps[i]), int(targets[i]) if partial else None)
        if key not in memo:
            memo[key] = expected(oracle, blocks[i], int(caps[i]), int(targets[i]) if partial else None)
        eret, eout = memo[key]
        assert int(ret[i]) == eret, (route, layout, i, kinds[i], int(ret[i]), eret)
        room = int(targets[i]) if partial else int(slot[i])      # the expand writes [0, ret) of it, nothing else
        ar.expect(org_dst + slot_at(i), eout + bytes([SENT]) * (room - len(eout)))
        ar.far(org_dst, slot_at(i), max(room, 1))
        res.append((int(ret[i]), eout))
    assert (ret[n_real:] == 0).all(), "a filler block returned something else than 0"
    ar.check()
    if fillers:                                 # the fillers' slots (and everything between them) stay sentinel
        assert bool((ar.view(160 * MiB, fillers * cap) == SENT).all())
    if not partial:
        res.nseq, res.slow = gu.ws_lists(ws, n)
        res.slow = res.slow[res.slow < n_real]
        res.ws = ws
        cnt = gu.check_vs_oracle(oracle, blocks[:n_real], caps[:n_real], kinds[:n_real], res, route)
        assert cnt["accepted"] > 0 and (cnt["rejected"] > 0 or mode == "stride")
    return res, ar


@pytest.mark.parametrize("route", list(ROUTES))
def test_decode_routes_at_far_offsets(lib, oracle, route):
    """Every route with its P50 blocks at slot starts on, one byte short of and past 2^31 and 2^32 (and one across
    2^32), its hostile blocks past 2^31 and 2^32, sources in runs across both lines; one call and the two phases."""
    for k, phases in ((0, "one"), (1, "split"), (2, "one")):
        decode_far(lib, oracle, route, ("off", k), phases)
        torch.cuda.empty_cache()


@pytest.mark.parametrize("route", [r for r in ROUTES if r != "R3"])
def test_decode_routes_at_far_strides(lib, oracle, route):
    """Three blocks at i * dstStride with dstStride about 2^31 + 2^20 (odd and even, the odd one from an odd base): block
    1 past 2^31, block 2 past 2^32; the middle one takes the generic kernel or is rejected."""
    for k, phases in ((0, "one"), (1, "split")):
        decode_far(lib, oracle, route, ("stride", k), phases)
        torch.cuda.empty_cache()


@pytest.mark.parametrize("n_blocks", [8192, 8200])
def test_bench_shaped_batch_past_4_gib(lib, oracle, n_blocks):
    """64 KB blocks at dstStride = 2^19 + 4096, all reading one compressed P50 block (every srcOff equal): 8 192 through
    R2 and 8 200 through R3.  Blocks 8 129 and up lie above 2^32 (their bulk stores from the rows kernel); compared on the
    device, gaps included."""
    stride = (1 << 19) + 4096
    need(n_blocks * stride + 2 * GiB)
    with open(gu.__file__.replace("gpu_util.py", "golden/p50_seed0_64k.lz4block"), "rb") as f:
        blk = f.read()
    r, want = oracle.decompress(blk, 65536)
    assert r == 65536
    assert 8128 * stride + 65536 < L32 < 8129 * stride
    comp = dev_u8(b"\x00" * 16 + blk + b"\x00" * 16)
    offs = torch.full((n_blocks,), 16, dtype=torch.int64, device=DEV)
    sizes = torch.full((n_blocks,), len(blk), dtype=torch.int32, device=DEV)
    out = torch.full((n_blocks * stride,), SENT, dtype=torch.uint8, device=DEV)
    ret = torch.full((n_blocks,), UNWRITTEN, dtype=torch.int32, device=DEV)
    wsb = int(lib.LZ4B200_decompress_workspace_bytes_for(n_blocks, 0, 65536))
    assert gu.route(n_blocks, 65536, ws_bytes=wsb) == ("R2" if n_blocks <= 8192 else "R3")
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    assert lib.LZ4B200_decompress_blocks(comp.data_ptr(), offs.data_ptr(), sizes.data_ptr(), out.data_ptr(), None,
                                         stride, None, 65536, ret.data_ptr(), n_blocks, ws.data_ptr(), wsb,
                                         stream()) == 0
    torch.cuda.synchronize()
    assert bool((ret == 65536).all())
    rows = out.view(n_blocks, stride)
    row = dev_u8(want)
    for a in range(0, n_blocks, 1024):
        chunk = rows[a:a + 1024]
        assert torch.equal(chunk[:, :65536], row.expand(chunk.shape[0], 65536)), "blocks %d.." % a
        assert bool((chunk[:, 65536:] == SENT).all()), "gap after blocks %d.." % a
    assert len(gu.ws_lists(ws, n_blocks)[1]) == 0, "no block of this batch is the generic kernel's"


def test_wide_batch_with_its_workspace_past_4_gib(lib, oracle):
    """R5 with 520 blocks at a capacity of 4 MiB: the workspace is about 4.4 GB, so the marks of blocks 512 and up and
    all of tileFirst and tileFlag lie past 2^32.  Most blocks are one repeated compressed block, a few distinct P50 and
    periodic blocks go last."""
    n, cap = 520, 4 << 20
    wsb = int(lib.LZ4B200_decompress_workspace_bytes_for(n, 0, cap))
    assert wsb > L32 + 64 * MiB
    stride = cap + 16
    need(wsb + n * stride + 512 * MiB)
    common = oracle.compress(oracle.datagen(cap, 0.5, 11), 1)[1]
    last = [oracle.compress(oracle.datagen(cap - 3 * k, 0.5, 60 + k), 1)[1] for k in range(4)]
    last += [oracle.compress((bytes(range(1, 200)) * (cap // 199 + 1))[:cap - 5], 1)[1],
             oracle.compress(bytes(cap), 1)[1]]
    blocks = [common] * (n - len(last)) + last
    buf, offs, sizes = gu.pack_host_blocks([common] + last)
    idx = [0] * (n - len(last)) + list(range(1, len(last) + 1))
    offs, sizes = offs[idx], sizes[idx]
    comp = dev_u8(np.concatenate([buf, np.zeros(16, np.uint8)]))
    out = torch.full((n * stride,), SENT, dtype=torch.uint8, device=DEV)
    ret = torch.full((n,), UNWRITTEN, dtype=torch.int32, device=DEV)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    assert gu.route(n, cap, ws_bytes=wsb) == "R5"
    assert lib.LZ4B200_decompress_blocks(comp.data_ptr(), gu.to_dev(offs).data_ptr(), gu.to_dev(sizes).data_ptr(),
                                         out.data_ptr(), None, stride, None, cap, ret.data_ptr(), n, ws.data_ptr(), wsb,
                                         stream()) == 0
    torch.cuda.synchronize()
    rows = out.view(n, stride)
    r0, w0 = oracle.decompress(common, cap)
    assert r0 == cap
    want0 = dev_u8(w0)
    for a in range(0, n - len(last), 64):
        b = min(a + 64, n - len(last))
        assert torch.equal(rows[a:b, :cap], want0.expand(b - a, cap)), "blocks %d.." % a
    assert bool((rows[:, cap:] == SENT).all())
    rets = ret.cpu().numpy()
    assert (rets[:n - len(last)] == cap).all()
    for j, blk in enumerate(last):
        i = n - len(last) + j
        er, eo = oracle.decompress(blk, cap)
        assert rets[i] == er and er > 0, (i, rets[i], er)
        assert rows[i, :er].cpu().numpy().tobytes() == eo, i
        assert bool((rows[i, er:cap] == SENT).all()), i
    res = gu.Decoded()
    res.ws = ws
    nseq, slow = gu.ws_lists(ws, n)
    marks, tile_first = gu.wide_workspace(res, n, cap)
    assert (nseq[:n - len(last)] == nseq[0]).all()
    marks0 = marks(0, int(nseq[0]))
    for b in (511, 512, n - len(last) - 1):                  # marks of blocks 512 and up lie past 2^32
        assert (marks(b, int(nseq[b])) == marks0).all(), b
    nt = (cap + 61439) // 61440
    first0 = [int(v) for v in tile_first(0, nt)]
    assert first0[0] == 0 and first0[-1] == nseq[0]
    for b in (511, 512, 513, n - len(last) - 1):            # the repeated block's index, however far its entries lie
        assert [int(v) for v in tile_first(b, nt)] == first0, b
    assert len(slow) == 0 or set(slow.tolist()) <= set(range(n - len(last), n)), slow


# ------------------------------------------------------------------------------------------
# compressors and pack kernels at far strides
# ------------------------------------------------------------------------------------------
SRC_STRIDE = L31 + MiB + 3
DST_STRIDE = L31 + 2 * MiB + 5
DST_ORG = 7


def compress_far(lib, ar, raws, room, call):
    """Put raws at SRC_ORG + i * SRC_STRIDE, run call(src, dst, sizes, ret, consumed) with slot i at
    DST_ORG + i * DST_STRIDE and return (ret, consumed, slot bytes [0, ret)) per block"""
    n = len(raws)
    for i, r in enumerate(raws):
        ar.put(SRC_ORG + i * SRC_STRIDE, r)
        ar.far(SRC_ORG, i * SRC_STRIDE, len(r))
    sizes = torch.tensor([len(r) for r in raws], dtype=torch.int32, device=DEV)
    ret = torch.full((n,), UNWRITTEN, dtype=torch.int32, device=DEV)
    cons = torch.full((n,), UNWRITTEN, dtype=torch.int32, device=DEV)
    assert call(ar.ptr(SRC_ORG), ar.ptr(DST_ORG), sizes.data_ptr(), ret.data_ptr(), cons.data_ptr()) == 0
    torch.cuda.synchronize()
    rets, cs = ret.cpu().numpy(), cons.cpu().numpy()
    out = []
    for i in range(n):
        at = DST_ORG + i * DST_STRIDE
        out.append((int(rets[i]), int(cs[i]), ar.view(at, max(int(rets[i]), 0)).cpu().numpy().tobytes()))
        ar.far(DST_ORG, i * DST_STRIDE, room)
    return out


def check_slots(ar, want_bytes, room, loose):
    """the model: each slot's returned bytes, then sentinel to its room and past it; `loose`: the bytes between the
    returned ones and the room may hold anything"""
    dont = []
    for i, b in enumerate(want_bytes):
        at = DST_ORG + i * DST_STRIDE
        ar.expect(at, b if loose else b + bytes([SENT]) * (room - len(b)))
        if loose and room > len(b):
            dont.append((at + len(b), room - len(b)))
    ar.check(dont)


def test_compressors_at_far_strides(lib, oracle):
    """The exact, destSize and parallel compressors at srcStride and dstStride of about 2^31 + odd: blocks 1 and 2 past
    2^31 and 2^32, guard bytes past every slot's room."""
    st = stream()
    raws = [bytes(oracle.datagen(65536 - 11 * k, 0.5, 90 + k)) for k in range(3)]
    cap = mg.compress_bound(65536)
    ar = Arena()
    got = compress_far(lib, ar, raws, cap, lambda s, d, sz, r, c: lib.LZ4B200_compress_blocks(
        s, SRC_STRIDE, sz, 0, d, DST_STRIDE, cap, 1, r, 3, st))
    want = [oracle.compress(r, 1, cap) for r in raws]
    assert [(g[0], g[2]) for g in got] == want
    check_slots(ar, [w[1] for w in want], cap, False)
    del ar
    torch.cuda.empty_cache()

    target = 20000
    ar = Arena()
    got = compress_far(lib, ar, raws, target, lambda s, d, sz, r, c: lib.LZ4B200_compress_blocks_destSize(
        s, SRC_STRIDE, sz, 0, d, DST_STRIDE, target, 1, r, c, 3, st))
    want = [oracle.compress_dest_size(r, target, 1)[:3] for r in raws]
    assert [tuple(g) for g in got] == want
    check_slots(ar, [w[2] for w in want], target, False)
    del ar
    torch.cuda.empty_cache()

    # the parallel compressor: one launch (all blocks <= 64 KB), then one per block size (blocks above 64 KB are the
    # byte-identical encoder's)
    for raws_p in (raws, [raws[0], bytes(oracle.datagen(100000, 0.5, 95)), raws[2][:30000]]):
        capp = mg.compress_bound(max(len(r) for r in raws_p))
        ar = Arena()
        got = compress_far(lib, ar, raws_p, capp, lambda s, d, sz, r, c: lib.LZ4B200_compress_blocks_parallel(
            s, SRC_STRIDE, sz, 0, d, DST_STRIDE, capp, 1, r, 3, st))
        want = [M.compress(r, 1, capp, oracle) for r in raws_p]
        assert [(g[0], g[2]) for g in got] == [(w.ret, w.out) for w in want]
        check_slots(ar, [w.out for w in want], capp, False)
        del ar
        torch.cuda.empty_cache()


HC_CALLS = ("hc", "hc_dest", "hc_opt", "hc_opt_dest")


@pytest.mark.parametrize("call", HC_CALLS)
def test_hc_calls_at_far_strides(lib, oracle, call):
    """The four HC calls at srcStride and dstStride of about 2^31 + odd against the host build, on golden inputs whose
    return value at the bound is pinned."""
    import hc_emul as he
    opt = "opt" in call
    fill = call.endswith("dest")
    level = 12 if opt else 9
    doc, ins = he.golden("kat_hc_opt.json" if opt else "kat_hc.json")
    picks = [(iid, rb) for iid, lv, rb, _, _ in doc["vectors"] if lv == level and 1000 <= ins[iid]["size"] <= 65536][:3]
    assert len(picks) == 3
    raws = [bytes(mg.make_input(oracle, ins[iid]["size"], ins[iid]["kind"], ins[iid]["seed"])) for iid, _ in picks]
    limit = 4096 if fill else mg.compress_bound(65536)
    nws = getattr(lib, "LZ4B200_compress_blocks_%sworkspace_bytes" % ("hc_opt_" if opt else "hc_"))(3)
    ws = torch.empty(int(nws), dtype=torch.uint8, device=DEV)
    fn = getattr(lib, "LZ4B200_compress_blocks_" + {"hc": "hc", "hc_dest": "hc_destSize", "hc_opt": "hc_opt",
                                                   "hc_opt_dest": "hc_opt_destSize"}[call])
    st = stream()
    ar = Arena()
    if fill:
        got = compress_far(lib, ar, raws, limit, lambda s, d, sz, r, c: fn(
            s, SRC_STRIDE, sz, 0, d, DST_STRIDE, limit, level, r, c, 3, ws.data_ptr(), int(nws), st))
        want = [(host_hc_opt_dest if opt else host_hc_dest)(r, limit, level) for r in raws]
        assert [tuple(g) for g in got] == want
        check_slots(ar, [w[2] for w in want], limit, True)
    else:
        got = compress_far(lib, ar, raws, limit, lambda s, d, sz, r, c: fn(
            s, SRC_STRIDE, sz, 0, d, DST_STRIDE, limit, level, r, 3, ws.data_ptr(), int(nws), st))
        want = [(host_hc_opt if opt else host_hc)(r, limit, level) for r in raws]
        assert [(g[0], g[2]) for g in got] == want
        assert [g[0] for g in got] == [rb for _, rb in picks], "the golden return values at the bound"
        check_slots(ar, [w[1] for w in want], limit, True)


@pytest.mark.parametrize("call,level", [("hc", 3), ("hc", 9), ("hc_dest", 3), ("hc_dest", 9),
                                        ("hc_opt", 10), ("hc_opt", 12), ("hc_opt_dest", 10), ("hc_opt_dest", 12)])
def test_hc_workspace_slots_past_the_lines(lib, oracle, call, level):
    """16 384 + 37 blocks of 1 .. 4 KB on the minimum workspace: all 16 384 slots run, slots 8 192 and up start past
    2^31 (HC-opt: 6 553 and up past 2^31, 13 106 and up past 2^32), slots 0 .. 36 take a second block.  Every block on a slot past 2^31 and 64
    others against the host build (levels 3 and 9, whose host parse is slow: a sample, and all of them against
    calls of 4 096 blocks, whose slots lie below 2^31); every block through an oracle round trip."""
    opt = "opt" in call
    fill = call.endswith("dest")
    n = 16384 + 37
    slot_bytes = 262144 + (4099 * 16 if opt else 0)
    wsb = int(getattr(lib, "LZ4B200_compress_blocks_%sworkspace_bytes" % ("hc_opt_" if opt else "hc_"))(n))
    assert wsb == 16384 * slot_bytes
    need(wsb + 256 * MiB)
    rng = np.random.default_rng(level)
    sizes_h = rng.integers(1024, 4097, n).astype(np.int32)
    data = oracle.datagen(n * 4096, 0.5, 300 + level)
    src = dev_u8(np.concatenate([data, np.zeros(16, np.uint8)]))
    limit = 1500 if fill else mg.compress_bound(4096)
    dst_stride = mg.compress_bound(4096) + 3
    fn = getattr(lib, "LZ4B200_compress_blocks_" + {"hc": "hc", "hc_dest": "hc_destSize", "hc_opt": "hc_opt",
                                                   "hc_opt_dest": "hc_opt_destSize"}[call])
    sizes = gu.to_dev(sizes_h)

    def run(lo, hi):
        """blocks [lo, hi) in one call on the minimum workspace: (ret, consumed, slots)"""
        m = hi - lo
        nbytes = int(getattr(lib, "LZ4B200_compress_blocks_%sworkspace_bytes" % ("hc_opt_" if opt else "hc_"))(m))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        dst = torch.full((m * dst_stride + 16,), SENT, dtype=torch.uint8, device=DEV)
        ret = torch.full((m,), UNWRITTEN, dtype=torch.int32, device=DEV)
        cons = torch.full((m,), UNWRITTEN, dtype=torch.int32, device=DEV)
        tail = (ret.data_ptr(), cons.data_ptr()) if fill else (ret.data_ptr(),)
        assert fn(src.data_ptr() + lo * 4096, 4096, sizes.data_ptr() + 4 * lo, 0, dst.data_ptr(), dst_stride, limit,
                  level, *tail, m, ws.data_ptr(), nbytes, stream()) == 0
        torch.cuda.synchronize()
        del ws
        torch.cuda.empty_cache()
        return ret.cpu().numpy(), cons.cpu().numpy(), dst.cpu().numpy()[:m * dst_stride]

    ret, cons, dst = run(0, n)
    assert (ret != UNWRITTEN).all() and (ret > 0).all()
    blk = lambda i: data[i * 4096:i * 4096 + sizes_h[i]].tobytes()
    outb = lambda d, r, i: d[i * dst_stride:i * dst_stride + int(r[i])].tobytes()
    for i in range(n):                                      # the oracle round trip
        c = int(cons[i]) if fill else int(sizes_h[i])
        assert oracle.decompress(outb(dst, ret, i), c) == (c, blk(i)[:c]), i
        assert (dst[i * dst_stride + min(limit, mg.compress_bound(int(sizes_h[i]))):(i + 1) * dst_stride] == SENT).all(), i
    far_slots = [i for i in range(n) if (i % 16384) * slot_bytes >= L31]
    assert far_slots[0] == (6553 if opt else 8192) and (not opt or far_slots.index(13106) > 0)
    # the 37 pairs that share a slot, and 27 more below 2^31
    others = sorted(set(range(37)) | set(range(16384, n)) | set(rng.choice(np.arange(37, 8192), 27, replace=False).tolist()))
    if opt:
        check = far_slots + others
    else:
        # the same blocks in calls of 4 096, whose workspaces (1 GiB) end below 2^31
        parts = [run(a, min(a + 4096, n)) for a in range(0, n, 4096)]
        small_ret, small_cons, small_dst = (np.concatenate([p[j] for p in parts]) for j in range(3))
        for i in range(n):
            assert (ret[i], cons[i] if fill else 0, outb(dst, ret, i)) == \
                (small_ret[i], small_cons[i] if fill else 0, outb(small_dst, small_ret, i)), i
        check = [8192, 13105, 13106, 16383] + others[:12]
    for i in check:
        if fill:
            host = (host_hc_opt_dest if opt else host_hc_dest)(blk(i), limit, level)
            assert (int(ret[i]), int(cons[i]), outb(dst, ret, i)) == host, i
        else:
            host = (host_hc_opt if opt else host_hc)(blk(i), limit, level)
            assert (int(ret[i]), outb(dst, ret, i)) == host, i


PACK_STRIDE = L31 + 3 * MiB + 1


@pytest.mark.parametrize("frame,header", [(False, 0), (False, 4), (True, 4)])
def test_pack_at_far_strides(lib, oracle, frame, header):
    """LZ4B200_pack_blocks (headers 0 and 4) and LZ4B200_pack_frame_blocks with slotStride and rawStride of about
    2^31 + odd, against gu.pack_model"""
    n = 3
    ar = Arena()
    sizes = np.array([40000, 0, 65536], dtype=np.int32) if frame else np.array([40000, 1, 65521], dtype=np.int32)
    slots = [bytes(oracle.datagen(65536, 0.3, 120 + i)) for i in range(n)]
    raw = [bytes(oracle.datagen(65536, 0.7, 130 + i)) for i in range(n)]
    for i in range(n):
        ar.put(DST_ORG + i * PACK_STRIDE, slots[i])
        ar.far(DST_ORG, i * PACK_STRIDE, 65536)
        if frame:
            ar.put(SRC_ORG + i * PACK_STRIDE, raw[i])
            ar.far(SRC_ORG, i * PACK_STRIDE, 65536)
    compact = b"".join(slots)
    fr = (b"".join(raw), 65536, 65536, 0) if frame else None
    want_off, want = gu.pack_model(compact, 65536, sizes, header, fr)
    d_sizes = gu.to_dev(sizes)
    packed = torch.full((len(want) + 64,), SENT, dtype=torch.uint8, device=DEV)
    off = torch.full((n + 1,), -1, dtype=torch.int64, device=DEV)
    if frame:
        rc = lib.LZ4B200_pack_frame_blocks(ar.ptr(DST_ORG), PACK_STRIDE, d_sizes.data_ptr(), ar.ptr(SRC_ORG),
                                           PACK_STRIDE, 65536, 0, n, packed.data_ptr(), off.data_ptr(), stream())
    else:
        rc = lib.LZ4B200_pack_blocks(ar.ptr(DST_ORG), PACK_STRIDE, d_sizes.data_ptr(), n, packed.data_ptr(),
                                     off.data_ptr(), header, stream())
    assert rc == 0
    torch.cuda.synchronize()
    assert (off.cpu().numpy() == want_off).all()
    p = packed.cpu().numpy()
    assert p[:len(want)].tobytes() == want and (p[len(want):] == SENT).all()
    ar.check()


@pytest.mark.parametrize("frame", [False, True])
def test_pack_output_past_4_gib_from_one_slot(lib, oracle, frame):
    """slotStride = 0 (and rawStride = 0): 66 000 blocks from one slot, more than 4 GiB of packed output.  outOff
    against an int64 cumsum, the headers past 2^32 and the payloads, all on the device."""
    n = 66000
    bs = 65552
    pays = np.where(np.arange(n) % 2 == 0, 65536, bs) if frame else np.full(n, 65536)
    total = int((pays + 4).sum())
    assert total > L32
    need(total + 2 * GiB)
    slot = dev_u8(oracle.datagen(bs + 16, 0.5, 140))
    raw = dev_u8(oracle.datagen(bs + 16, 0.5, 141))
    sizes = torch.full((n,), 65536, dtype=torch.int32, device=DEV)
    if frame:
        sizes[1::2] = 0                                         # did not fit: stored raw
    packed = torch.full((total + 64,), SENT, dtype=torch.uint8, device=DEV)
    off = torch.full((n + 1,), -1, dtype=torch.int64, device=DEV)
    if frame:
        rc = lib.LZ4B200_pack_frame_blocks(slot.data_ptr(), 0, sizes.data_ptr(), raw.data_ptr(), 0, bs, 0, n,
                                           packed.data_ptr(), off.data_ptr(), stream())
    else:
        rc = lib.LZ4B200_pack_blocks(slot.data_ptr(), 0, sizes.data_ptr(), n, packed.data_ptr(), off.data_ptr(), 4,
                                     stream())
    assert rc == 0
    torch.cuda.synchronize()
    want_off = torch.zeros(n + 1, dtype=torch.int64, device=DEV)
    want_off[1:] = torch.cumsum(torch.as_tensor(pays + 4, device=DEV), 0)
    assert torch.equal(off, want_off)
    hdr = lambda v: torch.tensor(list(int(v).to_bytes(4, "little")), dtype=torch.uint8, device=DEV)
    if frame:                                  # pairs: [65536][slot 65536][65552 | raw bit][raw 65552]
        row = torch.cat([hdr(65536), slot[:65536], hdr(bs | 0x80000000), raw[:bs]])
    else:
        row = torch.cat([hdr(65536), slot[:65536]])
    per = row.numel()
    rows = packed[:total].view(-1, per)
    for a in range(0, rows.shape[0], 4096):
        chunk = rows[a:a + 4096]
        assert torch.equal(chunk, row.expand_as(chunk)), "rows %d.." % a
    assert bool((packed[total:] == SENT).all())
    far = [k for k in range(n) if int(want_off[k]) >= L32][:3]
    assert far, "no block past 2^32"
    for k in far:
        o = int(want_off[k])
        h = int(pays[k]) | (0x80000000 if frame and k % 2 else 0)
        assert packed[o:o + 4].cpu().numpy().tobytes() == h.to_bytes(4, "little"), k


# ------------------------------------------------------------------------------------------
# blocks of up to INT_MAX bytes
# ------------------------------------------------------------------------------------------
INT_MAX = L31 - 1
PERIOD = 4096


def long_block(total, prefix):
    """literals `prefix` (PERIOD bytes), one match at offset PERIOD that brings the output to total - 16, then 16
    literals: decodes to [(prefix, total - 16), (tail, 16)] (pattern, bytes: the pattern repeated)"""
    tail = bytes(range(200, 216))
    return gu.lz4_seq(prefix, PERIOD, total - 16 - PERIOD) + gu.lz4_seq(tail, None), [(prefix, total - 16), (tail, 16)]


def long_length(ext_sum, field):
    """a block whose literal-length (field="lit") or match-length ("match") continuation of 0xFF bytes sums past ext_sum:
    the literals run past the input; the match (4 literals 0x07, offset 4) is decoded if it fits the capacity, then 5
    literals 0x01.  Returns (block, closed form of what it decodes to if valid)."""
    k = ext_sum // 255 + 1
    if field == "lit":
        return bytes([0xF0]) + b"\xff" * k + b"\x00" + b"\x07" * 64, None
    ml = 4 + 15 + 255 * k
    blk = bytes([0x4F]) + b"\x07" * 4 + bytes([4, 0]) + b"\xff" * k + b"\x00" + bytes([0x50]) + b"\x01" * 5
    return blk, [(b"\x07", 4 + ml), (b"\x01", 5)]


def check_closed_form(out, pieces):
    """out[0 ..] on the device against pieces (pattern, bytes): each pattern repeated over its bytes"""
    at = 0
    for pat, n in pieces:
        p = dev_u8(pat)
        reps = n // len(pat)
        for a in range(0, reps, 1 << 16):
            b = min(a + (1 << 16), reps)
            seg = out[at + a * len(pat):at + b * len(pat)].view(b - a, len(pat))
            assert torch.equal(seg, p.expand(b - a, len(pat))), (at, a)
        rest = n - reps * len(pat)
        assert torch.equal(out[at + reps * len(pat):at + n], p[:rest])
        at += n
    return at


def test_blocks_up_to_int_max(lib, oracle):
    """One block, capacity 2^31 - 1 (R6: the parallel scan, then the generic kernel): a valid block that decodes to
    2^31 - 1 - k bytes, the same block one byte short of capacity, and blocks whose literal-length or match-length
    continuations sum past 2^28 (the scan's run-length guard), 2^31 and 2^32 (about 8.4 MB and 16.8 MB of input).
    Return values against the oracle; the bytes of accepted blocks against their closed form on the device, and nothing
    written by a rejected one."""
    total = INT_MAX - 5
    need(L31 + 256 * MiB)
    prefix = bytes(np.random.default_rng(3).integers(1, 256, PERIOD, dtype=np.uint8))
    blk, pieces = long_block(total, prefix)
    cases = [(blk, INT_MAX, pieces), (blk, total - 1, pieces)]
    for s in (1 << 28, L31, L32):
        for field in ("lit", "match"):
            b, form = long_length(s, field)
            cases.append((b, INT_MAX, form))
    out = torch.empty(INT_MAX + 16, dtype=torch.uint8, device=DEV)
    verdicts = []
    for blk_i, cap, form in cases:
        er = oracle.decompress(blk_i, cap)[0]
        out[:64].fill_(SENT)
        out[total:].fill_(SENT)
        comp = dev_u8(b"\x00" * 16 + blk_i + b"\x00" * 16)
        offs = torch.tensor([16], dtype=torch.int64, device=DEV)
        sizes = torch.tensor([len(blk_i)], dtype=torch.int32, device=DEV)
        ret = torch.full((1,), UNWRITTEN, dtype=torch.int32, device=DEV)
        wsb = int(lib.LZ4B200_decompress_workspace_bytes_for(1, 0, cap))
        assert gu.route(1, cap, ws_bytes=wsb) == "R6"
        ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
        assert lib.LZ4B200_decompress_blocks(comp.data_ptr(), offs.data_ptr(), sizes.data_ptr(), out.data_ptr(), None,
                                             0, None, cap, ret.data_ptr(), 1, ws.data_ptr(), wsb, stream()) == 0
        torch.cuda.synchronize()
        r = int(ret[0])
        assert r == er, (len(blk_i), cap, r, er)
        verdicts.append(r)
        if r < 0:
            assert bool((out[:64] == SENT).all()), "a rejected block wrote"
        else:
            assert check_closed_form(out, form) == r
            if r == total:
                assert bool((out[total:] == SENT).all()), "wrote past the return value"
        del comp, ws
    assert verdicts[0] == total and verdicts[1] < 0
    assert verdicts[3] == 4 + 4 + 15 + 255 * ((1 << 28) // 255 + 1) + 5, "the 2^28 match fits the capacity"
    assert all(v < 0 for v in verdicts[4:]) and verdicts[2] < 0


def test_compressors_refuse_a_size_past_the_max_input(lib):
    """LZ4_MAX_INPUT_SIZE + 1 returns 0 and writes nothing in the exact, destSize and HC batch calls"""
    n = 0x7E000000 + 1
    need(n + 512 * MiB)
    src = torch.zeros(n + 16, dtype=torch.uint8, device=DEV)
    dst = torch.full((1 << 20,), SENT, dtype=torch.uint8, device=DEV)
    ret = torch.full((1,), UNWRITTEN, dtype=torch.int32, device=DEV)
    cons = torch.full((1,), UNWRITTEN, dtype=torch.int32, device=DEV)
    st = stream()
    ws = torch.empty(int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(1)), dtype=torch.uint8, device=DEV)
    cap = 1 << 19
    calls = [
        lambda: lib.LZ4B200_compress_blocks(src.data_ptr(), 0, None, n, dst.data_ptr(), cap, cap, 1, ret.data_ptr(), 1, st),
        lambda: lib.LZ4B200_compress_blocks_destSize(src.data_ptr(), 0, None, n, dst.data_ptr(), cap, cap, 1,
                                                     ret.data_ptr(), cons.data_ptr(), 1, st),
        lambda: lib.LZ4B200_compress_blocks_hc(src.data_ptr(), 0, None, n, dst.data_ptr(), cap, cap, 9, ret.data_ptr(),
                                               1, ws.data_ptr(), ws.numel(), st),
        lambda: lib.LZ4B200_compress_blocks_hc_destSize(src.data_ptr(), 0, None, n, dst.data_ptr(), cap, cap, 9,
                                                        ret.data_ptr(), cons.data_ptr(), 1, ws.data_ptr(), ws.numel(), st),
        lambda: lib.LZ4B200_compress_blocks_hc_opt(src.data_ptr(), 0, None, n, dst.data_ptr(), cap, cap, 12,
                                                   ret.data_ptr(), 1, ws.data_ptr(), ws.numel(), st),
        lambda: lib.LZ4B200_compress_blocks_hc_opt_destSize(src.data_ptr(), 0, None, n, dst.data_ptr(), cap, cap, 12,
                                                            ret.data_ptr(), cons.data_ptr(), 1, ws.data_ptr(),
                                                            ws.numel(), st),
    ]
    for j, call in enumerate(calls):
        ret.fill_(UNWRITTEN)
        assert call() == 0, j
        torch.cuda.synchronize()
        assert int(ret[0]) == 0, (j, int(ret[0]))
        assert bool((dst == SENT).all()), j


# ------------------------------------------------------------------------------------------
# host buffers past 4 GiB
# ------------------------------------------------------------------------------------------
def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def test_host_decode_into_a_pageable_buffer_past_4_gib(lib, oracle):
    """LZ4B200_decompress_blocks_host over 66 000 blocks that share one compressed block, into a pageable host
    destination larger than 4 GiB"""
    n, cap = 66000, 65536
    if mem_available() < 6 * GiB:
        pytest.skip("needs about 6 GB of free host memory, %.1f GB available" % (mem_available() / 1e9))
    with open(gu.__file__.replace("gpu_util.py", "golden/p50_seed0_64k.lz4block"), "rb") as f:
        blk = f.read()
    r, want = oracle.decompress(blk, cap)
    src = np.frombuffer(b"\x00" * 16 + blk + b"\x00" * 16, np.uint8).copy()
    offs = np.full(n, 16, dtype=np.int64)
    sizes = np.full(n, len(blk), dtype=np.int32)
    dst = np.full(n * cap + 64, SENT, dtype=np.uint8)
    assert dst.nbytes > L32
    rets = np.full(n, UNWRITTEN, dtype=np.int32)
    rc = lib.LZ4B200_decompress_blocks_host(src.ctypes.data, offs.ctypes.data, sizes.ctypes.data, dst.ctypes.data, cap,
                                            cap, rets.ctypes.data, n)
    assert rc == 0
    assert (rets == r).all()
    rows = dst[:n * cap].reshape(n, cap)
    w = np.frombuffer(want, np.uint8)
    for a in range(0, n, 4096):
        assert (rows[a:a + 4096] == w).all(), a
    assert (dst[n * cap:] == SENT).all()
    del dst, rows
