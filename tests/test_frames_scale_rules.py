"""The batched frame decode at scale without a GPU, and the frames tests/test_gpu_frames_scale.py decodes on the GPU.

Frames built here:
  - the many-frame batches: 4 095 .. 16 389 small frames of every class (most of them 64 KB), with empty frames,
    stored-raw blocks, checksummed frames and frames that fail at the header, in the chain, in a block or at a checksum,
    and the budgets that put each class's first LZ4B200_ERR_LIMIT on chosen frames of lz4_frames_scan_kernel's rounds
    (1 024 threads x 4 frames);
  - the far frame: one 64 KB-class frame of 65 540 blocks whose content passes 2^32 bytes, with its content size and
    content checksum.  Block i decodes to its index (8 bytes, little endian) and then a fill byte of its own, so every
    block differs from its neighbours; the compressed blocks are 275 bytes, so the frame is 18 MB.
    tests/golden/frames_scale.json holds the reference's digests of its content and its LZ4F_decompress outcome.

The tests here check the host build of fc_xxh32 on the far content against the reference's digest, the index passes on
the far frame with its source past 2^32, and that the index passes put LZ4B200_ERR_LIMIT where the batches plan it."""
import ctypes as C
import hashlib
import struct

import numpy as np
import pytest

import frame_checksum_model as fm
import frame_corpus as fc
import host_build
from conftest import load_golden

BLOCK = 65536
L32 = 1 << 32
REJECT, SKIP, VERIFY = 0, 1, 2                      # FC_SUMS_* (lz4_frame_core.h); "plain": LZ4B200_decompress_frames
MODES = {"plain": REJECT, "skip": SKIP, "verify": VERIFY}
INDEPENDENT = (1 << 6) | (1 << 5)                   # FLG: version 01, independent blocks

# ------------------------------------------------------------------------------------------
# the far frame
# ------------------------------------------------------------------------------------------
FAR_FULL = 65539                                    # full 64 KB blocks, then a short compressed one
FAR_TAIL = 19
FAR_BLOCKS = FAR_FULL + 1
FAR_SIZE = FAR_FULL * BLOCK + FAR_TAIL              # 2^32 + 3 x 65 536 + 19
FAR_RAW = frozenset(range(4097, FAR_FULL, 8192))    # stored-raw blocks (8), the first at 2^28 + 64 KB


def far_fill(i):
    return (i * 37 + 11) & 0xFF


def run_block(lead, fill, n):
    """an LZ4 block of n >= 18 bytes: the 8 lead bytes and one fill byte as literals, a match at offset 1 that repeats the
    fill byte, five literal fill bytes"""
    ml = n - 14
    v = ml - 4
    ext = b"" if v < 15 else b"\xff" * ((v - 15) // 255) + bytes([(v - 15) % 255])
    return bytes([(9 << 4) | min(v, 15)]) + lead + bytes([fill]) + b"\x01\x00" + ext + bytes([0x50]) + bytes([fill]) * 5


def far_frame(xxh, content_size=FAR_SIZE):
    """the far frame with content checksum xxh; content_size: the header's content-size field"""
    out = [fc.header(INDEPENDENT | 8 | fm.FLG_CONTENT_SUM, 4 << 4, content_size)]
    for i in range(FAR_BLOCKS):
        n = BLOCK if i < FAR_FULL else FAR_TAIL
        lead = struct.pack("<Q", i)
        if i in FAR_RAW:
            out.append(struct.pack("<I", n | 0x80000000) + lead + bytes([far_fill(i)]) * (n - 8))
        else:
            p = run_block(lead, far_fill(i), n)
            out.append(struct.pack("<I", len(p)) + p)
    out.append(struct.pack("<II", 0, xxh))
    return b"".join(out)


def far_content():
    """the far frame's content, FAR_SIZE bytes (numpy)"""
    buf = np.empty(FAR_SIZE, dtype=np.uint8)
    idx = np.arange(FAR_BLOCKS, dtype="<u8")
    fill = far_fill(idx).astype(np.uint8)
    full = buf[:FAR_FULL * BLOCK].reshape(FAR_FULL, BLOCK)
    full[:, 8:] = fill[:FAR_FULL, None]
    full[:, :8] = idx[:FAR_FULL].view(np.uint8).reshape(-1, 8)
    tail = buf[FAR_FULL * BLOCK:]
    tail[8:] = fill[-1]
    tail[:8] = idx[-1:].view(np.uint8)
    return buf


# ------------------------------------------------------------------------------------------
# the many-frame batches
# ------------------------------------------------------------------------------------------
SCAN_ROUND = 4096                                   # frames per round of lz4_frames_scan_kernel
BATCHES = [4095, 4096, 4097, 3 * 4096 + 5, 4 * 4096 + 5]


def limit_targets(n):
    """where a class's first LZ4B200_ERR_LIMIT goes in a batch of n: 4 095 (the last item of thread 1 023 in round 0),
    4 096 (the first frame of round 1), item 2 or 3 of a thread in the last full round from round 2 on, the last frame"""
    t = [4095, 4096]
    full = n // SCAN_ROUND
    if full >= 3:
        t.append((full - 1) * SCAN_ROUND + 4 * 37 + 2 + full % 2)
    t.append(n - 1)
    return sorted({x for x in t if x < n})


class Entry:
    """one distinct frame of the pool: bytes, capacity, class (-1: fails at the header in every mode), valid blocks of its
    chain, whether the chain reaches its end, its checksum flags"""

    def __init__(self, frame, cap, cls, blocks, complete=True):
        self.frame, self.cap, self.cls, self.blocks, self.complete = frame, cap, cls, blocks, complete
        self.sums = cls >= 0 and bool(frame[4] & (fm.FLG_BLOCK_SUM | fm.FLG_CONTENT_SUM))

    def pass1(self, mode):
        """(class, valid blocks, complete) as the index pass sees it without a budget; class -1: failed at the header"""
        if self.cls < 0 or (self.sums and mode == "plain"):
            return -1, 0, False
        return self.cls, self.blocks, self.complete


_pools = {}


def pool(oracle):
    """(weights, entries, anchors): the distinct frames of the batches; anchors[c]: a one-block frame of class c"""
    if "pool" in _pools:
        return _pools["pool"]
    rng = np.random.default_rng(1234)
    d = oracle.datagen(1 << 16, 0.5, 77).tobytes()
    noise = rng.integers(0, 256, 4096, dtype=np.uint8).tobytes()
    ents, weights = [], []

    def add(w, e):
        weights.append(w)
        ents.append(e)

    def frame(bsid, pieces, raw=(), bsum=False, csum=False, csize=True):
        total = sum(len(p) for p in pieces)
        return fm.frame_of_blocks(oracle, pieces, bsid, raw=raw, block_sum=bsum, content_sum=csum,
                                  content_size=total if csize else None), total

    for k in range(24):                              # 64 KB class: one or two blocks, hundreds of bytes to a few KB
        a = int(rng.integers(0, 60000))
        n1, n2 = int(rng.integers(200, 3000)), int(rng.integers(0, 1500))
        pieces = [d[a:a + n1]] + ([noise[:n2] if k % 3 == 0 else d[a + n1:a + n1 + n2]] if n2 > 100 else [])
        bsum, csum = k % 4 == 1 or k % 4 == 3, k % 4 >= 2
        f, total = frame(4, pieces, raw=(1,) if k % 3 == 0 else (), bsum=bsum, csum=csum, csize=k % 2 == 0)
        add(20, Entry(f, total + int(rng.integers(0, 100)), 0, len(pieces)))
    for bsid, w in ((5, 1.0), (6, 0.5), (7, 0.25)):  # the larger classes: rare, small
        for k in range(3):
            pieces = [d[1000 * k:1000 * k + 700 + 300 * bsid]] + ([noise[:500]] if k == 1 else [])
            f, total = frame(bsid, pieces, raw=(1,) if k == 1 else (), csum=k == 2, csize=k != 0)
            add(w, Entry(f, total, bsid - 4, len(pieces)))
    for bsid in (4, 5, 6, 7):                        # empty frames: no blocks
        add(2 if bsid == 4 else 0.3, Entry(frame(bsid, [], csize=False)[0], 1, bsid - 4, 0))
    add(2, Entry(frame(4, [], csum=True, csize=False)[0], 1, 0, 0))
    good, total = frame(4, [d[:1500], noise[:300]], raw=(1,))
    add(1, Entry(b"\x05" + good[1:], total, -1, 0))                          # bad magic
    bad = bytearray(good)
    bad[fc.header_len(good) - 1] ^= 0x40
    add(1, Entry(bytes(bad), total, -1, 0))                                  # header checksum
    add(1, Entry(frame(4, [], csize=False)[0][:-4], 1, 0, 0, False))        # chain: no EndMark, no block
    add(1, Entry(frame(6, [], csize=False)[0][:-2], 1, 2, 0, False))
    add(1, Entry(good[:fc.header_len(good) + 40], total, 0, 0, False))       # chain: cut inside the first block
    add(1, Entry(good, total - 1, 0, 2))                                     # LZ4B200_ERR_DSTSIZE
    hl = fc.header_len(good)
    add(1, Entry(good[:hl] + struct.pack("<I", 1) + b"\xf0" + struct.pack("<I", 0), total, 0, 1))   # malformed block
    f, total = frame(4, [d[5000:7000]], bsum=True, csum=True)
    b = bytearray(f)
    b[-1] ^= 0x10                                                            # content checksum
    add(1, Entry(bytes(b), total, 0, 1))
    b = bytearray(f)
    b[hl + 4 + 10] ^= 0x10                                                   # compressed payload: block checksum
    add(1, Entry(bytes(b), total, 0, 1))
    anchors = [Entry(frame(4 + c, [d[9000:9000 + 400 + 100 * c]])[0], 400 + 100 * c, c, 1) for c in range(4)]
    w = np.array(weights, dtype=np.float64)
    _pools["pool"] = (w / w.sum(), ents, anchors)
    return _pools["pool"]


def many_batch(oracle, n, rot=0):
    """n entries: seeded picks from the pool, and anchors[(j + rot) % 4] at limit_targets(n)[j]"""
    p, ents, anchors = pool(oracle)
    pick = np.random.default_rng(n).choice(len(ents), size=n, p=p)
    batch = [ents[i] for i in pick]
    for j, t in enumerate(limit_targets(n)):
        batch[t] = anchors[(j + rot) % 4]
    return batch


def plan(batch, mode, budget):
    """per entry: LZ4B200_ERR_LIMIT where the budget rule puts it, else None (the frame's own result); the chain walk
    stops after budget + 1 blocks (fc.budget_rule, with the pass the mode runs)"""
    run, out = [0, 0, 0, 0], []
    for e in batch:
        c, nb, complete = e.pass1(mode)
        if c < 0:
            out.append(None)
            continue
        if nb > budget[c]:
            k = budget[c] + 1
        elif not complete:
            out.append(None)
            continue
        else:
            k = nb
        out.append(fc.ERR_LIMIT if run[c] + k > budget[c] else None)
        run[c] += k
    return out


def need(batch, mode):
    n = [0, 0, 0, 0]
    for e in batch:
        c, nb, complete = e.pass1(mode)
        if c >= 0 and complete:
            n[c] += nb
    return n


def limit_budget(batch, mode, rot):
    """the budget that gives class (j + rot) % 4 its first LZ4B200_ERR_LIMIT at limit_targets(n)[j], and the other classes
    their need; returns (budget, {class: target})"""
    targets = limit_targets(len(batch))
    budget = need(batch, mode)
    want = {}
    for j, t in enumerate(targets):
        c = (j + rot) % 4
        before = need(batch[:t], mode)[c]
        budget[c] = before + batch[t].pass1(mode)[1] - 1
        want[c] = t
    return budget, want


def first_limits(status):
    """{class: first index with LZ4B200_ERR_LIMIT} of a status list paired with classes"""
    out = {}
    for f, (st, c) in enumerate(status):
        if st == fc.ERR_LIMIT and c not in out:
            out[c] = f
    return out


# ------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------
_ll, _llp, _ip = C.c_longlong, C.POINTER(C.c_longlong), C.POINTER(C.c_int)


def emul():
    h = host_build.require()
    h.frames_xxh32_host.restype = C.c_uint
    h.frames_xxh32_host.argtypes = [C.c_void_p, C.c_ulonglong, C.c_uint]
    fn = h.frames_index_mode_host
    fn.restype = _ll
    fn.argtypes = [C.c_void_p, _llp, _llp, _llp, _ll, _llp, C.c_int] + [_llp] * 7 + [_ip, _ip, _llp]
    return h


def index_mode(src_ptr, offs, sizes, caps, mb, mode):
    """frames_index_mode_host: frame f at src_ptr + offs[f]"""
    n = len(offs)
    P = lambda a, t: a.ctypes.data_as(C.POINTER(t))                                    # noqa: E731
    off, size, cap, mba = (np.array(x, dtype=np.int64) for x in (offs, sizes, caps, mb))
    outs = [np.zeros(n, dtype=np.int64) for _ in range(6)]
    ent = max(int(sum(mb)), 1)
    tso, tsz, trl, tmk = np.zeros(ent, np.int64), np.zeros(ent, np.int32), np.zeros(ent, np.int32), np.zeros(ent, np.int64)
    got = emul().frames_index_mode_host(src_ptr, P(off, _ll), P(size, _ll), P(cap, _ll), n, P(mba, _ll), mode,
                                        *[P(o, _ll) for o in outs], P(tso, _ll), P(tsz, C.c_int), P(trl, C.c_int),
                                        P(tmk, _ll))
    assert got == sum(mb)
    status, cls, count, base, consumed, sums = (o.tolist() for o in outs)
    return dict(status=status, cls=cls, count=count, base=base, consumed=consumed, sums=sums, tabSrcOff=tso,
                tabSrcSize=tsz, tabRawLen=trl, tabMark=tmk)


@pytest.fixture(scope="module")
def golden():
    return load_golden("frames_scale.json")


@pytest.fixture(scope="module")
def content():
    return far_content()


def test_far_content_digests(content, golden):
    """the content's SHA-256 and the host build of fc_xxh32 against the reference's XXH32: the 64-bit length path"""
    assert golden["content_size"] == FAR_SIZE > L32 + 3 * BLOCK + 17
    assert hashlib.sha256(memoryview(content)).hexdigest() == golden["sha256"]
    assert golden["xxh32"] == golden["xxh32_streamed"]
    assert emul().frames_xxh32_host(content.ctypes.data, FAR_SIZE, 0) == golden["xxh32"]


def test_far_frame_index_passes_past_4_gib(golden):
    """frames_index_mode_host on the far frame at a source offset past 2^32: the count and consumed length of the
    reference, and table entries at that offset plus each block's place in the frame"""
    f = far_frame(golden["xxh32"])
    assert len(f) == golden["frame_size"] and hashlib.sha256(f).hexdigest() == golden["frame_sha256"]
    assert golden["lz4f"]["error"] is None and golden["lz4f"]["size"] == FAR_SIZE
    blocks, consumed = fm.walk(f)
    assert consumed == golden["lz4f"]["consumed"] == len(f) and len(blocks) == FAR_BLOCKS
    buf = np.frombuffer(b"\0" * 16 + f + b"\0" * 16, dtype=np.uint8)
    far = L32 + 12345
    for mode in (SKIP, VERIFY):
        r = index_mode(buf.ctypes.data + 16 - far, [far], [len(f)], [FAR_SIZE], [FAR_BLOCKS, 0, 0, 0], mode)
        assert (r["status"], r["cls"], r["count"], r["consumed"]) == ([fc.OK], [0], [FAR_BLOCKS], [len(f)])
        assert r["tabSrcOff"].tolist() == [far + o for o, _, _ in blocks]
        assert r["tabRawLen"].tolist() == [sz if raw else -1 for _, sz, raw in blocks]
        assert r["tabSrcSize"].tolist() == [0 if raw else sz for _, sz, raw in blocks]
        assert not r["tabMark"].any()                       # no block checksums
    r = index_mode(buf.ctypes.data + 16 - far, [far], [len(f)], [FAR_SIZE], [FAR_BLOCKS - 1, 0, 0, 0], VERIFY)
    assert r["status"] == [fc.ERR_LIMIT] and r["consumed"] == [0]
    r = index_mode(buf.ctypes.data + 16 - far, [far], [len(f)], [FAR_SIZE], [FAR_BLOCKS, 0, 0, 0], REJECT)
    assert r["status"] == [fc.ERR_UNSUPPORTED]


def test_far_frame_blocks():
    """the hand-built blocks decode to the far content's pieces (the oracle's decoder)"""
    from oracle.pyoracle import Oracle
    o = Oracle()
    for i, n in ((0, BLOCK), (1, BLOCK), (FAR_FULL, FAR_TAIL)):
        lead = struct.pack("<Q", i)
        assert o.decompress(run_block(lead, far_fill(i), n), BLOCK) == (n, lead + bytes([far_fill(i)]) * (n - 8))
    assert len(run_block(lead, 1, BLOCK)) == 275


@pytest.mark.parametrize("n", BATCHES)
@pytest.mark.parametrize("mode", sorted(MODES))
def test_many_frame_batches_place_limit_where_planned(oracle, n, mode):
    """the index passes on every batch and rotation: the classes, counts and statuses the pool declares, and each
    class's first LZ4B200_ERR_LIMIT on its planned frame"""
    assert len(set(limit_targets(n))) >= 1 and max(limit_targets(n)) == n - 1
    for rot in range(4):
        batch = many_batch(oracle, n, rot)
        frames = [e.frame for e in batch]
        buf, offs = fc.layout(frames, seed=n)
        src = np.frombuffer(buf, dtype=np.uint8)
        caps = [e.cap for e in batch]
        full = need(batch, mode)
        r = index_mode(src.ctypes.data, offs, [len(f) for f in frames], caps, full, MODES[mode])
        for k, e in enumerate(batch):
            c, nb, complete = e.pass1(mode)
            assert r["cls"][k] == c, k
            if c >= 0 and complete:
                assert r["count"][k] == nb and r["status"][k] in (fc.OK,), k
            else:
                assert r["status"][k] not in (fc.OK, fc.ERR_LIMIT), k
        assert fc.ERR_LIMIT not in r["status"]
        budget, want = limit_budget(batch, mode, rot)
        r = index_mode(src.ctypes.data, offs, [len(f) for f in frames], caps, budget, MODES[mode])
        planned = plan(batch, mode, budget)
        assert first_limits(zip(planned, r["cls"])) == want
        assert first_limits(zip(r["status"], r["cls"])) == want
        for k, p in enumerate(planned):
            assert (r["status"][k] == fc.ERR_LIMIT) == (p == fc.ERR_LIMIT), k
