"""Routes R5 and R6 of lz4k_launch_decode (one capacity above 64 KB: the parallel scan, then the tile index and the tiles
kernel, or the generic kernel) on the corpus of tests/big_corpus.py, against the oracle, and the host pipeline and the
frame decoder over blocks of 256 KB .. 4 MB.

Every decode call asserts its route and goes through gpu_util.check_vs_oracle (return value incl. the negative error
position, bytes, and the untouched bytes of every slot past the return value).  It also checks:
  - the slow list: in R5 exactly the accepted blocks with a run-dense tile, in R6 every accepted block with output;
  - nSeq of every accepted block against the Python restatement (big_corpus.seq_list) and the one-thread scan (R1);
  - in R5, the wide marks and tileFirst of accepted blocks against the restatement (big_corpus.wide_marks, tile_first).
The corpus places offset errors and capacity events in chosen lanes of the parallel scan, compressed sizes on its
thresholds (2 047 / 2 048, 65 535 / 65 536 bytes), decoded sizes and matches on tile edges, and sources two tiles back;
tests/test_big_corpus_emul.py pins these claims on the CPU.  The host pipeline runs once with its default chunks and once,
in a child process, with 1 MiB chunks (LZ4B200_HOST_CHUNK_MB is read once per process).
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import big_corpus as bc
import frame_oracle as fo
from gpu_util import arrange, check_vs_oracle, corrupt, decode_batch, decode_batch_uniform, sha, wide_workspace

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CAPS = (65537, 122880, 300000, 4 << 20)
MiB = 1 << 20


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    assert lib.LZ4B200_device_count() > 0, "GPU tests need a CUDA device"
    assert "LZ4K_SCAN_IMPL" not in os.environ, "the route tests assume the default scan dispatch"
    return lib


@pytest.fixture(scope="module")
def ncta():
    """CTAs of the persistent expand kernels: one per SM"""
    return torch.cuda.get_device_properties(0).multi_processor_count


_corpora, _seqs = {}, {}


def corpus(oracle, cap):
    """(blocks, kinds, oracle return values) of big_corpus at capacity cap"""
    if cap not in _corpora:
        c = bc.big_corpus(oracle, cap, seed=cap % 1009)
        _corpora[cap] = ([b for _, b in c], [k for k, _ in c], [oracle.decompress(b, cap)[0] for _, b in c])
    return _corpora[cap]


def seqs_of(blk):
    key = sha(blk)
    if key not in _seqs:
        _seqs[key] = bc.seq_list(blk)
    return _seqs[key]


def reverse_offsets(n, cap):
    """destination offsets in reverse block order with odd gaps"""
    gaps = 1 + 2 * (np.arange(n, dtype=np.int64) % 7)
    off = np.cumsum(cap + gaps[::-1]) - cap
    return off[::-1].copy()


TOTAL = {}


def tally(key, v):
    TOTAL[key] = TOTAL.get(key, 0) + v


def check(oracle, cap, bs, ks, res, want_route, marks=True):
    """check_vs_oracle, plus the slow list, nSeq and (R5) the wide marks and tileFirst of the accepted blocks"""
    n = len(bs)
    cnt = check_vs_oracle(oracle, bs, [cap] * n, ks, res, want_route)
    rets = [r for r, _ in res]
    acc = [i for i, r in enumerate(rets) if r > 0]
    slow = sorted(res.slow.tolist())
    if want_route == "R5":
        assert slow == [i for i in acc if ks[i] == "runs-over"], (cap, slow)
    else:
        assert slow == acc, (cap, len(slow), len(acc))
    rd_marks, rd_first = wide_workspace(res, n, cap) if want_route == "R5" else (None, None)
    for i in acc:
        sq = seqs_of(bs[i])
        assert int(res.nseq[i]) == len(sq), (cap, i, ks[i], int(res.nseq[i]), len(sq))
        if rd_marks is not None and marks:
            assert np.array_equal(rd_marks(i, len(sq)), bc.wide_marks(sq)), (cap, i, ks[i], "wide marks")
            want_first = bc.tile_first(sq)
            assert np.array_equal(rd_first(i, len(want_first) - 1), want_first), (cap, i, ks[i], "tileFirst")
            tally("marks compared", len(sq))
            tally("tileFirst compared", len(want_first))
    tally("%s rejected" % want_route, cnt["rejected"])
    tally("%s accepted" % want_route, cnt["accepted"])
    tally("%s run-overflow hand-offs" % want_route, cnt["overflow handed off"])
    return cnt


@pytest.mark.parametrize("cap", CAPS)
def test_big_corpus_in_every_workspace_and_layout(lib, oracle, cap):
    """The whole corpus in one batch: R5 (aligned stride, one call; reverse-order odd destinations, scan and expand as two
    calls), R6 with the small workspace (odd stride, two calls) and R6 with one byte less than R5 needs (reverse-order
    odd destinations).  nSeq also against the one-thread scan of R1."""
    blocks, kinds, rets = corpus(oracle, cap)
    n = len(blocks)
    wide = int(lib.LZ4B200_decompress_workspace_bytes_for(n, 0, cap))
    rev = reverse_offsets(n, cap)
    check(oracle, cap, blocks, kinds, decode_batch_uniform(blocks, cap), "R5")
    check(oracle, cap, blocks, kinds, decode_batch_uniform(blocks, cap, dst_off=rev, phases="split"), "R5")
    check(oracle, cap, blocks, kinds, decode_batch_uniform(blocks, cap, wide=False, stride=cap | 1, phases="split"), "R6")
    check(oracle, cap, blocks, kinds, decode_batch_uniform(blocks, cap, dst_off=rev, ws_bytes=wide - 1), "R6")
    acc = [i for i, r in enumerate(rets) if r > 0]
    one = decode_batch([blocks[i] for i in acc], [cap] * len(acc))
    assert one.route == "R1"
    for k, i in enumerate(acc):
        assert one[k][0] == rets[i] and int(one.nseq[k]) == len(seqs_of(blocks[i])), (cap, i, kinds[i])
    lanes = [ln for _, _, ln in bc.lane_event_blocks(cap, seed=cap % 1009 + 1)]
    tally("lane-event blocks", 4 * len(lanes))
    print("cap %d: %d blocks (%d accepted), %d lane-event blocks finished by lanes %s; totals %s" % (
        cap, n, len(acc), len(lanes), sorted(set(lanes)), TOTAL))


@pytest.mark.parametrize("phases", ["one", "split"])
def test_batch_sizes_around_the_cta_count(lib, oracle, ncta, phases):
    """Batches of 1, 7, ncta - 1, ncta, ncta + 1 and 2 ncta + 5 blocks with hostile blocks on the CTA columns of the
    tiles kernel (with ncta blocks each CTA takes every tile of one block and waits on its own previous tile), odd and
    aligned strides, R5 and R6"""
    for cap in (122880, 300000):
        blocks, kinds, rets = corpus(oracle, cap)
        for n in (1, 7, ncta - 1, ncta, ncta + 1, 2 * ncta + 5):
            idx = arrange(kinds, rets, n, ncta, seed=n)
            bs, ks = [blocks[i] for i in idx], [kinds[i] for i in idx]
            stride = (cap + 64) | 1 if n % 2 else None
            check(oracle, cap, bs, ks, decode_batch_uniform(bs, cap, stride=stride, phases=phases), "R5")
            if n in (7, ncta):
                check(oracle, cap, bs, ks, decode_batch_uniform(bs, cap, wide=False, stride=stride, phases=phases), "R6")
    cap = 4 * MiB                                        # ncta blocks of 69 tiles
    blocks, kinds, rets = corpus(oracle, cap)
    idx = arrange(kinds, rets, ncta, ncta, seed=phases == "one")
    bs, ks = [blocks[i] for i in idx], [kinds[i] for i in idx]
    check(oracle, cap, bs, ks, decode_batch_uniform(bs, cap, stride=cap + 17 if phases == "one" else None, phases=phases),
          "R5", marks=False)
    print("batch sizes around %d CTAs, %s: totals %s" % (ncta, phases, TOTAL))


def test_ragged_batch_of_one_and_69_tile_blocks(lib, oracle, ncta):
    cap = 4 * MiB
    raws = [oracle.datagen(cap if i % 2 else 40000 + 977 * i, (0.2, 0.5, 0.9)[i % 3], 300 + i) for i in range(ncta + 1)]
    blocks = [oracle.compress(r, 1)[1] for r in raws]
    blocks[5] = blocks[5][:-1]
    blocks[ncta] = corrupt(np.random.default_rng(1), blocks[ncta])
    kinds = ["datagen"] * len(blocks)
    for phases in ("one", "split"):
        check(oracle, cap, blocks, kinds, decode_batch_uniform(blocks, cap, dst_off=reverse_offsets(len(blocks), cap),
                                                               phases=phases), "R5", marks=phases == "one")


def test_64_mib_capacity(lib, oracle):
    """64 MiB is the largest capacity of the tiles kernel (1 093 tiles); one byte more takes the generic kernel"""
    cap = 64 * MiB
    _, c = oracle.compress(oracle.datagen(cap, 0.5, 64), 1)
    rng = np.random.default_rng(64)
    big = bc.threshold_blocks(cap, seed=5)[-1][1]        # <= 65 535 bytes that decode to 15 MB and more
    blocks = [c, c[:-1], c[:len(c) // 2], corrupt(rng, c), big]
    kinds = ["datagen", "broken", "broken", "broken", "threshold"]
    for cp, rt in ((cap, "R5"), (cap + 1, "R6")):
        res = decode_batch_uniform(blocks, cp, stride=cp + 17)
        cnt = check(oracle, cp, blocks, kinds, res, rt, marks=False)
        assert res[0][0] == cap and res[4][0] >= 15 * MiB and cnt["rejected"] >= 2, cnt
        if rt == "R5":
            rd_marks, rd_first = wide_workspace(res, len(blocks), cp)
            sq = seqs_of(big)
            assert np.array_equal(rd_marks(4, len(sq)), bc.wide_marks(sq))
            assert np.array_equal(rd_first(4, bc.tiles_of(res[4][0])), bc.tile_first(sq))
            first = rd_first(0, bc.tiles_of(cap))                 # the P0.5 block: the tile index is non-decreasing
            assert len(first) == 1093 + 1 and (np.diff(first.astype(np.int64)) >= 0).all() and first[-1] <= res.nseq[0]
            tally("tileFirst compared", bc.tiles_of(res[4][0]) + 1)


# ------------------------------------------------------------------------------------------
# host pipeline and frames over big blocks
# ------------------------------------------------------------------------------------------
def _host_blocks(oracle):
    bs, n = 4 * MiB, 40
    raw = oracle.datagen(n * bs - 12345, 0.5, 91)
    blocks = [oracle.compress(raw[i * bs:(i + 1) * bs], 1)[1] for i in range(n)]
    rng = np.random.default_rng(40)
    for i in (2, 5, 37, 39):                             # the first and the last chunk of 16 blocks
        blocks[i] = {2: blocks[i][:-1], 37: blocks[i] + b"\x00"}.get(i) or corrupt(rng, blocks[i])
    return blocks


def _host_call(lib, blocks, cap):
    sizes = np.array([len(b) for b in blocks], dtype=np.int32)
    offs = np.concatenate([[0], np.cumsum(sizes[:-1], dtype=np.int64)]).astype(np.int64)
    src = np.frombuffer(b"".join(blocks) + b"\x00" * 16, dtype=np.uint8)
    out = np.zeros(len(blocks) * cap, dtype=np.uint8)
    rets = np.zeros(len(blocks), dtype=np.int32)
    rc = lib.LZ4B200_decompress_blocks_host(src.ctypes.data, offs.ctypes.data, sizes.ctypes.data, out.ctypes.data,
                                            cap, cap, rets.ctypes.data, len(blocks))
    assert rc == 0
    return rets, [out[i * cap:i * cap + max(int(r), 0)].tobytes() for i, r in enumerate(rets)]


def test_host_pipeline_over_several_chunks(lib, oracle, tmp_path):
    """40 blocks of 4 MiB: 16 per 64 MiB chunk, three chunks on different streams; then 1 MiB chunks in a child process:
    one block per chunk, 40 tiles kernels through the four streams"""
    cap = 4 * MiB
    blocks = _host_blocks(oracle)
    want = [oracle.decompress(b, cap) for b in blocks]
    rets, outs = _host_call(lib, blocks, cap)
    for i, ((er, eo), r, o) in enumerate(zip(want, rets, outs)):
        assert r == er and (r < 0 or o == eo), (i, int(r), er)
    assert sum(r < 0 for r, _ in want) >= 3
    env = dict(os.environ, LZ4B200_HOST_CHUNK_MB="1")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path)], env=env, timeout=600,
                       capture_output=True, text=True)
    assert p.returncode == 0, (p.stdout[-2000:], p.stderr[-4000:])
    assert np.load(str(tmp_path / "rets.npy")).tolist() == [r for r, _ in want]
    assert np.load(str(tmp_path / "sha.npy")).tolist() == [sha(o if r >= 0 else b"") for r, o in want]
    tally("host pipeline blocks", 2 * len(blocks))


def child_main(d):
    sys.path[:0] = [os.path.dirname(HERE), HERE]
    from lz4_b200 import _lib
    from oracle.pyoracle import Oracle
    rets, outs = _host_call(_lib.load(), _host_blocks(Oracle()), 4 * MiB)
    np.save(os.path.join(d, "rets.npy"), rets)
    np.save(os.path.join(d, "sha.npy"), np.array([sha(o) for o in outs]))


def _frame_call(lib, frame, cap):
    src = np.frombuffer(frame, dtype=np.uint8)
    dst = np.zeros(max(cap, 1), dtype=np.uint8)
    used = C.c_int64(-1)
    r = int(lib.LZ4B200_decompressFrame_host(src.ctypes.data, len(src), dst.ctypes.data, cap, C.byref(used)))
    return r, dst[:max(r, 0)].tobytes(), used.value


@pytest.mark.parametrize("bsid, nblocks", [(7, 150), (6, 300)])
def test_frames_of_several_groups(lib, oracle, bsid, nblocks):
    """A frame decodes in groups of 256 MiB of block slots (64 blocks of 4 MiB, 256 of 1 MiB): mixed block sizes from 1 B
    to the block size (tile edges and stored-raw blocks among them), into a buffer of exactly the decoded size (bounce
    buffer), one large enough for every group (direct), and one where the first group is direct and the next bounce;
    one byte short gives -5; a broken block in the last group and a content size off by one give -3."""
    bs = 1 << (8 + 2 * bsid)
    group = (256 * MiB) // bs
    rng = np.random.default_rng(bsid)
    menu = [1, 13, 61439, 61440, 61441, 122879, 122881, 300000, bs - 1, bs, bs // 3]
    sizes = [menu[i % len(menu)] if i % 5 else int(rng.integers(1, 5000)) for i in range(nblocks)]
    data = oracle.datagen(sum(sizes), 0.5, 100 + bsid).tobytes()
    cuts = np.concatenate([[0], np.cumsum(sizes)])
    pieces = [data[cuts[i]:cuts[i + 1]] for i in range(nblocks)]
    raw = {3, 17, nblocks - 2}
    for i in raw:
        pieces[i] = bytes(rng.integers(0, 256, sizes[i], dtype=np.uint8))
    want = b"".join(pieces)
    total = len(want)
    assert nblocks > group and total <= group * bs
    frame = fo.frame_of_blocks(oracle, pieces, bsid, content_size=total, raw=raw)
    assert fo.decompress_frame(oracle, frame) == (want, len(frame))
    for cap in (total, nblocks * bs, group * bs):      # bounce, direct, direct then bounce
        r, out, used = _frame_call(lib, frame, cap)
        assert (r, used) == (total, len(frame)) and out == want, (bsid, cap, r)
    assert _frame_call(lib, frame, total - 1)[0] == -5
    for cs in (total - 1, total + 1):
        assert _frame_call(lib, fo.frame_of_blocks(oracle, pieces, bsid, content_size=cs, raw=raw), total)[0] == -3
    k = nblocks - 3                                      # a compressed block of the last group, truncated by one byte
    assert k // group == (nblocks - 1) // group and k not in raw
    ok, c = oracle.compress(pieces[k], 1)
    assert oracle.decompress(c[:-1], bs)[0] < 0
    tail = fo.frame_of_blocks(oracle, pieces[k + 1:], bsid, raw={i - k - 1 for i in raw if i > k})
    head = fo.frame_of_blocks(oracle, pieces[:k], bsid, raw=raw)
    broken = head[:-4] + np.uint32(len(c) - 1).tobytes() + c[:-1] + tail[7:]
    assert _frame_call(lib, broken, nblocks * bs)[0] == -3
    tally("frame blocks", 5 * nblocks)
    tally("frame groups", 5 * ((nblocks + group - 1) // group))
    print("bsid %d: %d blocks, %d MB in %d groups; totals %s" % (bsid, nblocks, total >> 20, -(-nblocks // group), TOTAL))


if __name__ == "__main__":
    child_main(sys.argv[1])
