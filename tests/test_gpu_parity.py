"""GPU parity tests: the CUDA path, called through the C ABI, against the oracle and the golden
vectors.  Bit-exact: compressed bytes, decoded bytes and return values (incl. error codes)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from gpu_util import check_vs_oracle, decode_batch, decode_batch_uniform, dev, hostile_corpus, run_block, sha, to_dev

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    assert lib.LZ4B200_device_count() > 0, "GPU tests need a CUDA device"
    return lib


# ------------------------------------------------------------------------------------------
# decoder
# ------------------------------------------------------------------------------------------
def test_decode_golden_known_answers_batch(lib, kat_decode):
    res = decode_batch([bytes.fromhex(c["block"]) for c in kat_decode], [c["cap"] for c in kat_decode])
    for c, (ret, out) in zip(kat_decode, res):
        assert ret == c["ret"], c
        if ret >= 0:
            assert out.hex() == c["out"], c


def test_decode_golden_known_answers_dropin(lib, kat_decode):
    from lz4_b200 import block
    for c in kat_decode:
        ret, out = block.LZ4_decompress_safe(bytes.fromhex(c["block"]), c["cap"])
        assert ret == c["ret"], c
        if ret >= 0:
            assert out.hex() == c["out"], c


def test_decode_fixture_block(lib, oracle):
    from lz4_b200 import block
    blk = open(os.path.join(GOLDEN, "p50_seed0_64k.lz4block"), "rb").read()
    d = oracle.datagen(65536, 0.5, 0).tobytes()
    assert block.LZ4_decompress_safe(blk, 65536) == (65536, d)
    assert block.LZ4_decompress_safe(blk, 65537) == (65536, d)
    assert block.LZ4_decompress_safe(blk, 65535)[0] == oracle.decompress(blk, 65535)[0] < 0
    assert block.LZ4_decompress_safe(blk[:-1], 65536)[0] == oracle.decompress(blk[:-1], 65536)[0] < 0
    assert block.LZ4_decompress_safe(blk + b"\0", 65536)[0] == oracle.decompress(blk + b"\0", 65536)[0] < 0


def test_decode_noisy_source_vs_oracle(lib, oracle):
    """Per-block capacities (route R1): the hostile corpus of gpu_util -- datagen blocks against exact, slack and short
    capacities, truncated, extended and corrupted blocks (tests/fuzzer.c:588-622), 8 191 .. 8 193 sequences, run-table
    overflow, offset-0 / offset-1 runs, split-scan events -- at capacities from 20 bytes to 70 000, each block at its
    corpus capacity and at one up to 80 bytes above and below -> the oracle's verdict / value / bytes; the run-overflow
    blocks go to the generic kernel."""
    rng = np.random.default_rng(77)
    blocks, caps, kinds = [], [], []
    for cap in (20, 64, 100, 300, 1000, 5000, 65536, 70000):
        for kind, b in hostile_corpus(oracle, cap, seed=cap, n_corrupt=6):
            for c in (cap, cap + int(rng.integers(0, 80)), max(cap - int(rng.integers(0, 80)), 0)):
                blocks.append(b)
                caps.append(c)
                kinds.append(kind)
    res = decode_batch(blocks, caps)
    cnt = check_vs_oracle(oracle, blocks, caps, kinds, res, "R1")
    print("R1 %d blocks: %s" % (len(blocks), cnt))
    assert cnt["accepted"] > 300 and cnt["rejected"] > 2000 and cnt["overflow handed off"] >= 6, cnt


def test_decode_overlap_and_long_runs(lib, oracle):
    """Self-overlapping matches (offsets 1..40) and long literal / match runs."""
    blocks, caps = [], []
    for off in list(range(1, 41)) + [100, 255, 256, 1000]:
        seedlen = max(off, 5)
        lits = bytes((i * 7 + 3) & 0xFF for i in range(seedlen))
        for mlen in [4, 5, 19, 20, 70, 300, 1000]:
            body = bytearray()
            ll = len(lits)
            tok_l = min(ll, 15)
            tok_m = min(mlen - 4, 15)
            body.append((tok_l << 4) | tok_m)
            if ll >= 15:
                r = ll - 15
                while r >= 255:
                    body.append(255); r -= 255
                body.append(r)
            body += lits
            body += bytes([off & 0xFF, off >> 8])
            if mlen - 4 >= 15:
                r = mlen - 4 - 15
                while r >= 255:
                    body.append(255); r -= 255
                body.append(r)
            body += bytes([0x50]) + b"vwxyz"
            blocks.append(bytes(body))
            caps.append(ll + mlen + 5)
    res = decode_batch(blocks, caps)
    ok = 0
    for blk, cap, (ret, out) in zip(blocks, caps, res):
        assert (ret, out) == oracle.decompress(blk, cap)
        ok += ret == cap
    assert ok > 150       # (tiny ones violate the end-of-block distance rules and are rejected by both)


# ------------------------------------------------------------------------------------------
# encoder
# ------------------------------------------------------------------------------------------
def test_compress_golden_known_answers(lib, kat_compress):
    from lz4_b200 import block
    for c in kat_compress:
        ret, out = block.LZ4_compress_fast(bytes.fromhex(c["src"]), c.get("cap"), c["accel"])
        assert ret == c["ret"], c
        if ret > 0:
            assert out.hex() == c["out"], c


def test_compress_datagen_digests_byte_identical(lib, datagen_digests, oracle):
    from lz4_b200 import block
    cache = {}
    for row in datagen_digests["buffers"]:
        key = (row["size"], row["proba"], row["seed"])
        if key not in cache:
            cache[key] = oracle.datagen(*key)
        ret, out = block.LZ4_compress_fast(cache[key], None, row["accel"])
        assert ret == row["csize"], row
        assert sha(out) == row["comp_sha256"], row


def test_compress_stream_of_64k_blocks_batch(lib, datagen_digests, oracle):
    from lz4_b200 import batch
    import hashlib
    s = datagen_digests["stream"]
    d = oracle.datagen(s["size"], s["proba"], s["seed"])
    src = to_dev(d)
    slots, sizes, stride = batch.compress_blocks(src, s["block"], s["accel"])
    torch.cuda.synchronize()
    sz = sizes.cpu().numpy()
    assert sz.tolist() == s["csizes"]
    host = slots.cpu().numpy()
    h = hashlib.sha256()
    for i, n in enumerate(sz):
        h.update(host[i * stride:i * stride + n].tobytes())
    assert h.hexdigest() == s["stream_sha256"]
    # pack + decode round trip on the device
    packed, offs = batch.pack_blocks(slots, stride, sizes)
    out, rets = batch.decompress_blocks(packed, offs[:-1].contiguous(), sizes, s["block"])
    torch.cuda.synchronize()
    assert (rets.cpu().numpy() == s["block"]).all()
    assert torch.equal(out, src)
    assert int(offs[-1]) == int(sz.sum())


def test_compress_random_vs_oracle(lib, oracle):
    """Sizes around every boundary (13, 64K limit 65547, 4 MB byU32), limited output
    (fuzzer.c:479-486,698-727), accelerations incl. clamps (lz4.c:1386-1387)."""
    from lz4_b200 import block
    rng = np.random.default_rng(3)
    sizes = [0, 1, 5, 12, 13, 14, 20, 64, 100, 1000, 4096, 65535, 65536, 65546, 65547, 65548, 70000, 200000,
             1 << 20, (4 << 20) + 17]
    for trial in range(120):
        n = int(rng.choice(sizes))
        p = float(rng.choice([0.0, 0.1, 0.5, 0.9, 1.0]))
        d = oracle.datagen(n, p, 300 + trial)
        acc = int(rng.choice([1, 1, 1, 2, 8, 32, 1000, 65537, 70000, 0, -3]))
        eret, eout = oracle.compress(d, acc)
        ret, out = block.LZ4_compress_fast(d, None, acc)
        assert (ret, out) == (eret, eout), (n, p, acc)
        for cap in [eret, eret - 1, eret - int(rng.integers(1, 64)), max(eret // 2, 0), 1, 0]:
            e2 = oracle.compress(d, acc, cap)
            r2 = block.LZ4_compress_fast(d, cap, acc)
            assert r2[0] == e2[0] and (r2[0] == 0 or r2[1] == e2[1]), (n, p, acc, cap)


def test_compress_text_like_and_special_inputs(lib, oracle):
    from lz4_b200 import block
    words = [b"lorem", b"ipsum", b"dolor", b"sit", b"amet", b"consectetur", b"adipiscing", b"elit", b"sed", b"do"]
    rng = np.random.default_rng(9)
    text = b" ".join(words[int(i)] for i in rng.integers(0, len(words), 40000))
    cases = [text, text[:65536], b"\x00" * 200000, bytes(range(256)) * 1024, b"ab" * 50000,
             rng.integers(0, 256, 300000, dtype=np.uint8).tobytes(), b"a" * 65547, b"xyz" * 30000 + b"q"]
    for d in cases:
        for acc in (1, 5):
            assert block.LZ4_compress_fast(d, None, acc) == oracle.compress(d, acc)
        r, c = block.LZ4_compress_default(d)
        assert block.LZ4_decompress_safe(c, len(d)) == (len(d), d)


def test_extstate_and_usingdict_entry_points(lib, oracle):
    import ctypes as C
    d = oracle.datagen(30000, 0.5, 11)
    eret, eout = oracle.compress(d, 1)
    dst = np.zeros(oracle.compress_bound(len(d)), dtype=np.uint8)
    state = (C.c_uint64 * (16416 // 8))()
    r = lib.LZ4_compress_fast_extState(C.addressof(state), d.ctypes.data, dst.ctypes.data, len(d), len(dst), 1)
    assert r == eret and dst[:r].tobytes() == eout
    r = lib.LZ4_compress_fast_extState_fastReset(C.addressof(state), d.ctypes.data, dst.ctypes.data, len(d), len(dst), 1)
    assert r == eret and dst[:r].tobytes() == eout
    assert lib.LZ4_compress_fast_extState(None, d.ctypes.data, dst.ctypes.data, len(d), len(dst), 1) == 0
    assert lib.LZ4_compress_fast_extState(C.addressof(state) + 1, d.ctypes.data, dst.ctypes.data, len(d), len(dst), 1) == 0
    out = np.zeros(len(d), dtype=np.uint8)
    comp = np.frombuffer(eout, dtype=np.uint8)
    assert lib.LZ4_decompress_safe_usingDict(comp.ctypes.data, out.ctypes.data, len(comp), len(out), None, 0) == len(d)
    assert (out == d).all()
    assert lib.LZ4_decompress_safe_usingDict(comp.ctypes.data, out.ctypes.data, len(comp), len(out), d.ctypes.data, 100) < 0


def test_inplace_dropin_calls(lib, oracle):
    """In-place compression / decompression with the margins of lz4.h:619-678 (fuzzer.c:1143-1187)."""
    n = 65536
    d = oracle.datagen(n, 0.5, 21)
    eret, eout = oracle.compress(d, 1)
    # decompress in place: compressed data at the end of the output buffer
    margin = (eret >> 8) + 32
    buf = np.zeros(n + margin, dtype=np.uint8)
    start = len(buf) - eret
    buf[start:] = np.frombuffer(eout, dtype=np.uint8)
    r = lib.LZ4_decompress_safe(buf.ctypes.data + start, buf.ctypes.data, eret, n)
    assert r == n and (buf[:n] == d).all()
    # compress in place: source at the end of the buffer
    bound = oracle.compress_bound(n)
    buf2 = np.zeros(bound + n, dtype=np.uint8)
    buf2[bound:] = d
    r = lib.LZ4_compress_default(buf2.ctypes.data + bound, buf2.ctypes.data, n, bound)
    assert r == eret and buf2[:r].tobytes() == eout


# ------------------------------------------------------------------------------------------
# batched / host-buffer calls and full-size properties
# ------------------------------------------------------------------------------------------
def test_large_blocks_4mb_roundtrip(lib, oracle):
    """lz4frame-sized 4 MB blocks: byU32 / 5-byte-hash path of the encoder, generic decoder."""
    from lz4_b200 import batch
    bs = 4 << 20
    d = oracle.datagen_mt(3 * bs + 12345, 1 << 20, 0.5, 40)
    src = to_dev(d)
    slots, sizes, stride = batch.compress_blocks(src, bs, 1)
    torch.cuda.synchronize()
    host = slots.cpu().numpy()
    for i, n in enumerate(sizes.cpu().numpy()):
        eret, eout = oracle.compress(d[i * bs:(i + 1) * bs], 1)
        assert n == eret and host[i * stride:i * stride + n].tobytes() == eout
    packed, offs = batch.pack_blocks(slots, stride, sizes)
    out, rets = batch.decompress_blocks(packed, offs[:-1].contiguous(), sizes, bs)
    torch.cuda.synchronize()
    r = rets.cpu().numpy()
    assert r[:-1].tolist() == [bs] * 3 and r[-1] == 12345
    assert torch.equal(out[:len(d)], src)


def test_large_blocks_4mb_incompressible_and_malformed(lib, oracle):
    """4 MB blocks through the scan of large blocks (parallel lanes in global memory) and the generic expand kernel:
    incompressible data (literal runs of megabytes), truncated / corrupted / capacity-limited blocks -> the oracle's
    return value (incl. the negative error position) and bytes."""
    bs = 4 << 20
    rng = np.random.default_rng(41)
    raws = [oracle.datagen(bs, 0.0, 11).tobytes(),                       # incompressible
            oracle.datagen(bs, 0.5, 12).tobytes(),
            oracle.datagen(bs - 12345, 0.9, 13).tobytes(),
            bytes(rng.integers(0, 256, 1 << 20, dtype=np.uint8)) + b"\0" * (3 << 20)]
    blocks, caps = [], []
    for raw in raws:
        _, c = oracle.compress(raw, 1)
        n = len(raw)
        blocks += [c, c, c, c[:-1], c[:len(c) // 2], c + b"\0"]
        caps += [n, n + 100, n - 1, n, n, n]
        for _ in range(3):                                               # corrupt a few bytes
            b = bytearray(c)
            for _ in range(int(rng.integers(1, 4))):
                b[int(rng.integers(0, len(b)))] = int(rng.integers(0, 256))
            blocks.append(bytes(b))
            caps.append(n)
    res = decode_batch(blocks, caps)
    good = 0
    for blk, cap, (ret, out) in zip(blocks, caps, res):
        eret, eout = oracle.decompress(blk, cap)
        assert ret == eret, (len(blk), cap, ret, eret)
        if ret >= 0:
            assert out == eout
            good += 1
    assert good >= 8


def test_big_blocks_in_tiles_vs_oracle(lib, oracle):
    """Blocks above 64 KB with ONE capacity and the large workspace take the tiles kernel (60 KB output tiles, sources in
    earlier tiles read from global memory): valid, incompressible, periodic, truncated and corrupted blocks of 70 KB .. 4 MB
    -> the oracle's return value (incl. the negative error position) and bytes; the generic kernel (small workspace) must
    agree."""
    rng = np.random.default_rng(77)
    TILE = 61440
    def rep(seed, n):
        return (seed * (n // len(seed) + 2))[:n]
    noise = bytes(rng.integers(0, 256, 200000, dtype=np.uint8))
    raws = [oracle.datagen(4 << 20, 0.5, 21).tobytes(), oracle.datagen(1 << 20, 0.9, 22).tobytes(),
            oracle.datagen(300000, 0.0, 23).tobytes(), oracle.datagen(70001, 0.2, 24).tobytes(),
            b"\0" * (1 << 20), rep(b"ab", 250000), rep(noise[:255], 300001), rep(noise[:TILE], 4 * TILE + 3),
            rep(noise[:TILE + 1], 3 * TILE), rep(noise[:65535], 262144),
            noise + noise[:150000] + b"\0" * 130000 + noise[100:90000]]
    for group_cap in (None, 64):                                # exact capacity per block / 64 bytes of slack
        for raw in raws:
            _, c = oracle.compress(raw, 1)
            n = len(raw)
            cap = n if group_cap is None else n + group_cap
            blocks = [c, c[:-1], c[:len(c) // 2], c + b"\0"]
            for _ in range(2):
                b = bytearray(c)
                for _ in range(int(rng.integers(1, 4))):
                    b[int(rng.integers(0, len(b)))] = int(rng.integers(0, 256))
                blocks.append(bytes(b))
            res = decode_batch_uniform(blocks, cap, wide=True)
            res_small = decode_batch_uniform(blocks, cap, wide=False)
            assert (res.route, res_small.route) == ("R5", "R6")
            for blk, (ret, out), (ret2, out2) in zip(blocks, res, res_small):
                eret, eout = oracle.decompress(blk, cap)
                assert ret == eret and ret2 == eret, (n, cap, len(blk), ret, ret2, eret)
                if ret >= 0:
                    assert out == eout and out2 == eout, (n, cap, len(blk))
            assert res[0][0] == n
    # 200 KB of run-dense sequences (1 literal + an offset-1 match of 5 bytes: 4 runs per 6 bytes): every tile has more
    # runs than the table holds, and the block goes to the generic kernel once, however many tiles give up
    big = run_block(33333)
    n = 6 * 33333 + 29
    blocks = [big, big[:-1], big + b"\0", big]
    kinds = ["runs-over", "broken", "broken", "runs-over"]
    for cap, phases in ((n, "one"), (n + 64, "split")):
        res = decode_batch_uniform(blocks, cap, wide=True, phases=phases)
        cnt = check_vs_oracle(oracle, blocks, [cap] * 4, kinds, res, "R5")
        assert cnt["accepted"] == 2 and sorted(res.slow.tolist()) == [0, 3], (cap, cnt, res.slow)
        check_vs_oracle(oracle, blocks, [cap] * 4, kinds, decode_batch_uniform(blocks, cap, wide=False, phases=phases), "R6")
    # many big blocks at once: tile-major units across blocks, ragged sizes under one capacity
    raws = [oracle.datagen(int(rng.integers(70000, 600000)), float(rng.choice([0.2, 0.5, 0.9])), 100 + i).tobytes() for i in range(40)]
    blocks = [oracle.compress(r, 1)[1] for r in raws]
    res = decode_batch_uniform(blocks, 600000, wide=True)
    for r, (ret, out) in zip(raws, res):
        assert ret == len(r) and out == r


def test_host_buffer_batch_calls(lib, oracle):
    n_blocks, bs = 6000, 65536          # > one 256 MiB pipeline chunk
    total = n_blocks * bs - 777
    d = oracle.datagen_mt(total, 1 << 22, 0.5, 60)
    cap = oracle.compress_bound(bs)
    stride = (cap + 15) // 16 * 16
    slots = np.zeros(n_blocks * stride, dtype=np.uint8)
    csz = np.zeros(n_blocks, dtype=np.int32)
    rc = lib.LZ4B200_compress_blocks_host(d.ctypes.data, bs, bs, total - (n_blocks - 1) * bs, slots.ctypes.data,
                                          stride, cap, 1, csz.ctypes.data, n_blocks)
    assert rc == 0 and (csz > 0).all()
    for i in [0, 1, 4095, 4096, n_blocks - 1]:
        eret, eout = oracle.compress(d[i * bs:(i + 1) * bs], 1)
        assert csz[i] == eret and slots[i * stride:i * stride + eret].tobytes() == eout
    offs = (np.arange(n_blocks, dtype=np.int64) * stride)
    out = np.zeros(n_blocks * bs, dtype=np.uint8)
    rets = np.zeros(n_blocks, dtype=np.int32)
    rc = lib.LZ4B200_decompress_blocks_host(slots.ctypes.data, offs.ctypes.data, csz.ctypes.data, out.ctypes.data,
                                            bs, bs, rets.ctypes.data, n_blocks)
    assert rc == 0
    assert (rets[:-1] == bs).all() and rets[-1] == bs - 777
    assert (out[:total] == d).all()
    # broken blocks in the first and the last pipeline chunk (and one between): each gets the oracle's value, the other
    # blocks stay intact
    bad = [3, 1000, 2500, n_blocks - 10]
    csz[3] -= 1                                         # truncated
    csz[1000] += 1                                      # one byte appended (the slot's padding is zero)
    slots[2500 * stride] = 0xFF                         # first token
    slots[(n_blocks - 10) * stride + int(csz[n_blocks - 10]) // 2] ^= 0x40
    out[:] = 0
    rc = lib.LZ4B200_decompress_blocks_host(slots.ctypes.data, offs.ctypes.data, csz.ctypes.data, out.ctypes.data,
                                            bs, bs, rets.ctypes.data, n_blocks)
    assert rc == 0
    for k in bad:
        eret, eout = oracle.decompress(slots[k * stride:k * stride + int(csz[k])].tobytes(), bs)
        assert rets[k] == eret, (k, int(rets[k]), eret)
        if eret >= 0:
            assert out[k * bs:k * bs + eret].tobytes() == eout, k
    assert (rets[[3, 1000]] < 0).all()
    good = np.ones(n_blocks, dtype=bool)
    good[bad] = False
    assert (rets[good][:-1] == bs).all() and rets[-1] == bs - 777
    mask = np.repeat(good, bs)[:total]
    assert (out[:total][mask] == d[mask]).all()


def test_full_size_round_trip_property(lib, oracle):
    """1 GiB of 64 KB P50 blocks: compress -> pack -> decompress on the device equals the input;
    a sample of blocks is byte-identical to the oracle's compression."""
    from lz4_b200 import batch
    bs, n_blocks = 65536, 16384
    d = oracle.datagen_mt(n_blocks * bs, 64 << 20, 0.5, 0)
    src = to_dev(d)
    slots, sizes, stride = batch.compress_blocks(src, bs, 1)
    packed, offs = batch.pack_blocks(slots, stride, sizes)
    out, rets = batch.decompress_blocks(packed, offs[:-1].contiguous(), sizes, bs)
    torch.cuda.synchronize()
    assert bool((rets == bs).all())
    assert torch.equal(out, src)
    sz = sizes.cpu().numpy()
    ratio = (n_blocks * bs) / sz.sum()
    assert 1.5 < ratio < 1.75            # reference: 1.622 on this generator (SURVEY 8d)
    rng = np.random.default_rng(0)
    for i in rng.integers(0, n_blocks, 24):
        eret, eout = oracle.compress(d[i * bs:(i + 1) * bs], 1)
        got = slots[i * stride:i * stride + int(sz[i])].cpu().numpy().tobytes()
        assert sz[i] == eret and got == eout


def test_mixed_batch_fast_and_slow_lists(lib, oracle):
    """One batch mixing everything the two expand kernels see: RLE / periodic / text-like 64 KB blocks
    (long self-overlapping matches, periods 1..7 and 8..40), P10/P50/P90 datagen, incompressible blocks
    (compressed size > 65535 -> slow list), short and empty blocks, and a 300 KB block."""
    from lz4_b200 import batch
    rng = np.random.default_rng(12)
    words = [b"alpha", b"beta", b"gamma", b"delta", b"epsilon", b"zeta", b"eta", b"theta", b"iota", b"kappa"]
    blocks = []
    blocks.append(np.zeros(65536, dtype=np.uint8).tobytes())
    for period in (1, 2, 3, 5, 7, 8, 9, 13, 16, 31, 40):
        pat = bytes(rng.integers(0, 256, period, dtype=np.uint8))
        blocks.append((pat * (65536 // period + 1))[:65536])
    blocks.append(b" ".join(words[int(i)] for i in rng.integers(0, len(words), 20000))[:65536])
    for p, seed in ((0.1, 1), (0.5, 2), (0.9, 3), (0.9, 4), (0.0, 5), (0.0, 6), (1.0, 7)):
        blocks.append(oracle.datagen(65536, p, seed).tobytes())
    blocks.append(oracle.datagen(100, 0.5, 8).tobytes())
    blocks.append(b"")
    blocks.append(oracle.datagen(12, 0.5, 9).tobytes())
    blocks.append(oracle.datagen(300000, 0.5, 10).tobytes())
    blocks.append((b"abcdefgh" * 9000)[:65536 - 7])
    comp = [oracle.compress(b, 1)[1] for b in blocks]
    caps = [max(len(b), 1) for b in blocks]
    res = decode_batch(comp, caps)
    for b, c, cap, (ret, out) in zip(blocks, comp, caps, res):
        assert (ret, out) == oracle.decompress(c, cap)
        assert ret == len(b) and out == b
    # the same data compressed by the GPU must be byte-identical too (fixed 64 KB blocks only)
    full = [b for b in blocks if len(b) == 65536]
    src = to_dev(np.frombuffer(b"".join(full), dtype=np.uint8).copy())
    slots, sizes, stride = batch.compress_blocks(src, 65536, 1)
    torch.cuda.synchronize()
    host = slots.cpu().numpy()
    for i, (b, n) in enumerate(zip(full, sizes.cpu().numpy())):
        eret, eout = oracle.compress(b, 1)
        assert n == eret and host[i * stride:i * stride + n].tobytes() == eout
