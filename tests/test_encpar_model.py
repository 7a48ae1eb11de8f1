"""CPU checks of the host model of the parallel-parse compressor (tests/encpar_model.py), the reference that
tests/test_gpu_compress_routes.py compares the kernel with byte for byte.

The model is built from the documented rules (DESIGN.md 3.5), so these tests check that those rules describe the
compressor the project promises: every block is a valid LZ4 block at its exact capacity, obeys the format's end-of-block
rules, reproduces the ratios DESIGN.md 5 reports against the reference, and agrees with LZ4_compress_fast where the
parallel parse does not apply."""
import numpy as np
import pytest

import encpar_model as M

BS = 65536


def check_block(oracle, raw, r):
    """r (a model Result at compressBound) is a valid block of raw that obeys the end-of-block rules"""
    n = len(raw)
    assert r.ret == len(r.out) > 0
    assert oracle.decompress(r.out, n) == (n, raw)
    if n >= M.MIN_LENGTH:
        assert oracle.decompress(r.out, n + 64) == (n, raw)
        assert r.last >= M.LAST_LITERALS                                  # lz4.c:963-964
    for A, s, c, L, p in r.seqs:
        assert A <= s <= p <= n - M.MFLIMIT and 1 <= s - c <= 65535 and L >= 4 and s + L <= n - M.LAST_LITERALS
        assert p % r.step == 0                                            # only probed positions start a selection


def test_blocks_decode_at_exact_capacity(oracle):
    rng = np.random.default_rng(1)
    blocks = [oracle.datagen(BS, p, s).tobytes() for p, s in ((0.0, 1), (0.2, 2), (0.5, 3), (0.9, 4), (1.0, 5))]
    blocks += [b for _, b, _ in M.special_blocks()]
    blocks += [oracle.datagen(n, 0.5, n).tobytes() for n in (13, 14, 17, 100, 4107, 8203, 8204, 8205, 16396, 65535)]
    blocks.append(bytes(rng.integers(0, 4, BS, dtype=np.uint8)))
    for raw in blocks:
        for accel in (1, 5, 13, 1000):
            r = M.compress(raw, accel)
            check_block(oracle, raw, r)
            assert M.compress(raw, accel, r.ret).ret == r.ret
            assert M.compress(raw, accel, r.ret - 1).ret == 0


def test_ratio_reproduces_the_measured_gain_over_the_reference(oracle):
    """DESIGN.md 5: ratio against the reference's at acceleration 1 on datagen P50 / P90 / P20, measured with bench.py's
    generator (64 MiB segments, seed 0): +2.6 / +0.6 / +1.8 %.  The model must give the same to 0.2 points, and stay
    within the 2 % the header promises."""
    for proba, gain in ((0.5, 2.6), (0.9, 0.6), (0.2, 1.8)):
        nb = 48
        d = oracle.datagen_mt(nb * BS, 64 << 20, proba, 0)
        model = ref = 0
        for i in range(nb):
            blk = d[i * BS:(i + 1) * BS].tobytes()
            model += M.compress(blk).ret
            ref += oracle.compress(blk, 1)[0]
        got = 100.0 * (ref / model - 1.0)
        assert abs(got - gain) <= 0.2, (proba, got, gain)
        assert model <= ref * 1.02


def test_acceleration_steps():
    assert [M.step_of(a) for a in (-7, 0, 1, 4, 5, 12, 13, 20, 21, 1000, 65537, 1 << 30)] == \
        [1, 1, 1, 1, 2, 2, 3, 3, 4, 126, 8193, 8193]


def test_empty_short_and_large_blocks_agree_with_the_oracle(oracle):
    """n == 0, n < 13 (the last literals alone) and n > 65 536 (LZ4_compress_fast) give the oracle's bytes and verdict"""
    for n in list(range(0, 13)) + [65537, 70000, 200000]:
        raw = oracle.datagen(n, 0.5, n).tobytes()
        for cap in (None, 0, 1, max(n, 1), n + 1):
            r = M.compress(raw, 1, cap, oracle=oracle)
            want = oracle.compress(raw, 1, cap)
            assert (r.ret, r.out[:r.ret]) == want, (n, cap)


def test_rules_on_hand_made_blocks():
    # period 1 .. 4: the short-period rule gives p - d; periods 5 .. 8 the table
    for d in range(1, 9):
        raw = M.rle_block(d, d)
        r = M.compress(raw)
        A, s, c, L, p = r.seqs[0]
        assert len(r.seqs) == 1 and L == BS - 5 - s
        _, kind = M.candidates(np.frombuffer(raw, dtype=np.uint8), 1)
        assert kind[p] == (d if d <= 4 else 5), (d, kind[p])
    # one hash for every aligned position: the window's earliest word decides, a different word falls through to the
    # earlier windows' latest
    raw = M.collision_block(8, 15)
    b = np.frombuffer(raw, dtype=np.uint8)
    cand, kind = M.candidates(b, 1)
    assert (kind[0:BS - 12:4] != 0).sum() > 0
    assert set(np.unique(kind[8192:BS - 12:4]).tolist()) >= {5, 6}
    # the constructed blocks reach what they claim
    for name, raw, claim in M.special_blocks():
        assert M.reaches(M.compress(raw), claim), name
