"""Every decode route of lz4k_launch_decode on hostile batches, against the oracle: return value (incl. the negative
error position) and bytes of every block, the slow list (which blocks the generic kernel took over), and the bytes of
every destination slot the decoder may not touch (gpu_util.decode_batch*).

The route a call takes depends on the shape of the call alone (gpu_util.route); each test asserts the route it claims,
so that a change of the dispatch fails here instead of silently moving the coverage.  R1 (per-block capacities) is
covered here with the split phases and in test_gpu_parity.py::test_decode_noisy_source_vs_oracle; R5 / R6 (one capacity
above 64 KB) in test_gpu_big_routes.py, on a corpus of their own.  The last test runs the same saved corpus under every value of
the developer switch LZ4K_SCAN_IMPL, one process per value.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gpu_util import (arrange, check_vs_oracle, decode_batch, decode_batch_uniform, hostile_corpus, run_block, sha)

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


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


_corpora = {}


def corpus(oracle, cap):
    """(blocks, kinds, oracle return values) of hostile_corpus at capacity cap"""
    if cap not in _corpora:
        c = hostile_corpus(oracle, cap, seed=cap % 1009)
        _corpora[cap] = ([b for _, b in c], [k for k, _ in c], [oracle.decompress(b, cap)[0] for _, b in c])
    return _corpora[cap]


def run_uniform(oracle, cap, n, ncta, want_route, stride=None, phases="one", seed=0):
    blocks, kinds, rets = corpus(oracle, cap)
    idx = arrange(kinds, rets, n, ncta, seed)
    bs, ks = [blocks[i] for i in idx], [kinds[i] for i in idx]
    res = decode_batch_uniform(bs, cap, stride=stride, phases=phases)
    cnt = check_vs_oracle(oracle, bs, [cap] * n, ks, res, want_route)
    print("%s cap %d, %d blocks, %s: %s" % (want_route, cap, n, phases, cnt))
    return cnt


def odd(x):
    return x | 1


@pytest.mark.parametrize("cap", [16384, 20000, 32768, 65535, 65536])
def test_route_r2_split_scan(lib, oracle, ncta, cap):
    """One capacity in [16 KB, 64 KB], at most 8 192 blocks: split scan -> rows / generic.  Batches of 1, 7, 33 and 8 192
    blocks, hostile blocks in every slot of a warp and in the last, partial group; aligned and odd destination strides."""
    blocks, kinds, rets = corpus(oracle, cap)
    for i in [i for i, k in enumerate(kinds) if k in ("event", "runs-over", "seqs-over")]:   # one block per call
        res = decode_batch_uniform([blocks[i]], cap)
        check_vs_oracle(oracle, [blocks[i]], [cap], [kinds[i]], res, "R2")
    tot = {}
    for n, stride in ((7, odd(cap + 64)), (33, None), (8192, odd(cap + 100))):
        cnt = run_uniform(oracle, cap, n, ncta, "R2", stride=stride, phases="split" if (cap, n) == (65536, 33) else "one")
        tot = {k: tot.get(k, 0) + v for k, v in cnt.items()}
    assert tot["rejected"] >= 3000 and tot["accepted"] >= 500, tot
    if cap >= 32768:
        assert tot["overflow handed off"] >= 10, tot


@pytest.mark.parametrize("phases", ["one", "split"])
def test_route_r3_thread_scan_many_blocks(lib, oracle, ncta, phases):
    """One capacity of 64 KB and 8 193 blocks: the one-thread scan with narrow marks -> rows / generic; hostile blocks at
    0, 4 096 and 8 192."""
    cap, n = 65536, 8193
    blocks, kinds, rets = corpus(oracle, cap)
    idx = arrange(kinds, rets, n, ncta, seed=3)
    bad = [i for i, r in enumerate(rets) if r < 0]
    over = [i for i, k in enumerate(kinds) if k == "runs-over"]
    idx[0], idx[4096], idx[8192] = over[0], bad[1], bad[-2]
    bs, ks = [blocks[i] for i in idx], [kinds[i] for i in idx]
    res = decode_batch_uniform(bs, cap, stride=odd(cap + 64) if phases == "one" else None, phases=phases)
    cnt = check_vs_oracle(oracle, bs, [cap] * n, ks, res, "R3")
    print("R3 cap %d, %d blocks, %s: %s" % (cap, n, phases, cnt))
    assert 0 in res.slow
    assert cnt["rejected"] >= 3000 and cnt["accepted"] >= 1000 and cnt["overflow handed off"] >= 100, cnt


@pytest.mark.parametrize("cap", [64, 1000, 4096, 16383])
def test_route_r4_small_capacity(lib, oracle, ncta, cap):
    """One capacity below 16 KB: the one-thread scan with narrow marks (capacity / 4 + 2 slots) -> rows / generic."""
    blocks, kinds, rets = corpus(oracle, cap)
    tot = {}
    for n, stride, phases in ((len(blocks), None, "one"), (300, odd(cap + 64), "split")):
        cnt = run_uniform(oracle, cap, n, ncta, "R4", stride=stride, phases=phases, seed=n)
        tot = {k: tot.get(k, 0) + v for k, v in cnt.items()}
    assert tot["rejected"] >= 300 and tot["accepted"] >= 40, tot


def test_route_r1_with_split_phases(lib, oracle, ncta):
    """Per-block capacities (R1) as a scan call and an expand call, with the boundary blocks of the corpus."""
    blocks, kinds, caps = [], [], []
    for cap in (1000, 20000, 65536):
        b, k, _ = corpus(oracle, cap)
        blocks += b
        kinds += k
        caps += [cap] * len(b)
    rets = [oracle.decompress(b, c)[0] for b, c in zip(blocks, caps)]
    idx = arrange(kinds, rets, 2 * len(blocks), ncta, seed=5)
    bs, ks, cs = [blocks[i] for i in idx], [kinds[i] for i in idx], [caps[i] for i in idx]
    res = decode_batch(bs, cs, phases="split")
    cnt = check_vs_oracle(oracle, bs, cs, ks, res, "R1")
    print("R1 %d blocks, split: %s" % (len(bs), cnt))
    assert cnt["rejected"] >= 500 and cnt["overflow handed off"] >= 10, cnt


# ------------------------------------------------------------------------------------------
# the scan switch: the same corpus under LZ4K_SCAN_IMPL unset / thread / split / par, one process each
# ------------------------------------------------------------------------------------------
SHAPES = ("u65536", "u20000", "per", "u300000", "u300000small")


def _save_corpus(oracle, d):
    for name in SHAPES:
        if name == "per":
            blocks, _, _ = corpus(oracle, 65536)
            blocks = blocks + corpus(oracle, 1000)[0]
            caps = [(65536, 65535, 20000, 4096, 1000, 64)[i % 6] for i in range(len(blocks))]
        elif name.startswith("u300000"):
            raw = oracle.datagen(300000, 0.5, 31)
            _, c = oracle.compress(raw, 1)
            rng = np.random.default_rng(31)
            big = run_block(33333)
            blocks = [c, c[:-1], c[:len(c) // 2], c + b"\0", big, big[:-7]]
            for _ in range(6):
                b = bytearray(c)
                b[int(rng.integers(0, len(b)))] = int(rng.integers(0, 256))
                blocks.append(bytes(b))
            caps = [300000] * len(blocks)
        else:
            blocks = corpus(oracle, int(name[1:]))[0]
            caps = [int(name[1:])] * len(blocks)
        sizes = np.array([len(b) for b in blocks], dtype=np.int64)
        np.save(os.path.join(d, name + "_data.npy"), np.frombuffer(b"".join(blocks), dtype=np.uint8))
        np.save(os.path.join(d, name + "_sizes.npy"), sizes)
        np.save(os.path.join(d, name + "_caps.npy"), np.array(caps, dtype=np.int32))


def _load_corpus(d, name):
    data = np.load(os.path.join(d, name + "_data.npy")).tobytes()
    sizes = np.load(os.path.join(d, name + "_sizes.npy"))
    offs = np.concatenate([[0], np.cumsum(sizes)])
    blocks = [data[offs[i]:offs[i + 1]] for i in range(len(sizes))]
    return blocks, np.load(os.path.join(d, name + "_caps.npy"))


def child_main(d, tag):
    """decode every shape of the corpus saved in d; save return values, sequence counts and digests of the bytes"""
    for name in SHAPES:
        blocks, caps = _load_corpus(d, name)
        if name == "per":
            res = decode_batch(blocks, caps)
        else:
            res = decode_batch_uniform(blocks, int(caps[0]), wide=not name.endswith("small"))
        np.save(os.path.join(d, "%s_%s_ret.npy" % (tag, name)), np.array([r for r, _ in res], dtype=np.int32))
        np.save(os.path.join(d, "%s_%s_nseq.npy" % (tag, name)), res.nseq)
        np.save(os.path.join(d, "%s_%s_sha.npy" % (tag, name)), np.array([sha(o) for _, o in res]))


def test_scan_switch_differential(lib, oracle, tmp_path):
    """LZ4K_SCAN_IMPL is read once per process.  Under each value the children must agree with each other and with the
    oracle: return value, bytes, and the sequence count of every accepted block.  This is where the parallel scan runs on
    64 KB blocks with narrow marks, the split scan with per-block and small capacities (its list-overflow fallback), and
    the forced scans on a batch of blocks above 64 KB (which take the parallel scan all the same when the tiles kernel
    needs its wide marks)."""
    _save_corpus(oracle, str(tmp_path))
    tags = ("default", "thread", "split", "par")
    for tag in tags:
        env = dict(os.environ)
        env.pop("LZ4K_SCAN_IMPL", None)
        if tag != "default":
            env["LZ4K_SCAN_IMPL"] = tag
        p = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path), tag], env=env, timeout=600,
                           capture_output=True, text=True)
        assert p.returncode == 0, (tag, p.stdout[-2000:], p.stderr[-4000:])
    for name in SHAPES:
        blocks, caps = _load_corpus(str(tmp_path), name)
        want = [oracle.decompress(b, int(c)) for b, c in zip(blocks, caps)]
        wret = np.array([r for r, _ in want], dtype=np.int32)
        wsha = np.array([sha(o) for _, o in want])
        acc = wret > 0
        assert acc.sum() >= 3 and (~acc).sum() >= 3, name
        nseq0 = None
        for tag in tags:
            load = lambda what: np.load(os.path.join(str(tmp_path), "%s_%s_%s.npy" % (tag, name, what)))
            ret, nseq, dig = load("ret"), load("nseq"), load("sha")
            bad = np.nonzero(ret != wret)[0]
            assert len(bad) == 0, (tag, name, [(int(i), int(ret[i]), int(wret[i])) for i in bad[:5]])
            assert (dig == wsha).all(), (tag, name, np.nonzero(dig != wsha)[0][:5])
            if nseq0 is None:
                nseq0 = nseq
            assert (nseq[acc] == nseq0[acc]).all(), (tag, name, np.nonzero((nseq != nseq0) & acc)[0][:5])


if __name__ == "__main__":
    sys.path[:0] = [os.path.dirname(HERE), HERE]
    child_main(sys.argv[1], sys.argv[2])
