"""The CPU checker of LZ4_decompress_safe_partial (oracle_lz4_decompress_safe_partial in oracle/lz4_oracle.c) against
the reference's results.

tests/golden/kat_partial.json holds results of the compiled reference (tests/golden/make_golden_partial.py): the checker
must give every return value and every group's output digest, and the run digests.  Where oracle/_ref exists it is also
compared live.  Properties checked on the checker itself: ret <= outputSize, the prefix rule for valid blocks, and the
guard past outputSize (every call).
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_golden_partial as mg  # noqa: E402


@pytest.fixture(scope="module")
def kat():
    return mg.golden()


def test_checker_reproduces_the_reference(kat, oracle):
    doc, groups = kat
    paths, dst_dependent = set(), 0
    for name, cases, rets, digest in groups:
        res = []
        for src, t, c in cases:
            r, out, last_path, dep = oracle.decompress_partial_traced(src, t, c)
            res.append((r, None) if dep else (r, out))
            paths.add(last_path)
            dst_dependent += dep
        assert [r for r, _ in res] == rets and mg.run_digest(res) == digest, name
    assert sum(len(g[1]) for g in groups) > 20000
    assert paths == {0, 1, 2}                  # stops after literals, inside a match, and none (errors, target 0)
    assert 0 < dst_dependent < 1000            # offset-0 matches on the reference's cut path
    res = []
    for comp, t, c in mg.random_cases(oracle, doc["run_cases"]):
        r, out, _, dep = oracle.decompress_partial_traced(comp, t, c)
        res.append((r, None) if dep else (r, out))
    assert [mg.run_digest(res[k:k + doc["run_chunk"]]) for k in range(0, len(res), doc["run_chunk"])] == doc["run_digests"]


def test_partial_properties(oracle):
    """ret <= min(target, cap); a valid block at its exact size gives min(target, cap, decoded) bytes of the full decode"""
    for (bid, size, kind, seed) in mg.blocks():
        if size > 65536:
            continue
        raw, comp = mg.make_block(oracle, size, kind, seed)
        for t in {0, 1, 5, 12, 13, 64, 65, 1000, max(size - 1, 0), size, size + 3}:
            for c in (t, t + 7, max(t - 3, 0)):
                want = max(min(t, c, size), 0)
                assert oracle.decompress_partial(comp, t, c) == (want, raw[:want]), (bid, t, c)


def test_checker_against_live_reference(oracle, reference):
    rng = np.random.default_rng(77)
    for k in range(600):
        size = int(rng.choice([1, 30, 300, 3000, 30000, 65536, 70000]))
        comp = mg.make_block(reference, size, mg.KINDS[k % len(mg.KINDS)], 70000 + k)[1]
        v = [["exact"], ["trunc", int(rng.integers(1, len(comp) + 1))], ["ext", int(rng.integers(1, 12)), k],
             ["flip", int(rng.integers(0, len(comp))), int(rng.integers(1, 256))]][k % 4]
        src = mg.variant(comp, v)
        t = int(rng.choice([int(rng.integers(-1, 100)), int(rng.integers(0, size + 30)), size]))
        c = t if k % 3 else int(rng.integers(0, max(t, 1) + 1))
        r, out, _, dst_dependent = oracle.decompress_partial_traced(src, t, c)
        rr, rout = reference.decompress_partial(src, t, c)
        assert r == rr and (dst_dependent or out == rout), (k, size, v, t, c)
