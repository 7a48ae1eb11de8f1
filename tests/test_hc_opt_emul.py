"""CPU check of the HC optimal parse (levels 10 .. 12) the GPU runs: the host build of lz4_b200/csrc/lz4_hc_core.h
(tests/emul/hc_emul.cpp) must give the reference's LZ4_compress_HC and LZ4_compress_HC_destSize results on every
vector and run digest of tests/golden/kat_hc_opt.json, whatever the chain table and the price table hold at the start,
write nothing past its limit, and every output must decode through the oracle's decoder (at the input's size, or at
`consumed` for the fill mode).  Where oracle/_ref exists, extra seeded cases are compared with the reference live."""
import numpy as np
import pytest

import hc_emul as he
from hc_emul import host_hc_opt, host_hc_opt_dest, mg, mgd, mgo

FILLS = [(0xFFFF, 0), (0x3C5A, 0x7FFFFFFF), (0x0001, 0x80000000), (0x1234, 0xFFFFFFFF)]


@pytest.fixture(scope="module")
def inputs(oracle):
    doc, ins = he.golden("kat_hc_opt.json")
    data = {}
    for iid, i in ins.items():
        data[iid] = mg.make_input(oracle, i["size"], i["kind"], i["seed"])
        assert mg.digest(data[iid]) == i["sha256"], i
    return doc, ins, data


def test_plain_vectors_match_the_reference(oracle, inputs):
    doc, ins, data = inputs
    for k, (iid, lv, rb, rets, dig) in enumerate(doc["vectors"]):
        d, n = data[iid], ins[iid]["size"]
        chain, opt = FILLS[k % len(FILLS)]
        res = [host_hc_opt(d, cap, lv, chain, opt) for cap in mg.capacities(n, rb)]
        assert [r for r, _ in res] == rets and mg.run_digest(res) == dig, (ins[iid], lv)
        assert rb > 0 and oracle.decompress(res[mg.capacities(n, rb).index(rb)][1], n) == (n, d.tobytes())
    assert len(doc["vectors"]) > 250


def test_fill_vectors_match_the_reference(oracle, inputs):
    doc, ins, data = inputs
    for k, (iid, lv, rb, rets, cons, dig) in enumerate(doc["dest_vectors"]):
        d, n = data[iid], ins[iid]["size"]
        chain, opt = FILLS[(k + 1) % len(FILLS)]
        ts = mgd.targets(n, rb)
        res = [host_hc_opt_dest(d, t, lv, chain, opt) for t in ts]
        assert [r for r, _, _ in res] == rets and [c for _, c, _ in res] == cons, (ins[iid], lv)
        assert mgd.run_digest(res) == dig, (ins[iid], lv)
        for t, (r, c, out) in zip(ts, res):
            if t >= 1:
                assert r >= 1 and oracle.decompress(out, c) == (c, d[:c].tobytes()), (ins[iid], lv, t)
            else:
                assert (r, c) == (0, n)
    assert len(doc["dest_vectors"]) > 250


def test_run_digests_match_the_reference(oracle):
    doc, _ = he.golden("kat_hc_opt.json")
    runs, res = [], []
    for d, cap, lv in mgo.random_cases(oracle, doc["run_cases"], mgo.PLAIN_SEED):
        res.append(host_hc_opt(d, cap, lv, chain_fill=0x5555, opt_fill=0x01010101))
        if len(res) == doc["run_chunk"]:
            runs.append(mg.run_digest(res))
            res = []
    assert runs == doc["run_digests"]
    for d, t, lv in mgo.random_cases(oracle, doc["run_cases"], mgo.DEST_SEED):
        res.append(host_hc_opt_dest(d, t, lv, chain_fill=0xAAAA, opt_fill=0xFEFEFEFE))
        r, c, out = res[-1]
        assert oracle.decompress(out, c) == (c, d[:c].tobytes())
        if len(res) == doc["run_chunk"]:
            runs.append(mgd.run_digest(res))
            res = []
    assert runs[len(doc["run_digests"]):] == doc["dest_run_digests"]


def test_output_does_not_depend_on_the_starting_tables(oracle):
    """Chain table and price table filled with several values: the same bytes, values and consumed counts."""
    for k, kind in enumerate(["p50", "p90l60", "per1", "per3", "random", "p100"]):
        d = mg.make_input(oracle, 20000 + 7 * k, kind, 31 + k)
        b = mg.compress_bound(len(d))
        for lv in (10, 11, 12):
            want = [host_hc_opt(d, cap, lv) for cap in (b, b // 3)]
            want_d = [host_hc_opt_dest(d, t, lv) for t in (b, 2000)]
            for chain, opt in FILLS[1:] + [(0x8000, 0x00000003)]:
                assert [host_hc_opt(d, cap, lv, chain, opt) for cap in (b, b // 3)] == want, (kind, lv, chain, opt)
                assert [host_hc_opt_dest(d, t, lv, chain, opt) for t in (b, 2000)] == want_d, (kind, lv, chain, opt)


def test_levels_below_ten_are_not_this_parse():
    for lv in (9, 1, 0, -1):
        assert host_hc_opt(b"x" * 100, 200, lv)[0] == -1
        assert host_hc_opt_dest(b"x" * 100, 200, lv)[:2] == (-1, 100)


def test_live_against_the_reference(reference):
    rng = np.random.default_rng(1012)
    for k in range(200):
        n = int(rng.choice([0, 12, 13, 50, 777, 5000, 65536, 100000]))
        kind = mg.KINDS[int(rng.integers(0, len(mg.KINDS)))]
        d = mg.make_input(reference, n, kind, 93000 + k)
        b = mg.compress_bound(n)
        lv = int(rng.choice([10, 11, 12, 13, 50]))
        cap = int(rng.choice([b, b - 1, int(rng.integers(0, b + 1)), int(rng.integers(1, 64)), 1 << 30]))
        assert host_hc_opt(d, cap, lv) == mgo.reference_hc(reference, d, cap, lv), (n, kind, lv, cap)
        assert host_hc_opt_dest(d, cap, lv, opt_fill=0x7FFFFFFF) == mgo.reference_hc_dest(reference, d, cap, lv), \
            (n, kind, lv, cap)
