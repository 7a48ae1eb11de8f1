"""CPU check of the HC parse the GPU runs: the host build of lz4_b200/csrc/lz4_hc_core.h (tests/emul/hc_emul.cpp) must
give the reference's LZ4_compress_HC results on every vector and run digest of tests/golden/kat_hc.json, whatever the
chain table holds at the start, and every output must decode back to its input through the oracle's decoder at exactly
the input's size.  Where oracle/_ref exists, extra seeded cases are compared with the reference live."""
import numpy as np

import hc_emul as he
from hc_emul import host_hc, mg


def test_vectors_match_the_reference(oracle):
    doc, ins = he.golden("kat_hc.json")
    data = {}
    checked = 0
    for iid, lv, rb, rets, dig in doc["vectors"]:
        i = ins[iid]
        if iid not in data:
            data = {iid: mg.make_input(oracle, i["size"], i["kind"], i["seed"])}
            assert mg.digest(data[iid]) == i["sha256"], i
        d = data[iid]
        r0, out0 = host_hc(d, mg.compress_bound(i["size"]), lv)
        assert r0 == rb, (i, lv)
        res = [host_hc(d, cap, lv) for cap in mg.capacities(i["size"], rb)]
        assert [r for r, _ in res] == rets and mg.run_digest(res) == dig, (i, lv)
        assert oracle.decompress(out0, i["size"]) == (i["size"], d.tobytes()), (i, lv)
        checked += 1
    assert checked == len(doc["vectors"]) > 2000


def test_run_digests_match_the_reference(oracle):
    doc, _ = he.golden("kat_hc.json")
    runs, res = [], []
    for d, cap, lv in mg.random_cases(oracle, doc["run_cases"]):
        res.append(host_hc(d, cap, lv, chain_fill=0x3C5A))
        r, out = res[-1]
        if r > 0:
            assert oracle.decompress(out, len(d)) == (len(d), d.tobytes())
        if len(res) == doc["run_chunk"]:
            runs.append(mg.run_digest(res))
            res = []
    assert runs == doc["run_digests"]


def test_output_does_not_depend_on_the_initial_chain_table(oracle):
    for k, kind in enumerate(["p50", "per1", "per2", "p90l60"]):
        d = mg.make_input(oracle, 100000, kind, 77 + k)
        for lv in (3, 9):
            want = host_hc(d, mg.compress_bound(len(d)), lv)
            for fill in (0, 1, 0x8000, 0xFFFE):
                assert host_hc(d, mg.compress_bound(len(d)), lv, chain_fill=fill) == want, (kind, lv, fill)


def test_levels_above_nine_are_not_built():
    for lv in (10, 11, 12, 100):
        assert host_hc(b"x" * 100, 200, lv)[0] == -1


def test_live_against_the_reference(reference):
    rng = np.random.default_rng(99)
    for k in range(300):
        n = int(rng.choice([13, 50, 777, 5000, 65536, 131072]))
        kind = mg.KINDS[int(rng.integers(0, len(mg.KINDS)))]
        d = mg.make_input(reference, n, kind, 90000 + k)
        b = mg.compress_bound(n)
        lv = int(rng.integers(-2, 10))
        cap = int(rng.choice([b, b - 1, int(rng.integers(0, b)), n]))
        assert host_hc(d, cap, lv) == mg.reference_hc(reference, d, cap, lv), (n, kind, lv, cap)
