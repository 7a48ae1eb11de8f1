"""CPU check of the HC fill parse the GPU runs: the host build of lz4_b200/csrc/lz4_hc_core.h (tests/emul/hc_dest_emul.cpp)
must give the reference's LZ4_compress_HC_destSize results (ret, consumed and bytes) on every vector and run digest of
tests/golden/kat_hc_destsize.json, whatever the chain table holds at the start, write nothing at or past
min(target, bound), and every output must decode through the oracle's decoder to exactly the first `consumed` input
bytes.  Where oracle/_ref exists, extra seeded cases are compared with the reference live."""
import numpy as np
import pytest

import hc_dest_emul as hd
from hc_dest_emul import host_hc_dest, mg, mgd


@pytest.fixture(scope="module", autouse=True)
def emul():
    if hd.load() is None:
        pytest.skip("g++ not available")


def check_decodes(oracle, out, consumed, data):
    assert oracle.decompress(out, consumed) == (consumed, bytes(data[:consumed]))


def test_vectors_match_the_reference(oracle):
    doc, ins = hd.golden()
    data = {}
    checked = 0
    for iid, lv, rb, rets, cons, dig in doc["vectors"]:
        i = ins[iid]
        if iid not in data:
            data = {iid: mg.make_input(oracle, i["size"], i["kind"], i["seed"])}
            assert mg.digest(data[iid]) == i["sha256"], i
        d = data[iid]
        ts = mgd.targets(i["size"], rb)
        res = [host_hc_dest(d, t, lv, chain_fill=0x3C5A) for t in ts]
        assert [r for r, _, _ in res] == rets and [c for _, c, _ in res] == cons, (i, lv)
        assert mgd.run_digest(res) == dig, (i, lv)
        for t, (r, c, out) in zip(ts, res):
            if t >= 1:
                assert r >= 1
                check_decodes(oracle, out, c, d)
            else:
                assert (r, c) == (0, i["size"])
        checked += 1
    assert checked == len(doc["vectors"]) > 500


def test_run_digests_match_the_reference(oracle):
    doc, _ = hd.golden()
    runs, res = [], []
    for d, t, lv in mgd.random_cases(oracle, doc["run_cases"]):
        res.append(host_hc_dest(d, t, lv, chain_fill=0x1234))
        r, c, out = res[-1]
        if r > 0:
            check_decodes(oracle, out, c, d)
        if len(res) == doc["run_chunk"]:
            runs.append(mgd.run_digest(res))
            res = []
    assert runs == doc["run_digests"]


def test_small_targets_keep_the_output_inside(oracle):
    """Targets below 8 put the reference's reduced end before dst: the block ends in a literal run alone."""
    d = mg.make_input(oracle, 65536, "p50", 1)
    assert host_hc_dest(d, 1, 9)[:3] == (1, 0, b"\x00")
    for lv in (1, 2, 3, 9):
        for t in range(1, 17):
            r, c, out = host_hc_dest(d, t, lv)
            assert 1 <= r <= t, (lv, t)
            if t < 8:
                assert out == bytes([c << 4]) + d[:c].tobytes(), (lv, t)
            check_decodes(oracle, out, c, d)


def test_levels_above_nine_are_not_built():
    for lv in (10, 11, 12, 100):
        assert host_hc_dest(b"x" * 100, 200, lv)[0] == -1


def test_live_against_the_reference(reference):
    rng = np.random.default_rng(98)
    for k in range(300):
        n = int(rng.choice([0, 13, 50, 777, 5000, 65536, 131072]))
        kind = mg.KINDS[int(rng.integers(0, len(mg.KINDS)))]
        d = mg.make_input(reference, n, kind, 91000 + k)
        b = mg.compress_bound(n)
        lv = int(rng.integers(-2, 10))
        t = int(rng.choice([b, b - 1, int(rng.integers(-1, b)), int(rng.integers(1, 64)), n // 2, 1 << 30]))
        assert host_hc_dest(d, t, lv) == mgd.reference_hc_dest(reference, d, t, lv), (n, kind, lv, t)
