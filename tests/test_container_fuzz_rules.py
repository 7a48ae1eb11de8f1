"""The container fuzz (tests/container_fuzz.py) without a GPU: every model judge against the reference's judge on the
fuzz's cases where oracle/_ref is built (a disagreement blames the model), the models against the reference's run
digests of tests/golden/container_fuzz.json everywhere, and the host builds of the device steps on the fuzz's data:
the file walk (tests/emul/decompress_files_emul.cpp), the host readers' group plan and placement (files_plan_emul.cpp,
files_place_emul.cpp) on the mutated files, and the writers' index passes (compress_frames_emul.cpp,
compress_legacy_emul.cpp) on the fuzzed sizes, capacities and budgets."""
import os

import numpy as np
import pytest

import container_fuzz as F
import compress_legacy_model as LM
import decompress_files_model as DM
from conftest import load_golden


@pytest.fixture(scope="module")
def models(oracle):
    return F.Judge(oracle, use_reference=False)


# 16 seeds of 10 cases each by default; CONTAINER_FUZZ_LIVE_SEEDS=N runs N seeds (300: 3 000 cases)
LIVE_SEEDS = range(100, 100 + int(os.environ.get("CONTAINER_FUZZ_LIVE_SEEDS", "16")))


@pytest.mark.parametrize("seed", LIVE_SEEDS)
def test_models_match_the_reference(oracle, reference, models, seed):
    """every record of run_case -- writes at every capacity, mutated frames read with and without skipChecksums, the
    files read -- from the models equals the reference's"""
    ref = F.Judge(oracle, use_reference=True)
    n = 0
    for k, c in F.small_cases(seed, 10):
        datas = F.case_data(oracle, c)
        got, want = F.run_case(models, seed, k, c, datas), F.run_case(ref, seed, k, c, datas)
        assert len(got) == len(want)
        for g, w in zip(got, want):
            assert g[:2] == w[:2] and g[2] == w[2], (seed, k, g[0], g[1], w[1])
        n += len(got)
    assert n > 30


def test_run_digests(models):
    """the models reproduce the reference's run digests, so the generator and the models stay pinned without it"""
    doc = load_golden("container_fuzz.json")
    assert (doc["cases"], doc["chunk"], doc["max_total"]) == (F.DIGEST_CASES, F.DIGEST_CHUNK, F.SMALL)
    for seed in F.DIGEST_SEEDS:
        assert F.digest_run(models, seed) == doc["runs"][str(seed)], seed


def test_cases_are_deterministic():
    for seed in (1, 2026):
        for k in range(30):
            assert F.case(seed, k) == F.case(seed, k)
    levels = {F.case(1, k)["level"] for k in range(200)}
    assert levels == set(F.LEVELS)


@pytest.mark.parametrize("seed", [1, 2, 2026])
def test_files_emulator_matches_the_model(oracle, models, seed):
    """the host build of the walk, plan and placement of LZ4B200_decompress_files on the fuzz's mutated files, at
    capacities at, below and one below the decoded size"""
    import test_decompress_files_rules as R
    rng = np.random.default_rng(seed)
    for k, c in F.small_cases(seed, 5):
        datas = F.case_data(oracle, c)
        files = [f for _, f in F.mutated_files(oracle, c, F.written(models, c, datas), rng)]
        for skip in (False, True):
            mu, mb = DM.budget_needed(files, skip)
            sized = DM.decompress_files(oracle, files, [1 << 40] * len(files), mu, mb, skip, content=False)
            caps = [max((r if r >= 0 else p) - int(rng.integers(0, 2)), 0) for r, _, p, _ in sized]
            for size_only in (False, True):
                R._check(oracle, files, caps, mu, mb, skip, size_only)


def _attach(shim):
    import host_build
    lib = host_build.require()
    for name, res, args in shim:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


@pytest.mark.parametrize("seed", [1, 2026])
def test_host_plan_and_placement_on_mutated_files(oracle, models, seed):
    """the host readers' group plan and fold (tests/emul/files_plan_emul.cpp) and the host-to-device placement
    (tests/emul/files_place_emul.cpp) on the fuzz's mutated files, with groups small enough that their edges fall inside
    frames, at capacities at and one below each file's decoded size"""
    import test_decompress_files_host_rules as H
    import test_files_device_io_rules as P
    plan, place = _attach(H.SHIM), _attach(P.SHIM)
    rng = np.random.default_rng(seed)
    files = []
    for k, c in F.small_cases(seed, 4):
        files += [f for _, f in F.mutated_files(oracle, c, F.written(models, c, F.case_data(oracle, c)), rng)]
    for skip in (False, True):
        mu, mb = DM.budget_needed(files, skip)
        sized = DM.decompress_files(oracle, files, [1 << 40] * len(files), mu, mb, skip)
        caps = [max((r if r >= 0 else p) - int(rng.integers(0, 2)), 0) for r, _, p, _ in sized]
        dev_sized = H.device_sizes(plan, oracle, files, skip)
        for group_bytes in (64 << 10, 300 << 10, F.MIB):
            H.check_plan(plan, oracle, files, caps, skip, group_bytes, dev_sized)
            P.check_place(place, oracle, files, caps, skip, group_bytes)


@pytest.mark.parametrize("seed", [1, 2, 2026])
def test_writer_index_passes_on_fuzzed_batches(seed):
    """the index passes of LZ4B200_compress_frames and LZ4B200_compress_legacy (tests/emul/compress_frames_emul.cpp,
    compress_legacy_emul.cpp) on the fuzz's sizes and capacities, at the budget the batch needs, one block short and
    none"""
    import test_compress_frames_rules as WF
    import test_compress_legacy_rules as WL
    import compress_frames_model as CFM
    import host_build
    C, ll = WF.C, WF._ll
    llp, ip = C.POINTER(ll), C.POINTER(C.c_int)
    lib = host_build.require()
    lib.cframes_index_host.restype = ll
    lib.cframes_index_host.argtypes = [llp, llp, llp, ll, C.c_int, C.c_int, llp] + [llp] * 6 + [ip, llp, ip]
    lib.clegacy_index_host.restype = None
    lib.clegacy_index_host.argtypes = [llp, llp, llp, ll, ll] + [llp] * 5 + [llp, ip, llp, ip]
    rng = np.random.default_rng(seed)
    for k in range(40):
        c = dict(F.case(seed, k), bsum=False, csum=False)
        sizes = np.array([it["size"] for it in c["items"]], dtype=np.int64)
        caps = np.array([F.capacity(c, it, seed * 1000003 + k * 1009 + i) for i, it in enumerate(c["items"])],
                        dtype=np.int64)
        if c["legacy"]:
            need = sum(LM.n_chunks(n) for n, cap in zip(sizes, caps) if cap >= LM.bound(n))
            for budget in (need, max(need - 1, 0), 0):
                WL._check_batch(lib, sizes, caps, budget, rng)
        else:
            need = CFM.budget([n if cap >= CFM.bound(n, c["bsid"]) else -1 for n, cap in zip(sizes, caps)], c["bsid"])
            for budget in (need, [max(x - 1, 0) for x in need], [0, 0, 0, 0]):
                WF._check_batch(lib, sizes, caps, c["bsid"], budget, rng)
