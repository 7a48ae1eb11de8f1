"""Generate tests/golden/decompress_files.json by running the COMPILED REFERENCE TOOL (oracle/_ref/lz4).

    python tests/golden/make_golden_decompress_files.py

For every file of the corpus -- single frames, concatenations of frames, skippable frames, `lz4 -l` legacy streams,
trailing garbage, truncations at and around every unit boundary, the empty file -- it records the recipe that rebuilds
the file (tests/decompress_files_model.build_file) and what `lz4 -d -c` and `lz4 -d -c --no-frame-crc` do with the file
piped to their standard input: exit status, output length and SHA-256.  Frames the tool writes are recorded as the
recipe of the same bytes from the frame model (the maker checks the tool's output against the rebuild), and only a
linked-block frame, which the model cannot write, is kept verbatim.  Legacy streams are rebuilt from datagen with
LZ4_compress_default per 8 MiB chunk, checked the same way against `lz4 -l`.  One file per line."""
import hashlib
import json
import os
import random
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import decompress_files_model as dm        # noqa: E402
from oracle.pyoracle import Oracle         # noqa: E402

LZ4 = os.path.join(ROOT, "oracle", "_ref", "lz4")
MIB = 1 << 20


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


def run(args, data):
    r = subprocess.run([LZ4, "-q"] + args, input=data, capture_output=True)
    return r.returncode, r.stdout


def cli_frame(tmp, oracle, spec, opts):
    """what `lz4 -c opts` writes for the content of spec, read from a file (so that --content-size has a size)"""
    src = os.path.join(tmp, "in.bin")
    with open(src, "wb") as fh:
        fh.write(dm.fm.content(oracle.datagen, spec))
    r = subprocess.run([LZ4, "-q", "-c"] + opts + [src], capture_output=True, check=True)
    return r.stdout


def corpus(oracle, tmp):
    cases = []

    def add(name, parts, cut=None, flip=None):
        cases.append({"name": name, "parts": parts, "cut": cut, "flip": flip})

    # single frames of the library's frame model: every class, each checksum combination, with and without size
    for i, (spec, bsid) in enumerate([([30000, 0.5, 1, 0], 4), ([200000, 0.5, 2, 50000], 5), ([900000, 0.3, 3, 0], 6),
                                      ([1500000, 0.7, 4, 300000], 7), ([0, 0.5, 0, 0], 4), ([1, 0.5, 5, 0], 4)]):
        for k, (bsum, csum) in enumerate([(0, 0), (0, 1), (1, 0), (1, 1)]):
            add("frame%d_%d" % (i, k), [["frame", spec, bsid, bool((i + k) % 2), bsum, csum]])
    # frames the `lz4` tool writes: the frame model's bytes for the tool's options (block size ID, content size, block
    # and content checksums; -BD on one 4 MB block is written independent), checked against the tool in main()
    spec = [300000, 0.5, 11, 3000]
    for opts, (bsid, csize, bsum, csum) in [
            ([], (7, False, 0, 1)), (["-BX"], (7, False, 1, 1)), (["--content-size"], (7, True, 0, 1)),
            (["-B4"], (4, False, 0, 1)), (["-B5"], (5, False, 0, 1)), (["-B6"], (6, False, 0, 1)),
            (["-B7"], (7, False, 0, 1)), (["-BD"], (7, False, 0, 1)), (["--no-frame-crc"], (7, False, 0, 0)),
            (["-BX", "--content-size", "-B4"], (4, True, 1, 1)), (["-B5", "-BX"], (5, False, 1, 1))]:
        add("cli" + "".join(opts), [["frame", spec, bsid, csize, bsum, csum]])
        cases[-1]["cli"] = opts
    add("cli-BD-multi", [["hex", cli_frame(tmp, oracle, [140000, 1.0, 12, 0], ["-B4", "-BD"]).hex()]])
    # corrupted checksums and payloads, behind a good frame
    good = ["frame", [3000, 0.5, 13, 0], 4, False, 0, 1]
    bad = ["frame", [150000, 0.5, 14, 0], 4, False, 1, 1]
    g, b = (dm.build_file(oracle, {"parts": [p]}) for p in (good, bad))
    blocks, end = dm.fm.walk(b)
    for name, at in [("payload", blocks[0][0] + 100), ("blocksum", blocks[0][0] + blocks[0][1] + 1),
                     ("contentsum", end - 2)]:
        add("corrupt_" + name, [good, bad, good], flip=[len(g) + at])
    # concatenations of 1 .. 40 frames of mixed classes and checksum flags
    rng = random.Random(1234)
    pool = []
    for j in range(24):
        size = rng.choice([0, 1, 100, 5000, 70000, 300000, 1200000])
        pool.append(["frame", [size, rng.choice([0.2, 0.5, 0.9]), 100 + j, size // 4 if j % 3 == 0 else 0],
                     rng.choice([4, 5, 6, 7]), bool(rng.getrandbits(1)), rng.getrandbits(1), rng.getrandbits(1)])
    for n in (1, 2, 3, 5, 8, 13, 21, 40):
        add("concat%d" % n, [rng.choice(pool) for _ in range(n)])
    # skippable frames: all 16 magics, size 0, large, as the last unit, between frames
    for nib in range(16):
        add("skip%x" % nib, [["skip", nib, 3 * nib, nib], ["frame", [5000, 0.5, 20 + nib, 0], 4, False, 0, 1]])
    add("skip_empty", [["skip", 0, 0, 0]])
    add("skip_large", [["frame", [5000, 0.5, 40, 0], 4, False, 0, 1], ["skip", 5, 3 * MIB, 41],
                       ["frame", [7000, 0.5, 42, 0], 4, True, 1, 1]])
    add("skip_last", [["frame", [5000, 0.5, 43, 0], 4, False, 0, 1], ["skip", 15, 100, 44]])
    add("skip_many", [["skip", k % 16, k % 5, k] for k in range(200)] + [["frame", [100, 0.5, 45, 0], 4, False, 0, 1]])
    # legacy streams of `lz4 -l`
    for name, size in [("0", 0), ("1", 1), ("8m-1", 8 * MIB - 1), ("8m", 8 * MIB), ("8m+1", 8 * MIB + 1),
                       ("20m", 20 * MIB)]:
        add("legacy_" + name, [["legacy", [size, 0.5, 50, 0]]])
    add("legacy_frames", [["legacy", [100000, 0.5, 51, 0]], ["frame", [5000, 0.5, 52, 0], 4, False, 0, 1],
                          ["legacy", [9 * MIB, 0.4, 53, 0]], ["skip", 3, 10, 54]])
    add("legacy_legacy", [["legacy", [100000, 0.5, 55, 0]], ["legacy", [300, 0.5, 56, 0]]])
    add("legacy_block0", [["word", dm.LEGACY_MAGIC], ["word", 0]])
    add("legacy_block0_mid", [["legacy", [1000, 0.5, 57, 0]], ["word", 0]])
    add("legacy_bound", [["word", dm.LEGACY_MAGIC], ["word", dm.LEGACY_BOUND], ["hex", "00" * 64]])
    add("legacy_bound1", [["legacy", [1000, 0.5, 58, 0]], ["word", dm.LEGACY_BOUND + 1], ["hex", "00" * 64]])
    add("legacy_garbage_block", [["word", dm.LEGACY_MAGIC], ["word", 16], ["hex", "ff" * 16]])
    # trailing garbage
    for n in (1, 2, 3, 4, 7):
        add("trail%d" % n, [["frame", [3000, 0.5, 60, 0], 4, False, 0, 1], ["hex", "5a" * n]])
    add("trail_magicish", [["frame", [3000, 0.5, 61, 0], 4, False, 0, 1], ["word", 0x184D2205]])
    add("bad_start", [["word", 0x12345678], ["frame", [3000, 0.5, 62, 0], 4, False, 0, 1]])
    add("empty", [])
    # truncations at every unit boundary +- 1
    trunc = [["frame", [2000, 0.5, 70, 0], 4, True, 1, 1], ["skip", 2, 20, 71], ["legacy", [3000, 0.5, 72, 0]],
             ["frame", [2500, 0.5, 73, 0], 4, False, 0, 1]]
    ends, at = [], 0
    for p in trunc:
        at += len(dm.build_file(oracle, {"parts": [p]}))
        ends.append(at)
    for e in [0] + ends:
        for d in (-1, 0, 1):
            if 0 <= e + d < ends[-1]:
                add("trunc%d" % (e + d), trunc, e + d)
    return cases


def main():
    oracle = Oracle()
    out = []
    with tempfile.TemporaryDirectory() as tmp:
        for case in corpus(oracle, tmp):
            data = dm.build_file(oracle, case)
            if "cli" in case:                          # the rebuild of a frame the tool writes is the tool's
                assert cli_frame(tmp, oracle, case["parts"][0][1], case.pop("cli")) == data, case["name"]
            for part in case["parts"]:                 # the rebuild of a legacy stream is the tool's
                if part[0] == "legacy":
                    content = dm.fm.content(oracle.datagen, part[1])
                    rc, ref = run(["-l", "-c"], content)
                    assert rc == 0 and ref == dm.build_file(oracle, {"parts": [part]}), case["name"]
            row = dict(case, size=len(data), sha256=sha(data))
            for key, args in (("verify", ["-d", "-c"]), ("skip", ["-d", "-c", "--no-frame-crc"])):
                rc, got = run(args, data)
                row[key] = {"exit": rc, "size": len(got), "sha256": sha(got)}
            out.append(row)
    with open(os.path.join(HERE, "decompress_files.json"), "w") as fh:
        fh.write('{"source": "lz4 v1.10.0 programs/lz4 -d -c (and --no-frame-crc), each file piped to standard input",\n'
                 '"files": [\n' + ",\n".join(json.dumps(row) for row in out) + "\n]}\n")


if __name__ == "__main__":
    main()
