"""Generate tests/golden/compress_legacy.json by running the COMPILED REFERENCE TOOL (oracle/_ref/lz4).

    python tests/golden/make_golden_compress_legacy.py

For every case of tests/compress_legacy_model.corpus_cases() -- levels --fast=70000 .. -13, sizes 0 .. 2 x 8 MiB + 17 and
20 MiB, P50, P90, incompressible and zero data -- it records the length and SHA-256 of what `lz4 -l -c` writes with the
input piped to its standard input, and the legacy bound.  The inputs are rebuilt by the tests from their recipes (the
project's own datagen and numpy), so the tests never need the reference."""
import hashlib
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import compress_legacy_model as M          # noqa: E402
from oracle.pyoracle import Oracle         # noqa: E402

LZ4 = os.path.join(ROOT, "oracle", "_ref", "lz4")


def main():
    orc = Oracle()
    streams = []
    for cid, kind, size, seed, level in M.corpus_cases():
        data = M.corpus_data(orc, kind, size, seed)
        r = subprocess.run([LZ4, "-q", "-l", "-c"] + M.cli_args(level), input=data, capture_output=True, check=True)
        streams.append({"id": cid, "kind": kind, "size": size, "seed": seed, "level": level,
                        "length": len(r.stdout), "sha256": hashlib.sha256(r.stdout).hexdigest(),
                        "bound": M.bound(size)})
    with open(os.path.join(HERE, "compress_legacy.json"), "w") as fh:
        json.dump({"source": "lz4 v1.10.0 command-line tool: `lz4 -q -l -c <level>` with the input on standard input",
                   "streams": streams}, fh, indent=0)
        fh.write("\n")


if __name__ == "__main__":
    main()
