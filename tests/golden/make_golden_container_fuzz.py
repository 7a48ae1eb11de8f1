"""Writes tests/golden/container_fuzz.json: the run digests of the container fuzz (tests/container_fuzz.py) judged by the
reference -- LZ4F_compressFrame, LZ4F_decompress and the block compressors of oracle/_ref/libref_lz4.so.  For each seed,
one SHA-256 digest per chunk of cases over every (result, consumed, bytes) the judges give.  The file holds the recipe
(seeds, case counts) and digests only; tests/test_container_fuzz_rules.py rebuilds every case from its seed and checks
the host models against it.

    python tests/golden/make_golden_container_fuzz.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import container_fuzz as F  # noqa: E402
from oracle.pyoracle import Oracle  # noqa: E402


def main():
    judge = F.Judge(Oracle(), use_reference=True)
    doc = {"about": "run digests of tests/container_fuzz.py judged by the reference (tests/golden/"
                    "make_golden_container_fuzz.py)",
           "cases": F.DIGEST_CASES, "chunk": F.DIGEST_CHUNK, "max_total": F.SMALL,
           "runs": {str(s): F.digest_run(judge, s) for s in F.DIGEST_SEEDS}}
    with open(os.path.join(HERE, "container_fuzz.json"), "w") as f:
        json.dump(doc, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
