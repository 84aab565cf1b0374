"""Generates tests/golden/*.npz by running every script of tests/scenarios.py
through the REFERENCE oracle (oracle/_ref/libbng_ref.so = the reference's own
eBPF C sources compiled natively), and tests/golden/reference_digests.npz from
the re-seeded corpora of tests/test_oracle_differential.py and the mutated ones
of tests/test_oracle_fuzz.py.  Building that library needs the reference's
sources (oracle/Makefile, REF=...); the fixtures it writes are committed, so the
tests need neither.

    python tests/golden/make_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import harness  # noqa: E402
import scenarios  # noqa: E402
import test_oracle_differential as diff  # noqa: E402
import test_oracle_fuzz as fuzz  # noqa: E402
from oracle import pyoracle  # noqa: E402


def main():
    pyoracle.build("ref")
    for name, fn in scenarios.ALL_SCRIPTS.items():
        be = harness.OracleBackend("reference")
        res = harness.run_script(be, fn())
        path = os.path.join(HERE, name + ".npz")
        harness.save_golden(path, res)
        print(f"{name}: {len(res)} arrays, {os.path.getsize(path) / 1024:.0f} KiB")
    write_reference_digests()


def write_reference_digests():
    scripts = {diff.corpus_id(fam, s): lambda fam=fam, s=s: diff.FRESH[fam](s) for fam in diff.FRESH for s in diff.SEEDS}
    scripts.update({fuzz.corpus_id(p, s): lambda p=p, s=s: fuzz.fuzz_script(p, s) for p in fuzz.TARGETS for s in fuzz.FUZZ_SEEDS})
    out = {name: harness.digest(harness.run_script(harness.OracleBackend("reference"), fn())) for name, fn in scripts.items()}
    np.savez_compressed(harness.REFERENCE_DIGESTS, **out)


if __name__ == "__main__":
    main()
