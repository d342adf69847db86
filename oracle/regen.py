"""Regenerate the goldens under tests/golden/ from a reference checkout -- TEST INFRASTRUCTURE ONLY.

    ICNN_REFERENCE_DIR=<checkout> python -m oracle.regen [golden ...]      (from the repository root)

Every generator module has ``GOLDEN`` (its file under tests/golden/) and ``generate()`` -> {name: array}, except
``gen_golden``, which writes one file per entry of its ``CASES``: ``GOLDEN % case`` from ``generate(case)``.  The
generators are deterministic: a regeneration rewrites every file with identical bytes (tests/test_oracle_regen.py).
"""
import functools
import importlib
import os
import sys

import numpy as np

from oracle import refcode

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
GENERATORS = ("gen_golden", "gen_golden_grad", "gen_golden_adam", "gen_golden_gd_grad", "gen_golden_tfshim",
              "gen_golden_bundle_grad", "gen_golden_conv", "gen_golden_conv_grad", "gen_golden_conv_gd_grad",
              "gen_golden_td_grad")


def goldens(generators=GENERATORS):
    """-> [(file under tests/golden/, generate)] of the given generator modules."""
    out = []
    for name in generators:
        mod = importlib.import_module("oracle." + name)
        if name == "gen_golden":
            out += [(mod.GOLDEN % case[0], functools.partial(mod.generate, case[0])) for case in mod.CASES]
        else:
            out.append((mod.GOLDEN, mod.generate))
    return out


def write(golden, arrays):
    path = os.path.join(GOLDEN_DIR, golden)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez_compressed(path, **arrays)
    print("wrote %s: %d arrays, %d KB" % (path, len(arrays), os.path.getsize(path) // 1024), flush=True)


def main(generators=GENERATORS, only=()):
    """Write the goldens of ``generators`` (those named in ``only``, if any)."""
    if not refcode.available():
        sys.exit("no reference checkout at $ICNN_REFERENCE_DIR")
    for golden, generate in goldens(generators):
        if not only or golden in only:
            write(golden, generate())


if __name__ == "__main__":
    main(only=sys.argv[1:])
