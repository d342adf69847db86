"""Every golden under tests/golden/ regenerates bit for bit from a reference checkout: the generator list of
oracle/regen.py, one parameter per golden file (skipped without a checkout at $ICNN_REFERENCE_DIR)."""
import os

import numpy as np
import pytest

from oracle import refcode, regen

GOLDENS = regen.goldens()


@pytest.mark.skipif(not refcode.available(), reason="no reference checkout at $ICNN_REFERENCE_DIR")
@pytest.mark.parametrize("golden, generate", GOLDENS, ids=[g for g, _ in GOLDENS])
def test_golden_regenerates_from_the_reference(golden, generate, golden_dir):
    gold = np.load(os.path.join(golden_dir, golden))
    out = generate()
    assert set(out) == set(gold.files)
    for k, a in out.items():
        np.testing.assert_array_equal(np.asarray(a, dtype=gold[k].dtype), gold[k], err_msg=k)
