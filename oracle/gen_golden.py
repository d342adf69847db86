#!/usr/bin/env python
"""Generate tests/golden/*.npz by running the UNMODIFIED reference modules.

TEST INFRASTRUCTURE ONLY.  Needs a checkout of the reference (locuslab/icnn) at $ICNN_REFERENCE_DIR;
the tests read only the committed .npz files.  The three reference files import unchanged under numpy/scipy:
    lib/bundle_entropy.py        (solveBatch, solver='pc' / 'boyd')
    lib/bundle_entropy_dual.py   (solveBatch)
    RL/src/bundle_entropy.py     (solveBatch)
The PICNN f/g callback they are fed is oracle/picnn_np.py (the reference's own f is a
TensorFlow graph and TensorFlow is not installed) in float64; inputs are regenerated from the
seed by oracle/synth.py, and a checksum of the inputs is stored so generator drift is caught.

Usage:  python -m oracle.gen_golden [case ...]      -> tests/golden/<case>.npz
"""
import hashlib
import sys
import time

import numpy as np

from oracle import picnn_np, refcode, regen, synth

GOLDEN = "%s.npz"        # % case name

# (case name, config, B, nIter, variant, solver)
CASES = [
    ("c1_pc", "C1", 64, 5, "lib", "pc"),
    ("c1_dual", "C1", 64, 5, "dual", None),
    ("c1_rl", "C1", 64, 5, "rl", None),
    ("c1_boyd", "C1", 8, 5, "lib", "boyd"),
    ("c1_pc_long", "C1", 32, 20, "lib", "pc"),
    ("c3_pc", "C3", 16, 10, "lib", "pc"),
    ("c3_dual", "C3", 16, 10, "dual", None),
    ("c4_rl", "C4", 128, 5, "rl", None),
    ("c4_rl_long", "C4", 32, 12, "rl", None),
    ("t_pc", "T", 8, 10, "lib", "pc"),
    ("t_dual", "T", 8, 10, "dual", None),
    ("c2_pc", "C2", 4, 30, "lib", "pc"),
    ("c5_pc", "C5", 2, 8, "lib", "pc"),
    # round 2: the configs' OWN horizons (VERDICT r01 item 2a) -- KS = 51 at C5, 30 iterations at C2
    ("c3_pc_full", "C3", 32, 10, "lib", "pc"),
    ("c2_pc_full", "C2", 8, 30, "lib", "pc"),
    ("c5_pc_full", "C5", 2, 50, "lib", "pc"),
]


def inputs_digest(p, x, y0):
    h = hashlib.sha256()
    for arr in [x, y0] + [w for w in p.Wy if w is not None] + [w for w in p.Wz if w is not None]:
        h.update(np.ascontiguousarray(arr, dtype=np.float64).tobytes())
    return h.hexdigest()


def pack_ragged(lst, kmax, inner_shape, dtype=np.float64):
    B = len(lst)
    out = np.zeros((B, kmax) + tuple(inner_shape), dtype=dtype)
    for u, rows in enumerate(lst):
        for j, r in enumerate(rows):
            out[u, j] = r
    return out


def generate(name):
    """-> the arrays of tests/golden/<name>.npz: the UNMODIFIED reference module run on the seeded case."""
    _, cfgname, B, nIter, variant, solver = next(c for c in CASES if c[0] == name)
    cfg = synth.CONFIGS[cfgname]
    p, x, y0 = synth.make_inputs(cfgname, B=B)
    fg = picnn_np.make_fg(p, x, affine=cfg["affine"])
    if variant == "lib":
        mod = refcode.load("ref_pc", "lib/bundle_entropy.py")
        call = lambda: mod.solveBatch(fg, y0.copy(), nIter=nIter, solver=solver)  # noqa: E731
    elif variant == "dual":
        mod = refcode.load("ref_dual", "lib/bundle_entropy_dual.py")
        call = lambda: mod.solveBatch(fg, y0.copy(), nIter=nIter)  # noqa: E731
    else:
        mod = refcode.load("ref_rl", "RL/src/bundle_entropy.py")
        call = lambda: mod.solveBatch(fg, y0.copy(), nIter=nIter)  # noqa: E731
    t0 = time.time()
    with refcode.quiet():
        xf, A, b, lam, xs, nIters = call()
    counts = np.array([len(a) for a in A], dtype=np.int32)
    print("%-12s %-3s B=%-4d nIter=%-3d %-4s  %.1fs  k mean %.2f max %d  nIters mean %.2f" % (
        name, cfgname, B, nIter, variant, time.time() - t0, counts.mean(), counts.max(), np.mean(nIters)))
    kmax = max(1, int(counts.max()))
    n = cfg["n"]
    out = dict(
        config=cfgname, B=B, nIter=nIter, variant=variant, solver=solver or "",
        digest=inputs_digest(p, x, y0),
        x=xf, counts=counts, nIters=np.array(nIters, dtype=np.int32),
        lam=pack_ragged([list(l) if l is not None else [] for l in lam], kmax, ()),
        b=pack_ragged(b, kmax, ()),
    )
    if n <= 512:  # keep fixtures small: rows / iterates only for the small shapes
        out["A"] = pack_ragged(A, kmax, (n,))
        out["xs"] = pack_ragged(xs, kmax, (n,))
    return out


if __name__ == "__main__":
    regen.main(("gen_golden",), only=[GOLDEN % c for c in sys.argv[1:]])
