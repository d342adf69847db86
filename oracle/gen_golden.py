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

Usage:  python oracle/gen_golden.py [case ...]
"""
import contextlib
import hashlib
import importlib.util
import io
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import picnn_np, synth  # noqa: E402

REF = os.environ.get("ICNN_REFERENCE_DIR", "")


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


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


def compute_case(name, cfgname, B, nIter, variant, solver):
    """-> (arrays of the golden file, seconds, counts, nIters): the UNMODIFIED reference module run on the seeded case."""
    cfg = synth.CONFIGS[cfgname]
    p, x, y0 = synth.make_inputs(cfgname, B=B)
    fg = picnn_np.make_fg(p, x, affine=cfg["affine"])
    if variant == "lib":
        mod = _load("ref_pc", os.path.join(REF, "lib/bundle_entropy.py"))
        call = lambda: mod.solveBatch(fg, y0.copy(), nIter=nIter, solver=solver)  # noqa: E731
    elif variant == "dual":
        mod = _load("ref_dual", os.path.join(REF, "lib/bundle_entropy_dual.py"))
        call = lambda: mod.solveBatch(fg, y0.copy(), nIter=nIter)  # noqa: E731
    else:
        mod = _load("ref_rl", os.path.join(REF, "RL/src/bundle_entropy.py"))
        call = lambda: mod.solveBatch(fg, y0.copy(), nIter=nIter)  # noqa: E731
    t0 = time.time()
    with contextlib.redirect_stdout(io.StringIO()), np.errstate(all="ignore"):
        xf, A, b, lam, xs, nIters = call()
    dt = time.time() - t0
    counts = np.array([len(a) for a in A], dtype=np.int32)
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
    return out, dt, counts, nIters


def run_case(name, cfgname, B, nIter, variant, solver):
    out, dt, counts, nIters = compute_case(name, cfgname, B, nIter, variant, solver)
    path = os.path.join(ROOT, "tests", "golden", name + ".npz")
    np.savez_compressed(path, **out)
    print("%-12s %-3s B=%-4d nIter=%-3d %-4s  %.1fs  k mean %.2f max %d  nIters mean %.2f  -> %s (%d KB)" % (
        name, cfgname, B, nIter, variant, dt, counts.mean(), counts.max(), np.mean(nIters), path,
        os.path.getsize(path) // 1024))


if __name__ == "__main__":
    want = set(sys.argv[1:])
    for case in CASES:
        if not want or case[0] in want:
            run_case(*case)
