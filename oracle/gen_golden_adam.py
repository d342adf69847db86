#!/usr/bin/env python
"""Golden vectors for the RL Adam argmin from the reference's own `Agent.adam` body
(RL/src/icnn.py:160-215; the module imports TensorFlow, so the method source is cut out with ast
and exec'd with a stub `self`).  func = oracle fg_entr on the C4 (HalfCheetah) dims.
TEST INFRASTRUCTURE ONLY; needs a checkout of the reference at $ICNN_REFERENCE_DIR.
Usage:  python -m oracle.gen_golden_adam   -> tests/golden/adam.npz"""
import types

import numpy as np

from oracle import adam_np, refcode, regen, synth

GOLDEN = "adam.npz"


def generate():
    adam = refcode.extract("RL/src/icnn.py", ["Agent.adam"], {"np": np})["adam"]
    out = {}
    for tag, B in (("c4", 96),):
        p, x, _ = synth.make_inputs("C4", B=B)
        func = adam_np.make_fg_entr(p, x)
        stub = types.SimpleNamespace(dimA=p.n)
        with refcode.quiet() as buf:
            best = adam(stub, func, x)
        its = [int(s.split()[3]) for s in buf.getvalue().splitlines() if "Adam took" in s]
        out[tag + "_act_best"] = best
        out[tag + "_iters"] = np.array(its[-1] if its else 1000)
    return out


if __name__ == "__main__":
    regen.main(("gen_golden_adam",))
