"""The V3 two-sweep kernel's one-log update against ICNN_PC_TWOLOG=1.

The V3 build does not store u = G^T z.  Its update used to recover u_old = ry_old - logit(y_old) and form
ry_new = logit(y_new) + u_old + a du: two logs and two divisions per element.  By default it forms the same quantity
as ry_old + a du + log(y_new (1 - y_old) / (y_old (1 - y_new))), one log and one division.  ICNN_PC_TWOLOG=1 restores
the two-log expression.  The two differ by rounding only, so every decision (counts, permutation, status, finished
flags, iterations) is the same and y* and lambda agree to a few ulp.
"""
import numpy as np
import pytest

from test_gpu_k2_builds import CASES, LARGE, last_launch, max_affine_fg, orthogonal_fg, planned

pytestmark = pytest.mark.gpu
np.seterr(all="ignore")

ENV = ("ICNN_K2_SMALL", "ICNN_K2_PC", "ICNN_PC_V3", "ICNN_K2_WPS", "ICNN_K2_CS", "ICNN_K2_RESIDENT", "ICNN_PC_LEGACY",
       "ICNN_PC_PREFETCH", "ICNN_PC_SEED", "ICNN_PC_TWOLOG")


@pytest.fixture(autouse=True)
def clean_env(monkeypatch):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)


def solve(fg, n, B, nIter, monkeypatch, twolog):
    from icnn_b200 import bundle_entropy as be
    if twolog:
        monkeypatch.setenv("ICNN_PC_TWOLOG", "1")
    else:
        monkeypatch.delenv("ICNN_PC_TWOLOG", raising=False)
    r = be.solveBatch(fg, np.full((B, n), 0.5), nIter=nIter, return_state=True)
    st = r[6]
    out = dict(y=np.array(r[0]), lam=st.lam.cpu().numpy(), count=st.count.cpu().numpy(), perm=st.perm.cpu().numpy(),
               status=st.status.cpu().numpy(), finished=st.finished.cpu().numpy(), nIters=np.array(r[5]))
    return out, last_launch()


# the V3 cases of test_gpu_k2_builds.py (k >= 41 in the LARGE one), plus n_y = 4096 (C5's width)
BUILDS = {"v3-random": CASES["two-v3-8x4"] + (max_affine_fg,),
          "v3-k%d" % LARGE["two-v3-8x4"][2]: LARGE["two-v3-8x4"] + (orthogonal_fg,)}
BUILDS["v3-4096"] = (4096, 8, 20) + CASES["two-v3-8x4"][3:] + (max_affine_fg,)


@pytest.mark.parametrize("cid", list(BUILDS))
def test_one_log_update_matches_two_log(cid, monkeypatch):
    n, B, nIter, variant, want, kmin, env, make_fg = BUILDS[cid]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    KS = min(nIter, n) + 1
    plan = planned(n, KS, variant)
    assert plan[:6] == want, (plan, want)
    new, ran = solve(make_fg(n, B), n, B, nIter, monkeypatch, False)
    assert ran == plan, (ran, plan)
    ref, ran0 = solve(make_fg(n, B), n, B, nIter, monkeypatch, True)
    assert ran0 == plan, (ran0, plan)
    for key in ("count", "perm", "status", "finished", "nIters"):
        np.testing.assert_array_equal(new[key], ref[key], err_msg=key)
    assert new["count"].max() >= kmin, (new["count"], kmin)
    dy, dl = np.abs(new["y"] - ref["y"]).max(), np.abs(new["lam"] - ref["lam"]).max()
    print("%s: ran %s, counts %s, max |dy*| %.2e, max |dlambda| %.2e" % (cid, ran, list(new["count"]), dy, dl))
    assert dy <= 1e-13 and dl <= 1e-13, (dy, dl)
