"""The K2 dispatch table, pinned on the host: icnn_k2_plan returns the build icnn_bundle_step would launch for
(n_y, KS, solver) and the launch environment variables, without a device.  Every row of DESIGN.md §3 "Dispatch" is
checked on both sides of its boundaries, together with the KS limits (thread-per-sample kernel <= 10 slots, two-sweep
<= 62, any K2 <= 64, five-sweep shared memory at n_y = 8192) and each launch variable.  tests/test_gpu_k2_builds.py
runs the same builds on the device against the float64 oracle and checks with icnn_k2_last_launch that they ran.

A record is (family, warps per sample, column chunks | cluster size, V3, 16-byte rows, resident rows); minBlocks and
shared memory are checked where the table states them."""
import ctypes as C

import pytest

SMALL, TWO, FIVE = 0, 1, 2
ENV = ("ICNN_K2_SMALL", "ICNN_K2_PC", "ICNN_PC_V3", "ICNN_K2_WPS", "ICNN_K2_CS", "ICNN_K2_RESIDENT")


@pytest.fixture(autouse=True)
def clean_env(monkeypatch):
    """The plan reads the launch variables at every call: start each test from the default dispatch."""
    for k in ENV:
        monkeypatch.delenv(k, raising=False)


def plan_full(n, KS, solver="pc", variant="lib"):
    from icnn_b200 import _capi
    out = (C.c_int32 * _capi.K2_PLAN_LEN)()
    s = _capi.SOLVER_PC if solver == "pc" else _capi.SOLVER_NEWTON
    rc = _capi.lib.icnn_k2_plan(n, KS, s, _capi.VARIANT[variant], out)
    if rc != 0:
        return rc, _capi.lib.icnn_last_error().decode()
    return tuple(out)


def plan(n, KS, solver="pc", variant="lib"):
    r = plan_full(n, KS, solver, variant)
    assert len(r) == 8, r
    return r[:6]


def five(wps, cs=1, vec=1, res=0):
    return (FIVE, wps, cs, 0, vec, res)


def two(wps, nch, vec=1, v3=0):
    return (TWO, wps, nch, v3, vec, 0)


SMALL_REC = (SMALL, 0, 0, 0, 0, 0)

# (n_y, KS) -> build of the PC solver, by row of the dispatch table
PC_TABLE = [
    # n_y <= 8 and <= 10 slots: one thread per sample
    ((8, 9), SMALL_REC), ((8, 10), SMALL_REC), ((8, 11), two(1, 1)), ((9, 10), two(1, 1, vec=0)),
    # n_y <= 128: 1 warp, 1 chunk (scalar row loads when n_y % 4 != 0); <= 256: 1 warp, 2 chunks
    ((128, 11), two(1, 1)), ((129, 11), two(1, 2, vec=0)), ((132, 11), two(1, 2)), ((256, 11), two(1, 2)),
    # 256 < n_y <= 1024: five-sweep, 2 warps up to 512, then 4
    ((257, 11), five(2, vec=0)), ((260, 11), five(2)), ((512, 11), five(2)), ((513, 11), five(4, vec=0)),
    ((1024, 11), five(4)),
    # 1024 < n_y <= 2048: two-sweep 8 warps, 2 chunks; n_y % 4 != 0 -> five-sweep (SIMT Gram), 8 warps
    ((1025, 11), five(8, vec=0)), ((1028, 11), two(8, 2)), ((2048, 13), two(8, 2)), ((2050, 13), five(8, vec=0)),
    # 2048 < n_y <= 4096: V3 8 warps, 4 chunks while two samples fit an SM (KS <= 52 at 4096), else 16 warps, 2 chunks
    ((2052, 13), two(8, 4, v3=1)), ((4096, 51), two(8, 4, v3=1)), ((4096, 52), two(8, 4, v3=1)),
    ((4096, 53), two(16, 2)), ((4096, 57), two(16, 2)), ((4094, 11), five(8, vec=0)),
    # 4096 < n_y: 16 warps, 4 chunks while four n-vectors fit 227 KB, else five-sweep
    ((4098, 11), five(8, vec=0)), ((5000, 11), two(16, 4)), ((7000, 11), two(16, 4)), ((7200, 11), five(16)),
    ((8192, 11), five(16)), ((8192, 41), five(16)),
    # KS > 62: five-sweep at any n_y, warps by n_y, more warps (fewer samples per CTA) when the k x k matrices of
    # 8 / 4 samples do not fit one CTA, 16 when one CTA per SM is all that fits
    ((100, 62), two(1, 1)), ((100, 63), five(4)), ((100, 64), five(4)), ((200, 63), five(4)), ((513, 64), five(4, vec=0)),
    ((2048, 62), two(8, 2)), ((2048, 63), five(16)), ((2048, 64), five(16)),
]


@pytest.mark.parametrize("shape,want", PC_TABLE, ids=["n%d-KS%d" % s for s, _ in PC_TABLE])
def test_pc_dispatch_table(shape, want):
    assert plan(*shape) == want


# (variant, n_y, KS) -> build of the Newton solver: the five-sweep kernel, warps by n_y (1 up to 192, 2 up to 512,
# 4 up to 1024, then 8, or 16 when a single CTA per SM fits anyway)
NEWTON_TABLE = [
    (("rl", 6, 10), SMALL_REC), (("rl", 6, 11), five(1, vec=0)), (("dual", 8, 9), SMALL_REC), (("dual", 9, 10), five(1, vec=0)),
    (("dual", 159, 11), five(1, vec=0)), (("dual", 192, 11), five(1)), (("dual", 193, 11), five(2, vec=0)),
    (("dual", 512, 11), five(2)), (("dual", 513, 11), five(4, vec=0)), (("dual", 1024, 11), five(4)),
    (("dual", 1025, 11), five(8, vec=0)), (("dual", 2048, 13), five(8)), (("dual", 4096, 11), five(8)),
    (("dual", 4096, 41), five(16)), (("dual", 8192, 11), five(16)), (("lib", 2048, 13), five(8)),
    # eight one-warp samples per CTA hold KS <= 35 at n_y = 100; beyond, two warps and four samples, then four and two
    (("dual", 100, 35), five(1)), (("dual", 100, 36), five(2)), (("dual", 100, 64), five(4)), (("rl", 6, 64), five(4, vec=0)),
    (("dual", 200, 52), five(2)), (("dual", 200, 53), five(4)),
]


@pytest.mark.parametrize("shape,want", NEWTON_TABLE, ids=["%s-n%d-KS%d" % s for s, _ in NEWTON_TABLE])
def test_newton_dispatch_table(shape, want):
    variant, n, KS = shape
    assert plan(n, KS, "newton", variant) == want


def test_launch_bounds_and_shared_memory_of_the_table():
    """minBlocks and shared memory where the table states them: the 80-register 8-warp two-sweep build when three
    samples fit an SM, V3 at two CTAs per SM (a sample at n_y = 4096 / 51 slots needs 114 896 B), the 16-warp builds at
    one CTA per SM, the five-sweep 8-warp build at 3 CTAs while three fit in 225 KB."""
    assert plan_full(1028, 11)[6] == 3
    v3 = plan_full(4096, 51)
    assert v3[6] == 2 and v3[7] == 114896
    assert 2 * (plan_full(4096, 52)[7] + 1024) <= 228 * 1024
    assert plan_full(4096, 53)[6] == 1 and plan_full(5000, 11)[6] == 1
    assert plan_full(100, 11)[6] == 16 and plan_full(200, 11)[6] == 16       # one warp, 128-register build
    assert plan_full(1025, 11)[6] == 3 and plan_full(8192, 11)[6] == 1 and plan_full(512, 11)[6] == 3
    for shape in ((100, 11), (2048, 13), (4096, 52), (4096, 57), (5000, 11), (8192, 41), (1025, 11), (513, 11)):
        assert 0 < plan_full(*shape)[7] <= 227 * 1024, shape
    assert plan_full(8, 9)[6:] == (0, 0)


def test_shared_memory_edge_at_8192():
    """n_y = 8192 leaves the two-sweep kernel (four n-vectors are 256 KB) and the five-sweep kernel holds at most 41
    slots in 227 KB: one slot more is refused with a message, for either solver, instead of failing at launch."""
    for solver, variant in (("pc", "lib"), ("newton", "dual")):
        r = plan_full(8192, 41, solver, variant)
        assert r[:6] == five(16) and r[7] <= 227 * 1024, r
        rc, msg = plan_full(8192, 42, solver, variant)
        assert rc == -3 and "shared memory does not fit (n=8192, KS=42)" in msg, (rc, msg)
    rc, msg = plan_full(100, 65)
    assert rc == -3 and "KS=65 > 64" in msg


def test_arguments_are_checked_like_bundle_step():
    from icnn_b200 import _capi
    out = (C.c_int32 * _capi.K2_PLAN_LEN)()
    lib = _capi.lib
    assert lib.icnn_k2_plan(100, 11, _capi.SOLVER_PC, _capi.VARIANT["dual"], out) == -1
    assert b"Newton" in lib.icnn_last_error()
    assert lib.icnn_k2_plan(100, 11, 7, 0, out) == -1
    assert lib.icnn_k2_plan(100, 1, _capi.SOLVER_PC, 0, out) == -1
    assert lib.icnn_k2_plan(0, 11, _capi.SOLVER_PC, 0, out) == -1
    assert lib.icnn_k2_plan(100, 11, _capi.SOLVER_PC, 0, None) == -1
    assert lib.icnn_k2_last_launch(None) == -1
    assert lib.icnn_k2_last_launch(out) == 0          # no K2 enqueued on this thread: family -1
    assert out[0] == -1 and list(out)[1:] == [0] * 7


# (variables, (variant, n_y, KS)) -> build
ENV_TABLE = [
    # ICNN_K2_PC=legacy: the PC solver keeps the five-sweep kernel wherever the two-sweep one would run
    ({"ICNN_K2_PC": "legacy"}, ("lib", 100, 11), five(1)),
    ({"ICNN_K2_PC": "legacy"}, ("lib", 2048, 13), five(8)),
    ({"ICNN_K2_PC": "legacy"}, ("lib", 5000, 11), five(16)),
    ({"ICNN_K2_PC": "legacy"}, ("lib", 8, 9), SMALL_REC),
    # ICNN_PC_V3=0: the four-vector 16-warp build instead of V3
    ({"ICNN_PC_V3": "0"}, ("lib", 4096, 51), two(16, 2)),
    ({"ICNN_PC_V3": "0"}, ("lib", 2052, 13), two(16, 2)),
    # ICNN_K2_SMALL=0: the group kernels at n_y <= 8
    ({"ICNN_K2_SMALL": "0"}, ("lib", 8, 9), two(1, 1)),
    ({"ICNN_K2_SMALL": "0"}, ("rl", 6, 6), five(1, vec=0)),
    # the five-sweep launch variables reach only shapes that take the five-sweep kernel
    ({"ICNN_K2_RESIDENT": "1"}, ("lib", 2048, 13), two(8, 2)),
    ({"ICNN_K2_RESIDENT": "1"}, ("lib", 159, 11), two(1, 2, vec=0)),
    ({"ICNN_K2_WPS": "16"}, ("lib", 4096, 13), two(8, 4, v3=1)),
    ({"ICNN_K2_RESIDENT": "1", "ICNN_K2_PC": "legacy"}, ("lib", 512, 11), five(2, res=1)),
    ({"ICNN_K2_RESIDENT": "1", "ICNN_K2_PC": "legacy"}, ("lib", 159, 11), five(1, vec=0, res=1)),
    ({"ICNN_K2_RESIDENT": "1", "ICNN_K2_PC": "legacy"}, ("lib", 2048, 13), five(8, cs=2, res=1)),
    ({"ICNN_K2_RESIDENT": "1"}, ("dual", 2048, 13), five(8, cs=2, res=1)),
    ({"ICNN_K2_RESIDENT": "1", "ICNN_K2_CS": "8"}, ("dual", 4096, 13), five(8, cs=8, res=1)),
    ({"ICNN_K2_CS": "2"}, ("dual", 2048, 13), five(8, cs=2)),
    ({"ICNN_K2_CS": "4"}, ("dual", 2048, 13), five(8, cs=4)),
    ({"ICNN_K2_CS": "8"}, ("dual", 2048, 13), five(8, cs=8)),
    ({"ICNN_K2_CS": "1"}, ("dual", 2048, 13), five(8)),
    ({"ICNN_K2_CS": "3"}, ("dual", 2048, 13), five(8)),          # not a cluster size: ignored
    ({"ICNN_K2_WPS": "16"}, ("dual", 2048, 13), five(16)),
    ({"ICNN_K2_WPS": "16"}, ("lib", 2050, 13), five(16, vec=0)),
    ({"ICNN_K2_WPS": "4"}, ("dual", 2048, 13), five(4)),
    ({"ICNN_K2_WPS": "3"}, ("dual", 2048, 13), five(8)),          # not a warp count: ignored
    ({"ICNN_K2_WPS": "3"}, ("dual", 4096, 41), five(8)),          # but set: no 16-warp upgrade (default five(16))
    ({"ICNN_K2_WPS": "1"}, ("dual", 100, 35), five(1)),
]


@pytest.mark.parametrize("env,shape,want", ENV_TABLE)
def test_launch_variables(env, shape, want, monkeypatch):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    variant, n, KS = shape
    assert plan(n, KS, "pc" if variant == "lib" else "newton", variant) == want


def test_launch_variables_are_read_at_every_call(monkeypatch):
    assert plan(2048, 13) == two(8, 2)
    monkeypatch.setenv("ICNN_K2_PC", "legacy")
    assert plan(2048, 13) == five(8)
    monkeypatch.delenv("ICNN_K2_PC")
    assert plan(2048, 13) == two(8, 2)


def test_pinned_warp_count_that_does_not_fit_is_refused(monkeypatch):
    """ICNN_K2_WPS pins the warp count: no fall back to more warps when the samples of one CTA do not fit."""
    monkeypatch.setenv("ICNN_K2_WPS", "1")
    rc, msg = plan_full(100, 36, "newton", "dual")
    assert rc == -3 and "shared memory does not fit (n=100, KS=36)" in msg, msg


def test_cluster_that_does_not_fit_is_refused(monkeypatch):
    monkeypatch.setenv("ICNN_K2_CS", "8")
    rc, msg = plan_full(20, 11, "newton", "dual")                  # 8 slices of 4 columns leave one empty
    assert rc == -3 and "ICNN_K2_CS=8 does not fit (n=20, KS=11)" in msg, msg
