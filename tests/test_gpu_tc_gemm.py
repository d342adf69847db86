"""The wgmma tensor-core GEMM (tc_gemm_kernel, icnn_b200/csrc/picnn_tc.cu) tested on its own, under every tile
variant and split-K factor, against float64.

Which variant a launch takes normally follows the device's SM count and the grid, so on its own the suite would
exercise an accident of the shapes (<128,3> not at all, split-K 8 only at a few batch sizes).  Every test here
pins the variant with icnn_tc_set_tuning and asserts with icnn_tc_last_launch that the pinned variant ran; an
autouse fixture restores the automatic choice after each test and checks that it took.

  A-F  C = A B^T through icnn_tc_gemm_selftest (mode 2) at ragged shapes: exact integer arithmetic, the TF32 lo
       path, signed data, the chunked-accumulation bias (with a negative control), pad columns / guard bands /
       non-finite propagation, determinism and row invariance.
  G-J  the fused epilogues through the library: K1 forward / backward (modes 0, 1), the x-path gates (mode 3), the
       GD training backward (GDB instantiation) and the fused bundle loop (mode 1 with the bundle-slot scatter).
"""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from oracle import bundle_np, gd_grad_np, picnn_np, synth

pytestmark = pytest.mark.gpu
np.seterr(all="ignore")

# id -> (cfg, splitk) for icnn_tc_set_tuning, and the {BN, NST, splitk} the launch must report (None = automatic)
VARIANTS = {
    "auto": ((-1, -1), None),
    "128x3": ((0, -1), (128, 3, 1)),
    "64x4-S1": ((1, 1), (64, 4, 1)),
    "64x4-S2": ((1, 2), (64, 4, 2)),
    "64x4-S4": ((1, 4), (64, 4, 4)),
    "64x4-S8": ((1, 8), (64, 4, 8)),
    "64x2": ((2, -1), (64, 2, 1)),
}
PINNED = [v for v in VARIANTS if v != "auto"]

# (M, N, K): every M in {1, 17, 64, 127, 128, 129, 300}, N in {1, 7, 33, 64, 65, 128, 129, 200} and K in
# {1, 3, 4, 5, 16, 17, 31, 32, 33, 100, 1028, 5120} appears; K <= 224 leaves some ranks of an 8-way split-K cluster
# without a k-block (K = 32: one k-block for eight ranks)
SHAPES = [(1, 1, 1), (17, 7, 3), (64, 33, 4), (127, 65, 5), (128, 64, 16), (129, 129, 17), (300, 200, 31),
          (128, 128, 32), (17, 200, 33), (300, 1, 100), (1, 128, 1028), (64, 129, 5120), (129, 33, 1028),
          (127, 200, 100), (300, 65, 5120), (1, 7, 32), (17, 64, 17), (64, 1, 31), (128, 129, 1028), (129, 7, 5120),
          (300, 128, 33), (127, 1, 16), (64, 200, 3), (1, 65, 100), (128, 33, 5), (300, 129, 4)]
SHAPE_IDS = ["M%dxN%dxK%d" % s for s in SHAPES]

GUARD = 64          # floats of sentinel before and after C
SENTINEL = 0x5EED5EED
ENV_KNOBS = ("ICNN_TC_CFG", "ICNN_TC_SPLITK", "ICNN_TC_CH")
REPORT = {}         # measured figures, printed at the end of the module (pytest -s)


def _lib():
    from icnn_b200 import _capi
    return _capi


def ld4(k):
    return (k + 3) & ~3


def pin(vid, ch=-1):
    cfg, sk = VARIANTS[vid][0]
    assert _lib().lib.icnn_tc_set_tuning(cfg, sk, ch) == 0, _lib().lib.icnn_last_error()


def last_launch():
    out = (C.c_int32 * 5)()
    assert _lib().lib.icnn_tc_last_launch(out) == 0
    return tuple(out)


def check_launch(vid, mode, ch=None, splitk=None):
    """The calling thread's last tensor-core GEMM ran the pinned variant (``splitk`` overrides the pinned factor where
    the mode cannot split)."""
    bn, nst, s, c, md = last_launch()
    assert md == mode, (vid, last_launch())
    want = VARIANTS[vid][1]
    if want is None:
        assert (bn, nst) in ((128, 3), (64, 4), (64, 2)) and s in (1, 2, 4, 8) and (s == 1 or (bn, nst) == (64, 4))
    else:
        assert (bn, nst, s) == (want[0], want[1], want[2] if splitk is None else splitk), (vid, last_launch())
    if ch is not None:
        assert c == ch, (vid, last_launch())


def record(key, vid, value, agg=max):
    d = REPORT.setdefault(key, {})
    d[vid] = agg(d[vid], value) if vid in d else value


@pytest.fixture(autouse=True)
def automatic_tuning():
    """Every test leaves the GEMM on its automatic choice: pytest runs all files in one process, and a leaked pin
    would silently change what the rest of the suite exercises.  The reset is checked on two probes whose automatic
    variant is known on any device with >= 16 SMs: one tile with 32 k-blocks splits 8 ways, one k-block does not."""
    yield
    capi = _lib()
    assert capi.lib.icnn_tc_set_tuning(-1, -1, -1) == 0
    if any(k in os.environ for k in ENV_KNOBS):
        return
    for (M, N, K), want in (((128, 64, 1024), (64, 4, 8, 1, 2)), ((1, 1, 1), (64, 4, 1, 1, 2))):
        A = torch.ones(M, K, device="cuda")
        gemm(A, torch.ones(N, K, device="cuda"))
        assert last_launch() == want, (M, N, K, last_launch())


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\ntc_gemm measured on %s (%d SMs):" % (torch.cuda.get_device_name(),
                                                     torch.cuda.get_device_properties(0).multi_processor_count))
        for key, d in REPORT.items():
            print("  %-44s %s" % (key, "  ".join("%s %+.3e" % (v, d[v]) for v in VARIANTS if v in d)))


def gemm(A, B, scratch_fill=float("nan")):
    """C = A B^T (float32 [M, K], [N, K]) through icnn_tc_gemm_selftest.  The scratch that holds the split operands is
    filled with ``scratch_fill`` first (the ld4 pad columns keep it: the split kernel writes only columns < K), and C is
    pre-filled with NaN inside an allocation whose guard bands before and after M*N hold a sentinel; the guards are
    checked here, the absence of NaN by the callers."""
    capi = _lib()
    A, B = A.contiguous(), B.contiguous()
    M, K = A.shape
    N = B.shape[0]
    scratch = torch.full(((2 * M + 2 * N) * ld4(K),), scratch_fill, device=A.device)
    buf = torch.full((GUARD + M * N + GUARD,), float("nan"), device=A.device)
    iv = buf.view(torch.int32)
    iv[:GUARD] = SENTINEL
    iv[GUARD + M * N:] = SENTINEL
    Cm = buf[GUARD:GUARD + M * N]
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    capi.check(capi.lib.icnn_tc_gemm_selftest(A.data_ptr(), B.data_ptr(), Cm.data_ptr(), M, N, K, scratch.data_ptr(),
                                              stream))
    torch.cuda.synchronize()
    assert bool((iv[:GUARD] == SENTINEL).all()) and bool((iv[GUARD + M * N:] == SENTINEL).all()), \
        "tc_gemm wrote outside C[M, N]"
    return Cm.view(M, N).clone()


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def int_operands(M, N, K, seed):
    g = gen(seed)
    A = torch.randint(-32, 33, (M, K), generator=g, device="cuda").float()
    B = torch.randint(-32, 33, (N, K), generator=g, device="cuda").float()
    return A, B


def ref64(A, B):
    return A.double() @ B.double().T


# ---------------------------------------------------------------------------------------------------------------
# A-F: the GEMM on its own
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("vid", list(VARIANTS))
def test_integer_products_are_exact(vid, shape):
    """A. Integer operands in [-32, 32] are exact in TF32 (the lo parts are 0) and every partial sum is an integer
    below 2^24, so any correct order of summation gives A B^T exactly.  Catches any indexing, swizzle, k-step
    descriptor, tail, epilogue or DSMEM-reduction error however small.  The scratch is NaN-filled, so a read of the
    ld4 pad columns would show up as NaN, and C is NaN-prefilled, so an element left unwritten would too."""
    M, N, K = shape
    pin(vid)
    A, B = int_operands(M, N, K, seed=M * 7919 + N * 104729 + K)
    Cm = gemm(A, B)
    check_launch(vid, 2)
    ref = ref64(A, B)
    assert bool(torch.isfinite(Cm).all()), "non-finite entries"
    bad = Cm.double() != ref
    assert not bool(bad.any()), (int(bad.sum()), torch.nonzero(bad)[:5].tolist())


def lo_path_operand(rows, K, g):
    """fp32(t (1 + 2^-13)) with t a positive TF32 value (10-bit mantissa) in [0.5, 4): 2^-13 is below TF32's smallest
    relative half-ulp (2^-12), so hi = t and lo ~ +2^-13 t, one sign everywhere."""
    j = torch.randint(0, 1024, (rows, K), generator=g, device="cuda").double()
    e = torch.randint(-1, 2, (rows, K), generator=g, device="cuda").double()
    t = (1.0 + j / 1024.0) * torch.pow(2.0, e)
    return (t * (1.0 + 2.0 ** -13)).float()


@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("vid", list(VARIANTS))
def test_lo_terms_are_summed(vid, shape):
    """B. Every operand carries a large TF32 remainder of one sign, so a missing A_hi B_lo or A_lo B_hi term moves
    every entry by ~2^-13 relative (with random-sign remainders the same defect would shrink to ~2^-13 / sqrt(K)).
    Bound: 2^-19, 64x below that defect."""
    M, N, K = shape
    pin(vid)
    g = gen(K * 31 + M + 5 * N)
    A, B = lo_path_operand(M, K, g), lo_path_operand(N, K, g)
    Cm = gemm(A, B)
    check_launch(vid, 2)
    ref = ref64(A, B)
    rel = ((Cm.double() - ref).abs() / ref).max().item()
    record("B lo path: max rel err", vid, rel)
    assert rel <= 2.0 ** -19, rel


@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("vid", list(VARIANTS))
def test_signed_data_error_bound(vid, shape):
    """C. randn operands: |C - C64| <= (2^-19 + ceil(K/16) 2^-24) (|A| |B|^T) elementwise.  The second term covers the
    round-to-nearest adds of the K = 16 chunks into the running sum (and of the split-K partials).  The first covers
    the 3xTF32 split (~2^-21) plus one truncation per wgmma instruction; that part is an assumption about the tensor
    core's accumulator, not a documented or independently measured property."""
    M, N, K = shape
    pin(vid)
    g = gen(K * 131 + 17 * M + N)
    A = torch.randn(M, K, generator=g, device="cuda")
    B = torch.randn(N, K, generator=g, device="cuda")
    Cm = gemm(A, B)
    check_launch(vid, 2)
    scale = A.double().abs() @ B.double().abs().T
    ratio = ((Cm.double() - ref64(A, B)).abs() / scale).max().item()
    record("C signed: max |C-C64| / (|A||B|^T)", vid, ratio)
    assert ratio <= 2.0 ** -19 + math.ceil(K / 16) * 2.0 ** -24, ratio


BIAS_T = 1e-6


@pytest.mark.parametrize("vid", list(VARIANTS))
def test_chunked_accumulation_removes_the_truncation_bias(vid):
    """D. Positive operands at K = 5120: the tensor core does not round its FP32 accumulator to nearest, so one long
    accumulation drifts by a signed relative bias.  With the default chunk (K = 16 per round-to-nearest add) the signed
    mean relative error over all entries must stay within T; pinned to ch = 64 (K = 1024 per chunk, no chunking to
    speak of) the same measurement must show at least 4 T -- the test can see the defect it guards against."""
    M, N, K = 256, 256, 5120
    g = gen(5120)
    A = torch.rand(M, K, generator=g, device="cuda")
    B = torch.rand(N, K, generator=g, device="cuda")
    ref = ref64(A, B)
    means = {}
    for ch in (1, 64):
        pin(vid, ch)
        Cm = gemm(A, B)
        check_launch(vid, 2, ch=ch)
        means[ch] = ((Cm.double() - ref) / ref).mean().item()
        record("D bias: signed mean rel err, ch=%d" % ch, vid, means[ch])
    assert abs(means[1]) <= BIAS_T, means
    assert abs(means[64]) >= 4 * BIAS_T, means


NAN_PATTERNS = {"qnan": 0x7FC00000, "nan-all-ones": 0x7FFFFFFF, "neg-nan-all-ones": -1}


@pytest.mark.parametrize("nan", list(NAN_PATTERNS))
@pytest.mark.parametrize("vid", list(VARIANTS))
def test_non_finite_stays_in_its_row_and_column(vid, nan):
    """E. One row of A is NaN and one row of B is +Inf: exactly that row and that column of C are non-finite, every
    other entry stays exact (integer data), under every variant including the 8-way split-K, whose partial tiles
    meet in distributed shared memory.  0x7FFFFFFF is the NaN the GPU's own arithmetic produces: the TF32 rounding of
    the split must not carry it into +-0 or Inf."""
    M, N, K = 129, 65, 1028
    pin(vid)
    A, B = int_operands(M, N, K, seed=3)
    ref = ref64(A, B)
    ri, ci = 77, 40
    A.view(torch.int32)[ri, :] = NAN_PATTERNS[nan]
    B[ci, :] = float("inf")
    Cm = gemm(A, B)
    check_launch(vid, 2)
    nonfin = ~torch.isfinite(Cm)
    want = torch.zeros_like(nonfin)
    want[ri, :] = True
    want[:, ci] = True
    assert torch.equal(nonfin, want), (int(nonfin.sum()), int(want.sum()))
    keep = ~want
    assert torch.equal(Cm.double()[keep], ref[keep])


@pytest.mark.parametrize("vid", list(VARIANTS))
def test_pad_columns_and_guard_band(vid):
    """E. K % 4 != 0 shapes with the scratch NaN-filled and C NaN-prefilled between sentinel guard bands (``gemm``
    checks the guards): the result is finite and exact, so the ld4 pad columns were never read and every element of C
    was written, and nothing outside [M, N] was."""
    pin(vid)
    for M, N, K in ((300, 200, 31), (129, 129, 17), (17, 7, 3), (128, 33, 5), (64, 129, 5117)):
        A, B = int_operands(M, N, K, seed=K)
        Cm = gemm(A, B, scratch_fill=float("nan"))
        check_launch(vid, 2)
        assert bool(torch.isfinite(Cm).all()) and torch.equal(Cm.double(), ref64(A, B)), (M, N, K)


@pytest.mark.parametrize("vid", PINNED)
def test_deterministic_and_row_invariant(vid):
    """F. Under a pinned variant two calls give identical bits, and rows [37:70) computed as their own problem equal
    the same rows of the full problem bit for bit: per-row arithmetic depends only on K, the split factor and the
    chunk length once the variant is pinned."""
    pin(vid)
    g = gen(99)
    M, N, K = 300, 129, 1028
    A = torch.randn(M, K, generator=g, device="cuda")
    B = torch.randn(N, K, generator=g, device="cuda")
    c1 = gemm(A, B)
    c2 = gemm(A, B)
    check_launch(vid, 2)
    assert torch.equal(c1.view(torch.int32), c2.view(torch.int32))
    sub = gemm(A[37:70], B)
    check_launch(vid, 2)
    assert torch.equal(sub.view(torch.int32), c1[37:70].view(torch.int32))


@pytest.mark.parametrize("vid", ["64x4-S8"])
def test_rejected_override_leaves_the_pin_in_place(vid):
    pin(vid)
    assert _lib().lib.icnn_tc_set_tuning(3, -1, -1) == -1
    assert _lib().lib.icnn_tc_set_tuning(-1, 3, -1) == -1
    gemm(*int_operands(128, 64, 1024, seed=1))
    check_launch(vid, 2, ch=1 if "ICNN_TC_CH" not in os.environ else None)


# ---------------------------------------------------------------------------------------------------------------
# G-J: the fused epilogues through the library
# ---------------------------------------------------------------------------------------------------------------
_CACHE = {}


def _case(key):
    """(params, x, y, affine, net) of a K1 case, built once per module."""
    if key not in _CACHE:
        import icnn_b200
        from icnn_b200.workloads import synth_params
        if isinstance(key[0], str):
            name, B = key
            cfg = synth.CONFIGS[name]
            p, x, y0 = synth.make_inputs(name, B=B)
            affine = cfg["affine"]
        else:
            (m, n, hidden), B = key
            p = synth_params(31, m, n, list(hidden))
            x = np.random.RandomState(32).randn(B, m).astype(np.float32).astype(np.float64)
            affine = False
        y = np.random.RandomState(11).uniform(0.02, 0.98, size=(B, p.n)).astype(np.float32).astype(np.float64)
        _CACHE[key] = (p, x, y, affine, icnn_b200.PICNN.from_params(p))
    return _CACHE[key]


def _oracle(key, fn):
    k = ("oracle",) + key
    if k not in _CACHE:
        _CACHE[k] = fn()
    return _CACHE[k]


K1_CASES = [(("C3", 77), 1e-5), (((13, 37, (50, 21, 33)), 200), 1e-5), (("T", 130), 1e-5), (("C5", 70), 5e-5)]


@pytest.mark.parametrize("key,tol", K1_CASES, ids=["C3-77", "13x37x50.21.33-200", "T-130", "C5-70"])
@pytest.mark.parametrize("vid", list(VARIANTS))
def test_k1_forward_backward_epilogues(vid, key, tol):
    """G. Modes 0 and 1 (K1 f and df/dy) under each variant against the float64 oracle, with the tolerances of
    test_fg_matches_oracle.  The workspace is filled with NaN bytes after bind(): the ld4 pads of the K-concatenated
    operands and of the delta buffers are never written, so a read of one would poison f or g."""
    p, x, y, affine, net = _case(key)
    pin(vid)
    fg = net.bind(x, affine=affine)
    fg.ws.fill_(0xFF)
    f, g = fg(y)
    check_launch(vid, 1)
    fo, go = _oracle(key, lambda: picnn_np.make_fg(p, x, affine=affine)(y))
    assert np.isfinite(f).all() and np.isfinite(g).all()
    assert np.abs(f - fo).max() <= tol * max(1.0, np.abs(fo).max())
    assert np.abs(g - go).max() <= tol * max(1.0, np.abs(go).max())


@pytest.mark.parametrize("vid", list(VARIANTS))
def test_k1_nan_iterate_stays_in_its_row(vid):
    """A NaN row of the iterate reaches the GEMMs as the NaN the GPU's arithmetic produces (0x7FFFFFFF, from the
    s y + t gating): f of that row must come out non-finite (the bundle step flags such samples; g may stay finite,
    act'(NaN) takes the alpha branch), and every other row of f and g must be bit-identical to the clean batch."""
    p, x, y, affine, net = _case(("C3", 77))
    pin(vid)
    fg = net.bind(x, affine=affine)
    f0, g0 = fg(y)
    yn = y.copy()
    yn[5, :] = np.nan
    f, g = fg(yn)
    check_launch(vid, 1)
    assert not np.isfinite(f[5])
    rest = np.arange(len(y)) != 5
    np.testing.assert_array_equal(f[rest], f0[rest])
    np.testing.assert_array_equal(g[rest], g0[rest])


GATE_VARIANTS = ["128x3", "64x4-S8", "64x2"]


def _check_gates(p, x, cz, cy, d):
    ocz, ocy, od = picnn_np.gates(p, x)
    for i in range(p.L + 1):
        for got, want in ((cz[i], ocz[i]), (cy[i], ocy[i]), (d[i], od[i])):
            if want is None:
                assert got is None
                continue
            gv = got.cpu().numpy().astype(np.float64)
            assert gv.shape == want.shape
            assert np.abs(gv - want).max() <= 1e-5 * max(1.0, np.abs(want).max()), i


@pytest.mark.parametrize("key", [((13, 37, (50, 21, 33)), 200), ("T", 300)], ids=["13x37x50.21.33-200", "T-300"])
@pytest.mark.parametrize("vid", GATE_VARIANTS)
def test_gate_epilogue(vid, key):
    """H. Mode 3 (x-path gates: bias, per-range ReLU, scatter; range boundaries at 50 / 87 / 137 in the first case)
    against the float64 oracle.  A forced split-K factor must not reach mode 3, which has no split-K epilogue."""
    p, x, y, affine, net = _case(key)
    assert net._xpath
    pin(vid)
    cz, cy, d = net.gates(x)
    check_launch(vid, 3, splitk=1)
    _check_gates(p, x, cz, cy, d)


@pytest.mark.parametrize("vid", ["64x2"])
def test_gate_epilogue_with_nan_workspace(vid):
    """H. The same through icnn_picnn_gates directly, with the workspace (split x / u operands, ld4 pitch) NaN-filled."""
    capi = _lib()
    p, x, y, affine, net = _case(((13, 37, (50, 21, 33)), 200))
    pin(vid)
    B, L = x.shape[0], p.L
    e = lambda w: torch.empty(B, w, dtype=torch.float32, device="cuda")  # noqa: E731
    cz = [None] + [e(p.hidden[i - 1]) for i in range(1, L + 1)]
    cy = [e(p.n) for _ in range(L + 1)]
    d = [e(p.hidden[i]) if i < L else e(1) for i in range(L + 1)]
    ws = torch.full((capi.lib.icnn_picnn_gates_workspace_bytes(net._h, B),), 0xFF, dtype=torch.uint8, device="cuda")
    xd = torch.as_tensor(x, dtype=torch.float32, device="cuda")
    pz, py, pd = capi.ptr_array(cz), capi.ptr_array(cy), capi.ptr_array(d)
    capi.check(capi.lib.icnn_picnn_gates(net._h, xd.data_ptr(), B, C.cast(pz, capi._fpp), C.cast(py, capi._fpp),
                                         C.cast(pd, capi._fpp), ws.data_ptr(),
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    check_launch(vid, 3)
    _check_gates(p, x, cz, cy, d)


RTOL = 2e-4


def _relerr(a, b):
    return float(np.abs(np.asarray(a, dtype=np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def _gdb_case(dims, B):
    """test_gpu_gd_grad._dims_case: W^y scaled by 3 so that the GD iterates move; the oracle kink floor is cached."""
    key = ("gdb", dims, B)
    if key not in _CACHE:
        import icnn_b200
        from icnn_b200.workloads import synth_params
        m, n, hidden = dims
        seed = 21
        p = synth_params(seed, m, n, list(hidden))
        for i in range(len(p.Wy)):
            p.Wy[i] = (p.Wy[i].astype(np.float32) * np.float32(3.0)).astype(np.float64)
        rs = np.random.RandomState(seed + 1)
        x = rs.randn(B, m).astype(np.float32).astype(np.float64)
        y0 = np.full((B, n), 0.5)
        tY = (rs.uniform(size=(B, n)) < 0.2).astype(np.float64)
        _CACHE[key] = dict(p=p, x=x, y0=y0, tY=tY, net=icnn_b200.PICNN.from_params(p), oracle={}, floor=None)
    return _CACHE[key]


def _gdb_oracle(c, keep, nIter, lr, mom):
    k = (tuple(keep), nIter, lr, mom)
    if k not in c["oracle"]:
        p, xs, ys, ts = c["p"], c["x"][keep], c["y0"][keep], c["tY"][keep]
        scale = 2.0 / c["tY"].size
        yo, go = gd_grad_np.gd_backward(p, picnn_np.gates(p, xs), ys, nIter, lr, mom, lambda y: scale * (y - ts))
        c["oracle"][k] = (yo, go, gd_grad_np.xpath_backward(p, xs, go["dcy"], go["dcz"]))
    return c["oracle"][k]


def _gdb_floor(c, nIter, lr, mom):
    """Rows of the float64 oracle that a float32-sized (1e-7 relative) perturbation of W^y moves past the tolerances
    (max over three perturbations): kink flips are a property of the iteration, not of the device arithmetic."""
    import copy
    if c["floor"] is None:
        p, x, y0, tY = c["p"], c["x"], c["y0"], c["tY"]
        scale = 2.0 / tY.size
        y1, g1 = gd_grad_np.gd_backward(p, picnn_np.gates(p, x), y0, nIter, lr, mom, lambda y: scale * (y - tY))
        rs = np.random.RandomState(99)
        floor = 0
        for rep in range(3):
            pp = copy.deepcopy(p)
            for i in range(len(pp.Wy)):
                pp.Wy[i] = pp.Wy[i] * (1.0 + 1e-7 * rs.choice([-1.0, 1.0], size=pp.Wy[i].shape))
            y2, g2 = gd_grad_np.gd_backward(pp, picnn_np.gates(pp, x), y0, nIter, lr, mom, lambda y: scale * (y - tY))
            moved = np.abs(y1 - y2).max(axis=1) >= 1e-4
            for l in range(p.L + 1):
                for k in ("dcy", "dcz"):
                    if g1[k][l] is not None:
                        moved |= (np.abs(g1[k][l] - g2[k][l]).max(axis=1) / max(np.abs(g1[k][l]).max(), 1e-30)) >= RTOL
            floor = max(floor, int(moved.sum()))
        c["floor"] = floor
    return c["floor"]


def gd_grad_matches_oracle(c, nIter, lr, mom, check):
    """The kink-row handling of test_gpu_gd_grad.test_matches_oracle: rows whose y_N or gate adjoints land on the other
    side of a ReLU kink are dropped (<= 2 % of the batch, and no more than the float64 oracle itself loses under a
    float32-sized perturbation, plus one), both sides are rerun on the rest, and every gradient array must then agree
    to RTOL of its largest entry.  ``check()`` runs after every device call."""
    import icnn_b200
    p, x, y0, tY, net = c["p"], c["x"], c["y0"], c["tY"], c["net"]
    B = x.shape[0]
    keep = np.arange(B)
    dropped = 0
    for attempt in range(4):
        xs, ys, ts = x[keep], y0[keep], tY[keep]
        yo, go, xo = _gdb_oracle(c, keep, nIter, lr, mom)
        yN, gr = icnn_b200.gd_grad.gd_grad(net.bind(xs), ys, ts, nIter=nIter, lr=lr, momentum=mom, x=xs,
                                           loss_scale=2.0 / tY.size)
        check()
        bad = np.abs(yN - yo).max(axis=1) >= 1e-4
        for l in range(p.L + 1):
            for k in ("dcy", "dcz"):
                if go[k][l] is not None:
                    dd = np.abs(gr[k][l].astype(np.float64) - go[k][l]).max(axis=1) / max(np.abs(go[k][l]).max(), 1e-30)
                    bad |= dd >= RTOL
        if not bad.any():
            break
        dropped += int(bad.sum())
        keep = keep[~bad]
    assert not bad.any() and dropped <= 0.02 * B, (dropped, B)
    if dropped:
        floor = _gdb_floor(c, nIter, lr, mom)
        assert dropped <= floor + 1, (dropped, floor)
    assert np.median(np.abs(yN - yo).max(axis=1)) < 2e-6
    errs = {}
    for l in range(p.L + 1):
        errs["Wy%d" % l] = _relerr(gr["Wy"][l], go["dWy"][l])
        errs["Wyu%d" % l] = _relerr(gr["Wyu"][l], xo["dWyu"][l])
        if l > 0:
            errs["Wz%d" % l] = _relerr(gr["Wz"][l], go["dWz"][l])
            errs["Wzu%d" % l] = _relerr(gr["Wzu"][l], xo["dWzu"][l])
    for l in range(p.L):
        errs["Wu%d" % l] = _relerr(gr["Wu"][l], xo["dWu"][l])
    assert max(errs.values()) < RTOL, errs


GDB_CASES = [((12, 37, (50, 21, 33)), 77, 10, 0.02, 0.5), ((64, 512, (1024, 1024)), 200, 6, 0.01, 0.9)]


@pytest.mark.parametrize("gdb_mode", ["stored", "twopass"])
@pytest.mark.parametrize("case", GDB_CASES, ids=["12x37x50.21.33-77", "64x512x1024.1024-200"])
@pytest.mark.parametrize("vid", ["64x4-S1", "64x4-S2", "64x4-S4", "64x4-S8", "64x2"])
def test_gd_training_backward_epilogues(vid, case, gdb_mode, monkeypatch):
    """I. The GDB instantiation (tangent forward, backward with the delta / dCz / Dacc accumulations, the batched
    stored-pattern tangent GEMM) under each 64-wide variant, in the default stored-pattern mode and in ICNN_GDB=twopass,
    against the float64 restatement of TensorFlow's double backprop."""
    dims, B, nIter, lr, mom = case
    if gdb_mode == "twopass":
        monkeypatch.setenv("ICNN_GDB", "twopass")
    else:
        monkeypatch.delenv("ICNN_GDB", raising=False)
    c = _gdb_case(dims, B)
    pin(vid)
    gd_grad_matches_oracle(c, nIter, lr, mom, lambda: check_launch(vid, last_launch()[4]))
    assert last_launch()[4] in (0, 1)


FUSED = [("T", 160, 10), ("C2", 70, 8)]


@pytest.mark.parametrize("case", FUSED, ids=["T-160-10", "C2-70-8"])
@pytest.mark.parametrize("vid", list(VARIANTS))
def test_fused_bundle_loop(vid, case):
    """J. Mode 1 with the bundle-slot scatter through perm: the eager fused loop (a captured graph would bake in the
    launch configuration) against the float64 oracle, with the criterion of test_fused_vs_oracle: median y* error
    within max(1e-5, 4 x the oracle's own float32 noise floor), kink-flipped rows no more than the floor's plus
    max(2 %, 2.5 rows), and an objective gap as good as the oracle's."""
    from icnn_b200 import bundle_entropy as be
    name, B, nIter = case
    cfg = synth.CONFIGS[name]
    p, x, y0 = synth.make_inputs(name, B=B)
    variant = cfg["variant"]

    def oracle():
        o = bundle_np.solve_batch(picnn_np.make_fg(p, x, affine=cfg["affine"]), y0.copy(), nIter=nIter, variant=variant)
        o32 = bundle_np.solve_batch(picnn_np.make_fg(p, x, affine=cfg["affine"], dtype=np.float32, out_dtype=np.float64),
                                    y0.copy(), nIter=nIter, variant=variant)
        return o[0], o32[0]
    yo, yo32 = _oracle(("fused",) + case, oracle)
    net = _case((name, B))[4]
    pin(vid)
    r = be.solveBatch(net.bind(x, affine=cfg["affine"]), y0.copy(), nIter=nIter, variant=variant, graph=False)
    check_launch(vid, 1)
    d = np.abs(r[0] - yo).max(axis=1)
    floor = np.abs(yo32 - yo).max(axis=1)
    record("J fused %s-%d: median |y*-y*64|" % (name, B), vid, float(np.median(d)))
    assert np.median(d) < max(1e-5, 4 * np.median(floor)), (np.median(d), np.median(floor))
    assert np.mean(d > 1e-4) <= np.mean(floor > 1e-4) + max(0.02, 2.5 / B)
    fg64 = picnn_np.make_fg(p, x, affine=cfg["affine"])
    obj = lambda y: fg64(y)[0] + np.sum(y * np.log(y) + (1 - y) * np.log(1 - y), axis=1)  # noqa: E731
    gap = (obj(r[0]) - obj(yo)) / np.maximum(1.0, np.abs(obj(yo)))
    assert np.median(np.abs(gap)) < 1e-5 and gap.max() < 1e-3, gap
