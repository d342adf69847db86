"""CPU-only checks of the boundary: the shared library loads, exports every symbol the header
declares, rejects bad arguments, and fails loudly (no CPU fallback) without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_header_symbol():
    from icnn_b200 import _capi
    hdr = open(os.path.join(ROOT, "include", "icnn_b200.h")).read()
    declared = set(re.findall(r"\b(icnn_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(_capi.SYMBOLS), declared ^ set(_capi.SYMBOLS)
    lib = C.CDLL(_capi.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name
    assert _capi.lib.icnn_abi_version() == _capi.ABI_VERSION


def test_struct_layouts_match_header_sizes():
    from icnn_b200 import _capi
    # 3 int32 (+pad) + 17 pointers ; cfg: 4 int32 + 2 double + 2 int32
    assert C.sizeof(_capi.BundleBufs) == 16 + 20 * 8   # 3 int32 (+pad) + 20 pointers (ABI v2: + f64, iter_stats, vec_ws)
    assert C.sizeof(_capi.BundleCfg) == 16 + 16 + 8
    assert C.sizeof(_capi.Gates) == 8 + 3 * 8 + 12 + 4
    assert C.sizeof(_capi.PicnnDesc) == 8 + 8 + 8 + 8 + 8


def test_bad_arguments_are_rejected_without_touching_the_gpu():
    from icnn_b200 import _capi
    rc = _capi.lib.icnn_picnn_create(None, None, None)
    assert rc == -1 and b"null" in _capi.lib.icnn_last_error()
    bufs = _capi.BundleBufs()
    assert _capi.lib.icnn_bundle_init(C.byref(bufs), 5, None) == -1
    cfg = _capi.BundleCfg()
    assert _capi.lib.icnn_bundle_step(C.byref(cfg), C.byref(bufs), 0, None) == -1
    assert _capi.lib.icnn_gd_backward(None, None, None, None, 1.0, 3, 0.01, 0.3, None, None, None, None) == -1
    assert _capi.lib.icnn_gd_backward_workspace_bytes(None, 4, 3) == 0
    with pytest.raises(_capi.IcnnError):
        _capi.check(-1)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    import icnn_b200
    from icnn_b200 import bundle_entropy, workloads
    p, x, y0 = workloads.make_inputs("C1", B=4)
    with pytest.raises(RuntimeError, match="CUDA"):
        icnn_b200.PICNN.from_params(p)
    with pytest.raises(RuntimeError, match="CUDA"):
        bundle_entropy.solveBatch(lambda y: (np.zeros(4), np.zeros_like(y)), y0)


def test_unknown_solver_raises_like_reference():
    # lib/bundle_entropy.py:232  raise RuntimeError("Solver unknown: "+solver)
    from icnn_b200 import bundle_entropy
    with pytest.raises(RuntimeError, match="Solver unknown"):
        bundle_entropy._make_cfg("lib", "simplex", 10, None, None, 0, 8, 9)
    assert bundle_entropy._make_cfg("lib", "boyd", 10, None, None, 0, 8, 9).solver == 1
    assert bundle_entropy._make_cfg("rl", "pc", 5, None, None, 0, 6, 6).line_search == 1
    assert bundle_entropy._make_cfg("dual", "pc", 10, None, None, 0, 8, 9).line_search == 0


def test_dropin_module_names_exist():
    import importlib.util
    for sub in ("dropin", "dropin_rl"):
        path = os.path.join(ROOT, "icnn_b200", sub, "bundle_entropy.py")
        assert os.path.exists(path)
        spec = importlib.util.spec_from_file_location("bundle_entropy_" + sub, path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        assert callable(mod.solveBatch)


def test_device_list_environment_variable(monkeypatch):
    """ICNN_DEVICES (SURVEY.md section 5: "env var for device list"): entry LOCAL_RANK of the list, else torch's current device."""
    import torch
    from icnn_b200.picnn import default_device
    monkeypatch.delenv("ICNN_DEVICES", raising=False)
    assert default_device() == torch.device("cuda")
    monkeypatch.setenv("ICNN_DEVICES", "4,5,6,7")
    monkeypatch.setenv("LOCAL_RANK", "2")
    assert default_device() == torch.device("cuda", 6)
    monkeypatch.delenv("LOCAL_RANK")
    assert default_device() == torch.device("cuda", 4)
    monkeypatch.setenv("ICNN_DEVICES", "3")
    monkeypatch.setenv("LOCAL_RANK", "5")
    assert default_device() == torch.device("cuda", 3)


def test_plain_c_consumer_compiles_and_links_without_a_gpu(tmp_path):
    """include/icnn_b200.h is valid C99 (no C++-isms, no torch types) and tests/c_abi/smoke.c -- the plain-C consumer
    the GPU suite runs -- compiles and links against libicnn_b200.so here (it is executed by the GPU test only)."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr_only = tmp_path / "hdr.c"
    hdr_only.write_text('#include "icnn_b200.h"\nint main(void) { return ICNN_ABI_VERSION > 0 ? 0 : 1; }\n')
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(root, "include"),
                           "-c", str(hdr_only), "-o", str(tmp_path / "hdr.o")])
    lib = os.path.join(root, "icnn_b200")
    subprocess.check_call(["gcc", "-O1", "-std=c99", "-I", os.path.join(root, "include"), "-I", "/usr/local/cuda/include",
                           os.path.join(root, "tests", "c_abi", "smoke.c"), "-o", str(tmp_path / "smoke"),
                           "-L", lib, "-l:libicnn_b200.so", "-L", "/usr/local/cuda/lib64", "-lcudart", "-lm",
                           "-Wl,-rpath," + lib + ":/usr/local/cuda/lib64"])
    assert (tmp_path / "smoke").exists()


def test_ragged_result_views_follow_perm_and_count():
    """Host logic of the 6-tuple: A / b / lam / xs are lazy list-of-lists views over the dense slot buffers, in the
    sample's LOGICAL order (perm maps logical index -> physical slot; pruning permutes perm only).  Exercised on CPU
    tensors -- BundleState only stores pointers, no kernel runs."""
    import torch
    from icnn_b200.bundle_entropy import BundleState, _Rows
    B, n, KS = 3, 4, 5
    st = BundleState(B, n, KS, torch.device("cpu"), keep_xs=True, nIter=4)
    st.G.copy_(torch.arange(B * KS * n, dtype=torch.float32).reshape(B, KS, n))
    st.ys.copy_(-torch.arange(B * KS * n, dtype=torch.float64).reshape(B, KS, n))
    st.h.copy_(torch.arange(B * KS, dtype=torch.float64).reshape(B, KS) * 0.5)
    st.lam.copy_(torch.arange(B * KS, dtype=torch.float64).reshape(B, KS) * 0.25)
    st.perm.copy_(torch.tensor([[3, 0, 1, 2, 4], [4, 3, 2, 1, 0], [0, 1, 2, 3, 4]], dtype=torch.int32))
    st.count.copy_(torch.tensor([2, 0, 4], dtype=torch.int32))
    A, b, lam, xs = (_Rows(st, k) for k in ("A", "b", "lam", "xs"))
    assert len(A) == B and [len(a) for a in A] == [2, 0, 4]                      # nActive = len(G[j])
    np.testing.assert_array_equal(np.array(A[0]), st.G[0, [3, 0]].numpy())        # logical order = perm order
    np.testing.assert_array_equal(np.array(xs[0]), st.ys[0, [3, 0]].numpy())
    assert b[0] == [0.5 * 3, 0.0] and A[1] == [] and b[1] == [] and lam[1] is None and xs[1] == []
    np.testing.assert_array_equal(lam[2], st.lam[2, :4].numpy())
    assert isinstance(A[2][1], np.ndarray) and A[2][1].shape == (n,) and A[-1] is A[2]
    assert [len(a) for a in A[0:2]] == [2, 0]
    import pytest
    with pytest.raises(IndexError):
        A[3]
    st2 = BundleState(B, n, KS, torch.device("cpu"), keep_xs=False, nIter=4)
    st2.count.fill_(1)
    st2.perm.copy_(st.perm)
    with pytest.raises(RuntimeError):
        _Rows(st2, "xs")[0]
    assert st.compatible(B, n, KS, torch.device("cpu"), True, 3, False, False) and not st.compatible(B, n, KS + 1, torch.device("cpu"), True, 3, False, False)
    assert not st.compatible(B, n, KS, torch.device("cpu"), True, 9, False, False)      # more iterations than nactive holds


def test_solver_configuration_mirrors_the_three_reference_copies():
    """_make_cfg: defaults of lib / dual / RL copies (nIter 10/10/5, line search on/off/on, prune thresholds 1e-8/0/0),
    'boyd' accepted, an unknown solver raises the reference's message (lib/bundle_entropy.py:232)."""
    import pytest
    from icnn_b200 import _capi
    from icnn_b200.bundle_entropy import VARIANT_DEFAULTS, _make_cfg
    assert [VARIANT_DEFAULTS[v]["nIter"] for v in ("lib", "dual", "rl")] == [10, 10, 5]
    c = _make_cfg("lib", "pc", 10, None, None, 0, 159, 11)
    assert (c.variant, c.solver, c.line_search, c.nIter) == (_capi.VARIANT["lib"], _capi.SOLVER_PC, 1, 10) and c.prune_thr == 1e-8
    assert abs(c.rank_tol - 16.0 * 159 * np.finfo(np.float64).eps) < 1e-30
    assert _make_cfg("lib", "boyd", 10, None, None, 0, 8, 9).solver == _capi.SOLVER_NEWTON
    d = _make_cfg("dual", "newton", 10, None, None, 0, 8, 9)
    assert (d.variant, d.solver, d.line_search, d.prune_thr) == (_capi.VARIANT["dual"], _capi.SOLVER_NEWTON, 0, 0.0)
    r = _make_cfg("rl", "newton", 5, None, 1e-3, 7, 6, 6)
    assert (r.variant, r.line_search, r.max_inner, r.rank_tol) == (_capi.VARIANT["rl"], 1, 7, 1e-3)
    with pytest.raises(RuntimeError, match="Solver unknown: foo"):
        _make_cfg("lib", "foo", 10, None, None, 0, 8, 9)
