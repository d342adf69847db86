"""CPU checks of the conv PICNN boundary: parse_variables infers the reference's completion architecture from its
TensorFlow variable dict and names every bad variable; the torch helper evaluated from that dict reproduces the
reference graph's goldens; the descriptor struct matches the C header."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _olivetti_vars():
    from oracle.gen_golden_tfshim import conv_case, conv_variables
    net, _x, _y = conv_case("conv_olivetti")
    return conv_variables(net)


def test_parse_variables_infers_the_reference_architecture():
    from icnn_b200.conv_picnn import parse_variables
    spec = parse_variables(_olivetti_vars(), 64, 32)
    assert spec.convs == [(32, 8, 4), (64, 4, 2), (64, 3, 1)] and spec.fcs == [512, 1]
    assert all(a.dtype == np.float32 for a in spec.vars.values())
    # TF names with the ':0' suffix are accepted too
    v = {k + ":0": a for k, a in _olivetti_vars().items()}
    assert parse_variables(v, 64, 32).convs == spec.convs


@pytest.mark.parametrize("defect,name", [
    ("missing", "z1_yu_u/b"), ("missing", "u2/BatchNormalization/moving_variance"), ("extra", "z3_yu/W"),
    ("shape", "z2_zu_proj/W"), ("shape", "u3/W"), ("negative", "z4_zu_proj/W"), ("negative", "z1_zu_proj/W")])
def test_parse_variables_names_the_bad_variable(defect, name):
    from icnn_b200.conv_picnn import parse_variables
    v = _olivetti_vars()
    if defect == "missing":
        del v[name]
    elif defect == "extra":
        v[name] = np.zeros((3, 3, 1, 64))
    elif defect == "shape":
        v[name] = v[name][..., :-1]
    else:
        v[name] = v[name].copy()
        v[name].flat[5] = -1e-3
    with pytest.raises(ValueError, match=name.replace("/", ".")):
        parse_variables(v, 64, 32)


def test_parse_variables_checks_the_strides_against_the_dense_width():
    from icnn_b200.conv_picnn import parse_variables
    with pytest.raises(ValueError, match="u3/W"):
        parse_variables(_olivetti_vars(), 64, 32, strides=[2, 2, 1])
    assert parse_variables(_olivetti_vars(), 64, 32, strides=[2, 4, 1]).convs == [(32, 8, 2), (64, 4, 4), (64, 3, 1)]


def test_torch_helper_from_the_variables_matches_the_reference_goldens():
    """tests/conv_energy.py (float64, literal batch-norm, NHWC flattening) against E_ / dE_dy_ of the reference's
    own completion Model with non-zero biases and non-identity batch-norm statistics (17 x 9 included)."""
    import conv_energy
    from icnn_b200.conv_picnn import parse_variables
    from oracle.gen_golden_conv import CASES, case
    gold = np.load(os.path.join(ROOT, "tests", "golden", "conv", "conv_picnn.npz"))
    for tag in CASES:
        v, x, y, H, W = case(tag)
        f, g = conv_energy.fg(parse_variables(v, H, W), x, y)
        assert np.abs(f - gold[tag + "_f"]).max() <= 1e-9 * np.abs(f).max(), tag
        assert np.abs(g - gold[tag + "_g"]).max() <= 1e-9 * np.abs(g).max(), tag


def test_descriptor_struct_matches_the_header(tmp_path):
    from icnn_b200 import _capi
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "icnn_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu\\n", sizeof(icnn_conv_picnn_desc), '
                   'offsetof(icnn_conv_picnn_desc, Ld), offsetof(icnn_conv_picnn_desc, bred)); return 0; }\n')
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "sz")])
    size, off_ld, off_bred = map(int, subprocess.check_output([str(tmp_path / "sz")]).split())
    assert C.sizeof(_capi.ConvPicnnDesc) == size
    assert _capi.ConvPicnnDesc.Ld.offset == off_ld and _capi.ConvPicnnDesc.bred.offset == off_bred


def test_conv_entry_points_reject_bad_arguments_without_a_gpu():
    from icnn_b200 import _capi
    lib = _capi.lib
    assert lib.icnn_conv_picnn_create(None, None, None) == -1
    d = _capi.ConvPicnnDesc()
    h = C.c_void_p()
    assert lib.icnn_conv_picnn_create(C.byref(d), C.byref(h), None) == -1 and b"H and W" in lib.icnn_last_error()
    assert lib.icnn_conv_picnn_workspace_bytes(None, 4) == 0
    assert lib.icnn_conv_picnn_fg(None, None, None, None, None, 0, None, None, 0, None, None, None) == -1
    assert lib.icnn_conv_solve_batch_fused(None, None, None, None, None, None) == -1
    assert lib.icnn_conv_gd_solve(None, None, None, None, None, None, 3, 0.01, 0.9, None, None) == -1
    assert lib.icnn_conv_picnn_destroy(None) == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    import icnn_b200
    with pytest.raises(RuntimeError, match="CUDA"):
        icnn_b200.ConvPICNN.from_variables(_olivetti_vars(), 64, 32)
