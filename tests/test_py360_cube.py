"""CPU: py360convert's cubemap conversions (c2e / e2c, external/py360convert/c2e.py, e2c.py) — the numpy restatement
against the golden minted by executing the reference, the host face-type table, the cube layout helpers and the
reference's exception types. The kernels themselves are checked in test_gpu_py360_cube.py."""
import ctypes

import numpy as np
import pytest
import torch

import _py360_cube_oracle as oc
from panfusion_b200 import py360


@pytest.fixture(scope="module")
def gold():
    return np.load(oc.GOLDEN)


def test_restatement_matches_reference_golden_bit_for_bit(gold):
    """The golden holds the SHA-256 (dtype, shape, bytes) and the sum of every reference output."""
    for k, (fw, (h, w), mode, tag, C, fmt) in enumerate(oc.C2E_CASES):
        got = oc.c2e(oc.as_horizon(oc.c2e_input(k), fmt), h, w, mode)
        assert got.dtype == np.float64 and got.shape == (h, w, C)
        assert oc.digest(got) == str(gold[f"c2e{k}_sha256"]), (k, got.sum() - gold[f"c2e{k}_sum"])
    for k, (fw, _, mode, tag, C, fmt) in enumerate(oc.E2C_CASES):
        got = oc.e2c(oc.e2c_input(k), fw, mode)
        assert got.dtype == (np.uint8 if tag == "u8" else np.float32) and got.shape == (fw, 6 * fw, C)
        assert oc.digest(got) == str(gold[f"e2c{k}_sha256"]), (k, got.astype(np.float64).sum() - gold[f"e2c{k}_sum"])


@pytest.mark.parametrize("hw", oc.FACETYPE_HW)
def test_face_type_table_matches_reference(gold, hw):
    """The host ceiling-row table and the mapping pf_c2e_py360 applies to it give the reference's face of every pixel."""
    h, w = hw
    ref = gold[f"facetype_{h}x{w}"].astype(np.int32)
    assert np.array_equal(py360.equirect_facetype(h, w), ref)
    assert np.array_equal(oc.facetype(h, w), ref)
    ceil = py360.ceil_rows(h, w)
    assert ceil.dtype == np.int32 and ceil.shape == (w // 4,)


def test_cube_border_table_shape_and_range():
    for fw in (1, 2, 48, 64):
        bt = py360.cube_border(fw)
        assert bt.shape == (6, 4 * fw + 4) and bt.dtype == np.int32
        assert bt.min() >= -1 and bt.max() < fw * 6 * fw
        # U and D carry zero pads only at the two ends of their pad columns, the side faces none
        assert (bt[:4] >= 0).all() and (bt[4:] == -1).sum() == 8


@pytest.mark.parametrize("as_torch", [False, True])
def test_layout_helpers_round_trip(as_torch):
    cube = np.random.default_rng(3).integers(0, 256, (5, 30, 3)).astype(np.uint8)
    x = torch.from_numpy(cube) if as_torch else cube
    eq = (lambda a, b: torch.equal(a, b)) if as_torch else np.array_equal
    faces = py360.cube_h2list(x)
    assert len(faces) == 6 and all(tuple(f.shape) == (5, 5, 3) for f in faces)
    assert eq(py360.cube_list2h(faces), x)
    d = py360.cube_h2dict(x)
    assert list(d) == ["F", "R", "B", "L", "U", "D"] and eq(d["U"], faces[4])
    assert eq(py360.cube_dict2h(d), x)
    dice = py360.cube_h2dice(x)
    assert tuple(dice.shape) == (15, 20, 3)
    assert eq(py360.cube_dice2h(dice), x)
    # dice layout: F at (row 1, col 1) as is, R mirrored left-right at (1, 2), U upside down at (0, 1), corners empty
    assert eq(dice[5:10, 5:10], faces[0])
    assert eq(dice[5:10, 10:15], faces[1].flip(1) if as_torch else faces[1][:, ::-1])
    assert eq(dice[0:5, 5:10], faces[4].flip(0) if as_torch else faces[4][::-1])
    assert int(dice[0:5, 0:5].sum()) == 0


def test_reference_exception_types():
    cube = np.zeros((8, 48, 3), np.uint8)
    with pytest.raises(NotImplementedError):
        py360.c2e(cube, 16, 32, mode="bicubic", cube_format="horizon")
    with pytest.raises(NotImplementedError):
        py360.c2e(cube, 16, 32, cube_format="cross")
    with pytest.raises(AssertionError):
        py360.c2e(cube, 16, 36, cube_format="horizon")                   # w % 8 != 0
    with pytest.raises(AssertionError):
        py360.c2e(np.zeros((8, 40, 3), np.uint8), 16, 32, cube_format="horizon")
    with pytest.raises(AssertionError):
        py360.c2e(np.zeros((8, 48), np.uint8), 16, 32, cube_format="horizon")
    with pytest.raises(AssertionError):
        py360.c2e([cube[:, :8]] * 5, 16, 32, cube_format="list")
    with pytest.raises(AssertionError):
        py360.e2c(np.zeros((16, 32), np.uint8), 8)
    with pytest.raises(NotImplementedError):
        py360.e2c(np.zeros((16, 32, 3), np.uint8), 8, mode="bicubic")
    with pytest.raises(NotImplementedError):
        py360.e2c(np.zeros((16, 32, 3), np.uint8), 8, cube_format="cross")


def test_c_abi_rejects_bad_arguments_before_any_launch():
    from panfusion_b200 import _lib
    lib = _lib.lib()
    p = ctypes.c_void_p(16)  # never dereferenced: every check below returns before a launch
    assert lib.pf_c2e_py360(None, None, 1, 8, 3, 16, 32, None, None, 0, None) == -1
    assert b"null pointer" in lib.pf_last_error()
    assert lib.pf_c2e_py360(p, p, 1, 8, 3, 16, 36, p, p, 0, None) == -1
    assert b"multiple of 8" in lib.pf_last_error()
    assert lib.pf_c2e_py360(p, p, 1, 0, 3, 16, 32, p, p, 0, None) == -1
    assert lib.pf_c2e_py360(p, p, 1, 8, 3, 16, 32, p, p, 2, None) == -3
    assert b"unknown mode" in lib.pf_last_error()
    assert lib.pf_e2c_py360(p, p, 1, 1, 32, 3, 8, 0, None) == -1
    assert b"bad shape" in lib.pf_last_error()
    assert lib.pf_e2c_py360(p, p, 1, 16, 32, 3, 8, 7, None) == -3
    with pytest.raises(NotImplementedError):
        _lib.check(-3)
