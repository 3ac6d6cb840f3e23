"""CPU (-m "not gpu"): the C-ABI library builds, loads and exports exactly what include/panfusion_b200.h declares;
host-side logic that needs no GPU (packing, camera records, schedule)."""
import ctypes
import re
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent


def _declared():
    text = (ROOT / "include" / "panfusion_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(pf_[a-z0-9_]+)\s*\(", text)))


def test_library_builds_and_exports_every_declared_symbol():
    from panfusion_b200 import _lib, build
    build.build()
    lib = ctypes.CDLL(str(_lib.LIB_PATH))
    declared = _declared()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    assert sorted(_lib.EXPORTS) == declared
    assert lib.pf_version() >= 100


def test_bad_arguments_fail_loudly_without_gpu():
    """Argument validation happens before any CUDA call: error code + message, mapped to Python exceptions."""
    from panfusion_b200 import _lib
    lib = _lib.lib()
    rc = lib.pf_e2p(None, None, 0, 1, 1, 8, 16, 4, 4, None, 0, 0, None)
    assert rc == -1 and b"null pointer" in lib.pf_last_error()
    with pytest.raises(ValueError):
        _lib.check(rc)
    assert lib.pf_gemm_pick_block_n(320, 0) == 160 and lib.pf_gemm_pick_block_n(128, 0) == 128
    assert lib.pf_gemm_pick_block_n(100, 0) == 0


def _gemm_args(**fields):
    """A valid one-tap fp16 pf_gemm_args (M = 512, N = Kc = 320) with `fields` overridden; its pointers are never
    dereferenced."""
    from panfusion_b200 import _lib
    a = _lib.GemmArgs()
    a.A, a.a_rows, a.a_ld, a.B, a.b_ld, a.dtype = 0x10000, 512, 320, 0x20000, 320, 1
    a.M, a.N, a.Kc, a.num_taps = 512, 320, 320, 1
    a.out, a.out_ld, a.out_dtype = 0x30000, 320, 1
    for k, v in fields.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("field,value,extra,operand", [
    ("residual", 0x40008, dict(res_ld=320, res_dtype=1), b"residual"),
    ("rowbias", 0x40004, dict(rowbias_ld=320, rows_per_group=64), b"rowbias"),
    ("rowbias", 0x40000, dict(rowbias_ld=322, rows_per_group=64), b"rowbias"),
    ("splitk_ws", 0x40008, dict(k_splits=2), b"splitk_ws"),
    ("row_stats_out", 0x40004, {}, b"row_stats_out"),
])
def test_misaligned_epilogue_operands_are_rejected_without_gpu(field, value, extra, operand):
    """The epilogues and the split-K reduce access residual, rowbias and splitk_ws 16 bytes and row_stats_out 8 bytes at a
    time: pf_gemm_taps refuses a misaligned one (or a rowbias row stride that misaligns its rows) before any CUDA call,
    naming the operand. The pointers are never dereferenced."""
    import ctypes as C
    from panfusion_b200 import _lib
    lib = _lib.lib()
    a = _gemm_args(**{field: value}, **extra)
    rc = lib.pf_gemm_taps(C.byref(a), None)
    assert rc == -1 and operand in lib.pf_last_error(), lib.pf_last_error()


_GEGLU = dict(act=3, N=512, out_ld=256)  # PF_ACT_GEGLU: 512 packed columns -> 256 outputs
_LN = dict(ln_stats=0x40000, ln_slots=4, ln_colsum=0x50000, ln_eps=1e-5)


@pytest.mark.parametrize("fields,cause", [
    (dict(_GEGLU, block_n=128), b"GEGLU runs only at block_n 256"),
    (dict(_GEGLU, N=640, out_ld=320, block_n=160), b"GEGLU runs only at block_n 256"),
    (dict(_GEGLU, out_dtype=0), b"GEGLU needs map_mode 0 and a 16-bit output"),
    (dict(_GEGLU, num_taps=2, b_ld=640), b"GEGLU needs one tap"),
    (dict(row_stats_out=0x40000, num_taps=2, b_ld=640), b"fused LayerNorm needs one tap and no rowbias"),
    (dict(_LN, rowbias=0x60000, rowbias_ld=320, rows_per_group=64), b"fused LayerNorm needs one tap and no rowbias"),
    (dict(N=512, block_n=256), b"unsupported block_n 256"),
    (dict(block_n=64 | (1 << 16)), b"unsupported block_n 65600"),
], ids=["geglu_bn128", "geglu_bn160", "geglu_fp32_out", "geglu_two_taps", "row_stats_two_taps", "ln_stats_rowbias",
        "bn256_without_geglu", "bn_high_bits"])
def test_gemm_contract_is_checked_without_gpu(fields, cause):
    """GEGLU runs only at block_n = 256 with one tap and a 16-bit output, the fused LayerNorm needs one tap and no row
    bias, and block_n is 0, 64, 128, 160 or (GEGLU) 256: pf_gemm_taps refuses anything else before any CUDA call, with
    a message that names the cause."""
    import ctypes as C
    from panfusion_b200 import _lib
    lib = _lib.lib()
    rc = lib.pf_gemm_taps(C.byref(_gemm_args(**fields)), None)
    assert rc == -1 and cause in lib.pf_last_error(), lib.pf_last_error()


def test_no_cpu_path():
    from panfusion_b200 import geometry
    with pytest.raises(Exception):
        geometry.e2p(torch.zeros(1, 1, 8, 16), 90, 0, 0, (4, 4))  # CPU tensor: refused, never computed on the host


def test_camera_record_matches_oracle_rotations():
    from oracle import geometry as og
    from panfusion_b200.geometry import _camera_record
    for fov, th, ph in [(90.0, 0.0, 0.0), (75.0, 45.0, 30.0), (100.0, 200.0, -60.0)]:
        rec = np.array(_camera_record("e2p", fov, th, ph, 16, 24))
        R1, R2 = og.camera_rotations(th, ph)
        np.testing.assert_allclose(rec[:9].reshape(3, 3), R1, atol=1e-15)
        np.testing.assert_allclose(rec[9:18].reshape(3, 3), R2, atol=1e-15)
        assert rec[18] == np.tan(np.radians(fov / 2.0))
        rec = np.array(_camera_record("p2e", fov, th, ph, 16, 24))
        np.testing.assert_allclose(rec[:9].reshape(3, 3), np.linalg.inv(R1), atol=1e-15)


def test_geglu_and_conv_packing():
    from panfusion_b200.packing import pack_conv3x3, pack_geglu
    w = torch.arange(2 * 3 * 9, dtype=torch.float32).reshape(2, 3, 3, 3)
    p = pack_conv3x3(w)
    assert p.shape == (2, 27) and p[1, 4 * 3 + 2] == w[1, 2, 1, 1]  # tap (1,1), channel 2
    W = torch.randn(640, 8)
    b = torch.randn(640)
    wp, bp = pack_geglu(W, b, 160)
    assert torch.equal(wp[:80], W[:80]) and torch.equal(wp[80:160], W[320:400]) and torch.equal(wp[160:240], W[80:160])
    assert torch.equal(bp[80:160], b[320:400])


def test_schedule_matches_oracle():
    from oracle.sampler import DDIM
    from panfusion_b200.sampler import DDIMSchedule
    a, b = DDIMSchedule(), DDIM()
    a.set_timesteps(50)
    b.set_timesteps(50)
    assert torch.equal(a.timesteps, b.timesteps)
    x, e = torch.randn(8, dtype=torch.float64), torch.randn(8, dtype=torch.float64)
    for t in (981, 501, 1):
        cx, ce = a.coefficients(t)
        torch.testing.assert_close(cx * x + ce * e, b.step(e, t, x).double(), rtol=1e-5, atol=1e-6)


def test_camera_table_dedup():
    from panfusion_b200.eppa import CameraTables
    cams = dict(FoV=torch.full((4,), 90.0), theta=torch.tensor([0.0, 180.0, 0.0, 180.0]), phi=torch.zeros(4))
    key, groups = CameraTables.dedup(CameraTables.camera_key(cams), 2)
    assert groups == 1 and len(key[0]) == 2
    cams["theta"] = torch.tensor([0.0, 180.0, 90.0, 270.0])
    key, groups = CameraTables.dedup(CameraTables.camera_key(cams), 2)
    assert groups == 2 and len(key[0]) == 4


def test_row_stats_slots_ignore_tile_requests():
    """A fused-LayerNorm PRODUCER's slot layout is a function of N alone (never of a tile-width request), and the query
    gives the same answer before and after the caller has filled in row_stats_out."""
    import ctypes as C
    from panfusion_b200 import _lib
    lib = _lib.lib()
    for n, want in ((320, 4), (640, 8), (1280, 16), (128, 2), (64, 2)):
        seen = set()
        for req in (0, 64, 128, 160, 256):
            a = _lib.GemmArgs()
            a.N, a.M, a.Kc, a.num_taps, a.block_n = n, 512, n, 1, req
            seen.add(lib.pf_gemm_row_stats_slots(C.byref(a)))
            a.row_stats_out = 1
            seen.add(lib.pf_gemm_row_stats_slots(C.byref(a)))
        assert seen == {want}, (n, seen)


def test_packed_bias_tile_layout_helper():
    """ops.bias_tile_dense inverts the lane-interleaved tile layout documented at pf_bias_tile_pack
    (include/panfusion_b200.h): element (r, c) of a 128 x 64 tile sits at (((r/32)*16 + c/4)*32 + r%32)*4 + c%4."""
    import torch
    from panfusion_b200 import ops
    dense = torch.arange(128 * 64, dtype=torch.float32).reshape(128, 64)
    r, c = torch.meshgrid(torch.arange(128), torch.arange(64), indexing="ij")
    pos = (((r // 32) * 16 + c // 4) * 32 + r % 32) * 4 + c % 4
    assert sorted(pos.flatten().tolist()) == list(range(128 * 64))  # a permutation of the tile
    stored = torch.empty(128 * 64)
    stored[pos.flatten()] = dense.flatten()
    assert torch.equal(ops.bias_tile_dense(stored), dense)
    # one 16-byte piece of a warp = 32 lanes x 4 floats, contiguous
    w, e = 2, 5
    piece = stored[((w * 16 + e) * 32) * 4:((w * 16 + e) * 32 + 32) * 4].reshape(32, 4)
    assert torch.equal(piece, dense[w * 32:(w + 1) * 32, e * 4:(e + 1) * 4])
