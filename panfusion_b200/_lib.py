"""ctypes binding of the C-ABI library (include/panfusion_b200.h).

There is no fallback: if the shared object is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import os

import torch

PF_F32, PF_F16, PF_BF16 = 0, 1, 2
PF_ACT_NONE, PF_ACT_SILU, PF_ACT_GELU, PF_ACT_GEGLU = 0, 1, 2, 3
PF_MAX_TAPS = 16
PF_CAM_DOUBLES = 20

_DTYPES = {torch.float32: PF_F32, torch.float16: PF_F16, torch.bfloat16: PF_BF16}

LIB_PATH = Path(__file__).resolve().parent / "lib" / "libpanfusion_b200.so"
if os.environ.get("PF_LIB_PATH"):  # A/B of two builds of the SAME C-ABI (scripts/): never a different implementation
    LIB_PATH = Path(os.environ["PF_LIB_PATH"])


class PFError(RuntimeError):
    pass


class GemmArgs(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("a_rows", C.c_int64), ("a_ld", C.c_int32),
        ("B", C.c_void_p), ("b_ld", C.c_int32), ("dtype", C.c_int32),
        ("M", C.c_int32), ("N", C.c_int32), ("Kc", C.c_int32), ("num_taps", C.c_int32),
        ("tap_off", C.c_int32 * PF_MAX_TAPS), ("block_n", C.c_int32),
        ("out", C.c_void_p), ("out_ld", C.c_int32), ("out_dtype", C.c_int32),
        ("bias", C.c_void_p), ("rowbias", C.c_void_p), ("rowbias_ld", C.c_int32), ("rows_per_group", C.c_int32),
        ("residual", C.c_void_p), ("res_ld", C.c_int32), ("res_dtype", C.c_int32),
        ("act", C.c_int32),
        ("map_mode", C.c_int32), ("Hm", C.c_int32), ("Wm", C.c_int32), ("i0", C.c_int32), ("j0", C.c_int32),
        ("Hout", C.c_int32), ("Wout", C.c_int32),
        ("k_splits", C.c_int32), ("splitk_ws", C.c_void_p),
        ("out_sy", C.c_int32), ("out_sx", C.c_int32), ("out_a", C.c_int32), ("out_b", C.c_int32),
        ("row_stats_out", C.c_void_p), ("ln_stats", C.c_void_p), ("ln_slots", C.c_int32), ("ln_colsum", C.c_void_p),
        ("ln_eps", C.c_float),
    ]


class FmhaArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("out", C.c_void_p),
        ("dtype", C.c_int32), ("B", C.c_int32), ("H", C.c_int32), ("Lq", C.c_int32), ("Lk", C.c_int32),
        ("head_dim", C.c_int32),
        ("q_ld", C.c_int32), ("k_ld", C.c_int32), ("v_ld", C.c_int32), ("out_ld", C.c_int32),
        ("q_bstride", C.c_int64), ("k_bstride", C.c_int64), ("v_bstride", C.c_int64),
        ("scale", C.c_float), ("bias", C.c_void_p), ("bias_bstride", C.c_int64), ("bias_ld", C.c_int32),
        ("bias_flags", C.c_void_p), ("flags_bstride", C.c_int64), ("flags_ld", C.c_int32),
        ("bias_tile_off", C.c_void_p),
    ]


_lib = None


def lib() -> C.CDLL:
    """Load (once) the native library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise PFError(
                f"{LIB_PATH} not found: build it with `python -m panfusion_b200.build` "
                "(panfusion_b200 has no non-CUDA path)")
        l = C.CDLL(str(LIB_PATH))
        l.pf_last_error.restype = C.c_char_p
        for name in EXPORTS:
            getattr(l, name)  # AttributeError if the header and the library diverge
        _lib = l
    return _lib


# every symbol include/panfusion_b200.h declares (checked by tests/test_cabi.py against the header text)
EXPORTS = [
    "pf_last_error", "pf_version", "pf_check_device",
    "pf_e2p", "pf_e2p_shared", "pf_e2p_py360", "pf_c2e_py360", "pf_e2c_py360", "pf_p2e",
    "pf_gemm_taps", "pf_gemm_pick_block_n", "pf_gemm_splitk_plan", "pf_gemm_row_stats_slots",
    "pf_fmha_fwd", "pf_bias_tile_flags", "pf_bias_tile_scan", "pf_bias_tile_pack",
    "pf_groupnorm_ws_floats", "pf_groupnorm_stats", "pf_conv_prep", "pf_gn_prep_ws_floats", "pf_gn_prep", "pf_layernorm",
    "pf_conv_in", "pf_copy2d", "pf_pad_pano", "pf_softmax_rows", "pf_tensor_to_image", "pf_timestep_embed", "pf_cfg_ddim_step", "pf_cfg_ddim_step_dev",
    "pf_eppa_tables", "pf_eppa_pe", "pf_cpattn_tables", "pf_cpattn_gather", "pf_cpattn_attn", "pf_mp2e",
    "pf_allgather_views", "pf_enable_peer_access", "pf_comm_alloc", "pf_comm_free", "pf_ipc_export", "pf_ipc_open",
    "pf_ipc_close", "pf_embed_tokens", "pf_add_noise", "pf_mse_loss_ws_floats", "pf_mse_loss", "pf_gaussian_sample",
]


def check(rc: int) -> None:
    if rc != 0:
        msg = lib().pf_last_error().decode(errors="replace")
        if rc == -1:
            raise ValueError(msg)
        if rc == -3:
            raise NotImplementedError(msg)
        raise PFError(f"[{rc}] {msg}")


def dtype_code(dt: torch.dtype) -> int:
    try:
        return _DTYPES[dt]
    except KeyError:
        raise ValueError(f"unsupported dtype {dt}") from None


def ptr(t: torch.Tensor | None) -> int | None:
    if t is None:
        return None
    return t.data_ptr()


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def require_cuda(*tensors: torch.Tensor) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise PFError("panfusion_b200 kernels need CUDA tensors (there is no CPU path)")
