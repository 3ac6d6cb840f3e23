"""Thin Python wrappers over the C-ABI kernels (raw pointers + current CUDA stream). No math happens here."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch
from torch import Tensor

from . import _lib
from ._lib import (PF_ACT_GEGLU, PF_ACT_GELU, PF_ACT_NONE, PF_ACT_QUICK_GELU, PF_ACT_SILU, FmhaArgs,  # noqa: F401
                   GemmArgs)


# number of CUDA kernels launched through this module (bench.py reports it as `gpu_launches`)
LAUNCHES = 0


def _count(n: int = 1) -> None:
    global LAUNCHES
    LAUNCHES += n


def _vp(t: Optional[Tensor]):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _st():
    return C.c_void_p(_lib.stream_ptr())


# optional per-shape tile choice measured by scripts/tune_gemm.py: (M, N, Kc, taps) -> block_n (absent: pf_gemm_pick_block_n)
GEMM_LOG = None
# Split-K (pf_gemm_splitk_plan: only skinny deep-K problems — output tiles for at most half the SMs, >= 64 K-slabs, i.e. the 8x8 / 16x16-level
# convolutions of a small batch, which otherwise stream their weights through a handful of SMs). The K partition depends on the
# problem's M, so a sharded rank and the single-GPU run round a few convolutions differently (fp32 summation order):
# PF_SPLIT_K=0 (or ops.SPLIT_K = False) restores the bit-identical sharded == unsharded behaviour the tests check.
SPLIT_K = __import__("os").environ.get("PF_SPLIT_K", "1") != "0"
_TUNED: dict = {}


def _load_tuning() -> None:
    import json
    from pathlib import Path
    f = Path(__file__).with_name("gemm_tuning.json")
    if f.exists():
        for k, v in json.loads(f.read_text()).get("choice", {}).items():
            _TUNED[tuple(int(x) for x in k.split(","))] = int(v)


_load_tuning()


def pick_block_n(n: int, act: int = PF_ACT_NONE) -> int:
    return int(_lib.lib().pf_gemm_pick_block_n(int(n), int(act)))


def gemm_taps(A: Tensor, B: Tensor, out: Tensor, *, M: int, Kc: int, taps: Sequence[int] = (0,),
              bias: Optional[Tensor] = None, rowbias: Optional[Tensor] = None, rows_per_group: int = 0,
              residual: Optional[Tensor] = None, act: int = PF_ACT_NONE,
              image_map: Optional[tuple] = None, block_n: int = 0, k_splits: Optional[int] = None,
              row_stats: bool = False, ln: Optional[tuple] = None, scatter: Optional[tuple] = None):
    """acc = sum_t A[m + taps[t], :Kc] @ B[:, t*Kc:(t+1)*Kc]^T ; see include/panfusion_b200.h (pf_gemm_taps).

    A: [a_rows, a_ld] 16-bit, B: [N, len(taps)*Kc] 16-bit packed weight, out: [rows, n_out].
    image_map = (Hm, Wm, i0, j0, Hout, Wout) selects map_mode 1.
    Fused LayerNorm (see pf_gemm_args): row_stats=True makes this GEMM a PRODUCER — returns (out, stats) with
    stats [M, slots, 2] fp32 partial (sum, sum of squares) per output row; ln=(stats, colsum, eps) makes it a CONSUMER
    whose B holds gamma-scaled weights (engine._LinLN).
    """
    _lib.require_cuda(A, B, out)
    assert A.dim() == 2 and B.dim() == 2 and out.dim() == 2
    assert A.stride(1) == 1 and B.stride(1) == 1 and out.stride(1) == 1
    a = GemmArgs()
    a.A, a.a_rows, a.a_ld = A.data_ptr(), A.shape[0], A.stride(0)
    a.B, a.b_ld = B.data_ptr(), B.stride(0)
    a.dtype = _lib.dtype_code(A.dtype)
    assert B.dtype == A.dtype
    a.M, a.N, a.Kc, a.num_taps = int(M), B.shape[0], int(Kc), len(taps)
    for i, t in enumerate(taps):
        a.tap_off[i] = int(t)
    if block_n == -1:  # heuristic only (tuner baseline)
        block_n = 0
    elif not block_n and act != PF_ACT_GEGLU:
        block_n = _TUNED.get((int(M), B.shape[0], int(Kc), len(taps), int(image_map is not None),
                              int(residual is not None)), 0)  # tile width
    a.block_n = int(block_n)
    if GEMM_LOG is not None:
        GEMM_LOG.append((int(M), B.shape[0], int(Kc), len(taps), int(act), image_map is not None,
                         residual is not None, out.dtype == torch.float32))
    a.out, a.out_ld, a.out_dtype = out.data_ptr(), out.stride(0), _lib.dtype_code(out.dtype)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous()
        a.bias = bias.data_ptr()
    if rowbias is not None:
        assert rowbias.dtype == torch.float32 and rowbias.stride(1) == 1
        a.rowbias, a.rowbias_ld, a.rows_per_group = rowbias.data_ptr(), rowbias.stride(0), int(rows_per_group)
    if residual is not None:
        assert residual.stride(1) == 1
        a.residual, a.res_ld, a.res_dtype = residual.data_ptr(), residual.stride(0), _lib.dtype_code(residual.dtype)
    a.act = int(act)
    if image_map is not None:
        a.map_mode = 1
        a.Hm, a.Wm, a.i0, a.j0, a.Hout, a.Wout = (int(v) for v in image_map)
        if scatter is not None:  # (sy, sx, a, b): write phase (a, b) of the (sy, sx)-times larger output image
            a.out_sy, a.out_sx, a.out_a, a.out_b = (int(v) for v in scatter)
    stats = None
    if row_stats:
        slots = int(_lib.lib().pf_gemm_row_stats_slots(C.byref(a)))
        stats = torch.empty((int(M), slots, 2), dtype=torch.float32, device=A.device)
        a.row_stats_out = stats.data_ptr()
    if ln is not None:
        ln_stats, colsum, eps = ln
        assert ln_stats.dtype == torch.float32 and ln_stats.is_contiguous() and ln_stats.shape[0] == int(M)
        assert colsum.dtype == torch.float32 and colsum.is_contiguous() and colsum.numel() == B.shape[0]
        a.ln_stats, a.ln_slots, a.ln_colsum, a.ln_eps = ln_stats.data_ptr(), ln_stats.shape[1], colsum.data_ptr(), float(eps)
    ws = None
    if k_splits is None:
        k_splits = _lib.lib().pf_gemm_splitk_plan(C.byref(a)) if (SPLIT_K and not row_stats and ln is None) else 1
    if k_splits > 1:
        a.block_n = 0  # split-K runs with the heuristic's (widest) tile: operand bytes per FLOP matter
        ws = torch.empty(k_splits * int(M) * B.shape[0], dtype=torch.float32, device=A.device)
        a.k_splits, a.splitk_ws = int(k_splits), ws.data_ptr()
        _count(1)
    _count(1)
    _lib.check(_lib.lib().pf_gemm_taps(C.byref(a), _st()))
    return (out, stats) if row_stats else out


def bias_tile_flags(bias: Tensor) -> Tensor:
    """bias fp32 [G, Lq, Lk] -> uint8 [G, ceil(Lq/128), ceil(Lk/64)], 1 where the tile is entirely -1."""
    assert bias.dtype == torch.float32 and bias.dim() == 3 and bias.stride(2) == 1
    G, Lq, Lk = bias.shape
    flags = torch.empty((G, (Lq + 127) // 128, (Lk + 63) // 64), dtype=torch.uint8, device=bias.device)
    _count(1)
    _lib.check(_lib.lib().pf_bias_tile_flags(_vp(bias), G, Lq, Lk, bias.stride(1), C.c_int64(bias.stride(0)),
                                             _vp(flags), _st()))
    return flags


def bias_pack_tiles(bias: Tensor):
    """Dense fp32 bias [G, Lq, Lk] -> (store [n_live, 128 * 64] fp32, tile_off int32 [G, ceil(Lq/128), ceil(Lk/64)]): only the
    128 x 64 tiles that are not entirely -1 are kept (pf_bias_tile_flags -> pf_bias_tile_scan -> pf_bias_tile_pack). A stored
    tile is lane-interleaved for the attention kernel; `bias_tile_dense` gives back its [128, 64] view."""
    assert bias.dtype == torch.float32 and bias.dim() == 3 and bias.stride(2) == 1
    G, Lq, Lk = bias.shape
    flags = bias_tile_flags(bias)
    tile_off = torch.empty(flags.shape, dtype=torch.int32, device=bias.device)
    n_live = torch.empty(1, dtype=torch.int32, device=bias.device)
    lib = _lib.lib()
    _count(1)
    _lib.check(lib.pf_bias_tile_scan(_vp(flags), flags.numel(), _vp(tile_off), _vp(n_live), _st()))
    n = int(n_live.item())  # host sync: table construction is a one-off per camera set
    store = torch.empty((max(n, 1), 128 * 64), dtype=torch.float32, device=bias.device)
    _count(1)
    _lib.check(lib.pf_bias_tile_pack(_vp(bias), G, Lq, Lk, bias.stride(1), C.c_int64(bias.stride(0)), _vp(tile_off),
                                     _vp(store), _st()))
    return store, tile_off


def bias_tile_dense(tile: Tensor) -> Tensor:
    """One stored tile [8192] (pf_bias_tile_pack's layout [row / 32][col / 4][row % 32][col % 4]) -> dense [128, 64]."""
    return tile.reshape(4, 16, 32, 4).permute(0, 2, 1, 3).reshape(128, 64)


def fmha(q: Tensor, k: Tensor, v: Tensor, out: Tensor, *, heads: int, head_dim: int, scale: float,
         bias: Optional[Tensor] = None, bias_flags: Optional[Tensor] = None, bias_tiles: Optional[tuple] = None) -> Tensor:
    """out[b, l, h*d:(h+1)*d] = softmax(q_h k_h^T * scale + bias) v_h; see pf_fmha_fwd.

    q: [B, Lq, >=H*d] view (last stride 1), k/v: [B, Lk, >=H*d] views — slices of a fused QKV buffer are fine.
    bias: fp32 [Lq, Lk] (shared by batches and heads) or [B, Lq, Lk].
    """
    _lib.require_cuda(q, k, v, out)
    a = FmhaArgs()
    B, Lq = q.shape[0], q.shape[1]
    Lk = k.shape[1]
    for t in (q, k, v, out):
        assert t.dim() == 3 and t.stride(2) == 1
    a.q, a.k, a.v, a.out = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr()
    a.dtype = _lib.dtype_code(q.dtype)
    a.B, a.H, a.Lq, a.Lk, a.head_dim = B, int(heads), Lq, Lk, int(head_dim)
    a.q_ld, a.k_ld, a.v_ld, a.out_ld = q.stride(1), k.stride(1), v.stride(1), out.stride(1)
    a.q_bstride, a.k_bstride, a.v_bstride = q.stride(0), k.stride(0), v.stride(0)
    assert out.stride(0) == Lq * out.stride(1)
    a.scale = float(scale)
    if bias_tiles is not None:
        store, tile_off = bias_tiles  # tile-packed bias: store [n, 128, 64] fp32, tile_off int32 [G, QT, KT] (G = 1: shared)
        assert bias is None and store.dtype == torch.float32 and store.is_contiguous() and tile_off.dtype == torch.int32
        assert tile_off.dim() == 3 and tile_off.is_contiguous()
        assert tile_off.shape[1] == (Lq + 127) // 128 and tile_off.shape[2] == (Lk + 63) // 64 and tile_off.shape[0] in (1, B)
        a.bias, a.bias_tile_off = store.data_ptr(), tile_off.data_ptr()
        a.flags_ld = tile_off.stride(1)
        a.flags_bstride = tile_off.stride(0) if tile_off.shape[0] > 1 else 0
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.stride(-1) == 1
        a.bias = bias.data_ptr()
        if bias.dim() == 3:
            a.bias_bstride, a.bias_ld = (bias.stride(0) if bias.shape[0] > 1 else 0), bias.stride(1)
        else:
            a.bias_bstride, a.bias_ld = 0, bias.stride(0)
        if bias_flags is not None:
            assert bias_flags.dtype == torch.uint8 and bias_flags.dim() == 3 and bias_flags.is_contiguous()
            assert bias_flags.shape[1] == (Lq + 127) // 128 and bias_flags.shape[2] == (Lk + 63) // 64
            a.bias_flags = bias_flags.data_ptr()
            a.flags_bstride = bias_flags.stride(0) if (bias.dim() == 3 and bias.shape[0] > 1) else 0
            a.flags_ld = bias_flags.stride(1)
    _count(1)
    _lib.check(_lib.lib().pf_fmha_fwd(C.byref(a), _st()))
    return out


# ------------------------------------------------------------------------------------------------
# normalisation / preparation
# ------------------------------------------------------------------------------------------------
_GN_COUNTERS: dict = {}
_GN_SLOTS = 1 << 16


def _gn_counter_slot(device, n: int) -> Tensor:
    """n zeroed ints from a per-device ring (the kernel restores them to zero). Calls in flight at the same time —
    the two branch streams — always get different slots; a slot is only reused ~65k images later."""
    ent = _GN_COUNTERS.get(device)
    if ent is None:
        ent = _GN_COUNTERS[device] = [torch.zeros(_GN_SLOTS, dtype=torch.int32, device=device), 0]
    buf, pos = ent
    if pos + n > _GN_SLOTS:
        pos = 0
    ent[1] = pos + n
    return buf[pos:pos + n]


def groupnorm_stats(x: Tensor, N: int, H: int, W: int, groups: int, eps: float, circ: int = 0) -> Tensor:
    """x: [N*H*W, C] tokens -> mean_rstd [N, groups, 2] fp32 (statistics over the circularly extended image)."""
    Cc = x.shape[1]
    lib = _lib.lib()
    ws = torch.empty(lib.pf_groupnorm_ws_floats(N, groups), dtype=torch.float32, device=x.device)
    out = torch.empty((N, groups, 2), dtype=torch.float32, device=x.device)
    _count(1)
    _lib.check(lib.pf_groupnorm_stats(_vp(x), _lib.dtype_code(x.dtype), N, H, W, Cc, x.stride(0), groups, circ,
                                      _f(eps), _vp(ws), _vp(_gn_counter_slot(x.device, N)), _vp(out), _st()))
    return out


def _f(v: float):
    return C.c_float(float(v))


def conv_prep(x: Tensor, N: int, H: int, W: int, *, stats: Optional[Tensor] = None, gamma: Optional[Tensor] = None,
              beta: Optional[Tensor] = None, groups: int = 32, act: int = PF_ACT_NONE, circ: int = 0, up: int = 1,
              phases: int = 1, halo: int = 1) -> Tensor:
    """-> [phases * N * Ho * Wo, C] tap-GEMM A operand (see pf_conv_prep)."""
    Cc = x.shape[1]
    Hu, Wu = H * up, (W + 2 * circ) * up
    if phases == 4:
        Ho, Wo = Hu // 2 + 1, Wu // 2 + 1
    else:
        Ho, Wo = Hu + 2 * halo, Wu + 2 * halo
    out = torch.empty((phases * N * Ho * Wo, Cc), dtype=x.dtype, device=x.device)
    _count(1)
    _lib.check(_lib.lib().pf_conv_prep(_vp(x), _vp(out), _lib.dtype_code(x.dtype), N, H, W, Cc, x.stride(0),
                                       _vp(stats), _vp(gamma), _vp(beta), groups, act, circ, up, phases, halo, _st()))
    return out


def gn_prep(x: Tensor, N: int, H: int, W: int, *, gamma: Tensor, beta: Tensor, groups: int, eps: float,
            act: int = PF_ACT_NONE, circ_stats: int = 0, circ: int = 0, up: int = 1, phases: int = 1, halo: int = 1,
            x2: Optional[Tensor] = None, want_cat: bool = False):
    """GroupNorm statistics + apply (+SiLU) + conv_prep layout (pf_gn_prep: a statistics and an apply launch); with x2
    the normalised tensor is the channel concatenation cat(x, x2) and want_cat also returns that raw concatenation.
    -> out [phases * N * Ho * Wo, C] (and cat [N*H*W, C] if want_cat)."""
    C1, C2 = x.shape[1], (x2.shape[1] if x2 is not None else 0)
    Cc = C1 + C2
    Hu, Wu = H * up, (W + 2 * circ) * up
    if phases == 4:
        Ho, Wo = Hu // 2 + 1, Wu // 2 + 1
    else:
        Ho, Wo = Hu + 2 * halo, Wu + 2 * halo
    lib = _lib.lib()
    out = torch.empty((phases * N * Ho * Wo, Cc), dtype=x.dtype, device=x.device)
    cat = torch.empty((N * H * W, Cc), dtype=x.dtype, device=x.device) if want_cat else None
    ws = torch.empty(lib.pf_gn_prep_ws_floats(N, groups), dtype=torch.float32, device=x.device)
    _count(2)
    _lib.check(lib.pf_gn_prep(_vp(x), x.stride(0), C1, _vp(x2), x2.stride(0) if x2 is not None else 0, C2, _vp(cat),
                              _vp(out), _lib.dtype_code(x.dtype), N, H, W, groups, _f(eps), _vp(gamma), _vp(beta), act,
                              circ_stats, circ, up, phases, halo, _vp(ws), _vp(_gn_counter_slot(x.device, N)), _st()))
    return (out, cat) if want_cat else out


def layernorm(x: Tensor, gamma: Tensor, beta: Tensor, eps: float = 1e-5, pe: Optional[Tensor] = None) -> Tensor:
    T, Cc = x.shape
    out = torch.empty((T, Cc), dtype=x.dtype, device=x.device)
    pe_rows = pe.shape[0] if pe is not None else 0
    if pe is not None:
        assert pe.dtype == torch.float32 and pe.is_contiguous() and pe.shape[1] == Cc and T % pe_rows == 0
    _count(1)
    _lib.check(_lib.lib().pf_layernorm(_vp(x), x.stride(0), _vp(out), out.stride(0), _lib.dtype_code(x.dtype), T, Cc,
                                       _vp(pe), pe_rows, _vp(gamma), _vp(beta), _f(eps), _st()))
    return out


def conv_in(x: Tensor, w: Tensor, b: Optional[Tensor], dtype: torch.dtype, circ: bool, act: int = PF_ACT_NONE) -> Tensor:
    """x NCHW fp32 -> tokens [N*H*W, Cout]."""
    N, Cin, H, W = x.shape
    Cout = w.shape[0]
    out = torch.empty((N * H * W, Cout), dtype=dtype, device=x.device)
    _count(1)
    _lib.check(_lib.lib().pf_conv_in(_vp(x), _vp(w), _vp(b), _vp(out), _lib.dtype_code(dtype), N, Cin, H, W, Cout,
                                     int(circ), int(act), _st()))
    return out


def copy2d(src: Tensor, dst: Tensor) -> None:
    """dst[:, :cols] = src (row-strided 16-bit 2-D copy); src/dst may be column slices."""
    rows, cols = src.shape
    assert dst.shape == src.shape and src.stride(1) == 1 and dst.stride(1) == 1
    _count(1)
    _lib.check(_lib.lib().pf_copy2d(_vp(src), src.stride(0), _vp(dst), dst.stride(0), C.c_longlong(rows), cols, _st()))


def softmax_rows(s: Tensor, out: Tensor, scale: float) -> Tensor:
    """out[r] = softmax(scale * s[r]) — s fp32 [rows, cols], out 16-bit [rows, cols] (row strides free)."""
    assert s.dtype == torch.float32 and s.dim() == 2 and out.shape == s.shape and s.stride(1) == 1 and out.stride(1) == 1
    _count(1)
    _lib.check(_lib.lib().pf_softmax_rows(_vp(s), C.c_longlong(s.stride(0)), _vp(out), C.c_longlong(out.stride(0)),
                                          _lib.dtype_code(out.dtype), C.c_longlong(s.shape[0]), s.shape[1], _f(scale),
                                          _st()))
    return out


def tensor_to_image(x: Tensor) -> Tensor:
    """x fp32 [..., C, H, W] in [-1, 1] -> uint8 [..., H, W, C] on the device."""
    assert x.dtype == torch.float32 and x.dim() >= 3
    x = x.contiguous()
    Cc, H, W = x.shape[-3:]
    n = x.numel() // (Cc * H * W)
    out = torch.empty((*x.shape[:-3], H, W, Cc), dtype=torch.uint8, device=x.device)
    _count(1)
    _lib.check(_lib.lib().pf_tensor_to_image(_vp(x), _vp(out), C.c_longlong(n), Cc, H, W, _st()))
    return out


def timestep_embed(t: Tensor, dim: int, dtype: torch.dtype) -> Tensor:
    n = t.numel()
    out = torch.empty((n, dim), dtype=dtype, device=t.device)
    _count(1)
    _lib.check(_lib.lib().pf_timestep_embed(_vp(t), _vp(out), _lib.dtype_code(dtype), n, dim, _st()))
    return out


def cfg_ddim_step(x: Tensor, eps: Tensor, out: Tensor, guidance: float, alpha_t: float, alpha_prev: float,
                  roll: int = 0) -> Tensor:
    """x, out fp32 [..., W]; eps fp32 with 2x the elements of x ([uncond; text])."""
    assert x.dtype == eps.dtype == out.dtype == torch.float32 and x.is_contiguous() and eps.is_contiguous()
    assert eps.numel() == 2 * x.numel() and out.is_contiguous() and out.numel() == x.numel()
    _count(1)
    _lib.check(_lib.lib().pf_cfg_ddim_step(_vp(x), _vp(eps), _vp(out), C.c_longlong(x.numel()), x.shape[-1], int(roll),
                                           _f(guidance), _f(alpha_t), _f(alpha_prev), _st()))
    return out


def cfg_ddim_step_dev(x: Tensor, eps: Tensor, out: Tensor, guidance: float, coef: Tensor, roll: int = 0) -> Tensor:
    """Same as cfg_ddim_step with (c_x, c_eps) in a 2-float device tensor (graph-replayable)."""
    assert x.dtype == eps.dtype == out.dtype == coef.dtype == torch.float32
    assert x.is_contiguous() and eps.is_contiguous() and out.is_contiguous() and eps.numel() == 2 * x.numel()
    _count(1)
    _lib.check(_lib.lib().pf_cfg_ddim_step_dev(_vp(x), _vp(eps), _vp(out), C.c_longlong(x.numel()), x.shape[-1],
                                               int(roll), _f(guidance), _vp(coef), _st()))
    return out


def add_noise(x0: Tensor, noise: Tensor, t: Tensor, alphas_cumprod: Tensor) -> Tensor:
    """diffusers add_noise (PanFusion.py:84-85): x0, noise fp32 [B, ...], t int64 [B], alphas_cumprod fp32 [T] -> fp32 like x0."""
    _lib.require_cuda(x0, noise, t, alphas_cumprod)
    assert x0.dtype == noise.dtype == alphas_cumprod.dtype == torch.float32 and t.dtype == torch.int64
    assert x0.shape == noise.shape and x0.is_contiguous() and noise.is_contiguous() and t.is_contiguous()
    assert t.numel() == x0.shape[0] and alphas_cumprod.is_contiguous()
    out = torch.empty_like(x0)
    _count(1)
    _lib.check(_lib.lib().pf_add_noise(_vp(x0), _vp(noise), _vp(out), _vp(t), _vp(alphas_cumprod), alphas_cumprod.numel(),
                                       x0.shape[0], C.c_longlong(x0.numel() // x0.shape[0]), _st()))
    return out


def gaussian_sample(moments: Tensor, eps: Tensor, latent_channels: int, scale: float) -> Tensor:
    """moments fp32 [N*HW, ld] rows = [mean | logvar | ...], eps fp32 NCHW [N, L, h, w] -> z fp32 NCHW (pf_gaussian_sample)."""
    _lib.require_cuda(moments, eps)
    assert moments.dtype == eps.dtype == torch.float32 and moments.dim() == 2 and moments.stride(1) == 1 and eps.is_contiguous()
    N, L, h, w = eps.shape
    assert L == latent_channels and moments.shape[0] == N * h * w and moments.shape[1] >= 2 * L
    out = torch.empty_like(eps)
    _count(1)
    _lib.check(_lib.lib().pf_gaussian_sample(_vp(moments), moments.stride(0), _vp(eps), _vp(out), N, L, h * w, _f(scale), _st()))
    return out


_MSE_WS = {}


def mse_loss(a: Tensor, b: Tensor) -> Tensor:
    """torch.nn.functional.mse_loss(a, b) (mean; PanFusion.py:92-93) -> fp32 scalar tensor, launch-independent summation order."""
    _lib.require_cuda(a, b)
    assert a.dtype == b.dtype == torch.float32 and a.shape == b.shape and a.is_contiguous() and b.is_contiguous()
    lib = _lib.lib()
    ent = _MSE_WS.get(a.device)
    if ent is None:  # per-device partials + counter; calls on one device are ordered by the stream they are issued on
        ent = _MSE_WS[a.device] = (torch.empty(lib.pf_mse_loss_ws_floats(), dtype=torch.float32, device=a.device),
                                   torch.zeros(1, dtype=torch.int32, device=a.device))
    out = torch.empty((), dtype=torch.float32, device=a.device)
    _count(1)
    _lib.check(lib.pf_mse_loss(_vp(a), _vp(b), C.c_longlong(a.numel()), _vp(ent[0]), _vp(ent[1]), _vp(out), _st()))
    return out


# ------------------------------------------------------------------------------------------------
# EPPA tables
# ------------------------------------------------------------------------------------------------
_BLUR5 = None


def _blur5():
    """5 taps of kornia's sigma-1 gaussian, computed like kornia does (fp32 torch ops), as a ctypes float[5]."""
    global _BLUR5
    if _BLUR5 is None:
        x = torch.arange(5, dtype=torch.float32) - 2
        g = torch.exp(-x.pow(2.0) / 2.0)
        g = g / g.sum()
        _BLUR5 = (C.c_float * 5)(*g.tolist())
    return _BLUR5


def eppa_tables(cams_e2p: Tensor, cams_p2e: Tensor, m: int, ph: int, pw: int, eh: int, ew: int):
    """cams_*: [V, 20] float64 device records -> (bias1 [V/m, E, m*P], bias2 [V/m, m*P, E]) fp32."""
    V = cams_e2p.shape[0]
    P, E = ph * pw, eh * ew
    dev = cams_e2p.device
    ws_idx = torch.empty(4 * V * (P + E), dtype=torch.int32, device=dev)
    ws_w = torch.empty(4 * V * (P + E), dtype=torch.float32, device=dev)
    bias1 = torch.empty((V // m, E, m * P), dtype=torch.float32, device=dev)
    bias2 = torch.empty((V // m, m * P, E), dtype=torch.float32, device=dev)
    _count(3)
    _lib.check(_lib.lib().pf_eppa_tables(_vp(cams_e2p), _vp(cams_p2e), V, m, ph, pw, eh, ew, _blur5(), _vp(ws_idx),
                                         _vp(ws_w), _vp(bias1), _vp(bias2), _st()))
    return bias1, bias2


def eppa_pe(cams_e2p: Tensor, ph: int, pw: int, eh: int, ew: int, freq_bands: Tensor):
    """-> (pers_pe [V*P, 4N], equi_pe [E, 4N]) fp32 SphericalPE tables."""
    V = cams_e2p.shape[0]
    nf = freq_bands.numel()
    dev = cams_e2p.device
    pers_pe = torch.empty((V * ph * pw, 4 * nf), dtype=torch.float32, device=dev)
    equi_pe = torch.empty((eh * ew, 4 * nf), dtype=torch.float32, device=dev)
    fb = freq_bands.to(device=dev, dtype=torch.float32).contiguous()
    _count(1)
    _lib.check(_lib.lib().pf_eppa_pe(_vp(cams_e2p), V, ph, pw, eh, ew, _vp(fb), nf, _vp(pers_pe), _vp(equi_pe), _st()))
    return pers_pe, equi_pe


# ------------------------------------------------------------------------------------------------
# MVDiffusion CPAttn
# ------------------------------------------------------------------------------------------------
CP_SLOTS = 18


def cpattn_tables(homo_l: Tensor, homo_r: Tensor, h: int, w: int, img_size: int):
    """homo_l / homo_r fp32 [G, m, 2, 3, 3] on the device -> (pos fp32 [G, m, h*w, 18, 4], mask uint8 [G, m, h*w, 18])."""
    _lib.require_cuda(homo_l, homo_r)
    assert homo_l.dtype == homo_r.dtype == torch.float32 and homo_l.is_contiguous() and homo_r.is_contiguous()
    assert homo_l.shape == homo_r.shape and homo_l.dim() == 5 and tuple(homo_l.shape[2:]) == (2, 3, 3)
    G, m = homo_l.shape[:2]
    pos = torch.empty((G, m, h * w, CP_SLOTS, 4), dtype=torch.float32, device=homo_l.device)
    mask = torch.empty((G, m, h * w, CP_SLOTS), dtype=torch.uint8, device=homo_l.device)
    _count(1)
    _lib.check(_lib.lib().pf_cpattn_tables(_vp(homo_l), _vp(homo_r), G, m, h, w, img_size, _vp(pos), _vp(mask), _st()))
    return pos, mask


def cpattn_gather(x: Tensor, B: int, m: int, h: int, w: int, pos: Tensor, mask: Tensor, freq_bands: Tensor):
    """x tokens [B*m*h*w, >=C] 16-bit -> (keys [B*m*h*w*18, C] 16-bit, stats fp32 [B*m*h*w*18, 2, 2]) (pf_cpattn_gather)."""
    _lib.require_cuda(x, pos, mask, freq_bands)
    C = 4 * freq_bands.numel()
    assert x.dim() == 2 and x.stride(1) == 1 and x.shape[0] == B * m * h * w and x.shape[1] >= C
    assert pos.dtype == torch.float32 and pos.is_contiguous() and mask.dtype == torch.uint8 and mask.is_contiguous()
    assert freq_bands.dtype == torch.float32 and freq_bands.is_contiguous()
    G = pos.shape[0]
    assert tuple(pos.shape) == (G, m, h * w, CP_SLOTS, 4) and tuple(mask.shape) == (G, m, h * w, CP_SLOTS)
    rows = B * m * h * w * CP_SLOTS
    keys = torch.empty((rows, C), dtype=x.dtype, device=x.device)
    stats = torch.empty((rows, 2, 2), dtype=torch.float32, device=x.device)
    _count(1)
    _lib.check(_lib.lib().pf_cpattn_gather(_vp(x), x.stride(0), _lib.dtype_code(x.dtype), B, m, h, w, C, G, _vp(pos),
                                           _vp(mask), _vp(freq_bands), _vp(keys), _vp(stats), _st()))
    return keys, stats


def cpattn_attn(q: Tensor, kv: Tensor, out: Tensor, scale: float) -> Tensor:
    """q [T, >=C], kv [T*18, >=2C] (K | V), out [T, >=C], all 16-bit, last stride 1; heads of width 32 (pf_cpattn_attn)."""
    _lib.require_cuda(q, kv, out)
    ntok, ch = out.shape
    assert q.stride(1) == kv.stride(1) == out.stride(1) == 1 and q.shape[0] == ntok and kv.shape[0] == ntok * CP_SLOTS
    assert q.dtype == kv.dtype == out.dtype
    _count(1)
    _lib.check(_lib.lib().pf_cpattn_attn(_vp(q), q.stride(0), _vp(kv), kv.stride(0), _vp(out), out.stride(0),
                                         _lib.dtype_code(q.dtype), C.c_longlong(ntok), ch, _f(scale), _st()))
    return out


def mp2e(views: Tensor, fov_deg, theta_deg, phi_deg, out_hw) -> Tensor:
    """Stitch m uint8 views [m, hp, wp, C] (device) into one uint8 panorama [H, W, C] (pf_mp2e, mp2e.py:6-30)."""
    from . import geometry
    _lib.require_cuda(views)
    assert views.dtype == torch.uint8 and views.dim() == 4 and views.is_contiguous()
    m, hp, wp, ch = views.shape
    cams, _ = geometry.camera_records("p2e", list(map(float, fov_deg)), list(map(float, theta_deg)),
                                      list(map(float, phi_deg)), m, hp, wp, views.device)
    H, W = (int(v) for v in out_hw)
    out = torch.empty((H, W, ch), dtype=torch.uint8, device=views.device)
    _count(1)
    _lib.check(_lib.lib().pf_mp2e(_vp(views), m, hp, wp, ch, _vp(cams), H, W, _vp(out), _st()))
    return out
