"""fp64 restatements of the tap-GEMM (pf_gemm_taps), flash-attention (pf_fmha_fwd) and implicit-GEMM convolution
(pf_conv_circ, pf_faedt_conv, pf_conv2d_nhwc, pf_hnet_conv) contracts of include/panfusion_b200.h, and the error bound
a correct kernel meets on every output element.

The bound scales with the magnitude of the terms that make up each element, not with max|ref|: an element that is
small because its terms cancel may carry the rounding of its large terms, but one wrong tap, row or column changes an
element by about its own magnitude, far above the bound.

  tap-GEMM   |got - ref| <= 2^-14 * mag + ulp_out(ref)
             mag = (|A| @ |B|^T) + |bias| + |rowbias| (times 1.13 through GELU / SiLU) + |residual|
             2^-14 is ~10x the sqrt(K) * 2^-24 of fp32 accumulation at K = 9 * 1280.
             LayerNorm consumer: mag over the normalised input, plus 2^-8 * (|x - mean| * rstd) @ |W|^T (the fused form
             does not round LN(x) to 16 bits, the stand-alone pair does).
  attention  |got - ref| <= 2u * (P @ |V|) + u * |ref| + 2^-20, u = 2^-11 (fp16) / 2^-8 (bf16): the kernel rounds
             P to 16 bits before P V and rounds the output once.
  conv_mma   |got - ref| <= 2^-14 * (|x| * |w| + |bias| + |residual|) + ulp_out(ref)  (the implicit-GEMM convolution
             of csrc/conv_mma.cuh behind pf_conv_circ, pf_faedt_conv, pf_conv2d_nhwc and pf_hnet_conv; * is the
             convolution with the layer's own padding). ReLU is 1-Lipschitz and needs no factor. The deepest K any model
             passes is HorizonNet's first ConvCompressH, 9 * 2048 = 18432: sqrt(K) * 2^-24 = 8.1e-6, and ten times that
             rounds to the same power of two, 2^-14 (7.5x there, 9.5x at the tap-GEMM's 9 * 1280).

Every function here runs on whichever device its inputs live on (the CPU tests use the same code at small sizes).
"""
from __future__ import annotations

import math

import torch

GEMM_REL = 2.0 ** -14
ACT_LIP = 1.13          # max |d/dx| of erf-GELU (1.129) and of SiLU (1.100)
LN_SLACK = 2.0 ** -8
OUT_FLOOR = 2.0 ** -24
FMHA_FLOOR = 2.0 ** -20

ACT_NONE, ACT_SILU, ACT_GELU, ACT_GEGLU = 0, 1, 2, 3  # PF_ACT_*


def ulp_out(ref: torch.Tensor, out_dtype: torch.dtype) -> torch.Tensor:
    """Rounding of the fp32 result to the output type (0 for fp32 outputs)."""
    if out_dtype == torch.float32:
        return torch.zeros_like(ref)
    rel = 2.0 ** -10 if out_dtype == torch.float16 else 2.0 ** -7
    return torch.clamp(rel * ref.abs(), min=OUT_FLOOR)


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _silu(x):
    return x * torch.sigmoid(x)


def tap_gemm_ref(A, B, out_rows: int, out_dtype: torch.dtype, *, M: int, Kc: int, taps=(0,), bias=None, rowbias=None,
                 rows_per_group: int = 0, residual=None, act: int = ACT_NONE, image_map=None, scatter=None,
                 ln_eps=None, geglu_bn: int = 0):
    """(ref, bound), both fp64 [out_rows, n_out]; rows the contract does not write are NaN in both.

    Arguments mean what they mean to ops.gemm_taps; `residual` is the [out_rows, n_out] view the kernel reads,
    `ln_eps` makes this a LayerNorm consumer (A normalised over its Kc columns, B holding the gamma-scaled weights),
    `geglu_bn` is the tile width the GEGLU weights were packed for."""
    dev = A.device
    A64, B64 = A.double(), B.double()
    a_rows, N = A.shape[0], B.shape[0]
    m = torch.arange(M, device=dev)
    acc = torch.zeros((M, N), dtype=torch.float64, device=dev)
    mag = torch.zeros_like(acc)
    for t, off in enumerate(taps):
        idx = m + int(off)
        inside = (idx >= 0) & (idx < a_rows)
        a = A64[idx.clamp(0, a_rows - 1), :Kc] * inside[:, None]
        if ln_eps is not None:
            assert len(taps) == 1
            a = (a - a.mean(1, keepdim=True)) / torch.sqrt(a.var(1, unbiased=False, keepdim=True) + ln_eps)
        w = B64[:, t * Kc:(t + 1) * Kc]
        acc += a @ w.T
        mag += a.abs() @ w.abs().T
    err = (GEMM_REL + (LN_SLACK if ln_eps is not None else 0.0)) * mag
    if image_map is not None:
        Hm, Wm, i0, j0, Hout, Wout = image_map
        sy, sx, oa, ob = scatter if scatter is not None else (1, 1, 0, 0)
        img, r = m // (Hm * Wm), m % (Hm * Wm)
        i, j = r // Wm, r % Wm
        valid = (i >= i0) & (i < i0 + Hout) & (j >= j0) & (j < j0 + Wout)
        orow = ((img * Hout + i - i0) * sy + oa) * (Wout * sx) + (j - j0) * sx + ob
        group = img
    else:
        valid = torch.ones(M, dtype=torch.bool, device=dev)
        orow = m
        group = m // rows_per_group if rowbias is not None else m
    if bias is not None:
        acc += bias.double()
        err += GEMM_REL * bias.double().abs()
    if rowbias is not None:
        rb = rowbias.double()[group.clamp(max=rowbias.shape[0] - 1)]
        acc += rb
        err += GEMM_REL * rb.abs()
    if act in (ACT_SILU, ACT_GELU):
        acc = (_silu if act == ACT_SILU else _gelu)(acc)
        err = ACT_LIP * err
    elif act == ACT_GEGLU:
        half = geglu_bn // 2
        va, vg = acc.reshape(M, N // geglu_bn, 2, half).unbind(2)
        ea, eg = err.reshape(M, N // geglu_bn, 2, half).unbind(2)
        gg = _gelu(vg)
        acc = (va * gg).reshape(M, N // 2)
        err = (ea * (gg.abs() + ACT_LIP * eg) + ACT_LIP * va.abs() * eg).reshape(M, N // 2)
    n_out = acc.shape[1]
    ref = torch.full((out_rows, n_out), float("nan"), dtype=torch.float64, device=dev)
    bound = torch.full_like(ref, float("nan"))
    ref[orow[valid]] = acc[valid]
    bound[orow[valid]] = err[valid]
    if residual is not None:
        res = residual.double()
        ref += res
        bound += GEMM_REL * res.abs()
    return ref, bound + ulp_out(ref, out_dtype)


def merge(parts):
    """Combine (ref, bound) pairs of calls that write disjoint rows of one output (the upsample phases)."""
    ref, bound = parts[0]
    for r, b in parts[1:]:
        ref = torch.where(torch.isnan(ref), r, ref)
        bound = torch.where(torch.isnan(bound), b, bound)
    return ref, bound


def conv_ref(x, w, bias, *, Cout: int, kh: int, kw: int, stride_h: int, stride_w: int, ph: int, pw: int, circ: bool,
             relu: bool, out_dtype: torch.dtype, residual=None, res_before_relu: bool = False, Ho: int | None = None,
             Wo: int | None = None, out_rows: int | None = None, out_ld: int | None = None, out_off: int = 0,
             chunk: int = 0):
    """(ref, bound) of one conv_mma launch, both fp64 [out_rows, out_ld] (out_rows >= M = B * Ho * Wo); every element
    the launch must not write (rows past M, columns outside [out_off, out_off + Cout)) is NaN in both.

    x: the channels-last fp16 input [B, H, W, Cin_pad] (padded channels included); w: the packed fp16 weight
    [kh * kw][Cin_pad][Cw] (tap-major ky, kx; columns past Cout are ignored); bias: fp32 [>= Cout]; residual: fp16
    [M, Cout] rows (the kernel reads it with row stride Cout). Input row iy = oy * stride_h + ky - ph reads zero outside
    [0, H); input column ix = ox * stride_w + kx - pw reads zero outside [0, W), or x[..., ix mod W] when circ (corners
    zero). Ho / Wo default to the symmetric-padding output size; the stride-2 data-gradient phases pass their own.
    Epilogue: + bias, then ReLU, then + residual; with res_before_relu the residual goes before the ReLU.
    `chunk` > 0 computes that many images at a time (full-resolution layers on the device)."""
    B, H, W, cin = x.shape
    taps, cin_w, _cw = w.shape
    assert taps == kh * kw and cin_w == cin, (tuple(x.shape), tuple(w.shape), kh, kw)
    Ho = (H + 2 * ph - kh) // stride_h + 1 if Ho is None else Ho
    Wo = (W + 2 * pw - kw) // stride_w + 1 if Wo is None else Wo
    M = B * Ho * Wo
    out_rows = M if out_rows is None else out_rows
    out_ld = Cout if out_ld is None else out_ld
    dev = x.device
    wt = w.double().reshape(kh, kw, cin, -1).permute(3, 2, 0, 1)[:Cout].contiguous()
    wa = wt.abs()
    rows_end, cols_end = (Ho - 1) * stride_h + kh - ph, (Wo - 1) * stride_w + kw - pw  # exclusive, in input coordinates
    accs, mags = [], []
    for b0 in range(0, B, chunk or B):
        xb = x[b0:b0 + (chunk or B)].double().permute(0, 3, 1, 2)
        if circ:
            xb = xb[..., torch.arange(-pw, cols_end, device=dev) % W]
        else:
            xb = torch.nn.functional.pad(xb, (pw, max(0, cols_end - W)))
        xb = torch.nn.functional.pad(xb, (0, 0, ph, max(0, rows_end - H)))
        conv = lambda a, f: torch.nn.functional.conv2d(a, f, stride=(stride_h, stride_w))[:, :, :Ho, :Wo]
        accs.append(conv(xb, wt).permute(0, 2, 3, 1).reshape(-1, Cout))
        mags.append(conv(xb.abs(), wa).permute(0, 2, 3, 1).reshape(-1, Cout))
        del xb
    acc, mag = torch.cat(accs), torch.cat(mags)
    bias64 = bias[:Cout].double().to(dev)
    acc += bias64
    err = GEMM_REL * (mag + bias64.abs())
    res = None if residual is None else residual.reshape(M, Cout).double()
    if res is not None:
        err += GEMM_REL * res.abs()
        if res_before_relu:
            acc += res
    if relu:
        acc = acc.clamp_min(0.0)
    if res is not None and not res_before_relu:
        acc += res
    ref = torch.full((out_rows, out_ld), float("nan"), dtype=torch.float64, device=dev)
    bound = torch.full_like(ref, float("nan"))
    ref[:M, out_off:out_off + Cout] = acc
    bound[:M, out_off:out_off + Cout] = err
    return ref, bound + ulp_out(ref, out_dtype)


def fmha_ref(q, k, v, *, heads: int, head_dim: int, scale: float, bias=None, chunk: int = 1024):
    """(ref, P @ |V|), fp64 [B, Lq, heads * head_dim]; q / k / v: [B, L, >= heads * head_dim] views; bias fp32 [Lq, Lk] or
    [B or 1, Lq, Lk]. Chunked over batches, heads and queries (at most chunk x Lk scores at a time)."""
    B, Lq, Lk, d = q.shape[0], q.shape[1], k.shape[1], head_dim
    scale = float(torch.tensor(scale, dtype=torch.float32))  # the kernel receives it as a float
    ref = torch.empty((B, Lq, heads * d), dtype=torch.float64, device=q.device)
    pv = torch.empty_like(ref)
    for b in range(B):
        bb = None
        if bias is not None:
            bb = bias if bias.dim() == 2 else bias[b if bias.shape[0] > 1 else 0]
        for h in range(heads):
            cols = slice(h * d, (h + 1) * d)
            kh, vh = k[b, :, cols].double(), v[b, :, cols].double()
            for q0 in range(0, Lq, chunk):
                rows = slice(q0, min(q0 + chunk, Lq))
                s = (q[b, rows, cols].double() @ kh.T) * scale
                if bb is not None:
                    s = s + bb[rows].double()
                p = torch.softmax(s, -1)
                ref[b, rows, cols] = p @ vh
                pv[b, rows, cols] = p @ vh.abs()
    return ref, pv


def fmha_bound(ref, pv, dtype: torch.dtype):
    u = 2.0 ** -11 if dtype == torch.float16 else 2.0 ** -8
    return 2 * u * pv + u * ref.abs() + FMHA_FLOOR


def worst_ratio(got, ref, bound) -> float:
    """max |got - ref| / bound over the elements the contract writes; every other element of `got` must still hold the
    NaN it was filled with (a kernel that writes outside its rows fails here). A NaN where a value is due counts as inf."""
    got = got.double()
    written = ~torch.isnan(ref)
    stray = int((~torch.isnan(got[~written])).sum())
    assert stray == 0, f"{stray} elements written outside the contract's rows"
    r = ((got - ref).abs() / bound)[written]
    return float(torch.nan_to_num(r, nan=math.inf).max())
