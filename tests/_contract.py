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
  cpattn gather  |got - ref| <= 2^-21 * (sum_t w_t |x_t| + 1) + ulp_out(ref)  (pf_cpattn_gather, one key element: four
             bilinear taps x_t with weights w_t, plus sin or cos of the fp32 product xy_rel * f). The weights carry <= 3
             fp32 roundings (two subtractions, one product), the fma chain over the four taps <= 4, the PE add 1: 8 units
             of 2^-24 = 2^-21 of the tap magnitude. sincosf is within 2 ulp of a value <= 1, 2^-22, under the "+ 1".
             A masked key must be exactly zero (its bound is the smallest positive double).
  cpattn stats   |got - ref| <= n * 2^-24 * (sum |k|, sum k^2) + 2^-60, n = 16 * ceil(C / 512) + 6, against the fp64
             (sum, sum of squares) of the STORED 16-bit key row k: each lane adds 16 rounded values per 512 channels in
             fp32, then five shuffle-tree adds.
  cpattn attn    |got - ref| <= 2^-17 * (1 + A) * (P @ |V|) + ulp_out(ref)  (pf_cpattn_attn, one query against its 18
             keys per 32-wide head). The kernel keeps P in fp32, so no 16-bit term enters before the output rounding.
             A = scale * max_s sum_d |q_d k_sd| bounds the logits: the fp32 dot product errs by <= 33 units of 2^-24 * A
             and a logit error e moves P by a relative 2e (66 A units); expf (2), the 18-term denominator (18), the
             reciprocal and its product (2) and the 18-term fma chain of P V (18) add 40 units. 64 (1 + A) units is
             2^-18 (1 + A); 2^-17 leaves a factor of two.

The normalisation and sampler kernels (csrc/norm.cu, csrc/elementwise.cu), u = 2^-24:
  gn stats   (pf_groupnorm_stats, the statistics launch of pf_gn_prep) mean and rstd of each (image, group) over the image
             circularly extended by circ_stats columns, a duplicated column weighted w = 2 (3 when both seams cover it).
             w x and w x^2 are exact in fp32 (a 16-bit x has <= 11 significant bits, w <= 2 bits), so only additions
             round: a thread adds ceil(ceil(HW / slabs) / ppi) pixels, the CTA adds its ppi lanes, then cpg channels, all
             in fp32; slabs are added in fp64. With n = ceil(ceil(HW / slabs) / ppi) + ppi + cpg, S1 = sum w |x| and
             S2 = sum w x^2 over `count` = H (W + 2 circ_stats) cpg terms:
               |dmean| <= n u S1 / count + u |mean|                       (the fp32 store adds the last term)
               dvar    <= n u S2 / count + 2 |mean| n u S1 / count <= 3 n u S2 / count   ((S1 / count)^2 <= S2 / count)
               |drstd| / rstd <= 1/2 * 3 n u (S2 / count) / (var + eps) + 2u   (fp64 sqrt and the fp32 store)
             This is the one-pass form the kernel computes; for a near-constant group the bound is vacuous by design.
  gn apply   (pf_conv_prep / the apply launch of pf_gn_prep) y = x sc + sh with sc = fl(rstd gamma), sh = fl(beta - mean sc)
             from the fp32 (mean, rstd) the launch reads: four roundings of the x term, four of the mean term and two
             of beta: |dy| <= 4u ((|x| + |mean|) rstd |gamma| + |beta|) (sh carries the cancellation, so the bound is
             not on |x - mean|). SiLU (silu_f: ex2.approx, rcp.approx, <= 2 ulp each, the argument's product and the
             final product) adds 1.13 |dy| + 2^-20 (1 + |y|) |silu(y)|. Halo and phase padding, the raw concatenation
             and conv_prep without statistics are exact.
  layernorm  (pf_layernorm) f = fl(x + pe), then the two-pass fp32 form in one warp: each lane adds 8 ceil(C / 256)
             values, then 5 shuffles: n = 8 ceil(C / 256) + 5, dmean <= n u sum|f| / C + u |mean|; the squares carry
             (n + 4) u of var (d = f - mean rounds, d^2 rounds, the sum, / C) plus the (dmean)^2 / var the shifted centre
             adds, + eps rounds once, rsqrtf is within 2 ulp (4u): drstd / rstd <= 1/2 (n + 5) u var / (var + eps) +
             dmean^2 / (2 (var + eps)) + 4u. Output: |do| <= |gamma| rstd (dmean + |f - mean| (3u + drstd / rstd)) +
             u |o|, then the 16-bit store.
  row stats  (pf_embed_tokens) the row is exactly fl16(fl32(tok[id] + pos[t % L])); its (sum, sum of squares) as the
             cpattn stats with n = 2 ceil(C / 64) + 5 (a lane adds a pair, then the pair to its sum, per 64 channels).
  cfg ddim   (pf_cfg_ddim_step[_dev]) e = eu + g (ec - eu), v = c_x x + c_eps e in fp32, stored at column (col + roll) mod
             W: |dv| <= 2u (|c_x x| + 2 |c_eps e| + 2 |c_eps g (ec - eu)| + |v|) (first order, doubled).
  timestep   (pf_timestep_embed) [cos(t f_i) | sin(t f_i)], f_i = 10000^(-i / half). The fp32 argument t f_i carries
             logf (2u), two products (2u) and expf (4u) of ln f_i, then the product by t: |darg| <= u (4 |ln f_i| + 5)
             |t f_i|; cosf / sinf add 2 ulp of a value <= 1 (2^-22).

The remaining element-wise kernels of csrc/elementwise.cu, u = 2^-24:
  conv_in    (pf_conv_in) 3 x 3, pad 1 convolution of fp32 NCHW x with fp32 weights: rows zero-padded, columns
             zero-padded or wrapped (circ). A thread seeds its fp32 accumulator with the bias and adds the K = 9 Cin taps
             by fmaf, one rounding each, so the sequential-FMA bound holds: |dacc| <= gamma_K (|b| + sum |x| |w|),
             gamma_K = K u / (1 - K u). SiLU adds what it adds in gn apply (1.13 |dacc| + 2^-20 (1 + |y|) |silu(y)|),
             then the 16-bit store one output ulp. An element whose terms and bias are all zero (the zero-padded output
             channels) must be exactly zero.
  softmax    (pf_softmax_rows) p_j = e_j / sum e, e_j = expf(fl(fl(x_j - m) scale)), m the row's unscaled maximum (exact).
             The argument carries two roundings, an absolute error of 2u |a_j| (a_j = (x_j - m) scale <= 0), which moves
             e_j by a relative 2u |a_j|: large only where e_j = e^{a_j} is tiny. expf adds 2 ulp (4u; build.py uses
             no fast-math). The denominator adds positive terms: a thread adds ceil(cols / 256) of them, then a 5-level
             shuffle tree and the 8 warp partials in series, so dS <= sum_j e_j (2u |a_j| + 4u) + n_S u S with
             n_S = ceil(cols / 256) + 13. The reciprocal and the product round once each: |dp_j| <= p_j (2u |a_j| + 4u +
             dS / S + 2u), then the 16-bit store.
  gaussian   (pf_gaussian_sample) z = (mean + exp(0.5 clamp(logvar, -30, 20)) eps) scale; 0.5 lv is exact, expf 4u, the
             product, the sum and the scale one rounding each: |dz| <= |scale| (5u |t| + u |mean + t|) + u |z|,
             t = std eps. The clamp propagates NaN like torch.clamp: a NaN mean or logvar gives a NaN z.
  mse        (pf_mse_loss) sum (a - b)^2 / n over a fixed partition of 296 chunks of ceil(n / 296) elements. d = a - b
             rounds (2u of d^2), a thread's fmaf chain adds ceil(chunk / 256) terms, a 5-level shuffle tree and the 8
             warp partials in series follow, all on non-negative values: n_M = ceil(chunk / 256) + 14 and each chunk's
             fp32 sum errs by <= n_M u of its sum. The 296 partials are added and divided by n in fp64 (2^-50, under the
             slack), then rounded to fp32: |dloss| <= n_M u sum d^2 / n + u loss.

The FAED training kernels (csrc/faed_train.cu), u = 2^-24, f = fl32(inv_n / S) (inv_n / S is exact in fp64: S is a
power of two; the kernels round it to fp32 once):
  wgrad part  (pf_faedt_wgrad's fp32 partial of one pixel chunk, in ws [nch][k^2][Cin][Cdy]) the chunk's
             sum_p x[p (+) tap, ci] dy[p, co] on mma.sync m16n8k16 with an fp32 accumulator: fp16 x fp16 products are
             exact in fp32, so only the accumulation rounds. One k-step adds 16 products to the accumulator; the tensor
             core aligns them to the largest exponent and truncates, once when it sums the products and once when it
             adds the accumulator, each time losing < 2^-23 of a magnitude <= the chunk's sum_p |x| |dy| so far.
             Truncation errors all have the same sign, so they add linearly: |dpart| <= ceil(chunk / 16) 2^-22
             sum_chunk |x| |dy|. (The convolution core's 2^-14 is the statistical sqrt(K) form; a partial sums one chunk
             only, so the worst case stays small: 326 k-steps, 7.8e-5, at the largest chunk the models make, 5216 pixels
             of the first layer at 4 x 512 x 1024.) The dY column sums for
             db (ws [nch][Cdy] after the partials) are one thread's fp32 chain over the chunk: chunk u sum_chunk |dy|.
  wgrad reduce  given the kernel's own partials, dw = fl(fl(sum_c part_c) f) summed in chunk order:
             |dw - f sum_c part_c| <= nch u f sum_c |part_c| + u |dw|; db the same over the column sums.
  wgrad      end to end against fp64 f sum_p x dy: the two bounds above with sum_c |part_c| <= sum |x| |dy|.
  bn stats   (pf_faedt_bn_stats) chunks of row_chunk(P) rows, L = 256 / C lanes per channel, each lane a Welford
             chain over n_w <= ceil(chunk / L) rows, then L - 1 Chan merges into lane 0, then nch Chan merges. The chunk
             counts are exact integers. A Welford update rounds mu + d / k with error rho <= 3u A (A = max |z|: the
             mean is large against the spread, so A, not the spread, sets the scale), and a rounding at update j moves
             the lane mean by rho j / k afterwards: |dmean_lane| <= 3u A (n + 1) / 2. The same rounding moves M2 by
             rho j (2 |mu_n - mu_j| + |mu_j - mu_{j-1}|) to first order (the later updates re-centre on the perturbed
             mean); the products and sums add (n_w + 3) u M2. A Chan merge with delta = mean_b - mean_a and weight
             w = n_a n_b / n_ab rounds the mean by 4u A and M2 by 2u (M2_a + M2_b + delta^2 w) + 4u delta^2 w, and
             carries the means' errors into M2 as 2 |delta| w (dmean_a + dmean_b). The reference runs the kernel's
             partition and merge order in fp64 and sums these terms. invstd = 1 / sqrt(M2 / n + eps): half the
             relative error of M2 / n over var + eps, plus 4u (division, eps add, sqrtf, reciprocal); the unbiased
             variance M2 / (n - 1) adds 2u. n is an fp32 count; past 2^24 it rounds by u. pending must be bit-equal
             to stats rows 0 and 2.
  bn apply   (pf_faedt_bn_apply) given the launch's fp32 stats: (z - mean), * invstd, * gamma, + beta each round once:
             |dy| <= 3u |z - mean| invstd |gamma| + u |y|; ReLU is 1-Lipschitz; + residual rounds u |out|; fp16 store.
  bn bwd     (pf_faedt_bn_bwd) g' = g (mask > 0) with the mask the STORED fp16 ReLU output, xhat = (z - mean) invstd from
             the launch's fp32 stats (2u |xhat|). Per chunk (sum g', sum g' xhat) as the statistics' partition: n_w + L
             additions, (n_w + L) u sum |g'| and (n_w + L + 3) u sum |g' xhat|; nch more additions merge them; sums =
             the merged sums / P (one more u), dgamma = f sum g' xhat, dbeta = f sum g' (one more u). Given the launch's
             sums, dz = gamma invstd (g' - s0 - xhat s1): 4u |gamma invstd| (|g'| + |s0| + 2 |xhat s1|) + fp16 store.
  upsample   (pf_faedt_upsample) the weights are 0, 0.25, 0.75 or 1 and their products; w x is exact in fp32 and the two
             lerps round <= 4 times: 4u (sum |w| |x|) + fp16 store. The backward gathers <= 4 x 4 outputs: <= 9 roundings
             of the adjoint's magnitude, 10u (W^T |g|) + fp16 store.
  loss       (pf_faedt_loss) pred = tanhf(o): <= 2 ulp of the fp64 tanh (2^-22 |pred| + 2^-149). loss = mean |pred - t|
             over 3 B H W: a thread adds 3 ceil(M / 262144) terms (1024 x 256 threads grid-stride), an 8-level tree, the
             final kernel adds 4 partials per thread and another 8-level tree: n = 3 ceil(M / 262144) + 20;
             |dloss| <= (n u sum |d| + 2^-22 sum |pred| + u sum |d|) / count + u loss. seed = fl16(sign(d) (1 - pred^2) S)
             with the kernel's pred: |seed - sign (1 - pred^2) S| <= 2^-11 |.| + 2u S + 2^-25 (fp32 products, the fp16
             rounding); where |d| is within pred's error the sign is not defined and seed may be 0 or either sign,
             except o = 0 against a zero target: tanhf(0) = 0 exactly, so d = 0 and sign(0) = 0 give a zero seed.
             Channels 3..15 are exactly zero.
  exact      pf_faedt_prep, pf_faedt_interleave and pf_faedt_pack (forward layout, stride-1 flipped kernel, the four
             stride-2 phase kernels, zero padding) move or round values once: bit-equal.
  adam       (pf_faedt_adam) torch.optim.Adam(foreach=False)'s five fp32 kernels, each rounding once: bit-equal.

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


CP_SLOTS = 18
GATHER_REL = 2.0 ** -21
CPATTN_REL = 2.0 ** -17
EXACT = torch.finfo(torch.float64).tiny  # bound of an element that must be exactly its reference


def cpattn_gather_ref(x, B: int, m: int, h: int, w: int, C: int, G: int, pos, mask, freq, out_dtype: torch.dtype,
                      neighbours=(-1, 1)):
    """(ref, bound), fp64 [B * m * h * w * 18, C]: the key rows pf_cpattn_gather writes.

    x: the [B * m * h * w, >= C] 16-bit tokens; pos fp32 [G, m, h * w, 18, 4] (grid_sample position in the neighbour's
    map, xy_rel); mask uint8 [G, m, h * w, 18]; freq fp32 [C / 4]; G = 1 (every batch element shares the tables) or B.
    Row ((b * m + i) * P + q) * 18 + s samples view i - 1 (s < 9) or i + 1 (ring order) of batch element b bilinearly
    with zero padding (grid_sample, align_corners=True, at the unnormalised position) and adds
    [sin(x f), sin(y f), cos(x f), cos(y f)] of the fp32-rounded products xy_rel * f, evaluated in fp64.
    `neighbours` are the view offsets of slots 0-8 and 9-17."""
    P = h * w
    dev = x.device
    xv = x[:, :C].reshape(B, m, P, C)
    f32 = freq.float().reshape(-1)
    N = C // 4
    ref = torch.empty((B, m, P, CP_SLOTS, C), dtype=torch.float64, device=dev)
    bound = torch.empty_like(ref)
    side = torch.arange(CP_SLOTS, device=dev) < 9
    for b in range(B):
        g = 0 if G == 1 else b
        for i in range(m):
            p = pos[g, i].double()                                             # [P, 18, 4]
            fx, fy = torch.floor(p[..., 0]), torch.floor(p[..., 1])
            ax, ay = p[..., 0] - fx, p[..., 1] - fy
            wts = ((1 - ax) * (1 - ay), ax * (1 - ay), (1 - ax) * ay, ax * ay)  # nw, ne, sw, se
            acc = torch.zeros((P, CP_SLOTS, C), dtype=torch.float64, device=dev)
            mag = torch.zeros_like(acc)
            for t in range(4):
                xx, yy = fx.long() + (t & 1), fy.long() + (t >> 1)
                inside = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
                idx = (yy.clamp(0, h - 1) * w + xx.clamp(0, w - 1))            # [P, 18]
                left = xv[b, (i + neighbours[0]) % m].double()[idx]            # [P, 18, C]
                right = xv[b, (i + neighbours[1]) % m].double()[idx]
                val = torch.where(side[None, :, None], left, right)
                wt = (wts[t] * inside)[..., None]
                acc += wt * val
                mag += wt * val.abs()
            rel = pos[g, i, :, :, 2:].float()                                  # [P, 18, 2]
            arg = (rel[..., :, None] * f32).double()                           # fp32 products, [P, 18, 2, N]
            pe = torch.cat([arg.sin(), arg.cos()], -2).reshape(P, CP_SLOTS, 4 * N)
            live = mask[g, i].bool()[..., None]
            ref[b, i] = torch.where(live, acc + pe, 0.0)
            bound[b, i] = GATHER_REL * (mag + 1.0)
    ref = ref.reshape(-1, C)
    bound = bound.reshape(-1, C) + ulp_out(ref, out_dtype)
    masked = torch.stack([~mask[0 if G == 1 else b].bool() for b in range(B)]).reshape(-1)
    bound[masked] = EXACT
    return ref, bound


def _row_sums(rows, n: int):
    """(ref, bound), fp64 [rows, 2]: (sum, sum of squares) of 16-bit rows summed in fp32 chains of n additions."""
    k = rows.double()
    ref = torch.stack([k.sum(1), (k * k).sum(1)], 1)
    bound = n * U * torch.stack([k.abs().sum(1), (k * k).sum(1)], 1) + 2.0 ** -60
    return ref, bound


def cpattn_stats_ref(keys, C: int):
    """(ref, bound), fp64 [rows, 2]: (sum, sum of squares) of each stored 16-bit key row (pf_cpattn_gather's stats)."""
    return _row_sums(keys[:, :C], 16 * -(-C // 512) + 6)


def cpattn_attn_ref(q, kv, C: int, scale: float, out_dtype: torch.dtype, chunk: int = 4096):
    """(ref, bound), fp64 [T, C]: pf_cpattn_attn, out[t, head] = softmax_s(q_t,head . k_ts,head * scale) v_ts,head over
    the 18 key rows t * 18 + s of kv (K in columns [0, C), V in [C, 2C)), heads of width 32. Chunked over tokens."""
    T, H = q.shape[0], C // 32
    scale = float(torch.tensor(scale, dtype=torch.float32))
    ref = torch.empty((T, C), dtype=torch.float64, device=q.device)
    bound = torch.empty_like(ref)
    for t0 in range(0, T, chunk):
        t1 = min(T, t0 + chunk)
        qh = q[t0:t1, :C].double().reshape(-1, H, 1, 32)
        kvc = kv[t0 * CP_SLOTS:t1 * CP_SLOTS].double()
        k = kvc[:, :C].reshape(-1, CP_SLOTS, H, 32).transpose(1, 2)          # [t, H, 18, 32]
        v = kvc[:, C:2 * C].reshape(-1, CP_SLOTS, H, 32).transpose(1, 2)
        s = (qh @ k.transpose(-1, -2)) * scale                                  # [t, H, 1, 18]
        a = ((qh.abs() @ k.abs().transpose(-1, -2)) * scale).amax(-1, keepdim=True)
        p = torch.softmax(s, -1)
        ref[t0:t1] = (p @ v).reshape(-1, C)
        bound[t0:t1] = (CPATTN_REL * (1.0 + a) * (p @ v.abs())).reshape(-1, C)
    return ref, bound + ulp_out(ref, out_dtype)


U = 2.0 ** -24
SILU_REL = 2.0 ** -20


def _f32(v: float) -> float:
    """A Python float as the kernel receives it (a C float argument)."""
    return float(torch.tensor(v, dtype=torch.float32))


def gn_partition(entry: str, H: int, W: int, C: int):
    """(slabs, ppi) of the statistics launch: pf_gn_prep cuts an image into <= 32 slabs of >= 16 pixels with 512-thread
    CTAs, pf_groupnorm_stats into <= 64 with 256-thread CTAs; a CTA covers ppi pixels per step (C / 8 lanes each)."""
    threads, cap = (512, 32) if entry == "pf_gn_prep" else (256, 64)
    return min(max(H * W // 16, 1), cap), max(1, threads // (C // 8))


def gn_operand(g, N: int, H: int, W: int, C: int, groups: int, dtype: torch.dtype, seam: int = 2):
    """Channels-last tokens [N * H * W, C] that make GroupNorm indexing bugs visible: each (image, group) has its own
    scale s in [0.5, 2] and offset in [-4 s, 4 s], and the `seam` columns at either edge are shifted by +s (left) and
    -s (right), so the two sides of the circular seam differ."""
    cpg = C // groups
    s = (0.5 + 1.5 * torch.rand(N, 1, 1, groups, 1, generator=g))
    off = s * (8 * torch.rand(N, 1, 1, groups, 1, generator=g) - 4)
    x = torch.randn(N, H, W, groups, cpg, generator=g) * s + off
    if seam:
        x[:, :, :min(seam, W)] += s
        x[:, :, max(0, W - seam):] -= s
    return x.reshape(N * H * W, C).to(dtype)


def gn_stats_ref(x, N: int, H: int, W: int, groups: int, circ_stats: int, eps: float, partition):
    """(ref, bound), fp64 [N, groups, 2]: GroupNorm (mean, rstd) of x [N * H * W, C] (the concatenation, channels
    last) over each image circularly extended by circ_stats columns; `partition` = gn_partition(...)."""
    slabs, ppi = partition
    C = x.shape[1]
    cpg, hw = C // groups, H * W
    n = -(-(-(-hw // slabs)) // ppi) + ppi + cpg
    col = torch.arange(W, device=x.device)
    w = (1.0 + (col < circ_stats).double() + (col >= W - circ_stats).double())[None, :, None, None]
    count = H * (W + 2 * circ_stats) * cpg
    eps = _f32(eps)
    ref = torch.empty((N, groups, 2), dtype=torch.float64, device=x.device)
    bound = torch.empty_like(ref)
    for b in range(N):
        xb = x[b * hw:(b + 1) * hw].double().reshape(H, W, groups, cpg)
        s1 = (w * xb).sum((0, 1, 3))
        a1 = (w * xb.abs()).sum((0, 1, 3))
        s2 = (w * xb * xb).sum((0, 1, 3))
        mean = s1 / count
        var = (w * (xb - mean[None, None, :, None]) ** 2).sum((0, 1, 3)) / count
        rstd = 1.0 / torch.sqrt(var + eps)
        ref[b, :, 0], ref[b, :, 1] = mean, rstd
        bound[b, :, 0] = n * U * a1 / count + U * mean.abs()
        bound[b, :, 1] = rstd * (1.5 * n * U * (s2 / count) / (var + eps) + 2 * U)
        del xb
    return ref, bound


def _layout(t, circ: int, up: int, phases: int, halo: int, fill: float):
    """[N, H, W, C] -> the pf_conv_prep layout [phases * N * Ho * Wo, C], `fill` in the halo / phase padding."""
    W = t.shape[2]
    if circ:
        t = t[:, :, (torch.arange(W + 2 * circ, device=t.device) - circ) % W]
    if up > 1:
        t = t.repeat_interleave(up, 1).repeat_interleave(up, 2)
    pad = 1 if phases == 4 else halo
    t = torch.nn.functional.pad(t, (0, 0, pad, pad, pad, pad), value=fill)
    if phases == 4:
        t = torch.stack([t[:, py::2, px::2] for py in (0, 1) for px in (0, 1)])
    return t.reshape(-1, t.shape[-1])


def gn_apply_ref(x, N: int, H: int, W: int, mean_rstd, gamma, beta, *, act: int, circ: int, up: int, phases: int,
                 halo: int, out_dtype: torch.dtype):
    """(ref, bound), fp64 [phases * N * Ho * Wo, C]: pf_conv_prep (and pf_gn_prep's apply launch) on x [N * H * W, C]
    with the fp32 mean_rstd [N, groups, 2] the launch reads (None: no normalisation, the layout alone is exact).
    Halo and phase-padding positions must be exactly zero."""
    C = x.shape[1]
    y = x.double().reshape(N, H, W, C)
    if mean_rstd is None:
        assert act == ACT_NONE
        dy = torch.full_like(y, EXACT)
    else:
        cpg = C // mean_rstd.shape[1]
        mr = mean_rstd.double().repeat_interleave(cpg, 1)[:, None, None]     # [N, 1, 1, C, 2]
        mean, rstd = mr[..., 0], mr[..., 1]
        g, b = gamma.double(), beta.double()
        dy = 4 * U * ((y.abs() + mean.abs()) * rstd * g.abs() + b.abs())
        y = (y - mean) * rstd * g + b
        if act == ACT_SILU:
            s = _silu(y)
            dy = ACT_LIP * dy + SILU_REL * (1.0 + y.abs()) * s.abs()
            y = s
        dy = dy + ulp_out(y, out_dtype)
    return _layout(y, circ, up, phases, halo, 0.0), _layout(dy, circ, up, phases, halo, EXACT)


def layernorm_ref(x, pe, gamma, beta, eps: float, out_dtype: torch.dtype, chunk: int = 1 << 15):
    """(ref, bound), fp64 [T, C]: pf_layernorm, LayerNorm(fl32(x[t] + pe[t % pe_rows])) * gamma + beta for the rows of
    the 16-bit view x [T, C] (any row stride); pe fp32 [pe_rows, C] or None."""
    T, C = x.shape
    n = 8 * -(-C // 256) + 5
    eps = _f32(eps)
    g, b = gamma.double(), beta.double()
    ref = torch.empty((T, C), dtype=torch.float64, device=x.device)
    bound = torch.empty_like(ref)
    for t0 in range(0, T, chunk):
        t1 = min(T, t0 + chunk)
        f = x[t0:t1].float()
        if pe is not None:
            f = f + pe[torch.arange(t0, t1, device=x.device) % pe.shape[0]]  # the fp32 add the kernel does
        f = f.double()
        mean = f.mean(1, keepdim=True)
        d = f - mean
        var = (d * d).mean(1, keepdim=True)
        rstd = 1.0 / torch.sqrt(var + eps)
        o = d * rstd * g + b
        dmean = n * U * f.abs().mean(1, keepdim=True) + U * mean.abs()
        rel = 0.5 * (n + 5) * U * var / (var + eps) + dmean ** 2 / (2 * (var + eps)) + 4 * U
        ref[t0:t1] = o
        bound[t0:t1] = g.abs() * rstd * (dmean + d.abs() * (3 * U + rel)) + U * o.abs() + ulp_out(o, out_dtype)
    return ref, bound


def row_stats_ref(tok, pos, ids, L: int, out_dtype: torch.dtype):
    """pf_embed_tokens -> (row [T, C] in out_dtype, exact: fl16(fl32(tok[id] + pos[t % L]))), then (ref, bound) fp64
    [T, 2] of the (sum, sum of squares) of that stored row."""
    T, C = ids.numel(), tok.shape[1]
    row = (tok[ids] + pos[torch.arange(T, device=ids.device) % L]).to(out_dtype)
    return (row, *_row_sums(row, 2 * -(-C // 64) + 5))


def cfg_ddim_ref(x, eps, coef, guidance: float, roll: int):
    """(ref, bound), fp64 shaped like x: pf_cfg_ddim_step[_dev] on x fp32 [..., W], eps [uncond | text] with 2 x.numel()
    elements, coef fp32 (c_x, c_eps) as the sampler's coef_table holds them; element (.., col) goes to column
    (col + roll) mod W."""
    W = x.shape[-1]
    xr = x.double().reshape(-1, W)
    eu, ec = eps.double().reshape(2, -1, W).unbind(0)
    g = _f32(guidance)
    cx, ce = (float(c) for c in coef.double().cpu())
    e = eu + g * (ec - eu)
    v = cx * xr + ce * e
    bound = 2 * U * ((cx * xr).abs() + 2 * (ce * e).abs() + 2 * (ce * g * (ec - eu)).abs() + v.abs()) + EXACT
    return v.roll(roll, -1).reshape(x.shape), bound.roll(roll, -1).reshape(x.shape)


def timestep_ref(t, dim: int, out_dtype: torch.dtype):
    """(ref, bound), fp64 [n, dim]: diffusers Timesteps(dim, flip_sin_to_cos=True, freq_shift=0) of t fp32 [n]."""
    half = dim // 2
    lnf = -math.log(10000.0) * torch.arange(half, dtype=torch.float64, device=t.device) / half
    arg = t.double()[:, None] * torch.exp(lnf)
    ref = torch.cat([arg.cos(), arg.sin()], 1)
    b = U * (4 * lnf.abs() + 5) * arg.abs() + 2.0 ** -22
    return ref, torch.cat([b, b], 1) + ulp_out(ref, out_dtype)


def conv_in_ref(x, w, b, circ: bool, act: int, out_dtype: torch.dtype):
    """(ref, bound), fp64 tokens [N * H * W, Cout]: pf_conv_in of the fp32 NCHW x [N, Cin, H, W] the kernel reads with
    fp32 weights w [Cout, Cin, 3, 3] and bias b [Cout] (None: no bias)."""
    W = x.shape[-1]
    xd = x.double()
    xd = xd[..., torch.arange(-1, W + 1, device=x.device) % W] if circ else torch.nn.functional.pad(xd, (1, 1))
    xd = torch.nn.functional.pad(xd, (0, 0, 1, 1))
    wd = w.double()
    acc = torch.nn.functional.conv2d(xd, wd)
    mag = torch.nn.functional.conv2d(xd.abs(), wd.abs())
    if b is not None:
        acc += b.double()[:, None, None]
        mag += b.double().abs()[:, None, None]
    K = w.shape[1] * 9
    err = K * U / (1 - K * U) * mag
    if act == ACT_SILU:
        s = _silu(acc)
        err = ACT_LIP * err + SILU_REL * (1.0 + acc.abs()) * s.abs()
        acc = s
    tok = lambda t: t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])
    ref, mag = tok(acc), tok(mag)
    bound = tok(err) + ulp_out(ref, out_dtype)
    return ref, torch.where(mag == 0, torch.full_like(bound, EXACT), bound)


def softmax_rows_ref(s, scale: float, out_dtype: torch.dtype):
    """(ref, bound), fp64 [rows, cols]: pf_softmax_rows of the fp32 logits s [rows, cols] (any row stride) at the fp32
    value of `scale`."""
    scale = _f32(scale)
    x = s.double()
    a = (x - x.amax(1, keepdim=True)) * scale
    e = torch.exp(a)
    S = e.sum(1, keepdim=True)
    n_s = -(-s.shape[1] // 256) + 13
    rel_e = 2 * U * a.abs() + 4 * U
    dS = (e * rel_e).sum(1, keepdim=True) + n_s * U * S
    p = e / S
    return p, p * (rel_e + dS / S + 2 * U) + ulp_out(p, out_dtype)


def gaussian_sample_ref(moments, ld: int, eps, L: int, scale: float):
    """(ref, bound), fp64 NCHW like eps [N, L, h, w]: pf_gaussian_sample of the channels-last fp32 moments rows of
    width ld ([mean (L) | logvar (L) | ...], N * h * w rows from moments' first element). NaN where mean or logvar is
    NaN (ref and bound)."""
    N, _, h, w = eps.shape
    rows = moments.as_strided((N * h * w, 2 * L), (ld, 1))
    m4 = rows.double().reshape(N, h, w, 2 * L).permute(0, 3, 1, 2)
    mean, logvar = m4[:, :L], m4[:, L:].clamp(-30.0, 20.0)
    scale = _f32(scale)
    t = torch.exp(0.5 * logvar) * eps.double()
    ref = (mean + t) * scale
    bound = abs(scale) * (5 * U * t.abs() + U * (mean + t).abs()) + U * ref.abs() + EXACT
    return ref, bound


MSE_CTAS = 296  # elementwise.cu: the fixed partition of pf_mse_loss


def mse_ref(a, b):
    """(ref, bound), fp64 scalars: pf_mse_loss of the fp32 a, b (any shape, n elements)."""
    n = a.numel()
    d2 = (a.double() - b.double()).reshape(-1) ** 2
    chunk = -(-n // MSE_CTAS)
    n_m = -(-chunk // 256) + 14
    ref = d2.sum() / n
    return ref, n_m * U * ref + U * ref + EXACT


def worst_ratio(got, ref, bound) -> float:
    """max |got - ref| / bound over the elements the contract writes; every other element of `got` must still hold the
    NaN it was filled with (a kernel that writes outside its rows fails here). A NaN where a value is due counts as inf."""
    got = got.double()
    written = ~torch.isnan(ref)
    stray = int((~torch.isnan(got[~written])).sum())
    assert stray == 0, f"{stray} elements written outside the contract's rows"
    r = ((got - ref).abs() / bound)[written]
    return float(torch.nan_to_num(r, nan=math.inf).max())


# ---- FAED training (csrc/faed_train.cu) -----------------------------------------------------------------------------

WGRAD_STAGE = 32  # pixels per wgrad pipeline stage
WGRAD_KSTEP = 2.0 ** -22  # per mma k-step, of the chunk's sum |x| |dy|


def faedt_factor(inv_n: float, scale: float) -> float:
    """f = fl32(inv_n / S), the factor every parameter gradient is reduced with."""
    return _f32(inv_n / scale)


def wgrad_chunk(P: int, taps: int, Cin: int, Cdy: int) -> int:
    """Pixels per wgrad chunk: at most 2^24 partial floats and at most ceil(P / 1024) chunks, a multiple of 32."""
    cap = max(1, (1 << 24) // (taps * Cin * Cdy))
    nch = min(-(-P // 1024), cap)
    chunk = -(-P // nch)
    return -(-chunk // WGRAD_STAGE) * WGRAD_STAGE


def wgrad_ref(x, dy, *, Ho: int, Wo: int, k: int, stride: int, pad: int, chunk: int | None = None):
    """pf_faedt_wgrad's partition of x fp16 [B, H, W, Cin] (rows outside [0, H) zero, columns circular) against dy fp16
    [B, Ho, Wo, Cdy]: dict of fp64 `part` / `part_bound` [nch, k^2, Cin, Cdy], `dbpart` / `dbpart_bound` [nch, Cdy],
    and the unscaled end-to-end sums `w` / `w_bound` [k^2, Cin, Cdy], `b` / `b_bound` [Cdy] (multiply by f)."""
    B, H, W, Cin = x.shape
    Cdy = dy.shape[-1]
    P, taps = B * Ho * Wo, k * k
    chunk = chunk or wgrad_chunk(P, taps, Cin, Cdy)
    nch = -(-P // chunk)
    dev = x.device
    padrows = nch * chunk - P
    d = torch.nn.functional.pad(dy.reshape(P, Cdy).double(), (0, 0, 0, padrows)).reshape(nch, chunk, Cdy)
    da = d.abs()
    p = torch.arange(P, device=dev)
    b, oy, ox = p // (Ho * Wo), (p // Wo) % Ho, p % Wo
    part = torch.empty((nch, taps, Cin, Cdy), dtype=torch.float64, device=dev)
    mag = torch.empty_like(part)
    for t in range(taps):
        iy = oy * stride + t // k - pad
        ix = (ox * stride + t % k - pad) % W
        inside = ((iy >= 0) & (iy < H)).double()[:, None]
        xt = x[b, iy.clamp(0, H - 1), ix].double() * inside
        xt = torch.nn.functional.pad(xt, (0, 0, 0, padrows)).reshape(nch, chunk, Cin)
        part[:, t] = xt.transpose(1, 2) @ d
        mag[:, t] = xt.abs().transpose(1, 2) @ da
        del xt
    dbpart, dbmag = d.sum(1), da.sum(1)
    steps = -(-chunk // 16)
    return dict(part=part, part_bound=steps * WGRAD_KSTEP * mag + EXACT, dbpart=dbpart,
                dbpart_bound=chunk * U * dbmag + EXACT, w=part.sum(0),
                w_bound=(steps * WGRAD_KSTEP + nch * U) * mag.sum(0), b=dbpart.sum(0),
                b_bound=(chunk + nch) * U * dbmag.sum(0), nch=nch, chunk=chunk)


def wgrad_layout(t, Cin_w: int, Cout: int, k: int):
    """[k^2, Cin, Cdy] -> dw's torch layout [Cout, Cin_w, k, k]."""
    return t[:, :Cin_w, :Cout].permute(2, 1, 0).reshape(Cout, Cin_w, k, k)


def wgrad_reduce_ref(part, f: float):
    """(ref, bound) of f * sum_c part_c in chunk order, given the kernel's fp32 partials [nch, ...]."""
    p = part.double()
    ref = f * p.sum(0)
    return ref, p.shape[0] * U * f * p.abs().sum(0) + U * ref.abs() + EXACT


BN_EPS = 1e-5


def bn_row_chunk(P: int) -> int:
    """Rows per chunk of the BatchNorm reductions: at most 512 chunks, at least 256 rows each."""
    return max(256, -(-P // 512))


def _chan_merge(acc, b, A):
    """Merge lane / chunk b into acc in fp64, carrying the error bounds of the kernel's fp32 Chan merge."""
    n, mean, m2, em, e2 = acc
    nb, mb, m2b, emb, e2b = b
    nab = n + nb
    live = nb > 0
    delta = mb - mean
    w = torch.where(live, n * nb / nab.clamp(min=1), torch.zeros_like(n))
    q = delta * delta * w
    e2n = e2 + e2b + 2 * delta.abs() * w * (em + emb) + 2 * U * (m2 + m2b + q) + 4 * U * q
    emn = (n * em + nb * emb) / nab.clamp(min=1) + 4 * U * A
    meann = mean + delta * nb / nab.clamp(min=1)
    pick = lambda new, old: torch.where(live, new, old)
    return (nab, pick(meann, mean), pick(m2 + m2b + q, m2), pick(emn, em), pick(e2n, e2))


def bn_stats_ref(z, block: int = 64):
    """pf_faedt_bn_stats of z fp16 [P, C]: dict of fp64 per-chunk `count` (exact), `mean` / `mean_bound`, `m2` /
    `m2_bound` [nch, C], and the merged `stats` / `stats_bound` [3, C] (mean, invstd, unbiased var)."""
    P, Cc = z.shape
    L = 256 // Cc
    chunk = bn_row_chunk(P)
    nch = -(-P // chunk)
    nw = -(-chunk // L)
    dev = z.device
    A = z.double().abs().amax(0)
    outs = {key: [] for key in ("count", "mean", "m2", "em", "e2")}
    for c0 in range(0, nch, block):
        c1 = min(nch, c0 + block)
        r0, r1 = c0 * chunk, min(P, c1 * chunk)
        zz = torch.full(((c1 - c0) * chunk, Cc), float("nan"), dtype=torch.float64, device=dev)
        zz[:r1 - r0] = z[r0:r1].double()
        zz = torch.nn.functional.pad(zz.reshape(c1 - c0, chunk, Cc), (0, 0, 0, nw * L - chunk), value=float("nan"))
        v = zz.reshape(c1 - c0, nw, L, Cc)                           # row t * L + lane of each chunk
        valid = ~torch.isnan(v)
        v0 = torch.where(valid, v, torch.zeros_like(v))
        cnt = valid.double().cumsum(1)
        mu = v0.cumsum(1) / cnt.clamp(min=1)                          # running means
        n = cnt[:, -1]
        mean = mu[:, -1]
        m2 = (torch.where(valid, v0 - mean[:, None], torch.zeros_like(v0)) ** 2).sum(1)
        prev = torch.cat([mu[:, :1], mu[:, :-1]], 1)
        move = cnt * (2 * (mean[:, None] - mu).abs() + (mu - prev).abs())
        e2 = 3 * U * A * torch.where(valid & (cnt >= 2), move, torch.zeros_like(move)).sum(1) + (nw + 3) * U * m2
        em = 3 * U * A * (n + 1) / 2
        acc = tuple(t[:, 0] for t in (n, mean, m2, em, e2))
        for lane in range(1, L):
            acc = _chan_merge(acc, tuple(t[:, lane] for t in (n, mean, m2, em, e2)), A)
        for key, t in zip(outs, acc):
            outs[key].append(t)
        del zz, v, valid, v0, cnt, mu, prev, move
    part = {key: torch.cat(t) for key, t in outs.items()}
    zero = torch.zeros(Cc, dtype=torch.float64, device=dev)
    acc = (zero, zero, zero, zero, zero)
    for i in range(nch):
        acc = _chan_merge(acc, tuple(part[key][i] for key in outs), A)
    n, mean, m2, em, e2 = acc
    eps = _f32(BN_EPS)
    var = m2 / n
    inv = 1.0 / torch.sqrt(var + eps)
    nu = U if P > (1 << 24) else 0.0
    stats = torch.stack([mean, inv, m2 / (n - 1)])
    bound = torch.stack([em + EXACT, inv * (0.5 * (e2 / n + nu * var) / (var + eps) + 4 * U),
                         e2 / (n - 1) + (2 * U + nu) * m2 / (n - 1)])
    return dict(count=part["count"], mean=part["mean"], mean_bound=part["em"] + EXACT, m2=part["m2"],
                m2_bound=part["e2"] + EXACT, stats=stats, stats_bound=bound, nch=nch, chunk=chunk)


def bn_apply_ref(z, stats, gamma, beta, relu: bool, residual=None):
    """(ref, bound) fp64 [P, C] of pf_faedt_bn_apply given the launch's fp32 stats [>= 2, C]."""
    mean, inv = stats[0].double(), stats[1].double()
    g, b = gamma.double(), beta.double()
    c = z.double() - mean
    y = c * inv * g + b
    bound = 3 * U * c.abs() * inv * g.abs() + U * y.abs()
    if relu:
        y = y.clamp_min(0.0)
    if residual is not None:
        y = y + residual.double()
        bound = bound + U * y.abs()
    return y, bound + ulp_out(y, torch.float16)


def bn_bwd_ref(g, mask, z, stats, gamma, f: float):
    """pf_faedt_bn_bwd given the launch's fp32 stats: dict of fp64 per-chunk `part` / `part_bound` [nch, 2, C],
    `sums` / `sums_bound` [2, C] and `dgamma`, `dbeta` (each with `_bound`), and dz_ref(sums) -> (ref, bound)."""
    P, Cc = z.shape
    L = 256 // Cc
    chunk = bn_row_chunk(P)
    nch = -(-P // chunk)
    nw = -(-chunk // L)
    gp = g.double()
    if mask is not None:
        gp = gp * (mask.double() > 0)
    mean, inv = stats[0].double(), stats[1].double()
    xh = (z.double() - mean) * inv
    gx = gp * xh
    pad = nch * chunk - P
    cs = lambda t: torch.nn.functional.pad(t, (0, 0, 0, pad)).reshape(nch, chunk, Cc).sum(1)
    s_g, s_gx, a_g, a_gx = cs(gp), cs(gx), cs(gp.abs()), cs(gx.abs())
    part = torch.stack([s_g, s_gx], 1)
    part_bound = torch.stack([(nw + L) * U * a_g, (nw + L + 3) * U * a_gx], 1) + EXACT
    tot = part.sum(0)
    tot_bound = part_bound.sum(0) + nch * U * torch.stack([a_g.sum(0), a_gx.sum(0)])
    nu = U if P > (1 << 24) else 0.0
    sums = tot / P
    sums_bound = tot_bound / P + (U + nu) * sums.abs()
    gam = gamma.double()

    def dz_ref(sums_k):
        s0, s1 = sums_k[0].double(), sums_k[1].double()
        ref = gam * inv * (gp - s0 - xh * s1)
        bound = 4 * U * (gam * inv).abs() * (gp.abs() + s0.abs() + 2 * (xh * s1).abs())
        return ref, bound + ulp_out(ref, torch.float16)
    return dict(part=part, part_bound=part_bound, sums=sums, sums_bound=sums_bound, dgamma=f * tot[1],
                dgamma_bound=f * tot_bound[1] + U * f * tot[1].abs(), dbeta=f * tot[0],
                dbeta_bound=f * tot_bound[0] + U * f * tot[0].abs(), dz_ref=dz_ref, nch=nch)


def _up2(x):
    return torch.nn.functional.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)


def upsample_ref(x):
    """(ref, bound) fp64 [B, 2H, 2W, C] of pf_faedt_upsample on x fp16 [B, H, W, C]."""
    xd = x.double().permute(0, 3, 1, 2)
    ref = _up2(xd).permute(0, 2, 3, 1)
    mag = _up2(xd.abs()).permute(0, 2, 3, 1)
    return ref, 4 * U * mag + ulp_out(ref, torch.float16)


def upsample_bwd_ref(g, H: int, W: int):
    """(ref, bound) fp64 [B, H, W, C] of pf_faedt_upsample_bwd: the adjoint of the bilinear x2 applied to g fp16
    [B, 2H, 2W, C]."""
    B, Cc = g.shape[0], g.shape[-1]
    gd = g.double().permute(0, 3, 1, 2)
    outs = []
    for t in (gd, gd.abs()):
        xr = torch.zeros((B, Cc, H, W), dtype=torch.float64, device=g.device, requires_grad=True)
        with torch.enable_grad():
            (gx,) = torch.autograd.grad(_up2(xr), xr, t)
        outs.append(gx.permute(0, 2, 3, 1))
    return outs[0], 10 * U * outs[1] + ulp_out(outs[0], torch.float16)


def loss_ref(o, target, B: int, H: int, W: int):
    """pf_faedt_loss: dict of fp64 `pred` / `pred_bound` [B, 3, H, W], `d` (tanh(o) - target) and `loss` /
    `loss_bound`."""
    pred = torch.tanh(o[..., :3].double()).permute(0, 3, 1, 2)
    d = pred - (target.double() if target is not None else 0.0)
    M = B * H * W
    n = 3 * -(-M // (1024 * 256)) + 20
    count = 3.0 * M
    loss = d.abs().sum() / count
    lb = ((n + 1) * U * d.abs().sum() + 2.0 ** -22 * pred.abs().sum()) / count + U * loss
    return dict(pred=pred, pred_bound=2.0 ** -22 * pred.abs() + 2.0 ** -149, d=d, loss=loss, loss_bound=lb)


def seed_check(seed, pred_k, d, pred_bound, S: float):
    """(worst err/bound, number of elements whose sign is defined) of pf_faedt_loss's seed fp16 [B, H, W, 16] against
    sign(d) (1 - pred^2) S computed from the kernel's fp32 pred [B, 3, H, W]; d = tanh(o) - target in fp64. Where
    |d| <= pred's error the sign is not defined: there the seed must be 0 or either sign of the same magnitude.
    Channels 3..15 must be exactly zero."""
    assert not seed[..., 3:].any(), "seed channels 3..15 are not zero"
    got = seed[..., :3].permute(0, 3, 1, 2).double()
    p = pred_k.double()
    mag = (1 - p * p) * S
    bound = 2.0 ** -11 * mag.abs() + 2 * U * S + 2.0 ** -25
    big = mag.abs() + bound >= 65520.0             # may round to inf in fp16
    clear = d.abs() > pred_bound
    want = torch.sign(d) * mag
    err = torch.where(clear, (got - want).abs(), torch.minimum((got.abs() - mag).abs(), got.abs()))
    r = err / bound
    inf_ok = torch.isinf(got) & big & ((torch.sign(got) == torch.sign(d)) | ~clear)
    r = torch.where(inf_ok, torch.zeros_like(r), r)
    # tanhf(0) = 0 exactly: where the target is 0 too, d = 0 and sign(0) = 0 makes the seed exactly zero
    r = torch.where((d == 0) & (p == 0) & (got != 0), torch.full_like(r, math.inf), r)
    return float(torch.nan_to_num(r, nan=math.inf).max()), int(clear.sum())


def prep_ref(src):
    """pf_faedt_prep: fp32 [B, 3, H, W] -> fp16 [B, H, W, 16], channels 3..15 zero."""
    out = torch.zeros(src.shape[0], src.shape[2], src.shape[3], 16, dtype=torch.float16, device=src.device)
    out[..., :3] = src.permute(0, 2, 3, 1).half()
    return out


def interleave_ref(ph):
    """pf_faedt_interleave: phases [4, B, H/2, W/2, C] -> [B, H, W, C], dx[b, 2q + r, 2p + c] = phases[2r + c]."""
    _, B, h, w, Cc = ph.shape
    return ph.reshape(2, 2, B, h, w, Cc).permute(2, 3, 0, 4, 1, 5).reshape(B, 2 * h, 2 * w, Cc)


def pack_ref(w, k: int, stride: int, cin_pad: int, cw: int, dg_rows: int, dg_cw: int):
    """pf_faedt_pack of w fp32 [Cout, Cin, k, k]: (fwd fp16 [k^2, cin_pad, cw], dg fp16) with zero padding; dg is the
    flipped kernel [k^2, dg_rows, dg_cw] at stride 1 or the four phase kernels [4, 4, dg_rows, dg_cw] (phase (r, c)
    tap (ty, tx) = w[.., 3 - 2 ty - r, 3 - 2 tx - c]) at stride 2."""
    Cout, Cin = w.shape[:2]
    fwd = torch.zeros(k * k, cin_pad, cw, dtype=torch.float32, device=w.device)
    fwd[:, :Cin, :Cout] = w.permute(2, 3, 1, 0).reshape(k * k, Cin, Cout)
    if stride == 1:
        taps = w.flip(2, 3).permute(2, 3, 0, 1).reshape(k * k, Cout, Cin)
    else:
        taps = torch.cat([w[:, :, [3 - r, 1 - r]][:, :, :, [3 - c, 1 - c]].permute(2, 3, 0, 1).reshape(4, Cout, Cin)
                          for r in (0, 1) for c in (0, 1)])
    dg = torch.zeros(k * k, dg_rows, dg_cw, dtype=torch.float32, device=w.device)
    dg[:, :Cout, :Cin] = taps
    return fwd.half(), dg.half()
