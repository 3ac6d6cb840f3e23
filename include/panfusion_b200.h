/*
 * panfusion_b200 — C ABI of the H100 (sm_90a) denoise hot path of PanFusion.
 *
 * Every entry point takes plain device pointers, sizes and a CUDA stream (cudaStream_t passed as void*).
 * The caller (PyTorch on the host side) owns every buffer; the library keeps no hidden state except a
 * thread-local error string. All functions return 0 on success or a negative PF_ERR_* code; launches are
 * asynchronous on the given stream and CUDA-graph capturable (no allocation, no host sync inside), except
 * pf_frechet_fp64, which reads its convergence test back once per Jacobi sweep.
 *
 * Each declaration cites the reference interface (file:line under the upstream repo) it replaces.
 * Tensors are row-major; "tokens" layout means [N*H*W, C] channels-last, "NCHW" is the reference's layout.
 */
#ifndef PANFUSION_B200_H
#define PANFUSION_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PF_OK 0
#define PF_ERR_INVALID (-1)     /* bad argument (message in pf_last_error) */
#define PF_ERR_CUDA (-2)        /* CUDA runtime / driver failure */
#define PF_ERR_UNSUPPORTED (-3) /* shape / dtype not supported by the sm_90a kernels */

typedef enum { PF_F32 = 0, PF_F16 = 1, PF_BF16 = 2 } pf_dtype;

/* error convention: reference raises Python exceptions (utils/pano.py:85,
 * external/Perspective_and_Equirectangular/utils.py:15); here: return code + message. */
const char* pf_last_error(void);
int pf_version(void);
/* returns 0 iff the current device is compute capability 9.0 (H100); the library has no other path */
int pf_check_device(void);

/* ------------------------------------------------------------------------------------------------
 * Spherical resampling (K1/K2): external/Perspective_and_Equirectangular/e2p.py:54-76, p2e.py:52-77
 * The sampling grid is computed in-kernel (fp64 per output pixel) from the camera record; no grid is
 * stored. Sampling follows kornia.remap -> F.grid_sample(align_corners=True, padding_mode='zeros').
 *
 * Camera record: PF_CAM_DOUBLES doubles, device memory, one per batch element (cam_stride = 1) or a single
 * record broadcast over the batch (cam_stride = 0):
 *   [0:9)  R1  row-major   (e2p: Rodrigues(z * rad(theta));   p2e: inv(R1))
 *   [9:18) R2  row-major   (e2p: Rodrigues(R1 y * rad(-phi)); p2e: inv(R2))
 *   [18] w_len = tan(rad(wfov/2))   [19] h_len = tan(rad(hfov/2))
 * mode: 0 = bilinear, 1 = nearest (round-half-even).
 * ------------------------------------------------------------------------------------------------ */
#define PF_CAM_DOUBLES 20

/* e2p(e_img[B,C,He,We]) -> [B,C,h,w]   (e2p.py:54-76; grid math e2p.py:9-51) */
int pf_e2p(const void* src, void* dst, int dtype, int B, int C, int He, int We, int h, int w,
           const double* cams, int cam_stride, int mode, void* stream);

/* e2p of B cameras over B / src_repeat source panoramas: src[B/src_repeat, C, He, We], camera b reads source b / src_repeat
 * (PanFusion.init_noise, models/pano/PanFusion.py:30-43, expands ONE panorama to its m views before e2p; feature-map
 * warps of a CFG batch read 2 panoramas from 16 cameras). Same result as pf_e2p on the expanded tensor; the source is read
 * from HBM once. */
int pf_e2p_shared(const void* src, void* dst, int dtype, int B, int src_repeat, int C, int He, int We, int h, int w,
                  const double* cams, int cam_stride, int mode, void* stream);

/* py360convert.e2p (external/py360convert/e2p.py:6-43, utils.py:104-132,231-243): the dataset's pixel-space convention
 * (utils/pano.py:160-161 `Equirectangular.to_perspective`, dataset/PanoDataset.py:138) — channels-last src[H, W, C] (uint8 when
 * is_u8, else fp32) -> dst[num_cams, h, w, C]; half-pixel centres (uv2coor), longitude wrap-around, pole rows padded with the
 * first / last row rolled by W/2, scipy 'wrap' boundaries, float64 grid math, integers rounded half up.
 * Camera record: PF_CAM360_DOUBLES doubles = Rx, Ry, Ri (row-major; rotation_matrix(v,[1,0,0]), rotation_matrix(-yaw,[0,1,0]),
 * rotation_matrix(in_rot, z Rx Ry)), tan(h_fov/2), tan(v_fov/2). mode: 0 bilinear, 1 nearest; anything else is
 * PF_ERR_UNSUPPORTED like the reference's NotImplementedError('unknown mode'). */
#define PF_CAM360_DOUBLES 29
int pf_e2p_py360(const void* src, void* dst, int is_u8, int H, int W, int C, int h, int w, const double* cams,
                 int num_cams, int mode, void* stream);

/* py360convert.c2e (external/py360convert/c2e.py:6-64, utils.py:40-64,135-173): horizon cube cube[face_w, 6*face_w, C]
 * (faces F R B L U D, uint8 when is_u8, else fp32) -> dst[h, w, C] float64, the dtype the reference returns (its padded
 * faces are float64). w must be a multiple of 8 (c2e.py:26). Face coordinates in float32 as numpy computes them, clip /
 * scale / bilinear weights in float64, scipy 'wrap' sampling of the (face_w + 2)-padded faces.
 *   ceil_rows[w / 4]: the ceiling row of each column of one quarter (equirect_facetype: h // 2 - round(arctan(cos(lon))
 *                     * h / pi) in float64 on the host), device memory.
 *   border[6][4 * face_w + 4]: horizon-cube pixel index (row * 6 * face_w + col) of every pad sample of each face, -1 for
 *                     a zero pad: [row face_w][face_w], [row face_w + 1][face_w], [col face_w][face_w + 2],
 *                     [col face_w + 1][face_w + 2]; device memory. panfusion_b200/py360.py builds both tables.
 * mode: 0 bilinear, 1 nearest; anything else is PF_ERR_UNSUPPORTED. */
int pf_c2e_py360(const void* cube, double* dst, int is_u8, int face_w, int C, int h, int w, const int* ceil_rows,
                 const int* border, int mode, void* stream);

/* py360convert.e2c (external/py360convert/e2c.py:6-40): src[H, W, C] (uint8 when is_u8, else fp32) -> horizon cube
 * dst[face_w, 6 * face_w, C] in the source dtype; the grid (xyzcube -> xyz2uv -> uv2coor) in float32, sampled like
 * pf_e2p_py360 (integers rounded half up). mode: 0 bilinear, 1 nearest; anything else is PF_ERR_UNSUPPORTED. */
int pf_e2c_py360(const void* src, void* dst, int is_u8, int H, int W, int C, int face_w, int mode, void* stream);

/* p2e(p_img[B,C,hp,wp]) -> equi[B,C,He,We] (already multiplied by mask), mask[B,1,He,We] uint8 (may be NULL)
 * (p2e.py:52-77; grid math p2e.py:9-49) */
int pf_p2e(const void* src, void* dst, uint8_t* mask, int dtype, int B, int C, int hp, int wp, int He, int We,
           const double* cams, int cam_stride, int mode, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Tap-GEMM (wgmma / TMA): the one dense-contraction engine behind nn.Linear (K8, K10) and the
 * 3x3 / 1x1 convolutions (K9, K11) of the UNet walk in models/pano/MVGenModel.py:85-295.
 *
 *   acc[m, n] = sum_{t < num_taps} sum_{k < Kc} A[m + tap_off[t], k] * B[n, t*Kc + k]      (fp32 accumulate)
 *   v        = act(acc + bias[n] + rowbias[group(m), n])           (GEGLU: v = a * gelu(g), see below)
 *   out[row(m), n] = v + residual[row(m), n]
 *
 * A is a row-major [a_rows, a_ld] 16-bit matrix (rows outside [0, a_rows) read as zero), B the packed
 * weight [N, num_taps*Kc]. A 3x3 convolution is 9 taps over a zero-haloed channels-last image
 * ("padded-flat" layout); the M-space -> output-row map drops halo rows:
 *   map_mode 0: row(m) = m, group(m) = m / rows_per_group
 *   map_mode 1: m -> (img, i, j) with i = (m / Wm) % Hm, j = m % Wm; valid iff i0 <= i < i0+Hout and
 *               j0 <= j < j0+Wout; row(m) = (img*Hout + i-i0)*Wout + (j-j0); group(m) = img
 * act: PF_ACT_GEGLU expects B (and bias) packed so that every 256-wide column tile holds 128 value columns followed
 * by their 128 gate columns; it writes N/2 output columns. GEGLU runs only at block_n = 256 and needs one tap,
 * map_mode 0, a 16-bit output, k_splits <= 1 and no residual or rowbias. PF_ACT_GELU is erf-GELU (F.gelu),
 * PF_ACT_QUICK_GELU is CLIP's x * sigmoid(1.702 x); both apply wherever PF_ACT_SILU does (epilogues, split-K reduce).
 * Constraints: Kc % 64 == 0, N % block_n == 0, block_n in {64,128,160} (256 only with GEGLU), a_ld/b_ld % 8 == 0.
 * A call outside the contract returns PF_ERR_INVALID with a message before any CUDA call.
 * Alignment (checked, PF_ERR_INVALID otherwise): A, B, out, residual, rowbias, splitk_ws and ln_stats 16 bytes;
 * row_stats_out 8 bytes; out_ld, res_ld % 8 == 0 and rowbias_ld % 4 == 0 (elements), so every row stays aligned.
 * ------------------------------------------------------------------------------------------------ */
enum { PF_ACT_NONE = 0, PF_ACT_SILU = 1, PF_ACT_GELU = 2, PF_ACT_GEGLU = 3, PF_ACT_QUICK_GELU = 4 };
#define PF_MAX_TAPS 16

typedef struct pf_gemm_args {
  const void* A;
  int64_t a_rows;
  int32_t a_ld;
  const void* B;
  int32_t b_ld;
  int32_t dtype; /* PF_F16 | PF_BF16 (A and B) */
  int32_t M, N, Kc, num_taps;
  int32_t tap_off[PF_MAX_TAPS];
  int32_t block_n; /* 0 = auto (pf_gemm_pick_block_n), else 64, 128, 160, or 256 with GEGLU */
  void* out;
  int32_t out_ld;
  int32_t out_dtype; /* PF_F32 or same as dtype */
  const float* bias;
  const float* rowbias;
  int32_t rowbias_ld;
  int32_t rows_per_group;
  const void* residual;
  int32_t res_ld;
  int32_t res_dtype;
  int32_t act;
  int32_t map_mode, Hm, Wm, i0, j0, Hout, Wout;
  /* split-K (long-K, few-tile problems: the 8x8 / 16x16 level convolutions): k_splits > 1 partitions the K-slabs over
   * k_splits CTAs per tile; partial accumulators go to splitk_ws (fp32, k_splits * M * N elements, caller-owned) and
   * a second kernel reduces them in a fixed order and applies the epilogue. 0 / 1 = off. */
  int32_t k_splits;
  float* splitk_ws;
  /* LayerNorm fused around the GEMM (diffusers BasicTransformerBlock norm1/2/3 -> to_q|k|v / to_q / GEGLU proj, and
   * models/modules/transformer.py:159-160 norm2 -> ff): instead of a LayerNorm kernel between two linears,
   *   PRODUCER (row_stats_out != NULL): besides `out`, writes per output row the partial (sum, sum of squares) of the
   *     final fp32 values of every column slot: row_stats_out[m][slot][2], slots = pf_gemm_row_stats_slots(args).
   *   CONSUMER (ln_stats != NULL): A is the UN-normalised tensor, B holds gamma-scaled weights W'[n,k] = gamma[k] W[n,k],
   *     ln_colsum[n] = sum_k W'[n,k] (of the 16-bit rounded W'), bias[n] = sum_k beta[k] W[n,k] + b[n]; the epilogue applies
   *     acc <- rstd[m] * (acc - mean[m] * ln_colsum[n]) with mean / rstd from ln_stats[m][ln_slots][2] over K = Kc*num_taps
   *     elements, biased variance, eps = ln_eps — algebraically LayerNorm(A) W^T + b with the normalised tensor never
   *     stored. Both sides need one tap, no rowbias, no split-K, the plain row map and a 16-bit output; the consumer
   *     may also run the GEGLU epilogue. */
  /* map_mode 1 with an output SCATTER (0 / 1 = off): the valid pixel (i, j) of image img is written to row
   *   ((img*Hout + i-i0)*out_sy + out_a) * (Wout*out_sx) + (j-j0)*out_sx + out_b
   * i.e. phase (out_a, out_b) of an image up-sampled by (out_sy, out_sx). Upsample2D's nearest-x2 followed by a 3x3
   * convolution (MVGenModel.py:272-277) is exactly four 2x2 convolutions of the ORIGINAL image, one per output phase, with
   * summed weights: 16 instead of 36 tap-GEMMs per input pixel and no up-sampled copy. */
  int32_t out_sy, out_sx, out_a, out_b;
  float* row_stats_out;
  const float* ln_stats;
  int32_t ln_slots;
  const float* ln_colsum;
  float ln_eps;
} pf_gemm_args;

int pf_gemm_taps(const pf_gemm_args* args, void* stream);
/* number of column slots a producer with these args writes per row of row_stats_out: 2 per column tile, and a producer's
 * tile width is a function of N alone (block_n requests are ignored), so the statistics are bit-identical for any M */
int pf_gemm_row_stats_slots(const pf_gemm_args* args);
/* suggested k_splits for this problem (1 = do not split); only M, N, Kc, num_taps, act, map_mode, dtypes are read */
int pf_gemm_splitk_plan(const pf_gemm_args* args);
/* block_n that block_n = 0 selects for this N: 160, 128 or 64 (the widest that divides N), for GEGLU 256; 0 if none
 * divides N (used by the host-side weight packer for GEGLU) */
int pf_gemm_pick_block_n(int N, int act);

/* ------------------------------------------------------------------------------------------------
 * Flash attention forward (wgmma): out = softmax(q k^T * scale + bias) v, fp32 softmax / accumulation.
 * Replaces xformers.ops.memory_efficient_attention at models/modules/transformer.py:71 (EPPA: head_dim 32,
 * additive fp32 bias shared by every head — transformer.py:68 materialises it per head, this never does) and the
 * bmm-softmax-bmm of the diffusers attention blocks walked at models/pano/MVGenModel.py:104,116,185,190,227,241
 * (head_dim 64, self and 77-token text cross attention).
 * q/k/v: 16-bit, element (b, l, h, d) at ptr[b*bstride + l*ld + h*head_dim + d] (so fused QKV buffers work
 * in place); out: [B, Lq, out_ld] same dtype. bias: fp32 [*, Lq, bias_ld], batch b reads bias + b*bias_bstride
 * (0 = one table for all batches), or NULL. Any Lq / Lk >= 1 (ragged tiles are masked).
 * ------------------------------------------------------------------------------------------------ */
typedef struct pf_fmha_args {
  const void* q;
  const void* k;
  const void* v;
  void* out;
  int32_t dtype;
  int32_t B, H, Lq, Lk, head_dim;
  int32_t q_ld, k_ld, v_ld, out_ld;
  int64_t q_bstride, k_bstride, v_bstride;
  float scale;
  const float* bias;
  int64_t bias_bstride;
  int32_t bias_ld;
  /* optional block-sparsity hint for the bias: flags[b][ceil(Lq/128)][ceil(Lk/64)] bytes, non-zero = every entry of
   * that 128x64 bias tile is exactly -1 (no geometric correspondence, SURVEY.md A.4: ~85% of the EPPA tiles), so the
   * kernel substitutes the constant instead of reading the tile. NULL = read everything. Build with
   * pf_bias_tile_flags. */
  const uint8_t* bias_flags;
  int64_t flags_bstride;
  int32_t flags_ld;
  /* tile-PACKED bias (the resident form of the EPPA tables): `bias` is then the store [n_live][128 * 64] fp32 (lane-interleaved tiles) built by
   * pf_bias_tile_pack and bias_tile_off[bias batch][ceil(Lq/128)][ceil(Lk/64)] (row stride flags_ld, batch stride
   * flags_bstride, in tiles) holds each tile's index in it, or -1 for a tile that is entirely -1 (no correspondence).
   * bias_ld / bias_bstride / bias_flags are unused. The reference materialises the dense tensor PER HEAD
   * (models/modules/transformer.py:68); this keeps ~15 % of ONE copy. */
  const int32_t* bias_tile_off;
} pf_fmha_args;

int pf_fmha_fwd(const pf_fmha_args* args, void* stream);
/* flags[g][qt][kt] = 1 iff bias[g][qt*128 .. , kt*64 ..] is entirely == -1.0f (tiles clipped at Lq / Lk) */
int pf_bias_tile_flags(const float* bias, int G, int Lq, int Lk, int bias_ld, int64_t bias_bstride, uint8_t* flags,
                       void* stream);
/* exclusive scan of the live (flag == 0) tiles: tile_off[t] = index among the live tiles or -1; n_live[0] = their number */
int pf_bias_tile_scan(const uint8_t* flags, int num_tiles, int32_t* tile_off, int32_t* n_live, void* stream);
/* packed[tile_off[g][qt][kt]] <- the dense 128 x 64 tile (zero outside [Lq, Lk]); constant tiles are skipped. Inside a
 * tile the 8192 floats are LANE-INTERLEAVED for the attention kernel (thread = query row): element (r, c) sits at
 * (((r / 32) * 16 + c / 4) * 32 + r % 32) * 4 + c % 4, so one 16-byte load of a warp covers 512 contiguous bytes. */
int pf_bias_tile_pack(const float* bias, int G, int Lq, int Lk, int bias_ld, int64_t bias_bstride, const int32_t* tile_off,
                      float* packed, void* stream);

/* ------------------------------------------------------------------------------------------------
 * GroupNorm statistics of a channels-last image x[N, H, W, C] (row stride ld), computed over the image
 * circularly extended by `circ` columns on each side — the reference normalises the padded tensor
 * (models/pano/MVGenModel.py:110-115 wraps each panorama ResnetBlock2D in utils/pano.py:74-105 pad/unpad), so
 * columns {0..circ-1, W-circ..W-1} count twice. ws: scratch of pf_groupnorm_ws_floats(N, groups) floats.
 * counters: N ints that are ZERO on entry (the kernel restores them to zero; concurrent calls need distinct slots):
 * the last CTA of each image reduces the partial sums in a fixed order, so the result is deterministic.
 * mean_rstd: [N, groups, 2] fp32 (mean, 1/sqrt(var + eps)), biased variance like torch.nn.GroupNorm.
 * ------------------------------------------------------------------------------------------------ */
int pf_groupnorm_ws_floats(int N, int groups);
int pf_groupnorm_stats(const void* x, int dtype, int N, int H, int W, int C, int ld, int groups, int circ,
                       float eps, float* ws, int* counters, float* mean_rstd, void* stream);

/* GroupNorm-apply (+SiLU) fused with building the tap-GEMM A operand (replaces norm+nonlinearity of diffusers
 * ResnetBlock2D / Transformer2DModel.norm, pad_pano/unpad_pano utils/pano.py:74-105, Upsample2D's nearest x2,
 * Downsample2D's stride-2 gather; call sites MVGenModel.py:98-277).
 *   source image S = x circularly extended by `circ` columns per side, then nearest-upsampled by `up` (1|2);
 *   phases == 1: out[N, Hu + 2*halo, Wu + 2*halo, C], zero halo (halo = 1 for a 3x3 conv input, 0 = plain apply)
 *   phases == 4: out[4][N][Hu/2 + 1][Wu/2 + 1][C], phase (py,px) element (i,j) = zero-padded S at (2i+py, 2j+px)
 * mean_rstd == NULL skips the normalisation; act: PF_ACT_NONE | PF_ACT_SILU. */
int pf_conv_prep(const void* x, void* out, int dtype, int N, int H, int W, int C, int ld, const float* mean_rstd,
                 const float* gamma, const float* beta, int groups, int act, int circ, int up, int phases, int halo,
                 void* stream);

/* pf_groupnorm_stats + pf_conv_prep (same semantics, same reference call sites), optionally over the channel concatenation
 * of two tensors (torch.cat([hidden, skip], dim=1) at MVGenModel.py:223,231,246,254):
 *   x = cat(x1[N*H*W, C1], x2[N*H*W, C2]) (x2 may be NULL); if cat_out != NULL the raw concatenation [N*H*W, C1+C2] is also
 *   written (the ResnetBlock2D shortcut convolution reads it);
 *   statistics over the image circularly extended by circ_stats columns (duplicated columns count twice), applied with
 *   gamma / beta (+ SiLU) while building the conv_prep layout (circ, up, phases, halo as in pf_conv_prep).
 * Two launches: the statistics with one CTA per slab of each image, then the apply pass with up to 64 CTAs per image (the
 * source is re-read from L2). ws: pf_gn_prep_ws_floats(N, groups) floats of scratch; counters: N ints that are ZERO on
 * entry (restored to zero by the kernel; concurrent launches need distinct slots). The partition of every sum depends on
 * H*W only, never on N: results are bit-identical for any batch size. */
int pf_gn_prep_ws_floats(int N, int groups);
int pf_gn_prep(const void* x1, int ld1, int C1, const void* x2, int ld2, int C2, void* cat_out, void* out, int dtype,
               int N, int H, int W, int groups, float eps, const float* gamma, const float* beta, int act,
               int circ_stats, int circ, int up, int phases, int halo, float* ws, int* counters, void* stream);

/* out[t, :] = LayerNorm(x[t, :] + pe[t % pe_rows, :]) * gamma + beta (pe fp32, may be NULL);
 * models/modules/transformer.py:157-160 (EPPA norm1 on x + query_pe / context, norm2) and the diffusers
 * BasicTransformerBlock norm1/2/3. */
int pf_layernorm(const void* x, int ldx, void* out, int ldo, int dtype, int T, int C, const float* pe, int pe_rows,
                 const float* gamma, const float* beta, float eps, void* stream);

/* conv_in (MVGenModel.py:85-91): NCHW fp32 latent [N,Cin,H,W] -> tokens [N*H*W, Cout] 16-bit; 3x3 pad 1;
 * circ != 0 wraps columns (== pad_pano(1) -> conv -> unpad_pano(1)). w fp32 [Cout,Cin,3,3], bias fp32 [Cout].
 * act = PF_ACT_SILU applies SiLU to the result: the first convolution of the ControlNet conditioning embedding on the
 * 3-channel layout image (diffusers ControlNetConditioningEmbedding [3P], consumed at MVGenModel.py:66-83). */
int pf_conv_in(const float* x, const float* w, const float* bias, void* out, int dtype, int N, int Cin, int H, int W,
               int Cout, int circ, int act, void* stream);

/* strided 2-D copy of 16-bit rows; src and dst may be column slices of wider tensors */
int pf_copy2d(const void* src, int src_ld, void* dst, int dst_ld, long long rows, int cols, void* stream);

/* pad_pano (utils/pano.py:74-99): out[r, j] = x[r, (j - pad) mod W] for j in [0, W + 2*pad) — circular padding of the
 * longitude axis of a contiguous tensor whose leading dims are flattened into `rows`; any pad >= 1 (F.pad's circular
 * mode limits pad <= W, this does not). elem_bytes in {1, 2, 4, 8}. */
int pf_pad_pano(const void* x, void* out, int elem_bytes, long long rows, int W, int pad, void* stream);

/* out[r, :cols] = softmax(scale * s[r, :cols]) — fp32 logits [rows, ld] -> 16-bit probabilities [rows, ldo].
 * The VAE mid-block attention (diffusers AutoencoderKL [3P], called through decode_latent, PanoGenerator.py:272-278)
 * has ONE head of width 512, outside the flash kernel's head sizes: it runs as pf_gemm_taps (Q K^T, fp32 out) ->
 * pf_softmax_rows -> pf_gemm_taps (P V). */
int pf_softmax_rows(const float* s, long long ld, void* out, long long ldo, int dtype, long long rows, int cols,
                    float scale, void* stream);

/* tensor_to_image (models/modules/utils.py:9-15): x fp32 [n, C, H, W] in [-1, 1] -> uint8 [n, H, W, C] =
 * round(clamp(x / 2 + 0.5, 0, 1) * 255), round-half-to-even like torch.round. */
int pf_tensor_to_image(const float* x, unsigned char* out, long long n, int C, int H, int W, void* stream);

/* diffusers Timesteps(dim, flip_sin_to_cos=True, freq_shift=0) (MVGenModel.py:55,59): t fp32 [n] -> [n, dim] */
int pf_timestep_embed(const float* t, void* out, int dtype, int n, int dim, void* stream);

/* CLIP text embeddings (transformers CLIPTextEmbeddings [3P] behind PanoGenerator.encode_text, models/pano/PanoGenerator.py:
 * 197-211): out[t, :] = tok_emb[ids[t], :] + pos_emb[t % L, :] (fp32 tables -> 16-bit tokens) and row_stats[t] = (sum, sum of
 * squares, 0, 0) of the stored row — the two-slot statistics the first encoder layer's fused LayerNorm consumes
 * (pf_gemm_args.ln_stats). ids int64 [T]; an id outside [0, vocab) traps (torch raises IndexError). */
int pf_embed_tokens(const long long* ids, const float* tok_emb, const float* pos_emb, void* out, int dtype,
                    float* row_stats, int T, int L, int C, int vocab, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Forward half of the training step (models/pano/PanFusion.py:64-98, SURVEY.md 8f rank 4). The backward of the UNets, of
 * EPPA and of the LoRA adapters, the optimizer and the gradient all-reduce are NOT built.
 * pf_add_noise: diffusers SchedulerMixin.add_noise [3P] as called at PanFusion.py:84-85 —
 *   out[b, :] = sqrt(abar[t[b]]) * x0[b, :] + sqrt(1 - abar[t[b]]) * noise[b, :]   (fp32 [B, per_sample], t int64 [B],
 *   abar = alphas_cumprod fp32 [num_train_timesteps]; a timestep outside the table traps).
 * pf_mse_loss: torch.nn.functional.mse_loss(a, b) with mean reduction (PanFusion.py:92-93), out[0] = sum((a-b)^2) / n,
 *   summed in a launch-independent order (fixed chunks, partials added in index order in fp64). ws: pf_mse_loss_ws_floats()
 *   floats; counter: one zero-initialised int32, re-armed by the kernel.
 * ------------------------------------------------------------------------------------------------ */
/* Latent sampling at the end of the VAE encoder (diffusers DiagonalGaussianDistribution.sample [3P] + the scaling of
 * PanoGenerator.encode_image, models/pano/PanoGenerator.py:218-224): moments = channels-last rows of width ld holding
 * [mean (L) | logvar (L) | ...] for N images of HW pixels; eps, out NCHW fp32 [N, L, HW];
 * out = (mean + exp(0.5 * clamp(logvar, -30, 20)) * eps) * scale. */
int pf_gaussian_sample(const float* moments, int ld, const float* eps, float* out, int N, int L, int HW, float scale,
                       void* stream);
int pf_add_noise(const float* x0, const float* noise, float* out, const long long* t, const float* alphas_cumprod,
                 int num_train_timesteps, int B, long long per_sample, void* stream);
int pf_mse_loss_ws_floats(void);
int pf_mse_loss(const float* a, const float* b, long long n, float* ws, int* counter, float* out, void* stream);

/* Classifier-free-guidance combine + DDIM update (+ roll of the result by `roll` columns):
 *   e = eps[0:count] + guidance * (eps[count:2count] - eps[0:count])        (PanoGenerator.py:253-262)
 *   out[.., (col+roll) % W] = sqrt(a_prev) * (x - sqrt(1-a_t) e) / sqrt(a_t) + sqrt(1-a_prev) e   (DDIM, eta 0)
 * replaces combine_cls_free_guide_pred + DDIMScheduler.step (PanFusion.py:159-162) + torch.roll
 * (PanoGenerator.py:264-269) of the following step. x, out fp32 [count] viewed as rows of W. */
int pf_cfg_ddim_step(const float* x, const float* eps, float* out, long long count, int W, int roll, float guidance,
                     float alpha_t, float alpha_prev, void* stream);
/* same update with the two coefficients read from DEVICE memory: coef[0] = sqrt(a_prev/a_t),
 * coef[1] = sqrt(1-a_prev) - coef[0]*sqrt(1-a_t) — lets one captured CUDA graph serve every denoising step. */
int pf_cfg_ddim_step_dev(const float* x, const float* eps, float* out, long long count, int W, int roll,
                         float guidance, const float* coef, void* stream);

/* ------------------------------------------------------------------------------------------------
 * EPPA geometry tables (models/pano/utils.py:10-106, models/modules/transformer.py:185-201).
 * pf_eppa_tables: correspondence bias for both attention directions of V views (groups of m views per batch
 * element) straight from the camera records (device, PF_CAM_DOUBLES each; e2p and p2e flavours):
 *   bias1[V/m][eh*ew][m*ph*pw]  query = pano pixel, keys = view pixels   (modules.py:46)
 *   bias2[V/m][m*ph*pw][eh*ew]  query = view pixel, keys = pano pixels   (modules.py:53)
 * blur5: HOST pointer to the 5 taps of the sigma-1 gaussian. ws_idx / ws_w: scratch of 4*V*(ph*pw+eh*ew) each.
 * pf_eppa_pe: SphericalPE tables, fp32: pers_pe[V*ph*pw][4*n_freqs], equi_pe[eh*ew][4*n_freqs].
 * ------------------------------------------------------------------------------------------------ */
int pf_eppa_tables(const double* cams_e2p, const double* cams_p2e, int V, int m, int ph, int pw, int eh, int ew,
                   const float* blur5, int* ws_idx, float* ws_w, float* bias1, float* bias2, void* stream);
int pf_eppa_pe(const double* cams_e2p, int V, int ph, int pw, int eh, int ew, const float* freq_bands, int n_freqs,
               float* pers_pe, float* equi_pe, void* stream);

/* ------------------------------------------------------------------------------------------------
 * MVDiffusion correspondence-aware attention CPAttn (external/MVDiffusion/pano/modules.py:22-86,
 * pano/utils.py:7-123): each pixel of view i attends to the 3x3 window around its homography correspondence in
 * views (i-1) mod m and (i+1) mod m — 18 keys per query, key slot s = n*9 + (di+1)*3 + (dj+1) (n = 0: view i-1,
 * n = 1: view i+1; di offsets x, dj offsets y).
 * pf_cpattn_tables: homo_l / homo_r fp32 [G][m][2][9] row-major (per camera group, view i, neighbour n):
 *   homo_l = K_n R_n^-1 R_i K_i^-1 (correspondences, utils.py:26-27), homo_r = K_i R_i^-1 R_n K_n^-1
 *   (back-projection, modules.py:57-58). Query pixel (y, x) of the h x h level sits at image pixel
 *   (s/2 + s x, s/2 + s y), s = img_size / h. Writes, per (g, i, query pixel, slot):
 *   pos fp32 [G*m*h*w*18][4] = (grid_sample x, y in the neighbour's pixel units, xy_rel x, y) and
 *   mask uint8 [G*m*h*w*18] (window position strictly inside the image, utils.py:74-75).
 * pf_cpattn_gather: x = tokens [B*m*h*w, ldx] 16-bit (batch element b uses camera group b when G == B, group 0
 *   when G == 1) -> keys [B*m*h*w*18, C] 16-bit = (bilinear sample + PosEmbedding(xy_rel)) * mask with
 *   freq_bands[C/4] (transformer.py:169-209), and stats fp32 [B*m*h*w*18][2][2] = per-row (sum, sum of squares)
 *   in slot 0 and zeros in slot 1: the ln_stats operand of pf_gemm_args (norm1 folded into the K|V GEMM).
 * pf_cpattn_attn: q [ntok, ldq], kv [ntok*18, ldkv] = K in columns [0, C) and V in [C, 2C), out [ntok, ldo];
 *   heads of width 32, softmax over the 18 keys in fp32 (masked keys included, like the reference).
 * ------------------------------------------------------------------------------------------------ */
int pf_cpattn_tables(const float* homo_l, const float* homo_r, int G, int m, int h, int w, int img_size, float* pos,
                     uint8_t* mask, void* stream);
int pf_cpattn_gather(const void* x, int ldx, int dtype, int B, int m, int h, int w, int C, int G, const float* pos,
                     const uint8_t* mask, const float* freq_bands, void* keys, float* stats, void* stream);
int pf_cpattn_attn(const void* q, int ldq, const void* kv, int ldkv, void* out, int ldo, int dtype, long long ntok,
                   int C, float scale, void* stream);

/* mp2e (external/Perspective_and_Equirectangular/mp2e.py as MvDiffusion.inference_and_save calls it, no mode):
 * views uint8 [m, hp, wp, C] (C <= 4) -> out uint8 [He, We, C] = sum_v img_v w_v / sum_v w_v truncated, 255 where no
 * view reaches; img_v / w_v are the view and its horizontal weight ramp warped by p2e's numpy path (cv2.remap with
 * interpolation None = nearest, map rounded half to even, BORDER_WRAP) times the frustum mask. cams_p2e: m p2e camera
 * records (PF_CAM_DOUBLES each, device). */
int pf_mp2e(const uint8_t* views, int m, int hp, int wp, int C, const double* cams_p2e, int He, int We, uint8_t* out,
            void* stream);

/* ------------------------------------------------------------------------------------------------
 * FAED (models/faed/FAED.py:50-103, encoder models/faed/modules.py:5-36,176-264). Activations are channels-last fp16
 * [B, H, W, C]; CircularPadding(p) (modules.py:5-19: rows zero-padded, columns wrapped, corners zero) is addressing
 * inside pf_conv_circ, no padded copy.
 * pf_faed_prep (FAED.py:70, Encoder.forward's x[:, :3], modules.py:249): src [B, C, H, W] uint8 (is_u8) or fp32, first
 * 3 channels -> dst fp16 [B, H, W, 16] = src / 127.5 - 1 in fp32, rounded once; channels 3..15 are zero. */
int pf_faed_prep(const void* src, int is_u8, int B, int C, int H, int W, void* dst, void* stream);
/* Conv2d = CircularPadding(pad) + unpadded nn.Conv2d (modules.py:22-36) with BN folded into w/bias, then ReLU (relu != 0),
 * then + residual (ResBlock, modules.py:59-65). x fp16 [B, H, W, Cin], w fp16 [k*k][Cin][Cout] (tap-major ky, kx), bias
 * fp32 [Cout], residual fp16 [B, Ho, Wo, Cout] or NULL, out [B, Ho, Wo, Cout] fp16 or fp32 (out_dtype PF_F16 / PF_F32).
 * Layers: k 3/5/7/9 stride 1 pad k/2, or k 4 stride 2 pad 1; Cin 16/32/64/128, Cout 32/64/128 (Cin >= 64 -> Cout 64/128,
 * Cin 16 -> Cout 32); anything else is PF_ERR_UNSUPPORTED. */
int pf_conv_circ(const void* x, int B, int H, int W, int Cin, const void* w, const float* bias, int Cout, int k,
                 int stride, int pad, int relu, const void* residual, void* out, int out_dtype, void* stream);
/* FAED.py:72-77: x fp32 [B, h, w, C] -> out fp32 [B, C*h], out[b, c*h + y] = weight[y] * mean_x x[b, y, x, c];
 * weight [h] = cos(linspace(pi/2, -pi/2, h)) in fp32 (device). */
int pf_faed_pool(const float* x, int B, int h, int w, int C, const float* weight, float* out, void* stream);
/* FAED.py:80-90: sum[d] += sum_i X[i], cov_sum[d, d] += X^T X in fp64 for X fp32 [n, d]; every element is summed over i in
 * order, so repeated calls give identical bits. */
int pf_faed_stats(const float* features, int n, int d, double* sum, double* cov_sum, void* stream);
/* FAED.py:92-103 + torchmetrics _compute_fid: out[0] = |mu1 - mu2|^2 + tr S1 + tr S2 - 2 sum sqrt(eig(S1 S2)) in fp64,
 * S = (cov_sum - n mu mu^T) / (n - 1), mu = sum / n. The square-root term is the nuclear norm of L1^T L2 with
 * S_i = L_i L_i^T, both from one-sided Jacobi iterations (negative rounding-level eigenvalues clamped to 0). ws: device,
 * pf_frechet_ws_doubles(d) doubles; d % 64 == 0; n1, n2 >= 2. sweeps: host int[3] (or NULL) <- the sweeps of the
 * Jacobi iterations on S1, S2 and L1^T L2. Synchronizes the stream once per Jacobi sweep; a Jacobi
 * that does not converge in 100 sweeps returns PF_ERR_UNSUPPORTED. */
long long pf_frechet_ws_doubles(int d);
int pf_frechet_fp64(const double* sum1, const double* cov_sum1, long long n1, const double* sum2,
                    const double* cov_sum2, long long n2, int d, double* ws, double* out, int* sweeps, void* stream);

/* ------------------------------------------------------------------------------------------------
 * FID and Inception Score (models/pano/EvalPanoGen.py:30-49: torchmetrics FrechetInceptionDistance / InceptionScore over
 * torch-fidelity's FeatureExtractorInceptionV3, the network of torchmetrics' NoTrainInceptionV3). Activations are
 * channels-last fp16 [B, H, W, C]. FID's statistics and distance are pf_faed_stats and pf_frechet_fp64 at d = 2048.
 * pf_inception_prep (FeatureExtractorInceptionV3.forward: x.float(), interpolate_bilinear_2d_like_tensorflow1x to
 * 299x299 with align_corners=False, method 'slow', then (x - 128) / 128): src [B, 3, H, W] uint8 (is_u8 = 1) or fp32 in
 * [0, 1] (is_u8 = 0: torchmetrics' normalize=True, (x * 255).byte() truncation applied per pixel) -> dst fp16
 * [B, 299, 299, 16], channels 3..15 zero. Each op is one fp32 op, as torch runs it. */
int pf_inception_prep(const void* src, int is_u8, int B, int H, int W, void* dst, void* stream);
/* Width Cw of pf_conv2d_nhwc's packed weight and bias: Cout rounded up to 32 if Cout <= 32, else to a multiple of 64. */
int pf_conv2d_packed_cout(int Cout);
/* BasicConv2d (conv without bias + BatchNorm(eps 1e-3) + ReLU) with BN folded into w / bias: zero-padded kh x kw
 * convolution (kh, kw <= 7, per-axis pad < k, stride 1 or 2, the same on both axes), then ReLU if relu != 0. The
 * implicit-GEMM mma.sync core of pf_conv_circ. x fp16 [B, H, W, Cin] with Cin % 16 == 0; w fp16 [kh*kw][Cin][Cw]
 * (tap-major ky, kx; zero columns past Cout); bias fp32 [Cw]. out fp16 or fp32 (out_dtype) [B, Ho, Wo, out_ld] of which
 * channels [out_off, out_off + Cout) are written and the rest left untouched: a branch writes its slice of the
 * concat buffer. Cout, out_ld and out_off even. */
int pf_conv2d_nhwc(const void* x, int B, int H, int W, int Cin, const void* w, const float* bias, int Cout, int kh,
                   int kw, int stride, int ph, int pw, int relu, void* out, int out_dtype, int out_ld, int out_off,
                   void* stream);
/* 3x3 pools of the FID InceptionV3 on fp16 [B, H, W, C] (C % 8 == 0) -> out [B, Ho, Wo, out_ld] channels
 * [out_off, out_off + C) (multiples of 8). PF_POOL_MAX: F.max_pool2d (stem, Mixed_6a / 7a with stride 2 pad 0; Mixed_7c's
 * pool branch with stride 1 pad 1). PF_POOL_AVG_EXCL_PAD: F.avg_pool2d(count_include_pad=False), fp32 sum in tap order,
 * rounded once (Mixed_5b..7b's pool branch, stride 1 pad 1). */
#define PF_POOL_MAX 0
#define PF_POOL_AVG_EXCL_PAD 1
int pf_pool2d_nhwc(const void* x, int B, int H, int W, int C, int mode, int stride, int pad, void* out, int out_ld,
                   int out_off, void* stream);
/* FeatureExtractorInceptionV3's head: x fp32 [B, HW, C] (Mixed_7c, HW = 8x8) -> pool3 fp32 [B, C] (the mean over HW,
 * adaptive_avg_pool2d) and logits fp32 [B, N] = pool3 @ fc_w^T with fc_w fp32 [N, C] ('logits_unbiased': no bias).
 * Every output is summed in a fixed order, independent of B. */
int pf_inception_head(const float* x, int B, int HW, int C, const float* fc_w, int N, float* pool3, float* logits,
                      void* stream);
/* torchmetrics InceptionScore.compute after its randperm: logits fp32 [n, C], perm int64 [n] (device) -> out fp32 [2] =
 * (mean, unbiased std) over the torch.chunk(splits) chunks (ceil(n / splits) rows each) of exp(mean KL(p || chunk mean
 * p)), computed in fp64; one chunk gives std = nan. ws: device, pf_inception_score_ws_doubles(n, C, splits) doubles. */
long long pf_inception_score_ws_doubles(int n, int C, int splits);
int pf_inception_score(const float* logits, const long long* perm, int n, int C, int splits, double* ws, float* out,
                       void* stream);

/* ------------------------------------------------------------------------------------------------
 * CLIP score (models/pano/EvalPanoGen.py:33-46: torchmetrics CLIPScore('openai/clip-vit-base-patch16') over
 * transformers' CLIPProcessor / CLIPModel). Both towers' layers run on pf_gemm_taps (PF_ACT_QUICK_GELU) and pf_fmha_fwd.
 * pf_clip_prep_taps (host only, no CUDA call): the tap table of CLIPImageProcessor's resize for an H x W image — short
 *   side to 224, long side to int(224 * long / short) (no resample when the short side is 224) with Pillow's 8-bit
 *   bicubic filter — restricted to the 224 columns and rows the centre crop keeps (left = (Wr - 224) / 2, top =
 *   (Hr - 224) / 2). taps: host, pf_clip_prep_taps_ints(H, W) ints = {Kx, Ky, 0, 0}, then per kept column (start,
 *   count, Kx coefficients), then per kept row (start, count, Ky coefficients); coefficients in 22-bit fixed point.
 * pf_clip_prep: src [B, 3, H, W] uint8 (is_u8 = 1) or fp32 in [0, 1] (is_u8 = 0: converted per pixel as
 *   uint8(x * 255), truncated) and taps (device copy of pf_clip_prep_taps(H, W)) -> out [B * 196, 768], fp16 or fp32
 *   (out_dtype): row b * 196 + py * 14 + px is patch (py, px) of the normalised 224 x 224 crop in the (c, kh, kw) order
 *   of patch_embedding.weight.reshape(768, -1). The resample is integer-only (bit-identical to PIL.Image.resize), the
 *   intermediate image never leaves registers; then x / 255 in fp64 rounded to fp32 and (x - mean) / std in fp32.
 * pf_clip_embed: patches fp32 [B * 196, C] (the patch-embedding GEMM) -> out 16-bit [B * 197, C] =
 *   pre_layrnorm(cat(class_emb, patches) + pos_emb) per image (class_emb [C], pos_emb [197, C], gamma, beta fp32), and
 *   row_stats [B * 197][2][2] = (sum, sum of squares, 0, 0) of each stored row, the ln_stats of layer 0's folded LN1
 *   (the layout of pf_embed_tokens). C % 64 == 0, C <= 1024.
 * pf_clip_score: img_emb, txt_emb fp32 [B, D] -> scores fp32 [B] = 100 * <img / |img|, txt / |txt|> in fp32, and
 *   score_sum[0] (fp64, device) += the scores summed in sample order: repeated runs give identical bits. */
int pf_clip_prep_taps_ints(int H, int W);
int pf_clip_prep_taps(int H, int W, int* taps);
int pf_clip_prep(const void* src, int is_u8, int B, int H, int W, const int* taps, void* out, int out_dtype,
                 void* stream);
int pf_clip_embed(const float* patches, const float* class_emb, const float* pos_emb, const float* gamma,
                  const float* beta, float eps, int B, int C, void* out, int dtype, float* row_stats, void* stream);
int pf_clip_score(const float* img_emb, const float* txt_emb, int B, int D, float* scores, double* score_sum,
                  void* stream);

/* ------------------------------------------------------------------------------------------------
 * View-sharded step (SURVEY.md 8e): device-initiated all-gather over NVLink peer mappings, capturable in a CUDA graph.
 * The reference has no model parallelism (Lightning DDP over prompts, main.py:63); this is the exchange the view partition
 * needs: models/pano/modules.py:44-48 lets every panorama query attend to the keys / values of ALL views, so each rank
 * publishes the projected K|V of its local views before every EPPA block (and the eps outputs at the end of the step).
 *   local         this rank's slice (slice_bytes, multiple of 16)
 *   peer_data     DEVICE array [nranks] of pointers: every rank's receive buffer [nranks][slice_bytes] for this call site,
 *                 mapped into this process (CUDA IPC / peer access); entry `rank` is the own buffer
 *   peer_flags    DEVICE array [nranks] of pointers to every rank's nranks flag words (zero-initialised, uint32)
 *   my_flags      == peer_flags[rank];  state: 2 zero-initialised uint32 of this rank (epoch, CTA counter)
 * On return (stream order) the own receive buffer holds every rank's slice in rank order. One kernel: push to all peers,
 * publish the epoch, wait for all peers; a peer that never arrives makes the kernel trap after ~15 s instead of hanging. */
/* Receive buffers of the device-side collectives: cudaMalloc'ed (zero-filled) by pf_comm_alloc, exported as a 64-byte CUDA IPC
 * handle, opened by the peers ON THEIR device (cudaIpcOpenMemHandle with lazy peer access — NVLink on an HGX board). */
int pf_comm_alloc(long long bytes, void** ptr);
int pf_comm_free(void* ptr);
int pf_ipc_export(const void* ptr, unsigned char handle[64]);
int pf_ipc_open(const unsigned char handle[64], void** ptr);
int pf_ipc_close(void* ptr);
/* let kernels of the CURRENT device store into memory of `peer_device` (cudaDeviceEnablePeerAccess; idempotent) — needed once
 * per peer before pf_allgather_views pushes into IPC-mapped buffers that live on the other GPUs of the node */
int pf_enable_peer_access(int peer_device);
int pf_allgather_views(const void* local, long long slice_bytes, void* const* peer_data, unsigned int* const* peer_flags,
                       unsigned int* my_flags, unsigned int* state, int rank, int nranks, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PANFUSION_B200_H */
