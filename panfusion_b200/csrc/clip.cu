// CLIP score (torchmetrics CLIPScore over transformers' CLIPProcessor / CLIPModel, as models/pano/EvalPanoGen.py:33-46
// builds it): CLIPImageProcessor's Pillow bicubic resize, centre crop and normalisation written as ViT-B/16 patch rows,
// the vision embeddings with pre_layrnorm, and the cosine-score reduction. The transformer layers of both towers run on
// pf_gemm_taps (PF_ACT_QUICK_GELU) and pf_fmha_fwd.
#include <math.h>

#include <vector>

#include "pf_common.cuh"

namespace pf {
namespace clip {

constexpr int kSize = 224;               // CLIPImageProcessor's shortest_edge and crop_size
constexpr int kPatch = 16;               // ViT-B/16
constexpr int kGrid = kSize / kPatch;    // 14 x 14 patches
constexpr int kPrecision = 22;           // Pillow's 8-bit resample: 32 - 8 - 2 fractional bits
constexpr int kTapHeader = 4;            // Kx, Ky, 0, 0

// ---------------------------------------------------------------------------------------------------------------------
// Host: the tap tables of Pillow's 8-bit bicubic resample (a = -0.5), for the 224 output columns / rows that survive the
// centre crop. Coefficients are evaluated in double in Pillow's order, normalised by their sum, then rounded half away
// from zero to 22-bit fixed point.
// ---------------------------------------------------------------------------------------------------------------------
static double bicubic(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

static int axis_ksize(int in, int out) {
  const double scale = (double)in / out, fs = scale < 1.0 ? 1.0 : scale;
  return (int)ceil(2.0 * fs) * 2 + 1;
}

// rows [first, first + kSize) of an in -> out resample: per row (start, count, coeffs[ksize])
static void axis_taps(int in, int out, int first, int ksize, int* dst) {
  const double scale = (double)in / out, fs = scale < 1.0 ? 1.0 : scale, support = 2.0 * fs, ss = 1.0 / fs;
  std::vector<double> k(ksize);
  for (int i = 0; i < kSize; ++i) {
    const int xx = first + i;
    const double center = (xx + 0.5) * scale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in) xmax = in;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      const double w = bicubic((x + xmin - center + 0.5) * ss);
      k[x] = w;
      ww += w;
    }
    int* row = dst + (size_t)i * (2 + ksize);
    row[0] = xmin;
    row[1] = xmax;
    for (int x = 0; x < ksize; ++x) {
      const double v = x < xmax ? (ww != 0.0 ? k[x] / ww : k[x]) : 0.0;
      row[2 + x] = v < 0 ? (int)(-0.5 + v * (1 << kPrecision)) : (int)(0.5 + v * (1 << kPrecision));
    }
  }
}

// CLIPImageProcessor (transformers 4.26.1): short side -> 224, long side -> int(224 * long / short); no resample when
// the short side is already 224
static void resized(int H, int W, int* Hr, int* Wr) {
  const int s = H < W ? H : W;
  if (s == kSize) {
    *Hr = H, *Wr = W;
  } else if (W <= H) {
    *Wr = kSize, *Hr = (int)((double)(kSize * (long long)H) / W);
  } else {
    *Hr = kSize, *Wr = (int)((double)(kSize * (long long)W) / H);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// pf_clip_prep: one thread per output element of the patch rows. The vertical pass sums the horizontal pass's uint8
// results of its tap rows, each computed in registers from the source; both passes accumulate in int32 from 1 << 21
// and clip (x >> 22) to [0, 255], as Pillow does. Then rescale (double) and normalise (float), one rounding per op.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int clip8(int v) {
  v >>= kPrecision;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

__device__ __forceinline__ int load_u8(const void* src, int is_u8, size_t i) {
  if (is_u8) return static_cast<const uint8_t*>(src)[i];
  // to_pil_image of a float image: (x * 255).astype(uint8), a truncation (inputs in [0, 1])
  const float v = __fmul_rn(static_cast<const float*>(src)[i], 255.f);
  return (int)truncf(fminf(fmaxf(v, 0.f), 255.f));
}

__global__ void __launch_bounds__(256)
prep_kernel(const void* __restrict__ src, int is_u8, int B, int H, int W, const int* __restrict__ taps,
            void* __restrict__ out, int out_f32) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  constexpr int kRow = 3 * kPatch * kPatch;  // 768 = (c, kh, kw)
  if (idx >= (long long)B * kGrid * kGrid * kRow) return;
  const int col = (int)(idx % kRow);
  const long long prow = idx / kRow;
  const int b = (int)(prow / (kGrid * kGrid)), p = (int)(prow % (kGrid * kGrid));
  const int c = col >> 8, y = (p / kGrid) * kPatch + ((col >> 4) & 15), x = (p % kGrid) * kPatch + (col & 15);
  const int Kx = __ldg(taps), Ky = __ldg(taps + 1);
  const int* tx = taps + kTapHeader + x * (2 + Kx);
  const int* ty = taps + kTapHeader + kSize * (2 + Kx) + y * (2 + Ky);
  const int x0 = __ldg(tx), nx = __ldg(tx + 1), y0 = __ldg(ty), ny = __ldg(ty + 1);
  const size_t plane = ((size_t)b * 3 + c) * H * W;
  int acc = 1 << (kPrecision - 1);
  for (int j = 0; j < ny; ++j) {
    const size_t r = plane + (size_t)(y0 + j) * W + x0;
    int h = 1 << (kPrecision - 1);
    for (int i = 0; i < nx; ++i) h += load_u8(src, is_u8, r + i) * __ldg(tx + 2 + i);
    acc += clip8(h) * __ldg(ty + 2 + j);
  }
  const int u = clip8(acc);
  // rescale(1/255): uint8 * Python float in float64, cast to float32; normalize in float32 with OpenAI's mean / std
  const float mean = c == 0 ? (float)0.48145466 : (c == 1 ? (float)0.4578275 : (float)0.40821073);
  const float stdv = c == 0 ? (float)0.26862954 : (c == 1 ? (float)0.26130258 : (float)0.27577711);
  const float v = __double2float_rn(__dmul_rn((double)u, 1.0 / 255.0));
  const float o = __fdiv_rn(__fsub_rn(v, mean), stdv);
  if (out_f32)
    static_cast<float*>(out)[idx] = o;
  else
    static_cast<__half*>(out)[idx] = __float2half_rn(o);
}

// ---------------------------------------------------------------------------------------------------------------------
// pf_clip_embed: one warp per output row; e = (row 0: class_embedding, else the patch row) + position, then
// pre_layrnorm (two-pass fp32 statistics over the row held in registers), stored 16-bit with the (sum, sum of squares)
// of the stored row for layer 0's folded LayerNorm.
// ---------------------------------------------------------------------------------------------------------------------
template <bool BF16>
__global__ void __launch_bounds__(256)
embed_kernel(const float* __restrict__ patches, const float* __restrict__ cls, const float* __restrict__ pos,
             const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int B, int P, int C,
             uint16_t* __restrict__ out, float* __restrict__ stats) {
  const int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (t >= B * (P + 1)) return;
  const int b = t / (P + 1), r = t % (P + 1);
  const float* src = r == 0 ? cls : patches + ((size_t)b * P + r - 1) * C;
  const float* pr = pos + (size_t)r * C;
  const int n = C / 64;
  float2 e[16];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    if (i < n) {
      const int c = i * 64 + lane * 2;
      const float2 v = __ldg(reinterpret_cast<const float2*>(src + c)), q = __ldg(reinterpret_cast<const float2*>(pr + c));
      e[i] = make_float2(v.x + q.x, v.y + q.y);
      s += e[i].x + e[i].y;
    }
  }
  const float mean = warp_sum(s) / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    if (i < n) {
      const float dx = e[i].x - mean, dy = e[i].y - mean;
      q = fmaf(dx, dx, fmaf(dy, dy, q));
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
  float ss = 0.f, sq = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    if (i < n) {
      const int c = i * 64 + lane * 2;
      const float2 g = __ldg(reinterpret_cast<const float2*>(gamma + c)), be = __ldg(reinterpret_cast<const float2*>(beta + c));
      const uint32_t w = pack2<BF16>(fmaf((e[i].x - mean) * rstd, g.x, be.x), fmaf((e[i].y - mean) * rstd, g.y, be.y));
      const float2 st = unpack2<BF16>(w);  // statistics of the stored 16-bit row
      ss += st.x + st.y;
      sq = fmaf(st.x, st.x, fmaf(st.y, st.y, sq));
      *reinterpret_cast<uint32_t*>(out + (size_t)t * C + c) = w;
    }
  }
  ss = warp_sum(ss);
  sq = warp_sum(sq);
  if (lane == 0) reinterpret_cast<float4*>(stats)[t] = make_float4(ss, sq, 0.f, 0.f);
}

// ---------------------------------------------------------------------------------------------------------------------
// pf_clip_score: one CTA. Warp w scores samples w, w + 8, ... in fp32 (norms, normalised products, 100x) with a fixed
// lane order; thread 0 then adds the scores in sample order in fp64 to the state.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
score_kernel(const float* __restrict__ img, const float* __restrict__ txt, int B, int D, float* __restrict__ scores,
             double* __restrict__ state) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int b = w; b < B; b += 8) {
    const float* ip = img + (size_t)b * D;
    const float* tp = txt + (size_t)b * D;
    float si = 0.f, st = 0.f;
    for (int d = lane; d < D; d += 32) {
      si = fmaf(ip[d], ip[d], si);
      st = fmaf(tp[d], tp[d], st);
    }
    const float ni = sqrtf(warp_sum(si)), nt = sqrtf(warp_sum(st));
    float dot = 0.f;
    for (int d = lane; d < D; d += 32) dot = fmaf(__fdiv_rn(ip[d], ni), __fdiv_rn(tp[d], nt), dot);
    dot = warp_sum(dot);
    if (lane == 0) scores[b] = __fmul_rn(100.f, dot);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int b = 0; b < B; ++b) s += (double)scores[b];
    *state += s;
  }
}

}  // namespace clip
}  // namespace pf

using namespace pf;
using namespace pf::clip;

extern "C" int pf_clip_prep_taps_ints(int H, int W) {
  if (H <= 0 || W <= 0) return 0;
  int Hr, Wr;
  resized(H, W, &Hr, &Wr);
  return kTapHeader + kSize * (4 + axis_ksize(W, Wr) + axis_ksize(H, Hr));
}

extern "C" int pf_clip_prep_taps(int H, int W, int* taps) {
  PF_CHECK_ARG(taps, "pf_clip_prep_taps: null pointer");
  PF_CHECK_ARG(H > 0 && W > 0 && H < (1 << 16) && W < (1 << 16), "pf_clip_prep_taps: bad size %dx%d", H, W);
  int Hr, Wr;
  resized(H, W, &Hr, &Wr);
  const int Kx = axis_ksize(W, Wr), Ky = axis_ksize(H, Hr);
  taps[0] = Kx, taps[1] = Ky, taps[2] = 0, taps[3] = 0;
  axis_taps(W, Wr, (Wr - kSize) / 2, Kx, taps + kTapHeader);
  axis_taps(H, Hr, (Hr - kSize) / 2, Ky, taps + kTapHeader + kSize * (2 + Kx));
  return PF_OK;
}

extern "C" int pf_clip_prep(const void* src, int is_u8, int B, int H, int W, const int* taps, void* out, int out_dtype,
                            void* stream) {
  PF_CHECK_ARG(src && taps && out, "pf_clip_prep: null pointer");
  PF_CHECK_ARG(out_dtype == PF_F16 || out_dtype == PF_F32, "pf_clip_prep: out_dtype must be PF_F16 or PF_F32");
  PF_CHECK_ARG(B > 0 && H > 0 && W > 0 && H < (1 << 16) && W < (1 << 16) && (long long)B * 3 * H * W < (1LL << 40) &&
                   (long long)B * kGrid * kGrid * 3 * kPatch * kPatch < (1LL << 40),
               "pf_clip_prep: bad shape B=%d H=%d W=%d", B, H, W);
  PF_CHECK_ARG((reinterpret_cast<uintptr_t>(taps) & 3) == 0 && (is_u8 || (reinterpret_cast<uintptr_t>(src) & 3) == 0) &&
                   (reinterpret_cast<uintptr_t>(out) & (out_dtype == PF_F32 ? 3 : 1)) == 0,
               "pf_clip_prep: misaligned operand");
  const long long n = (long long)B * kGrid * kGrid * 3 * kPatch * kPatch;
  prep_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, is_u8, B, H, W, taps, out, out_dtype == PF_F32);
  PF_CHECK_LAUNCH("clip prep_kernel");
  return PF_OK;
}

extern "C" int pf_clip_embed(const float* patches, const float* class_emb, const float* pos_emb, const float* gamma,
                             const float* beta, float eps, int B, int C, void* out, int dtype, float* row_stats,
                             void* stream) {
  PF_CHECK_ARG(patches && class_emb && pos_emb && gamma && beta && out && row_stats, "pf_clip_embed: null pointer");
  PF_CHECK_ARG(dtype == PF_BF16 || dtype == PF_F16, "pf_clip_embed: 16-bit output required");
  PF_CHECK_ARG(B > 0 && C > 0 && C % 64 == 0 && C <= 1024 && (long long)B * (kGrid * kGrid + 1) * 32 < (1LL << 31),
               "pf_clip_embed: bad shape B=%d C=%d (C %% 64 == 0, C <= 1024)", B, C);
  // float2 loads of the fp32 operands, 4-byte stores of the 16-bit pairs, one float4 of statistics per row
  PF_CHECK_ARG(((reinterpret_cast<uintptr_t>(patches) | reinterpret_cast<uintptr_t>(class_emb) |
                 reinterpret_cast<uintptr_t>(pos_emb) | reinterpret_cast<uintptr_t>(gamma) |
                 reinterpret_cast<uintptr_t>(beta)) & 7) == 0 &&
                   (reinterpret_cast<uintptr_t>(out) & 3) == 0 && (reinterpret_cast<uintptr_t>(row_stats) & 15) == 0,
               "pf_clip_embed: fp32 operands must be 8-byte, out 4-byte and row_stats 16-byte aligned");
  const int P = kGrid * kGrid, blocks = (B * (P + 1) + 7) / 8;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PF_BF16)
    embed_kernel<true><<<blocks, 256, 0, st>>>(patches, class_emb, pos_emb, gamma, beta, eps, B, P, C,
                                                static_cast<uint16_t*>(out), row_stats);
  else
    embed_kernel<false><<<blocks, 256, 0, st>>>(patches, class_emb, pos_emb, gamma, beta, eps, B, P, C,
                                                 static_cast<uint16_t*>(out), row_stats);
  PF_CHECK_LAUNCH("clip embed_kernel");
  return PF_OK;
}

extern "C" int pf_clip_score(const float* img_emb, const float* txt_emb, int B, int D, float* scores, double* score_sum,
                             void* stream) {
  PF_CHECK_ARG(img_emb && txt_emb && scores && score_sum, "pf_clip_score: null pointer");
  PF_CHECK_ARG(B > 0 && D > 0 && (long long)B * D < (1LL << 31), "pf_clip_score: bad shape B=%d D=%d", B, D);
  PF_CHECK_ARG(((reinterpret_cast<uintptr_t>(img_emb) | reinterpret_cast<uintptr_t>(txt_emb) |
                 reinterpret_cast<uintptr_t>(scores)) & 3) == 0 && (reinterpret_cast<uintptr_t>(score_sum) & 7) == 0,
               "pf_clip_score: misaligned operand");
  score_kernel<<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(img_emb, txt_emb, B, D, scores, score_sum);
  PF_CHECK_LAUNCH("clip score_kernel");
  return PF_OK;
}
