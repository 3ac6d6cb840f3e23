// FID / Inception Score (torchmetrics FrechetInceptionDistance / InceptionScore over torch-fidelity's
// FeatureExtractorInceptionV3, as EvalPanoGen builds them, models/pano/EvalPanoGen.py:30-49): the TF1-style resize
// and normalisation, the zero-padded convolutions of the FID InceptionV3 (on the implicit-GEMM core shared with FAED),
// its pools, the pool3 / logits head and the Inception Score reduction.
//
// Activations are channels-last fp16 [B, H, W, C]; Mixed_7c writes fp32 so the head reads fp32.
#include "conv_mma.cuh"

namespace pf {
namespace inception {

constexpr int kPrepC = 16;  // 3 image channels + 13 zero channels: the first layer's one 16-wide MMA k-step
constexpr int kSize = 299;  // torch-fidelity's input resolution

// ---------------------------------------------------------------------------------------------------------------------
// pf_inception_prep: torch-fidelity's interpolate_bilinear_2d_like_tensorflow1x (align_corners=False, 'slow') to
// 299x299, then (x - 128) / 128, rounded once to fp16. Every step is one fp32 op (no FMA contraction), as torch runs it.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float load_px(const void* src, int is_u8, size_t i) {
  if (is_u8) return (float)static_cast<const uint8_t*>(src)[i];
  // torchmetrics' normalize=True: (imgs * 255).byte(), which truncates (inputs in [0, 1])
  const float v = __fmul_rn(static_cast<const float*>(src)[i], 255.f);
  return truncf(fminf(fmaxf(v, 0.f), 255.f));
}

__global__ void __launch_bounds__(256)
prep_kernel(const void* __restrict__ src, int is_u8, int B, int H, int W, float sy, float sx,
            __half* __restrict__ dst) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  constexpr long long HW = (long long)kSize * kSize;
  if (idx >= B * HW) return;
  const int b = (int)(idx / HW), oy = (int)(idx % HW) / kSize, ox = (int)(idx % HW) % kSize;
  const float gy = __fmul_rn((float)oy, sy), gx = __fmul_rn((float)ox, sx);
  const int y0 = (int)gy, x0 = (int)gx;  // g >= 0: .long() truncates
  const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
  const float dy = __fsub_rn(gy, (float)y0), dx = __fsub_rn(gx, (float)x0);
  __align__(16) __half v[kPrepC];
#pragma unroll
  for (int c = 0; c < kPrepC; ++c) v[c] = __float2half_rn(0.f);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const size_t base = ((size_t)b * 3 + c) * H * W;
    const float a00 = load_px(src, is_u8, base + (size_t)y0 * W + x0);
    const float a01 = load_px(src, is_u8, base + (size_t)y0 * W + x1);
    const float a10 = load_px(src, is_u8, base + (size_t)y1 * W + x0);
    const float a11 = load_px(src, is_u8, base + (size_t)y1 * W + x1);
    const float r0 = __fadd_rn(a00, __fmul_rn(__fsub_rn(a01, a00), dx));
    const float r1 = __fadd_rn(a10, __fmul_rn(__fsub_rn(a11, a10), dx));
    const float o = __fadd_rn(r0, __fmul_rn(__fsub_rn(r1, r0), dy));
    v[c] = __float2half_rn(__fdiv_rn(__fsub_rn(o, 128.f), 128.f));
  }
  uint4* d = reinterpret_cast<uint4*>(dst + idx * kPrepC);
  d[0] = reinterpret_cast<const uint4*>(v)[0];
  d[1] = reinterpret_cast<const uint4*>(v)[1];
}

// ---------------------------------------------------------------------------------------------------------------------
// pf_pool2d_nhwc: 3x3 max (padding never wins) or average with count_include_pad=False (fp32 sum in tap order), fp16
// in and out, 8 channels per thread, written at out[pixel * out_ld + out_off + c].
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
pool_kernel(const __half* __restrict__ x, int B, int H, int W, int C, int avg, int stride, int pad, int Ho, int Wo,
            __half* __restrict__ out, int out_ld, int out_off) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int G = C / 8;
  if (idx >= (long long)B * Ho * Wo * G) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int ox = (int)(pix % Wo), oy = (int)(pix / Wo % Ho), b = (int)(pix / ((long long)Wo * Ho));
  float s[8];
  __half2 mx[4];
#pragma unroll
  for (int q = 0; q < 8; ++q) s[q] = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) mx[q] = __half2half2(__ushort_as_half((unsigned short)0xFC00));  // -inf
  int cnt = 0;
  for (int ky = 0; ky < 3; ++ky) {
    const int iy = oy * stride - pad + ky;
    if (iy < 0 || iy >= H) continue;
    for (int kx = 0; kx < 3; ++kx) {
      const int ix = ox * stride - pad + kx;
      if (ix < 0 || ix >= W) continue;
      const uint4 raw = *reinterpret_cast<const uint4*>(x + (((size_t)b * H + iy) * W + ix) * C + g * 8);
      const __half2* h = reinterpret_cast<const __half2*>(&raw);
      ++cnt;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (avg) {
          const float2 f = __half22float2(h[q]);
          s[2 * q] = __fadd_rn(s[2 * q], f.x);
          s[2 * q + 1] = __fadd_rn(s[2 * q + 1], f.y);
        } else {
          mx[q] = __hmax2(mx[q], h[q]);
        }
      }
    }
  }
  __align__(16) __half2 o[4];
#pragma unroll
  for (int q = 0; q < 4; ++q)
    o[q] = avg ? __floats2half2_rn(__fdiv_rn(s[2 * q], (float)cnt), __fdiv_rn(s[2 * q + 1], (float)cnt)) : mx[q];
  *reinterpret_cast<uint4*>(out + (size_t)pix * out_ld + out_off + g * 8) = *reinterpret_cast<const uint4*>(o);
}

// ---------------------------------------------------------------------------------------------------------------------
// pf_inception_head: pool3 = the fp32 mean over the HW positions (summed in order), logits = pool3 @ fc_w^T in fp32, one
// warp per output with a fixed lane order, so a row's values do not depend on the batch.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
mean_kernel(const float* __restrict__ x, int B, int HW, int C, float* __restrict__ pool3) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * C) return;
  const int b = idx / C, c = idx % C;
  const float* p = x + (size_t)b * HW * C + c;
  float s = 0.f;
  for (int i = 0; i < HW; ++i) s = __fadd_rn(s, p[(size_t)i * C]);
  pool3[idx] = __fdiv_rn(s, (float)HW);
}

__global__ void __launch_bounds__(256)
fc_kernel(const float* __restrict__ pool3, int B, int C, const float* __restrict__ w, int N, float* __restrict__ out) {
  const int o = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (o >= B * N) return;
  const int b = o / N, n = o % N;
  const float* x = pool3 + (size_t)b * C;
  const float* wr = w + (size_t)n * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s = __fmaf_rn(x[c], wr[c], s);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if (lane == 0) out[o] = s;
}

// ---------------------------------------------------------------------------------------------------------------------
// pf_inception_score: torchmetrics InceptionScore.compute in fp64 after the host's randperm: gather, softmax and
// log_softmax per row, torch.chunk into ceil(n / splits)-row chunks, KL of each row to its chunk's mean probability,
// exp(mean KL) per chunk, then the mean and the unbiased std over the chunks.
// ---------------------------------------------------------------------------------------------------------------------
__device__ double block_reduce(double v, double* red, bool is_max) {
  // fixed-order tree over 256 threads
  const int t = threadIdx.x;
  red[t] = v;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if (t < off) red[t] = is_max ? fmax(red[t], red[t + off]) : red[t] + red[t + off];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(256)
softmax_kernel(const float* __restrict__ logits, const long long* __restrict__ perm, int C, double* __restrict__ prob,
               double* __restrict__ logp) {
  __shared__ double red[256];
  const int i = blockIdx.x;
  const float* x = logits + (size_t)perm[i] * C;
  double m = -INFINITY;
  for (int c = threadIdx.x; c < C; c += 256) m = fmax(m, (double)x[c]);
  m = block_reduce(m, red, true);
  double s = 0.0;
  for (int c = threadIdx.x; c < C; c += 256) s += exp((double)x[c] - m);
  s = block_reduce(s, red, false);
  const double ls = log(s);
  for (int c = threadIdx.x; c < C; c += 256) {
    const double z = (double)x[c] - m;
    prob[(size_t)i * C + c] = exp(z) / s;
    logp[(size_t)i * C + c] = z - ls;
  }
}

// log of chunk k's mean probability of class c
__global__ void __launch_bounds__(256)
chunk_mean_kernel(const double* __restrict__ prob, int n, int C, int cs, double* __restrict__ logm) {
  const int k = blockIdx.y, c = blockIdx.x * 256 + threadIdx.x;
  if (c >= C) return;
  const int r0 = k * cs, r1 = min(n, r0 + cs);
  double s = 0.0;
  for (int r = r0; r < r1; ++r) s += prob[(size_t)r * C + c];
  logm[(size_t)k * C + c] = log(s / (double)(r1 - r0));
}

__global__ void __launch_bounds__(256)
chunk_kl_kernel(const double* __restrict__ prob, const double* __restrict__ logp, const double* __restrict__ logm,
                int n, int C, int cs, double* __restrict__ kl) {
  __shared__ double red[256];
  const int k = blockIdx.x, r0 = k * cs, r1 = min(n, r0 + cs);
  double s = 0.0;
  for (int r = r0; r < r1; ++r)
    for (int c = threadIdx.x; c < C; c += 256) {
      const size_t e = (size_t)r * C + c;
      s += prob[e] * (logp[e] - logm[(size_t)k * C + c]);
    }
  s = block_reduce(s, red, false);
  if (threadIdx.x == 0) kl[k] = exp(s / (double)(r1 - r0));
}

__global__ void score_kernel(const double* kl, int chunks, float* out) {
  double mean = 0.0, ss = 0.0;
  for (int k = 0; k < chunks; ++k) mean += kl[k];
  mean /= chunks;
  for (int k = 0; k < chunks; ++k) ss += (kl[k] - mean) * (kl[k] - mean);
  out[0] = (float)mean;
  out[1] = (float)sqrt(ss / (double)(chunks - 1));  // one chunk: 0 / 0 = nan, as torch.std gives
}

}  // namespace inception
}  // namespace pf

using namespace pf;
using namespace pf::inception;
using pf::convmma::ConvArgs;
using pf::convmma::launch_conv;

extern "C" int pf_inception_prep(const void* src, int is_u8, int B, int H, int W, void* dst, void* stream) {
  PF_CHECK_ARG(src && dst, "pf_inception_prep: null pointer");
  PF_CHECK_ARG(B > 0 && H > 0 && W > 0 && (long long)B * 3 * H * W < (1LL << 40) &&
                   (long long)B * kSize * kSize < (1LL << 31),
               "pf_inception_prep: bad shape B=%d H=%d W=%d", B, H, W);
  // torch-fidelity computes in / out in Python (double) and rounds it to an fp32 tensor
  const float sy = (float)((double)H / kSize), sx = (float)((double)W / kSize);
  const long long n = (long long)B * kSize * kSize;
  prep_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, is_u8, B, H, W, sy, sx, static_cast<__half*>(dst));
  PF_CHECK_LAUNCH("inception prep_kernel");
  return PF_OK;
}

extern "C" int pf_conv2d_packed_cout(int Cout) { return Cout <= 32 ? 32 : (Cout + 63) / 64 * 64; }

extern "C" int pf_conv2d_nhwc(const void* x, int B, int H, int W, int Cin, const void* w, const float* bias, int Cout,
                              int kh, int kw, int stride, int ph, int pw, int relu, void* out, int out_dtype,
                              int out_ld, int out_off, void* stream) {
  PF_CHECK_ARG(x && w && bias && out, "pf_conv2d_nhwc: null pointer");
  PF_CHECK_ARG(out_dtype == PF_F16 || out_dtype == PF_F32, "pf_conv2d_nhwc: out_dtype must be PF_F16 or PF_F32");
  PF_CHECK_ARG(B > 0 && H > 0 && W > 0 && Cin > 0 && Cin % 16 == 0 && Cout > 0 && Cout % 2 == 0,
               "pf_conv2d_nhwc: bad shape B=%d H=%d W=%d Cin=%d Cout=%d (Cin % 16 == 0, even Cout)", B, H, W, Cin,
               Cout);
  PF_CHECK_ARG(kh >= 1 && kh <= 7 && kw >= 1 && kw <= 7 && (stride == 1 || stride == 2) && ph >= 0 && ph < kh &&
                   pw >= 0 && pw < kw,
               "pf_conv2d_nhwc: kernel %dx%d stride %d pad (%d, %d) unsupported (k <= 7, stride 1/2, pad < k)", kh,
               kw, stride, ph, pw);
  PF_CHECK_ARG(out_ld % 2 == 0 && out_off % 2 == 0 && out_off >= 0 && out_off + Cout <= out_ld,
               "pf_conv2d_nhwc: output slice [%d, %d) of row stride %d (even offset and stride)", out_off,
               out_off + Cout, out_ld);
  const int Ho = (H + 2 * ph - kh) / stride + 1, Wo = (W + 2 * pw - kw) / stride + 1;
  PF_CHECK_ARG(H + 2 * ph >= kh && W + 2 * pw >= kw, "pf_conv2d_nhwc: image %dx%d smaller than the kernel", H, W);
  const long long M = (long long)B * Ho * Wo;
  PF_CHECK_ARG(M < (1LL << 31) && (long long)B * H * W < (1LL << 31), "pf_conv2d_nhwc: tensor too large");
  const int Cw = pf_conv2d_packed_cout(Cout);
  ConvArgs a{static_cast<const __half*>(x), static_cast<const __half*>(w), bias, nullptr, out, B, H, W, Cin, Cout,
             Ho, Wo, kh, kw, stride, ph, pw, relu, out_dtype == PF_F32, Cw, out_ld, out_off, (int)M};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int kc = Cin % 64 == 0 ? 64 : (Cin % 32 == 0 ? 32 : 16);
  if (Cw == 32) return kc == 16 ? launch_conv<16, 32, false>(a, st) : launch_conv<32, 32, false>(a, st);  // <64, 32> spills
  if (kc == 16) return launch_conv<16, 64, false>(a, st);
  if (kc == 32) return launch_conv<32, 64, false>(a, st);
  return launch_conv<64, 64, false>(a, st);
}

extern "C" int pf_pool2d_nhwc(const void* x, int B, int H, int W, int C, int mode, int stride, int pad, void* out,
                              int out_ld, int out_off, void* stream) {
  PF_CHECK_ARG(x && out, "pf_pool2d_nhwc: null pointer");
  PF_CHECK_ARG(mode == PF_POOL_MAX || mode == PF_POOL_AVG_EXCL_PAD, "pf_pool2d_nhwc: unknown mode %d", mode);
  PF_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && (stride == 1 || stride == 2) && (pad == 0 || pad == 1)
                   && H + 2 * pad >= 3 && W + 2 * pad >= 3,
               "pf_pool2d_nhwc: bad shape B=%d H=%d W=%d C=%d stride=%d pad=%d (C %% 8 == 0, 3x3, stride 1/2, pad 0/1)",
               B, H, W, C, stride, pad);
  PF_CHECK_ARG(out_ld % 8 == 0 && out_off % 8 == 0 && out_off >= 0 && out_off + C <= out_ld,
               "pf_pool2d_nhwc: output slice [%d, %d) of row stride %d (multiples of 8)", out_off, out_off + C, out_ld);
  const int Ho = (H + 2 * pad - 3) / stride + 1, Wo = (W + 2 * pad - 3) / stride + 1;
  const long long n = (long long)B * Ho * Wo * (C / 8);
  PF_CHECK_ARG((long long)B * H * W * C < (1LL << 40) && n < (1LL << 31), "pf_pool2d_nhwc: tensor too large");
  pool_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(x), B, H, W, C, mode == PF_POOL_AVG_EXCL_PAD, stride, pad, Ho, Wo,
      static_cast<__half*>(out), out_ld, out_off);
  PF_CHECK_LAUNCH("inception pool_kernel");
  return PF_OK;
}

extern "C" int pf_inception_head(const float* x, int B, int HW, int C, const float* fc_w, int N, float* pool3,
                                 float* logits, void* stream) {
  PF_CHECK_ARG(x && fc_w && pool3 && logits, "pf_inception_head: null pointer");
  PF_CHECK_ARG(B > 0 && HW > 0 && C > 0 && N > 0 && (long long)B * HW * C < (1LL << 40) &&
                   (long long)B * N < (1LL << 31) && (long long)B * C < (1LL << 31),
               "pf_inception_head: bad shape B=%d HW=%d C=%d N=%d", B, HW, C, N);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  mean_kernel<<<(B * C + 255) / 256, 256, 0, st>>>(x, B, HW, C, pool3);
  fc_kernel<<<(unsigned)(((long long)B * N + 7) / 8), 256, 0, st>>>(pool3, B, C, fc_w, N, logits);
  PF_CHECK_LAUNCH("inception head");
  return PF_OK;
}

extern "C" long long pf_inception_score_ws_doubles(int n, int C, int splits) {
  return 2LL * n * C + (long long)splits * (C + 1);
}

extern "C" int pf_inception_score(const float* logits, const long long* perm, int n, int C, int splits, double* ws,
                                  float* out, void* stream) {
  PF_CHECK_ARG(logits && perm && ws && out, "pf_inception_score: null pointer");
  PF_CHECK_ARG(n > 0 && C > 0 && splits > 0 && (long long)n * C < (1LL << 31),
               "pf_inception_score: bad shape n=%d C=%d splits=%d", n, C, splits);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int cs = (n + splits - 1) / splits, chunks = (n + cs - 1) / cs;  // torch.chunk
  double *prob = ws, *logp = ws + (size_t)n * C, *logm = logp + (size_t)n * C, *kl = logm + (size_t)splits * C;
  softmax_kernel<<<n, 256, 0, st>>>(logits, perm, C, prob, logp);
  chunk_mean_kernel<<<dim3((C + 255) / 256, chunks), 256, 0, st>>>(prob, n, C, cs, logm);
  chunk_kl_kernel<<<chunks, 256, 0, st>>>(prob, logp, logm, n, C, cs, kl);
  score_kernel<<<1, 1, 0, st>>>(kl, chunks, out);
  PF_CHECK_LAUNCH("inception score");
  return PF_OK;
}
