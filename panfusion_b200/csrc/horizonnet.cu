// HorizonNet's layout network (external/HorizonNet/model.py HorizonNet('resnet50', use_rnn=True), the `net` of
// models/horizonnet/HorizonNet.py): input normalisation, the circular-padded ResNet-50 and GlobalHeightStage
// convolutions (on the implicit-GEMM core of conv_mma.cuh), GlobalHeightConv's width upsampling, the recurrence of the
// two-layer bidirectional LSTM (its input projections run on pf_gemm_taps) and the Linear(1024, 12) head.
//
// Activations are channels-last fp16 [B, H, W, C]. wrap_lr_pad turns every convolution with W padding p into
// LR_PAD(p) + Conv2d(padding=(p, 0)): rows zero-padded, columns wrapped, corners zero. That is the CIRC addressing of
// conv_mma.cuh (a no-op for 1x1), so no padded copy is made.
#include <cooperative_groups.h>

#include "conv_mma.cuh"

namespace cg = cooperative_groups;

namespace pf {
namespace hnet {

constexpr int kPrepC = 16;  // the stem's operand: 3 image channels + 13 zero channels (one 16-wide MMA k-step)
constexpr int kH = 512, kW = 1024;
constexpr int kHidden = 512;                  // LSTM hidden size
constexpr int kGates = 4 * kHidden;           // gate rows per direction (i, f, g, o)
constexpr int kFeat = 1024;                   // LSTM input width and [fwd | bwd] output width
constexpr int kCluster = 16;                  // CTAs per direction
constexpr int kUnits = kHidden / kCluster;    // hidden units per CTA
constexpr int kRows = 4 * kUnits;             // W_hh rows per CTA
constexpr int kMaxB = 16;                     // samples per pf_lstm_bidir launch
constexpr int kLstmThreads = 256;
constexpr size_t kLstmSmem = (size_t)kRows * kHidden * 2          // W_hh slice, fp16
                             + 2ull * kMaxB * kHidden * 4         // h_{t-1} / h_t, all 512 units, fp32
                             + (size_t)kMaxB * kRows * 4          // W_hh h for this CTA's rows
                             + 2ull * kMaxB * kUnits * 4;         // this CTA's new h and its c
static_assert(kLstmSmem <= 227 * 1024, "LSTM shared memory");

// ---------------------------------------------------------------------------------------------------------------------
// pf_hnet_prep: (x[:, :3] - mean) / std as two fp32 ops (HorizonNet._prepare_x), rounded once to fp16, NCHW ->
// [B, 512, 1024, 16]
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
prep_kernel(const float* __restrict__ src, int B, int C, __half* __restrict__ dst) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  constexpr long long HW = (long long)kH * kW;
  if (idx >= B * HW) return;
  const long long b = idx / HW, p = idx % HW;
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
  __align__(16) __half v[kPrepC];
#pragma unroll
  for (int c = 0; c < kPrepC; ++c) v[c] = __float2half_rn(0.f);
#pragma unroll
  for (int c = 0; c < 3; ++c)
    v[c] = __float2half_rn(__fdiv_rn(__fsub_rn(src[(b * C + c) * HW + p], mean[c]), stdv[c]));
  uint4* d = reinterpret_cast<uint4*>(dst + idx * kPrepC);
  d[0] = reinterpret_cast<const uint4*>(v)[0];
  d[1] = reinterpret_cast<const uint4*>(v)[1];
}

// ---------------------------------------------------------------------------------------------------------------------
// pf_hnet_height_upsample: GlobalHeightConv's tail for one scale. cat(x[..., -1:], x, x[..., :1]) -> bilinear
// (align_corners=False) to width f * (w + 2) with the height unchanged -> [..., f:-f] -> reshape(B, C * h, T), written as
// rows t * B + b of the LSTM input. The width scale is exactly 1 / f and no kept column clamps its source index, so the
// fp32 weights are exact; the sum is torch's upsample_bilinear2d_out_frame expression with h0lambda = 1, h1lambda = 0.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
height_upsample_kernel(const __half* __restrict__ x, int B, int h, int w, int C, int f, int T,
                       __half* __restrict__ out, int out_off) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int CH = C * h;
  if (idx >= (long long)T * B * CH) return;
  const int ch = (int)(idx % CH), row = (int)(idx / CH);  // row = t * B + b
  const int t = row / B, b = row % B, c = ch / h, y = ch % h;
  const float scale = __fdiv_rn((float)(w + 2), (float)(f * (w + 2)));
  const float src = fmaxf(__fsub_rn(__fmul_rn(scale, (float)(t + f) + 0.5f), 0.5f), 0.f);
  const int x0 = (int)src;
  const int x1 = x0 + (x0 < w + 1 ? 1 : 0);
  const float l1 = __fsub_rn(src, (float)x0), l0 = __fsub_rn(1.f, l1);
  // padded column p holds original column (p - 1) mod w
  const int c0 = x0 == 0 ? w - 1 : (x0 == w + 1 ? 0 : x0 - 1);
  const int c1 = x1 == 0 ? w - 1 : (x1 == w + 1 ? 0 : x1 - 1);
  const __half* r0 = x + ((size_t)b * h + y) * w * C + c;
  const __half* r1 = r0 + (y < h - 1 ? (size_t)w * C : 0);  // the h1 + h1p row, weighted 0
  const float a = __fadd_rn(__fmul_rn(l0, __half2float(r0[(size_t)c0 * C])), __fmul_rn(l1, __half2float(r0[(size_t)c1 * C])));
  const float z = __fadd_rn(__fmul_rn(l0, __half2float(r1[(size_t)c0 * C])), __fmul_rn(l1, __half2float(r1[(size_t)c1 * C])));
  const float v = __fadd_rn(__fmul_rn(1.f, a), __fmul_rn(0.f, z));
  out[(size_t)row * kFeat + out_off + ch] = __float2half_rn(v);
}

// ---------------------------------------------------------------------------------------------------------------------
// pf_lstm_bidir: the recurrence of one bidirectional LSTM layer. One 16-CTA cluster per direction; CTA r owns hidden
// units [32 r, 32 r + 32), i.e. the 128 W_hh rows of their i, f, g, o gates (128 x 512 fp16 = 128 KB of shared memory,
// loaded once for all steps). Every CTA keeps the whole h_{t-1} of its direction in shared memory; per step it computes
// its 128 gate rows (fp32, one warp per 16 rows, lanes split K and reduce in a fixed butterfly), updates c and h of its
// 32 units, writes h to the output and pushes it into every peer's next h buffer through distributed shared memory,
// then the cluster barrier (release / acquire) separates the steps. h is double-buffered, so one barrier per step
// suffices. Every sample's arithmetic is the same for any B.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cluster_arrive_release() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_wait_acquire() {
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }

__global__ void __launch_bounds__(kLstmThreads, 1)
lstm_bidir_kernel(const float* __restrict__ xproj, const __half* __restrict__ whh, int T, int B,
                  __half* __restrict__ out) {
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __half* Ws = reinterpret_cast<__half*>(smem_raw);                          // [kRows][kHidden]
  float* hbuf = reinterpret_cast<float*>(Ws + kRows * kHidden);              // [2][kMaxB][kHidden]
  float* gates = hbuf + 2 * kMaxB * kHidden;                                 // [kMaxB][kRows]
  float* hnew = gates + kMaxB * kRows;                                       // [kMaxB][kUnits]
  float* cst = hnew + kMaxB * kUnits;                                        // [kMaxB][kUnits]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rank = (int)cluster.block_rank(), dir = blockIdx.x / kCluster;

  {
    const uint4* src = reinterpret_cast<const uint4*>(whh + (size_t)(dir * kCluster + rank) * kRows * kHidden);
    uint4* dst = reinterpret_cast<uint4*>(Ws);
    for (int i = tid; i < kRows * kHidden / 8; i += kLstmThreads) dst[i] = src[i];
    for (int i = tid; i < B * kHidden; i += kLstmThreads) hbuf[i] = 0.f;  // h_{-1} = 0
    for (int i = tid; i < B * kUnits; i += kLstmThreads) cst[i] = 0.f;    // c_{-1} = 0
  }
  cluster.sync();  // every CTA of the cluster runs and has zeroed its h_{-1} before anyone pushes into it

  for (int s = 0; s < T; ++s) {
    const int t = dir == 0 ? s : T - 1 - s;
    const float* hc = hbuf + (s & 1) * kMaxB * kHidden;
    // gates[b][r] = W_hh[r] . h_{t-1}[b]; lane l takes k = 2 l + 64 i, i < 8
    for (int rr = 0; rr < kRows / 8; ++rr) {
      const int r = warp * (kRows / 8) + rr;
      float2 wf[8];
#pragma unroll
      for (int i = 0; i < 8; ++i)
        wf[i] = __half22float2(*reinterpret_cast<const __half2*>(Ws + r * kHidden + 2 * lane + 64 * i));
      for (int b = 0; b < B; ++b) {
        const float* hb = hc + b * kHidden + 2 * lane;
        float acc = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float2 hv = *reinterpret_cast<const float2*>(hb + 64 * i);
          acc = __fmaf_rn(wf[i].x, hv.x, acc);
          acc = __fmaf_rn(wf[i].y, hv.y, acc);
        }
        acc = warp_sum(acc);
        if (lane == 0) gates[b * kRows + r] = acc;
      }
    }
    __syncthreads();
    for (int e = tid; e < B * kUnits; e += kLstmThreads) {
      const int b = e / kUnits, u = e % kUnits;
      const float* xp = xproj + ((size_t)t * B + b) * (2 * kGates) + dir * kGates + rank * kUnits + u;
      const float* g = gates + b * kRows + u;
      const float gi = __fadd_rn(xp[0], g[0]), gf = __fadd_rn(xp[kHidden], g[kUnits]);
      const float gg = __fadd_rn(xp[2 * kHidden], g[2 * kUnits]), go = __fadd_rn(xp[3 * kHidden], g[3 * kUnits]);
      const float c = __fadd_rn(__fmul_rn(sigmoid_f(gf), cst[e]), __fmul_rn(sigmoid_f(gi), tanhf(gg)));
      const float hv = __fmul_rn(sigmoid_f(go), tanhf(c));
      cst[e] = c;
      hnew[e] = hv;
      out[((size_t)t * B + b) * kFeat + dir * kHidden + rank * kUnits + u] = __float2half_rn(hv);
    }
    if (s + 1 == T) break;
    __syncthreads();
    // push this CTA's 32 new units of every sample into every peer's next h buffer (float4 pieces)
    float* hn = hbuf + ((s + 1) & 1) * kMaxB * kHidden;
    const int pieces = B * (kUnits / 4);
    for (int e = tid; e < kCluster * pieces; e += kLstmThreads) {
      const int peer = e / pieces, q = e % pieces, b = q / (kUnits / 4), u4 = q % (kUnits / 4);
      const float4 v = reinterpret_cast<const float4*>(hnew)[q];
      float* dst = cluster.map_shared_rank(hn + b * kHidden + rank * kUnits + u4 * 4, peer);
      *reinterpret_cast<float4*>(dst) = v;
    }
    cluster_arrive_release();
    cluster_wait_acquire();
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// pf_hnet_head: out = x @ W^T + b (Linear(1024, 12)) in fp32, one warp per output with a fixed lane order, scattered as
// view(T, B, 3, 4).permute(1, 2, 0, 3): channel 0 -> cor [B, 1, 4T], channels 1, 2 -> bon [B, 2, 4T].
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
head_kernel(const __half* __restrict__ x, int T, int B, const float* __restrict__ w, const float* __restrict__ bias,
            float* __restrict__ bon, float* __restrict__ cor) {
  const int o = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (o >= T * B * 12) return;
  const int n = o % 12, row = o / 12, t = row / B, b = row % B;
  const __half* xr = x + (size_t)row * kFeat;
  const float* wr = w + (size_t)n * kFeat;
  float s = 0.f;
  for (int k = lane; k < kFeat; k += 32) s = __fmaf_rn(__half2float(xr[k]), wr[k], s);
  s = warp_sum(s);
  if (lane) return;
  s = __fadd_rn(s, bias[n]);
  const int ch = n / 4, col = t * 4 + n % 4;
  if (ch == 0)
    cor[(size_t)b * 4 * T + col] = s;
  else
    bon[((size_t)b * 2 + ch - 1) * 4 * T + col] = s;
}

// occupancy of the recurrence's 16-CTA clusters on the current device: -1 before the first query
int g_lstm_clusters = -1;

int lstm_setup() {
  if (g_lstm_clusters >= 0) return PF_OK;
  int rc = check_cuda(cudaFuncSetAttribute(lstm_bidir_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1),
                      "cudaFuncSetAttribute(NonPortableClusterSizeAllowed)");
  if (rc) return rc;
  rc = check_cuda(cudaFuncSetAttribute(lstm_bidir_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLstmSmem),
                  "cudaFuncSetAttribute(lstm_bidir_kernel)");
  if (rc) return rc;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kCluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.gridDim = dim3(2 * kCluster);
  cfg.blockDim = dim3(kLstmThreads);
  cfg.dynamicSmemBytes = kLstmSmem;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  rc = check_cuda(cudaOccupancyMaxActiveClusters(&n, lstm_bidir_kernel, &cfg), "cudaOccupancyMaxActiveClusters");
  if (rc) return rc;
  g_lstm_clusters = n;
  return PF_OK;
}

}  // namespace hnet
}  // namespace pf

using namespace pf;
using namespace pf::hnet;
using pf::convmma::ConvArgs;
using pf::convmma::launch_conv;

extern "C" int pf_hnet_prep(const float* src, int B, int C, int H, int W, void* dst, void* stream) {
  PF_CHECK_ARG(src && dst, "pf_hnet_prep: null pointer");
  PF_CHECK_ARG(B > 0 && C >= 3 && H == kH && W == kW && (long long)B * C * H * W < (1LL << 40) &&
                   (long long)B * H * W < (1LL << 31),
               "pf_hnet_prep: bad shape B=%d C=%d H=%d W=%d (need C >= 3, H x W = 512 x 1024)", B, C, H, W);
  const long long n = (long long)B * H * W;
  prep_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(src, B, C,
                                                                                          static_cast<__half*>(dst));
  PF_CHECK_LAUNCH("hnet prep_kernel");
  return PF_OK;
}

extern "C" int pf_hnet_conv(const void* x, int B, int H, int W, int Cin, const void* w, const float* bias, int Cout,
                            int k, int stride_h, int stride_w, int relu, const void* residual, void* out,
                            int out_dtype, void* stream) {
  PF_CHECK_ARG(x && w && bias && out, "pf_hnet_conv: null pointer");
  PF_CHECK_ARG(out_dtype == PF_F16 || out_dtype == PF_F32, "pf_hnet_conv: out_dtype must be PF_F16 or PF_F32");
  PF_CHECK_ARG(B > 0 && H > 0 && W > 0, "pf_hnet_conv: bad shape B=%d H=%d W=%d", B, H, W);
  PF_CHECK_ARG(k == 1 || k == 3 || k == 7, "pf_hnet_conv: kernel %d unsupported (1, 3 or 7)", k);
  PF_CHECK_ARG((stride_h == 1 && stride_w == 1) || (stride_h == 2 && stride_w == 2) || (stride_h == 2 && stride_w == 1),
               "pf_hnet_conv: stride (%d, %d) unsupported ((1, 1), (2, 2) or (2, 1))", stride_h, stride_w);
  PF_CHECK_ARG(Cin == 16 || (Cin > 0 && Cin % 64 == 0), "pf_hnet_conv: Cin=%d unsupported (16 or a multiple of 64)",
               Cin);
  PF_CHECK_ARG(Cout == 32 || Cout == 64 || (Cout > 0 && Cout % 128 == 0),
               "pf_hnet_conv: Cout=%d unsupported (32, 64 or a multiple of 128)", Cout);
  const int pad = k / 2;
  PF_CHECK_ARG(pad < W && H + 2 * pad >= k, "pf_hnet_conv: image %dx%d too small for the %dx%d kernel", H, W, k, k);
  const int Ho = (H + 2 * pad - k) / stride_h + 1, Wo = (W + 2 * pad - k) / stride_w + 1;
  const long long M = (long long)B * Ho * Wo;
  PF_CHECK_ARG(M * Cout < (1LL << 31) && (long long)B * H * W * Cin < (1LL << 31), "pf_hnet_conv: tensor too large");
  // rows zero-padded and columns wrapped by pad = k / 2; the weight is packed [k*k][Cin][Cout]
  ConvArgs a{static_cast<const __half*>(x), static_cast<const __half*>(w), bias,
             static_cast<const __half*>(residual), out, B, H, W, Cin, Cout, Ho, Wo, k, k, stride_h, pad, pad, relu,
             out_dtype == PF_F32, Cout, Cout, 0, (int)M, stride_w};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (Cin == 16) {
    PF_CHECK_ARG(Cout == 64, "pf_hnet_conv: Cin=16 runs only the stem (Cout 64), not Cout=%d", Cout);
    return launch_conv<16, 64, true, true, true>(a, st);
  }
  if (Cout == 32) return launch_conv<32, 32, true, true, true>(a, st);
  if (Cout == 64) return launch_conv<64, 64, true, true, true>(a, st);
  return launch_conv<64, 128, true, true, true>(a, st);
}

extern "C" int pf_hnet_height_upsample(const void* x, int B, int h, int w, int C, int T, void* out, int out_off,
                                       void* stream) {
  PF_CHECK_ARG(x && out, "pf_hnet_height_upsample: null pointer");
  PF_CHECK_ARG(B > 0 && h > 0 && w > 0 && C > 0 && T > 0 && T % w == 0 && (long long)T * B * C * h < (1LL << 31),
               "pf_hnet_height_upsample: bad shape B=%d h=%d w=%d C=%d T=%d (T a multiple of w)", B, h, w, C, T);
  PF_CHECK_ARG(out_off >= 0 && out_off + C * h <= kFeat,
               "pf_hnet_height_upsample: slice [%d, %d) outside the %d-wide LSTM input", out_off, out_off + C * h,
               kFeat);
  const long long n = (long long)T * B * C * h;
  height_upsample_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(x), B, h, w, C, T / w, T, static_cast<__half*>(out), out_off);
  PF_CHECK_LAUNCH("height_upsample_kernel");
  return PF_OK;
}

extern "C" int pf_lstm_bidir_clusters(int* clusters) {
  PF_CHECK_ARG(clusters, "pf_lstm_bidir_clusters: null pointer");
  const int rc = lstm_setup();
  if (rc) return rc;
  *clusters = g_lstm_clusters;
  return PF_OK;
}

extern "C" int pf_lstm_bidir(const float* xproj, const void* whh, int T, int B, void* out, void* stream) {
  PF_CHECK_ARG(xproj && whh && out, "pf_lstm_bidir: null pointer");
  PF_CHECK_ARG(T > 0 && B > 0 && B <= kMaxB && (long long)T * B * 2 * kGates < (1LL << 31),
               "pf_lstm_bidir: bad shape T=%d B=%d (1 <= B <= %d)", T, B, kMaxB);
  PF_CHECK_ARG((reinterpret_cast<uintptr_t>(whh) & 15) == 0, "pf_lstm_bidir: whh must be 16-byte aligned");
  int rc = lstm_setup();
  if (rc) return rc;
  if (g_lstm_clusters < 1) {
    set_error("pf_lstm_bidir: this device cannot hold a %d-CTA cluster with %zu bytes of shared memory per CTA",
              kCluster, kLstmSmem);
    return PF_ERR_UNSUPPORTED;
  }
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kCluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.gridDim = dim3(2 * kCluster);
  cfg.blockDim = dim3(kLstmThreads);
  cfg.dynamicSmemBytes = kLstmSmem;
  cfg.stream = static_cast<cudaStream_t>(stream);
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  rc = check_cuda(cudaLaunchKernelEx(&cfg, lstm_bidir_kernel, xproj, static_cast<const __half*>(whh), T, B,
                                     static_cast<__half*>(out)),
                  "cudaLaunchKernelEx(lstm_bidir_kernel)");
  if (rc) return rc;
  PF_CHECK_LAUNCH("lstm_bidir_kernel");
  return PF_OK;
}

extern "C" int pf_hnet_head(const void* x, int T, int B, const float* w, const float* bias, float* bon, float* cor,
                            void* stream) {
  PF_CHECK_ARG(x && w && bias && bon && cor, "pf_hnet_head: null pointer");
  PF_CHECK_ARG(T > 0 && B > 0 && (long long)T * B * 12 < (1LL << 31), "pf_hnet_head: bad shape T=%d B=%d", T, B);
  const long long n = (long long)T * B * 12;
  head_kernel<<<(unsigned)((n + 7) / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(x), T, B, w, bias, bon, cor);
  PF_CHECK_LAUNCH("hnet head_kernel");
  return PF_OK;
}
