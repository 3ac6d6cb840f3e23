// FAED autoencoder training (models/faed/FAED.py:13-33 over models/faed/modules.py's AutoEncoder): the training-mode
// forward, its backward and Adam, all on the device.
//
// Activations are channels-last fp16 [B, H, W, C] as in pf_conv_circ. Gradients of activations carry a power-of-two
// loss scale S (the seed is sign * S instead of sign / N, which would be below fp16's normal range); every fp32
// parameter gradient is multiplied by 1 / (S * N) where it is reduced. All reductions run in a fixed order over
// fixed-size chunks whose size depends only on the shape, so the bits do not depend on the grid or on timing.
#include "conv_mma.cuh"

namespace pf {
namespace faedt {

using convmma::cp_async16;
using convmma::cp_async_commit;
using convmma::cp_async_wait;
using convmma::ldsm_x4_t;
using convmma::mma16816;

constexpr float kBnEps = 1e-5f;
constexpr float kBnMomentum = 0.1f;
constexpr int kGrowthInterval = 2000;  // torch.cuda.amp.GradScaler's growth_interval

__device__ __forceinline__ void mark_nonfinite(float v, int* flag) {
  if (!isfinite(v)) *flag = 1;  // every writer stores the same value
}

// rows per chunk of a [P][C] reduction: at most 512 chunks, at least 256 rows each
__host__ __device__ inline int row_chunk(long long P) {
  long long c = (P + 511) / 512;
  return (int)(c < 256 ? 256 : c);
}

// ---------------------------------------------------------------------------------------------------------------------
// Input: pano fp32 [B, 3, H, W] -> fp16 [B, H, W, 16] (channels 3..15 zero)
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
prep_kernel(const float* __restrict__ src, int B, int H, int W, __half* __restrict__ dst) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long HW = (long long)H * W;
  if (idx >= B * HW) return;
  const long long b = idx / HW, p = idx % HW;
  __align__(16) __half v[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) v[c] = __float2half_rn(c < 3 ? src[(b * 3 + c) * HW + p] : 0.f);
  uint4* d = reinterpret_cast<uint4*>(dst + idx * 16);
  d[0] = reinterpret_cast<const uint4*>(v)[0];
  d[1] = reinterpret_cast<const uint4*>(v)[1];
}

// ---------------------------------------------------------------------------------------------------------------------
// Weight gradient of a circular convolution: dW[tap][ci][co] = sum_p X[p (+) tap, ci] * dY[p, co], K = pixels.
// CTA tile BM input channels x BN output channels, one tap, one pixel chunk; WM x WN warps of 32 x 32. Both operands
// are pixel-major in shared memory ([k][m] and [k][n]), so A is read with ldmatrix.trans like B. Each CTA writes an fp32
// partial [chunk][tap][Cin][Cdy]; the (tap 0, ci tile 0) CTAs also write the chunk's column sums of dY for db.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kWBK = 32;  // pixels per stage
constexpr int kWStages = 3;

struct WgradArgs {
  const __half* x;
  const __half* dy;
  float* part;
  float* dbpart;
  int B, H, W, Cin, Ho, Wo, Cdy, k, stride, pad, P, chunk, ci_tiles;
};

template <int BM, int BN>
__global__ void __launch_bounds__(BM / 32 * BN / 32 * 32)
wgrad_kernel(WgradArgs a) {
  constexpr int WM = BM / 32, WN = BN / 32, NTH = WM * WN * 32;
  constexpr int X_LD = BM + 8, D_LD = BN + 8;
  constexpr int STAGE = kWBK * (X_LD + D_LD);
  __shared__ __align__(16) __half smem[kWStages * STAGE];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp % WM, wn = warp / WM;
  const int ci_t = blockIdx.y % a.ci_tiles, tap = blockIdx.y / a.ci_tiles;
  const int ky = tap / a.k, kx = tap % a.k;
  const int ci0 = ci_t * BM;
  const int p0 = blockIdx.x * a.chunk;
  const int p1 = min(a.P, p0 + a.chunk);
  const int steps = (p1 - p0 + kWBK - 1) / kWBK;
  const int HoWo = a.Ho * a.Wo;
  const bool do_db = a.dbpart && tap == 0 && ci_t == 0;

  auto load = [&](int s, int buf) {
    __half* Xs = smem + buf * STAGE;
    __half* Ds = Xs + kWBK * X_LD;
    const int pb = p0 + s * kWBK;
    for (int idx = tid; idx < kWBK * (BM / 8); idx += NTH) {
      const int row = idx / (BM / 8), ch = idx % (BM / 8);
      const int p = pb + row, ci = ci0 + ch * 8;
      bool valid = p < p1 && ci < a.Cin;
      const __half* src = a.x;
      if (valid) {
        const int b = p / HoWo, r = p % HoWo;
        const int iy = (r / a.Wo) * a.stride + ky - a.pad;
        int ix = (r % a.Wo) * a.stride + kx - a.pad;
        ix = ix < 0 ? ix + a.W : (ix >= a.W ? ix - a.W : ix);
        valid = iy >= 0 && iy < a.H;
        if (valid) src = a.x + ((size_t)(b * a.H + iy) * a.W + ix) * a.Cin + ci;
      }
      cp_async16(smem_u32(Xs + row * X_LD + ch * 8), src, valid);
    }
    for (int idx = tid; idx < kWBK * (BN / 8); idx += NTH) {
      const int row = idx / (BN / 8), ch = idx % (BN / 8);
      const int p = pb + row, co = ch * 8;
      const bool valid = p < p1 && co < a.Cdy;
      cp_async16(smem_u32(Ds + row * D_LD + ch * 8), valid ? a.dy + (size_t)p * a.Cdy + co : a.dy, valid);
    }
  };

  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;
  float dbsum = 0.f;

#pragma unroll
  for (int s = 0; s < kWStages - 1; ++s) {
    if (s < steps) load(s, s);
    cp_async_commit();
  }
  for (int s = 0; s < steps; ++s) {
    cp_async_wait<kWStages - 2>();
    __syncthreads();
    if (s + kWStages - 1 < steps) load(s + kWStages - 1, (s + kWStages - 1) % kWStages);
    cp_async_commit();
    const __half* Xs = smem + (s % kWStages) * STAGE;
    const __half* Ds = Xs + kWBK * X_LD;
    if (do_db && tid < BN)
      for (int r = 0; r < kWBK; ++r) dbsum += __half2float(Ds[r * D_LD + tid]);
#pragma unroll
    for (int kk = 0; kk < kWBK; kk += 16) {
      uint32_t af[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int krow = kk + (lane & 7) + ((lane >> 4) << 3);
        const int col = wm * 32 + mt * 16 + ((lane >> 3) & 1) * 8;
        ldsm_x4_t(smem_u32(Xs + krow * X_LD + col), af[mt][0], af[mt][1], af[mt][2], af[mt][3]);
      }
#pragma unroll
      for (int np = 0; np < 2; ++np) {
        uint32_t b0, b1, b2, b3;
        const int krow = kk + (lane & 15), col = wn * 32 + np * 16 + (lane >> 4) * 8;
        ldsm_x4_t(smem_u32(Ds + krow * D_LD + col), b0, b1, b2, b3);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma16816(acc[mt][2 * np], af[mt], b0, b1);
          mma16816(acc[mt][2 * np + 1], af[mt], b2, b3);
        }
      }
    }
  }
  cp_async_wait<0>();

  float* out = a.part + ((size_t)blockIdx.x * a.k * a.k + tap) * a.Cin * a.Cdy;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const int co = wn * 32 + nt * 8 + (lane & 3) * 2;
      if (co >= a.Cdy) continue;  // Cdy is a multiple of 8
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ci = ci0 + wm * 32 + mt * 16 + (lane >> 2) + h * 8;
        if (ci >= a.Cin) continue;
        *reinterpret_cast<float2*>(out + (size_t)ci * a.Cdy + co) =
            make_float2(acc[mt][nt][2 * h], acc[mt][nt][2 * h + 1]);
      }
    }
  if (do_db && tid < BN && tid < a.Cdy) a.dbpart[(size_t)blockIdx.x * a.Cdy + tid] = dbsum;
}

// dw [Cout][Cin_w][k][k] (torch layout) = factor * sum over chunks in order; threads run co fastest (coalesced reads)
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ part, int nch, int taps, int Cin, int Cdy, int Cin_w, int Cout,
                    const double* __restrict__ scale, double inv_n, float* __restrict__ dw, int* flag) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= taps * Cin_w * Cout) return;
  const int co = idx % Cout, ci = (idx / Cout) % Cin_w, tap = idx / (Cout * Cin_w);
  const size_t stride = (size_t)taps * Cin * Cdy;
  const float* p = part + ((size_t)tap * Cin + ci) * Cdy + co;
  float s = 0.f;
  for (int c = 0; c < nch; ++c) s += p[c * stride];
  const float v = s * (float)(inv_n / scale[0]);
  dw[((size_t)co * Cin_w + ci) * taps + tap] = v;
  mark_nonfinite(v, flag);
}

__global__ void __launch_bounds__(128)
db_reduce_kernel(const float* __restrict__ dbpart, int nch, int Cdy, int Cout, const double* __restrict__ scale,
                 double inv_n, float* __restrict__ db, int* flag) {
  const int co = blockIdx.x * blockDim.x + threadIdx.x;
  if (co >= Cout) return;
  float s = 0.f;
  for (int c = 0; c < nch; ++c) s += dbpart[(size_t)c * Cdy + co];
  const float v = s * (float)(inv_n / scale[0]);
  db[co] = v;
  mark_nonfinite(v, flag);
}

__host__ __device__ inline int wgrad_chunk(long long P, int taps, int Cin, int Cdy) {
  // at most 2^24 partial floats and at most ceil(P / 1024) chunks; a multiple of the stage depth
  long long cap = (1LL << 24) / ((long long)taps * Cin * Cdy);
  if (cap < 1) cap = 1;
  long long nch = (P + 1023) / 1024;
  if (nch > cap) nch = cap;
  long long chunk = (P + nch - 1) / nch;
  chunk = (chunk + kWBK - 1) / kWBK * kWBK;
  return (int)chunk;
}

// ---------------------------------------------------------------------------------------------------------------------
// BatchNorm2d, training mode, on z [P][C] (P = B*H*W). Per-chunk Welford (count, mean, M2), merged in chunk order with
// Chan's formula; never sum(z^2) - mean^2 (the conv bias makes the mean large against the spread).
// stats [3][C]: batch mean, 1 / sqrt(biased var + eps), unbiased var.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void chan_merge(float& n, float& mean, float& m2, float nb, float mb, float m2b) {
  if (nb == 0.f) return;
  const float nab = n + nb, delta = mb - mean;
  mean += delta * (nb / nab);
  m2 += m2b + delta * delta * (n * nb / nab);
  n = nab;
}

__global__ void __launch_bounds__(256)
bn_stats_part_kernel(const __half* __restrict__ z, long long P, int C, int chunk, float* __restrict__ part) {
  __shared__ float sh[3][256];
  const int tid = threadIdx.x, c = tid % C, lane = tid / C, L = 256 / C;
  const long long r0 = (long long)blockIdx.x * chunk, r1 = min(P, r0 + chunk);
  float n = 0.f, mean = 0.f, m2 = 0.f;
  for (long long r = r0 + lane; r < r1; r += L) {
    const float v = __half2float(z[r * C + c]);
    n += 1.f;
    const float d = v - mean;
    mean += d / n;
    m2 += d * (v - mean);
  }
  sh[0][tid] = n;
  sh[1][tid] = mean;
  sh[2][tid] = m2;
  __syncthreads();
  if (lane == 0) {
    for (int l = 1; l < L; ++l) chan_merge(n, mean, m2, sh[0][l * C + c], sh[1][l * C + c], sh[2][l * C + c]);
    float* o = part + (size_t)blockIdx.x * 3 * C;
    o[c] = n;
    o[C + c] = mean;
    o[2 * C + c] = m2;
  }
}

__global__ void bn_stats_merge_kernel(const float* __restrict__ part, int nch, int C, float* __restrict__ stats) {
  const int c = threadIdx.x;
  if (c >= C) return;
  float n = 0.f, mean = 0.f, m2 = 0.f;
  for (int i = 0; i < nch; ++i) {
    const float* p = part + (size_t)i * 3 * C;
    chan_merge(n, mean, m2, p[c], p[C + c], p[2 * C + c]);
  }
  stats[c] = mean;
  stats[C + c] = 1.f / sqrtf(m2 / n + kBnEps);
  stats[2 * C + c] = m2 / (n - 1.f);
}

// out = [relu]((z - mean) * invstd * gamma + beta) [+ residual]
__global__ void __launch_bounds__(256)
bn_apply_kernel(const __half* __restrict__ z, long long n, int C, const float* __restrict__ stats,
                const float* __restrict__ gamma, const float* __restrict__ beta, int relu,
                const __half* __restrict__ residual, __half* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const int c = (int)(idx % C);
  float v = (__half2float(z[idx]) - stats[c]) * stats[C + c] * gamma[c] + beta[c];
  if (relu) v = fmaxf(v, 0.f);
  if (residual) v += __half2float(residual[idx]);
  out[idx] = __float2half_rn(v);
}

// BN backward. g' = g * (mask > 0 if mask); per chunk sum g' and sum g' * xhat in row order, merged in chunk order.
__global__ void __launch_bounds__(256)
bn_bwd_part_kernel(const __half* __restrict__ g, const __half* __restrict__ mask, const __half* __restrict__ z,
                   long long P, int C, int chunk, const float* __restrict__ stats, float* __restrict__ part) {
  __shared__ float sh[2][256];
  const int tid = threadIdx.x, c = tid % C, lane = tid / C, L = 256 / C;
  const long long r0 = (long long)blockIdx.x * chunk, r1 = min(P, r0 + chunk);
  const float mean = stats[c], inv = stats[C + c];
  float sg = 0.f, sgx = 0.f;
  for (long long r = r0 + lane; r < r1; r += L) {
    const long long i = r * C + c;
    float gv = __half2float(g[i]);
    if (mask && !(__half2float(mask[i]) > 0.f)) gv = 0.f;
    sg += gv;
    sgx += gv * ((__half2float(z[i]) - mean) * inv);
  }
  sh[0][tid] = sg;
  sh[1][tid] = sgx;
  __syncthreads();
  if (lane == 0) {
    for (int l = 1; l < L; ++l) {
      sg += sh[0][l * C + c];
      sgx += sh[1][l * C + c];
    }
    part[(size_t)blockIdx.x * 2 * C + c] = sg;
    part[(size_t)blockIdx.x * 2 * C + C + c] = sgx;
  }
}

// sums [2][C] <- mean g', mean g' xhat; dgamma = factor * sum g' xhat, dbeta = factor * sum g'
__global__ void bn_bwd_merge_kernel(const float* __restrict__ part, int nch, int C, long long P,
                                    const double* __restrict__ scale, double inv_n, float* __restrict__ sums,
                                    float* __restrict__ dgamma, float* __restrict__ dbeta, int* flag) {
  const int c = threadIdx.x;
  if (c >= C) return;
  float sg = 0.f, sgx = 0.f;
  for (int i = 0; i < nch; ++i) {
    sg += part[(size_t)i * 2 * C + c];
    sgx += part[(size_t)i * 2 * C + C + c];
  }
  sums[c] = sg / (float)P;
  sums[C + c] = sgx / (float)P;
  const float f = (float)(inv_n / scale[0]);
  dgamma[c] = sgx * f;
  dbeta[c] = sg * f;
  mark_nonfinite(dgamma[c], flag);
  mark_nonfinite(dbeta[c], flag);
}

// dz = gamma * invstd * (g' - mean g' - xhat * mean g' xhat)
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const __half* __restrict__ g, const __half* __restrict__ mask, const __half* __restrict__ z,
                    long long n, int C, const float* __restrict__ stats, const float* __restrict__ gamma,
                    const float* __restrict__ sums, __half* __restrict__ dz) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const int c = (int)(idx % C);
  float gv = __half2float(g[idx]);
  if (mask && !(__half2float(mask[idx]) > 0.f)) gv = 0.f;
  const float xh = (__half2float(z[idx]) - stats[c]) * stats[C + c];
  dz[idx] = __float2half_rn(gamma[c] * stats[C + c] * (gv - sums[c] - xh * sums[C + c]));
}

// ---------------------------------------------------------------------------------------------------------------------
// F.interpolate(scale_factor=2, mode='bilinear', align_corners=False): src = max((o + 0.5) * 0.5 - 0.5, 0), clamped
// at the far edge (no wrap). The backward is a gather over the <= 4 outputs per axis that read an input.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void up_src(int o, int n, int& i0, int& i1, float& l1) {
  const float s = fmaxf((o + 0.5f) * 0.5f - 0.5f, 0.f);
  i0 = (int)s;
  i1 = i0 + (i0 < n - 1 ? 1 : 0);
  l1 = s - (float)i0;
}

__device__ __forceinline__ float up_weight(int o, int n, int i) {
  int i0, i1;
  float l1;
  up_src(o, n, i0, i1, l1);
  return (i0 == i ? 1.f - l1 : 0.f) + (i1 == i ? l1 : 0.f);
}

__global__ void __launch_bounds__(256)
upsample_kernel(const __half* __restrict__ x, int B, int H, int W, int C, __half* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int Ho = 2 * H, Wo = 2 * W;
  if (idx >= (long long)B * Ho * Wo * C) return;
  const int c = (int)(idx % C);
  const long long pix = idx / C;
  const int ox = (int)(pix % Wo), oy = (int)((pix / Wo) % Ho), b = (int)(pix / ((long long)Wo * Ho));
  int y0, y1, x0, x1;
  float ly, lx;
  up_src(oy, H, y0, y1, ly);
  up_src(ox, W, x0, x1, lx);
  auto at = [&](int y, int xx) { return __half2float(x[(((size_t)b * H + y) * W + xx) * C + c]); };
  const float v = (1.f - ly) * ((1.f - lx) * at(y0, x0) + lx * at(y0, x1)) +
                  ly * ((1.f - lx) * at(y1, x0) + lx * at(y1, x1));
  out[idx] = __float2half_rn(v);
}

__global__ void __launch_bounds__(256)
upsample_bwd_kernel(const __half* __restrict__ g, int B, int H, int W, int C, __half* __restrict__ dx) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * H * W * C) return;
  const int Ho = 2 * H, Wo = 2 * W;
  const int c = (int)(idx % C);
  const long long pix = idx / C;
  const int ix = (int)(pix % W), iy = (int)((pix / W) % H), b = (int)(pix / ((long long)W * H));
  float s = 0.f;
  for (int oy = max(2 * iy - 1, 0); oy <= min(2 * iy + 2, Ho - 1); ++oy) {
    const float wy = up_weight(oy, H, iy);
    if (wy == 0.f) continue;
    float r = 0.f;
    for (int ox = max(2 * ix - 1, 0); ox <= min(2 * ix + 2, Wo - 1); ++ox) {
      const float wx = up_weight(ox, W, ix);
      if (wx != 0.f) r += wx * __half2float(g[(((size_t)b * Ho + oy) * Wo + ox) * C + c]);
    }
    s += wy * r;
  }
  dx[idx] = __float2half_rn(s);
}

// ---------------------------------------------------------------------------------------------------------------------
// Loss: pred = tanh(o), loss = mean |pred - target| over B*3*H*W, seed = sign(pred - target) * (1 - pred^2) * S.
// o fp32 [B, H, W, 4] (outconv, channel 3 unused), target fp32 [B, 3, H, W], seed fp16 [B, H, W, 16] (3..15 zero).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kLossBlocks = 1024;

__device__ __forceinline__ float block_sum256(float v, float* red) {
  const int t = threadIdx.x;
  red[t] = v;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if (t < off) red[t] += red[t + off];
    __syncthreads();
  }
  return red[0];
}

__global__ void __launch_bounds__(256)
loss_part_kernel(const float* __restrict__ o, const float* __restrict__ target, int B, int H, int W,
                 const double* __restrict__ scale, float* __restrict__ pred, __half* __restrict__ seed,
                 float* __restrict__ part) {
  __shared__ float red[256];
  const long long HW = (long long)H * W, M = B * HW;
  const float S = (float)scale[0];
  float acc = 0.f;
  for (long long m = (long long)blockIdx.x * 256 + threadIdx.x; m < M; m += (long long)gridDim.x * 256) {
    const long long b = m / HW, p = m % HW;
    __align__(16) __half sv[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) sv[c] = __float2half_rn(0.f);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float pr = tanhf(o[m * 4 + c]);
      const float d = pr - (target ? target[(b * 3 + c) * HW + p] : 0.f);
      acc += fabsf(d);
      const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : d);  // sign(0) = 0, NaN stays NaN
      sv[c] = __float2half_rn(sg * (1.f - pr * pr) * S);
      if (pred) pred[(b * 3 + c) * HW + p] = pr;
    }
    uint4* d = reinterpret_cast<uint4*>(seed + m * 16);
    d[0] = reinterpret_cast<const uint4*>(sv)[0];
    d[1] = reinterpret_cast<const uint4*>(sv)[1];
  }
  const float s = block_sum256(acc, red);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

__global__ void __launch_bounds__(256)
loss_final_kernel(const float* __restrict__ part, int n, double count, float* __restrict__ loss, int* flag) {
  __shared__ float red[256];
  float acc = 0.f;
  for (int i = threadIdx.x; i < n; i += 256) acc += part[i];
  const float s = block_sum256(acc, red);
  if (threadIdx.x == 0) {
    loss[0] = (float)(s / count);
    mark_nonfinite(loss[0], flag);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Adam (torch.optim.Adam, foreach=False: lerp, mul + addcmul, sqrt / bias_correction2_sqrt + eps, addcdiv) over the flat
// fp32 parameters, skipped entirely when the non-finite flag is set. ctl: lr, scale (double); ictl: step, growth
// tracker, skipped steps, non-finite flag (int32). Also applies the pending BatchNorm running statistics.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
            long long n, float* __restrict__ run, const float* __restrict__ pending, long long n_run,
            const double* __restrict__ ctl, const int* __restrict__ ictl, double beta1, double beta2, double eps) {
  if (ictl[3]) return;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < n_run) run[idx] = kBnMomentum * pending[idx] + (1.f - kBnMomentum) * run[idx];
  if (idx >= n) return;
  const double step = (double)(ictl[0] + 1);
  // torch's five fp32 kernels, each rounding once: Python's doubles cast to fp32 where torch passes them; division by
  // the bias correction is a multiplication by its reciprocal, taken in double and rounded to fp32 once, as torch's div
  // by a CPU scalar is; lerp, addcmul and addcdiv compute self + w * (x) with one fused multiply-add. The intrinsics
  // keep nvcc from contracting across what torch rounds separately.
  const double bc1 = 1.0 - pow(beta1, step), bc2 = 1.0 - pow(beta2, step);
  const float step_size = (float)(-(ctl[0] / bc1));
  const float inv_bc2 = (float)(1.0 / sqrt(bc2));
  const float gv = g[idx];
  const float mv = __fmaf_rn((float)(1.0 - beta1), __fsub_rn(gv, m[idx]), m[idx]);
  const float vv = __fmaf_rn((float)(1.0 - beta2), __fmul_rn(gv, gv), __fmul_rn(v[idx], (float)beta2));
  const float denom = __fadd_rn(__fmul_rn(__fsqrt_rn(vv), inv_bc2), (float)eps);
  p[idx] = __fmaf_rn(step_size, __fdiv_rn(mv, denom), p[idx]);
  m[idx] = mv;
  v[idx] = vv;
}

__global__ void step_end_kernel(double* ctl, int* ictl, long long* num_batches) {
  if (ictl[3]) {
    ctl[1] *= 0.5;
    ictl[1] = 0;
    ictl[2] += 1;
    ictl[3] = 0;
  } else {
    ictl[0] += 1;
    *num_batches += 1;
    if (++ictl[1] == kGrowthInterval) {
      ctl[1] *= 2.0;
      ictl[1] = 0;
    }
  }
}

// forward [k*k][cin_pad][cw] and dgrad weights from w [Cout][Cin][k][k] (fp32). Stride 1: the flipped kernel
// [k*k][dg_rows][dg_cw] (dg_rows >= Cout, dg_cw >= Cin). Stride 2 (k = 4): four 2x2 phase kernels [4][4][dg_rows][dg_cw],
// phase (r, c) tap (ty, tx) = w[.., 3 - 2 ty - r, 3 - 2 tx - c].
__global__ void __launch_bounds__(256)
pack_kernel(const float* __restrict__ w, int Cout, int Cin, int k, int stride, __half* __restrict__ fwd, int cin_pad,
            int cw, __half* __restrict__ dg, int dg_rows, int dg_cw) {
  const int taps = k * k;
  const long long nf = (long long)taps * cin_pad * cw, nd = dg ? (long long)taps * dg_rows * dg_cw : 0;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < nf) {
    const int co = (int)(idx % cw), ci = (int)((idx / cw) % cin_pad), tap = (int)(idx / ((long long)cw * cin_pad));
    fwd[idx] = __float2half_rn(co < Cout && ci < Cin ? w[((size_t)co * Cin + ci) * taps + tap] : 0.f);
  } else if (idx < nf + nd) {
    const long long j = idx - nf;
    const int ci = (int)(j % dg_cw), co = (int)((j / dg_cw) % dg_rows), t = (int)(j / ((long long)dg_cw * dg_rows));
    int ky, kx;
    if (stride == 1) {
      ky = k - 1 - t / k;
      kx = k - 1 - t % k;
    } else {
      const int ph = t / 4, tt = t % 4;
      ky = 3 - 2 * (tt / 2) - ph / 2;
      kx = 3 - 2 * (tt % 2) - ph % 2;
    }
    dg[j] = __float2half_rn(co < Cout && ci < Cin ? w[((size_t)co * Cin + ci) * taps + ky * k + kx] : 0.f);
  }
}

// phase outputs [4][B, H/2, W/2, C] -> dx [B, H, W, C], dx[2q + r][2p + c] = phase (r, c)
__global__ void __launch_bounds__(256)
interleave_kernel(const __half* __restrict__ ph, int B, int H, int W, int C, __half* __restrict__ dx) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = (long long)B * H * W * C;
  if (idx >= n) return;
  const int c = (int)(idx % C);
  const long long pix = idx / C;
  const int x = (int)(pix % W), y = (int)((pix / W) % H), b = (int)(pix / ((long long)W * H));
  const int phase = (y & 1) * 2 + (x & 1);
  dx[idx] = ph[(size_t)phase * (n / 4) + ((((size_t)b * (H / 2) + y / 2) * (W / 2) + x / 2) * C + c)];
}

}  // namespace faedt
}  // namespace pf

using namespace pf;
using namespace pf::faedt;
using pf::convmma::ConvArgs;
using pf::convmma::launch_conv;

static unsigned blocks_for(long long n) { return (unsigned)((n + 255) / 256); }

extern "C" int pf_faedt_prep(const float* src, int B, int H, int W, void* dst, void* stream) {
  PF_CHECK_ARG(src && dst, "pf_faedt_prep: null pointer");
  PF_CHECK_ARG(B > 0 && H > 0 && W > 0 && (long long)B * H * W * 16 < (1LL << 31), "pf_faedt_prep: bad shape");
  prep_kernel<<<blocks_for((long long)B * H * W), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, B, H, W, static_cast<__half*>(dst));
  PF_CHECK_LAUNCH("faedt prep_kernel");
  return PF_OK;
}

extern "C" int pf_faedt_conv(const void* x, int B, int H, int W, int Cin, const void* w, const float* bias, int Cout,
                             int Cw, int kh, int kw, int stride, int ph, int pw, int Ho, int Wo, const void* residual,
                             void* out, int out_ld, int out_dtype, void* stream) {
  PF_CHECK_ARG(x && w && bias && out, "pf_faedt_conv: null pointer");
  PF_CHECK_ARG(B > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && kh > 0 && kw > 0 && (stride == 1 || stride == 2) &&
                   ph >= 0 && pw >= 0 && pw < W,
               "pf_faedt_conv: bad shape");
  // rows outside [0, H) read zeros; columns wrap once, so they must stay within [-W, 2W)
  PF_CHECK_ARG((Wo - 1) * stride + kw - 1 - pw < 2 * W, "pf_faedt_conv: output width %d wraps more than once", Wo);
  PF_CHECK_ARG(out_dtype == PF_F16 || out_dtype == PF_F32, "pf_faedt_conv: out_dtype must be PF_F16 or PF_F32");
  PF_CHECK_ARG(Cout > 0 && Cout % 2 == 0 && Cout <= Cw && out_ld >= Cout && out_ld % 2 == 0 &&
                   (!residual || out_ld == Cout),
               "pf_faedt_conv: Cout=%d Cw=%d out_ld=%d", Cout, Cw, out_ld);
  const long long M = (long long)B * Ho * Wo;
  PF_CHECK_ARG(M * (Cw > Cin ? Cw : Cin) < (1LL << 31) && (long long)B * H * W * Cin < (1LL << 31),
               "pf_faedt_conv: tensor too large");
  ConvArgs a{static_cast<const __half*>(x), static_cast<const __half*>(w), bias,
             static_cast<const __half*>(residual), out, B, H, W, Cin, Cout, Ho, Wo, kh, kw, stride, ph, pw, 0,
             out_dtype == PF_F32, Cw, out_ld, 0, (int)M, stride};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int kc = Cin >= 64 ? 64 : Cin;
  if (Cin % kc == 0) {
    if (kc == 16 && Cw == 32) return launch_conv<16, 32, true>(a, st);
    if (kc == 32 && Cw == 32) return launch_conv<32, 32, true>(a, st);
    if (kc == 32 && Cw == 64) return launch_conv<32, 64, true>(a, st);
    if (kc == 64 && Cw == 32) return launch_conv<64, 32, true>(a, st);
    if (kc == 64 && Cw == 64) return launch_conv<64, 64, true>(a, st);
    if (kc == 64 && Cw == 128) return launch_conv<64, 128, true>(a, st);
  }
  set_error("pf_faedt_conv: Cin=%d -> Cw=%d is not an FAED autoencoder layer or adjoint", Cin, Cw);
  return PF_ERR_UNSUPPORTED;
}

extern "C" long long pf_faedt_wgrad_ws_floats(int B, int Ho, int Wo, int Cin, int Cdy, int k) {
  const long long P = (long long)B * Ho * Wo;
  const int chunk = wgrad_chunk(P, k * k, Cin, Cdy);
  const long long nch = (P + chunk - 1) / chunk;
  return nch * ((long long)k * k * Cin * Cdy + Cdy);
}

extern "C" int pf_faedt_wgrad(const void* x, int B, int H, int W, int Cin, const void* dy, int Ho, int Wo, int Cdy,
                              int Cin_w, int Cout, int k, int stride, int pad, float* ws, const double* scale,
                              double inv_n, float* dw, float* db, int* flag, void* stream) {
  PF_CHECK_ARG(x && dy && ws && scale && dw && flag, "pf_faedt_wgrad: null pointer");
  PF_CHECK_ARG(B > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && k > 0 && (stride == 1 || stride == 2) && pad < W,
               "pf_faedt_wgrad: bad shape");
  PF_CHECK_ARG(Cin % 8 == 0 && Cin <= 128 && Cdy % 8 == 0 && Cdy <= 128 && Cin_w > 0 && Cin_w <= Cin && Cout > 0 &&
                   Cout <= Cdy,
               "pf_faedt_wgrad: channels Cin=%d Cdy=%d Cin_w=%d Cout=%d", Cin, Cdy, Cin_w, Cout);
  const long long P = (long long)B * Ho * Wo;
  PF_CHECK_ARG(P * (Cin > Cdy ? Cin : Cdy) < (1LL << 31) && (long long)B * H * W * Cin < (1LL << 31),
               "pf_faedt_wgrad: tensor too large");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int taps = k * k, chunk = wgrad_chunk(P, taps, Cin, Cdy);
  const int nch = (int)((P + chunk - 1) / chunk);
  const int BM = Cin <= 32 ? 32 : 64;
  const int BN = Cdy <= 32 ? 32 : (Cdy <= 64 ? 64 : 128);
  WgradArgs a{static_cast<const __half*>(x), static_cast<const __half*>(dy), ws, db ? ws + (size_t)nch * taps * Cin * Cdy : nullptr,
              B, H, W, Cin, Ho, Wo, Cdy, k, stride, pad, (int)P, chunk, (Cin + BM - 1) / BM};
  const dim3 grid(nch, taps * a.ci_tiles);
  if (BM == 32 && BN == 32) wgrad_kernel<32, 32><<<grid, 32, 0, st>>>(a);
  else if (BM == 32 && BN == 64) wgrad_kernel<32, 64><<<grid, 64, 0, st>>>(a);
  else if (BM == 64 && BN == 32) wgrad_kernel<64, 32><<<grid, 64, 0, st>>>(a);
  else if (BM == 64 && BN == 64) wgrad_kernel<64, 64><<<grid, 128, 0, st>>>(a);
  else if (BM == 64 && BN == 128) wgrad_kernel<64, 128><<<grid, 256, 0, st>>>(a);
  else {
    set_error("pf_faedt_wgrad: Cin=%d Cdy=%d has no tile", Cin, Cdy);
    return PF_ERR_UNSUPPORTED;
  }
  PF_CHECK_LAUNCH("wgrad_kernel");
  wgrad_reduce_kernel<<<blocks_for((long long)taps * Cin_w * Cout), 256, 0, st>>>(ws, nch, taps, Cin, Cdy, Cin_w,
                                                                                 Cout, scale, inv_n, dw, flag);
  if (db) db_reduce_kernel<<<1, 128, 0, st>>>(a.dbpart, nch, Cdy, Cout, scale, inv_n, db, flag);
  PF_CHECK_LAUNCH("wgrad_reduce_kernel");
  return PF_OK;
}

extern "C" long long pf_faedt_bn_ws_floats(long long P, int C) {
  return (P + row_chunk(P) - 1) / row_chunk(P) * 3LL * C + 2LL * C;
}

static int bn_check(long long P, int C, const char* what) {
  if (!(P > 1 && (C == 32 || C == 64 || C == 128) && P * C < (1LL << 40))) {
    set_error("%s: bad shape P=%lld C=%d (C 32/64/128, P > 1)", what, P, C);
    return PF_ERR_INVALID;
  }
  return PF_OK;
}

extern "C" int pf_faedt_bn_stats(const void* z, long long P, int C, float* ws, float* stats, float* pending,
                                 void* stream) {
  PF_CHECK_ARG(z && ws && stats && pending, "pf_faedt_bn_stats: null pointer");
  if (int rc = bn_check(P, C, "pf_faedt_bn_stats")) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int chunk = row_chunk(P), nch = (int)((P + chunk - 1) / chunk);
  bn_stats_part_kernel<<<nch, 256, 0, st>>>(static_cast<const __half*>(z), P, C, chunk, ws);
  bn_stats_merge_kernel<<<1, 128, 0, st>>>(ws, nch, C, stats);
  PF_CHECK_LAUNCH("bn_stats");
  // the running-statistics update (mean and unbiased var) waits for the step's end: a skipped step leaves them
  cudaError_t e = cudaMemcpyAsync(pending, stats, C * sizeof(float), cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(pending + C, stats + 2 * C, C * sizeof(float), cudaMemcpyDeviceToDevice, st);
  return check_cuda(e, "pf_faedt_bn_stats copy");
}

extern "C" int pf_faedt_bn_apply(const void* z, long long P, int C, const float* stats, const float* gamma,
                                 const float* beta, int relu, const void* residual, void* out, void* stream) {
  PF_CHECK_ARG(z && stats && gamma && beta && out, "pf_faedt_bn_apply: null pointer");
  if (int rc = bn_check(P, C, "pf_faedt_bn_apply")) return rc;
  bn_apply_kernel<<<blocks_for(P * C), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(z), P * C, C, stats, gamma, beta, relu, static_cast<const __half*>(residual),
      static_cast<__half*>(out));
  PF_CHECK_LAUNCH("bn_apply_kernel");
  return PF_OK;
}

extern "C" int pf_faedt_bn_bwd(const void* g, const void* mask, const void* z, long long P, int C, const float* stats,
                               const float* gamma, float* ws, const double* scale, double inv_n, float* dgamma,
                               float* dbeta, int* flag, void* dz, void* stream) {
  PF_CHECK_ARG(g && z && stats && gamma && ws && scale && dgamma && dbeta && flag && dz,
               "pf_faedt_bn_bwd: null pointer");
  if (int rc = bn_check(P, C, "pf_faedt_bn_bwd")) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int chunk = row_chunk(P), nch = (int)((P + chunk - 1) / chunk);
  const __half *gh = static_cast<const __half*>(g), *mh = static_cast<const __half*>(mask),
               *zh = static_cast<const __half*>(z);
  float* sums = ws + (size_t)nch * 3 * C;
  bn_bwd_part_kernel<<<nch, 256, 0, st>>>(gh, mh, zh, P, C, chunk, stats, ws);
  bn_bwd_merge_kernel<<<1, 128, 0, st>>>(ws, nch, C, P, scale, inv_n, sums, dgamma, dbeta, flag);
  bn_bwd_apply_kernel<<<blocks_for(P * C), 256, 0, st>>>(gh, mh, zh, P * C, C, stats, gamma, sums,
                                                         static_cast<__half*>(dz));
  PF_CHECK_LAUNCH("bn_bwd");
  return PF_OK;
}

extern "C" int pf_faedt_upsample(const void* x, int B, int H, int W, int C, void* out, void* stream) {
  PF_CHECK_ARG(x && out, "pf_faedt_upsample: null pointer");
  PF_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && 4LL * B * H * W * C < (1LL << 40), "pf_faedt_upsample: bad shape");
  upsample_kernel<<<blocks_for(4LL * B * H * W * C), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(x), B, H, W, C, static_cast<__half*>(out));
  PF_CHECK_LAUNCH("upsample_kernel");
  return PF_OK;
}

extern "C" int pf_faedt_upsample_bwd(const void* g, int B, int H, int W, int C, void* dx, void* stream) {
  PF_CHECK_ARG(g && dx, "pf_faedt_upsample_bwd: null pointer");
  PF_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && 4LL * B * H * W * C < (1LL << 40),
               "pf_faedt_upsample_bwd: bad shape");
  upsample_bwd_kernel<<<blocks_for((long long)B * H * W * C), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(g), B, H, W, C, static_cast<__half*>(dx));
  PF_CHECK_LAUNCH("upsample_bwd_kernel");
  return PF_OK;
}

extern "C" long long pf_faedt_loss_ws_floats(void) { return kLossBlocks; }

extern "C" int pf_faedt_loss(const float* o, const float* target, int B, int H, int W, const double* scale, float* ws,
                             float* loss, float* pred, void* seed, int* flag, void* stream) {
  PF_CHECK_ARG(o && scale && ws && loss && seed && flag, "pf_faedt_loss: null pointer");
  PF_CHECK_ARG(B > 0 && H > 0 && W > 0 && (long long)B * H * W * 16 < (1LL << 40), "pf_faedt_loss: bad shape");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  loss_part_kernel<<<kLossBlocks, 256, 0, st>>>(o, target, B, H, W, scale, pred, static_cast<__half*>(seed), ws);
  loss_final_kernel<<<1, 256, 0, st>>>(ws, kLossBlocks, 3.0 * B * H * W, loss, flag);
  PF_CHECK_LAUNCH("loss");
  return PF_OK;
}

extern "C" int pf_faedt_adam(float* params, const float* grads, float* m, float* v, long long n, float* running,
                             const float* pending, long long n_running, double* ctl, int* ictl,
                             long long* num_batches, double beta1, double beta2, double eps, void* stream) {
  PF_CHECK_ARG(params && grads && m && v && ctl && ictl && num_batches && (n_running == 0 || (running && pending)),
               "pf_faedt_adam: null pointer");
  PF_CHECK_ARG(n > 0 && n_running >= 0 && n_running <= n, "pf_faedt_adam: bad sizes");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  adam_kernel<<<blocks_for(n), 256, 0, st>>>(params, grads, m, v, n, running, pending, n_running, ctl, ictl, beta1,
                                             beta2, eps);
  step_end_kernel<<<1, 1, 0, st>>>(ctl, ictl, num_batches);
  PF_CHECK_LAUNCH("adam");
  return PF_OK;
}

extern "C" int pf_faedt_pack(const float* w, int Cout, int Cin, int k, int stride, void* fwd, int cin_pad, int cw,
                             void* dg, int dg_rows, int dg_cw, void* stream) {
  PF_CHECK_ARG(w && fwd, "pf_faedt_pack: null pointer");
  PF_CHECK_ARG(Cout > 0 && Cin > 0 && k > 0 && cin_pad >= Cin && cw >= Cout && (stride == 1 || (stride == 2 && k == 4)) &&
                   (!dg || (dg_rows >= Cout && dg_cw >= Cin && (stride == 2 || k % 2 == 1))),
               "pf_faedt_pack: bad shape");
  const long long n = (long long)k * k * cin_pad * cw + (dg ? (long long)k * k * dg_rows * dg_cw : 0);
  pack_kernel<<<blocks_for(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      w, Cout, Cin, k, stride, static_cast<__half*>(fwd), cin_pad, cw, static_cast<__half*>(dg), dg_rows, dg_cw);
  PF_CHECK_LAUNCH("pack_kernel");
  return PF_OK;
}

extern "C" int pf_faedt_interleave(const void* phases, int B, int H, int W, int C, void* dx, void* stream) {
  PF_CHECK_ARG(phases && dx, "pf_faedt_interleave: null pointer");
  PF_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && H % 2 == 0 && W % 2 == 0, "pf_faedt_interleave: bad shape");
  interleave_kernel<<<blocks_for((long long)B * H * W * C), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __half*>(phases), B, H, W, C, static_cast<__half*>(dx));
  PF_CHECK_LAUNCH("interleave_kernel");
  return PF_OK;
}
