// Small bandwidth-bound kernels at the edges of the UNet walk (models/pano/MVGenModel.py:52-60,85-91,279-295) and of
// the sampling loop (models/pano/PanFusion.py:146-162, PanoGenerator.py:253-269).
#include "pf_common.cuh"

namespace pf {

// ------------------------------------------------------------------------------------------------
// conv_in: NCHW fp32 latent [N,Cin<=8,H,W] -> channels-last tokens [N*H*W, Cout] (3x3, pad 1; `circ` wraps
// columns == pad_pano(1) -> conv -> unpad_pano(1), MVGenModel.py:87-91). Weights fp32 [Cout, Cin, 3, 3].
// thread <-> (pixel, 8 output channels)
// ------------------------------------------------------------------------------------------------
template <bool BF16>
__global__ void __launch_bounds__(256)
conv_in_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
               uint16_t* __restrict__ out, int N, int Cin, int H, int W, int Cout, int circ, int act) {
  // weights transposed into shared memory as [Cin*9][Cout] (+bias row): lanes read consecutive output channels
  extern __shared__ float s_w[];
  const int K = Cin * 9;
  for (int i = threadIdx.x; i < K * Cout; i += blockDim.x) {
    const int co = i % Cout, k = i / Cout;  // k = ci*9 + tap
    s_w[i] = w[(size_t)co * K + k];
  }
  float* s_b = s_w + K * Cout;
  for (int i = threadIdx.x; i < Cout; i += blockDim.x) s_b[i] = bias ? bias[i] : 0.f;
  __syncthreads();
  const int vecs = Cout / 8;
  if ((W & 3) == 0) {
    // register blocking: 4 consecutive pixels x 8 output channels per thread — each weight vector read from shared
    // memory feeds 4 pixels, each input value up to 3 taps (the unblocked loop was smem-bandwidth bound)
    const int Wq = W >> 2;
    const long long total = (long long)N * H * Wq * vecs;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
      const int v = int(idx % vecs);
      const long long quad = idx / vecs;
      const int xq = int(quad % Wq) * 4, yy = int((quad / Wq) % H), n = int(quad / ((long long)Wq * H));
      float acc[4][8];
#pragma unroll
      for (int pp = 0; pp < 4; ++pp)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[pp][e] = s_b[v * 8 + e];
      for (int ci = 0; ci < Cin; ++ci) {
        const float* xp = x + ((size_t)n * Cin + ci) * H * W;
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
          const int sy = yy + dy - 1;
          if (sy < 0 || sy >= H) continue;
          float in[6];
#pragma unroll
          for (int t = 0; t < 6; ++t) {
            int sx = xq + t - 1;
            bool ok = true;
            if (circ) sx = sx < 0 ? sx + W : (sx >= W ? sx - W : sx);
            else ok = sx >= 0 && sx < W;
            in[t] = ok ? __ldg(xp + sy * W + sx) : 0.f;
          }
#pragma unroll
          for (int dx = 0; dx < 3; ++dx) {
            const float4* wr = reinterpret_cast<const float4*>(s_w + (size_t)(ci * 9 + dy * 3 + dx) * Cout + v * 8);
            const float4 w0 = wr[0], w1 = wr[1];
            const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
            for (int pp = 0; pp < 4; ++pp)
#pragma unroll
              for (int e = 0; e < 8; ++e) acc[pp][e] = fmaf(in[pp + dx], wv[e], acc[pp][e]);
          }
        }
      }
      const size_t pix0 = ((size_t)n * H + yy) * W + xq;
      if (act == PF_ACT_SILU) {
#pragma unroll
        for (int pp = 0; pp < 4; ++pp)
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[pp][e] = silu_f(acc[pp][e]);
      }
#pragma unroll
      for (int pp = 0; pp < 4; ++pp)
        *reinterpret_cast<uint4*>(out + (pix0 + pp) * Cout + v * 8) =
            make_uint4(pack2<BF16>(acc[pp][0], acc[pp][1]), pack2<BF16>(acc[pp][2], acc[pp][3]),
                       pack2<BF16>(acc[pp][4], acc[pp][5]), pack2<BF16>(acc[pp][6], acc[pp][7]));
    }
    return;
  }
  const long long total = (long long)N * H * W * vecs;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int v = int(idx % vecs);
    const long long pix = idx / vecs;
    const int xx = int(pix % W), yy = int((pix / W) % H), n = int(pix / ((long long)W * H));
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = s_b[v * 8 + e];
    for (int ci = 0; ci < Cin; ++ci) {
      const float* xp = x + ((size_t)n * Cin + ci) * H * W;
#pragma unroll
      for (int dy = 0; dy < 3; ++dy) {
        const int sy = yy + dy - 1;
        if (sy < 0 || sy >= H) continue;
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          int sx = xx + dx - 1;
          if (circ) {
            sx = sx < 0 ? sx + W : (sx >= W ? sx - W : sx);
          } else if (sx < 0 || sx >= W) {
            continue;
          }
          const float val = __ldg(xp + sy * W + sx);
          const float4* wr = reinterpret_cast<const float4*>(s_w + (size_t)(ci * 9 + dy * 3 + dx) * Cout + v * 8);
          const float4 w0 = wr[0], w1 = wr[1];
          acc[0] = fmaf(val, w0.x, acc[0]); acc[1] = fmaf(val, w0.y, acc[1]);
          acc[2] = fmaf(val, w0.z, acc[2]); acc[3] = fmaf(val, w0.w, acc[3]);
          acc[4] = fmaf(val, w1.x, acc[4]); acc[5] = fmaf(val, w1.y, acc[5]);
          acc[6] = fmaf(val, w1.z, acc[6]); acc[7] = fmaf(val, w1.w, acc[7]);
        }
      }
    }
    if (act == PF_ACT_SILU) {
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = silu_f(acc[e]);
    }
    *reinterpret_cast<uint4*>(out + (size_t)pix * Cout + v * 8) =
        make_uint4(pack2<BF16>(acc[0], acc[1]), pack2<BF16>(acc[2], acc[3]), pack2<BF16>(acc[4], acc[5]),
                   pack2<BF16>(acc[6], acc[7]));
  }
}

// strided 2-D copy of 16-bit rows; src and dst may be column slices of wider tensors
__global__ void __launch_bounds__(256)
copy2d_kernel(const uint16_t* __restrict__ src, int src_ld, uint16_t* __restrict__ dst, int dst_ld, long long rows,
              int cols) {
  const int vecs = cols / 8;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * vecs) return;
  const long long r = idx / vecs;
  const int v = int(idx % vecs);
  *reinterpret_cast<uint4*>(dst + r * dst_ld + v * 8) = __ldg(reinterpret_cast<const uint4*>(src + r * src_ld + v * 8));
}

// pad_pano (utils/pano.py:74-99): circular padding of the last (longitude) axis; rows = every leading dim flattened
template <typename T>
__global__ void __launch_bounds__(256)
pad_pano_kernel(const T* __restrict__ x, T* __restrict__ out, long long rows, int W, int pad) {
  const int Wo = W + 2 * pad;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * Wo) return;
  const long long r = idx / Wo;
  int j = int(idx % Wo) - pad;
  j %= W;
  if (j < 0) j += W;
  out[idx] = __ldg(x + r * W + j);
}

// row softmax of fp32 logits -> 16-bit probabilities (the VAE mid-block attention: one head of width 512, computed as
// two tap-GEMMs around this kernel). One CTA per row; three passes over a row that stays in L1/L2.
template <bool BF16>
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ s, long long ld, uint16_t* __restrict__ out, long long ldo, int cols,
                    float scale) {
  __shared__ float red[8];
  const float* row = s + (size_t)blockIdx.x * ld;
  uint16_t* orow = out + (size_t)blockIdx.x * ldo;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float m = -INFINITY;
  for (int c = threadIdx.x; c < cols; c += 256) m = fmaxf(m, row[c]);
#pragma unroll
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red[warp] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
  __syncthreads();
  float sum = 0.f;
  for (int c = threadIdx.x; c < cols; c += 256) sum += expf((row[c] - m) * scale);
  sum = warp_sum(sum);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) sum += red[w];
  const float inv = 1.0f / sum;
  for (int c = 2 * threadIdx.x; c < cols; c += 512) {
    const float a = expf((row[c] - m) * scale) * inv;
    const float b = c + 1 < cols ? expf((row[c + 1] - m) * scale) * inv : 0.f;
    if (c + 1 < cols) *reinterpret_cast<uint32_t*>(orow + c) = pack2<BF16>(a, b);
    else orow[c] = (uint16_t)(pack2<BF16>(a, 0.f) & 0xffffu);
  }
}

// tensor_to_image (models/modules/utils.py:9-15): float [-1,1] planes [n, C, H, W] -> uint8 [n, H, W, C]
__global__ void __launch_bounds__(256)
tensor_to_image_kernel(const float* __restrict__ x, uint8_t* __restrict__ out, long long total, int C, int H, int W) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over the OUTPUT [n, H, W, C]
  if (idx >= total) return;
  const int c = int(idx % C);
  long long r = idx / C;
  const int xx = int(r % W);
  r /= W;
  const int yy = int(r % H);
  const long long n = r / H;
  float v = __ldg(x + ((n * C + c) * H + yy) * (long long)W + xx) / 2.0f + 0.5f;
  v = fminf(fmaxf(v, 0.f), 1.f);
  out[idx] = (uint8_t)rintf(v * 255.0f);
}

// diffusers Timesteps(dim, flip_sin_to_cos=True, downscale_freq_shift=0): [cos(t f_i) | sin(t f_i)], f_i = 10000^(-i/half)
template <bool BF16>
__global__ void timestep_embed_kernel(const float* __restrict__ t, uint16_t* __restrict__ out, int n, int dim) {
  const int half = dim / 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * half) return;
  const int r = idx / half, i = idx % half;
  const float freq = expf(-logf(10000.0f) * float(i) / float(half));
  const float ang = t[r] * freq;
  const float c = cosf(ang), s = sinf(ang);
  if constexpr (BF16) {
    reinterpret_cast<__nv_bfloat16*>(out)[(size_t)r * dim + i] = __float2bfloat16_rn(c);
    reinterpret_cast<__nv_bfloat16*>(out)[(size_t)r * dim + half + i] = __float2bfloat16_rn(s);
  } else {
    reinterpret_cast<__half*>(out)[(size_t)r * dim + i] = __float2half_rn(c);
    reinterpret_cast<__half*>(out)[(size_t)r * dim + half + i] = __float2half_rn(s);
  }
}

// CFG combine + DDIM update (+ optional column roll of the result): PanoGenerator.py:253-262, DDIMScheduler.step,
// PanoGenerator.py:264-269. eps holds [uncond | text] halves of `count` elements each; x, out are [rows, W] fp32.
__global__ void __launch_bounds__(256)
cfg_ddim_kernel(const float* __restrict__ x, const float* __restrict__ eps, float* __restrict__ out, long long count,
                int W, int roll, float guidance, float c_x, float c_eps, const float* __restrict__ coef_dev) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= count) return;
  if (coef_dev) {  // coefficients read from device memory so a captured CUDA graph can be replayed for any step
    c_x = coef_dev[0];
    c_eps = coef_dev[1];
  }
  const float eu = eps[idx], ec = eps[count + idx];
  const float e = eu + guidance * (ec - eu);
  const float v = c_x * x[idx] + c_eps * e;
  long long o = idx;
  if (roll) {
    const int col = int(idx % W);
    int nc = (col + roll) % W;
    if (nc < 0) nc += W;
    o = idx - col + nc;
  }
  out[o] = v;
}

// ------------------------------------------------------------------------------------------------
// Forward half of the training step (models/pano/PanFusion.py:64-98; SURVEY.md 8f rank 4 — the backward is not built)
// ------------------------------------------------------------------------------------------------
// diffusers SchedulerMixin.add_noise [3P] as called at PanFusion.py:84-85: one timestep per sample,
// out = sqrt(abar[t]) * x0 + sqrt(1 - abar[t]) * noise, every product and the sum rounded separately like the eager ops.
__global__ void __launch_bounds__(256)
add_noise_kernel(const float* __restrict__ x0, const float* __restrict__ noise, float* __restrict__ out,
                 const long long* __restrict__ t, const float* __restrict__ abar, int T, long long per_sample) {
  const int b = blockIdx.y;
  const long long tt = t[b];
  if (tt < 0 || tt >= T) __trap();  // torch raises IndexError
  const float a = __ldg(abar + tt);
  const float sa = __fsqrt_rn(a), s1 = __fsqrt_rn(__fsub_rn(1.0f, a));
  const long long base = (long long)b * per_sample;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_sample; i += (long long)gridDim.x * blockDim.x)
    out[base + i] = __fadd_rn(__fmul_rn(sa, __ldg(x0 + base + i)), __fmul_rn(s1, __ldg(noise + base + i)));
}

constexpr int MSE_CTAS = 296;  // fixed partition (2 per SM): the summation order never depends on the launch

// torch.nn.functional.mse_loss, mean reduction (PanFusion.py:92-93). Deterministic: element i always belongs to CTA
// i / chunk, a CTA sums its chunk in a fixed thread-strided order, the last CTA to finish adds the MSE_CTAS partials in
// index order in fp64 and re-arms the counter.
__global__ void __launch_bounds__(256)
mse_loss_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n, float* __restrict__ ws,
                int* __restrict__ counter, float* __restrict__ out) {
  __shared__ float red[8];
  __shared__ int s_last;
  const long long chunk = (n + MSE_CTAS - 1) / MSE_CTAS;
  const long long lo = (long long)blockIdx.x * chunk, hi = (lo + chunk < n) ? lo + chunk : n;
  float acc = 0.f;
  for (long long i = lo + threadIdx.x; i < hi; i += 256) {
    const float d = __ldg(a + i) - __ldg(b + i);
    acc = fmaf(d, d, acc);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w];
    ws[blockIdx.x] = s;
    __threadfence();
    s_last = (atomicAdd(counter, 1) == MSE_CTAS - 1);
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    __threadfence();
    double tot = 0.0;
    for (int i = 0; i < MSE_CTAS; ++i) tot += (double)__ldcg(ws + i);
    out[0] = (float)(tot / (double)n);
    *counter = 0;
  }
}

// diffusers DiagonalGaussianDistribution.sample + the scaling of PanoGenerator.encode_image (PanoGenerator.py:218-224):
// moments are channels-last rows [mean(0..L) | logvar(L..2L) | ...] (the fp32 output tile of the encoder's last tap-GEMM),
// eps and out are NCHW. z = (mean + exp(0.5 * clamp(logvar, -30, 20)) * eps) * scale, products and sum rounded separately.
__global__ void __launch_bounds__(256)
gaussian_sample_kernel(const float* __restrict__ moments, int ld, const float* __restrict__ eps, float* __restrict__ out,
                       long long total, int L, int HW, float scale) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over out [N, L, HW]
  if (idx >= total) return;
  const int px = int(idx % HW);
  const long long r = idx / HW;
  const int c = int(r % L);
  const long long n = r / L;
  const float* row = moments + (n * HW + px) * (long long)ld;
  const float mean = __ldg(row + c);
  const float logvar = fminf(fmaxf(__ldg(row + L + c), -30.0f), 20.0f);
  const float stdv = expf(__fmul_rn(0.5f, logvar));
  out[idx] = __fmul_rn(__fadd_rn(mean, __fmul_rn(stdv, __ldg(eps + idx))), scale);
}

}  // namespace pf

extern "C" int pf_conv_in(const float* x, const float* w, const float* bias, void* out, int dtype, int N, int Cin,
                          int H, int W, int Cout, int circ, int act, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(x && w && out, "pf_conv_in: null pointer");
  PF_CHECK_ARG(dtype == PF_BF16 || dtype == PF_F16, "pf_conv_in: 16-bit output dtype required");
  PF_CHECK_ARG(N > 0 && Cin > 0 && H > 0 && W > 0 && Cout > 0 && Cout % 8 == 0, "pf_conv_in: bad shape");
  PF_CHECK_ARG(act == PF_ACT_NONE || act == PF_ACT_SILU, "pf_conv_in: act must be none or silu");
  const long long total = (long long)N * H * ((W & 3) ? W : W / 4) * (Cout / 8);
  long long want = (total + 255) / 256;
  const unsigned blocks = (unsigned)(want < sm_count() * 4 ? want : sm_count() * 4);  // persistent-ish: weights staged once per CTA
  const size_t smem = ((size_t)Cin * 9 * Cout + Cout) * sizeof(float);
  PF_CHECK_ARG(smem <= 200 * 1024, "pf_conv_in: Cin*9*Cout too large for shared memory");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc;
  if (dtype == PF_BF16) {
    auto k = conv_in_kernel<true>;
    if ((rc = check_cuda(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "conv_in attr"))) return rc;
    k<<<blocks, 256, smem, st>>>(x, w, bias, static_cast<uint16_t*>(out), N, Cin, H, W, Cout, circ, act);
  } else {
    auto k = conv_in_kernel<false>;
    if ((rc = check_cuda(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "conv_in attr"))) return rc;
    k<<<blocks, 256, smem, st>>>(x, w, bias, static_cast<uint16_t*>(out), N, Cin, H, W, Cout, circ, act);
  }
  PF_CHECK_LAUNCH("conv_in_kernel");
  return PF_OK;
}

extern "C" int pf_copy2d(const void* src, int src_ld, void* dst, int dst_ld, long long rows, int cols, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(src && dst, "pf_copy2d: null pointer");
  PF_CHECK_ARG(rows > 0 && cols > 0 && cols % 8 == 0 && src_ld % 8 == 0 && dst_ld % 8 == 0 && src_ld >= cols && dst_ld >= cols,
               "pf_copy2d: bad shape rows=%lld cols=%d", rows, cols);
  PF_CHECK_ARG(((uintptr_t)src & 15) == 0 && ((uintptr_t)dst & 15) == 0, "pf_copy2d: pointers must be 16-byte aligned");
  const long long total = rows * (cols / 8);
  copy2d_kernel<<<(unsigned)((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint16_t*>(src), src_ld, static_cast<uint16_t*>(dst), dst_ld, rows, cols);
  PF_CHECK_LAUNCH("copy2d_kernel");
  return PF_OK;
}

extern "C" int pf_pad_pano(const void* x, void* out, int elem_bytes, long long rows, int W, int pad, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(x && out, "pf_pad_pano: null pointer");
  PF_CHECK_ARG(elem_bytes == 1 || elem_bytes == 2 || elem_bytes == 4 || elem_bytes == 8,
               "pf_pad_pano: elem_bytes must be 1, 2, 4 or 8");
  PF_CHECK_ARG(rows > 0 && W > 0 && pad > 0, "pf_pad_pano: bad shape rows=%lld W=%d pad=%d", rows, W, pad);
  const long long total = rows * (W + 2LL * pad);
  PF_CHECK_ARG(total <= 2147483647LL * 256, "pf_pad_pano: tensor too large");
  const unsigned blocks = (unsigned)((total + 255) / 256);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (elem_bytes) {
    case 1: pad_pano_kernel<uint8_t><<<blocks, 256, 0, st>>>(static_cast<const uint8_t*>(x), static_cast<uint8_t*>(out), rows, W, pad); break;
    case 2: pad_pano_kernel<uint16_t><<<blocks, 256, 0, st>>>(static_cast<const uint16_t*>(x), static_cast<uint16_t*>(out), rows, W, pad); break;
    case 4: pad_pano_kernel<uint32_t><<<blocks, 256, 0, st>>>(static_cast<const uint32_t*>(x), static_cast<uint32_t*>(out), rows, W, pad); break;
    default: pad_pano_kernel<uint64_t><<<blocks, 256, 0, st>>>(static_cast<const uint64_t*>(x), static_cast<uint64_t*>(out), rows, W, pad); break;
  }
  PF_CHECK_LAUNCH("pad_pano_kernel");
  return PF_OK;
}

extern "C" int pf_softmax_rows(const float* s, long long ld, void* out, long long ldo, int dtype, long long rows,
                               int cols, float scale, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(s && out, "pf_softmax_rows: null pointer");
  PF_CHECK_ARG(dtype == PF_BF16 || dtype == PF_F16, "pf_softmax_rows: 16-bit output dtype required");
  PF_CHECK_ARG(rows > 0 && rows <= 2147483647LL && cols > 0 && ld >= cols && ldo >= cols && ldo % 2 == 0,
               "pf_softmax_rows: bad shape rows=%lld cols=%d", rows, cols);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PF_BF16) softmax_rows_kernel<true><<<(unsigned)rows, 256, 0, st>>>(s, ld, static_cast<uint16_t*>(out), ldo, cols, scale);
  else softmax_rows_kernel<false><<<(unsigned)rows, 256, 0, st>>>(s, ld, static_cast<uint16_t*>(out), ldo, cols, scale);
  PF_CHECK_LAUNCH("softmax_rows_kernel");
  return PF_OK;
}

extern "C" int pf_tensor_to_image(const float* x, unsigned char* out, long long n, int C, int H, int W, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(x && out, "pf_tensor_to_image: null pointer");
  PF_CHECK_ARG(n > 0 && C > 0 && H > 0 && W > 0, "pf_tensor_to_image: bad shape");
  const long long total = n * C * H * W;
  PF_CHECK_ARG(total <= 2147483647LL * 256, "pf_tensor_to_image: tensor too large");
  tensor_to_image_kernel<<<(unsigned)((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, out, total, C, H, W);
  PF_CHECK_LAUNCH("tensor_to_image_kernel");
  return PF_OK;
}

// ------------------------------------------------------------------------------------------------
// CLIP text embeddings (transformers CLIPTextEmbeddings [3P], called through PanoGenerator.encode_text,
// models/pano/PanoGenerator.py:197-211): x[t, :] = token_embedding[ids[t], :] + position_embedding[t % L, :], plus the
// per-row (sum, sum of squares) the first layer's fused LayerNorm consumes (two slots per row, the second zero).
// One warp per token.
// ------------------------------------------------------------------------------------------------
namespace pf {
template <bool BF16>
__global__ void __launch_bounds__(256)
embed_tokens_kernel(const long long* __restrict__ ids, const float* __restrict__ tok, const float* __restrict__ pos,
                    uint16_t* __restrict__ out, float* __restrict__ stats, int T, int L, int C, int vocab) {
  const int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  long long id = ids[t];
  if (id < 0 || id >= vocab) __trap();  // torch.nn.Embedding raises an IndexError for such ids
  const float* tr = tok + (size_t)id * C;
  const float* pr = pos + (size_t)(t % L) * C;
  float s = 0.f, q = 0.f;
  for (int c = lane * 2; c < C; c += 64) {
    const float a = __ldg(tr + c) + __ldg(pr + c), b = __ldg(tr + c + 1) + __ldg(pr + c + 1);
    const uint32_t w = pack2<BF16>(a, b);
    const float2 r = unpack2<BF16>(w);  // statistics of the STORED (16-bit) row, like a LayerNorm kernel reading it would see
    s += r.x + r.y;
    q = fmaf(r.x, r.x, fmaf(r.y, r.y, q));
    *reinterpret_cast<uint32_t*>(out + (size_t)t * C + c) = w;
  }
  s = warp_sum(s);
  q = warp_sum(q);
  if (lane == 0) {
    reinterpret_cast<float4*>(stats)[t] = make_float4(s, q, 0.f, 0.f);
  }
}
}  // namespace pf

extern "C" int pf_embed_tokens(const long long* ids, const float* tok_emb, const float* pos_emb, void* out, int dtype,
                               float* row_stats, int T, int L, int C, int vocab, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(ids && tok_emb && pos_emb && out && row_stats, "pf_embed_tokens: null pointer");
  PF_CHECK_ARG(dtype == PF_BF16 || dtype == PF_F16, "pf_embed_tokens: 16-bit output required");
  PF_CHECK_ARG(T > 0 && L > 0 && C > 0 && C % 2 == 0 && vocab > 0, "pf_embed_tokens: bad shape T=%d L=%d C=%d", T, L, C);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int blocks = (T + 7) / 8;
  if (dtype == PF_BF16)
    embed_tokens_kernel<true><<<blocks, 256, 0, st>>>(ids, tok_emb, pos_emb, static_cast<uint16_t*>(out), row_stats, T, L, C, vocab);
  else
    embed_tokens_kernel<false><<<blocks, 256, 0, st>>>(ids, tok_emb, pos_emb, static_cast<uint16_t*>(out), row_stats, T, L, C, vocab);
  PF_CHECK_LAUNCH("embed_tokens_kernel");
  return PF_OK;
}

extern "C" int pf_timestep_embed(const float* t, void* out, int dtype, int n, int dim, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(t && out && n > 0 && dim > 0 && dim % 2 == 0, "pf_timestep_embed: bad arguments");
  PF_CHECK_ARG(dtype == PF_BF16 || dtype == PF_F16, "pf_timestep_embed: 16-bit output dtype required");
  const int total = n * dim / 2;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PF_BF16) timestep_embed_kernel<true><<<(total + 127) / 128, 128, 0, st>>>(t, static_cast<uint16_t*>(out), n, dim);
  else timestep_embed_kernel<false><<<(total + 127) / 128, 128, 0, st>>>(t, static_cast<uint16_t*>(out), n, dim);
  PF_CHECK_LAUNCH("timestep_embed_kernel");
  return PF_OK;
}

extern "C" int pf_cfg_ddim_step(const float* x, const float* eps, float* out, long long count, int W, int roll,
                                float guidance, float alpha_t, float alpha_prev, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(x && eps && out && count > 0 && W > 0 && count % W == 0, "pf_cfg_ddim_step: bad arguments");
  PF_CHECK_ARG(alpha_t > 0.f && alpha_t <= 1.f && alpha_prev > 0.f && alpha_prev <= 1.f, "pf_cfg_ddim_step: bad alphas");
  // x_prev = sqrt(a_prev) * (x - sqrt(1-a_t) e) / sqrt(a_t) + sqrt(1-a_prev) e
  const double sa = sqrt((double)alpha_prev / (double)alpha_t);
  const float c_x = (float)sa;
  const float c_eps = (float)(sqrt(1.0 - (double)alpha_prev) - sa * sqrt(1.0 - (double)alpha_t));
  cfg_ddim_kernel<<<(unsigned)((count + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, eps, out, count, W, roll, guidance, c_x, c_eps, nullptr);
  PF_CHECK_LAUNCH("cfg_ddim_kernel");
  return PF_OK;
}

extern "C" int pf_cfg_ddim_step_dev(const float* x, const float* eps, float* out, long long count, int W, int roll,
                                    float guidance, const float* coef, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(x && eps && out && coef && count > 0 && W > 0 && count % W == 0, "pf_cfg_ddim_step_dev: bad arguments");
  cfg_ddim_kernel<<<(unsigned)((count + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, eps, out, count, W, roll, guidance, 0.f, 0.f, coef);
  PF_CHECK_LAUNCH("cfg_ddim_kernel");
  return PF_OK;
}

extern "C" int pf_add_noise(const float* x0, const float* noise, float* out, const long long* t, const float* alphas_cumprod,
                            int num_train_timesteps, int B, long long per_sample, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(x0 && noise && out && t && alphas_cumprod && num_train_timesteps > 0 && B > 0 && B <= 65535 && per_sample > 0,
               "pf_add_noise: bad arguments");
  long long bx = (per_sample + 255) / 256;
  if (bx > 1184) bx = 1184;
  add_noise_kernel<<<dim3((unsigned)bx, B), 256, 0, static_cast<cudaStream_t>(stream)>>>(x0, noise, out, t, alphas_cumprod,
                                                                                        num_train_timesteps, per_sample);
  PF_CHECK_LAUNCH("add_noise_kernel");
  return PF_OK;
}

extern "C" int pf_mse_loss_ws_floats(void) { return pf::MSE_CTAS; }

extern "C" int pf_mse_loss(const float* a, const float* b, long long n, float* ws, int* counter, float* out, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(a && b && ws && counter && out && n > 0, "pf_mse_loss: bad arguments");
  mse_loss_kernel<<<MSE_CTAS, 256, 0, static_cast<cudaStream_t>(stream)>>>(a, b, n, ws, counter, out);
  PF_CHECK_LAUNCH("mse_loss_kernel");
  return PF_OK;
}

extern "C" int pf_gaussian_sample(const float* moments, int ld, const float* eps, float* out, int N, int L, int HW, float scale,
                                  void* stream) {
  using namespace pf;
  PF_CHECK_ARG(moments && eps && out && N > 0 && L > 0 && HW > 0 && ld >= 2 * L, "pf_gaussian_sample: bad arguments");
  const long long total = (long long)N * L * HW;
  gaussian_sample_kernel<<<(unsigned)((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(moments, ld, eps, out,
                                                                                                       total, L, HW, scale);
  PF_CHECK_LAUNCH("gaussian_sample_kernel");
  return PF_OK;
}
