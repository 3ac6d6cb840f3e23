// FAED (PanFusion's Fréchet AutoEncoder Distance, models/faed/FAED.py:50-103): the FAED encoder's circular-padded
// convolutions (models/faed/modules.py:5-36,176-264), the latitude-weighted W-mean pooling (FAED.py:69-78), the fp64
// feature statistics (FAED.py:80-90) and the Fréchet distance (FAED.py:92-103 + torchmetrics' _compute_fid) in fp64.
//
// Activations are channels-last fp16 [B, H, W, C]. CircularPadding(p) zero-pads rows and wraps columns (corners are
// zero), so the convolution addresses its operand directly: input row iy = oy*s + ky - p is zero outside [0, H), input
// column ix = ox*s + kx - p is taken modulo W. No padded copy is made. pf_conv_circ runs the implicit-GEMM core of
// conv_mma.cuh (shared with the FID InceptionV3) with circular padding.
#include "conv_mma.cuh"

namespace pf {
namespace faed {

constexpr int kPrepC = 16;  // the first layer's operand: 3 image channels + 13 zero channels (one 16-wide MMA k-step)

// ---------------------------------------------------------------------------------------------------------------------
// pf_faed_prep: x = img.float32 / 127.5 - 1 (FAED.py:70), rounded once to fp16, NCHW -> [B, H, W, 16]
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
prep_kernel(const void* __restrict__ src, int is_u8, int B, int C, int H, int W, __half* __restrict__ dst) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long HW = (long long)H * W;
  if (idx >= B * HW) return;
  const long long b = idx / HW, p = idx % HW;
  __align__(16) __half v[kPrepC];
#pragma unroll
  for (int c = 0; c < kPrepC; ++c) v[c] = __float2half_rn(0.f);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const long long s = (b * C + c) * HW + p;
    const float f = is_u8 ? (float)static_cast<const uint8_t*>(src)[s] : static_cast<const float*>(src)[s];
    v[c] = __float2half_rn(__fsub_rn(__fdiv_rn(f, 127.5f), 1.0f));
  }
  uint4* d = reinterpret_cast<uint4*>(dst + idx * kPrepC);
  d[0] = reinterpret_cast<const uint4*>(v)[0];
  d[1] = reinterpret_cast<const uint4*>(v)[1];
}

// ---------------------------------------------------------------------------------------------------------------------
// pf_faed_pool: torch.mean(features, dim=3) * cos(linspace(pi/2, -pi/2, h)) flattened channel-major (FAED.py:72-77)
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
pool_kernel(const float* __restrict__ x, int B, int h, int w, int C, const float* __restrict__ weight,
            float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * h * C) return;
  const int c = idx % C, y = (idx / C) % h, b = idx / (C * h);
  const float* p = x + ((size_t)(b * h + y) * w) * C + c;
  float s = 0.f;
  for (int i = 0; i < w; ++i) s += p[(size_t)i * C];
  out[(size_t)b * C * h + c * h + y] = __fmul_rn(weight[y], __fdiv_rn(s, (float)w));
}

// ---------------------------------------------------------------------------------------------------------------------
// pf_faed_stats: sum += X.sum(0), cov_sum += X^T X in fp64 (FAED.py:80-90). Every output is one thread's sum over the
// samples in index order, then added to the state, so the bits do not depend on the launch.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
stats_kernel(const float* __restrict__ X, int n, int d, double* __restrict__ sum, double* __restrict__ cov) {
  __shared__ double xa[16][16], xb[16][16];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int a = blockIdx.y * 16 + ty, b = blockIdx.x * 16 + tx;
  double acc = 0.0, s = 0.0;
  for (int i0 = 0; i0 < n; i0 += 16) {
    const int i = i0 + ty;
    xa[ty][tx] = i < n && blockIdx.y * 16 + tx < d ? (double)X[(size_t)i * d + blockIdx.y * 16 + tx] : 0.0;
    xb[ty][tx] = i < n && b < d ? (double)X[(size_t)i * d + b] : 0.0;
    __syncthreads();
    const int lim = min(16, n - i0);
    for (int k = 0; k < lim; ++k) {
      acc = __fma_rn(xa[k][ty], xb[k][tx], acc);  // the product of two floats is exact in fp64
      s = __dadd_rn(s, xb[k][tx]);
    }
    __syncthreads();
  }
  if (a < d && b < d) cov[(size_t)a * d + b] = __dadd_rn(cov[(size_t)a * d + b], acc);
  if (blockIdx.y == 0 && ty == 0 && b < d) sum[b] = __dadd_rn(sum[b], s);
}

// ---------------------------------------------------------------------------------------------------------------------
// pf_frechet_fp64. For PSD S1, S2: sum sqrt(eig(S1 S2)) = sum of the singular values of L1^T L2 for any factors
// S_i = L_i L_i^T. L_i^T = diag(sqrt(max(lambda, 0))) U^T comes from a one-sided (Hestenes) Jacobi on S_i, and the
// singular values of G = L1^T L2 from a second one. Jacobi rotates row pairs in round-robin order (n/2 disjoint pairs
// per launch, one CTA per pair, reductions in a fixed order), so the result is deterministic, and it never leaves the
// PSD cone: an eigenvalue that rounding made slightly negative is clamped to 0, which is what Re(sqrt()) of the
// reference's tiny negative eigenvalues gives.
// ---------------------------------------------------------------------------------------------------------------------
constexpr double kJacobiTol = 1e-13;  // |<a_i, a_j>| / (|a_i| |a_j|) below this counts as orthogonal
constexpr int kMaxSweeps = 100;  // a full-rank d = 512 covariance with condition 1.7e9 takes 30

template <int N>
__device__ __forceinline__ void block_sum(double* v, double* red) {
  // fixed-order tree over 256 threads, N values at once
  const int t = threadIdx.x;
#pragma unroll
  for (int q = 0; q < N; ++q) red[q * 256 + t] = v[q];
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if (t < off)
#pragma unroll
      for (int q = 0; q < N; ++q) red[q * 256 + t] = __dadd_rn(red[q * 256 + t], red[q * 256 + t + off]);
    __syncthreads();
  }
#pragma unroll
  for (int q = 0; q < N; ++q) v[q] = red[q * 256];
  __syncthreads();
}

// cov = (cov_sum - n mu mu^T) / (n - 1), mu = sum / n (FAED.py:96-101)
__global__ void __launch_bounds__(256)
cov_kernel(const double* __restrict__ sum, const double* __restrict__ cov_sum, long long n, int d,
           double* __restrict__ cov) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)d * d) return;
  const int i = (int)(idx / d), j = (int)(idx % d);
  const double mi = sum[i] / (double)n, mj = sum[j] / (double)n;
  cov[idx] = (cov_sum[idx] - (double)n * (mi * mj)) / (double)(n - 1);
}

// scal[0] = |mu1 - mu2|^2, scal[1] = tr S1, scal[2] = tr S2
__global__ void __launch_bounds__(256)
scalars_kernel(const double* sum1, long long n1, const double* sum2, long long n2, const double* S1,
               const double* S2, int d, double* scal) {
  __shared__ double red[3 * 256];
  double v[3] = {0.0, 0.0, 0.0};
  for (int i = threadIdx.x; i < d; i += 256) {
    const double diff = sum1[i] / (double)n1 - sum2[i] / (double)n2;
    v[0] += diff * diff;
    v[1] += S1[(size_t)i * d + i];
    v[2] += S2[(size_t)i * d + i];
  }
  block_sum<3>(v, red);
  if (threadIdx.x == 0)
    for (int q = 0; q < 3; ++q) scal[q] = v[q];
}

// out[0] = |A|_F^2
__global__ void __launch_bounds__(256)
sumsq_kernel(const double* A, long long len, double* out) {
  __shared__ double red[256];
  double x[1] = {0.0};
  for (long long e = threadIdx.x; e < len; e += 256) x[0] = __fma_rn(A[e], A[e], x[0]);
  block_sum<1>(x, red);
  if (threadIdx.x == 0) out[0] = x[0];
}

__global__ void identity_kernel(double* V, int d) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < (long long)d * d) V[idx] = (idx / d == idx % d) ? 1.0 : 0.0;
}

// one round of the round-robin schedule: pair k of round r is (r, n-1) for k = 0, else ((r+k), (r-k)) mod (n-1)
__global__ void __launch_bounds__(256)
jacobi_round_kernel(double* A, double* V, int n, int round, const double* fro2, unsigned long long* off_max) {
  __shared__ double red[3 * 256];
  __shared__ double rot[2];
  const int k = blockIdx.x, m = n - 1;
  int i = k == 0 ? round : (round + k) % m;
  int j = k == 0 ? m : (round - k + m) % m;
  if (i > j) {
    const int t = i;
    i = j;
    j = t;
  }
  double* ai = A + (size_t)i * n;
  double* aj = A + (size_t)j * n;
  double v[3] = {0.0, 0.0, 0.0};
  for (int e = threadIdx.x; e < n; e += 256) {
    const double x = ai[e], y = aj[e];
    v[0] = __fma_rn(x, x, v[0]);
    v[1] = __fma_rn(y, y, v[1]);
    v[2] = __fma_rn(x, y, v[2]);
  }
  block_sum<3>(v, red);
  if (threadIdx.x == 0) {
    const double al = v[0], be = v[1], ga = v[2];
    double c = 1.0, s = 0.0;
    if (al > 0.0 && be > 0.0) {
      const double off = fabs(ga) / (sqrt(al) * sqrt(be));
      // A pair whose inner product is below tol * |A|_F^2 (invariant under the rotations) is rotated but does not hold
      // the sweep back: such pairs are rounding-level rows of a rank-deficient S and move sum |a_i| by less than the
      // eigenvalues' own rounding. Without this the rank-deficient cases take 5-10x more sweeps for the same result.
      if (fabs(ga) > kJacobiTol * fro2[0])
        atomicMax(off_max, (unsigned long long)__double_as_longlong(off));  // non-negative doubles order as integers
      if (off > kJacobiTol) {
        const double zeta = (be - al) / (2.0 * ga);
        const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        c = 1.0 / sqrt(1.0 + t * t);
        s = c * t;
      }
    }
    rot[0] = c;
    rot[1] = s;
  }
  __syncthreads();
  const double c = rot[0], s = rot[1];
  if (s == 0.0) return;
  for (int e = threadIdx.x; e < n; e += 256) {
    const double x = ai[e], y = aj[e];
    ai[e] = c * x - s * y;
    aj[e] = s * x + c * y;
  }
  if (V) {
    double* vi = V + (size_t)i * n;
    double* vj = V + (size_t)j * n;
    for (int e = threadIdx.x; e < n; e += 256) {
      const double x = vi[e], y = vj[e];
      vi[e] = c * x - s * y;
      vj[e] = s * x + c * y;
    }
  }
}

// rows of A are lambda_i u_i^T and rows of V are u_i^T: V row i <- sqrt(max(<A_i, V_i>, 0)) V_i   (= L^T)
__global__ void __launch_bounds__(256)
scale_rows_kernel(const double* A, double* V, int n) {
  __shared__ double red[256];
  const double* a = A + (size_t)blockIdx.x * n;
  double* v = V + (size_t)blockIdx.x * n;
  double x[1] = {0.0};
  for (int e = threadIdx.x; e < n; e += 256) x[0] = __fma_rn(a[e], v[e], x[0]);
  block_sum<1>(x, red);
  const double s = sqrt(fmax(x[0], 0.0));
  for (int e = threadIdx.x; e < n; e += 256) v[e] *= s;
}

// C[a][b] = sum_k P[a][k] Q[b][k], d % 64 == 0; 64x64 tiles, 4x4 per thread
__global__ void __launch_bounds__(256)
gemm_nt_kernel(const double* __restrict__ P, const double* __restrict__ Q, double* __restrict__ Cm, int d) {
  __shared__ double Ps[16][64 + 1], Qs[16][64 + 1];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int a0 = blockIdx.y * 64, b0 = blockIdx.x * 64;
  double acc[4][4] = {};
  for (int k0 = 0; k0 < d; k0 += 16) {
    for (int e = threadIdx.x; e < 16 * 64; e += 256) {
      const int r = e / 16, kk = e % 16;
      Ps[kk][r] = P[(size_t)(a0 + r) * d + k0 + kk];
      Qs[kk][r] = Q[(size_t)(b0 + r) * d + k0 + kk];
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      double p[4], q[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        p[u] = Ps[kk][ty + 16 * u];
        q[u] = Qs[kk][tx + 16 * u];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int w = 0; w < 4; ++w) acc[u][w] = __fma_rn(p[u], q[w], acc[u][w]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int w = 0; w < 4; ++w) Cm[(size_t)(a0 + ty + 16 * u) * d + b0 + tx + 16 * w] = acc[u][w];
}

// out = |mu1 - mu2|^2 + tr S1 + tr S2 - 2 sum_i |G_i|   (rows of G orthogonal: their norms are its singular values)
__global__ void __launch_bounds__(256)
finish_kernel(const double* G, int n, const double* scal, double* out) {
  __shared__ double red[256];
  double x[1] = {0.0};
  for (int r = threadIdx.x; r < n; r += 256) {
    const double* g = G + (size_t)r * n;
    double s = 0.0;
    for (int e = 0; e < n; ++e) s = __fma_rn(g[e], g[e], s);
    x[0] += sqrt(s);
  }
  block_sum<1>(x, red);
  if (threadIdx.x == 0) out[0] = scal[0] + scal[1] + scal[2] - 2.0 * x[0];
}

int jacobi(double* A, double* V, int n, double* fro2, unsigned long long* off_dev, cudaStream_t st,
           const char* what, int* sweeps) {
  sumsq_kernel<<<1, 256, 0, st>>>(A, (long long)n * n, fro2);
  for (int sweep = 0; sweep < kMaxSweeps; ++sweep) {
    int rc = check_cuda(cudaMemsetAsync(off_dev, 0, sizeof(unsigned long long), st), "cudaMemsetAsync");
    if (rc) return rc;
    for (int r = 0; r < n - 1; ++r) jacobi_round_kernel<<<n / 2, 256, 0, st>>>(A, V, n, r, fro2, off_dev);
    PF_CHECK_LAUNCH("jacobi_round_kernel");
    unsigned long long bits = 0;
    rc = check_cuda(cudaMemcpyAsync(&bits, off_dev, sizeof(bits), cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync");
    if (rc) return rc;
    rc = check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize");
    if (rc) return rc;
    double off;
    memcpy(&off, &bits, sizeof(off));
    if (off <= kJacobiTol) {  // a whole sweep without a rotation
      if (sweeps) *sweeps = sweep + 1;
      return PF_OK;
    }
  }
  set_error("pf_frechet_fp64: the Jacobi iteration for %s did not converge in %d sweeps", what, kMaxSweeps);
  return PF_ERR_UNSUPPORTED;
}

}  // namespace faed
}  // namespace pf

using namespace pf;
using namespace pf::faed;
using pf::convmma::ConvArgs;
using pf::convmma::launch_conv;

extern "C" int pf_faed_prep(const void* src, int is_u8, int B, int C, int H, int W, void* dst, void* stream) {
  PF_CHECK_ARG(src && dst, "pf_faed_prep: null pointer");
  PF_CHECK_ARG(B > 0 && C >= 3 && H > 0 && W > 0 && (long long)B * H * W < (1LL << 31),
               "pf_faed_prep: bad shape B=%d C=%d H=%d W=%d (need C >= 3)", B, C, H, W);
  const long long n = (long long)B * H * W;
  prep_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(src, is_u8, B, C, H, W,
                                                                                          static_cast<__half*>(dst));
  PF_CHECK_LAUNCH("prep_kernel");
  return PF_OK;
}

extern "C" int pf_conv_circ(const void* x, int B, int H, int W, int Cin, const void* w, const float* bias, int Cout,
                            int k, int stride, int pad, int relu, const void* residual, void* out, int out_dtype,
                            void* stream) {
  PF_CHECK_ARG(x && w && bias && out, "pf_conv_circ: null pointer");
  PF_CHECK_ARG(B > 0 && H > 0 && W > 0 && k > 0 && stride > 0 && pad >= 0, "pf_conv_circ: bad shape");
  PF_CHECK_ARG(out_dtype == PF_F16 || out_dtype == PF_F32, "pf_conv_circ: out_dtype must be PF_F16 or PF_F32");
  const bool s1 = stride == 1 && (k == 3 || k == 5 || k == 7 || k == 9) && pad == k / 2;
  const bool s2 = stride == 2 && k == 4 && pad == 1;
  if (!(s1 || s2)) {
    set_error("pf_conv_circ: k=%d stride=%d pad=%d is not a FAED encoder layer (k 3/5/7/9 stride 1 pad k/2, or k 4 "
              "stride 2 pad 1)", k, stride, pad);
    return PF_ERR_UNSUPPORTED;
  }
  if (!(Cin == 16 || Cin == 32 || Cin == 64 || Cin == 128) || !(Cout == 32 || Cout == 64 || Cout == 128)) {
    set_error("pf_conv_circ: Cin=%d Cout=%d unsupported (Cin 16/32/64/128, Cout 32/64/128)", Cin, Cout);
    return PF_ERR_UNSUPPORTED;
  }
  PF_CHECK_ARG(pad < W, "pf_conv_circ: circular padding %d needs W > pad (W=%d)", pad, W);
  PF_CHECK_ARG(!(s2 && (H % 2 || W % 2)), "pf_conv_circ: the stride-2 layer needs even H and W (H=%d W=%d)", H, W);
  // one N tile of width Cout (grid.y = 1), circular W; the weight is packed [k*k][Cin][Cout]
  ConvArgs a{static_cast<const __half*>(x), static_cast<const __half*>(w), bias,
             static_cast<const __half*>(residual), out, B, H, W, Cin, Cout,
             (H + 2 * pad - k) / stride + 1, (W + 2 * pad - k) / stride + 1, k, k, stride, pad, pad, relu,
             out_dtype == PF_F32, Cout, Cout, 0, 0};
  const long long M = (long long)B * a.Ho * a.Wo;
  PF_CHECK_ARG(M > 0 && M * (Cout > Cin ? Cout : Cin) < (1LL << 31), "pf_conv_circ: tensor too large");
  a.M = (int)M;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int kc = Cin >= 64 ? 64 : Cin;
  if (kc == 16 && Cout == 32) return launch_conv<16, 32, true>(a, st);
  if (kc == 32 && Cout == 32) return launch_conv<32, 32, true>(a, st);
  if (kc == 32 && Cout == 64) return launch_conv<32, 64, true>(a, st);
  if (kc == 64 && Cout == 64) return launch_conv<64, 64, true>(a, st);
  if (kc == 64 && Cout == 128) return launch_conv<64, 128, true>(a, st);
  set_error("pf_conv_circ: Cin=%d -> Cout=%d is not a FAED encoder layer", Cin, Cout);
  return PF_ERR_UNSUPPORTED;
}

extern "C" int pf_faed_pool(const float* x, int B, int h, int w, int C, const float* weight, float* out,
                            void* stream) {
  PF_CHECK_ARG(x && weight && out, "pf_faed_pool: null pointer");
  PF_CHECK_ARG(B > 0 && h > 0 && w > 0 && C > 0 && (long long)B * h * w * C < (1LL << 31),
               "pf_faed_pool: bad shape B=%d h=%d w=%d C=%d", B, h, w, C);
  const int n = B * h * C;
  pool_kernel<<<(n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, B, h, w, C, weight, out);
  PF_CHECK_LAUNCH("pool_kernel");
  return PF_OK;
}

extern "C" int pf_faed_stats(const float* features, int n, int d, double* sum, double* cov_sum, void* stream) {
  PF_CHECK_ARG(features && sum && cov_sum, "pf_faed_stats: null pointer");
  PF_CHECK_ARG(n > 0 && d > 0 && (long long)n * d < (1LL << 31) && (long long)d * d < (1LL << 31),
               "pf_faed_stats: bad shape n=%d d=%d", n, d);
  const dim3 grid((d + 15) / 16, (d + 15) / 16);
  stats_kernel<<<grid, dim3(16, 16), 0, static_cast<cudaStream_t>(stream)>>>(features, n, d, sum, cov_sum);
  PF_CHECK_LAUNCH("stats_kernel");
  return PF_OK;
}

extern "C" long long pf_frechet_ws_doubles(int d) { return 4LL * d * d + 8; }

extern "C" int pf_frechet_fp64(const double* sum1, const double* cov_sum1, long long n1, const double* sum2,
                               const double* cov_sum2, long long n2, int d, double* ws, double* out, int* sweeps,
                               void* stream) {
  PF_CHECK_ARG(sum1 && cov_sum1 && sum2 && cov_sum2 && ws && out, "pf_frechet_fp64: null pointer");
  PF_CHECK_ARG(n1 >= 2 && n2 >= 2, "pf_frechet_fp64: more than one sample is required on both sides (n1=%lld "
               "n2=%lld)", n1, n2);
  PF_CHECK_ARG(d > 0 && d % 64 == 0 && (long long)d * d < (1LL << 31), "pf_frechet_fp64: d=%d must be a positive "
               "multiple of 64", d);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t dd = (size_t)d * d;
  double *S1 = ws, *S2 = ws + dd, *V1 = ws + 2 * dd, *V2 = ws + 3 * dd, *scal = ws + 4 * dd;
  double* fro2 = scal + 3;
  unsigned long long* off = reinterpret_cast<unsigned long long*>(scal + 4);
  const unsigned g = (unsigned)((dd + 255) / 256);
  cov_kernel<<<g, 256, 0, st>>>(sum1, cov_sum1, n1, d, S1);
  cov_kernel<<<g, 256, 0, st>>>(sum2, cov_sum2, n2, d, S2);
  scalars_kernel<<<1, 256, 0, st>>>(sum1, n1, sum2, n2, S1, S2, d, scal);
  identity_kernel<<<g, 256, 0, st>>>(V1, d);
  identity_kernel<<<g, 256, 0, st>>>(V2, d);
  PF_CHECK_LAUNCH("frechet setup");
  int rc = jacobi(S1, V1, d, fro2, off, st, "sigma1", sweeps);
  if (rc) return rc;
  rc = jacobi(S2, V2, d, fro2, off, st, "sigma2", sweeps ? sweeps + 1 : nullptr);
  if (rc) return rc;
  scale_rows_kernel<<<d, 256, 0, st>>>(S1, V1, d);
  scale_rows_kernel<<<d, 256, 0, st>>>(S2, V2, d);
  gemm_nt_kernel<<<dim3(d / 64, d / 64), 256, 0, st>>>(V1, V2, S1, d);  // G = L1^T L2 into S1
  PF_CHECK_LAUNCH("frechet factors");
  rc = jacobi(S1, nullptr, d, fro2, off, st, "L1^T L2", sweeps ? sweeps + 2 : nullptr);
  if (rc) return rc;
  finish_kernel<<<1, 256, 0, st>>>(S1, d, scal, out);
  PF_CHECK_LAUNCH("finish_kernel");
  return PF_OK;
}
