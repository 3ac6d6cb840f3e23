// Implicit-GEMM convolution on mma.sync m16n8k16 (fp16 in, fp32 accumulate), shared by FAED's circular-padded encoder
// (faed.cu, pf_conv_circ) and the FID InceptionV3 (inception.cu, pf_conv2d_nhwc).
//
// GEMM view: M = B*Ho*Wo output pixels, N = Cout, K = kh*kw taps x Cin. A k-step is one tap x KC input channels
// (KC = 64, 32 or 16, whichever divides Cin), so narrow layers are not zero-padded to 64.
// CTA: 128 pixels x BN output channels (column tile blockIdx.y), 8 warps as 4 (M, 32 rows) x 2 (N, BN/2 columns);
// 3-stage cp.async ring; the A rows are gathered per pixel (16-byte pieces, zero-filled for taps outside the image) and
// the B rows are the packed weight [tap][Cin][Cw] (Cw = Cout padded to the N tile with zero columns). Shared rows are
// padded by 16 bytes so the ldmatrix phases hit distinct banks.
// Padding is addressing, no padded copy: input row iy = oy*s + ky - ph is zero outside [0, H); input column
// ix = ox*s + kx - pw is zero outside [0, W), or taken modulo W when CIRC (FAED's CircularPadding: corners zero). CIRC is
// a template parameter so that neither kind of layer pays for the other's address test in the load loop.
// The epilogue adds the bias (BN folded), applies ReLU, adds an optional fp16 residual [M][Cout] and stores fp16 or fp32
// at out[m * out_ld + out_off + col] for col < Cout, so a branch writes straight into its slice of a concat buffer.
// Two more template parameters serve HorizonNet's ResNet-50 (horizonnet.cu) without costing the other layers anything:
// RES_BEFORE_RELU adds the residual before the ReLU (torchvision's Bottleneck, relu(bn3(conv3) + identity)), and
// STRIDE_HW takes the column stride from stride_w instead of stride (ConvCompressH's stride (2, 1)).
#pragma once
#include "pf_common.cuh"

namespace pf {
namespace convmma {
// Internal linkage: each .cu that includes this header gets its own kernel instances and launch state, so no kernel
// template is registered by two translation units (the library is built without relocatable device code).
namespace {

constexpr int kBM = 128;  // output pixels per CTA
constexpr int kThreads = 256;
constexpr int kStages = 3;

struct ConvArgs {
  const __half* x;
  const __half* w;
  const float* bias;
  const __half* residual;
  void* out;
  int B, H, W, Cin, Cout, Ho, Wo, kh, kw, stride, ph, pw, relu, out_f32;
  int Cw;              // packed weight / bias width (Cout rounded up to the N tile)
  int out_ld, out_off;  // output row stride and channel offset, in elements
  int M;
  int stride_w;  // column stride, read only by STRIDE_HW instances
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int KC, int BN>
struct ConvTile {
  static constexpr int A_LD = KC + 8, B_LD = BN + 8;  // halves
  static constexpr int A_HALVES = kBM * A_LD, B_HALVES = KC * B_LD;
  static constexpr int STAGE_HALVES = A_HALVES + B_HALVES;
  static constexpr int SMEM = kStages * STAGE_HALVES * 2;
  static constexpr int CPR = KC / 8;                    // 16-byte pieces per A row
  static constexpr int A_ITERS = kBM * CPR / kThreads;  // pieces per thread
  static constexpr int NT = BN / 16;                    // n8 tiles per warp
};

template <int KC, int BN, bool CIRC, bool RES_BEFORE_RELU = false, bool STRIDE_HW = false>
__global__ void __launch_bounds__(kThreads)
conv_mma_kernel(ConvArgs a) {
  using T = ConvTile<KC, BN>;
  static_assert(T::A_ITERS >= 1 && T::NT % 2 == 0, "tile");
  constexpr int A_IT = T::A_ITERS;
  extern __shared__ __align__(16) __half smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp & 3, wn = warp >> 2;
  const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * BN;
  const int HoWo = a.Ho * a.Wo;

  // per-thread A pieces: the pixel's image offset and its top-left input coordinate
  int a_base[A_IT], a_y[A_IT], a_x[A_IT], a_dst[A_IT];
#pragma unroll
  for (int i = 0; i < A_IT; ++i) {
    const int idx = tid + i * kThreads, row = idx / T::CPR, ch = idx % T::CPR;
    const int m = m0 + row;
    a_dst[i] = row * T::A_LD + ch * 8;
    if (m < a.M) {
      const int b = m / HoWo, r = m % HoWo;
      a_base[i] = b * a.H;
      a_y[i] = (r / a.Wo) * a.stride - a.ph;
      a_x[i] = (r % a.Wo) * (STRIDE_HW ? a.stride_w : a.stride) - a.pw;
    } else {
      a_base[i] = 0;
      a_y[i] = -(1 << 20);  // never inside the image: zero-filled
      a_x[i] = 0;
    }
  }
  const int chunks = a.Cin / KC;
  const int steps = a.kh * a.kw * chunks;

  auto load = [&](int s, int buf) {
    __half* As = smem + buf * T::STAGE_HALVES;
    __half* Bs = As + T::A_HALVES;
    const int tap = s / chunks, c0 = (s % chunks) * KC;
    const int ky = tap / a.kw, kx = tap % a.kw;
#pragma unroll
    for (int i = 0; i < A_IT; ++i) {
      const int ch = (tid + i * kThreads) % T::CPR;
      const int iy = a_y[i] + ky;
      int ix = a_x[i] + kx;
      bool valid = iy >= 0 && iy < a.H;
      if constexpr (CIRC)
        ix = ix < 0 ? ix + a.W : (ix >= a.W ? ix - a.W : ix);
      else
        valid = valid && ix >= 0 && ix < a.W;
      const __half* src = valid ? a.x + ((size_t)(a_base[i] + iy) * a.W + ix) * a.Cin + c0 + ch * 8 : a.x;
      cp_async16(smem_u32(As + a_dst[i]), src, valid);
    }
    const __half* wsrc = a.w + ((size_t)tap * a.Cin + c0) * a.Cw + n0;
    for (int idx = tid; idx < KC * BN / 8; idx += kThreads) {
      const int r = idx / (BN / 8), c = idx % (BN / 8);
      cp_async16(smem_u32(Bs + r * T::B_LD + c * 8), wsrc + (size_t)r * a.Cw + c * 8, true);
    }
  };

  float acc[2][T::NT][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < T::NT; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

#pragma unroll
  for (int s = 0; s < kStages - 1; ++s) {
    if (s < steps) load(s, s);
    cp_async_commit();
  }
  for (int s = 0; s < steps; ++s) {
    cp_async_wait<kStages - 2>();
    __syncthreads();  // stage s landed for every thread; stage s-1's buffer is free
    if (s + kStages - 1 < steps) load(s + kStages - 1, (s + kStages - 1) % kStages);
    cp_async_commit();
    const __half* As = smem + (s % kStages) * T::STAGE_HALVES;
    const __half* Bs = As + T::A_HALVES;
#pragma unroll
    for (int kk = 0; kk < KC; kk += 16) {
      uint32_t af[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int row = wm * 32 + mt * 16 + (lane & 15), col = kk + (lane >> 4) * 8;
        ldsm_x4(smem_u32(As + row * T::A_LD + col), af[mt][0], af[mt][1], af[mt][2], af[mt][3]);
      }
#pragma unroll
      for (int np = 0; np < T::NT / 2; ++np) {
        uint32_t b0, b1, b2, b3;
        const int krow = kk + (lane & 15), col = wn * (BN / 2) + np * 16 + (lane >> 4) * 8;
        ldsm_x4_t(smem_u32(Bs + krow * T::B_LD + col), b0, b1, b2, b3);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma16816(acc[mt][2 * np], af[mt], b0, b1);
          mma16816(acc[mt][2 * np + 1], af[mt], b2, b3);
        }
      }
    }
  }
  cp_async_wait<0>();

  // epilogue: + bias (BN folded), ReLU, + residual, 16-bit or fp32 store of the columns < Cout
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < T::NT; ++nt) {
      const int col = n0 + wn * (BN / 2) + nt * 8 + (lane & 3) * 2;
      if (col >= a.Cout) continue;  // Cout is even, so col + 1 < Cout too
      const float bias0 = a.bias[col], bias1 = a.bias[col + 1];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + wm * 32 + mt * 16 + (lane >> 2) + h * 8;
        if (m >= a.M) continue;
        float v0 = acc[mt][nt][2 * h] + bias0, v1 = acc[mt][nt][2 * h + 1] + bias1;
        if (RES_BEFORE_RELU && a.residual) {
          const float2 r = __half22float2(*reinterpret_cast<const __half2*>(a.residual + (size_t)m * a.Cout + col));
          v0 += r.x;
          v1 += r.y;
        }
        if (a.relu) {
          v0 = fmaxf(v0, 0.f);
          v1 = fmaxf(v1, 0.f);
        }
        if (!RES_BEFORE_RELU && a.residual) {
          const float2 r = __half22float2(*reinterpret_cast<const __half2*>(a.residual + (size_t)m * a.Cout + col));
          v0 += r.x;
          v1 += r.y;
        }
        const size_t o = (size_t)m * a.out_ld + a.out_off + col;
        if (a.out_f32)
          *reinterpret_cast<float2*>(static_cast<float*>(a.out) + o) = make_float2(v0, v1);
        else
          *reinterpret_cast<__half2*>(static_cast<__half*>(a.out) + o) = __floats2half2_rn(v0, v1);
      }
    }
}

template <int KC, int BN, bool CIRC, bool RES_BEFORE_RELU = false, bool STRIDE_HW = false>
int launch_conv(const ConvArgs& a, cudaStream_t st) {
  using T = ConvTile<KC, BN>;
  static bool attr_set = false;  // per-kernel opt-in to > 48 KB of dynamic shared memory
  if (!attr_set) {
    const int rc = check_cuda(
        cudaFuncSetAttribute(conv_mma_kernel<KC, BN, CIRC, RES_BEFORE_RELU, STRIDE_HW>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, T::SMEM),
        "cudaFuncSetAttribute(conv_mma_kernel)");
    if (rc) return rc;
    attr_set = true;
  }
  const dim3 grid((unsigned)((a.M + kBM - 1) / kBM), (unsigned)(a.Cw / BN));
  conv_mma_kernel<KC, BN, CIRC, RES_BEFORE_RELU, STRIDE_HW><<<grid, kThreads, T::SMEM, st>>>(a);
  PF_CHECK_LAUNCH("conv_mma_kernel");
  return PF_OK;
}

}  // namespace
}  // namespace convmma
}  // namespace pf
