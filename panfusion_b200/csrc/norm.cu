// Normalisation + convolution-input preparation kernels (HBM-bound, channels-last, 16-byte vector accesses).
//
//  * pf_groupnorm_stats : GroupNorm statistics of a channels-last image, optionally over the circularly padded
//    image (the reference normalises the W+2*circ wide tensor: models/pano/MVGenModel.py:110-115 wraps every
//    panorama ResnetBlock2D in pad_pano(2)/unpad_pano(2), so columns {0,1,W-2,W-1} count twice). It is the
//    statistics launch of pf_gn_prep with its own partition of the image.
//  * pf_conv_prep       : GroupNorm-apply (+SiLU) fused with building the tap-GEMM's A operand: circular column
//    extension (utils/pano.py:74-105), nearest x2 upsampling (Upsample2D), zero halo, or the four stride-2
//    phase images (Downsample2D). Replaces norm1/norm2 + nonlinearity of ResnetBlock2D, Transformer2DModel.norm,
//    and ~60 pad_pano / unpad_pano copies per step.
//  * pf_gn_prep         : pf_groupnorm_stats + pf_conv_prep as two launches of one kernel (statistics, then apply),
//    optionally over the skip concatenation of two tensors.
//  * pf_layernorm       : LayerNorm(x + pe) per token (models/modules/transformer.py:157-160, diffusers
//    BasicTransformerBlock norm1/2/3).
#include "pf_common.cuh"

namespace pf {

// ------------------------------------------------------------------------------------------------
// conv_prep: thread <-> (output position, 8-channel vector)
// ------------------------------------------------------------------------------------------------
struct PrepParams {
  const uint16_t* x;
  uint16_t* out;
  const float* mean_rstd;  // [N, groups, 2] or null (no normalisation)
  const float* gamma;
  const float* beta;
  int N, H, W, C, ld, groups, act, circ, up, phases, halo;
  int Ho, Wo;           // output positions per image (incl. halo / phase padding)
  long long total_vecs;  // N * phases * Ho * Wo * C/8
};

// grid = (ceil(Wo * C/8 / 256), N * phases * Ho): one output row per blockIdx.y, so the per-channel scale/shift of the
// row's image is built once per CTA in shared memory and the inner loop is load -> 8 FMA (+SiLU) -> store.
template <bool BF16>
__global__ void __launch_bounds__(256) conv_prep_kernel(const PrepParams p) {
  extern __shared__ float s_ss[];  // [2][C] scale, shift
  const int vecs = p.C / 8;
  int rowid = blockIdx.y;
  const int i = rowid % p.Ho;
  rowid /= p.Ho;
  const int n = rowid % p.N;
  const int ph = rowid / p.N;
  if (p.mean_rstd) {
    const int cpg = p.C / p.groups;
    for (int c = threadIdx.x; c < p.C; c += blockDim.x) {
      const int g = c / cpg;
      const float mean = __ldg(p.mean_rstd + ((size_t)n * p.groups + g) * 2);
      const float rstd = __ldg(p.mean_rstd + ((size_t)n * p.groups + g) * 2 + 1);
      const float sc = rstd * __ldg(p.gamma + c);
      s_ss[c] = sc;
      s_ss[p.C + c] = __ldg(p.beta + c) - mean * sc;
    }
    __syncthreads();
  }
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= p.Wo * vecs) return;
  const int j = idx / vecs, v = idx - j * vecs;
  const int We = p.W + 2 * p.circ;
  const int Hu = p.H * p.up, Wu = We * p.up;
  int yy, xx;
  if (p.phases == 4) {
    yy = 2 * i + (ph >> 1) - 1;
    xx = 2 * j + (ph & 1) - 1;
  } else {
    yy = i - p.halo;
    xx = j - p.halo;
  }
  uint4 outv = make_uint4(0, 0, 0, 0);
  if (yy >= 0 && yy < Hu && xx >= 0 && xx < Wu) {
    const int sy = yy / p.up;
    int sx = xx / p.up - p.circ;
    if (sx < 0) sx += p.W;
    else if (sx >= p.W) sx -= p.W;
    const uint4 raw = __ldg(reinterpret_cast<const uint4*>(p.x + ((size_t)n * p.H * p.W + (size_t)sy * p.W + sx) * p.ld + v * 8));
    if (p.mean_rstd || p.act) {
      const uint32_t w4[4] = {raw.x, raw.y, raw.z, raw.w};
      float f[8];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 t = unpack2<BF16>(w4[e]);
        f[2 * e] = t.x;
        f[2 * e + 1] = t.y;
      }
      if (p.mean_rstd) {
        const float4 s0 = *reinterpret_cast<const float4*>(s_ss + v * 8), s1 = *reinterpret_cast<const float4*>(s_ss + v * 8 + 4);
        const float4 h0 = *reinterpret_cast<const float4*>(s_ss + p.C + v * 8), h1 = *reinterpret_cast<const float4*>(s_ss + p.C + v * 8 + 4);
        f[0] = fmaf(f[0], s0.x, h0.x); f[1] = fmaf(f[1], s0.y, h0.y); f[2] = fmaf(f[2], s0.z, h0.z); f[3] = fmaf(f[3], s0.w, h0.w);
        f[4] = fmaf(f[4], s1.x, h1.x); f[5] = fmaf(f[5], s1.y, h1.y); f[6] = fmaf(f[6], s1.z, h1.z); f[7] = fmaf(f[7], s1.w, h1.w);
      }
      if (p.act == PF_ACT_SILU) {
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = silu_f(f[e]);
      }
      outv = make_uint4(pack2<BF16>(f[0], f[1]), pack2<BF16>(f[2], f[3]), pack2<BF16>(f[4], f[5]),
                        pack2<BF16>(f[6], f[7]));
    } else {
      outv = raw;
    }
  }
  *reinterpret_cast<uint4*>(p.out + ((size_t)blockIdx.y * p.Wo + j) * p.C + v * 8) = outv;
}

// ------------------------------------------------------------------------------------------------
// gn_prep: GroupNorm statistics, then GroupNorm-apply (+SiLU) + conv_prep layout (pf_gn_prep); the statistics launch
// alone is pf_groupnorm_stats.
//
// STATS launch, grid (slabs, N): CTA (s, n) sums slab s of image n per channel — the slabs are a fixed partition of the
// image into pixel ranges that depends on the image size ONLY — and publishes per-group partials (two sources = the skip
// concatenation torch.cat([hidden, skip], 1), optionally also written out raw). The LAST CTA of the image to arrive
// reduces the partials in slab order into mean / rstd and re-arms counters[n]. No floating-point sum depends on the batch
// size, so the result is the same, bit for bit, for any N (a view-sharded rank reproduces the single-GPU run).
// APPLY launch, grid (ctas, N): CTA (c, n) produces its share of image n's output positions; the source pixels are
// re-read from L2, not HBM.
// ------------------------------------------------------------------------------------------------
constexpr int GN_MAX_SLABS = 64;   // upper bound of the statistics partition of one image (sizes the workspace)
constexpr int GN_PREP_SLABS = 32;  // pf_gn_prep: at most 32 slabs per image
constexpr int GN_APPLY_CTAS = 64;  // pf_gn_prep: at most 64 apply CTAs per image

struct GnPrepParams {
  const uint16_t* x1;
  const uint16_t* x2;   // second source of a channel concatenation, or null
  uint16_t* cat_out;    // raw concatenation [N*H*W, C] or null
  uint16_t* out;
  const float* gamma;
  const float* beta;
  float* ws;            // [N][slabs][groups][2] partials
  float* mean_rstd;     // [N][groups][2]
  int* counters;        // [N], zero on entry and on exit of the statistics launch
  int slabs;            // statistics partition of an image: a function of H*W only
  int N, H, W, C1, C2, ld1, ld2, groups, act, circ_stats, circ, up, phases, halo;
  int Ho, Wo;
  float count, eps;
};

template <bool BF16, bool STATS>
__global__ void __launch_bounds__(512, 2) gn_prep_kernel(const GnPrepParams p) {
  extern __shared__ float s_acc[];  // statistics: [ppi][2][C] partials; apply: [2][C] scale / shift
  const int C = p.C1 + p.C2;
  const int vecs = C / 8, vecs1 = p.C1 / 8;
  const int ppi = blockDim.x / vecs;  // blockDim.x is a multiple of vecs
  const int v = threadIdx.x % vecs, pl = threadIdx.x / vecs;
  const int n = blockIdx.y;
  const int hw = p.H * p.W;
  const bool second = v >= vecs1;
  const int ld = second ? p.ld2 : p.ld1;
  const uint16_t* src = second ? p.x2 + (size_t)n * hw * p.ld2 + (v - vecs1) * 8 : p.x1 + (size_t)n * hw * p.ld1 + v * 8;
  const int cpg = C / p.groups;
  float* mr = p.mean_rstd + (size_t)n * p.groups * 2;
  if constexpr (STATS) {
    const int sl = blockIdx.x;
    const int per = (hw + p.slabs - 1) / p.slabs;
    const int p_begin = sl * per, p_end = min(hw, p_begin + per);
    float s[8], q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
    auto accum = [&](const uint4& raw, int px) {
      float wgt = 1.f;
      if (p.circ_stats > 0) {
        const int col = px % p.W;
        wgt += (col < p.circ_stats ? 1.f : 0.f) + (col >= p.W - p.circ_stats ? 1.f : 0.f);
      }
      const uint32_t w4[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack2<BF16>(w4[e]);
        s[2 * e] += wgt * f.x;
        q[2 * e] += wgt * f.x * f.x;
        s[2 * e + 1] += wgt * f.y;
        q[2 * e + 1] += wgt * f.y * f.y;
      }
      if (p.cat_out) *reinterpret_cast<uint4*>(p.cat_out + ((size_t)n * hw + px) * C + v * 8) = raw;
    };
    int px = p_begin + pl;
    // four independent 16-byte loads in flight per thread
    for (; px + 3 * ppi < p_end; px += 4 * ppi) {
      const uint4 r0 = __ldg(reinterpret_cast<const uint4*>(src + (size_t)px * ld));
      const uint4 r1 = __ldg(reinterpret_cast<const uint4*>(src + (size_t)(px + ppi) * ld));
      const uint4 r2 = __ldg(reinterpret_cast<const uint4*>(src + (size_t)(px + 2 * ppi) * ld));
      const uint4 r3 = __ldg(reinterpret_cast<const uint4*>(src + (size_t)(px + 3 * ppi) * ld));
      accum(r0, px);
      accum(r1, px + ppi);
      accum(r2, px + 2 * ppi);
      accum(r3, px + 3 * ppi);
    }
    for (; px < p_end; px += ppi) accum(__ldg(reinterpret_cast<const uint4*>(src + (size_t)px * ld)), px);
    float* mine = s_acc + (size_t)pl * 2 * C;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      mine[v * 8 + e] = s[e];
      mine[C + v * 8 + e] = q[e];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
      float a = s_acc[i];
      for (int l = 1; l < ppi; ++l) a += s_acc[(size_t)l * 2 * C + i];
      s_acc[i] = a;
    }
    __syncthreads();
    for (int g = threadIdx.x; g < p.groups; g += blockDim.x) {
      float a = 0.f, b = 0.f;
      for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
        a += s_acc[c];
        b += s_acc[C + c];
      }
      float* o = p.ws + (((size_t)n * p.slabs + sl) * p.groups + g) * 2;
      o[0] = a;
      o[1] = b;
    }
    __shared__ int s_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(&p.counters[n], 1) == p.slabs - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    for (int g = threadIdx.x; g < p.groups; g += blockDim.x) {
      double a = 0.0, b = 0.0;
      for (int c = 0; c < p.slabs; ++c) {
        const float* o = p.ws + (((size_t)n * p.slabs + c) * p.groups + g) * 2;
        a += __ldcg(o);
        b += __ldcg(o + 1);
      }
      const double mean = a / p.count;
      double var = b / p.count - mean * mean;
      if (var < 0.0) var = 0.0;
      mr[g * 2 + 0] = float(mean);
      mr[g * 2 + 1] = float(1.0 / sqrt(var + double(p.eps)));
    }
    if (threadIdx.x == 0) p.counters[n] = 0;  // the next launch is ordered behind this one by the stream
  } else {
    // scale / shift of this image into shared memory
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const int g = c / cpg;
      const float mean = __ldcg(mr + g * 2), rstd = __ldcg(mr + g * 2 + 1);
      const float sc = rstd * __ldg(p.gamma + c);
      s_acc[c] = sc;
      s_acc[C + c] = __ldg(p.beta + c) - mean * sc;
    }
    __syncthreads();
    const int We = p.W + 2 * p.circ;
    const int Hu = p.H * p.up, Wu = We * p.up;
    const int total = p.phases * p.Ho * p.Wo;
    const int ctas = gridDim.x;
    const int per_o = (total + ctas - 1) / ctas;
    const int o_begin = blockIdx.x * per_o, o_end = min(total, o_begin + per_o);
    const float4 s0 = *reinterpret_cast<const float4*>(s_acc + v * 8), s1 = *reinterpret_cast<const float4*>(s_acc + v * 8 + 4);
    const float4 h0 = *reinterpret_cast<const float4*>(s_acc + C + v * 8), h1 = *reinterpret_cast<const float4*>(s_acc + C + v * 8 + 4);
    const size_t img_out = (size_t)p.Ho * p.Wo;
    const int hw_o = p.Ho * p.Wo;
    // (output position) -> (source pixel offset or -1 for the zero halo, output vector pointer)
    auto locate = [&](int o, long long& soff, uint4*& dst) {
      const int ph = o / hw_o;
      const int r = o - ph * hw_o;
      const int i = r / p.Wo, j = r - i * p.Wo;
      int yy, xx;
      if (p.phases == 4) {
        yy = 2 * i + (ph >> 1) - 1;
        xx = 2 * j + (ph & 1) - 1;
      } else {
        yy = i - p.halo;
        xx = j - p.halo;
      }
      soff = -1;
      if (yy >= 0 && yy < Hu && xx >= 0 && xx < Wu) {
        const int sy = yy / p.up;
        int sx = xx / p.up - p.circ;
        if (sx < 0) sx += p.W;
        else if (sx >= p.W) sx -= p.W;
        soff = ((long long)sy * p.W + sx) * ld;
      }
      dst = reinterpret_cast<uint4*>(p.out + (((size_t)ph * p.N + n) * img_out + r) * C + v * 8);  // [phases][N][Ho][Wo][C]
    };
    auto finish = [&](const uint4& raw, bool live, uint4* dst) {
      uint4 outv = make_uint4(0, 0, 0, 0);
      if (live) {
        const uint32_t w4[4] = {raw.x, raw.y, raw.z, raw.w};
        float f[8];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 t = unpack2<BF16>(w4[e]);
          f[2 * e] = t.x;
          f[2 * e + 1] = t.y;
        }
        f[0] = fmaf(f[0], s0.x, h0.x); f[1] = fmaf(f[1], s0.y, h0.y); f[2] = fmaf(f[2], s0.z, h0.z); f[3] = fmaf(f[3], s0.w, h0.w);
        f[4] = fmaf(f[4], s1.x, h1.x); f[5] = fmaf(f[5], s1.y, h1.y); f[6] = fmaf(f[6], s1.z, h1.z); f[7] = fmaf(f[7], s1.w, h1.w);
        if (p.act == PF_ACT_SILU) {
#pragma unroll
          for (int e = 0; e < 8; ++e) f[e] = silu_f(f[e]);
        }
        outv = make_uint4(pack2<BF16>(f[0], f[1]), pack2<BF16>(f[2], f[3]), pack2<BF16>(f[4], f[5]), pack2<BF16>(f[6], f[7]));
      }
      *dst = outv;
    };
    const uint4 z4 = make_uint4(0, 0, 0, 0);
    int o = o_begin + pl;
    for (; o + 3 * ppi < o_end; o += 4 * ppi) {  // four independent L2 loads in flight per thread
      long long so[4];
      uint4* dst[4];
      uint4 raw[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) locate(o + u * ppi, so[u], dst[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u) raw[u] = so[u] >= 0 ? __ldcg(reinterpret_cast<const uint4*>(src + so[u])) : z4;
#pragma unroll
      for (int u = 0; u < 4; ++u) finish(raw[u], so[u] >= 0, dst[u]);
    }
    for (; o < o_end; o += ppi) {
      long long so;
      uint4* dst;
      locate(o, so, dst);
      const uint4 raw = so >= 0 ? __ldcg(reinterpret_cast<const uint4*>(src + so)) : z4;
      finish(raw, so >= 0, dst);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm(x + pe): one warp per token, two-pass in registers
// ------------------------------------------------------------------------------------------------
template <bool BF16, int MAXV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const uint16_t* __restrict__ x, int ldx, const float* __restrict__ pe, int pe_rows, int T, int C,
                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                 uint16_t* __restrict__ out, int ldo) {
  const int lane = threadIdx.x & 31;
  const int warps_total = (gridDim.x * blockDim.x) >> 5;
  const int vecs = C / 8;
  // affine parameters staged once per CTA in shared memory (each warp then visits many tokens)
  extern __shared__ float s_gb[];  // [2][C]
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    s_gb[c] = __ldg(gamma + c);
    s_gb[C + c] = __ldg(beta + c);
  }
  __syncthreads();
  for (int tok = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; tok < T; tok += warps_total) {
    float f[MAXV][8];
    float sum = 0.f;
    const uint16_t* xr = x + (size_t)tok * ldx;
    const float* per = pe ? pe + (size_t)(tok % pe_rows) * C : nullptr;
#pragma unroll
    for (int r = 0; r < MAXV; ++r) {
      const int v = lane + r * 32;
      if (v < vecs) {
        const uint4 raw = __ldg(reinterpret_cast<const uint4*>(xr + v * 8));
        const uint32_t w4[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 t = unpack2<BF16>(w4[e]);
          f[r][2 * e] = t.x;
          f[r][2 * e + 1] = t.y;
        }
        if (per) {
          const float4 a = __ldg(reinterpret_cast<const float4*>(per + v * 8));
          const float4 b = __ldg(reinterpret_cast<const float4*>(per + v * 8 + 4));
          f[r][0] += a.x; f[r][1] += a.y; f[r][2] += a.z; f[r][3] += a.w;
          f[r][4] += b.x; f[r][5] += b.y; f[r][6] += b.z; f[r][7] += b.w;
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) sum += f[r][e];
      }
    }
    const float mean = warp_sum(sum) / float(C);
    float sq = 0.f;
#pragma unroll
    for (int r = 0; r < MAXV; ++r) {
      const int v = lane + r * 32;
      if (v < vecs) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float d = f[r][e] - mean;
          sq += d * d;
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(sq) / float(C) + eps);
    uint16_t* orow = out + (size_t)tok * ldo;
#pragma unroll
    for (int r = 0; r < MAXV; ++r) {
      const int v = lane + r * 32;
      if (v < vecs) {
        const float4 ga = *reinterpret_cast<const float4*>(s_gb + v * 8), gb = *reinterpret_cast<const float4*>(s_gb + v * 8 + 4);
        const float4 ba = *reinterpret_cast<const float4*>(s_gb + C + v * 8), bb4 = *reinterpret_cast<const float4*>(s_gb + C + v * 8 + 4);
        const float gg[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
        const float bb[8] = {ba.x, ba.y, ba.z, ba.w, bb4.x, bb4.y, bb4.z, bb4.w};
        float o[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = (f[r][e] - mean) * rstd * gg[e] + bb[e];
        *reinterpret_cast<uint4*>(orow + v * 8) = make_uint4(pack2<BF16>(o[0], o[1]), pack2<BF16>(o[2], o[3]),
                                                             pack2<BF16>(o[4], o[5]), pack2<BF16>(o[6], o[7]));
      }
    }
  }
}

}  // namespace pf

extern "C" int pf_groupnorm_ws_floats(int N, int groups) { return N * pf::GN_MAX_SLABS * groups * 2; }

extern "C" int pf_groupnorm_stats(const void* x, int dtype, int N, int H, int W, int C, int ld, int groups, int circ,
                                  float eps, float* ws, int* counters, float* mean_rstd, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(x && ws && counters && mean_rstd, "pf_groupnorm_stats: null pointer");
  PF_CHECK_ARG(dtype == PF_BF16 || dtype == PF_F16, "pf_groupnorm_stats: 16-bit dtype required");
  PF_CHECK_ARG(N > 0 && H > 0 && W > 0 && C > 0 && groups > 0 && C % groups == 0 && C % 8 == 0 && ld % 8 == 0 &&
                   ld >= C && C / 8 <= 512,
               "pf_groupnorm_stats: bad shape N=%d H=%d W=%d C=%d ld=%d groups=%d", N, H, W, C, ld, groups);
  PF_CHECK_ARG(circ >= 0 && circ <= W, "pf_groupnorm_stats: circ=%d out of range", circ);
  GnPrepParams p = {};
  p.x1 = static_cast<const uint16_t*>(x);
  p.ws = ws; p.mean_rstd = mean_rstd; p.counters = counters;
  p.N = N; p.H = H; p.W = W; p.C1 = C; p.ld1 = ld; p.ld2 = ld; p.groups = groups; p.circ_stats = circ;
  p.count = float(H) * float(W + 2 * circ) * float(C / groups);
  p.eps = eps;
  const int slabs = H * W / 16;  // >= 16 pixels per CTA; small images still spread over several SMs
  p.slabs = slabs < 1 ? 1 : (slabs > GN_MAX_SLABS ? GN_MAX_SLABS : slabs);
  const int vecs = C / 8;
  int ppi = 256 / vecs;
  if (ppi < 1) ppi = 1;
  const size_t smem = 2 * (size_t)C * ppi * sizeof(float);
  const dim3 grid(p.slabs, N);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PF_BF16) gn_prep_kernel<true, true><<<grid, vecs * ppi, smem, st>>>(p);
  else gn_prep_kernel<false, true><<<grid, vecs * ppi, smem, st>>>(p);
  PF_CHECK_LAUNCH("gn_prep_kernel(stats)");
  return PF_OK;
}

extern "C" int pf_conv_prep(const void* x, void* out, int dtype, int N, int H, int W, int C, int ld,
                            const float* mean_rstd, const float* gamma, const float* beta, int groups, int act,
                            int circ, int up, int phases, int halo, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(x && out, "pf_conv_prep: null pointer");
  PF_CHECK_ARG(dtype == PF_BF16 || dtype == PF_F16, "pf_conv_prep: 16-bit dtype required");
  PF_CHECK_ARG(N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && ld % 8 == 0 && ld >= C, "pf_conv_prep: bad shape");
  PF_CHECK_ARG(!mean_rstd || (gamma && beta && groups > 0 && C % groups == 0), "pf_conv_prep: GroupNorm needs gamma/beta/groups");
  PF_CHECK_ARG(act == PF_ACT_NONE || act == PF_ACT_SILU, "pf_conv_prep: act must be none or silu");
  PF_CHECK_ARG((up == 1 || up == 2) && (phases == 1 || phases == 4) && (halo == 0 || halo == 1) && circ >= 0 && circ <= W,
               "pf_conv_prep: bad geometry up=%d phases=%d halo=%d circ=%d", up, phases, halo, circ);
  PF_CHECK_ARG(!(phases == 4 && (up != 1 || halo != 1 || (H % 2) || ((W + 2 * circ) % 2))),
               "pf_conv_prep: stride-2 phase split needs up=1, halo=1 and even extents");
  PrepParams p;
  p.x = static_cast<const uint16_t*>(x);
  p.out = static_cast<uint16_t*>(out);
  p.mean_rstd = mean_rstd; p.gamma = gamma; p.beta = beta;
  p.N = N; p.H = H; p.W = W; p.C = C; p.ld = ld; p.groups = groups > 0 ? groups : 1; p.act = act;
  p.circ = circ; p.up = up; p.phases = phases; p.halo = halo;
  const int Hu = H * up, Wu = (W + 2 * circ) * up;
  if (phases == 4) {
    p.Ho = Hu / 2 + 1;
    p.Wo = Wu / 2 + 1;
  } else {
    p.Ho = Hu + 2 * halo;
    p.Wo = Wu + 2 * halo;
  }
  p.total_vecs = (long long)N * phases * p.Ho * p.Wo * (C / 8);
  const long long rows = (long long)N * phases * p.Ho;
  PF_CHECK_ARG(rows <= 2147483647LL / 1 && rows > 0, "pf_conv_prep: tensor too large");
  const size_t smem = mean_rstd ? 2 * (size_t)C * sizeof(float) : 0;
  PF_CHECK_ARG(smem <= 48 * 1024, "pf_conv_prep: C=%d too large", C);
  dim3 grid((unsigned)((p.Wo * (C / 8) + 255) / 256), (unsigned)rows);
  PF_CHECK_ARG(rows <= 65535LL * 32768LL, "pf_conv_prep: too many rows");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (rows > 65535) {
    // gridDim.y limit: fold rows into x is not needed for UNet shapes (N*(H+2) <= 65535); refuse loudly otherwise
    set_error("pf_conv_prep: N*phases*Ho = %lld exceeds 65535", rows);
    return PF_ERR_UNSUPPORTED;
  }
  if (dtype == PF_BF16) conv_prep_kernel<true><<<grid, 256, smem, st>>>(p);
  else conv_prep_kernel<false><<<grid, 256, smem, st>>>(p);
  PF_CHECK_LAUNCH("conv_prep_kernel");
  return PF_OK;
}

extern "C" int pf_gn_prep_ws_floats(int N, int groups) {
  return N * pf::GN_MAX_SLABS * groups * 2 + N * groups * 2;
}

extern "C" int pf_gn_prep(const void* x1, int ld1, int C1, const void* x2, int ld2, int C2, void* cat_out, void* out,
                          int dtype, int N, int H, int W, int groups, float eps, const float* gamma, const float* beta,
                          int act, int circ_stats, int circ, int up, int phases, int halo, float* ws, int* counters,
                          void* stream) {
  using namespace pf;
  PF_CHECK_ARG(x1 && out && gamma && beta && ws && counters, "pf_gn_prep: null pointer");
  PF_CHECK_ARG(dtype == PF_BF16 || dtype == PF_F16, "pf_gn_prep: 16-bit dtype required");
  if (!x2) C2 = 0;
  const int C = C1 + C2;
  PF_CHECK_ARG(N > 0 && H > 0 && W > 0 && C1 > 0 && C1 % 8 == 0 && C2 % 8 == 0 && ld1 % 8 == 0 &&
                   ld1 >= C1 && (!x2 || (ld2 % 8 == 0 && ld2 >= C2 && C2 > 0)) && groups > 0 && C % groups == 0 &&
                   C / 8 <= 512,
               "pf_gn_prep: bad shape N=%d H=%d W=%d C1=%d C2=%d groups=%d", N, H, W, C1, C2, groups);
  PF_CHECK_ARG(!cat_out || x2, "pf_gn_prep: cat_out needs a second source");
  PF_CHECK_ARG(act == PF_ACT_NONE || act == PF_ACT_SILU, "pf_gn_prep: act must be none or silu");
  PF_CHECK_ARG((up == 1 || up == 2) && (phases == 1 || phases == 4) && (halo == 0 || halo == 1) && circ >= 0 && circ <= W &&
                   circ_stats >= 0 && circ_stats <= W,
               "pf_gn_prep: bad geometry up=%d phases=%d halo=%d circ=%d", up, phases, halo, circ);
  PF_CHECK_ARG(!(phases == 4 && (up != 1 || halo != 1 || (H % 2) || ((W + 2 * circ) % 2))),
               "pf_gn_prep: stride-2 phase split needs up=1, halo=1 and even extents");
  GnPrepParams p;
  p.x1 = static_cast<const uint16_t*>(x1);
  p.x2 = static_cast<const uint16_t*>(x2);
  p.cat_out = static_cast<uint16_t*>(cat_out);
  p.out = static_cast<uint16_t*>(out);
  p.gamma = gamma; p.beta = beta;
  p.ws = ws;
  p.mean_rstd = ws + (size_t)N * GN_MAX_SLABS * groups * 2;
  p.counters = counters;
  p.N = N; p.H = H; p.W = W; p.C1 = C1; p.C2 = C2; p.ld1 = ld1; p.ld2 = x2 ? ld2 : ld1; p.groups = groups; p.act = act;
  p.circ_stats = circ_stats; p.circ = circ; p.up = up; p.phases = phases; p.halo = halo;
  const int Hu = H * up, Wu = (W + 2 * circ) * up;
  if (phases == 4) {
    p.Ho = Hu / 2 + 1;
    p.Wo = Wu / 2 + 1;
  } else {
    p.Ho = Hu + 2 * halo;
    p.Wo = Wu + 2 * halo;
  }
  p.count = float(H) * float(W + 2 * circ_stats) * float(C / groups);
  p.eps = eps;
  const int slabs = H * W / 16;  // >= 16 source pixels per slab; a function of the image size ONLY (batch-invariant sums)
  p.slabs = slabs < 1 ? 1 : (slabs > GN_PREP_SLABS ? GN_PREP_SLABS : slabs);
  const int vecs = C / 8;
  int ppi = 512 / vecs;
  if (ppi < 1) ppi = 1;
  const int threads = vecs * ppi;
  const size_t smem = 2 * (size_t)C * ppi * sizeof(float);  // <= 32 KB
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 g1(p.slabs, N);
  if (dtype == PF_BF16) gn_prep_kernel<true, true><<<g1, threads, smem, st>>>(p);
  else gn_prep_kernel<false, true><<<g1, threads, smem, st>>>(p);
  PF_CHECK_LAUNCH("gn_prep_kernel(stats)");
  const int ctas = p.phases * p.Ho * p.Wo / 16;  // >= 16 output positions per CTA
  const dim3 g2(ctas < 1 ? 1 : (ctas > GN_APPLY_CTAS ? GN_APPLY_CTAS : ctas), N);
  if (dtype == PF_BF16) gn_prep_kernel<true, false><<<g2, threads, smem, st>>>(p);
  else gn_prep_kernel<false, false><<<g2, threads, smem, st>>>(p);
  PF_CHECK_LAUNCH("gn_prep_kernel(apply)");
  return PF_OK;
}

extern "C" int pf_layernorm(const void* x, int ldx, void* out, int ldo, int dtype, int T, int C, const float* pe,
                            int pe_rows, const float* gamma, const float* beta, float eps, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(x && out && gamma && beta, "pf_layernorm: null pointer");
  PF_CHECK_ARG(dtype == PF_BF16 || dtype == PF_F16, "pf_layernorm: 16-bit dtype required");
  PF_CHECK_ARG(T > 0 && C > 0 && C % 8 == 0 && C <= 2048 && ldx % 8 == 0 && ldo % 8 == 0 && ldx >= C && ldo >= C,
               "pf_layernorm: bad shape T=%d C=%d", T, C);
  PF_CHECK_ARG(!pe || pe_rows > 0, "pf_layernorm: pe_rows must be positive");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int blocks = (T + 7) / 8;
  if (blocks > sm_count() * 8) blocks = sm_count() * 8;  // warps loop over tokens (affine parameters stay in registers)
  const uint16_t* xi = static_cast<const uint16_t*>(x);
  uint16_t* xo = static_cast<uint16_t*>(out);
  const int rounds = (C / 8 + 31) / 32;
#define PF_LN(BF, MV) layernorm_kernel<BF, MV><<<blocks, 256, 2 * (size_t)C * sizeof(float), st>>>(xi, ldx, pe, pe_rows, T, C, gamma, beta, eps, xo, ldo)
  if (dtype == PF_BF16) {
    if (rounds <= 2) PF_LN(true, 2); else if (rounds <= 5) PF_LN(true, 5); else PF_LN(true, 8);
  } else {
    if (rounds <= 2) PF_LN(false, 2); else if (rounds <= 5) PF_LN(false, 5); else PF_LN(false, 8);
  }
#undef PF_LN
  PF_CHECK_LAUNCH("layernorm_kernel");
  return PF_OK;
}
