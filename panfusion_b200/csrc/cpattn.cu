// Correspondence-aware attention of MVDiffusion (external/MVDiffusion/pano/modules.py:22-86, pano/utils.py:45-123):
// every pixel of view i attends to a 3x3 window around its homography correspondence in views i-1 and i+1 (ring
// order), 18 keys per query.
//
//   pf_cpattn_tables : per (camera group, view, query pixel, key slot) the grid_sample position in the neighbour's
//                      feature map, the in-image mask and the key's relative position xy_rel (the PE argument).
//                      Built once per (camera set, level); the homographies come from the host (fp32 torch.inverse,
//                      exactly as the reference computes them) and are applied here with the fp32 FMA chain that a
//                      CPU batched matmul uses, so positions and xy_rel reproduce the reference's bits.
//   pf_cpattn_gather : key rows [18 T, C] = (bilinear sample + PosEmbedding(xy_rel)) * mask, 16-bit, together with
//                      each row's (sum, sum of squares) so that norm1 folds into the K|V projection GEMM (ln_stats).
//   pf_cpattn_attn   : one query against its 18 keys per (pixel, head), head_dim 32, fp32 softmax, 16-bit output.
//
// Key slot s = n * 9 + (di + 1) * 3 + (dj + 1): n = 0 for view i-1, 1 for view i+1; the window offset di moves x and
// dj moves y (utils.py:58-62), the order in which the reference concatenates its keys.
#include "pf_common.cuh"

namespace pf {

constexpr int CP_SLOTS = 18;

// x' = H [x, y, 1]^T with the accumulation order of a CPU fp32 batched matmul: h0 x, then two FMAs
__device__ __forceinline__ void homog(const float* __restrict__ H, float x, float y, float& ox, float& oy) {
  float r[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float a = __fmul_rn(H[3 * k], x);
    a = __fmaf_rn(H[3 * k + 1], y, a);
    r[k] = __fmaf_rn(H[3 * k + 2], 1.f, a);
  }
  ox = __fdiv_rn(r[0], r[2]);
  oy = __fdiv_rn(r[1], r[2]);
}

// thread <-> (group g, view i, query pixel q, neighbour n): one correspondence, nine window taps
__global__ void __launch_bounds__(256)
cpattn_tables_kernel(const float* __restrict__ homo_l, const float* __restrict__ homo_r, int G, int m, int h, int w,
                     int img, float4* __restrict__ pos, uint8_t* __restrict__ mask) {
  const int P = h * w;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)G * m * P * 2) return;
  const int n = int(idx & 1);
  const long long gq = idx >> 1;          // (g * m + i) * P + q
  const int q = int(gq % P);
  const long long gi = gq / P;            // g * m + i
  const int s = img / h;                  // query_scale == key_scale (utils.py:48-49)
  const float fs = float(s);
  const float X = float(s / 2 + s * (q % w)), Y = float(s / 2 + s * (q / w));  // get_x_2d()[s//2::s, s//2::s]
  float hl[9], hr[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    hl[k] = __ldg(homo_l + (gi * 2 + n) * 9 + k);
    hr[k] = __ldg(homo_r + (gi * 2 + n) * 9 + k);
  }
  float cx, cy;
  homog(hl, X, Y, cx, cy);                              // get_correspondences (utils.py:26-38)
  const float px = __fsub_rn(__fdiv_rn(cx, fs), 0.5f);  // utils.py:51-52
  const float py = __fsub_rn(__fdiv_rn(cy, fs), 0.5f);
  const float fimg = float(img);
  const float sx = (w - 1) * 0.5f, sy = (h - 1) * 0.5f;
  const long long out0 = gq * CP_SLOTS + n * 9;
#pragma unroll
  for (int di = -1; di <= 1; ++di) {
#pragma unroll
    for (int dj = -1; dj <= 1; ++dj) {
      const float nx = __fadd_rn(px, float(di)), ny = __fadd_rn(py, float(dj));
      const float rx = __fmul_rn(__fadd_rn(nx, 0.5f), fs), ry = __fmul_rn(__fadd_rn(ny, 0.5f), fs);  // utils.py:63
      const bool ok = rx > 0.f && rx < fimg && ry > 0.f && ry < fimg;                                  // utils.py:74-75
      // grid_sample(align_corners=True) of the normalised grid (utils.py:67-70): normalise, then unnormalise as
      // ATen's CPU kernel does, (g + 1) * (size - 1) / 2
      const float gx = __fsub_rn(__fmul_rn(__fdiv_rn(nx, float(w - 1)), 2.f), 1.f);
      const float gy = __fsub_rn(__fmul_rn(__fdiv_rn(ny, float(h - 1)), 2.f), 1.f);
      float bx, by;
      homog(hr, rx, ry, bx, by);                                       // utils.py:77-84
      const float relx = __fdiv_rn(__fsub_rn(bx, X), fs);             // utils.py:91
      const float rely = __fdiv_rn(__fsub_rn(by, Y), fs);
      const long long o = out0 + (di + 1) * 3 + (dj + 1);
      pos[o] = make_float4(__fmul_rn(__fadd_rn(gx, 1.f), sx), __fmul_rn(__fadd_rn(gy, 1.f), sy), relx, rely);
      mask[o] = ok ? 1 : 0;
    }
  }
}

template <typename T>
__device__ __forceinline__ void load8(const T* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 f = unpack2<std::is_same<T, __nv_bfloat16>::value>(w4[e]);
    v[2 * e] = f.x;
    v[2 * e + 1] = f.y;
  }
}

template <typename T>
__device__ __forceinline__ void store8(T* p, const float (&v)[8], float& s, float& sq) {
  constexpr bool BF = std::is_same<T, __nv_bfloat16>::value;
  uint32_t w4[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    w4[e] = pack2<BF>(v[2 * e], v[2 * e + 1]);
    const float2 r = unpack2<BF>(w4[e]);  // statistics of the values the GEMM will read
    s += r.x + r.y;
    sq = fmaf(r.x, r.x, fmaf(r.y, r.y, sq));
  }
  *reinterpret_cast<uint4*>(p) = make_uint4(w4[0], w4[1], w4[2], w4[3]);
}

// warp <-> one key row (token, slot). Lane chunk c covers channels [8c, 8c + 8) and [2N + 8c, 2N + 8c + 8), N = C / 4:
// the PE layout is [sin(x f), sin(y f), cos(x f), cos(y f)] (transformer.py:201-208), so both halves share sincosf.
template <typename T>
__global__ void __launch_bounds__(256)
cpattn_gather_kernel(const T* __restrict__ x, int ldx, int B, int m, int h, int w, int C, int G,
                     const float4* __restrict__ pos, const uint8_t* __restrict__ mask, const float* __restrict__ freq,
                     T* __restrict__ keys, float4* __restrict__ stats) {
  const int P = h * w;
  const long long rows = (long long)B * m * P * CP_SLOTS;
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const long long tok = row / CP_SLOTS;
  const int slot = int(row % CP_SLOTS);
  const int b = int(tok / ((long long)m * P));
  const int i = int((tok / P) % m);
  const int q = int(tok % P);
  const int g = G == 1 ? 0 : b;
  const long long e = (((long long)g * m + i) * P + q) * CP_SLOTS + slot;
  T* dst = keys + row * (long long)C;
  const int chunks = C >> 4, N = C >> 2;
  if (!__ldg(mask + e)) {  // a masked key is the zero vector; it stays in the softmax (LN1(0) = beta)
    for (int c = lane; c < chunks; c += 32) {
      *reinterpret_cast<uint4*>(dst + 8 * c) = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(dst + 2 * N + 8 * c) = make_uint4(0, 0, 0, 0);
    }
    if (lane == 0) stats[row] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  const float4 p = __ldg(pos + e);
  const int j = slot < 9 ? (i + m - 1) % m : (i + 1) % m;
  const T* src = x + ((long long)b * m + j) * P * ldx;
  // bilinear taps of grid_sample (zero padding): nw, ne, sw, se
  const float fx = floorf(p.x), fy = floorf(p.y);
  const int x0 = int(fx), y0 = int(fy);
  const float wgt[4] = {(fx + 1.f - p.x) * (fy + 1.f - p.y), (p.x - fx) * (fy + 1.f - p.y),
                        (fx + 1.f - p.x) * (p.y - fy), (p.x - fx) * (p.y - fy)};
  long long off[4];
  bool in[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int xx = x0 + (t & 1), yy = y0 + (t >> 1);
    in[t] = xx >= 0 && xx < w && yy >= 0 && yy < h;
    off[t] = in[t] ? ((long long)yy * w + xx) * ldx : 0;
  }
  float s = 0.f, sq = 0.f;
  for (int c = lane; c < chunks; c += 32) {
    float lo[8], hi[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) lo[k] = hi[k] = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      if (!in[t]) continue;
      float a[8], bb[8];
      load8(src + off[t] + 8 * c, a);
      load8(src + off[t] + 2 * N + 8 * c, bb);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        lo[k] = fmaf(a[k], wgt[t], lo[k]);
        hi[k] = fmaf(bb[k], wgt[t], hi[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int ch = 8 * c + k;  // < 2N: sin part (x for ch < N, y otherwise)
      const float arg = __fmul_rn(ch < N ? p.z : p.w, __ldg(freq + (ch < N ? ch : ch - N)));
      float sn, cs;
      sincosf(arg, &sn, &cs);  // accurate range reduction: frequencies reach 2^79 at C = 320
      lo[k] += sn;
      hi[k] += cs;
    }
    store8(dst + 8 * c, lo, s, sq);
    store8(dst + 2 * N + 8 * c, hi, s, sq);
  }
  s = warp_sum(s);
  sq = warp_sum(sq);
  if (lane == 0) stats[row] = make_float4(s, sq, 0.f, 0.f);  // slot 0 = (sum, sum of squares), slot 1 = 0
}

// thread <-> (token, head): q . k_s for the 18 keys, softmax in fp32, o = sum p_s v_s (transformer.py:57-77)
template <typename T>
__global__ void __launch_bounds__(256)
cpattn_attn_kernel(const T* __restrict__ q, int ldq, const T* __restrict__ kv, int ldkv, T* __restrict__ out, int ldo,
                   long long ntok, int C, float scale) {
  const int H = C >> 5;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= ntok * H) return;
  const long long tok = idx / H;
  const int hd = int(idx % H) * 32;
  float qv[32];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    float t8[8];
    load8(q + tok * ldq + hd + 8 * c, t8);
#pragma unroll
    for (int k = 0; k < 8; ++k) qv[8 * c + k] = t8[k];
  }
  const T* kr = kv + tok * CP_SLOTS * (long long)ldkv + hd;
  float sc[CP_SLOTS];
  float mx = -INFINITY;
#pragma unroll
  for (int sl = 0; sl < CP_SLOTS; ++sl) {
    float acc = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float t8[8];
      load8(kr + sl * (long long)ldkv + 8 * c, t8);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc = fmaf(qv[8 * c + k], t8[k], acc);
    }
    sc[sl] = acc * scale;
    mx = fmaxf(mx, sc[sl]);
  }
  float den = 0.f;
#pragma unroll
  for (int sl = 0; sl < CP_SLOTS; ++sl) {
    sc[sl] = expf(sc[sl] - mx);
    den += sc[sl];
  }
  float o[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) o[k] = 0.f;
#pragma unroll
  for (int sl = 0; sl < CP_SLOTS; ++sl) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float t8[8];
      load8(kr + sl * (long long)ldkv + C + 8 * c, t8);
#pragma unroll
      for (int k = 0; k < 8; ++k) o[8 * c + k] = fmaf(sc[sl], t8[k], o[8 * c + k]);
    }
  }
  const float inv = 1.f / den;
  constexpr bool BF = std::is_same<T, __nv_bfloat16>::value;
  uint32_t w16[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) w16[k] = pack2<BF>(o[2 * k] * inv, o[2 * k + 1] * inv);
  uint4* d = reinterpret_cast<uint4*>(out + tok * ldo + hd);
#pragma unroll
  for (int c = 0; c < 4; ++c) d[c] = make_uint4(w16[4 * c], w16[4 * c + 1], w16[4 * c + 2], w16[4 * c + 3]);
}

}  // namespace pf

extern "C" int pf_cpattn_tables(const float* homo_l, const float* homo_r, int G, int m, int h, int w, int img_size,
                                float* pos, uint8_t* mask, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(homo_l && homo_r && pos && mask, "pf_cpattn_tables: null pointer");
  PF_CHECK_ARG(G > 0 && m > 1 && h >= 2 && w == h && img_size >= h && img_size % h == 0,
               "pf_cpattn_tables: bad shape G=%d m=%d h=%d w=%d img=%d", G, m, h, w, img_size);
  PF_CHECK_ARG((reinterpret_cast<uintptr_t>(pos) & 15) == 0, "pf_cpattn_tables: pos must be 16-byte aligned");
  const long long threads = (long long)G * m * h * w * 2;
  cpattn_tables_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      homo_l, homo_r, G, m, h, w, img_size, reinterpret_cast<float4*>(pos), mask);
  PF_CHECK_LAUNCH("cpattn_tables_kernel");
  return PF_OK;
}

extern "C" int pf_cpattn_gather(const void* x, int ldx, int dtype, int B, int m, int h, int w, int C, int G,
                                const float* pos, const uint8_t* mask, const float* freq_bands, void* keys, float* stats,
                                void* stream) {
  using namespace pf;
  PF_CHECK_ARG(x && pos && mask && freq_bands && keys && stats, "pf_cpattn_gather: null pointer");
  PF_CHECK_ARG(dtype == PF_BF16 || dtype == PF_F16, "pf_cpattn_gather: 16-bit dtype required");
  PF_CHECK_ARG(B > 0 && m > 1 && h >= 2 && w >= 2 && C > 0 && C % 32 == 0 && ldx >= C && ldx % 8 == 0 &&
                   (G == 1 || G == B),
               "pf_cpattn_gather: bad shape B=%d m=%d h=%d w=%d C=%d ldx=%d G=%d", B, m, h, w, C, ldx, G);
  PF_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(keys) |
                 reinterpret_cast<uintptr_t>(pos) | reinterpret_cast<uintptr_t>(stats)) & 15) == 0,
               "pf_cpattn_gather: x, keys, pos and stats must be 16-byte aligned");
  const long long rows = (long long)B * m * h * w * CP_SLOTS;
  const long long blocks = (rows + 7) / 8;
  PF_CHECK_ARG(blocks < (1LL << 31), "pf_cpattn_gather: too many rows");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PF_BF16)
    cpattn_gather_kernel<__nv_bfloat16><<<(unsigned)blocks, 256, 0, st>>>(
        static_cast<const __nv_bfloat16*>(x), ldx, B, m, h, w, C, G, reinterpret_cast<const float4*>(pos), mask,
        freq_bands, static_cast<__nv_bfloat16*>(keys), reinterpret_cast<float4*>(stats));
  else
    cpattn_gather_kernel<__half><<<(unsigned)blocks, 256, 0, st>>>(
        static_cast<const __half*>(x), ldx, B, m, h, w, C, G, reinterpret_cast<const float4*>(pos), mask, freq_bands,
        static_cast<__half*>(keys), reinterpret_cast<float4*>(stats));
  PF_CHECK_LAUNCH("cpattn_gather_kernel");
  return PF_OK;
}

extern "C" int pf_cpattn_attn(const void* q, int ldq, const void* kv, int ldkv, void* out, int ldo, int dtype,
                              long long ntok, int C, float scale, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(q && kv && out, "pf_cpattn_attn: null pointer");
  PF_CHECK_ARG(dtype == PF_BF16 || dtype == PF_F16, "pf_cpattn_attn: 16-bit dtype required");
  PF_CHECK_ARG(ntok > 0 && C > 0 && C % 32 == 0 && ldq >= C && ldkv >= 2 * C && ldo >= C && ldq % 8 == 0 &&
                   ldkv % 8 == 0 && ldo % 8 == 0,
               "pf_cpattn_attn: bad shape ntok=%lld C=%d ldq=%d ldkv=%d ldo=%d", ntok, C, ldq, ldkv, ldo);
  PF_CHECK_ARG(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(kv) | reinterpret_cast<uintptr_t>(out)) &
                15) == 0,
               "pf_cpattn_attn: q, kv and out must be 16-byte aligned");
  const long long threads = ntok * (C / 32);
  PF_CHECK_ARG((threads + 255) / 256 < (1LL << 31), "pf_cpattn_attn: too many tokens");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const unsigned blocks = (unsigned)((threads + 255) / 256);
  if (dtype == PF_BF16)
    cpattn_attn_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(q), ldq,
                                                              static_cast<const __nv_bfloat16*>(kv), ldkv,
                                                              static_cast<__nv_bfloat16*>(out), ldo, ntok, C, scale);
  else
    cpattn_attn_kernel<__half><<<blocks, 256, 0, st>>>(static_cast<const __half*>(q), ldq,
                                                       static_cast<const __half*>(kv), ldkv, static_cast<__half*>(out),
                                                       ldo, ntok, C, scale);
  PF_CHECK_LAUNCH("cpattn_attn_kernel");
  return PF_OK;
}
