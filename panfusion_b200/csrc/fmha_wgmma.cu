// Flash-attention forward on Hopper wgmma: S = Q K^T (both operands in shared memory) and O += P V (P from
// registers, V from shared memory), fp32 accumulators in registers, TMA-fed K/V ring, online softmax on the
// accumulator fragments, optional additive fp32 bias shared by all heads (the EPPA correspondence bias).
//
// Replaces: xformers.ops.memory_efficient_attention(q, k, v, attn_bias) at models/modules/transformer.py:71
// (EPPA, head dim 32, dense bias repeated per head at :68 — here never repeated) and the diffusers AttnProcessor
// bmm-softmax-bmm inside Transformer2DModel (MVGenModel.py:104,116,185,190,227,241; head dim 64, self and text
// cross attention).
//
// Tile: 128 queries x 64 keys. 288 threads: warps 0..3 and 4..7 are two consumer warpgroups of 64 queries each,
// warp 8 is the TMA producer. The S accumulator fragment of m64n64 has the register layout of the A operand of the
// next m64nDk16, so P never leaves registers.
#include <stdlib.h>

#include "pf_common.cuh"
#include "wgmma.cuh"

namespace pf {

constexpr int FA_BLOCK_M = 128;
constexpr int FA_BLOCK_N = 64;
constexpr int FA_THREADS = 288;

struct FmhaParams {
  int B, H, Lq, Lk;
  float scale_log2;  // softmax scale * log2(e)
  void* out;         // [B, Lq, out_ld] 16-bit, head h at columns [h*D, (h+1)*D)
  int out_ld;
  const float* bias;  // [bias_batches, Lq, bias_ld] or null
  long long bias_bstride;
  int bias_ld;
  // optional: per (128-query x 64-key) tile flag, 1 = every bias entry of the tile equals -1 (no correspondence):
  // the tile's loads are replaced by the constant. [bias_batches, ceil(Lq/128), ceil(Lk/64)] bytes.
  const uint8_t* bias_flags;
  long long flags_bstride;
  int flags_ld;
  // tile-packed bias (pf_bias_tile_pack): tile_off[bias batch][ceil(Lq/128)][ceil(Lk/64)] = index of the 128x64 tile in
  // `bias` (then a [n_live][128][64] store) or -1 for an all -1 tile; replaces bias_ld / bias_flags addressing
  const int* tile_off;
};

// ex2.approx.ftz: one MUFU op (exp2f() adds denormal / range fix-up instructions we do not need: inputs are <= 0)
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int D>
__host__ __device__ constexpr int fa_stages() { return D == 64 ? 2 : 4; }
template <int D>
__host__ __device__ constexpr int fmha_smem_bytes() {
  return FA_BLOCK_M * D * 2 + fa_stages<D>() * 2 * FA_BLOCK_N * D * 2 + 128;
}

// offset (floats) of element (row r, key k) inside one lane-interleaved packed 128 x 64 bias tile (pf_bias_tile_pack):
// 16-byte piece k/4 of row r sits at ((r/32)*16 + k/4)*32 + r%32 pieces from the tile start
__device__ __forceinline__ int packed_bias_off(int r, int k) {
  return (((r >> 5) * 16 + (k >> 2)) * 32 + (r & 31)) * 4 + (k & 3);
}

// Two CTAs per SM. The bias variants then spill a few registers (16 B at d = 32, 112 B at d = 64); without the bound they
// take 128 / 168 registers and fit one CTA per SM, which measured slower on an H100 SXM (700 W): EPPA attention at the
// C2 level-32 shapes 305 / 247 us against 376 / 358 us (scripts/fmha_bias_micro.py), the whole C2 step 20.0 vs 19.3 steps/s.
template <int D, bool BF16, bool HAS_BIAS>
__global__ void __launch_bounds__(FA_THREADS, 2)
fmha_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const FmhaParams p) {
  static_assert(D == 32 || D == 64, "head dim 32 (EPPA) or 64 (SD-2 UNet)");
  constexpr int STAGES = fa_stages<D>();
  constexpr int Q_BYTES = FA_BLOCK_M * D * 2;
  constexpr int KV_BYTES = FA_BLOCK_N * D * 2;  // one of K or V
  constexpr uint32_t SW_LAYOUT = (D == 64) ? 1u : 2u;           // wgmma layout type: 128B / 64B swizzle
  constexpr uint32_t SW_ATOM_BYTES = (D == 64) ? 1024u : 512u;  // 8 rows of D*2 bytes
  constexpr float LOG2E = 1.4426950408889634f;

  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + Q_BYTES;  // stage s: K at s*2*KV_BYTES, V right after
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + STAGES * 2 * KV_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;
  uint64_t* kv_empty = kv_full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.x % p.H;  // heads fastest: CTAs sharing a bias tile run together (L2 reuse)
  const int qt = blockIdx.x / p.H;
  const int b = blockIdx.y;
  const int q0 = qt * FA_BLOCK_M;
  const int n_tiles = (p.Lk + FA_BLOCK_N - 1) / FA_BLOCK_N;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 2);  // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      mbar_expect_tx(q_full, Q_BYTES);
      tma_load_4d(sQ, &tmQ, q_full, 0, h, q0, b);
      for (int j = 0; j < n_tiles; ++j) {
        const int s = j % STAGES;
        mbar_wait(&kv_empty[s], ((j / STAGES) & 1) ^ 1);
        mbar_expect_tx(&kv_full[s], 2 * KV_BYTES);
        uint8_t* dst = sKV + s * 2 * KV_BYTES;
        tma_load_4d(dst, &tmK, &kv_full[s], 0, h, j * FA_BLOCK_N, b);
        tma_load_4d(dst + KV_BYTES, &tmV, &kv_full[s], 0, h, j * FA_BLOCK_N, b);
      }
    }
    return;
  }

  // ---------------------------------- consumers ----------------------------------
  const int wg = threadIdx.x >> 7;                              // queries [64 wg, 64 wg + 64) of the tile
  const int rA = wg * 64 + (warp & 3) * 16 + (lane >> 2);       // tile rows of this thread: rA and rA + 8
  const int cq = 2 * (lane & 3);                                // key column of the fragment inside each 8-key group
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float oacc[D / 2];
  float sacc[FA_BLOCK_N / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) oacc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < FA_BLOCK_N / 2; ++i) sacc[i] = 0.f;
  const float* bias_rows[2] = {nullptr, nullptr};
  const uint8_t* flag_row = nullptr;
  const int* off_row = nullptr;
  if constexpr (HAS_BIAS) {
    if (p.tile_off) {
      off_row = p.tile_off + (long long)b * p.flags_bstride + (long long)qt * p.flags_ld;
    } else {
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int q = q0 + rA + 8 * hr;
        const int qq = q < p.Lq ? q : p.Lq - 1;
        bias_rows[hr] = p.bias + (long long)b * p.bias_bstride + (long long)qq * p.bias_ld;
      }
      if (p.bias_flags) flag_row = p.bias_flags + (long long)b * p.flags_bstride + (long long)qt * p.flags_ld;
    }
  }
  mbar_wait(q_full, 0);
  const uint64_t qdesc = make_wgmma_desc(smem_u32(sQ + wg * 64 * D * 2), 16, SW_ATOM_BYTES, SW_LAYOUT);

  for (int j = 0; j < n_tiles; ++j) {
    const int s = j % STAGES;
    const int k0 = j * FA_BLOCK_N;
    mbar_wait(&kv_full[s], (j / STAGES) & 1);
    const uint32_t k_addr = smem_u32(sKV + s * 2 * KV_BYTES);
    const uint64_t kdesc = make_wgmma_desc(k_addr, 16, SW_ATOM_BYTES, SW_LAYOUT);
    wgmma_fence();
    fence_regs(sacc);
#pragma unroll
    for (int k = 0; k < D / 16; ++k) Wgmma<FA_BLOCK_N, BF16>::ss(sacc, qdesc + 2 * k, kdesc + 2 * k, k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(sacc);

    // logits in log2 units; sacc[4 g + 2 hr + e] is (row rA + 8 hr, key 8 g + cq + e)
    if constexpr (HAS_BIAS) {
      int toff = 0;
      if (off_row) toff = off_row[j];
      const bool constant_tile = off_row ? toff < 0 : (flag_row != nullptr && flag_row[j] != 0);
      if (constant_tile) {
#pragma unroll
        for (int i = 0; i < FA_BLOCK_N / 2; ++i) sacc[i] = fmaf(sacc[i], p.scale_log2, -LOG2E);
      } else if (off_row) {
        const float* tb = p.bias + (long long)toff * (FA_BLOCK_M * FA_BLOCK_N);
#pragma unroll
        for (int g = 0; g < FA_BLOCK_N / 8; ++g)
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const float2 t = __ldg(reinterpret_cast<const float2*>(tb + packed_bias_off(rA + 8 * hr, 8 * g + cq)));
            sacc[4 * g + 2 * hr] = fmaf(t.x, LOG2E, sacc[4 * g + 2 * hr] * p.scale_log2);
            sacc[4 * g + 2 * hr + 1] = fmaf(t.y, LOG2E, sacc[4 * g + 2 * hr + 1] * p.scale_log2);
          }
      } else if (k0 + FA_BLOCK_N <= p.Lk) {
#pragma unroll
        for (int g = 0; g < FA_BLOCK_N / 8; ++g)
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const float2 t = __ldg(reinterpret_cast<const float2*>(bias_rows[hr] + k0 + 8 * g + cq));
            sacc[4 * g + 2 * hr] = fmaf(t.x, LOG2E, sacc[4 * g + 2 * hr] * p.scale_log2);
            sacc[4 * g + 2 * hr + 1] = fmaf(t.y, LOG2E, sacc[4 * g + 2 * hr + 1] * p.scale_log2);
          }
      } else {  // ragged last key tile of a dense table
#pragma unroll
        for (int g = 0; g < FA_BLOCK_N / 8; ++g)
#pragma unroll
          for (int hr = 0; hr < 2; ++hr)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int k = k0 + 8 * g + cq + e;
              const float bv = k < p.Lk ? __ldg(bias_rows[hr] + k) : 0.f;
              sacc[4 * g + 2 * hr + e] = fmaf(bv, LOG2E, sacc[4 * g + 2 * hr + e] * p.scale_log2);
            }
      }
    } else {
#pragma unroll
      for (int i = 0; i < FA_BLOCK_N / 2; ++i) sacc[i] *= p.scale_log2;
    }
    if (k0 + FA_BLOCK_N > p.Lk) {
#pragma unroll
      for (int g = 0; g < FA_BLOCK_N / 8; ++g)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (k0 + 8 * g + cq + e >= p.Lk) sacc[4 * g + e] = sacc[4 * g + 2 + e] = -INFINITY;
    }
    // online softmax: the four threads of a quad share a row
    float alpha[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float mx = -INFINITY;
#pragma unroll
      for (int g = 0; g < FA_BLOCK_N / 8; ++g) mx = fmaxf(mx, fmaxf(sacc[4 * g + 2 * hr], sacc[4 * g + 2 * hr + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[hr], mx);
      alpha[hr] = fast_exp2(m_run[hr] - m_new);  // 0 on the first tile
      m_run[hr] = m_new;
      float ls = 0.f;
#pragma unroll
      for (int g = 0; g < FA_BLOCK_N / 8; ++g)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float pv = fast_exp2(sacc[4 * g + 2 * hr + e] - m_new);
          sacc[4 * g + 2 * hr + e] = pv;
          ls += pv;
        }
      l_run[hr] = l_run[hr] * alpha[hr] + ls;  // per-thread partial row sum; the quad is summed at the end
    }
#pragma unroll
    for (int g = 0; g < D / 8; ++g) {
      oacc[4 * g] *= alpha[0];
      oacc[4 * g + 1] *= alpha[0];
      oacc[4 * g + 2] *= alpha[1];
      oacc[4 * g + 3] *= alpha[1];
    }
    // P as the register A operand of m64nDk16: keys [16 kk, 16 kk + 16) = S column groups 2 kk and 2 kk + 1
    uint32_t pa[FA_BLOCK_N / 16][4];
#pragma unroll
    for (int kk = 0; kk < FA_BLOCK_N / 16; ++kk) {
      pa[kk][0] = pack2<BF16>(sacc[8 * kk + 0], sacc[8 * kk + 1]);
      pa[kk][1] = pack2<BF16>(sacc[8 * kk + 2], sacc[8 * kk + 3]);
      pa[kk][2] = pack2<BF16>(sacc[8 * kk + 4], sacc[8 * kk + 5]);
      pa[kk][3] = pack2<BF16>(sacc[8 * kk + 6], sacc[8 * kk + 7]);
    }
    // V tile [64 keys][D]: MN-major B operand; 8-key groups are SW_ATOM_BYTES apart, one swizzle atom along D
    const uint32_t v_addr = k_addr + KV_BYTES;
    wgmma_fence();
    fence_regs(oacc);
#pragma unroll
    for (int kk = 0; kk < FA_BLOCK_N / 16; ++kk)
      Wgmma<D, BF16>::rs(oacc, pa[kk], make_wgmma_desc(v_addr + kk * 2 * SW_ATOM_BYTES, SW_ATOM_BYTES, SW_ATOM_BYTES, SW_LAYOUT),
                         1);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(oacc);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[s]);  // this warpgroup is done with K and V of the stage
  }

  // normalise and store
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    float l = l_run[hr];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.0f / l;
    const int q = q0 + rA + 8 * hr;
    if (q < p.Lq) {
      uint16_t* orow = static_cast<uint16_t*>(p.out) + ((long long)b * p.Lq + q) * p.out_ld + h * D;
#pragma unroll
      for (int g = 0; g < D / 8; ++g)
        *reinterpret_cast<uint32_t*>(orow + 8 * g + cq) =
            pack2<BF16>(oacc[4 * g + 2 * hr] * inv, oacc[4 * g + 2 * hr + 1] * inv);
    }
  }
}

static int make_qkv_tmap(CUtensorMap* tm, int dtype, const void* ptr, int B, int H, int L, int D, int ld,
                         long long bstride, int box_rows) {
  uint64_t dims[4] = {(uint64_t)D, (uint64_t)H, (uint64_t)L, (uint64_t)B};
  uint64_t str[3] = {(uint64_t)D * 2, (uint64_t)ld * 2, (uint64_t)bstride * 2};
  uint32_t box[4] = {(uint32_t)D, 1, (uint32_t)box_rows, 1};
  return make_tmap(tm, dtype, 4, ptr, dims, str, box, D == 64 ? 128 : 64);
}

template <int D, bool BF16, bool HAS_BIAS>
static int launch_fmha(const pf_fmha_args* a, cudaStream_t st) {
  CUtensorMap tmQ, tmK, tmV;
  int rc;
  if ((rc = make_qkv_tmap(&tmQ, a->dtype, a->q, a->B, a->H, a->Lq, D, a->q_ld, a->q_bstride, FA_BLOCK_M))) return rc;
  if ((rc = make_qkv_tmap(&tmK, a->dtype, a->k, a->B, a->H, a->Lk, D, a->k_ld, a->k_bstride, FA_BLOCK_N))) return rc;
  if ((rc = make_qkv_tmap(&tmV, a->dtype, a->v, a->B, a->H, a->Lk, D, a->v_ld, a->v_bstride, FA_BLOCK_N))) return rc;
  FmhaParams p;
  p.B = a->B; p.H = a->H; p.Lq = a->Lq; p.Lk = a->Lk;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.out = a->out; p.out_ld = a->out_ld;
  p.bias = a->bias; p.bias_bstride = a->bias_bstride; p.bias_ld = a->bias_ld;
  p.bias_flags = a->bias_flags; p.flags_bstride = a->flags_bstride; p.flags_ld = a->flags_ld;
  p.tile_off = a->bias_tile_off;
  auto kern = fmha_fwd_kernel<D, BF16, HAS_BIAS>;
  constexpr int SMEM = fmha_smem_bytes<D>();
  static bool attr_set = false;
  if (!attr_set) {
    rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM),
                    "cudaFuncSetAttribute(fmha)");
    if (rc) return rc;
    attr_set = true;
  }
  dim3 grid(((a->Lq + FA_BLOCK_M - 1) / FA_BLOCK_M) * a->H, a->B);
  kern<<<grid, FA_THREADS, SMEM, st>>>(tmQ, tmK, tmV, p);
  PF_CHECK_LAUNCH("fmha_fwd_kernel");
  return PF_OK;
}

}  // namespace pf

extern "C" int pf_fmha_fwd(const pf_fmha_args* a, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(a != nullptr, "pf_fmha_fwd: null args");
  PF_CHECK_ARG(a->dtype == PF_BF16 || a->dtype == PF_F16, "pf_fmha_fwd: dtype must be PF_F16 or PF_BF16");
  PF_CHECK_ARG(a->q && a->k && a->v && a->out, "pf_fmha_fwd: null operand");
  PF_CHECK_ARG(a->head_dim == 32 || a->head_dim == 64, "pf_fmha_fwd: head_dim %d unsupported (32 or 64)", a->head_dim);
  PF_CHECK_ARG(a->B > 0 && a->B <= 65535 && a->H > 0 && a->Lq > 0 && a->Lk > 0, "pf_fmha_fwd: empty shape");
  PF_CHECK_ARG(a->q_ld % 8 == 0 && a->k_ld % 8 == 0 && a->v_ld % 8 == 0 && a->out_ld % 8 == 0,
               "pf_fmha_fwd: leading dims must be multiples of 8 elements");
  PF_CHECK_ARG(((uintptr_t)a->q & 15) == 0 && ((uintptr_t)a->k & 15) == 0 && ((uintptr_t)a->v & 15) == 0 &&
                   ((uintptr_t)a->out & 15) == 0,
               "pf_fmha_fwd: operands must be 16-byte aligned");
  PF_CHECK_ARG(!a->bias || a->bias_tile_off || (a->bias_ld % 4 == 0 && ((uintptr_t)a->bias & 15) == 0 && a->bias_ld >= a->Lk),
               "pf_fmha_fwd: bias must be 16-byte aligned with bias_ld %% 4 == 0");
  PF_CHECK_ARG(!a->bias_tile_off || (a->bias && ((uintptr_t)a->bias & 15) == 0 && !a->bias_flags && a->flags_ld > 0),
               "pf_fmha_fwd: a tile-packed bias needs the packed store in `bias`, flags_ld = tiles per row, no bias_flags");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool bf = a->dtype == PF_BF16;
  const bool hb = a->bias != nullptr;
  if (a->head_dim == 64) {
    if (bf) return hb ? launch_fmha<64, true, true>(a, st) : launch_fmha<64, true, false>(a, st);
    return hb ? launch_fmha<64, false, true>(a, st) : launch_fmha<64, false, false>(a, st);
  }
  if (bf) return hb ? launch_fmha<32, true, true>(a, st) : launch_fmha<32, true, false>(a, st);
  return hb ? launch_fmha<32, false, true>(a, st) : launch_fmha<32, false, false>(a, st);
}
