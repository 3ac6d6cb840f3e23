// Tap-GEMM on Hopper: TMA (SWIZZLE_128B) -> shared-memory ring -> wgmma (m64 x BLOCK_N x k16 per warpgroup, fp32 in
// registers) -> epilogue. One kernel serves nn.Linear and every 1x1 / 3x3 convolution of the UNet walk
// (reference call sites: models/pano/MVGenModel.py:85-295 through diffusers ResnetBlock2D / Transformer2DModel,
//  models/modules/transformer.py:57-74,8-35). A convolution is a sum of `num_taps` GEMMs whose A operand is the
// same channels-last image shifted by a constant row offset (zero-haloed "padded-flat" layout), so the im2col
// matrix is never formed: each K-slab is one plain 2-D TMA box.
//
// 256 threads: warps 0..3 and 4..7 = two warpgroups, each owning 64 of the 128 tile rows through the main loop.
// There is no producer warp: thread 0 fills the ring before the loop, and the leader of whichever warpgroup releases
// a slot last issues the slot's next TMA loads, so no MMA-issuing warp ever blocks on the other warpgroup. After the last K-slab the accumulators are written to shared memory (over the now idle operand
// ring) and all 256 threads run the epilogue with two threads per tile row (even / odd 16-column chunks): bias / LayerNorm fold / per-image row bias / SiLU / GELU / GEGLU / residual,
// then either (EPI_TMA) swizzled [128][32] sub-tiles streamed out with TMA tile stores through two staging buffers
// behind the accumulators, or direct stores through the halo-dropping row map (convolutions, fp32 outputs, GEGLU),
// or raw fp32 split-K partials.
//
// Instantiations with a short ring (CTAS = 2) run TWO CTAs per SM (at most 128 registers per thread and 113 KB of
// shared memory per CTA): a tile has no overlap of its own between ring fill, main loop, accumulator dump and
// epilogue, so the tensor pipe is kept busy by the other CTA's main loop while one CTA fills or drains. A ninth
// (producer) warp would rule that out: registers are granted to whole warps, nine warps would leave two CTAs 96
// registers per thread, and the 160-wide tile alone holds 80 accumulators. The 256-wide GEGLU tile (128 accumulators,
// 133 KB accumulator dump) and split-K, which is planned at about one CTA per SM, keep a long ring and CTAS = 1.
#include <stdlib.h>

#include "gemm_common.cuh"
#include "wgmma.cuh"

namespace pf {

constexpr int GEMM_THREADS = 256;

constexpr int GEMM_SUB_BYTES = GEMM_BLOCK_M * 64;  // one [128][32] 16-bit sub-tile of the TMA-store epilogue, SWIZZLE_64B
// an SM has 228 KB of shared memory and every resident CTA reserves 1 KB of it
constexpr int GEMM_SMEM_CORESIDENT = 228 * 1024 / 2 - 1024;

__host__ __device__ constexpr int gemm_acc_ld(int block_n) { return block_n + 4; }  // floats; +4: conflict-free rows
// accumulator dump, rounded up to the 1024 bytes that keep the staging buffers behind it swizzle-aligned
__host__ __device__ constexpr int gemm_acc_bytes(int block_n) {
  return (GEMM_BLOCK_M * gemm_acc_ld(block_n) * 4 + 1023) / 1024 * 1024;
}
// the operand ring; after the main loop the same bytes hold the accumulators and (EPI_TMA) two staging sub-tiles
__host__ __device__ constexpr int gemm_ring_bytes(int block_n, int stages, bool epi_tma) {
  const int ring = stages * gemm_stage_bytes(block_n);
  const int epi = gemm_acc_bytes(block_n) + (epi_tma ? 2 * GEMM_SUB_BYTES : 0);
  return ((ring > epi ? ring : epi) + 1023) / 1024 * 1024;
}
// full barrier (8 bytes) and release counter (4 bytes) per stage, rounded up to keep s_bias 16-byte aligned
__host__ __device__ constexpr int gemm_bar_bytes(int stages) { return (stages * 12 + 15) / 16 * 16; }
__host__ __device__ constexpr int gemm_smem_bytes(int block_n, int stages, bool epi_tma) {
  return gemm_ring_bytes(block_n, stages, epi_tma) + gemm_bar_bytes(stages) +
         2 * block_n * 4 /*bias row + LayerNorm column sums*/;
}

template <int BLOCK_N, int STAGES, int CTAS, bool BF16, bool EPI_TMA>
__global__ void __launch_bounds__(GEMM_THREADS, CTAS)
gemm_taps_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmC, const GemmKernelParams p) {
  constexpr int A_BYTES = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;
  constexpr int STAGE_BYTES = gemm_stage_bytes(BLOCK_N);
  constexpr int RING_BYTES = gemm_ring_bytes(BLOCK_N, STAGES, EPI_TMA);
  constexpr int ACC_LD = gemm_acc_ld(BLOCK_N);
  constexpr int NCH = BLOCK_N / 16;
  constexpr int NACC = BLOCK_N / 2;  // fp32 accumulators per thread of an m64 x BLOCK_N warpgroup tile
  static_assert(BLOCK_N % 32 == 0 && BLOCK_N <= 256, "tile width");

  // 1024-byte alignment (128 B swizzle atoms) is requested on the declaration; verified once, never padded for
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  float* sacc = reinterpret_cast<float*>(smem);  // [128][ACC_LD] fp32, over the ring once the main loop is done
  uint8_t* staging = smem + gemm_acc_bytes(BLOCK_N);  // EPI_TMA: two [128][32] 16-bit sub-tiles, also inside the ring
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + RING_BYTES);
  uint32_t* released = reinterpret_cast<uint32_t*>(full_bar + STAGES);  // per slot: releases by the two warpgroups
  float* s_bias = reinterpret_cast<float*>(smem + RING_BYTES + gemm_bar_bytes(STAGES));  // [BLOCK_N]
  float* s_cs = s_bias + BLOCK_N;                                            // [BLOCK_N] LayerNorm column sums

  const int et = threadIdx.x;  // 0..255
  const int lane = et & 31;
  const int wg = et >> 7;  // warpgroup: tile rows [64 wg, 64 wg + 64)
  const int n_tiles = p.N / BLOCK_N;
  const int n_tile = int(blockIdx.x) % n_tiles;  // n fastest: concurrent CTAs share the A tile through L2
  const int m0 = (int(blockIdx.x) / n_tiles) * GEMM_BLOCK_M;
  const int n0 = n_tile * BLOCK_N;
  // split-K: this CTA owns K-slabs [kb_begin, kb_end)
  const int split = p.k_splits > 1 ? int(blockIdx.y) : 0;
  const int kb_begin = (p.k_splits > 1) ? (int)((long long)split * p.num_kb / p.k_splits) : 0;
  const int kb_end = (p.k_splits > 1) ? (int)((long long)(split + 1) * p.num_kb / p.k_splits) : p.num_kb;

  if (et == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      released[s] = 0u;
    }
    if constexpr (EPI_TMA) tma_prefetch_desc(&tmC);
    fence_barrier_init();
  }
  __syncthreads();

  // one K-slab into its ring slot (one thread): the A box of the slab's tap and the B box of the slab
  auto load_slab = [&](int kb) {
    const int s = (kb - kb_begin) % STAGES;
    const int tap = kb / p.kb_per_tap;
    const int kk = kb - tap * p.kb_per_tap;
    uint8_t* sa = smem + s * STAGE_BYTES;
    mbar_expect_tx(&full_bar[s], STAGE_BYTES);
    tma_load_2d(sa, &tmA, &full_bar[s], kk * GEMM_BLOCK_K, m0 + p.tap_off[tap]);
    tma_load_2d(sa + A_BYTES, &tmB, &full_bar[s], kb * GEMM_BLOCK_K, n0);
  };
  if (et == 0) {
    for (int kb = kb_begin; kb < kb_end && kb < kb_begin + STAGES; ++kb) load_slab(kb);
  }

  // ------------------------------ main loop ------------------------------
  if (p.bias && et < BLOCK_N) s_bias[et] = __ldg(p.bias + n0 + et);
  if (p.ln_stats && et < BLOCK_N) s_cs[et] = __ldg(p.ln_colsum + n0 + et);
  {
    float acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    // issue one K-slab's MMAs as one commit group (every range holds at least one slab)
    auto issue_slab = [&](int kb) {
      const int s = (kb - kb_begin) % STAGES;
      mbar_wait(&full_bar[s], ((kb - kb_begin) / STAGES) & 1);
      const uint32_t sa = smem_u32(smem + s * STAGE_BYTES);
      const uint64_t adesc = make_wgmma_desc(sa + wg * (64 * 128), 16, 1024, 1);
      const uint64_t bdesc = make_wgmma_desc(sa + A_BYTES, 16, 1024, 1);
      wgmma_fence();
      fence_regs(acc);
#pragma unroll
      for (int k = 0; k < GEMM_BLOCK_K / 16; ++k)  // +32 B per K step inside the 128 B swizzle row => +2 in (addr >> 4)
        Wgmma<BLOCK_N, BF16>::ss(acc, adesc + 2 * k, bdesc + 2 * k, 1);
      wgmma_commit();
      fence_regs(acc);
    };
    // The first slab is issued before the loop, so the zeroing above never meets an in-flight MMA at the loop head.
    // Without the peel ptxas sees the accumulators defined both by those moves and by MMAs still in flight, and
    // serialises every wgmma (a full wait after each m64 x BLOCK_N x k16, warning C7515).
    issue_slab(kb_begin);
    for (int kb = kb_begin + 1; kb < kb_end; ++kb) {
      issue_slab(kb);
      wgmma_wait<1>();  // the previous slab's MMAs have retired: this warpgroup releases its slot
      fence_regs(acc);
      // Each use of a slot adds 2 to its counter, one per warpgroup: the leader that finds it odd released last, both
      // warpgroups have read the slot, and that leader refills it. Nobody waits.
      if ((et & 127) == 0 && kb - 1 + STAGES < kb_end) {
        __threadfence_block();
        const uint32_t before = atomicAdd(&released[(kb - 1 - kb_begin) % STAGES], 1u);
        __threadfence_block();
        if (before & 1u) load_slab(kb - 1 + STAGES);
      }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    // every MMA of both warpgroups has read its operands before the ring is overwritten with the accumulators
    named_bar_sync(1, GEMM_THREADS);
    // fragment of m64nN: thread (warp w, lane l) holds rows 16w + l/4 (+8), columns 8j + 2(l%4) (+1)
    const int r0 = wg * 64 + ((et >> 5) & 3) * 16 + (lane >> 2);
    const int cb = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      *reinterpret_cast<float2*>(sacc + r0 * ACC_LD + 8 * j + cb) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(sacc + (r0 + 8) * ACC_LD + 8 * j + cb) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  named_bar_sync(1, GEMM_THREADS);

  // ------------------------------ epilogue -----------------------------------
  const int row = et & 127;
  const int half = et >> 7;  // even (0) / odd (1) 16-column chunks of the row
  const float* arow = sacc + row * ACC_LD;
  const int m = m0 + row;
  bool valid = m < p.M;
  long long orow = m;
  int group = 0;
  if (p.map_mode == 1) {
    const int hw = p.Hm * p.Wm;
    const int img = m / hw;
    const int r = m - img * hw;
    const int i = r / p.Wm;
    const int j = r - i * p.Wm;
    valid = valid && i >= p.i0 && i < p.i0 + p.Hout && j >= p.j0 && j < p.j0 + p.Wout;
    orow = ((long long)img * p.Hout * p.osy + (i - p.i0) * p.osy + p.oa) * (p.Wout * p.osx) + (j - p.j0) * p.osx + p.ob;
    group = img;
  } else if (p.rowbias) {
    group = m / p.rows_per_group;
  }
  if (!valid) group = 0;  // rows past M are computed (and clipped by the TMA store): keep their table reads in bounds
  float ln_a = 1.f, ln_b = 0.f;
  if (p.ln_stats && m < p.M) ln_row_coeffs(p, m, ln_a, ln_b);
  const float* rb_base = p.rowbias ? p.rowbias + (long long)group * p.rowbias_ld + n0 : nullptr;
  auto load16 = [&](int c, float (&o)[16]) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float4 t = *reinterpret_cast<const float4*>(arow + c + 4 * e);
      o[4 * e] = t.x;
      o[4 * e + 1] = t.y;
      o[4 * e + 2] = t.z;
      o[4 * e + 3] = t.w;
    }
  };

  if (p.k_splits > 1) {
    // split-K partial: raw fp32 accumulators, M-space rows (the reduce kernel applies row map + epilogue)
    if (m < p.M) {
      float* wrow = p.ws + ((long long)split * p.M + m) * p.N + n0;
#pragma unroll 1
      for (int ci = half; ci < NCH; ci += 2) {
        float o[16];
        load16(ci * 16, o);
        float4* dst = reinterpret_cast<float4*>(wrow + ci * 16);
#pragma unroll
        for (int e = 0; e < 4; ++e) dst[e] = make_float4(o[4 * e], o[4 * e + 1], o[4 * e + 2], o[4 * e + 3]);
      }
    }
  } else if constexpr (EPI_TMA) {
    // The tile leaves in [128][32] sub-tiles: the two threads of a row fill one 16-column chunk each, thread 0 hands the
    // sub-tile to a TMA store, and the next sub-tile goes to the other staging buffer while that store reads this one.
    static_assert(NCH % 2 == 0, "a sub-tile is one chunk of each of a row's two threads");
    const uint32_t sw = uint32_t((row >> 1) & 3);  // SWIZZLE_64B: 16-byte chunk index ^= address bits [7,9)
    float st_s = 0.f, st_q = 0.f;                   // row statistics of this thread's chunks = slot `half`
    // rows past M are computed and clipped by the TMA store: they read no residual
    const uint16_t* res_row =
        p.residual && m < p.M ? static_cast<const uint16_t*>(p.residual) + (long long)m * p.res_ld + n0 : nullptr;
#pragma unroll 1
    for (int ci = half; ci < NCH; ci += 2) {
      const int c = ci * 16;
      uint4 r0 = make_uint4(0u, 0u, 0u, 0u), r1 = r0;
      if (res_row) {
        r0 = __ldg(reinterpret_cast<const uint4*>(res_row + c));
        r1 = __ldg(reinterpret_cast<const uint4*>(res_row + c) + 1);
      }
      float o[16];
      load16(c, o);
      if (p.ln_stats) {
#pragma unroll
        for (int e = 0; e < 16; ++e) o[e] = fmaf(o[e], ln_a, s_cs[c + e] * ln_b);
      }
      if (p.bias) {
#pragma unroll
        for (int e = 0; e < 16; ++e) o[e] += s_bias[c + e];
      }
      if (rb_base) {
#pragma unroll
        for (int e = 0; e < 16; ++e) o[e] += __ldg(rb_base + c + e);
      }
      if (p.act == PF_ACT_SILU) {
#pragma unroll
        for (int e = 0; e < 16; ++e) o[e] = silu_f(o[e]);
      } else if (p.act == PF_ACT_GELU) {
#pragma unroll
        for (int e = 0; e < 16; ++e) o[e] = gelu_erf_f(o[e]);
      } else if (p.act == PF_ACT_QUICK_GELU) {
#pragma unroll
        for (int e = 0; e < 16; ++e) o[e] = quick_gelu_f(o[e]);
      }
      const int sub = c >> 5;
      uint8_t* sbuf = staging + (sub & 1) * GEMM_SUB_BYTES;
      uint8_t* srow = sbuf + row * 64;
      const uint32_t q0 = uint32_t((c >> 4) & 1) * 2;  // first 16-byte chunk of this 16-column group in the 64 B row
      uint4* s0 = reinterpret_cast<uint4*>(srow + (((q0 + 0) ^ sw) << 4));
      uint4* s1 = reinterpret_cast<uint4*>(srow + (((q0 + 1) ^ sw) << 4));
      if (p.residual) {  // rows past M add the zeros above
        float2 f;
        f = unpack2<BF16>(r0.x); o[0] += f.x; o[1] += f.y;
        f = unpack2<BF16>(r0.y); o[2] += f.x; o[3] += f.y;
        f = unpack2<BF16>(r0.z); o[4] += f.x; o[5] += f.y;
        f = unpack2<BF16>(r0.w); o[6] += f.x; o[7] += f.y;
        f = unpack2<BF16>(r1.x); o[8] += f.x; o[9] += f.y;
        f = unpack2<BF16>(r1.y); o[10] += f.x; o[11] += f.y;
        f = unpack2<BF16>(r1.z); o[12] += f.x; o[13] += f.y;
        f = unpack2<BF16>(r1.w); o[14] += f.x; o[15] += f.y;
      }
      if (p.row_stats) {
#pragma unroll
        for (int e = 0; e < 16; ++e) {
          st_s += o[e];
          st_q = fmaf(o[e], o[e], st_q);
        }
      }
      *s0 = make_uint4(pack2<BF16>(o[0], o[1]), pack2<BF16>(o[2], o[3]), pack2<BF16>(o[4], o[5]),
                       pack2<BF16>(o[6], o[7]));
      *s1 = make_uint4(pack2<BF16>(o[8], o[9]), pack2<BF16>(o[10], o[11]), pack2<BF16>(o[12], o[13]),
                       pack2<BF16>(o[14], o[15]));
      fence_proxy_async_smem();  // generic-proxy writes -> visible to the TMA store
      // the previous sub-tile's store has read its buffer before anyone passes this barrier and refills it
      if (et == 0) tma_store_wait_read();
      named_bar_sync(1, GEMM_THREADS);
      if (et == 0) {
        tma_store_2d(&tmC, sbuf, n0 + sub * 32, m0);
        tma_store_commit();
      }
    }
    if (p.row_stats && m < p.M)
      reinterpret_cast<float2*>(p.row_stats)[(long long)m * p.stat_slots + n_tile * 2 + half] = make_float2(st_s, st_q);
    if (et == 0) tma_store_wait_read();  // shared memory must outlive the last store's reads
  } else if (p.act == PF_ACT_GEGLU) {
    constexpr int HALF_N = BLOCK_N / 2;
    const int on0 = n_tile * HALF_N;
    if constexpr (HALF_N % 16 == 0) {
#pragma unroll 1
      for (int c = half * 16; c < HALF_N; c += 32) {
        if (!valid) break;
        float va[16], vg[16], o[16], ba[16], bg[16];
        load16(c, va);
        load16(HALF_N + c, vg);
        if (p.bias) {  // HALF_N and c are multiples of 16: 128-bit shared-memory loads
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            *reinterpret_cast<float4*>(ba + 4 * e) = *reinterpret_cast<const float4*>(s_bias + c + 4 * e);
            *reinterpret_cast<float4*>(bg + 4 * e) = *reinterpret_cast<const float4*>(s_bias + HALF_N + c + 4 * e);
          }
        } else {
#pragma unroll
          for (int e = 0; e < 16; ++e) ba[e] = bg[e] = 0.f;
        }
        if (p.ln_stats) {
#pragma unroll
          for (int e = 0; e < 16; ++e) {
            va[e] = fmaf(va[e], ln_a, s_cs[c + e] * ln_b);
            vg[e] = fmaf(vg[e], ln_a, s_cs[HALF_N + c + e] * ln_b);
          }
        }
#pragma unroll
        for (int e = 0; e < 16; e += 2)
          geglu_pair(va[e], va[e + 1], vg[e], vg[e + 1], ba[e], ba[e + 1], bg[e], bg[e + 1], o[e], o[e + 1]);
        if (p.out_f32) {
          float4* dst = reinterpret_cast<float4*>(static_cast<float*>(p.out) + orow * p.out_ld + on0 + c);
#pragma unroll
          for (int e = 0; e < 4; ++e) dst[e] = make_float4(o[4 * e], o[4 * e + 1], o[4 * e + 2], o[4 * e + 3]);
        } else {
          uint4* dst = reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.out) + orow * p.out_ld + on0 + c);
          dst[0] = make_uint4(pack2<BF16>(o[0], o[1]), pack2<BF16>(o[2], o[3]), pack2<BF16>(o[4], o[5]),
                              pack2<BF16>(o[6], o[7]));
          dst[1] = make_uint4(pack2<BF16>(o[8], o[9]), pack2<BF16>(o[10], o[11]), pack2<BF16>(o[12], o[13]),
                              pack2<BF16>(o[14], o[15]));
        }
      }
    }
  } else if (valid) {
    // direct stores (convolutions: halo-dropping row map; fp32 outputs)
#pragma unroll 1
    for (int ci = half; ci < NCH; ci += 2) {
      const int c = ci * 16;
      float o[16];
      load16(c, o);
      if (p.bias) {
#pragma unroll
        for (int e = 0; e < 16; ++e) o[e] += s_bias[c + e];
      }
      if (rb_base) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float4 t = __ldg(reinterpret_cast<const float4*>(rb_base + c) + e);
          o[4 * e] += t.x;
          o[4 * e + 1] += t.y;
          o[4 * e + 2] += t.z;
          o[4 * e + 3] += t.w;
        }
      }
      if (p.act == PF_ACT_SILU) {
#pragma unroll
        for (int e = 0; e < 16; ++e) o[e] = silu_f(o[e]);
      } else if (p.act == PF_ACT_GELU) {
#pragma unroll
        for (int e = 0; e < 16; ++e) o[e] = gelu_erf_f(o[e]);
      } else if (p.act == PF_ACT_QUICK_GELU) {
#pragma unroll
        for (int e = 0; e < 16; ++e) o[e] = quick_gelu_f(o[e]);
      }
      if (p.residual) {
        if (p.res_f32) {
          const float4* r4 =
              reinterpret_cast<const float4*>(static_cast<const float*>(p.residual) + orow * p.res_ld + n0 + c);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float4 t = r4[e];
            o[4 * e] += t.x;
            o[4 * e + 1] += t.y;
            o[4 * e + 2] += t.z;
            o[4 * e + 3] += t.w;
          }
        } else {
          const uint4* r16 =
              reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(p.residual) + orow * p.res_ld + n0 + c);
          const uint4 r0 = __ldg(r16), r1 = __ldg(r16 + 1);
          float2 f;
          f = unpack2<BF16>(r0.x); o[0] += f.x; o[1] += f.y;
          f = unpack2<BF16>(r0.y); o[2] += f.x; o[3] += f.y;
          f = unpack2<BF16>(r0.z); o[4] += f.x; o[5] += f.y;
          f = unpack2<BF16>(r0.w); o[6] += f.x; o[7] += f.y;
          f = unpack2<BF16>(r1.x); o[8] += f.x; o[9] += f.y;
          f = unpack2<BF16>(r1.y); o[10] += f.x; o[11] += f.y;
          f = unpack2<BF16>(r1.z); o[12] += f.x; o[13] += f.y;
          f = unpack2<BF16>(r1.w); o[14] += f.x; o[15] += f.y;
        }
      }
      if (p.out_f32) {
        float4* dst = reinterpret_cast<float4*>(static_cast<float*>(p.out) + orow * p.out_ld + n0 + c);
#pragma unroll
        for (int e = 0; e < 4; ++e) dst[e] = make_float4(o[4 * e], o[4 * e + 1], o[4 * e + 2], o[4 * e + 3]);
      } else {
        uint4* dst = reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.out) + orow * p.out_ld + n0 + c);
        dst[0] = make_uint4(pack2<BF16>(o[0], o[1]), pack2<BF16>(o[2], o[3]), pack2<BF16>(o[4], o[5]),
                            pack2<BF16>(o[6], o[7]));
        dst[1] = make_uint4(pack2<BF16>(o[8], o[9]), pack2<BF16>(o[10], o[11]), pack2<BF16>(o[12], o[13]),
                            pack2<BF16>(o[14], o[15]));
      }
    }
  }
}

// split-K reduce: fixed-order sum of the k_splits partials, then the same epilogue as the in-kernel one
// (bias, per-image row bias, activation, residual, halo-dropping row map). thread <-> (M-space row, 8 columns)
template <bool BF16>
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const GemmKernelParams p) {
  const int vecs = p.N / 8;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)p.M * vecs) return;
  const int m = int(idx / vecs), c = int(idx % vecs) * 8;
  bool valid = true;
  long long orow = m;
  int group = 0;
  if (p.map_mode == 1) {
    const int hw = p.Hm * p.Wm;
    const int img = m / hw;
    const int r = m - img * hw;
    const int i = r / p.Wm;
    const int j = r - i * p.Wm;
    valid = i >= p.i0 && i < p.i0 + p.Hout && j >= p.j0 && j < p.j0 + p.Wout;
    orow = ((long long)img * p.Hout * p.osy + (i - p.i0) * p.osy + p.oa) * (p.Wout * p.osx) + (j - p.j0) * p.osx + p.ob;
    group = img;
  } else if (p.rowbias) {
    group = m / p.rows_per_group;
  }
  if (!valid) return;
  float o[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) o[e] = 0.f;
  for (int sp = 0; sp < p.k_splits; ++sp) {
    const float4* w4 = reinterpret_cast<const float4*>(p.ws + ((long long)sp * p.M + m) * p.N + c);
    const float4 a = __ldcs(w4), b = __ldcs(w4 + 1);
    o[0] += a.x; o[1] += a.y; o[2] += a.z; o[3] += a.w;
    o[4] += b.x; o[5] += b.y; o[6] += b.z; o[7] += b.w;
  }
  if (p.bias) {
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] += __ldg(p.bias + c + e);
  }
  if (p.rowbias) {
    const float* rb = p.rowbias + (long long)group * p.rowbias_ld + c;
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] += __ldg(rb + e);
  }
  if (p.act == PF_ACT_SILU) {
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = silu_f(o[e]);
  } else if (p.act == PF_ACT_GELU) {
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = gelu_erf_f(o[e]);
  } else if (p.act == PF_ACT_QUICK_GELU) {
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = quick_gelu_f(o[e]);
  }
  if (p.residual) {
    if (p.res_f32) {
      const float4* r4 = reinterpret_cast<const float4*>(static_cast<const float*>(p.residual) + orow * p.res_ld + c);
      const float4 a = r4[0], b = r4[1];
      o[0] += a.x; o[1] += a.y; o[2] += a.z; o[3] += a.w;
      o[4] += b.x; o[5] += b.y; o[6] += b.z; o[7] += b.w;
    } else {
      const uint4 t = *reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(p.residual) + orow * p.res_ld + c);
      float2 f;
      f = unpack2<BF16>(t.x); o[0] += f.x; o[1] += f.y;
      f = unpack2<BF16>(t.y); o[2] += f.x; o[3] += f.y;
      f = unpack2<BF16>(t.z); o[4] += f.x; o[5] += f.y;
      f = unpack2<BF16>(t.w); o[6] += f.x; o[7] += f.y;
    }
  }
  if (p.out_f32) {
    float4* dst = reinterpret_cast<float4*>(static_cast<float*>(p.out) + orow * p.out_ld + c);
    dst[0] = make_float4(o[0], o[1], o[2], o[3]);
    dst[1] = make_float4(o[4], o[5], o[6], o[7]);
  } else {
    *reinterpret_cast<uint4*>(static_cast<uint16_t*>(p.out) + orow * p.out_ld + c) =
        make_uint4(pack2<BF16>(o[0], o[1]), pack2<BF16>(o[2], o[3]), pack2<BF16>(o[4], o[5]), pack2<BF16>(o[6], o[7]));
  }
}

// CTAS: CTAs per SM the instantiation is built for (register cap of the build, shared-memory budget, checked below)
template <int BLOCK_N, int STAGES, int CTAS, bool EPI_TMA>
static int launch_gemm(const pf_gemm_args* a, const GemmKernelParams& kp, cudaStream_t st) {
  CUtensorMap tmA, tmB, tmC;
  {
    uint64_t dims[2] = {(uint64_t)a->Kc, (uint64_t)a->a_rows};
    uint64_t str[1] = {(uint64_t)a->a_ld * 2};
    uint32_t box[2] = {GEMM_BLOCK_K, GEMM_BLOCK_M};
    int rc = make_tmap(&tmA, a->dtype, 2, a->A, dims, str, box, 128);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {(uint64_t)a->Kc * a->num_taps, (uint64_t)a->N};
    uint64_t str[1] = {(uint64_t)a->b_ld * 2};
    uint32_t box[2] = {GEMM_BLOCK_K, (uint32_t)BLOCK_N};
    int rc = make_tmap(&tmB, a->dtype, 2, a->B, dims, str, box, 128);
    if (rc) return rc;
  }
  tmC = tmA;
  if constexpr (EPI_TMA) {
    uint64_t dims[2] = {(uint64_t)a->N, (uint64_t)a->M};
    uint32_t box[2] = {32, GEMM_BLOCK_M};
    uint64_t str[1] = {(uint64_t)a->out_ld * 2};
    int rc = make_tmap(&tmC, a->dtype, 2, a->out, dims, str, box, 64);
    if (rc) return rc;
  }
  constexpr int SMEM = gemm_smem_bytes(BLOCK_N, STAGES, EPI_TMA);
  static_assert(SMEM <= 227 * 1024, "shared memory budget of one H100 CTA");
  static_assert(CTAS == 1 || SMEM <= GEMM_SMEM_CORESIDENT, "two CTAs per SM: 113 KB of shared memory each");
  const int m_tiles = (a->M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M;
  const dim3 grid(m_tiles * (a->N / BLOCK_N), kp.k_splits > 1 ? kp.k_splits : 1);
  const int bf = a->dtype == PF_BF16;
  auto kern = bf ? gemm_taps_kernel<BLOCK_N, STAGES, CTAS, true, EPI_TMA>
                 : gemm_taps_kernel<BLOCK_N, STAGES, CTAS, false, EPI_TMA>;
  static bool attr_set[2] = {false, false};  // per dtype: the two kernels share this function's statics
  if (!attr_set[bf]) {
    int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM),
                        "cudaFuncSetAttribute(gemm)");
    if (rc) return rc;
    // the registers and shared memory this build came out with must admit the CTAs per SM the schedule relies on
    int resident = 0;
    rc = check_cuda(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern, GEMM_THREADS, SMEM),
                    "cudaOccupancyMaxActiveBlocksPerMultiprocessor(gemm)");
    if (rc) return rc;
    if (resident < CTAS) {
      set_error("gemm_taps_kernel<%d, %d, %s>: %d CTA(s) per SM fit, built for %d", BLOCK_N, STAGES,
                EPI_TMA ? "tma" : "direct", resident, CTAS);
      return PF_ERR_UNSUPPORTED;
    }
    attr_set[bf] = true;
  }
  kern<<<grid, GEMM_THREADS, SMEM, st>>>(tmA, tmB, tmC, kp);
  PF_CHECK_LAUNCH("gemm_taps_kernel");
  return PF_OK;
}

// tile width pf_gemm_taps runs with: the caller's request, else the heuristic; the staged (TMA-store) epilogue
// that carries the fused-LayerNorm statistics has no 256-wide variant
static int resolve_block_n(const pf_gemm_args* a) {
  int bn = (a->block_n & 0xffff) ? (a->block_n & 0xffff) : pf_gemm_pick_block_n(a->N, a->act);
  // a statistics PRODUCER always uses the width the heuristic derives from N: the slot partition of the row sums (and so
  // their fp32 rounding) must not depend on M-specific tuning, or a sharded rank would not reproduce the full batch
  if (a->row_stats_out) bn = pf_gemm_pick_block_n(a->N, a->act);
  if ((a->row_stats_out || a->ln_stats) && a->act != PF_ACT_GEGLU && bn == 256) bn = 128;
  return bn;
}

}  // namespace pf

extern "C" int pf_gemm_row_stats_slots(const pf_gemm_args* a) {
  if (!a || a->N <= 0) return 0;
  pf_gemm_args producer = *a;  // the question is about a PRODUCER, whether or not the caller has set row_stats_out yet
  static float dummy;
  producer.row_stats_out = &dummy;
  const int bn = pf::resolve_block_n(&producer);
  return bn > 0 && a->N % bn == 0 ? 2 * (a->N / bn) : 0;
}

extern "C" int pf_gemm_pick_block_n(int N, int act) {
  // GEGLU tiles are epilogue-bound (one erf-GELU per output): the 256-wide tile halves the per-tile fixed cost
  if (act == PF_ACT_GEGLU && N % 256 == 0) return 256;
  if (N % 160 == 0) return 160;
  if (N % 128 == 0) return 128;
  if (N % 64 == 0) return 64;
  return 0;
}

extern "C" int pf_gemm_splitk_plan(const pf_gemm_args* a) {
  if (!a || a->act == PF_ACT_GEGLU || a->M <= 0 || a->N <= 0 || a->Kc <= 0) return 1;
  const int bn = pf_gemm_pick_block_n(a->N, a->act);
  if (!bn) return 1;
  const long long tiles = (long long)((a->M + 127) / 128) * (a->N / bn);
  const int num_kb = a->Kc / 64 * a->num_taps;
  const int sms = pf::sm_count();
  // Only the skinny deep-K problems: a sharded rank's 8x8 / 16x16-level convolutions have few output tiles and 90-360
  // K-slabs, i.e. a handful of SMs each streaming megabytes of weights at the per-SM L2 rate. Shapes that already cover
  // half the machine, or short K, lose more to the partial-sum traffic than they gain.
  if (tiles > sms / 2 || num_kb < 64) return 1;
  int s = (int)((sms + tiles - 1) / tiles);           // aim for ~1 CTA per SM
  const int max_by_k = num_kb / 16;                   // >= 16 K-slabs per split
  if (s > max_by_k) s = max_by_k;
  if (s > 16) s = 16;
  return s < 2 ? 1 : s;
}

extern "C" int pf_gemm_taps(const pf_gemm_args* a, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(a != nullptr, "pf_gemm_taps: null args");
  PF_CHECK_ARG(a->dtype == PF_BF16 || a->dtype == PF_F16, "pf_gemm_taps: dtype must be PF_F16 or PF_BF16");
  PF_CHECK_ARG(a->A && a->B && a->out, "pf_gemm_taps: null operand");
  PF_CHECK_ARG(a->M > 0 && a->N > 0 && a->Kc > 0, "pf_gemm_taps: empty problem M=%d N=%d Kc=%d", a->M, a->N, a->Kc);
  PF_CHECK_ARG(a->Kc % GEMM_BLOCK_K == 0, "pf_gemm_taps: Kc=%d must be a multiple of 64", a->Kc);
  PF_CHECK_ARG(a->num_taps >= 1 && a->num_taps <= PF_MAX_TAPS, "pf_gemm_taps: num_taps=%d out of range", a->num_taps);
  PF_CHECK_ARG(a->a_ld % 8 == 0 && a->b_ld % 8 == 0 && a->a_ld >= a->Kc && a->b_ld >= a->Kc * a->num_taps,
               "pf_gemm_taps: bad leading dims a_ld=%d b_ld=%d", a->a_ld, a->b_ld);
  PF_CHECK_ARG((reinterpret_cast<uintptr_t>(a->A) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->B) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(a->out) & 15) == 0,
               "pf_gemm_taps: operands must be 16-byte aligned");
  // the epilogues and the split-K reduce read / write these with 16-byte (row statistics: 8-byte) vector accesses
  PF_CHECK_ARG((reinterpret_cast<uintptr_t>(a->residual) & 15) == 0, "pf_gemm_taps: residual must be 16-byte aligned");
  PF_CHECK_ARG(!a->rowbias || ((reinterpret_cast<uintptr_t>(a->rowbias) & 15) == 0 && a->rowbias_ld % 4 == 0),
               "pf_gemm_taps: rowbias must be 16-byte aligned with rowbias_ld %% 4 == 0 (rowbias_ld=%d)", a->rowbias_ld);
  PF_CHECK_ARG((reinterpret_cast<uintptr_t>(a->splitk_ws) & 15) == 0, "pf_gemm_taps: splitk_ws must be 16-byte aligned");
  PF_CHECK_ARG((reinterpret_cast<uintptr_t>(a->row_stats_out) & 7) == 0,
               "pf_gemm_taps: row_stats_out must be 8-byte aligned");
  PF_CHECK_ARG(a->out_dtype == PF_F32 || a->out_dtype == a->dtype, "pf_gemm_taps: out_dtype must be f32 or dtype");
  PF_CHECK_ARG(!a->residual || a->res_dtype == PF_F32 || a->res_dtype == a->dtype,
               "pf_gemm_taps: res_dtype must be f32 or dtype");
  PF_CHECK_ARG(a->act >= PF_ACT_NONE && a->act <= PF_ACT_QUICK_GELU, "pf_gemm_taps: unknown act %d", a->act);
  // block_n: low 16 bits = tile width (0 = auto); the high bits are ignored (one schedule)
  int bn = pf::resolve_block_n(a);
  PF_CHECK_ARG(bn == 64 || bn == 128 || bn == 160 || bn == 256, "pf_gemm_taps: unsupported block_n %d (N=%d)", bn, a->N);
  PF_CHECK_ARG(a->N % bn == 0, "pf_gemm_taps: N=%d not a multiple of block_n=%d", a->N, bn);
  const int n_out = a->act == PF_ACT_GEGLU ? a->N / 2 : a->N;
  PF_CHECK_ARG(a->out_ld % 8 == 0 && a->out_ld >= n_out, "pf_gemm_taps: bad out_ld %d", a->out_ld);
  PF_CHECK_ARG(!a->residual || (a->res_ld % 8 == 0 && a->res_ld >= n_out), "pf_gemm_taps: bad res_ld %d", a->res_ld);
  PF_CHECK_ARG(!(a->act == PF_ACT_GEGLU && (a->residual || a->rowbias)),
               "pf_gemm_taps: GEGLU epilogue takes no residual/rowbias");
  if (a->map_mode == 1) {
    PF_CHECK_ARG(a->Hm > 0 && a->Wm > 0 && a->Hout > 0 && a->Wout > 0 && a->M % (a->Hm * a->Wm) == 0,
                 "pf_gemm_taps: bad image map Hm=%d Wm=%d M=%d", a->Hm, a->Wm, a->M);
    PF_CHECK_ARG(a->out_sy >= 0 && a->out_sx >= 0 && a->out_a >= 0 && a->out_b >= 0 &&
                     a->out_a < (a->out_sy > 0 ? a->out_sy : 1) && a->out_b < (a->out_sx > 0 ? a->out_sx : 1),
                 "pf_gemm_taps: bad output scatter (%d,%d) phase (%d,%d)", a->out_sy, a->out_sx, a->out_a, a->out_b);
    PF_CHECK_ARG((a->out_sy <= 1 && a->out_sx <= 1) || !a->residual, "pf_gemm_taps: the scattered output map takes no residual");
  } else {
    PF_CHECK_ARG(a->map_mode == 0, "pf_gemm_taps: unknown map_mode %d", a->map_mode);
    PF_CHECK_ARG(!a->rowbias || a->rows_per_group > 0, "pf_gemm_taps: rowbias needs rows_per_group");
  }

  GemmKernelParams kp;
  kp.M = a->M;
  kp.N = a->N;
  kp.kb_per_tap = a->Kc / GEMM_BLOCK_K;
  kp.num_kb = kp.kb_per_tap * a->num_taps;
  for (int t = 0; t < PF_MAX_TAPS; ++t) kp.tap_off[t] = t < a->num_taps ? a->tap_off[t] : 0;
  kp.out = a->out;
  kp.out_ld = a->out_ld;
  kp.out_f32 = a->out_dtype == PF_F32;
  kp.bias = a->bias;
  kp.rowbias = a->rowbias;
  kp.rowbias_ld = a->rowbias_ld;
  kp.rows_per_group = a->rows_per_group > 0 ? a->rows_per_group : 1;
  kp.residual = a->residual;
  kp.res_ld = a->res_ld;
  kp.res_f32 = a->res_dtype == PF_F32;
  kp.act = a->act;
  kp.map_mode = a->map_mode;
  kp.Hm = a->Hm;
  kp.Wm = a->Wm;
  kp.i0 = a->i0;
  kp.j0 = a->j0;
  kp.Hout = a->Hout;
  kp.Wout = a->Wout;
  kp.osy = a->out_sy > 0 ? a->out_sy : 1;
  kp.osx = a->out_sx > 0 ? a->out_sx : 1;
  kp.oa = a->out_a;
  kp.ob = a->out_b;
  kp.k_splits = a->k_splits > 1 ? a->k_splits : 1;
  kp.ws = a->splitk_ws;
  kp.row_stats = a->row_stats_out;
  kp.stat_slots = 2 * (a->N / bn);
  kp.ln_stats = a->ln_stats;
  kp.ln_slots = a->ln_slots;
  kp.ln_colsum = a->ln_colsum;
  kp.ln_inv_k = 1.0f / float((long long)a->Kc * a->num_taps);
  kp.ln_eps = a->ln_eps;
  PF_CHECK_ARG(kp.k_splits == 1 || (a->splitk_ws && a->act != PF_ACT_GEGLU && kp.k_splits <= kp.num_kb),
               "pf_gemm_taps: split-K needs a workspace, no GEGLU and k_splits <= K-slabs");
  const bool fused_ln = a->row_stats_out || a->ln_stats;
  if (fused_ln) {
    PF_CHECK_ARG(kp.k_splits == 1, "pf_gemm_taps: fused LayerNorm does not combine with split-K");
    PF_CHECK_ARG(!a->ln_stats || (a->ln_colsum && a->ln_slots > 0 && a->ln_slots % 2 == 0 && a->ln_eps > 0.f &&
                                  (reinterpret_cast<uintptr_t>(a->ln_stats) & 15) == 0),
                 "pf_gemm_taps: ln_stats needs ln_colsum, ln_slots and ln_eps");
    const bool plain16 = a->map_mode == 0 && a->out_dtype == a->dtype && (!a->residual || a->res_dtype == a->dtype);
    PF_CHECK_ARG(a->act == PF_ACT_GEGLU ? !a->row_stats_out : plain16,
                 "pf_gemm_taps: fused LayerNorm needs the plain row map with 16-bit output (consumer: or GEGLU)");
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (kp.k_splits > 1) {
    int rc;
    switch (bn) {
      // few tiles of 90-360 K-slabs, planned at about one CTA per SM: nothing to co-schedule, so the long rings
      case 64: rc = launch_gemm<64, 8, 1, false>(a, kp, st); break;
      case 128: rc = launch_gemm<128, 6, 1, false>(a, kp, st); break;
      case 160: rc = launch_gemm<160, 5, 1, false>(a, kp, st); break;
      default: rc = launch_gemm<256, 4, 1, false>(a, kp, st); break;
    }
    if (rc) return rc;
    const long long total = (long long)a->M * (a->N / 8);
    if (a->dtype == PF_BF16) splitk_reduce_kernel<true><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(kp);
    else splitk_reduce_kernel<false><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(kp);
    PF_CHECK_LAUNCH("splitk_reduce_kernel");
    return PF_OK;
  }
  // staged TMA-store epilogue: plain row map, 16-bit output, 16-bit (or no) residual, no GEGLU
  const bool epi_tma = a->map_mode == 0 && a->out_dtype == a->dtype && a->act != PF_ACT_GEGLU &&
                       (!a->residual || a->res_dtype == a->dtype) && bn != 256;
  if (epi_tma) {
    switch (bn) {
      case 64: return launch_gemm<64, 4, 2, true>(a, kp, st);
      case 128: return launch_gemm<128, 3, 2, true>(a, kp, st);
      case 160: return launch_gemm<160, 3, 2, true>(a, kp, st);
    }
  }
  switch (bn) {
    case 64: return launch_gemm<64, 4, 2, false>(a, kp, st);
    case 128: return launch_gemm<128, 3, 2, false>(a, kp, st);
    case 160: return launch_gemm<160, 3, 2, false>(a, kp, st);
    case 256: return launch_gemm<256, 4, 1, false>(a, kp, st);
  }
  return PF_ERR_UNSUPPORTED;
}
