// Tap-GEMM on Hopper: TMA (SWIZZLE_128B) -> shared-memory ring -> wgmma (m64 x BLOCK_N x k16 per warpgroup, fp32 in
// registers) -> epilogue. It runs every pf_gemm_taps call the persistent linear GEMM (gemm_linear.cu) does not take:
// the 3x3 convolutions and Upsample2D / Downsample2D phase convolutions of the UNet walk, fp32 outputs, row bias and
// split-K (reference call sites: models/pano/MVGenModel.py:85-295 through diffusers ResnetBlock2D /
// Transformer2DModel). A convolution is a sum of `num_taps` GEMMs whose A operand is the same channels-last image
// shifted by a constant row offset (zero-haloed "padded-flat" layout), so the im2col matrix is never formed. Taps whose
// offsets lie within GEMM_WIN_SPAN (8) rows of each other (the three taps of a 3x3 kernel row) read one A window of
// 128 + 8 rows, fetched once per 64-channel slab with one 2-D TMA box, and each tap's wgmma A operand starts 0..8 rows
// into it; only the B box is fetched per tap. A 3x3 convolution's tile so reads each A row 3 times per channel slab
// from L2 instead of 9. A GEMM whose taps are all further apart (1x1 convolutions, single-tap GEMMs) runs the plain
// slab ring: one A box and one B box per K-slab behind one barrier.
//
// 256 threads: warps 0..3 and 4..7 = two warpgroups, each owning 64 of the 128 tile rows through the main loop.
// There is no producer warp: thread 0 fills the ring before the loop, and the leader of whichever warpgroup releases
// a slot last issues the slot's next TMA loads, so no MMA-issuing warp ever blocks on the other warpgroup. After the
// last K-slab the accumulators are written to shared memory (over the now idle operand ring) and all 256 threads run
// the epilogue with two threads per tile row (even / odd 16-column chunks). It has two forms: raw fp32 split-K
// partials, or bias / per-image row bias / SiLU / GELU / QuickGELU / residual stored directly through the
// halo-dropping row map.
//
// Instantiations with a short ring (CTAS = 2) run TWO CTAs per SM (at most 128 registers per thread and 113 KB of
// shared memory per CTA): a tile has no overlap of its own between ring fill, main loop, accumulator dump and
// epilogue, so the tensor pipe is kept busy by the other CTA's main loop while one CTA fills or drains. A ninth
// (producer) warp would rule that out: registers are granted to whole warps, nine warps would leave two CTAs 96
// registers per thread, and the 160-wide tile alone holds 80 accumulators. Split-K, which is planned at about one CTA
// per SM, keeps a long ring and CTAS = 1.
#include <stdlib.h>

#include "gemm_common.cuh"
#include "wgmma.cuh"

namespace pf {

constexpr int GEMM_THREADS = 256;

// an SM has 228 KB of shared memory and every resident CTA reserves 1 KB of it
constexpr int GEMM_SMEM_CORESIDENT = 228 * 1024 / 2 - 1024;

__host__ __device__ constexpr int gemm_acc_ld(int block_n) { return block_n + 4; }  // floats; +4: conflict-free rows
// the operand ring; after the main loop the same bytes hold the [128][acc_ld] fp32 accumulators
__host__ __device__ constexpr int gemm_ring_bytes(int block_n, int stages) {
  const int ring = stages * gemm_stage_bytes(block_n);
  const int acc = GEMM_BLOCK_M * gemm_acc_ld(block_n) * 4;
  return ((ring > acc ? ring : acc) + 1023) / 1024 * 1024;
}
// full barrier (8 bytes) and release counter (4 bytes) per A slot and per B slot (at most STAGES of each), rounded up
// to keep s_bias 16-byte aligned
__host__ __device__ constexpr int gemm_bar_bytes(int stages) { return (2 * stages * 12 + 15) / 16 * 16; }
__host__ __device__ constexpr int gemm_smem_bytes(int block_n, int stages) {
  return gemm_ring_bytes(block_n, stages) + gemm_bar_bytes(stages) + block_n * 4 /*bias row*/;
}

template <int BLOCK_N, int STAGES, int CTAS, bool BF16>
__global__ void __launch_bounds__(GEMM_THREADS, CTAS)
gemm_taps_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmKernelParams p) {
  constexpr int B_BYTES = BLOCK_N * GEMM_BLOCK_K * 2;
  constexpr int RING_BYTES = gemm_ring_bytes(BLOCK_N, STAGES);
  constexpr int ACC_LD = gemm_acc_ld(BLOCK_N);
  constexpr int NCH = BLOCK_N / 16;
  constexpr int NACC = BLOCK_N / 2;  // fp32 accumulators per thread of an m64 x BLOCK_N warpgroup tile
  static_assert(BLOCK_N % 32 == 0 && BLOCK_N <= 160, "tile width");

  // 1024-byte alignment (128 B swizzle atoms) is requested on the declaration; verified once, never padded for
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  float* sacc = reinterpret_cast<float*>(smem);  // [128][ACC_LD] fp32, over the ring once the main loop is done
  // the ring: p.a_slots A windows, then STAGES B boxes (1024-byte multiples, so every slot is swizzle-aligned)
  const int a_bytes = p.a_rows * (GEMM_BLOCK_K * 2);
  uint8_t* const b_ring = smem + p.a_slots * a_bytes;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + RING_BYTES);
  uint64_t* b_full = a_full + STAGES;
  uint32_t* a_rel = reinterpret_cast<uint32_t*>(b_full + STAGES);  // per slot: releases by the two warpgroups
  uint32_t* b_rel = a_rel + STAGES;
  float* s_bias = reinterpret_cast<float*>(smem + RING_BYTES + gemm_bar_bytes(STAGES));  // [BLOCK_N]

  const int et = threadIdx.x;  // 0..255
  const int lane = et & 31;
  const int wg = et >> 7;  // warpgroup: tile rows [64 wg, 64 wg + 64)
  const int n_tiles = p.N / BLOCK_N;
  const int n_tile = int(blockIdx.x) % n_tiles;  // n fastest: concurrent CTAs share the A tile through L2
  const int m0 = (int(blockIdx.x) / n_tiles) * GEMM_BLOCK_M;
  const int n0 = n_tile * BLOCK_N;
  const int kpt = p.kb_per_tap;
  // split-K: this CTA owns units [u_begin, u_end), i.e. K-slabs [s_begin, s_end)
  const int split = p.k_splits > 1 ? int(blockIdx.y) : 0;
  const int u_begin = (p.k_splits > 1) ? (int)((long long)split * p.num_units / p.k_splits) : 0;
  const int u_end = (p.k_splits > 1) ? (int)((long long)(split + 1) * p.num_units / p.k_splits) : p.num_units;
  auto first_slab = [&](int u) {  // K-slab of unit u's first tap (u = num_units: the end of K)
    const int gu = u / kpt, ku = u - gu * kpt;
    return p.grp_first[gu] * kpt + (ku ? ku * (p.grp_first[gu + 1] - p.grp_first[gu]) : 0);
  };
  const int s_begin = first_slab(u_begin), s_end = first_slab(u_end);

  if (et == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&b_full[s], 1);
      a_rel[s] = b_rel[s] = 0u;
    }
    fence_barrier_init();
  }
  __syncthreads();

  // Where K-slab s sits in the K order: sorted tap i of group g at channel slab kk. The main loop never calls this: it
  // walks the order incrementally, so no division or table search lies between two slabs' MMAs.
  auto locate = [&](int s, int& gs, int& ks, int& is) {
    gs = 0;
    while (s >= p.grp_first[gs + 1] * kpt) ++gs;
    const int taps = p.grp_first[gs + 1] - p.grp_first[gs];
    const int r = s - p.grp_first[gs] * kpt;
    ks = r / taps;
    is = p.grp_first[gs] + r - ks * taps;
  };
  // One thread each: the A window of group ga at channel slab ka, and the B box of sorted tap ib at channel slab kb
  // (group gb). In a slab ring (every group a single tap, so units are slabs) a slab's A box and B box share slot and
  // barrier, and the A barriers and counters stay unused.
  auto load_a = [&](int slot, int ga, int ka, uint64_t* bar) {
    tma_load_2d(smem + slot * a_bytes, &tmA, bar, ka * GEMM_BLOCK_K, m0 + p.grp_off[ga]);
  };
  auto fill_a = [&](int slot, int ga, int ka) {
    mbar_expect_tx(&a_full[slot], a_bytes);
    load_a(slot, ga, ka, &a_full[slot]);
  };
  auto fill_b = [&](int slot, int gb, int kb, int ib) {
    mbar_expect_tx(&b_full[slot], B_BYTES + (p.slab_ring ? a_bytes : 0));
    if (p.slab_ring) load_a(slot, gb, kb, &b_full[slot]);
    tma_load_2d(b_ring + slot * B_BYTES, &tmB, &b_full[slot], (p.tap_src[ib] * kpt + kb) * GEMM_BLOCK_K, n0);
  };
  if (et == 0) {
    if (!p.slab_ring)
      for (int k = 0; k < p.a_slots && u_begin + k < u_end; ++k) {
        const int gu = (u_begin + k) / kpt;
        fill_a(k, gu, u_begin + k - gu * kpt);
      }
    for (int k = 0; k < STAGES && s_begin + k < s_end; ++k) {
      int gs, ks, is;
      locate(s_begin + k, gs, ks, is);
      fill_b(k, gs, ks, is);
    }
  }
  // Each use of a slot adds 2 to its counter, one per warpgroup: the leader that finds it odd released last, both
  // warpgroups have read the slot, and that leader refills it. Nobody waits.
  auto released_last = [](uint32_t* counter) {
    __threadfence_block();
    const uint32_t before = atomicAdd(counter, 1u);
    __threadfence_block();
    return (before & 1u) != 0u;
  };

  // ------------------------------ main loop ------------------------------
  if (p.bias && et < BLOCK_N) s_bias[et] = __ldg(p.bias + n0 + et);
  {
    float acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    // The MMA walk: K-slab s is tap t of group g (gsize taps, row shifts packed 4 bits per tap in gshift) at channel
    // slab kk; its A window and B box sit in ring slots a_slot / b_slot, whose barriers complete with parity a_par /
    // b_par. Every thread keeps the same walks, so whichever leader releases a slot last can refill it.
    int g = u_begin / kpt, kk = u_begin - g * kpt, t = 0;
    int gsize = p.grp_first[g + 1] - p.grp_first[g];
    uint64_t gshift = p.grp_shifts[g];
    int a_slot = 0, a_par = 0, b_slot = 0, b_par = 0;
    // The B load walk: the next B box to load, K-slab s + STAGES - 1 at step s, is sorted tap ib (of [ib0, ib_end),
    // group gb) at channel slab kb.
    int gb = 0, kb = 0, ib = 0;
    if (s_begin + STAGES < s_end) locate(s_begin + STAGES, gb, kb, ib);
    int ib0 = p.grp_first[gb], ib_end = p.grp_first[gb + 1];
    // The window load walk: the next window to load is unit ua, group ga at channel slab ka.
    int ua = u_begin + p.a_slots, ga = ua / kpt, ka = ua - ga * kpt;
    // issue one K-slab's MMAs as one commit group (every range holds at least one slab)
    auto issue_slab = [&]() {
      if (!p.slab_ring && t == 0) mbar_wait(&a_full[a_slot], a_par);  // the window's first tap
      mbar_wait(&b_full[b_slot], b_par);
      // the tap's 128 rows start its shift into the window; the 128 B swizzle follows the shared-memory address, as
      // the TMA wrote it, so a start that is not 1024-byte aligned needs no base offset
      const int shift = int(gshift >> (4 * t)) & 15;
      const uint32_t sa = smem_u32(smem + a_slot * a_bytes) + (shift + wg * 64) * (GEMM_BLOCK_K * 2);
      const uint64_t adesc = make_wgmma_desc(sa, 16, 1024, 1);
      const uint64_t bdesc = make_wgmma_desc(smem_u32(b_ring + b_slot * B_BYTES), 16, 1024, 1);
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
    issue_slab();
    for (int s = s_begin + 1; s < s_end; ++s) {
      if (++b_slot == STAGES) {
        b_slot = 0;
        b_par ^= 1;
      }
      const bool new_window = ++t == gsize;
      if (new_window) {
        t = 0;
        if (++kk == kpt) {
          kk = 0;
          ++g;
          gsize = p.grp_first[g + 1] - p.grp_first[g];
          gshift = p.grp_shifts[g];
        }
        if (++a_slot == p.a_slots) {
          a_slot = 0;
          a_par ^= 1;
        }
      }
      issue_slab();
      wgmma_wait<1>();  // slab s - 1 has retired: this warpgroup releases its B box, and its window if that was its last tap
      fence_regs(acc);
      const bool load_b = s - 1 + STAGES < s_end;
      const bool load_a = !p.slab_ring && new_window && ua < u_end;
      if ((et & 127) == 0) {
        const int bs = (b_slot ? b_slot : STAGES) - 1;
        if (load_b && released_last(&b_rel[bs])) fill_b(bs, gb, kb, ib);
        const int as = (a_slot ? a_slot : p.a_slots) - 1;
        if (load_a && released_last(&a_rel[as])) fill_a(as, ga, ka);
      }
      if (load_b && ++ib == ib_end) {
        if (++kb == kpt) {
          kb = 0;
          ++gb;
          ib0 = ib_end;
          ib_end = gb < p.num_groups ? p.grp_first[gb + 1] : ib_end;
        }
        ib = ib0;
      }
      if (load_a) {
        ++ua;
        if (++ka == kpt) {
          ka = 0;
          ++ga;
        }
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
  } else if (valid) {
    // direct stores through the row map
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
template <int BLOCK_N, int STAGES, int CTAS>
static int launch_gemm(const pf_gemm_args* a, GemmKernelParams kp, cudaStream_t st) {
  // STAGES B boxes, and as many A windows as the rest of the ring holds (a slab ring: STAGES 128-row boxes)
  const int a_slots = (gemm_ring_bytes(BLOCK_N, STAGES) - STAGES * BLOCK_N * GEMM_BLOCK_K * 2) /
                      (kp.a_rows * GEMM_BLOCK_K * 2);
  kp.a_slots = a_slots < STAGES ? a_slots : STAGES;
  // a window is refilled when the last tap of the window before it has retired: the ring needs two of them
  static_assert(gemm_ring_bytes(BLOCK_N, STAGES) - STAGES * BLOCK_N * GEMM_BLOCK_K * 2 >= 2 * GEMM_WIN_BYTES,
                "two A windows next to the B boxes");
  CUtensorMap tmA, tmB;
  {
    uint64_t dims[2] = {(uint64_t)a->Kc, (uint64_t)a->a_rows};
    uint64_t str[1] = {(uint64_t)a->a_ld * 2};
    uint32_t box[2] = {GEMM_BLOCK_K, (uint32_t)kp.a_rows};
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
  constexpr int SMEM = gemm_smem_bytes(BLOCK_N, STAGES);
  static_assert(SMEM <= 227 * 1024, "shared memory budget of one H100 CTA");
  static_assert(CTAS == 1 || SMEM <= GEMM_SMEM_CORESIDENT, "two CTAs per SM: 113 KB of shared memory each");
  const int m_tiles = (a->M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M;
  const dim3 grid(m_tiles * (a->N / BLOCK_N), kp.k_splits > 1 ? kp.k_splits : 1);
  const int bf = a->dtype == PF_BF16;
  auto kern = bf ? gemm_taps_kernel<BLOCK_N, STAGES, CTAS, true> : gemm_taps_kernel<BLOCK_N, STAGES, CTAS, false>;
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
      set_error("gemm_taps_kernel<%d, %d>: %d CTA(s) per SM fit, built for %d", BLOCK_N, STAGES, resident, CTAS);
      return PF_ERR_UNSUPPORTED;
    }
    attr_set[bf] = true;
  }
  kern<<<grid, GEMM_THREADS, SMEM, st>>>(tmA, tmB, kp);
  PF_CHECK_LAUNCH("gemm_taps_kernel");
  return PF_OK;
}

// tile width pf_gemm_taps runs with: the caller's request, else the heuristic. A statistics PRODUCER always uses the
// width the heuristic derives from N: the slot partition of the row sums (and so their fp32 rounding) must not depend
// on a per-call request, or a sharded rank would not reproduce the full batch.
static int resolve_block_n(const pf_gemm_args* a) {
  return a->block_n && !a->row_stats_out ? a->block_n : pf_gemm_pick_block_n(a->N, a->act);
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
  // GEGLU runs only at the 256-wide tile: its value and gate columns lie 128 apart in one thread's fragment
  if (act == PF_ACT_GEGLU) return N % 256 == 0 ? 256 : 0;
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
  const int bn = pf::resolve_block_n(a);
  const bool geglu = a->act == PF_ACT_GEGLU;
  const bool plain16 = a->map_mode == 0 && a->out_dtype == a->dtype && (!a->residual || a->res_dtype == a->dtype);
  if (geglu) {  // only the persistent linear GEMM has a GEGLU epilogue
    PF_CHECK_ARG(bn == 256, "pf_gemm_taps: GEGLU runs only at block_n 256, not %d (N=%d)", bn, a->N);
    PF_CHECK_ARG(a->num_taps == 1, "pf_gemm_taps: GEGLU needs one tap, not %d", a->num_taps);
    PF_CHECK_ARG(a->map_mode == 0 && a->out_dtype == a->dtype,
                 "pf_gemm_taps: GEGLU needs map_mode 0 and a 16-bit output");
    PF_CHECK_ARG(a->k_splits <= 1 && !a->residual && !a->rowbias,
                 "pf_gemm_taps: GEGLU takes no split-K, residual or rowbias");
  } else {
    PF_CHECK_ARG(bn == 64 || bn == 128 || bn == 160, "pf_gemm_taps: unsupported block_n %d (N=%d); 256 only with GEGLU",
                 bn, a->N);
  }
  PF_CHECK_ARG(a->N % bn == 0, "pf_gemm_taps: N=%d not a multiple of block_n=%d", a->N, bn);
  const int n_out = geglu ? a->N / 2 : a->N;
  PF_CHECK_ARG(a->out_ld % 8 == 0 && a->out_ld >= n_out, "pf_gemm_taps: bad out_ld %d", a->out_ld);
  PF_CHECK_ARG(!a->residual || (a->res_ld % 8 == 0 && a->res_ld >= n_out), "pf_gemm_taps: bad res_ld %d", a->res_ld);
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
  // Taps sorted by offset (equal offsets keep the caller's order) and cut into window groups: a tap joins the current
  // group while it lies within GEMM_WIN_SPAN rows of the group's first. The K order, and so the summation order,
  // depends on the tap offsets alone, never on M; a one-tap GEMM keeps the plain slab order.
  int order[PF_MAX_TAPS];
  for (int t = 0; t < a->num_taps; ++t) {
    int k = t;
    for (; k > 0 && a->tap_off[order[k - 1]] > a->tap_off[t]; --k) order[k] = order[k - 1];
    order[k] = t;
  }
  kp.num_groups = 0;
  for (int k = 0; k < PF_MAX_TAPS; ++k) kp.grp_shifts[k] = 0;
  int span = 0;
  for (int k = 0; k < a->num_taps; ++k) {
    const int off = a->tap_off[order[k]];
    if (k == 0 || (long long)off - kp.grp_off[kp.num_groups - 1] > GEMM_WIN_SPAN) {
      kp.grp_first[kp.num_groups] = k;
      kp.grp_off[kp.num_groups++] = off;
    }
    const int shift = off - kp.grp_off[kp.num_groups - 1];
    kp.grp_shifts[kp.num_groups - 1] |= uint64_t(shift) << (4 * (k - kp.grp_first[kp.num_groups - 1]));
    kp.tap_src[k] = order[k];
    span = span > shift ? span : shift;
  }
  kp.grp_first[kp.num_groups] = a->num_taps;
  kp.num_units = kp.num_groups * kp.kb_per_tap;
  kp.a_rows = GEMM_BLOCK_M + (span ? GEMM_WIN_SPAN : 0);
  kp.slab_ring = kp.num_groups == a->num_taps;
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
  PF_CHECK_ARG(kp.k_splits == 1 || (a->splitk_ws && kp.k_splits <= kp.num_units),
               "pf_gemm_taps: split-K needs a workspace and k_splits <= (tap window, channel slab) units");
  if (a->row_stats_out || a->ln_stats) {  // fused LayerNorm: only the persistent linear GEMM folds it
    PF_CHECK_ARG(kp.k_splits == 1, "pf_gemm_taps: fused LayerNorm does not combine with split-K");
    PF_CHECK_ARG(!a->ln_stats || (a->ln_colsum && a->ln_slots > 0 && a->ln_slots % 2 == 0 && a->ln_eps > 0.f &&
                                  (reinterpret_cast<uintptr_t>(a->ln_stats) & 15) == 0),
                 "pf_gemm_taps: ln_stats needs ln_colsum, ln_slots and ln_eps");
    PF_CHECK_ARG(a->num_taps == 1 && !a->rowbias, "pf_gemm_taps: fused LayerNorm needs one tap and no rowbias");
    PF_CHECK_ARG(plain16 && !(geglu && a->row_stats_out),
                 "pf_gemm_taps: fused LayerNorm needs the plain row map with 16-bit output (consumer: or GEGLU)");
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (kp.k_splits > 1) {
    int rc = PF_ERR_UNSUPPORTED;
    switch (bn) {
      // few tiles of 90-360 K-slabs, planned at about one CTA per SM: nothing to co-schedule, so the long rings
      case 64: rc = launch_gemm<64, 8, 1>(a, kp, st); break;
      case 128: rc = launch_gemm<128, 6, 1>(a, kp, st); break;
      case 160: rc = launch_gemm<160, 5, 1>(a, kp, st); break;
    }
    if (rc) return rc;
    const long long total = (long long)a->M * (a->N / 8);
    if (a->dtype == PF_BF16) splitk_reduce_kernel<true><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(kp);
    else splitk_reduce_kernel<false><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(kp);
    PF_CHECK_LAUNCH("splitk_reduce_kernel");
    return PF_OK;
  }
  // one-tap, plain-row-map calls with 16-bit output and 16-bit (or no) residual and no row bias: the persistent linear
  // GEMM (gemm_linear.cu). The checks above leave every GEGLU and fused-LayerNorm call in this class.
  if (a->num_taps == 1 && plain16 && !a->rowbias) return launch_gemm_linear(a, kp, bn, st);
  switch (bn) {
    case 64: return launch_gemm<64, 4, 2>(a, kp, st);
    case 128: return launch_gemm<128, 3, 2>(a, kp, st);
    case 160: return launch_gemm<160, 3, 2>(a, kp, st);
  }
  return PF_ERR_UNSUPPORTED;
}
