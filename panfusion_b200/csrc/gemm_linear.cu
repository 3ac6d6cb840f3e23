// Persistent, warp-specialized GEMM for the single-tap, plain-row-map calls of pf_gemm_taps with a 16-bit output:
// nn.Linear (proj_in, q|k|v, to_out, the Transformer tail, GEGLU, the text-tower and EPPA / CPAttn linears) and the
// resnet 1x1 shortcuts. Their K is short (320-1600), so in the tap-GEMM kernel a tile's MMAs are small next to what it
// pays serially per tile: the first ring fill, the fp32 accumulator dump through shared memory, the barriers and the
// stores. Here nothing of that lies between two tiles' MMAs:
//
// - One CTA per SM, min(tiles, SMs) CTAs; CTA b runs tiles b, b + gridDim.x, ... in the order n fastest, so the CTAs
//   running at the same time share A rows through L2.
// - 384 threads. Warpgroup 2 is the producer (setmaxnreg 40): one thread walks (tile, K-slab) without a break through
//   a ring of STAGES slots (a 128-row A box and a BLOCK_N-row B box behind one full barrier; one empty barrier with one
//   arrival per consumer warpgroup). It fills the next tile's first slabs while the consumers run the epilogue. Slot
//   and parity come from the running slab count, never from a per-tile index.
// - Warpgroups 0 and 1 are the consumers (setmaxnreg 232): rows [64 wg, 64 wg + 64) of the 128 x BLOCK_N tile. The
//   per-slab wgmma sequence, the K order and the first-slab peel are the tap-GEMM kernel's, so each accumulator is
//   bit-identical to it.
// - The epilogue works on the wgmma fragment in registers: LayerNorm fold, bias, activation (or GEGLU: value column c
//   and gate column 128 + c are fragment columns j and j + 16 of the same thread), residual, row statistics. The 16-bit
//   result goes into a swizzled staging buffer of the warpgroup, one thread hands it to TMA tile stores, and the
//   warpgroup goes straight to the next tile's MMAs; the store's read of the buffer is waited for at the next epilogue.
// - The 16-bit residual tile is fetched by the producer with TMA into its own slot, in the staging layout.
// - LayerNorm consumer: warps 1-3 of the producer warpgroup turn the row statistics of each tile's 128 rows into the
//   fold's two coefficients in one of two shared-memory slots, ahead of the consumers, so the epilogue never waits on
//   the global loads of the statistics.
#include "gemm_common.cuh"
#include "wgmma.cuh"

namespace pf {

constexpr int LIN_THREADS = 384;
constexpr int LIN_SUB_COLS = 32;                            // TMA store / residual boxes: 32 columns, SWIZZLE_64B
constexpr int LIN_SUB_BYTES = 64 * LIN_SUB_COLS * 2;        // one warpgroup's [64][32] 16-bit sub-tile
constexpr int LIN_RES_SUB_BYTES = GEMM_BLOCK_M * LIN_SUB_COLS * 2;  // one [128][32] residual sub-tile

// columns a tile writes: GEGLU halves the width
__host__ __device__ constexpr int lin_out_cols(int block_n, bool geglu) { return geglu ? block_n / 2 : block_n; }
__host__ __device__ constexpr int lin_ring_bytes(int block_n, int stages) { return stages * gemm_stage_bytes(block_n); }
__host__ __device__ constexpr int lin_staging_bytes(int block_n, bool geglu) {
  return 2 * 64 * lin_out_cols(block_n, geglu) * 2;
}
// GEGLU takes no residual: no residual slot
__host__ __device__ constexpr int lin_res_bytes(int block_n, bool geglu) { return geglu ? 0 : GEMM_BLOCK_M * block_n * 2; }
__host__ __device__ constexpr int lin_smem_bytes(int block_n, int stages, bool geglu) {
  return lin_ring_bytes(block_n, stages) + lin_staging_bytes(block_n, geglu) + lin_res_bytes(block_n, geglu) +
         2 * GEMM_BLOCK_M * 8 /*two slots of LayerNorm coefficients*/ + (2 * stages + 6) * 8;
}

// mean / rstd of one row from the producer's partial sums, as the two epilogue coefficients of the LayerNorm fold:
// acc <- acc * a + colsum[n] * b with a = rstd, b = -mean * rstd
__device__ __forceinline__ void ln_row_coeffs(const GemmKernelParams& p, long long m, float& a, float& b) {
  // slots come in pairs (two per column tile): 16-byte loads, four of them in flight, summed in slot order
  const float4* st = reinterpret_cast<const float4*>(p.ln_stats) + m * (p.ln_slots >> 1);
  const int pairs = p.ln_slots >> 1;
  float s = 0.f, q = 0.f;
  for (int i0 = 0; i0 < pairs; i0 += 4) {
    float4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = i0 + u < pairs ? __ldg(st + i0 + u) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      s += v[u].x;
      q += v[u].y;
      s += v[u].z;
      q += v[u].w;
    }
  }
  const float mean = s * p.ln_inv_k;
  const float var = fmaxf(q * p.ln_inv_k - mean * mean, 0.f);
  a = rsqrtf(var + p.ln_eps);
  b = -mean * a;
}

__device__ __forceinline__ void setmaxnreg_inc232() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory"); }
__device__ __forceinline__ void setmaxnreg_dec40() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory"); }

// byte offset of 16-bit element (row r, column c) in [c / 32][rows][32] sub-tiles of `rows` rows, SWIZZLE_64B (16-byte
// chunk index ^= (r >> 1) & 3); c is even, so the two elements (c, c + 1) are one 4-byte word
__device__ __forceinline__ uint32_t lin_sw_off(int r, int c, int rows) {
  return uint32_t((c >> 5) * rows * 64 + r * 64 + ((((c & 31) >> 3) ^ ((r >> 1) & 3)) << 4) + (c & 7) * 2);
}

template <int BLOCK_N, int STAGES, bool GEGLU, bool BF16>
__global__ void __launch_bounds__(LIN_THREADS, 1)
gemm_linear_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR,
                   const GemmKernelParams p) {
  constexpr int A_BYTES = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;
  constexpr int B_BYTES = BLOCK_N * GEMM_BLOCK_K * 2;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int NACC = BLOCK_N / 2;  // fp32 accumulators per consumer thread
  constexpr int OUT_N = lin_out_cols(BLOCK_N, GEGLU);
  constexpr int NSUB = OUT_N / LIN_SUB_COLS;
  static_assert(OUT_N % LIN_SUB_COLS == 0, "output tile in 32-column sub-tiles");
  static_assert(!GEGLU || BLOCK_N == 256, "GEGLU in registers: value and gate columns 128 apart");

  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* const staging = smem + lin_ring_bytes(BLOCK_N, STAGES);  // per warpgroup [NSUB][64][32]
  uint8_t* const res_tile = staging + lin_staging_bytes(BLOCK_N, GEGLU);  // [BLOCK_N / 32][128][32]
  float2* const ln_coef = reinterpret_cast<float2*>(res_tile + lin_res_bytes(BLOCK_N, GEGLU));  // [2][128] (a, b)
  uint64_t* const full = reinterpret_cast<uint64_t*>(ln_coef + 2 * GEMM_BLOCK_M);
  uint64_t* const empty = full + STAGES;
  uint64_t* const res_full = empty + STAGES;
  uint64_t* const res_empty = res_full + 1;
  uint64_t* const ln_full = res_empty + 1;  // [2]
  uint64_t* const ln_empty = ln_full + 2;   // [2]

  const int n_tiles = p.N / BLOCK_N;
  const int tiles = (p.M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M * n_tiles;
  const int kslabs = p.kb_per_tap;
  const bool has_res = p.residual != nullptr;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);  // one arrival per consumer warpgroup
    }
    mbar_init(res_full, 1);
    mbar_init(res_empty, 2);
    for (int s = 0; s < 2; ++s) {
      mbar_init(&ln_full[s], 96);  // one arrival per thread of warps 1-3 of the producer warpgroup
      mbar_init(&ln_empty[s], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    // ------------------------------ producer ------------------------------
    setmaxnreg_dec40();
    if (threadIdx.x >= 288) {
      if (!p.ln_stats) return;
      // LayerNorm coefficients of tile i's rows into slot i & 1
      int i = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++i) {
        const int m0 = (tile / n_tiles) * GEMM_BLOCK_M;
        mbar_wait(&ln_empty[i & 1], ((i >> 1) & 1) ^ 1);
        for (int r = threadIdx.x - 288; r < GEMM_BLOCK_M; r += 96) {
          float a = 1.f, b = 0.f;  // rows past M are clipped by the store
          if (m0 + r < p.M) ln_row_coeffs(p, m0 + r, a, b);
          ln_coef[(i & 1) * GEMM_BLOCK_M + r] = make_float2(a, b);
        }
        mbar_arrive(&ln_full[i & 1]);
      }
      return;
    }
    if (threadIdx.x != 256) return;
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (has_res) tma_prefetch_desc(&tmR);
    int slot = 0, par = 0, res_par = 0;
    // the residual of a tile is requested once its first slabs are on their way: by then the consumers are in (or
    // past) the previous tile's epilogue, whose residual read this load waits for
    const int res_after = (kslabs < STAGES ? kslabs : STAGES) - 1;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
      const int n0 = (tile % n_tiles) * BLOCK_N;
      const int m0 = (tile / n_tiles) * GEMM_BLOCK_M;
      for (int k = 0; k < kslabs; ++k) {
        mbar_wait(&empty[slot], par ^ 1);
        mbar_expect_tx(&full[slot], STAGE_BYTES);
        uint8_t* st = smem + slot * STAGE_BYTES;
        tma_load_2d(st, &tmA, &full[slot], k * GEMM_BLOCK_K, m0 + p.grp_off[0]);
        tma_load_2d(st + A_BYTES, &tmB, &full[slot], k * GEMM_BLOCK_K, n0);
        if (++slot == STAGES) {
          slot = 0;
          par ^= 1;
        }
        if (!GEGLU && has_res && k == res_after) {
          mbar_wait(res_empty, res_par ^ 1);
          mbar_expect_tx(res_full, lin_res_bytes(BLOCK_N, GEGLU));
#pragma unroll 1
          for (int s = 0; s < BLOCK_N / LIN_SUB_COLS; ++s)
            tma_load_2d(res_tile + s * LIN_RES_SUB_BYTES, &tmR, res_full, n0 + s * LIN_SUB_COLS, m0);
          res_par ^= 1;
        }
      }
    }
    return;
  }

  // ------------------------------ consumers ------------------------------
  setmaxnreg_inc232();
  const int et = threadIdx.x & 127;
  const int lane = threadIdx.x & 31;
  // fragment of m64nN: thread (warp w, lane l) holds rows 16w + l/4 (+8), columns 8j + 2(l%4) (+1)
  const int rl = ((et >> 5) << 4) + (lane >> 2);  // row of the warpgroup's 64 (and rl + 8)
  const int cb = 2 * (lane & 3);
  uint8_t* const my_staging = staging + wg * (NSUB * LIN_SUB_BYTES);
  if (et == 0) tma_prefetch_desc(&tmC);
  int slot = 0, par = 0, res_par = 0;
  float acc[NACC];

  for (int tile = blockIdx.x, ti = 0; tile < tiles; tile += gridDim.x, ++ti) {
    const int n_tile = tile % n_tiles;
    const int n0 = n_tile * BLOCK_N;
    const int m0 = (tile / n_tiles) * GEMM_BLOCK_M;

#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    auto issue_slab = [&]() {
      mbar_wait(&full[slot], par);
      const uint32_t sa = smem_u32(smem + slot * STAGE_BYTES) + wg * 64 * (GEMM_BLOCK_K * 2);
      const uint64_t adesc = make_wgmma_desc(sa, 16, 1024, 1);
      const uint64_t bdesc = make_wgmma_desc(smem_u32(smem + slot * STAGE_BYTES + A_BYTES), 16, 1024, 1);
      wgmma_fence();
      fence_regs(acc);
#pragma unroll
      for (int k = 0; k < GEMM_BLOCK_K / 16; ++k)  // +32 B per K step inside the 128 B swizzle row => +2 in (addr >> 4)
        Wgmma<BLOCK_N, BF16>::ss(acc, adesc + 2 * k, bdesc + 2 * k, 1);
      wgmma_commit();
      fence_regs(acc);
    };
    // the first slab is peeled, as in the tap-GEMM kernel: without it ptxas sees the accumulators defined both by the
    // zeroing and by MMAs in flight at the loop head and serialises every wgmma (C7515)
    issue_slab();
    int prev = slot;
    if (++slot == STAGES) {
      slot = 0;
      par ^= 1;
    }
    for (int k = 1; k < kslabs; ++k) {
      issue_slab();
      wgmma_wait<1>();  // slab k - 1 has retired: release its slot
      fence_regs(acc);
      if (et == 0) mbar_arrive(&empty[prev]);
      prev = slot;
      if (++slot == STAGES) {
        slot = 0;
        par ^= 1;
      }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    if (et == 0) mbar_arrive(&empty[prev]);

    // ------------------------------ epilogue ------------------------------
    const int ma = m0 + wg * 64 + rl, mb = ma + 8;  // the thread's two rows
    if (p.ln_stats) {
      mbar_wait(&ln_full[ti & 1], (ti >> 1) & 1);
      const float2 ca = ln_coef[(ti & 1) * GEMM_BLOCK_M + wg * 64 + rl];
      const float2 cc = ln_coef[(ti & 1) * GEMM_BLOCK_M + wg * 64 + rl + 8];
      const float la = ca.x, lb = ca.y, ha = cc.x, hb = cc.y;
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const float cs0 = __ldg(p.ln_colsum + n0 + 8 * j + cb), cs1 = __ldg(p.ln_colsum + n0 + 8 * j + cb + 1);
        acc[4 * j] = fmaf(acc[4 * j], la, cs0 * lb);
        acc[4 * j + 1] = fmaf(acc[4 * j + 1], la, cs1 * lb);
        acc[4 * j + 2] = fmaf(acc[4 * j + 2], ha, cs0 * hb);
        acc[4 * j + 3] = fmaf(acc[4 * j + 3], ha, cs1 * hb);
      }
    }
    if constexpr (GEGLU) {
      // value column c = 8j + cb (j < 16) and its gate column 128 + c (j + 16); the result replaces the value
#pragma unroll
      for (int j = 0; j < OUT_N / 8; ++j) {
        float ba0 = 0.f, ba1 = 0.f, bg0 = 0.f, bg1 = 0.f;
        if (p.bias) {
          ba0 = __ldg(p.bias + n0 + 8 * j + cb);
          ba1 = __ldg(p.bias + n0 + 8 * j + cb + 1);
          bg0 = __ldg(p.bias + n0 + OUT_N + 8 * j + cb);
          bg1 = __ldg(p.bias + n0 + OUT_N + 8 * j + cb + 1);
        }
        constexpr int G = 4 * (OUT_N / 8);
        geglu_pair(acc[4 * j], acc[4 * j + 1], acc[G + 4 * j], acc[G + 4 * j + 1], ba0, ba1, bg0, bg1, acc[4 * j],
                   acc[4 * j + 1]);
        geglu_pair(acc[4 * j + 2], acc[4 * j + 3], acc[G + 4 * j + 2], acc[G + 4 * j + 3], ba0, ba1, bg0, bg1,
                   acc[4 * j + 2], acc[4 * j + 3]);
      }
    } else {
      if (p.bias) {
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const float b0 = __ldg(p.bias + n0 + 8 * j + cb), b1 = __ldg(p.bias + n0 + 8 * j + cb + 1);
          acc[4 * j] += b0;
          acc[4 * j + 1] += b1;
          acc[4 * j + 2] += b0;
          acc[4 * j + 3] += b1;
        }
      }
      if (p.act == PF_ACT_SILU) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] = silu_f(acc[i]);
      } else if (p.act == PF_ACT_GELU) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] = gelu_erf_f(acc[i]);
      } else if (p.act == PF_ACT_QUICK_GELU) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] = quick_gelu_f(acc[i]);
      }
      if (has_res) {  // rows past M were zero-filled by the TMA load
        mbar_wait(res_full, res_par);
        res_par ^= 1;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const float2 ra = unpack2<BF16>(
              *reinterpret_cast<const uint32_t*>(res_tile + lin_sw_off(wg * 64 + rl, 8 * j + cb, GEMM_BLOCK_M)));
          const float2 rb = unpack2<BF16>(
              *reinterpret_cast<const uint32_t*>(res_tile + lin_sw_off(wg * 64 + rl + 8, 8 * j + cb, GEMM_BLOCK_M)));
          acc[4 * j] += ra.x;
          acc[4 * j + 1] += ra.y;
          acc[4 * j + 2] += rb.x;
          acc[4 * j + 3] += rb.y;
        }
      }
      if (p.row_stats) {
        // slot 2 n_tile + h sums the even (h = 0) / odd (h = 1) 16-column chunks of the row: fragment column group j
        // lies in chunk j / 2. Per lane in column order, then over the row's four lanes.
        float s[2][2] = {{0.f, 0.f}, {0.f, 0.f}}, q[2][2] = {{0.f, 0.f}, {0.f, 0.f}};  // [row a / b][h]
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          const int h = (j >> 1) & 1;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            s[0][h] += acc[4 * j + e];
            q[0][h] = fmaf(acc[4 * j + e], acc[4 * j + e], q[0][h]);
            s[1][h] += acc[4 * j + 2 + e];
            q[1][h] = fmaf(acc[4 * j + 2 + e], acc[4 * j + 2 + e], q[1][h]);
          }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            s[r][h] += __shfl_xor_sync(0xffffffffu, s[r][h], 1);
            q[r][h] += __shfl_xor_sync(0xffffffffu, q[r][h], 1);
            s[r][h] += __shfl_xor_sync(0xffffffffu, s[r][h], 2);
            q[r][h] += __shfl_xor_sync(0xffffffffu, q[r][h], 2);
          }
        if ((lane & 3) < 2) {  // lane h of the row's four writes slot 2 n_tile + h of both rows
          const int h = lane & 1;
          float2* st = reinterpret_cast<float2*>(p.row_stats) + n_tile * 2 + h;
          if (ma < p.M) st[(long long)ma * p.stat_slots] = make_float2(h ? s[0][1] : s[0][0], h ? q[0][1] : q[0][0]);
          if (mb < p.M) st[(long long)mb * p.stat_slots] = make_float2(h ? s[1][1] : s[1][0], h ? q[1][1] : q[1][0]);
        }
      }
    }

    // the previous tile's stores have read the staging buffer before anyone refills it
    if (et == 0) tma_store_wait_read();
    named_bar_sync(1 + wg, 128);
    if (et == 0) {  // every residual and coefficient read of this warpgroup lies before the barrier
      if (!GEGLU && has_res) mbar_arrive(res_empty);
      if (p.ln_stats) mbar_arrive(&ln_empty[ti & 1]);
    }
#pragma unroll
    for (int j = 0; j < OUT_N / 8; ++j) {
      *reinterpret_cast<uint32_t*>(my_staging + lin_sw_off(rl, 8 * j + cb, 64)) = pack2<BF16>(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<uint32_t*>(my_staging + lin_sw_off(rl + 8, 8 * j + cb, 64)) =
          pack2<BF16>(acc[4 * j + 2], acc[4 * j + 3]);
    }
    fence_proxy_async_smem();  // generic-proxy writes -> visible to the TMA store
    named_bar_sync(1 + wg, 128);
    if (et == 0) {
#pragma unroll 1
      for (int s = 0; s < NSUB; ++s)
        tma_store_2d(&tmC, my_staging + s * LIN_SUB_BYTES, n_tile * OUT_N + s * LIN_SUB_COLS, m0 + wg * 64);
      tma_store_commit();
    }
  }
  if (et == 0) tma_store_wait_read();  // shared memory must outlive the last stores' reads
}

template <int BLOCK_N, int STAGES, bool GEGLU>
static int launch_linear(const pf_gemm_args* a, const GemmKernelParams& kp, cudaStream_t st) {
  constexpr int OUT_N = lin_out_cols(BLOCK_N, GEGLU);
  CUtensorMap tmA, tmB, tmC, tmR;
  {
    uint64_t dims[2] = {(uint64_t)a->Kc, (uint64_t)a->a_rows};
    uint64_t str[1] = {(uint64_t)a->a_ld * 2};
    uint32_t box[2] = {GEMM_BLOCK_K, GEMM_BLOCK_M};
    int rc = make_tmap(&tmA, a->dtype, 2, a->A, dims, str, box, 128);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {(uint64_t)a->Kc, (uint64_t)a->N};
    uint64_t str[1] = {(uint64_t)a->b_ld * 2};
    uint32_t box[2] = {GEMM_BLOCK_K, (uint32_t)BLOCK_N};
    int rc = make_tmap(&tmB, a->dtype, 2, a->B, dims, str, box, 128);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {(uint64_t)(a->N / BLOCK_N * OUT_N), (uint64_t)a->M};
    uint64_t str[1] = {(uint64_t)a->out_ld * 2};
    uint32_t box[2] = {LIN_SUB_COLS, 64};
    int rc = make_tmap(&tmC, a->dtype, 2, a->out, dims, str, box, 64);
    if (rc) return rc;
  }
  tmR = tmC;
  if (a->residual) {
    uint64_t dims[2] = {(uint64_t)a->N, (uint64_t)a->M};
    uint64_t str[1] = {(uint64_t)a->res_ld * 2};
    uint32_t box[2] = {LIN_SUB_COLS, GEMM_BLOCK_M};
    int rc = make_tmap(&tmR, a->dtype, 2, a->residual, dims, str, box, 64);
    if (rc) return rc;
  }
  constexpr int SMEM = lin_smem_bytes(BLOCK_N, STAGES, GEGLU);
  static_assert(SMEM <= 227 * 1024, "shared memory budget of one H100 CTA");
  const int bf = a->dtype == PF_BF16;
  auto kern = bf ? gemm_linear_kernel<BLOCK_N, STAGES, GEGLU, true> : gemm_linear_kernel<BLOCK_N, STAGES, GEGLU, false>;
  static bool attr_set[2] = {false, false};  // per dtype
  if (!attr_set[bf]) {
    int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM),
                        "cudaFuncSetAttribute(gemm_linear)");
    if (rc) return rc;
    attr_set[bf] = true;
  }
  const long long tiles = (long long)((a->M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M) * (a->N / BLOCK_N);
  const int sms = sm_count();
  const unsigned grid = (unsigned)(tiles < sms ? tiles : sms);
  kern<<<grid, LIN_THREADS, SMEM, st>>>(tmA, tmB, tmC, tmR, kp);
  PF_CHECK_LAUNCH("gemm_linear_kernel");
  return PF_OK;
}

int launch_gemm_linear(const pf_gemm_args* a, const GemmKernelParams& kp, int bn, cudaStream_t st) {
  if (a->act == PF_ACT_GEGLU) return bn == 256 ? launch_linear<256, 4, true>(a, kp, st) : PF_ERR_UNSUPPORTED;
  switch (bn) {
    case 64: return launch_linear<64, 8, false>(a, kp, st);
    case 128: return launch_linear<128, 5, false>(a, kp, st);
    case 160: return launch_linear<160, 4, false>(a, kp, st);
  }
  return PF_ERR_UNSUPPORTED;
}

}  // namespace pf
