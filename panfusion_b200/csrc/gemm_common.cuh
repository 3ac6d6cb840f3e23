// Shared declarations of the two GEMM kernels behind pf_gemm_taps: the tap-GEMM (gemm_wgmma.cu) and the persistent
// linear GEMM (gemm_linear.cu), which takes the tap-GEMM's parameter block.
#pragma once
#include "pf_common.cuh"

namespace pf {

constexpr int GEMM_BLOCK_M = 128;
constexpr int GEMM_BLOCK_K = 64;  // 64 x 16-bit = 128 B = one swizzle row
// Taps whose offsets lie within GEMM_WIN_SPAN rows of each other share one A window of 128 + GEMM_WIN_SPAN rows.
// 8 covers a 3x3 kernel row (span 2) and an Upsample2D phase row (span 1) and keeps two windows and three 160-wide B
// boxes inside a co-resident CTA's 108 KB ring.
constexpr int GEMM_WIN_SPAN = 8;
constexpr int GEMM_WIN_BYTES = (GEMM_BLOCK_M + GEMM_WIN_SPAN) * GEMM_BLOCK_K * 2;

struct GemmKernelParams {
  int M, N, kb_per_tap;
  // K order: (window group, 64-channel slab, tap of the group). Taps are sorted by offset; group g holds sorted taps
  // [grp_first[g], grp_first[g + 1]) and its A window starts grp_off[g] rows from the tile. A unit is one
  // (group, channel slab) pair: one A window and one B box per tap of the group.
  int num_groups, num_units;
  int grp_first[PF_MAX_TAPS + 1];
  int grp_off[PF_MAX_TAPS];
  int tap_src[PF_MAX_TAPS];    // sorted tap: the caller's tap index, i.e. its block of B's columns
  // the operand ring: a_slots A windows of a_rows rows, then the B boxes. slab_ring: every group is a single tap, so
  // each K-slab's A box travels with its B box (one barrier per slot, as a plain GEMM's ring)
  int a_rows, a_slots, slab_ring;
  // group g: the rows its taps start past the window start (0..GEMM_WIN_SPAN), 4 bits per tap in sorted order
  unsigned long long grp_shifts[PF_MAX_TAPS];
  void* out;
  int out_ld;
  int out_f32;
  const float* bias;
  const float* rowbias;
  int rowbias_ld;
  int rows_per_group;
  const void* residual;
  int res_ld;
  int res_f32;
  int act;
  int map_mode, Hm, Wm, i0, j0, Hout, Wout;
  int osy, osx, oa, ob;  // output scatter of map_mode 1: row ((img*Hout + i-i0)*osy + oa), column ((j-j0)*osx + ob)
  int k_splits;     // > 1: blockIdx.y = split index, raw fp32 partials go to ws
  float* ws;        // [k_splits][M][N]
  // fused LayerNorm (see pf_gemm_args): producer side / consumer side
  float* row_stats;        // [M][stat_slots][2] or null
  int stat_slots;          // 2 * n_tiles
  const float* ln_stats;   // [M][ln_slots][2] or null
  int ln_slots;
  const float* ln_colsum;  // [N]
  float ln_inv_k, ln_eps;
};

__host__ __device__ constexpr int gemm_stage_bytes(int block_n) {
  return GEMM_BLOCK_M * GEMM_BLOCK_K * 2 + block_n * GEMM_BLOCK_K * 2;
}

// The persistent linear GEMM (gemm_linear.cu) for one-tap, plain-row-map calls with 16-bit output and residual, no row
// bias and no split-K, at tile width bn (GEGLU: bn = 256 only). kp is the tap-GEMM's parameter block.
int launch_gemm_linear(const pf_gemm_args* a, const GemmKernelParams& kp, int bn, cudaStream_t st);

}  // namespace pf
