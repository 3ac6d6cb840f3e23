// Spherical resampling kernels: equirect -> perspective (e2p) and perspective -> equirect (p2e).
// Reference: external/Perspective_and_Equirectangular/e2p.py:9-76, p2e.py:9-77 (grid built on the CPU in
// float64 numpy per camera, uploaded, then kornia.remap == F.grid_sample(align_corners=True, zeros)).
// Here the grid is evaluated in-kernel in fp64 per output pixel (amortised over the channel loop), rounded to
// fp32 exactly where the reference rounds (`.type(e_img.dtype)`), and pushed through the same fp32
// normalise / un-normalise round trip as kornia + ATen so the bilinear taps agree with the oracle.
//
// Two variants per direction:
//   * staged  : the source planes of a channel group are brought into shared memory with 1-D bulk async copies
//               (cp.async.bulk, mbarrier completion), double-buffered; taps are computed once per CTA and reused
//               for every channel. Used when a source plane fits in shared memory (all EPPA / latent shapes).
//   * direct  : gathers straight from global memory (L2) — any plane size (pixel-space panoramas).
#include "sphere_grid.cuh"

namespace pf {

// ---------------------------------------------------------------------------------------------------
// direct variant: thread <-> output pixel, loop over a channel slice. NCHW.
// grid = (ceil(hw_out/256), channel slices, B)
// ---------------------------------------------------------------------------------------------------
template <typename T, bool P2E>
__global__ void __launch_bounds__(256)
resample_direct_kernel(const T* __restrict__ src, T* __restrict__ dst, uint8_t* __restrict__ mask_out, int C,
                       int Hs, int Ws, int Hd, int Wd, const double* __restrict__ cams, int cam_stride, int mode,
                       int ch_per_slice) {
  const int b = blockIdx.z;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= Hd * Wd) return;
  const int r = pix / Wd, c = pix - r * Wd;
  const double* cam = cams + (size_t)b * cam_stride * PF_CAM_DOUBLES;
  float px, py;
  bool live = true;
  if constexpr (P2E) {
    p2e_grid(cam, r, c, Hd, Wd, Hs, Ws, px, py, live);
    if (mask_out && blockIdx.y == 0) mask_out[(size_t)b * Hd * Wd + pix] = live ? 1 : 0;
  } else {
    e2p_grid(cam, r, c, Hd, Wd, Hs, Ws, px, py);
  }
  Taps t;
  // p2e samples everywhere `inside` holds and multiplies by mask afterwards; sample * 0 == 0 for finite data
  make_taps(px, py, Hs, Ws, mode, live, t);
  const int c0 = blockIdx.y * ch_per_slice;
  const int c1 = min(C, c0 + ch_per_slice);
  const size_t splane = (size_t)Hs * Ws, dplane = (size_t)Hd * Wd;
  const T* sp = src + ((size_t)b * C + c0) * splane;
  T* dp = dst + ((size_t)b * C + c0) * dplane + pix;
  for (int ch = c0; ch < c1; ++ch) {
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (t.idx[k] >= 0) acc = __fadd_rn(acc, __fmul_rn(Cvt<T>::to_f(__ldg(sp + t.idx[k])), t.w[k]));
    }
    *dp = Cvt<T>::from_f(acc);
    sp += splane;
    dp += dplane;
  }
}

// ---------------------------------------------------------------------------------------------------
// staged variant: CTA <-> (batch b, channel range); taps for ALL output pixels live in registers
// (PIX_PER_THREAD each); source planes stream through a 2-deep shared-memory ring via cp.async.bulk.
// Output stores are fully coalesced (thread <-> consecutive x), source reads hit shared memory.
// ---------------------------------------------------------------------------------------------------
constexpr int STG_THREADS = 256;

template <typename T, bool P2E, int PPT>
__global__ void __launch_bounds__(STG_THREADS)
resample_staged_kernel(const T* __restrict__ src, T* __restrict__ dst, uint8_t* __restrict__ mask_out, int C,
                       int Hs, int Ws, int Hd, int Wd, const double* __restrict__ cams, int cam_stride, int mode,
                       int ch_per_cta, int ch_per_stage) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  const int splane = Hs * Ws, dplane = Hd * Wd;
  const uint32_t stage_bytes = uint32_t(ch_per_stage) * splane * sizeof(T);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem);
  T* buf0 = reinterpret_cast<T*>(smem + 128);
  T* buf1 = reinterpret_cast<T*>(smem + 128 + ((stage_bytes + 127) & ~127u));

  const int b = blockIdx.y;
  const int c_begin = blockIdx.x * ch_per_cta;
  const int c_end = min(C, c_begin + ch_per_cta);
  const int n_stages = (c_end - c_begin + ch_per_stage - 1) / ch_per_stage;
  const T* sbase = src + (size_t)b * C * splane;

  if (threadIdx.x == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto issue = [&](int st) {
    const int ca = c_begin + st * ch_per_stage;
    const int nch = min(ch_per_stage, c_end - ca);
    const uint32_t bytes = uint32_t(nch) * splane * sizeof(T);
    mbar_expect_tx(&bars[st & 1], bytes);
    bulk_load_1d((st & 1) ? buf1 : buf0, sbase + (size_t)ca * splane, bytes, &bars[st & 1]);
  };
  if (threadIdx.x == 0) {
    issue(0);
    if (n_stages > 1) issue(1);
  }

  // taps for this thread's output pixels (overlaps the first bulk copies)
  const double* cam = cams + (size_t)b * cam_stride * PF_CAM_DOUBLES;
  Taps taps[PPT];
#pragma unroll
  for (int i = 0; i < PPT; ++i) {
    const int pix = threadIdx.x + i * STG_THREADS;
    bool live = pix < dplane;
    float px = 0.f, py = 0.f;
    if (live) {
      const int r = pix / Wd, c = pix - r * Wd;
      if constexpr (P2E) {
        bool m;
        p2e_grid(cam, r, c, Hd, Wd, Hs, Ws, px, py, m);
        if (mask_out && blockIdx.x == 0) mask_out[(size_t)b * dplane + pix] = m ? 1 : 0;
        live = m;
      } else {
        e2p_grid(cam, r, c, Hd, Wd, Hs, Ws, px, py);
      }
    }
    make_taps(px, py, Hs, Ws, mode, live, taps[i]);
  }

  for (int st = 0; st < n_stages; ++st) {
    mbar_wait(&bars[st & 1], (st >> 1) & 1);
    const T* sb = (st & 1) ? buf1 : buf0;
    const int ca = c_begin + st * ch_per_stage;
    const int nch = min(ch_per_stage, c_end - ca);
    T* dp = dst + ((size_t)b * C + ca) * dplane;
    for (int ch = 0; ch < nch; ++ch) {
      const T* sp = sb + (size_t)ch * splane;
#pragma unroll
      for (int i = 0; i < PPT; ++i) {
        const int pix = threadIdx.x + i * STG_THREADS;
        if (pix < dplane) {
          float acc = 0.f;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            if (taps[i].idx[k] >= 0) acc = __fadd_rn(acc, __fmul_rn(Cvt<T>::to_f(sp[taps[i].idx[k]]), taps[i].w[k]));
          }
          dp[(size_t)ch * dplane + pix] = Cvt<T>::from_f(acc);
        }
      }
    }
    __syncthreads();  // everyone done with this buffer before it is refilled
    if (threadIdx.x == 0 && st + 2 < n_stages) issue(st + 2);
  }
}

// ---------------------------------------------------------------------------------------------------
// quad variant of the staged kernel (the default whenever the output width is a multiple of 4): thread <-> QPT groups
// of 4 CONSECUTIVE output pixels, so every store is one 16-byte (fp32) / 8-byte (16-bit) vector and a group without
// any live pixel — ~80 % of a p2e output, whose mask is false outside the camera frustum — costs one predicate and one
// vector store of zeros per channel. The output plane is cut into tiles of at most 4*QPT*256 pixels (blockIdx.z), so
// planes of any size keep their source in shared memory. `src_repeat` consecutive batch elements share one source
// image (B cameras looking at B / src_repeat panoramas: the source is then read once from HBM and again from L2).
// ---------------------------------------------------------------------------------------------------
template <typename T> struct Quad;
template <> struct Quad<float> {
  static __device__ __forceinline__ void store(float* p, const float* o) {
    __stcs(reinterpret_cast<float4*>(p), make_float4(o[0], o[1], o[2], o[3]));
  }
};
template <> struct Quad<__half> {
  static __device__ __forceinline__ void store(__half* p, const float* o) {
    const __half2 a = __floats2half2_rn(o[0], o[1]), b = __floats2half2_rn(o[2], o[3]);
    __stcs(reinterpret_cast<uint2*>(p), make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b)));
  }
};
template <> struct Quad<__nv_bfloat16> {
  static __device__ __forceinline__ void store(__nv_bfloat16* p, const float* o) {
    const __nv_bfloat162 a = __floats2bfloat162_rn(o[0], o[1]), b = __floats2bfloat162_rn(o[2], o[3]);
    __stcs(reinterpret_cast<uint2*>(p), make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b)));
  }
};

template <typename T, bool P2E, int QPT>
__global__ void __launch_bounds__(STG_THREADS, 2)
resample_quad_kernel(const T* __restrict__ src, T* __restrict__ dst, uint8_t* __restrict__ mask_out, int C,
                     int Hs, int Ws, int Hd, int Wd, const double* __restrict__ cams, int cam_stride, int mode,
                     int ch_per_cta, int ch_per_stage, int src_repeat, int tile_px) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  const int splane = Hs * Ws, dplane = Hd * Wd;
  const uint32_t stage_bytes = uint32_t(ch_per_stage) * splane * sizeof(T);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem);
  T* buf0 = reinterpret_cast<T*>(smem + 128);
  T* buf1 = reinterpret_cast<T*>(smem + 128 + ((stage_bytes + 127) & ~127u));

  const int b = blockIdx.y;
  const int c_begin = blockIdx.x * ch_per_cta;
  const int c_end = min(C, c_begin + ch_per_cta);
  const int n_stages = (c_end - c_begin + ch_per_stage - 1) / ch_per_stage;
  const int pix0 = blockIdx.z * tile_px;
  const int pix_end = min(dplane, pix0 + tile_px);
  const T* sbase = src + (size_t)(b / src_repeat) * C * splane;

  if (threadIdx.x == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto issue = [&](int st) {
    const int ca = c_begin + st * ch_per_stage;
    const int nch = min(ch_per_stage, c_end - ca);
    const uint32_t bytes = uint32_t(nch) * splane * sizeof(T);
    mbar_expect_tx(&bars[st & 1], bytes);
    bulk_load_1d((st & 1) ? buf1 : buf0, sbase + (size_t)ca * splane, bytes, &bars[st & 1]);
  };
  if (threadIdx.x == 0) {
    issue(0);
    if (n_stages > 1) issue(1);
  }

  const double* cam = cams + (size_t)b * cam_stride * PF_CAM_DOUBLES;
  Taps taps[QPT][4];
  bool any_live[QPT];
#pragma unroll
  for (int i = 0; i < QPT; ++i) {
    const int q0 = pix0 + 4 * (threadIdx.x + i * STG_THREADS);
    any_live[i] = false;
    uint32_t mbits = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int pix = q0 + j;
      bool live = pix < pix_end;
      float px = 0.f, py = 0.f;
      if (live) {
        const int r = pix / Wd, c = pix - r * Wd;
        if constexpr (P2E) {
          bool m;
          p2e_grid(cam, r, c, Hd, Wd, Hs, Ws, px, py, m);
          live = m;
          mbits |= (m ? 1u : 0u) << (8 * j);
        } else {
          e2p_grid(cam, r, c, Hd, Wd, Hs, Ws, px, py);
        }
      }
      make_taps(px, py, Hs, Ws, mode, live, taps[i][j]);
#pragma unroll
      for (int k = 0; k < 4; ++k) any_live[i] = any_live[i] || taps[i][j].idx[k] >= 0;
    }
    if constexpr (P2E) {
      if (mask_out && blockIdx.x == 0 && q0 < pix_end)
        *reinterpret_cast<uint32_t*>(mask_out + (size_t)b * dplane + q0) = mbits;
    }
  }

  for (int st = 0; st < n_stages; ++st) {
    mbar_wait(&bars[st & 1], (st >> 1) & 1);
    const T* sb = (st & 1) ? buf1 : buf0;
    const int ca = c_begin + st * ch_per_stage;
    const int nch = min(ch_per_stage, c_end - ca);
    T* dp = dst + ((size_t)b * C + ca) * dplane;
    for (int ch = 0; ch < nch; ++ch) {
      const T* sp = sb + (size_t)ch * splane;
#pragma unroll
      for (int i = 0; i < QPT; ++i) {
        const int q0 = pix0 + 4 * (threadIdx.x + i * STG_THREADS);
        if (q0 < pix_end) {
          float o[4] = {0.f, 0.f, 0.f, 0.f};
          if (any_live[i]) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                if (taps[i][j].idx[k] >= 0)
                  o[j] = __fadd_rn(o[j], __fmul_rn(Cvt<T>::to_f(sp[taps[i][j].idx[k]]), taps[i][j].w[k]));
              }
            }
          }
          Quad<T>::store(dp + (size_t)ch * dplane + q0, o);
        }
      }
    }
    __syncthreads();  // everyone done with this buffer before it is refilled
    if (threadIdx.x == 0 && st + 2 < n_stages) issue(st + 2);
  }
}

template <typename T, bool P2E>
static int launch_resample(const void* src, void* dst, uint8_t* mask, int B, int C, int Hs, int Ws, int Hd, int Wd,
                           const double* cams, int cam_stride, int mode, int src_repeat, cudaStream_t st) {
  const int dplane = Hd * Wd;
  const size_t plane_bytes = (size_t)Hs * Ws * sizeof(T);
  const bool aligned = (plane_bytes % 16 == 0) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
  // quad path: vector stores need a 4-pixel-aligned output plane; the mask is written 4 bytes at a time
  if (aligned && plane_bytes <= 48 * 1024 && C >= 4 && Wd % 4 == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0 &&
      (!mask || (reinterpret_cast<uintptr_t>(mask) & 3) == 0) && B <= 65535) {
    int ch_per_stage = (int)((48 * 1024) / plane_bytes);
    if (ch_per_stage > 16) ch_per_stage = 16;
    const int max_tile = 4 * 2 * STG_THREADS;  // QPT = 2
    const int tiles = (dplane + max_tile - 1) / max_tile;
    int tile_px = (dplane + tiles - 1) / tiles;
    tile_px = (tile_px + 3) & ~3;
    const int qpt = (tile_px + 4 * STG_THREADS - 1) / (4 * STG_THREADS);
    // exactly ONE wave of co-resident CTAs (2 per SM) when the problem allows it
    int ctas_per_bt = (sm_count() * 2) / (B * tiles);
    if (ctas_per_bt < 1) ctas_per_bt = 1;
    int ch_per_cta = (C + ctas_per_bt - 1) / ctas_per_bt;
    ch_per_cta = ((ch_per_cta + ch_per_stage - 1) / ch_per_stage) * ch_per_stage;
    const int grid_x = (C + ch_per_cta - 1) / ch_per_cta;
    const size_t stage_bytes = ((size_t)ch_per_stage * plane_bytes + 127) & ~size_t(127);
    const size_t smem = 128 + 128 + 2 * stage_bytes;
    dim3 grid(grid_x, B, tiles);
#define PF_LAUNCH_QUAD(QPT)                                                                                       \
  {                                                                                                               \
    auto kern = resample_quad_kernel<T, P2E, QPT>;                                                                \
    int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),       \
                        "cudaFuncSetAttribute(resample)");                                                        \
    if (rc) return rc;                                                                                            \
    kern<<<grid, STG_THREADS, smem, st>>>(static_cast<const T*>(src), static_cast<T*>(dst), mask, C, Hs, Ws, Hd,  \
                                          Wd, cams, cam_stride, mode, ch_per_cta, ch_per_stage, src_repeat,       \
                                          tile_px);                                                               \
  }
    if (qpt <= 1) PF_LAUNCH_QUAD(1)
    else PF_LAUNCH_QUAD(2)
#undef PF_LAUNCH_QUAD
    PF_CHECK_LAUNCH("resample_quad_kernel");
    return PF_OK;
  }
  if (src_repeat != 1) {
    set_error("pf_e2p/pf_p2e: src_repeat > 1 needs the staged quad path (output width %% 4 == 0, source plane <= 48 KB)");
    return PF_ERR_UNSUPPORTED;
  }
  // staged path: plane must fit twice (double buffer) in <= ~96 KB so two CTAs share an SM, <= 8 pixels/thread
  if (aligned && plane_bytes <= 48 * 1024 && dplane <= 8 * STG_THREADS && C >= 4) {
    int ch_per_stage = (int)((48 * 1024) / plane_bytes);
    if (ch_per_stage < 1) ch_per_stage = 1;
    if (ch_per_stage > 16) ch_per_stage = 16;
    // enough CTAs to fill every SM twice, but long enough channel runs to amortise the fp64 grid math
    int ch_per_cta = C;
    // exactly ONE wave of co-resident CTAs (2 per SM): a small overshoot of those slots costs a whole second wave
    const int want_ctas = sm_count() * 2;
    int ctas_per_b = want_ctas / B;
    if (ctas_per_b < 1) ctas_per_b = 1;
    ch_per_cta = (C + ctas_per_b - 1) / ctas_per_b;
    ch_per_cta = ((ch_per_cta + ch_per_stage - 1) / ch_per_stage) * ch_per_stage;
    if (ch_per_cta > C) ch_per_cta = ((C + ch_per_stage - 1) / ch_per_stage) * ch_per_stage;
    const int grid_x = (C + ch_per_cta - 1) / ch_per_cta;
    const size_t stage_bytes = ((size_t)ch_per_stage * plane_bytes + 127) & ~size_t(127);
    const size_t smem = 128 + 128 + 2 * stage_bytes;
    dim3 grid(grid_x, B);
    const int ppt = (dplane + STG_THREADS - 1) / STG_THREADS;
#define PF_LAUNCH_STG(PPT)                                                                                        \
  {                                                                                                               \
    auto kern = resample_staged_kernel<T, P2E, PPT>;                                                              \
    int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),       \
                        "cudaFuncSetAttribute(resample)");                                                        \
    if (rc) return rc;                                                                                            \
    kern<<<grid, STG_THREADS, smem, st>>>(static_cast<const T*>(src), static_cast<T*>(dst), mask, C, Hs, Ws, Hd,  \
                                          Wd, cams, cam_stride, mode, ch_per_cta, ch_per_stage);                  \
  }
    if (ppt <= 1) PF_LAUNCH_STG(1)
    else if (ppt <= 2) PF_LAUNCH_STG(2)
    else if (ppt <= 4) PF_LAUNCH_STG(4)
    else PF_LAUNCH_STG(8)
#undef PF_LAUNCH_STG
    PF_CHECK_LAUNCH("resample_staged_kernel");
    return PF_OK;
  }
  int ch_per_slice = C;
  {
    const long long blocks_xy = (long long)((dplane + 255) / 256) * B;
    int slices = (int)(((long long)sm_count() * 8 + blocks_xy - 1) / blocks_xy);
    if (slices < 1) slices = 1;
    if (slices > C) slices = C;
    ch_per_slice = (C + slices - 1) / slices;
  }
  dim3 grid((dplane + 255) / 256, (C + ch_per_slice - 1) / ch_per_slice, B);
  resample_direct_kernel<T, P2E><<<grid, 256, 0, st>>>(static_cast<const T*>(src), static_cast<T*>(dst), mask, C,
                                                       Hs, Ws, Hd, Wd, cams, cam_stride, mode, ch_per_slice);
  PF_CHECK_LAUNCH("resample_direct_kernel");
  return PF_OK;
}

template <bool P2E>
static int dispatch_resample(const void* src, void* dst, uint8_t* mask, int dtype, int B, int C, int Hs, int Ws,
                             int Hd, int Wd, const double* cams, int cam_stride, int mode, int src_repeat, void* stream) {
  const char* name = P2E ? "pf_p2e" : "pf_e2p";
  PF_CHECK_ARG(src && dst && cams, "%s: null pointer", name);
  PF_CHECK_ARG(B > 0 && C > 0 && Hs > 0 && Ws > 0 && Hd > 0 && Wd > 0, "%s: empty shape", name);
  PF_CHECK_ARG(B <= 65535, "%s: batch %d exceeds grid limit", name, B);
  PF_CHECK_ARG(cam_stride == 0 || cam_stride == 1, "%s: cam_stride must be 0 or 1", name);
  // reference: choose_mode() accepts 'bilinear'/'nearest' for tensors, ValueError otherwise (utils.py:5-15)
  PF_CHECK_ARG(mode == 0 || mode == 1, "%s: mode must be one of [bilinear, nearest]", name);
  PF_CHECK_ARG(src_repeat >= 1 && B % src_repeat == 0, "%s: src_repeat=%d must divide the batch %d", name, src_repeat, B);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (dtype) {
    case PF_F32:
      return launch_resample<float, P2E>(src, dst, mask, B, C, Hs, Ws, Hd, Wd, cams, cam_stride, mode, src_repeat, st);
    case PF_F16:
      return launch_resample<__half, P2E>(src, dst, mask, B, C, Hs, Ws, Hd, Wd, cams, cam_stride, mode, src_repeat, st);
    case PF_BF16:
      return launch_resample<__nv_bfloat16, P2E>(src, dst, mask, B, C, Hs, Ws, Hd, Wd, cams, cam_stride, mode, src_repeat, st);
  }
  set_error("%s: unknown dtype %d", name, dtype);
  return PF_ERR_INVALID;
}

}  // namespace pf

// ---------------------------------------------------------------------------------------------------
// py360convert convention (external/py360convert/e2p.py:6-43, utils.py:104-132): the pixel-space equirect -> perspective
// resampling of the dataset path (utils/pano.py:160-161, dataset/PanoDataset.py:138). Channels-last images [H, W, C],
// half-pixel centres, longitude wrap-around, pole rows padded with the first / last row rolled by W/2, scipy's legacy
// 'wrap' boundary (period n - 1), float64 grid math, integer images rounded half up. thread <-> output pixel.
// ---------------------------------------------------------------------------------------------------
namespace pf {

__device__ __forceinline__ double py360_wrap(double c, int n) {
  const double sz = double(n - 1);
  if (c < 0.0) c += sz * double((long long)(-c / sz) + 1);
  else if (c > sz) c -= sz * double((long long)(c / sz));
  return c;
}

// row r of the padded image [H + 2][W]: r < H plain, r == H the last row rolled by W/2, r == H+1 the first row rolled
__device__ __forceinline__ long long py360_src_index(int r, int x, int H, int W) {
  if (r < H) return (long long)r * W + x;
  const int xr = (x - W / 2 + W) % W;  // np.roll(row, W // 2)[x] == row[(x - W//2) mod W]
  return (long long)(r == H ? H - 1 : 0) * W + xr;
}

// utils.py:125-132 sample_equirec: scipy map_coordinates([cy, cx], order 1 or 0, mode='wrap') over the equirect image
// with its two pole rows appended, every channel of one output pixel. Shared by e2p and e2c.
template <typename T>
__device__ __forceinline__ void py360_sample_equirec(const T* __restrict__ src, int H, int W, int C, double cx,
                                                     double cy, int nearest, T* __restrict__ out) {
  const int HP = H + 2;
  const double y = py360_wrap(cy, HP), x = py360_wrap(cx, W);
  if (nearest) {
    int yi = int(floor(y + 0.5)), xi = int(floor(x + 0.5));
    if (yi > HP - 1) yi -= HP - 1;
    if (xi > W - 1) xi -= W - 1;
    const T* sp = src + py360_src_index(yi, xi, H, W) * C;
    for (int c = 0; c < C; ++c) out[c] = sp[c];
    return;
  }
  const int y0 = int(floor(y)), x0 = int(floor(x));
  const double ty = y - double(y0), tx = x - double(x0);
  int y1 = y0 + 1, x1 = x0 + 1;
  if (y1 > HP - 1) y1 -= HP - 1;
  if (x1 > W - 1) x1 -= W - 1;
  const T* p00 = src + py360_src_index(y0, x0, H, W) * C;
  const T* p01 = src + py360_src_index(y0, x1, H, W) * C;
  const T* p10 = src + py360_src_index(y1, x0, H, W) * C;
  const T* p11 = src + py360_src_index(y1, x1, H, W) * C;
  const double w00 = (1.0 - ty) * (1.0 - tx), w01 = (1.0 - ty) * tx, w10 = ty * (1.0 - tx), w11 = ty * tx;
  for (int c = 0; c < C; ++c) {
    const double val = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(double(p00[c]), w00), __dmul_rn(double(p01[c]), w01)),
                                           __dmul_rn(double(p10[c]), w10)), __dmul_rn(double(p11[c]), w11));
    if constexpr (sizeof(T) == 1) {
      const double r = floor(val + 0.5);
      out[c] = T(r < 0.0 ? 0.0 : (r > 255.0 ? 255.0 : r));
    } else {
      out[c] = T(val);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
e2p_py360_kernel(const T* __restrict__ src, T* __restrict__ dst, int H, int W, int C, int h, int w,
                 const double* __restrict__ cams, int nearest) {
  const int cam_i = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= h * w) return;
  const int i = pix / w, j = pix - i * w;
  const double* cam = cams + (size_t)cam_i * PF_CAM360_DOUBLES;
  // xyzpers: float32 linspace grids, z = 1, then three float64 rotations applied to the ROW vector
  double v[3] = {double(float(np_linspace(-cam[27], cam[27], w, j))), -double(float(np_linspace(-cam[28], cam[28], h, i))), 1.0};
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double* R = cam + 9 * r;
    double o[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
      o[k] = __dadd_rn(__dadd_rn(__dmul_rn(v[0], R[k]), __dmul_rn(v[1], R[3 + k])), __dmul_rn(v[2], R[6 + k]));
    v[0] = o[0]; v[1] = o[1]; v[2] = o[2];
  }
  const double uu = atan2(v[0], v[2]);
  const double vv = atan2(v[1], sqrt(v[0] * v[0] + v[2] * v[2]));
  const double cx = (uu / (2.0 * M_PI) + 0.5) * double(W) - 0.5;
  const double cy = (-vv / M_PI + 0.5) * double(H) - 0.5;
  py360_sample_equirec(src, H, W, C, cx, cy, nearest, dst + ((size_t)cam_i * h * w + pix) * C);
}

// numpy float32 math restated on the device: each float32 ufunc result is the float64 function rounded to float
// (correctly rounded but for rare double-rounding ties; numpy's own float32 kernels are within about one ulp of that).
__device__ __forceinline__ float f32_tan(float a) { return float(tan(double(a))); }
__device__ __forceinline__ float f32_sin(float a) { return float(sin(double(a))); }
__device__ __forceinline__ float f32_cos(float a) { return float(cos(double(a))); }
__device__ __forceinline__ float f32_atan2(float y, float x) { return float(atan2(double(y), double(x))); }

// np.linspace(start, stop, n, dtype=float32)[i]: float64 i * step, then + start, each rounded (no contraction into
// an FMA), then cast to float32; the last sample is `stop` exactly.
__device__ __forceinline__ float np_linspace_f32(double start, double stop, int n, int i) {
  if (n == 1) return float(start);
  if (i == n - 1) return float(stop);
  return float(__dadd_rn(__dmul_rn(double(i), (stop - start) / double(n - 1)), start));
}

// e2c.py:6-40: thread <-> one pixel of the horizon cube [fw, 6 fw, C]. xyzcube -> xyz2uv -> uv2coor in float32
// (utils.py:5-37,82-114), then the e2p sampler.
template <typename T>
__global__ void __launch_bounds__(256)
e2c_py360_kernel(const T* __restrict__ src, T* __restrict__ dst, int H, int W, int C, int fw, int nearest) {
  const int ow = 6 * fw;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= fw * ow) return;
  const int r = pix / ow, col = pix - r * ow;
  const int face = col / fw, c = col - face * fw;
  const float a = np_linspace_f32(-0.5, 0.5, fw, c), b = -np_linspace_f32(-0.5, 0.5, fw, r);
  float x, y, z;
  switch (face) {  // F R B L U D: the face's plane coordinate is +-0.5, the grid (a, b) spans the other two axes
    case 0: x = a; y = b; z = 0.5f; break;
    case 1: z = a; y = b; x = 0.5f; break;
    case 2: x = a; y = b; z = -0.5f; break;
    case 3: z = a; y = b; x = -0.5f; break;
    case 4: x = a; z = b; y = 0.5f; break;
    default: x = a; z = b; y = -0.5f; break;
  }
  const float u = f32_atan2(x, z);
  const float v = f32_atan2(y, __fsqrt_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(z, z))));
  const float cx = __fsub_rn(__fmul_rn(__fadd_rn(__fdiv_rn(u, float(2.0 * M_PI)), 0.5f), float(W)), 0.5f);
  const float cy = __fsub_rn(__fmul_rn(__fadd_rn(__fdiv_rn(-v, float(M_PI)), 0.5f), float(H)), 0.5f);
  py360_sample_equirec(src, H, W, C, double(cx), double(cy), nearest, dst + (size_t)pix * C);
}

// Pixel of the horizon cube behind sample (y, x) of padded face f of sample_cubefaces (utils.py:135-173), or -1 for
// one of its zero pads. Inside the face: the R / B column flip and the U row flip. On the two pad rows / columns: the
// host's border table, per face [row fw][fw], [row fw+1][fw], [col fw][fw+2], [col fw+1][fw+2].
__device__ __forceinline__ int c2e_src(int f, int y, int x, int fw, const int* __restrict__ border) {
  if (y < fw && x < fw) {
    if (f == 1 || f == 2) x = fw - 1 - x;
    if (f == 4) y = fw - 1 - y;
    return y * 6 * fw + f * fw + x;
  }
  const int* bt = border + (size_t)f * (4 * fw + 4);
  return __ldg(x < fw ? bt + (y - fw) * fw + x : bt + 2 * fw + (x - fw) * (fw + 2) + y);
}

template <typename T>
__device__ __forceinline__ double c2e_tap(const T* __restrict__ cube, int idx, int C, int ch) {
  return idx < 0 ? 0.0 : double(cube[(size_t)idx * C + ch]);
}

// c2e.py:6-64: thread <-> one equirect pixel, every channel. The face comes from the host's ceiling-row table
// (equirect_facetype, utils.py:47-64), the face coordinates from float32 math as numpy evaluates it, the clip and
// scale and the bilinear sum in float64 in scipy's term order ((v * wy) * wx, summed row-major) — the padded faces
// are float64, so the result is too.
template <typename T>
__global__ void __launch_bounds__(256)
c2e_py360_kernel(const T* __restrict__ cube, double* __restrict__ dst, int fw, int C, int h, int w,
                 const int* __restrict__ ceil_rows, const int* __restrict__ border, int nearest) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= h * w) return;
  const int i = pix / w, j = pix - i * w;
  // face type: the four side faces rolled by 3w/8, ceiling rows [0, ceil) are U, their mirror image D
  const int q4 = w / 4;
  const int xs = (j - 3 * w / 8 + w) % w;
  const int ceil_i = __ldg(ceil_rows + xs % q4);
  int face = xs / q4;
  if (i < ceil_i) face = 4;
  if (h - 1 - i < ceil_i) face = 5;
  // equirect_uvgrid: float32 linspace; v's halving is exact
  const float u = np_linspace_f32(-M_PI, M_PI, w, j);
  const float v = __fmul_rn(np_linspace_f32(M_PI, -M_PI, h, i), 0.5f);
  float fx, fy;
  if (face < 4) {
    const float a = __fsub_rn(u, float(__dmul_rn(M_PI, double(face)) * 0.5));
    fx = __fmul_rn(0.5f, f32_tan(a));
    fy = __fdiv_rn(__fmul_rn(-0.5f, f32_tan(v)), f32_cos(a));
  } else {
    const float cc = __fmul_rn(0.5f, f32_tan(__fsub_rn(float(M_PI / 2), face == 4 ? v : fabsf(v))));
    fx = __fmul_rn(cc, f32_sin(u));
    fy = __fmul_rn(face == 4 ? cc : -cc, f32_cos(u));
  }
  // clip to the face and scale to [0, fw]: always inside the (fw + 2)-wide padded face, so the 'wrap' boundary
  // never applies and the +1 neighbour is at most index fw + 1
  const double X = __dmul_rn(__dadd_rn(fmin(fmax(double(fx), -0.5), 0.5), 0.5), double(fw));
  const double Y = __dmul_rn(__dadd_rn(fmin(fmax(double(fy), -0.5), 0.5), 0.5), double(fw));
  double* out = dst + (size_t)pix * C;
  if (nearest) {
    const int idx = c2e_src(face, int(floor(Y + 0.5)), int(floor(X + 0.5)), fw, border);
    for (int ch = 0; ch < C; ++ch) out[ch] = c2e_tap(cube, idx, C, ch);
    return;
  }
  const int y0 = int(floor(Y)), x0 = int(floor(X));
  const double ty = Y - double(y0), tx = X - double(x0);
  const int i00 = c2e_src(face, y0, x0, fw, border), i01 = c2e_src(face, y0, x0 + 1, fw, border);
  const int i10 = c2e_src(face, y0 + 1, x0, fw, border), i11 = c2e_src(face, y0 + 1, x0 + 1, fw, border);
  const double wy0 = 1.0 - ty, wx0 = 1.0 - tx;
  for (int ch = 0; ch < C; ++ch) {
    double acc = __dmul_rn(__dmul_rn(c2e_tap(cube, i00, C, ch), wy0), wx0);
    acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(c2e_tap(cube, i01, C, ch), wy0), tx));
    acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(c2e_tap(cube, i10, C, ch), ty), wx0));
    out[ch] = __dadd_rn(acc, __dmul_rn(__dmul_rn(c2e_tap(cube, i11, C, ch), ty), tx));
  }
}

}  // namespace pf

extern "C" int pf_e2p_py360(const void* src, void* dst, int is_u8, int H, int W, int C, int h, int w, const double* cams,
                            int num_cams, int mode, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(src && dst && cams, "pf_e2p_py360: null pointer");
  PF_CHECK_ARG(H > 1 && W > 1 && C > 0 && h > 0 && w > 0 && num_cams > 0 && num_cams <= 65535, "pf_e2p_py360: bad shape");
  // py360convert raises NotImplementedError('unknown mode') for anything but bilinear / nearest (e2p.py:21-26)
  if (mode != 0 && mode != 1) {
    set_error("pf_e2p_py360: unknown mode");
    return PF_ERR_UNSUPPORTED;
  }
  dim3 grid((h * w + 255) / 256, num_cams);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (is_u8)
    e2p_py360_kernel<uint8_t><<<grid, 256, 0, st>>>(static_cast<const uint8_t*>(src), static_cast<uint8_t*>(dst), H, W, C, h, w, cams, mode);
  else
    e2p_py360_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float*>(src), static_cast<float*>(dst), H, W, C, h, w, cams, mode);
  PF_CHECK_LAUNCH("e2p_py360_kernel");
  return PF_OK;
}

extern "C" int pf_c2e_py360(const void* cube, double* dst, int is_u8, int face_w, int C, int h, int w,
                            const int* ceil_rows, const int* border, int mode, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(cube && dst && ceil_rows && border, "pf_c2e_py360: null pointer");
  PF_CHECK_ARG(face_w > 0 && C > 0 && h > 0 && w > 0, "pf_c2e_py360: empty shape");
  // c2e.py:26 asserts w % 8 == 0: the face-type roll by 3w/8 and the w/4 ceiling table need it
  PF_CHECK_ARG(w % 8 == 0, "pf_c2e_py360: w = %d must be a multiple of 8", w);
  PF_CHECK_ARG((long long)h * w < (1LL << 31) && (long long)face_w * 6 * face_w < (1LL << 31),
               "pf_c2e_py360: %d x %d panorama or face_w %d exceeds 2^31 pixels", h, w, face_w);
  if (mode != 0 && mode != 1) {
    set_error("pf_c2e_py360: unknown mode");
    return PF_ERR_UNSUPPORTED;
  }
  const unsigned blocks = unsigned(((long long)h * w + 255) / 256);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (is_u8)
    c2e_py360_kernel<uint8_t><<<blocks, 256, 0, st>>>(static_cast<const uint8_t*>(cube), dst, face_w, C, h, w, ceil_rows, border, mode);
  else
    c2e_py360_kernel<float><<<blocks, 256, 0, st>>>(static_cast<const float*>(cube), dst, face_w, C, h, w, ceil_rows, border, mode);
  PF_CHECK_LAUNCH("c2e_py360_kernel");
  return PF_OK;
}

extern "C" int pf_e2c_py360(const void* src, void* dst, int is_u8, int H, int W, int C, int face_w, int mode,
                            void* stream) {
  using namespace pf;
  PF_CHECK_ARG(src && dst, "pf_e2c_py360: null pointer");
  PF_CHECK_ARG(H > 1 && W > 1 && C > 0 && face_w > 0, "pf_e2c_py360: bad shape");
  PF_CHECK_ARG((long long)face_w * 6 * face_w < (1LL << 31) && (long long)(H + 2) * W < (1LL << 31),
               "pf_e2c_py360: face_w %d or %d x %d image exceeds 2^31 pixels", face_w, H, W);
  if (mode != 0 && mode != 1) {
    set_error("pf_e2c_py360: unknown mode");
    return PF_ERR_UNSUPPORTED;
  }
  const unsigned blocks = unsigned(((long long)face_w * 6 * face_w + 255) / 256);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (is_u8)
    e2c_py360_kernel<uint8_t><<<blocks, 256, 0, st>>>(static_cast<const uint8_t*>(src), static_cast<uint8_t*>(dst), H, W, C, face_w, mode);
  else
    e2c_py360_kernel<float><<<blocks, 256, 0, st>>>(static_cast<const float*>(src), static_cast<float*>(dst), H, W, C, face_w, mode);
  PF_CHECK_LAUNCH("e2c_py360_kernel");
  return PF_OK;
}

extern "C" int pf_e2p(const void* src, void* dst, int dtype, int B, int C, int He, int We, int h, int w,
                      const double* cams, int cam_stride, int mode, void* stream) {
  return pf::dispatch_resample<false>(src, dst, nullptr, dtype, B, C, He, We, h, w, cams, cam_stride, mode, 1, stream);
}

extern "C" int pf_e2p_shared(const void* src, void* dst, int dtype, int B, int src_repeat, int C, int He, int We, int h,
                             int w, const double* cams, int cam_stride, int mode, void* stream) {
  return pf::dispatch_resample<false>(src, dst, nullptr, dtype, B, C, He, We, h, w, cams, cam_stride, mode, src_repeat,
                                      stream);
}

extern "C" int pf_p2e(const void* src, void* dst, uint8_t* mask, int dtype, int B, int C, int hp, int wp, int He,
                      int We, const double* cams, int cam_stride, int mode, void* stream) {
  return pf::dispatch_resample<true>(src, dst, mask, dtype, B, C, hp, wp, He, We, cams, cam_stride, mode, 1, stream);
}
