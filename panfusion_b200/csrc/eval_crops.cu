// Evaluation crops and the ground-truth resize of EvalPanoGen (models/pano/EvalPanoGen.py:99-169,
// dataset/PanoDataset.py:140), uint8 in and uint8 out.
//
// pf_eval_crops is e2p (e2p.py:54-76) composed with the dtype conversions around it, so no fp32 crop tensor exists:
// the grid is e2p_grid and the taps make_taps, shared with pf_e2p (sphere_grid.cuh), and the taps are accumulated in
// the order and with the roundings of pf_e2p's fp32 path. normalize: texel float(x) / 255 (IEEE division, as torch
// computes `pano.float() / 255` on the CPU), store uint8(trunc(v * 255)) (the conversion of pf_inception_prep /
// pf_clip_prep for fp32 input). raw: texel float(x), store uint8(trunc(v)) (`.to(torch.uint8)`).
#include "sphere_grid.cuh"

namespace pf {

// thread <-> one output pixel of one crop, all three channels; grid (pixel blocks, crops)
__global__ void __launch_bounds__(256)
eval_crops_kernel(const uint8_t* __restrict__ src, int H, int W, int crops_per_pano, int h, int w,
                  const double* __restrict__ cams, int normalize, uint8_t* __restrict__ dst) {
  const int n = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= h * w) return;
  const int r = pix / w, c = pix - r * w;
  float px, py;
  e2p_grid(cams + (size_t)n * PF_CAM_DOUBLES, r, c, h, w, H, W, px, py);
  Taps t;
  make_taps(px, py, H, W, 0, true, t);
  const size_t splane = (size_t)H * W, dplane = (size_t)h * w;
  const uint8_t* sp = src + (size_t)(n / crops_per_pano) * 3 * splane;
  uint8_t* dp = dst + (size_t)n * 3 * dplane + pix;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (t.idx[k] >= 0) {
        const float x = float(__ldg(sp + t.idx[k]));
        acc = __fadd_rn(acc, __fmul_rn(normalize ? __fdiv_rn(x, 255.f) : x, t.w[k]));
      }
    }
    const float v = normalize ? __fmul_rn(acc, 255.f) : acc;
    dp[(size_t)ch * dplane] = uint8_t(truncf(fminf(fmaxf(v, 0.f), 255.f)));
    sp += splane;
  }
}

// cv2.resize(INTER_AREA) by exactly 2 on both axes (OpenCV 4.x resizeAreaFast_ for uint8): (a + b + c + d + 2) >> 2.
// thread <-> one output pixel of one plane
__global__ void __launch_bounds__(256)
resize_area2_kernel(const uint8_t* __restrict__ src, long long planes, int H, int W, uint8_t* __restrict__ dst) {
  const int ho = H / 2, wo = W / 2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= planes * ho * wo) return;
  const long long p = i / ((long long)ho * wo);
  const int rem = int(i - p * ho * wo);
  const int y = rem / wo, x = rem - y * wo;
  const uint8_t* s = src + (size_t)p * H * W + (size_t)(2 * y) * W + 2 * x;
  dst[i] = uint8_t((int(s[0]) + int(s[1]) + int(s[W]) + int(s[W + 1]) + 2) >> 2);
}

}  // namespace pf

extern "C" int pf_eval_crops(const uint8_t* src, int P, int H, int W, int crops_per_pano, int N, int h, int w,
                             const double* cams, int normalize, uint8_t* dst, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(src && dst && cams, "pf_eval_crops: null pointer");
  PF_CHECK_ARG(P > 0 && H > 1 && W > 1 && h > 0 && w > 0 && crops_per_pano > 0, "pf_eval_crops: empty shape");
  PF_CHECK_ARG(N > 0 && N <= 65535, "pf_eval_crops: N = %d crops must be in [1, 65535]", N);
  PF_CHECK_ARG((long long)N <= (long long)P * crops_per_pano,
               "pf_eval_crops: %d crops of %d per panorama read past the %d panoramas", N, crops_per_pano, P);
  PF_CHECK_ARG((long long)H * W < (1LL << 31) && (long long)h * w < (1LL << 31),
               "pf_eval_crops: an image exceeds 2^31 pixels");
  PF_CHECK_ARG(normalize == 0 || normalize == 1, "pf_eval_crops: normalize must be 0 or 1");
  dim3 grid((unsigned)((h * w + 255) / 256), N);
  eval_crops_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(src, H, W, crops_per_pano, h, w, cams,
                                                                         normalize, dst);
  PF_CHECK_LAUNCH("eval_crops_kernel");
  return PF_OK;
}

extern "C" int pf_resize_area2_u8(const uint8_t* src, int B, int C, int H, int W, int Ho, int Wo, uint8_t* dst,
                                  void* stream) {
  using namespace pf;
  PF_CHECK_ARG(src && dst, "pf_resize_area2_u8: null pointer");
  PF_CHECK_ARG(B > 0 && C > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0, "pf_resize_area2_u8: empty shape");
  const long long planes = (long long)B * C;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (Ho == H && Wo == W) {
    return check_cuda(cudaMemcpyAsync(dst, src, (size_t)planes * H * W, cudaMemcpyDeviceToDevice, st),
                      "pf_resize_area2_u8: copy");
  }
  // other factors round half to even in OpenCV's INTER_AREA, and non-integer ones weight partial pixels
  if (H != 2 * Ho || W != 2 * Wo) {
    set_error("pf_resize_area2_u8: %d x %d -> %d x %d is not a factor-2 downsampling", H, W, Ho, Wo);
    return PF_ERR_UNSUPPORTED;
  }
  const long long n = planes * Ho * Wo;
  resize_area2_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, planes, H, W, dst);
  PF_CHECK_LAUNCH("resize_area2_kernel");
  return PF_OK;
}
