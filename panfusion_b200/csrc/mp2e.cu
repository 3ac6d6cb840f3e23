// Panorama stitching of MVDiffusion (external/Perspective_and_Equirectangular/mp2e.py, p2e.py numpy path), all views of
// one panorama in one launch, uint8 in and out.
//
// For every view, p2e warps the uint8 image and a horizontal weight ramp (0 -> 1 -> 0 across the width) onto the
// panorama with cv2.remap and multiplies both by the frustum mask; the panorama is sum(img * w) / sum(w) truncated to
// uint8, 255 where no view reaches. The reference calls mp2e without a mode, and its numpy path then hands
// interpolation=None to cv2.remap, which is INTER_NEAREST: the map coordinate (float32) is rounded half to even and
// wraps around the image (BORDER_WRAP). The grid is p2e_grid (fp64, rounded to float32 like lon.astype(np.float32)).
// The blurred mask mp2e computes is never used and is not reproduced. Sums run in fp64 in view order, like numpy.
#include "sphere_grid.cuh"

namespace pf {

__device__ __forceinline__ int wrap_index(int v, int n) {
  v %= n;
  return v < 0 ? v + n : v;
}

// np.linspace(0, 1, w // 2) on the left half, np.linspace(1, 0, w // 2) on the right half (mp2e.py:14-17)
__device__ __forceinline__ double ramp(int x, int w) {
  const int h = w / 2;
  if (x < h) return np_linspace(0.0, 1.0, h, x);
  if (x < 2 * h) return np_linspace(1.0, 0.0, h, x - h);
  return 0.0;
}

// thread <-> one panorama pixel, every channel
__global__ void __launch_bounds__(256)
mp2e_kernel(const uint8_t* __restrict__ views, int m, int hp, int wp, int C, const double* __restrict__ cams, int He,
            int We, uint8_t* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= He * We) return;
  const int i = idx / We, j = idx % We;
  double num[4] = {0.0, 0.0, 0.0, 0.0};
  double den = 0.0;
  for (int v = 0; v < m; ++v) {
    float px, py;
    bool mask;
    p2e_grid(cams + (size_t)v * PF_CAM_DOUBLES, i, j, He, We, hp, wp, px, py, mask);
    const int x = wrap_index(__float2int_rn(px), wp), y = wrap_index(__float2int_rn(py), hp);
    const double w = mask ? ramp(x, wp) : 0.0;
    const uint8_t* src = views + (((size_t)v * hp + y) * wp + x) * C;
    for (int c = 0; c < C; ++c) num[c] = __dadd_rn(num[c], __dmul_rn(mask ? double(src[c]) : 0.0, w));
    den = __dadd_rn(den, w);
  }
  uint8_t* dst = out + (size_t)idx * C;
  for (int c = 0; c < C; ++c) {
    const double r = den == 0.0 ? 255.0 : __ddiv_rn(num[c], den);
    dst[c] = (uint8_t)fmin(r, 255.0);  // astype(np.uint8): truncation
  }
}

}  // namespace pf

extern "C" int pf_mp2e(const uint8_t* views, int m, int hp, int wp, int C, const double* cams_p2e, int He, int We,
                       uint8_t* out, void* stream) {
  using namespace pf;
  PF_CHECK_ARG(views && cams_p2e && out, "pf_mp2e: null pointer");
  PF_CHECK_ARG(m > 0 && hp > 0 && wp > 0 && C > 0 && C <= 4 && He > 0 && We > 0 && (long long)He * We < (1LL << 31),
               "pf_mp2e: bad shape m=%d hp=%d wp=%d C=%d He=%d We=%d", m, hp, wp, C, He, We);
  mp2e_kernel<<<(unsigned)((He * We + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(views, m, hp, wp, C,
                                                                                             cams_p2e, He, We, out);
  PF_CHECK_LAUNCH("mp2e_kernel");
  return PF_OK;
}
