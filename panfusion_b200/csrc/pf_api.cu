// C-ABI plumbing: error string, device check, TMA tensor-map encoding.
#include <stdarg.h>
#include <string.h>

#include "pf_common.cuh"

namespace pf {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return PF_OK;
  set_error("%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
  return PF_ERR_CUDA;
}

int sm_count() {
  static const int n = [] {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        v <= 0) {
      cudaGetLastError();
      v = 132;
    }
    return v;
  }();
  return n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int make_tmap(CUtensorMap* out, int dtype, int rank, const void* base, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled driver entry point unavailable (no CUDA driver?)");
    return PF_ERR_CUDA;
  }
  CUtensorMapDataType dt;
  if (dtype == PF_BF16)
    dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  else if (dtype == PF_F16)
    dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  else {
    set_error("make_tmap: dtype %d not a 16-bit float type", dtype);
    return PF_ERR_INVALID;
  }
  CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_NONE;
  if (swizzle_bytes == 128) sw = CU_TENSOR_MAP_SWIZZLE_128B;
  else if (swizzle_bytes == 64) sw = CU_TENSOR_MAP_SWIZZLE_64B;
  else if (swizzle_bytes == 32) sw = CU_TENSOR_MAP_SWIZZLE_32B;
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = fn(out, dt, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed: CUresult %d (rank %d, dims %llu,%llu box %u,%u base %p)", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0],
              rank > 1 ? box[1] : 0, base);
    return PF_ERR_CUDA;
  }
  return PF_OK;
}

}  // namespace pf

extern "C" {

const char* pf_last_error(void) { return pf::g_err; }

int pf_version(void) { return 100; }

int pf_check_device(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return pf::check_cuda(e, "cudaGetDevice");
  cudaDeviceProp p;
  e = cudaGetDeviceProperties(&p, dev);
  if (e != cudaSuccess) return pf::check_cuda(e, "cudaGetDeviceProperties");
  if (p.major != 9 || p.minor != 0) {
    pf::set_error("device %s is sm_%d%d; panfusion_b200 only has sm_90a kernels", p.name, p.major, p.minor);
    return PF_ERR_UNSUPPORTED;
  }
  return PF_OK;
}

}  // extern "C"
