// Host-side helpers of the TMA kernels (conv_tma.h).  Host code only.
#include "conv_tma.h"

#include <atomic>
#include <cstdlib>
#include <cstring>
#include <mutex>

namespace ltb {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

bool tma_encode_available() { return get_encode() != nullptr; }

bool encode_tmap_f16(CUtensorMap* tm, int rank, const void* base, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                     const cuuint32_t* box, int spatial_stride, CUtensorMapSwizzle swizzle) {
  EncodeTiledFn fn = get_encode();
  if (!fn) return false;
  cuuint32_t es[5] = {1, (cuuint32_t)spatial_stride, (cuuint32_t)spatial_stride, 1, 1};   // traversal stride of the W and H dimensions
  return fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box, es,
            CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

bool encode_nhwc_f16(CUtensorMap* tm, const void* base, int C, int W, int H, int N, int Ctot, const cuuint32_t* box,
                     int spatial_stride, CUtensorMapSwizzle swizzle) {
  const cuuint64_t pitch = (cuuint64_t)Ctot * 2;
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[3] = {pitch, W * pitch, (cuuint64_t)H * W * pitch};
  return encode_tmap_f16(tm, 4, base, dims, strides, box, spatial_stride, swizzle);
}

int device_sms() {
  static std::atomic<int> sms_cached{0};
  int sms = sms_cached.load();
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;   // H100 SXM
    sms_cached.store(sms);
  }
  return sms;
}

bool conv_is_3x3_same(const ConvParams& p) {
  if (p.nphases != 1 || p.ph[0].ntaps != 9 || p.sy != 1 || p.sx != 1 || p.osy != 1 || p.osx != 1) return false;
  for (int t = 0; t < 9; ++t)
    if (p.ph[0].dy[t] != t / 3 - 1 || p.ph[0].dx[t] != t % 3 - 1) return false;
  return p.IH == p.GH && p.IW == p.GW && p.OH == p.GH && p.OW == p.GW;
}

bool ab_switch_on(const char* name) {
  const char* e = std::getenv(name);
  return !(e && std::strcmp(e, "0") == 0);
}

}  // namespace ltb
