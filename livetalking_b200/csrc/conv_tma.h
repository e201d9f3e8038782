// Host-side helpers of the TMA kernels (conv_tma.cu): the one tensor-map encoding policy (fp16, L2 promotion 256 B,
// out-of-bounds elements read as zero), the SM count the persistent grids are sized by, and the routing tests the TMA conv
// kernels share.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "conv_params.h"

namespace ltb {

// the driver exports the tiled tensor-map encoder (looked up once)
bool tma_encode_available();
// fp16 tensor map, out-of-bounds elements read as zero; spatial_stride: traversal stride of dimensions 1 and 2.
// False if the driver entry point is missing or rejects the map.
bool encode_tmap_f16(CUtensorMap* tm, int rank, const void* base, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                     const cuuint32_t* box, int spatial_stride = 1, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B);
// 4-D (C, W, H, N) view of C channels of an NHWC fp16 tensor whose pixels are Ctot elements apart; base: the slice's first
// channel (tensor + channel offset)
bool encode_nhwc_f16(CUtensorMap* tm, const void* base, int C, int W, int H, int N, int Ctot, const cuuint32_t* box,
                     int spatial_stride = 1, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B);
// SM count of the current device (read once), the width of the persistent grid launches
int device_sms();
// 3x3 conv, stride 1, pad 1, whose output grid is its input map
bool conv_is_3x3_same(const ConvParams& p);
// TMA can address the channel slice [off, off + C) of a tensor with pixel pitch Ctot at ptr: 16-byte aligned start and pitch
inline bool tma_slice_ok(const void* ptr, int Ctot, int off) {
  return Ctot % 8 == 0 && off % 8 == 0 && reinterpret_cast<uintptr_t>(ptr) % 16 == 0;
}
// A/B switch of a conv kernel: off only when the environment variable is "0".  Read on every call, so that one process can
// plan the same layer both ways.
bool ab_switch_on(const char* name);

}  // namespace ltb
