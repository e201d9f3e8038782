// Host/device interface of the small-map split-K conv kernel (conv_smallmap.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "conv_params.h"

namespace ltb {

struct alignas(64) SmallmapParams {
  CUtensorMap tm_in;   // 4-D (C, W, H, N) fp16 NHWC input slice, box (64, bw, bh, bimg) with traversal stride sx, SWIZZLE_128B
  CUtensorMap tm_w;    // 2-D (K, Cout) over the layer's K-major weight rows [Cout][Ktot], box (64, 128), SWIZZLE_128B
  __half* out;
  const __half* res;
  const float* bias;
  int N, OH, OW, OCtot, oc_off, RCtot, rc_off, relu;
  int GH, GW, osy, osx, Cin;
  int np;        // pixels per tile (the wgmma N): bimg whole images of GH x GW grid points
  int bimg, ptiles, cotiles, nphases, ksplit;
  ConvPhase ph[kMaxPhases];
};

// ConvParams::smallmap layers on 8x8, 4x4 or 1x1 grids with Cin % 64 == 0 and Cout % 128 == 0 (see conv_smallmap.cu); false
// when LTB_CONV_SMALLMAP=0
bool conv_smallmap_supported(const ConvParams& p);
int conv_smallmap_make_plan(const ConvParams& p, SmallmapParams* out);
cudaError_t launch_conv_smallmap(const SmallmapParams& sp, cudaStream_t st);

}  // namespace ltb
