// Host/device interface of the ping-pong 64-channel residual 3x3 conv kernel (conv_pingpong.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "conv_params.h"

namespace ltb {

struct alignas(64) PingpongParams {
  CUtensorMap tm_in;   // 4-D (C, W, H, N) fp16 NHWC input slice, box (64, 10, 18, 1), SWIZZLE_128B, OOB -> 0 (= padding)
  CUtensorMap tm_w;    // 3-D (k, n, tap) over the tap-major weight copy [9][64][64], box (64, 64, 3)
  CUtensorMap tm_out;  // 4-D (C, W, H, N) fp16 NHWC output slice, box (64, 8, 16, 1), SWIZZLE_128B: stores clip at the map's edge
  const float* bias;
  int relu;
  int tiles_x, tiles_y, total_tiles;   // 16 x 8 pixel tiles
};

// 3x3 stride-1 pad-1 convs with Cin = Cout = 64 whose residual is their own input slice, on maps whose width is a multiple of 8,
// with enough tiles for the two MMA warpgroups of each CTA to alternate (see conv_pingpong.cu); false when LTB_CONV_PINGPONG=0
bool conv_pingpong_supported(const ConvParams& p);
// w_tap_major: device pointer to the [9][64][64] copy of the layer's weights.  Returns 0 on success.
int conv_pingpong_make_plan(const ConvParams& p, const __half* w_tap_major, PingpongParams* out);
cudaError_t launch_conv_pingpong(const PingpongParams& pp, cudaStream_t st);

}  // namespace ltb
