// Host/device interface of the row-pair 80 -> 32 channel 3x3 conv kernel (conv_rowpair.cu), with the optional fused 1x1 head.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "conv_params.h"

namespace ltb {

struct alignas(64) RowpairParams {
  CUtensorMap tm_x0;   // 4-D (C, W, H, N) fp16 NHWC input slice, box (64, 10, TH + 2, 1) at channel 0, SWIZZLE_128B, OOB -> 0
  CUtensorMap tm_x1;   // the same slice, box (16, 10, TH + 2, 1) at channel 64, SWIZZLE_32B (channels >= Cin read as 0)
  CUtensorMap tm_w0;   // 3-D (k, n, tap) over the tap-major weight copy [9][32][Cin], box (64, 32, 1), SWIZZLE_128B
  CUtensorMap tm_w1;   // the same, box (16, 32, 1) at k = 64, SWIZZLE_32B
  CUtensorMap tm_out;  // 4-D (C, W, H, N) fp16 NHWC output slice, box (32, 8, TH, 1), SWIZZLE_64B: stores clip at the map's edge
  const float* bias;
  // optional fused output head (conv_plan_fuse_head): pred[pix][j] = sigmoid(sum_c head_w[j][c] * y[pix][c] + head_b[j]) * 255
  // from the fp16-rounded activations, in the order of w2l_head_kernel; the activations are then not stored
  const float* head_w;
  const float* head_b;
  float* head_out;
  int relu;
  int H, W;
  int tiles_x, tiles_y, total_tiles;   // TH x 8 pixel tiles
};

// 3x3 stride-1 pad-1 convs with Cin = 80, Cout = 32 and no residual (the wav2lip256 output conv), with enough tiles for the
// two MMA warpgroups of each CTA to alternate (see conv_rowpair.cu); false when LTB_CONV_ROWPAIR=0
bool conv_rowpair_supported(const ConvParams& p);
// w_tap_major: device pointer to the [9][32][80] copy of the layer's weights.  Returns 0 on success.
int conv_rowpair_make_plan(const ConvParams& p, const __half* w_tap_major, RowpairParams* out);
cudaError_t launch_conv_rowpair(const RowpairParams& rp, cudaStream_t st);

}  // namespace ltb
