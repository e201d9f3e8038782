// Conv planning: the one place that turns a convolution into ConvParams, picks the kernel that runs it (the TMA halo kernel
// of conv_halo.cu, the ping-pong kernel of conv_pingpong.cu for the 64-channel residual 3x3 convs, the row-pair kernel of
// conv_rowpair.cu for the 80 -> 32 channel output conv, the small-map split-K kernel of conv_smallmap.cu for opted-in 8x8 / 4x4 / 1x1
// layers, or the cp.async gather kernel of conv_gather.cu), fuses epilogue extras
// and launches it.
#pragma once
#include <cuda_runtime.h>

#include "conv_halo.h"
#include "conv_pingpong.h"
#include "conv_rowpair.h"
#include "conv_smallmap.h"

struct ltb_conv_variant;   // include/ltb200.h

namespace ltb {

// channels [off, off + C) of an NHWC fp16 tensor whose pixels are Ctot elements apart
struct ConvSlice {
  const __half* p;
  int Ctot, off;
};

enum class ConvMode {
  Dense,       // KH x KW taps, stride (sy, sx), top / left padding (pad_t, pad_l)
  Transposed,  // ConvTranspose2d(k3, s2, p1, op1): four sub-pixel phases over the input grid, OH = 2 IH, Ktot = 9 Cin
  Upsample2x,  // nearest 2x upsample + 3x3 p1 conv: four 2x2 phases over the low-resolution input, Ktot = 16 Cin
};
struct ConvTaps {
  int KH, KW, sy, sx, pad_t, pad_l;
};

inline int conv_out_dim(int in, int k, int s, int pad) { return (in + 2 * pad - k) / s + 1; }

// w: fp16 [Cout][Ktot] K-major rows, the first tap at element w_koff; res.p may be null; taps are read in Dense mode only
ConvParams conv_params(ConvMode mode, int N, ConvSlice in, int IH, int IW, int Cin, ConvSlice out, int OH, int OW, int Cout,
                       ConvSlice res, const __half* w, int Ktot, int w_koff, const float* bias, bool relu, ConvTaps taps = {});

enum class ConvPath {
  Auto,    // the small-map kernel for a layer that opts in (ConvParams::smallmap) and fits it, else a TMA kernel (ping-pong,
           // row-pair or halo) when one supports the geometry and has its weights (w_tap, or none needed in GEMM mode), else gather
  Gather,  // gather kernel
  Halo,    // a TMA kernel (ping-pong, row-pair or halo), or fail
};
// the kernel a plan runs; the values are those ltb_conv_variant::kernel reports
enum class ConvKernel { Gather = 0, Halo = 1, Pingpong = 2, Rowpair = 3, Smallmap = 4 };
struct ConvPlan {
  ConvParams p{};
  ConvKernel kernel = ConvKernel::Gather;
  HaloPlan hp{};        // Halo only
  PingpongParams pp{};  // Pingpong only
  RowpairParams rp{};   // Rowpair only
  SmallmapParams sp{};  // Smallmap only
};

// w_tap: device copy of the weights in the halo kernel's tap-major layout (see launch_w_tap_major*); null if there is none.
// Grouped ops (p.group_slot) run on the halo kernel's GEMM mode or on the gather kernel, never with zbatch, split-K, the fused
// upsample or an epilogue fusion.  Returns 0, or 1 with the reason set as the last error.
int conv_plan(const ConvParams& p, const __half* w_tap, ConvPath path, ConvPlan* out);
// splitk_ws: zero-initialised fp32 workspace of ws_floats floats for the gather kernel's split-K (one per stream)
cudaError_t conv_launch(const ConvPlan& pl, cudaStream_t st, float* splitk_ws, size_t ws_floats);
// the kernel instance conv_launch runs for pl with (have_ws) or without a split-K workspace; false if no instance can run it
bool conv_plan_variant(const ConvPlan& pl, bool have_ws, size_t ws_floats, ltb_conv_variant* out);

// Epilogue fusions; each returns false, leaving the plan unchanged, when the plan cannot take it.
// GroupNorm statistics (sum, sum of squares per (image, group)) of the output, hw pixels per image: `stats` must be zeroed
// before the launch.
bool conv_plan_fuse_gn_stats(ConvPlan* pl, float* stats, int groups, int hw);
// 32 -> 3 head + sigmoid * 255 into out[pix][3] (w2l_head_kernel's arithmetic); the 32-channel activations are not stored
bool conv_plan_fuse_head(ConvPlan* pl, const float* w, const float* b, float* out);

}  // namespace ltb
