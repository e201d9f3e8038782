// Host/device interface of the halo-resident 3x3 conv / sub-pixel ConvT kernel (conv_halo.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstring>

#include "conv_params.h"

namespace ltb {

struct alignas(64) HaloParams {
  CUtensorMap tm_in;  // 4-D (C, W, H, N) fp16 NHWC channel slice, box (64, 10, 16*NSUB+2, 1), SWIZZLE_128B, OOB -> 0 (= padding)
  CUtensorMap tm_w;   // 3-D (k, n, tap) over the tap-major weight copy [9][Cout][Cin], box (64, BN, 3)
  __half* out;
  const __half* res;
  const float* bias;
  int N, M, Cin;  // M: GEMM-mode row count
  int OCtot, oc_off, RCtot, rc_off;
  int OH, OW, osy, osx;
  int GH, GW;            // tile-grid extent (= input H, W): tiles may overhang it, rows/columns beyond are masked
  int relu;
  // the residual is the conv's own input slice (3x3 stride-1, Cin == Cout): the epilogue takes it from the centre view of the
  // halo tiles in shared memory instead of reading res from global memory
  int res_halo;
  int halo_y0, halo_x0;  // halo origin relative to the tile origin (-1 for pad-1 conv, 0 for ConvT phases)
  // output offset of each accumulator slot (sub-pixel phase; slot order p0, p1, p3, p2, see conv_halo.cu SubpixelTable)
  int acc_oy[4], acc_ox[4];
  int tiles_x, tiles_y, tiles_n, total_tiles;
  // optional fused GroupNorm statistics of the OUTPUT tensor (sum, sum of squares per (image, group)), accumulated by the
  // epilogue from the fp16-rounded values: saves the separate statistics pass of the following GroupNorm
  float* gn_stats;
  int gn_groups, gn_cpg, gn_hw, gn_images;   // gn_images: number of images the statistics table covers (M / gn_hw)
  // optional fused output head (BN == Cout == 32 only): pred[pix][j] = sigmoid(sum_c head_w[j][c] * y[pix][c] + head_b[j]) * 255
  // computed from the fp16-rounded activations in the order of w2l_head_kernel (bit-identical); the activations
  // themselves are then not stored.  wav2lip256 output_block: avatars/wav2lip/models/wav2lip_v2.py:95-97.
  const float* head_w;
  const float* head_b;
  float* head_out;
  // grouped GEMM mode (ConvParams::group_slot): M-tiles are enumerated per group of group_rows rows, tiles_x = groups *
  // group_tiles; the weight map is 3-D (k, n, slot) over the bank and the bias of slot s starts at bias + s * bias_slot_stride
  const int* group_slot;
  int group_rows, group_tiles;
  long long bias_slot_stride;
#ifdef LTB_HALO_DIAG
  int dbg;      // diagnostic build only (tools/diag_halo.py): bit0 no epilogue global I/O, bit1 no epilogue at all,
                // bit2 no MMAs, bit3 no A loads, bit4 no B loads.  Never compiled into libltb200.so.
#endif
};

struct HaloPlan {
  HaloParams hp;
  int BN, NSUB, NACC, TAPS;  // TAPS = 9 (3x3 conv / ConvT halo mode) or 1 (TMA GEMM mode: 1x1 conv / linear)
  bool grouped;              // GEMM mode with per-group weight slots
};

bool conv_halo_supported(const ConvParams& p);
// w_tap_major: device pointer to the [9][Cout][Cin] copy of the layer's weights (unused in GEMM mode). returns 0 on success.
int conv_halo_make_plan(const ConvParams& p, const __half* w_tap_major, HaloPlan* out);
cudaError_t launch_conv_halo(const HaloPlan& pl, cudaStream_t st);
// K chunks of weights the variant launch_conv_halo runs for pl on `sms` SMs keeps resident (template argument RC); 0: streamed
int conv_halo_resident_chunks(const HaloPlan& pl, int sms);
bool conv_halo_gn_fusable(const HaloPlan& pl, int cout_total, int groups, int hw);
cudaError_t launch_w_tap_major(const __half* w, __half* wt, int cout, int cin, cudaStream_t st, int ntaps = 9);
// ConvT(k3,s2) weights: phase-major rows [Cout][9][Cin] (pack order of w2l_pack.py / pack_convT_w) -> the view-major slice
// order the sub-pixel issue loop expects (see conv_halo.cu SubpixelTable)
cudaError_t launch_w_tap_major_convT(const __half* w, __half* wt, int cout, int cin, cudaStream_t st);

}  // namespace ltb
