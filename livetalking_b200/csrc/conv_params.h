// Geometry description shared by the host-side layer planner and the implicit-GEMM conv kernels.
// One ConvParams describes Conv2d / ConvTranspose2d(+folded BN)(+residual)(+ReLU) on NHWC fp16
// tensors as   out[pix, co] = act( sum_{tap, ci} in[pix*stride + tap, ci] * W[co, tap, ci] + bias[co] (+ res[pix, co]) )
// (reference ops: avatars/wav2lip/models/conv.py:5-19 and :33-44).
// A stride-2 ConvTranspose is expressed as 4 sub-pixel "phases", each a dense stride-1 gather
// over the input grid that writes every second output pixel.
#pragma once
#include <cuda_fp16.h>
#include <cstdint>

namespace ltb {

constexpr int kMaxTaps = 16;
constexpr int kMaxPhases = 4;

struct ConvPhase {
  int ntaps;
  int koff;      // element offset along K of this phase's first tap inside a weight row
  int ooy, oox;  // output offset of this phase (sub-pixel position for ConvT)
  signed char dy[kMaxTaps];
  signed char dx[kMaxTaps];
};

struct ConvParams {
  // input  : NHWC, pixel pitch ICtot elements, channels [ic_off, ic_off+Cin) are consumed per tap
  const __half* in;
  int N, IH, IW, ICtot, ic_off, Cin;
  int sy, sx;  // input step per output-grid step
  // output grid (per phase) and output tensor
  int GH, GW;
  __half* out;
  int OH, OW, OCtot, oc_off;
  int osy, osx;  // output step per grid step (2 for ConvT phases)
  int Cout;
  // optional residual (same spatial mapping as out)
  const __half* res;
  int RCtot, rc_off;
  // weights [Cout][Ktot] fp16 (BN folded), bias fp32 [Cout]
  const __half* w;
  int Ktot;
  const float* bias;
  int relu;
  int M;  // N*GH*GW rows per phase
  int nphases;
  ConvPhase ph[kMaxPhases];
  // optional batching over grid.z (attention: one GEMM per (batch, head)): z = zo * zdiv + zi, element offsets added to
  // the in / w / out (/ res) base pointers.  zbatch <= 1 disables.
  int zbatch, zdiv;
  long long in_zo, in_zi, w_zo, w_zi, out_zo, out_zi;
  // optional split-K (small-M, weight-heavy layers): grid.z = ksplit CTAs each reduce a slice of the K loop and store
  // their fp32 partial tile to ws[split][M][Cout]; splitk_finalize sums the slices and applies bias/residual/activation.
  int ksplit;
  float* ws;
  // 1: nearest-neighbour 2x upsample fused with the 3x3 p1 conv that follows it (diffusers Upsample2D): 4 output phases, each a
  // 2x2 conv over the LOW-resolution input with pre-summed taps (16 weight slices [Cout][16][Cin], see ops.py
  // ConvWeight.upconv).  Halo kernel only (no gather fallback).
  int upconv;
  // optional grouped weights (cross-session batching of networks that differ per avatar): image n belongs to group
  // n / group_images and uses the weights / bias of bank slot group_slot[n / group_images] (read on the device, so one captured
  // graph serves any assignment), i.e. w + slot * w_slot_stride and bias + slot * bias_slot_stride (elements).  The bank holds
  // `slots` slots.  group_slot == nullptr: ungrouped.
  const int* group_slot;
  int group_images, slots;
  long long w_slot_stride, bias_slot_stride;
  // 1: the caller opts this layer in to the small-map split-K kernel (conv_smallmap.cu) where that kernel supports it
  int smallmap;
};

}  // namespace ltb
