// PFLD_GhostOne landmark network glue kernels (the UltraLight avatar generator, avatars/ultralight/genavatar.py ->
// face_detect_utils/get_landmark.py Landmark.detect): the convolutions run on the conv planner (ltb_op_conv2d) and the depthwise
// kernel (ltb_op_dwconv3x3); here are the two pieces around them.
//   * pfld_prep:  u8 BGR crops -> fp16 NHWC v / 255 in channels 0-2 (BGR: the reference does not swap), zeros in 3-15 (the conv
//                 kernels need Cin >= 16); v / 255 is the fp32 quotient, rounded to fp16 once
//   * pfld_head:  per image, the global average of the four multi-scale taps and the conv8 output (torch.cat of x1..x5), conv_out
//                 (1x1, bias) in fp32, + mean_face, scaled by the crop width / height and truncated (astype(np.int32))
#include "ltb_internal.h"
#include "ops.h"
#include "ptx_sm90.cuh"

namespace ltb {

// ------------------------------------------------------------------------------------------------ prep
// One thread = one pixel: three byte loads, two 16-byte stores.
__global__ void __launch_bounds__(256) pfld_prep_kernel(const uint8_t* __restrict__ bgr, long long npix, __half* __restrict__ out) {
  pdl_launch_dependents();
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < npix; i += (long long)gridDim.x * 256) {
    const uint8_t* p = bgr + i * 3;
    uint4 v;
    __half2* h = reinterpret_cast<__half2*>(&v);
    // np.asarray(x, np.float32) / 255.0 is the correctly rounded fp32 quotient
    h[0] = __halves2half2(__float2half_rn(__fdiv_rn((float)p[0], 255.f)), __float2half_rn(__fdiv_rn((float)p[1], 255.f)));
    h[1] = __halves2half2(__float2half_rn(__fdiv_rn((float)p[2], 255.f)), __float2half(0.f));
    h[2] = h[3] = __float2half2_rn(0.f);
    uint4* o = reinterpret_cast<uint4*>(out + i * kPfldInC);
    o[0] = v;
    o[1] = make_uint4(0, 0, 0, 0);
  }
}

cudaError_t launch_pfld_prep(const uint8_t* bgr, int N, int H, int W, __half* out, cudaStream_t st) {
  if (N <= 0 || H <= 0 || W <= 0 || (reinterpret_cast<uintptr_t>(out) & 15)) return cudaErrorInvalidValue;
  const long long npix = (long long)N * H * W;
  long long blocks = (npix + 255) / 256;
  if (blocks > 132 * 64) blocks = 132 * 64;
  return launch_kernel_plain(pfld_prep_kernel, dim3((unsigned)blocks), dim3(256), 0, st, bgr, npix, out);
}

// ------------------------------------------------------------------------------------------------ head
// One CTA per image.  Tap t: [N][hw[t]] pixels of pitch[t] halves; its real channels are ch[first .. first + nch[t]) (indices
// inside the pitch), concatenated in tap order into the nfeat features.  Per tap, thread i sums 8 channels (group i % G, G =
// pitch / 8) over the pixels i / G, i / G + T, ... (T = threads / G) in fp32; thread c then adds the T partials of channel c in
// slot order: a fixed summation order, so a replay is bit-identical.  The average is the sum divided by hw (AvgPool2d).
constexpr int kHeadThreads = 512;

__global__ void __launch_bounds__(kHeadThreads) pfld_head_kernel(const PfldTaps taps, const float* __restrict__ wt, const float* __restrict__ bias,
                                                                 const float* __restrict__ mean, const int* __restrict__ crop_wh, int nout,
                                                                 float* __restrict__ out_f, int* __restrict__ out_i) {
  pdl_launch_dependents();
  __shared__ float part[kHeadThreads * 8];
  __shared__ float avg[kPfldMaxPitch];
  __shared__ float feat[kPfldMaxFeat];
  const int n = blockIdx.x, tid = threadIdx.x;
  int first = 0;
#pragma unroll   // static indices into the parameter struct
  for (int t = 0; t < kPfldTaps; ++t) {
    const int pitch = taps.pitch[t], hw = taps.hw[t], G = pitch >> 3, T = kHeadThreads / G;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    if (tid < T * G) {
      const int g = tid % G;
      const __half* base = taps.p[t] + (size_t)n * hw * pitch + g * 8;
      for (int px = tid / G; px < hw; px += T) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(base + (size_t)px * pitch));
        const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = __half22float2(h[k]);
          acc[2 * k] += f.x;
          acc[2 * k + 1] += f.y;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) part[tid * 8 + k] = acc[k];
    __syncthreads();
    if (tid < pitch) {
      const int g = tid >> 3, k = tid & 7;
      float s = 0.f;
      for (int slot = 0; slot < T; ++slot) s += part[(slot * G + g) * 8 + k];
      avg[tid] = s / (float)hw;
    }
    __syncthreads();
    if (tid < taps.nch[t]) feat[first + tid] = avg[taps.ch[first + tid]];
    first += taps.nch[t];
    __syncthreads();
  }
  if (tid >= nout) return;
  float acc = __ldg(bias + tid);
  for (int j = 0; j < first; ++j) acc = fmaf(__ldg(wt + (size_t)j * nout + tid), feat[j], acc);
  // pre_landmark + mean_face, then [:, 0] *= w, [:, 1] *= h and astype(np.int32): fp32 add, fp32 multiply, truncation
  const float lm = __fadd_rn(acc, __ldg(mean + tid));
  const float v = __fmul_rn(lm, (float)__ldg(crop_wh + 2 * n + (tid & 1)));
  out_f[(size_t)n * nout + tid] = v;
  out_i[(size_t)n * nout + tid] = (int)v;
}

cudaError_t launch_pfld_head(const PfldTaps& taps, int N, const float* wt, const float* bias, const float* mean, const int* crop_wh, int nout,
                             float* out_f, int* out_i, cudaStream_t st) {
  if (N <= 0 || nout <= 0 || nout > kHeadThreads || (nout & 1)) return cudaErrorInvalidValue;
  int nfeat = 0;
  for (int t = 0; t < kPfldTaps; ++t) {
    if (!taps.p[t] || taps.hw[t] <= 0 || taps.pitch[t] < 8 || (taps.pitch[t] & 7) || taps.pitch[t] > kPfldMaxPitch || taps.nch[t] < 0 ||
        (reinterpret_cast<uintptr_t>(taps.p[t]) & 15))
      return cudaErrorInvalidValue;
    for (int c = 0; c < taps.nch[t]; ++c)
      if (nfeat + c >= kPfldMaxFeat || taps.ch[nfeat + c] >= taps.pitch[t]) return cudaErrorInvalidValue;
    nfeat += taps.nch[t];
  }
  return launch_kernel_plain(pfld_head_kernel, dim3(N), dim3(kHeadThreads), 0, st, taps, wt, bias, mean, crop_wh, nout, out_f, out_i);
}

}  // namespace ltb
