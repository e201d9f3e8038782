// HuBERT front-end kernels (SURVEY 8 row f4; reference: avatars/ultralight/audio2feature.py:14-56 -> transformers HubertModel,
// hubert-large-ls960-ft: feat_extract_norm "layer", conv_bias, do_stable_layer_norm).  The transformer layers and conv layers 1-6
// run on the wgmma conv / attention kernels; these are the pieces with no GEMM shape:
//   * Wav2Vec2 processor normalisation (zero mean / unit variance over the utterance) fused with conv layer 0 (1 -> 512, k 10, s 5)
//   * the positional convolution (Conv1d 1024 -> 1024, k 128, pad 64, 16 groups, weight-norm folded) + SamePad trim + GELU + residual
//   * the window gather of BaseASR._feature2chunks (base_asr.py:91-157) as HubertASR.run_step calls it (hubert.py:42-45)
#include "ltb_internal.h"
#include "ops.h"
#include "ptx_sm90.cuh"

namespace ltb {

// Every kernel takes a sequence count G: G windows of n samples stacked on the row dimension ([G][n] PCM, [G][T][C] activations,
// [G][B][R][D] windows).  Sequence g reads and writes only its own rows; G = 1 is the single-window layout.

// ------------------------------------------------------------------------------------------------ utterance statistics
// stats[4g + 0] = mean, stats[4g + 1] = 1 / sqrt(var + 1e-7) (population variance) of window g (one block per window) —
// Wav2Vec2FeatureExtractor.zero_mean_unit_var_norm, which normalises each input sequence on its own.
__global__ void __launch_bounds__(1024) wave_stats_kernel(const float* __restrict__ x, int n, float* __restrict__ stats) {
  __shared__ double s1[32], s2[32];
  x += (size_t)blockIdx.x * n;
  stats += 4 * blockIdx.x;
  double a = 0.0, b = 0.0;
  for (int i = threadIdx.x; i < n; i += 1024) {
    const double v = (double)x[i];
    a += v;
    b += v * v;
  }
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  if ((threadIdx.x & 31) == 0) s1[threadIdx.x >> 5] = a, s2[threadIdx.x >> 5] = b;
  __syncthreads();
  if (threadIdx.x == 0) {
    double sa = 0.0, sb = 0.0;
    for (int i = 0; i < 32; ++i) sa += s1[i], sb += s2[i];
    const double mean = sa / n;
    const double var = fmax(sb / n - mean * mean, 0.0);
    stats[0] = (float)mean;
    stats[1] = (float)(1.0 / sqrt(var + 1e-7));
  }
}

// out[t][c] = bias[c] + sum_k w[c][k] * (x[5t + k] - mean) * inv_std,  t < T0 = (n - 10) / 5 + 1 ; fp32 math, fp16 out [T0][512]
// per window (blockIdx.y)
__global__ void __launch_bounds__(256) hubert_conv0_kernel(const float* __restrict__ x, int n, const float* __restrict__ stats,
                                                           const float* __restrict__ w, const float* __restrict__ bias, int T0, int C,
                                                           __half* __restrict__ out) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  const int t = blockIdx.x, g = blockIdx.y;
  x += (size_t)g * n;
  stats += 4 * g;
  out += (size_t)g * T0 * C;
  __shared__ float xs[10];
  if (threadIdx.x < 10) xs[threadIdx.x] = (x[5 * t + threadIdx.x] - stats[0]) * stats[1];
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += 256) {
    float acc = bias ? bias[c] : 0.f;
#pragma unroll
    for (int k = 0; k < 10; ++k) acc = fmaf(w[c * 10 + k], xs[k], acc);
    out[(size_t)t * C + c] = __float2half_rn(acc);
  }
}

cudaError_t launch_hubert_conv0(const float* pcm, int G, int n, const float* w, const float* bias, int C, float* stats, __half* out,
                                cudaStream_t st) {
  if (n < 10 || G < 1 || G > 65535) return cudaErrorInvalidValue;
  wave_stats_kernel<<<G, 1024, 0, st>>>(pcm, n, stats);
  const int T0 = (n - 10) / 5 + 1;
  return launch_kernel_plain(hubert_conv0_kernel, dim3(T0, G), dim3(256), 0, st, pcm, n, stats, w, bias, T0, C, out);
}

// ------------------------------------------------------------------------------------------------ positional convolution
// h [T][D] fp16; w fp16 [D][K][D/G] (output channel, tap, input channel inside the group); out[t][co] = h[t][co] +
// gelu(bias[co] + sum_{k < K, ci < D/G} h[t + k - K/2][g*D/G + ci] * w[co][k][ci])  for t < T (the SamePad layer drops the extra
// last step an even kernel produces).  One block = 4 output channels of one group x 64 time steps; the group's input slab
// lives in shared memory (rows padded by one word: conflict-free column walks), weights stream through L1 as broadcasts.
// blockIdx.z = sequence: its T rows are zero-padded on their own, so no tap reads a neighbouring sequence.
constexpr int kPcK = 128, kPcCg = 64, kPcRows = 64 + kPcK - 1, kPcPitch = kPcCg / 2 + 1;   // pitch in 32-bit words

__device__ __forceinline__ float gelu_erf(float v) { return 0.5f * v * (1.f + erff(v * 0.70710678118654752f)); }

__global__ void __launch_bounds__(256) hubert_pos_conv_kernel(const __half* __restrict__ h, int T, int D, const __half* __restrict__ w,
                                                              const float* __restrict__ bias, __half* __restrict__ out) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  __shared__ uint32_t slab[kPcRows * kPcPitch];
  h += (size_t)blockIdx.z * T * D;
  out += (size_t)blockIdx.z * T * D;
  const int g = blockIdx.y, co = g * kPcCg + blockIdx.x * 4 + (threadIdx.x >> 6), tl = threadIdx.x & 63;
  for (int t0 = 0; t0 < T; t0 += 64) {
    __syncthreads();
    for (int i = threadIdx.x; i < kPcRows * (kPcCg / 2); i += 256) {
      const int r = i / (kPcCg / 2), c2 = i % (kPcCg / 2);
      const int t = t0 + r - kPcK / 2;
      slab[r * kPcPitch + c2] = (t >= 0 && t < T) ? *reinterpret_cast<const uint32_t*>(h + (size_t)t * D + g * kPcCg + 2 * c2) : 0u;
    }
    __syncthreads();
    float acc0 = 0.f, acc1 = 0.f;
    const uint4* wrow = reinterpret_cast<const uint4*>(w + (size_t)co * kPcK * kPcCg);
    for (int k = 0; k < kPcK; ++k) {
      const uint32_t* xr = slab + (tl + k) * kPcPitch;
#pragma unroll
      for (int q = 0; q < kPcCg / 8; ++q) {
        const uint4 wv = __ldg(wrow + k * (kPcCg / 8) + q);
        const __half2* wh = reinterpret_cast<const __half2*>(&wv);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t xw = xr[q * 4 + j];
          const float2 xf = __half22float2(*reinterpret_cast<const __half2*>(&xw)), wf = __half22float2(wh[j]);
          acc0 = fmaf(xf.x, wf.x, acc0);
          acc1 = fmaf(xf.y, wf.y, acc1);
        }
      }
    }
    const int t = t0 + tl;
    if (t < T) {
      const float v = gelu_erf(acc0 + acc1 + bias[co]);
      out[(size_t)t * D + co] = __float2half_rn(__half2float(h[(size_t)t * D + co]) + v);
    }
  }
}

cudaError_t launch_hubert_pos_conv(const __half* h, int G, int T, int D, int groups, int K, const __half* w, const float* bias, __half* out,
                                   cudaStream_t st) {
  if (K != kPcK || D % groups || D / groups != kPcCg || h == out || G < 1 || G > 65535) return cudaErrorInvalidValue;
  return launch_kernel_plain(hubert_pos_conv_kernel, dim3(kPcCg / 4, groups, G), dim3(256), 0, st, h, T, D, w, bias, out);
}

// ------------------------------------------------------------------------------------------------ window gather
// hidden fp16 [Tc][D] (Tc = conv frames); the reference trims / zero-pads it to T = (n - 80) / 320 rows (audio2feature.py:50-55), then
// frame i takes rows clamp(left .. right-1, 0, T-1), left = int((i + start) * mult) - int(win_l * mult) (base_asr.py:107-129).
// out_f32 [B][R][D] (what HubertASR queues, float32) and/or out_nhwc fp16 [B][D][R] (the U-Net's (B,32,32,16) NHWC input:
// audiofeat.reshape(16,32,32) -> channel = row, pixel = feature index; ultralight_avatar.py:162).  blockIdx.z = sequence g: it gathers
// from its own hidden rows [g*Tc, (g+1)*Tc) into its own B windows.
__global__ void __launch_bounds__(256) hubert_slice_kernel(const __half* __restrict__ hidden, int Tc, int T, int D, int B, int R, float start,
                                                           float mult, int win_l, float* __restrict__ out_f32, __half* __restrict__ out_nhwc) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  const int b = blockIdx.y, r = blockIdx.x, g = blockIdx.z;
  hidden += (size_t)g * Tc * D;
  if (out_f32) out_f32 += (size_t)g * B * R * D;
  if (out_nhwc) out_nhwc += (size_t)g * B * D * R;
  const int center = (int)(((float)b + start) * mult);
  const int left = (int)((float)center - (float)win_l * mult);
  const int row = min(max(left + r, 0), T - 1);
  for (int d = threadIdx.x; d < D; d += 256) {
    const __half v = row < Tc ? hidden[(size_t)row * D + d] : __float2half(0.f);
    if (out_f32) out_f32[((size_t)b * R + r) * D + d] = __half2float(v);
    if (out_nhwc) out_nhwc[((size_t)b * D + d) * R + r] = v;
  }
}

cudaError_t launch_hubert_slice(const __half* hidden, int G, int Tc, int T, int D, int B, int R, float start, float mult, int win_l,
                                float* out_f32, __half* out_nhwc, cudaStream_t st) {
  if (T < 1 || Tc < 1 || G < 1 || G > 65535) return cudaErrorInvalidValue;
  return launch_kernel_plain(hubert_slice_kernel, dim3(R, B, G), dim3(256), 0, st, hidden, Tc, T, D, B, R, start, mult, win_l, out_f32,
                             out_nhwc);
}

}  // namespace ltb
