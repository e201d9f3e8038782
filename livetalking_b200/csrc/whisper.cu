// Whisper front-end on the GPU (replaces the CPU/torch path of transformers.WhisperFeatureExtractor as called by
// Audio2Feature.audio2feat, avatars/musetalk/whisper/audio2feature.py:106-111) and the feature slicing of
// WhisperASR.run_step (avatars/audio_features/whisper.py:35-56, base_asr.py:91-133).
//
//   log-mel : zero-pad PCM to 30 s, STFT(n_fft 400, hop 160, periodic Hann, centre + reflect padding), |.|^2, drop the
//             last frame (3000 frames), 80 x 201 Slaney filterbank, log10(max(1e-10, .)), max(x, global_max - 8), (x+4)/4.
//             Only the frames that overlap real samples are transformed; the 30-s padding region is the constant
//             log10(1e-10) = -10 (before the global-max clamp), exactly what the reference computes for silence.
//   slicing : video frame i takes encoder steps c..c+9, c = int((i + start) * 2), clamped to [0, T-1], from all 5 hidden
//             states -> (50, 384) rows ordered (step-major, layer-minor).
//
// Every kernel takes a window count G (cross-session batching: one encoder forward for G sessions): PCM [G][n], log-mel
// [G][3000][80], hidden states [G*T][D], features [G][B][rows][D].  Window g reads and writes only its own slices, and has its own
// global maximum (WhisperFeatureExtractor clamps each utterance on its own).  G = 1 is the single-window layout.
#include "ops.h"

namespace ltb {

constexpr int kWNfft = 400, kWHop = 160, kWBins = 201, kWMels = 80, kWFrames = 3000, kWSamples = 480000;

__device__ __forceinline__ float w_sample(const float* __restrict__ pcm, int n, int i) {
  // index into the reflect-padded (by n_fft/2) version of the zero-padded 480000-sample signal
  if (i < 0) i = -i;
  if (i >= kWSamples) i = 2 * (kWSamples - 1) - i;
  return (i < n) ? pcm[i] : 0.f;
}

__device__ __forceinline__ int float_ordered(float f) {
  const int i = __float_as_int(f);
  return (i >= 0) ? i : (i ^ 0x7FFFFFFF);
}
__device__ __forceinline__ float ordered_float(int i) { return __int_as_float((i >= 0) ? i : (i ^ 0x7FFFFFFF)); }

// one block per active frame (blockIdx.x) of window blockIdx.y; writes log10 mel power to logspec[g][m * t_active + t] and folds
// the window's maximum into gmax[g]
__global__ void __launch_bounds__(256) whisper_stft_mel_kernel(const float* __restrict__ pcm, int n, const float* __restrict__ fb,
                                                               int t_active, float* __restrict__ logspec, int* __restrict__ gmax) {
  __shared__ double fr[kWNfft];
  __shared__ double tc[kWNfft], ts[kWNfft];
  __shared__ double pw[kWBins];
  __shared__ float red[8];
  const int t = blockIdx.x, g = blockIdx.y;
  pcm += (size_t)g * n;
  logspec += (size_t)g * kWMels * t_active;
  gmax += g;
  for (int i = threadIdx.x; i < kWNfft; i += 256) {
    const double w = 0.5 - 0.5 * cospi((double)i / 200.0);  // torch.hann_window(400) (periodic)
    fr[i] = (double)w_sample(pcm, n, t * kWHop + i - kWNfft / 2) * (double)(float)w;
    tc[i] = cospi((double)i / 200.0);
    ts[i] = sinpi((double)i / 200.0);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < kWBins; k += 256) {
    double re = 0.0, im = 0.0;
    int idx = 0;
    for (int j = 0; j < kWNfft; ++j) {
      re = fma(fr[j], tc[idx], re);
      im = fma(fr[j], ts[idx], im);
      idx += k;
      if (idx >= kWNfft) idx -= kWNfft;
    }
    pw[k] = re * re + im * im;
  }
  __syncthreads();
  float lmax = -INFINITY;
  if (threadIdx.x < kWMels) {
    const float* f = fb + (size_t)threadIdx.x * kWBins;
    double acc = 0.0;
    for (int k = 0; k < kWBins; ++k) acc = fma((double)f[k], pw[k], acc);
    const float v = log10f(fmaxf((float)acc, 1e-10f));
    logspec[(size_t)threadIdx.x * t_active + t] = v;
    lmax = v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lmax;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = red[0];
    for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
    atomicMax(gmax, float_ordered(m));
  }
}

__global__ void whisper_init_max_kernel(int* gmax, int G, int t_active) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < G) gmax[g] = float_ordered(t_active < kWFrames ? -10.f : -INFINITY);
}

// window blockIdx.y -> out16: fp16 [3000][80] (the NHWC input of conv1) ; out32 (optional): float [80][3000] = input_features
__global__ void __launch_bounds__(256) whisper_finalize_kernel(const float* __restrict__ logspec, int t_active, const int* __restrict__ gmax,
                                                               __half* __restrict__ out16, float* __restrict__ out32) {
  const int g = blockIdx.y;
  logspec += (size_t)g * kWMels * t_active;
  out16 += (size_t)g * kWFrames * kWMels;
  if (out32) out32 += (size_t)g * kWMels * kWFrames;
  const float floor_v = ordered_float(gmax[g]) - 8.0f;
  const int total = kWFrames * kWMels;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < total; i += gridDim.x * 256) {
    const int t = i / kWMels, m = i % kWMels;
    float v = (t < t_active) ? logspec[(size_t)m * t_active + t] : -10.f;
    v = (fmaxf(v, floor_v) + 4.0f) / 4.0f;
    out16[i] = __float2half_rn(v);
    if (out32) out32[(size_t)m * kWFrames + t] = v;
  }
}

cudaError_t launch_whisper_logmel(const float* pcm, int G, int n, const float* fb, float* logspec_ws, int* gmax, __half* out16, float* out32,
                                  cudaStream_t st) {
  if (n < 1 || n > kWSamples || G < 1 || G > 65535) return cudaErrorInvalidValue;
  int t_active = (n + kWNfft / 2 + kWHop - 1) / kWHop + 1;
  if (t_active > kWFrames) t_active = kWFrames;
  whisper_init_max_kernel<<<(G + 255) / 256, 256, 0, st>>>(gmax, G, t_active);
  whisper_stft_mel_kernel<<<dim3(t_active, G), 256, 0, st>>>(pcm, n, fb, t_active, logspec_ws, gmax);
  whisper_finalize_kernel<<<dim3(240, G), 256, 0, st>>>(logspec_ws, t_active, gmax, out16, out32);
  return cudaGetLastError();
}

struct HiddenPtrs {
  const __half* h[5];
};
__global__ void __launch_bounds__(128) whisper_slice_kernel(HiddenPtrs hp, int T, int D, int B, float start, float mult, __half* __restrict__ out,
                                                            int out_rows_per_frame) {
  const int i = blockIdx.y;         // video frame
  const int r = blockIdx.x;         // 0..49 : step j = r / 5, layer = r % 5
  const int g = blockIdx.z;         // window: its hidden rows [g*T, (g+1)*T), its B frames of out
  const int j = r / 5, layer = r % 5;
  const int center = (int)((float)(i + start) * mult);   // int(vid_idx * feature_idx_multiplier)
  int idx = center + j;                                   // window [0, 5] video frames * 2 = 10 steps
  idx = max(0, min(T - 1, idx));
  const uint4* src = reinterpret_cast<const uint4*>(hp.h[layer] + ((size_t)g * T + idx) * D);
  uint4* dst = reinterpret_cast<uint4*>(out + (((size_t)g * B + i) * out_rows_per_frame + r) * D);
  for (int v = threadIdx.x; v < D / 8; v += 128) dst[v] = src[v];
}

cudaError_t launch_whisper_slice(const __half* const* hidden5, int G, int T, int D, int B, float start, float mult, __half* out,
                                 int out_rows_per_frame, cudaStream_t st) {
  if (G < 1 || G > 65535 || B < 1 || B > 65535 || T < 1) return cudaErrorInvalidValue;
  HiddenPtrs hp;
  for (int i = 0; i < 5; ++i) hp.h[i] = hidden5[i];
  whisper_slice_kernel<<<dim3(50, B, G), 128, 0, st>>>(hp, T, D, B, start, mult, out, out_rows_per_frame);
  return cudaGetLastError();
}

}  // namespace ltb
