// Bandwidth-bound operators of the MuseTalk path (NHWC fp16 activations, fp32 statistics):
//   GroupNorm(+SiLU)  — diffusers ResnetBlock2D / Transformer2DModel / VAE norms   (K11, K12, K13 in SURVEY 2a)
//   LayerNorm         — BasicTransformerBlock norm1..3, Whisper encoder layer norms  (warp-shuffle reductions)
//   softmax           — attention probabilities (scaled, key-padding aware)
//   GEGLU / GELU      — transformer feed-forward, Whisper MLP / conv activations
//   nearest 2x upsample, channel-slice copy (concat), V transpose for the P.V GEMM, positional-encoding add
//     (avatars/musetalk/models/unet.py:12-27), VAE post-processing to u8 BGR (avatars/musetalk/models/vae.py:104-107).
#include "ltb_internal.h"
#include "ops.h"
#include "ptx_sm90.cuh"

namespace ltb {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.f + __expf(-x)); }
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }

// ------------------------------------------------------------------------------------------------ GroupNorm
// pass 1: per (image, group) sum and sum of squares.  A block is R pixel-rows x VPR 16-byte vectors (VPR = C/8): thread
// (r, v) owns channel vector v and walks pixels r, r+R, ... of its slab, so every warp load is a contiguous run of the
// NHWC row and the 8 per-channel partial sums stay in registers; groups are resolved once per thread at the end.
__global__ void __launch_bounds__(512) gn_stats_kernel(const __half* __restrict__ x, int HW, int C, int Ctot, int c_off, int groups, int R,
                                                       float* __restrict__ stats) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  __shared__ float s_sum[64], s_sq[64];
  const int n = blockIdx.y;
  const int cpg = C / groups;
  const int vpr = C / 8;
  // tiny maps launch a single warp: the table of up to 64 groups is zeroed and flushed in blockDim steps
  for (int i = threadIdx.x; i < groups; i += blockDim.x) s_sum[i] = s_sq[i] = 0.f;
  __syncthreads();
  const int per = (HW + gridDim.x - 1) / gridDim.x;
  const int p0 = blockIdx.x * per, p1 = min(HW, p0 + per);
  const int v = threadIdx.x % vpr, r = threadIdx.x / vpr;
  float a[8], b[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) a[j] = b[j] = 0.f;
  if (r < R) {
    const __half* base = x + ((size_t)n * HW) * Ctot + c_off + v * 8;
    int p = p0 + r;
    // two loads in flight per thread
    for (; p + R < p1; p += 2 * R) {
      const uint4 u0 = *reinterpret_cast<const uint4*>(base + (size_t)p * Ctot);
      const uint4 u1 = *reinterpret_cast<const uint4*>(base + (size_t)(p + R) * Ctot);
      const __half* h0 = reinterpret_cast<const __half*>(&u0);
      const __half* h1 = reinterpret_cast<const __half*>(&u1);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float f0 = __half2float(h0[j]), f1 = __half2float(h1[j]);
        a[j] += f0 + f1;
        b[j] += f0 * f0 + f1 * f1;
      }
    }
    for (; p < p1; p += R) {
      const uint4 u0 = *reinterpret_cast<const uint4*>(base + (size_t)p * Ctot);
      const __half* h0 = reinterpret_cast<const __half*>(&u0);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float f0 = __half2float(h0[j]);
        a[j] += f0;
        b[j] += f0 * f0;
      }
    }
    // fold the 8 channels into their groups (consecutive channels mostly share a group)
    int g = (v * 8) / cpg;
    float sa = 0.f, sb = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int gj = (v * 8 + j) / cpg;
      if (gj != g) {
        atomicAdd(&s_sum[g], sa);
        atomicAdd(&s_sq[g], sb);
        sa = sb = 0.f;
        g = gj;
      }
      sa += a[j];
      sb += b[j];
    }
    atomicAdd(&s_sum[g], sa);
    atomicAdd(&s_sq[g], sb);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < groups; i += blockDim.x) {
    atomicAdd(&stats[((size_t)n * groups + i) * 2 + 0], s_sum[i]);
    atomicAdd(&stats[((size_t)n * groups + i) * 2 + 1], s_sq[i]);
  }
}

// pass 2: y = x * a[c] + b[c] (+SiLU) with a = rstd*gamma, b = beta - mean*rstd*gamma staged per image in shared memory;
// one thread = 8 channels of one pixel (16-byte loads/stores), channel vector fixed per thread.
__global__ void __launch_bounds__(256) gn_apply_kernel(const __half* __restrict__ x, int HW, int C, int Ctot, int c_off, int groups,
                                                       float eps, const float* __restrict__ stats, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, int silu, __half* __restrict__ out, int OCtot,
                                                       int oc_off, size_t total_vec) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  extern __shared__ float s_ab[];  // [2][C]
  __shared__ float s_mean[64], s_rstd[64];
  const int n = blockIdx.y;
  const int cpg = C / groups;
  if (threadIdx.x < groups) {
    const float cnt = (float)HW * cpg;
    const float m = stats[((size_t)n * groups + threadIdx.x) * 2] / cnt;
    const float v = fmaxf(stats[((size_t)n * groups + threadIdx.x) * 2 + 1] / cnt - m * m, 0.f);
    s_mean[threadIdx.x] = m;
    s_rstd[threadIdx.x] = rsqrtf(v + eps);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += 256) {
    const int g = c / cpg;
    const float a = s_rstd[g] * gamma[c];
    s_ab[c] = a;
    s_ab[C + c] = beta[c] - s_mean[g] * a;
  }
  __syncthreads();
  const unsigned vpr = C / 8;  // vectors per pixel
  const unsigned tv = (unsigned)total_vec;   // per image: HW * C/8 < 2^31
  const unsigned stride = gridDim.x * 256u;
  const __half* xin = x + (size_t)n * HW * Ctot + c_off;
  __half* yout = out + (size_t)n * HW * OCtot + oc_off;
  // 4 independent 16-byte loads in flight per thread (a single dependent load per iteration left the kernel latency-bound
  // at ~1.6 TB/s)
  for (unsigned i0 = blockIdx.x * 256u + threadIdx.x; i0 < tv; i0 += 4 * stride) {
    uint4 v[4];
    unsigned pp[4];
    int cvv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const unsigned i = i0 + u * stride;
      pp[u] = i / vpr;
      cvv[u] = (int)(i - pp[u] * vpr) * 8;
      if (i < tv) v[u] = *reinterpret_cast<const uint4*>(xin + (size_t)pp[u] * Ctot + cvv[u]);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (i0 + u * stride >= tv) break;
      const int cv = cvv[u];
      const __half2* h = reinterpret_cast<const __half2*>(&v[u]);
      const float4 a0 = *reinterpret_cast<const float4*>(s_ab + cv), a1 = *reinterpret_cast<const float4*>(s_ab + cv + 4);
      const float4 b0 = *reinterpret_cast<const float4*>(s_ab + C + cv), b1 = *reinterpret_cast<const float4*>(s_ab + C + cv + 4);
      float y[8];
      float2 t;
      t = __half22float2(h[0]); y[0] = fmaf(t.x, a0.x, b0.x); y[1] = fmaf(t.y, a0.y, b0.y);
      t = __half22float2(h[1]); y[2] = fmaf(t.x, a0.z, b0.z); y[3] = fmaf(t.y, a0.w, b0.w);
      t = __half22float2(h[2]); y[4] = fmaf(t.x, a1.x, b1.x); y[5] = fmaf(t.y, a1.y, b1.y);
      t = __half22float2(h[3]); y[6] = fmaf(t.x, a1.z, b1.z); y[7] = fmaf(t.y, a1.w, b1.w);
      if (silu) {
#pragma unroll
        for (int j = 0; j < 8; ++j) y[j] = silu_f(y[j]);
      }
      uint4 o;
      __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) oh[j] = __floats2half2_rn(y[2 * j], y[2 * j + 1]);
      *reinterpret_cast<uint4*>(yout + (size_t)pp[u] * OCtot + cv) = o;
    }
  }
}

cudaError_t launch_gn_stats(const __half* x, int N, int HW, int C, int Ctot, int c_off, int groups, float* stats, cudaStream_t st) {
  if (C % groups != 0 || C % 8 != 0 || groups > 64 || C / 8 > 512 || (Ctot % 8) || (c_off % 8)) return cudaErrorInvalidValue;
  cudaError_t e = cudaMemsetAsync(stats, 0, (size_t)N * groups * 2 * sizeof(float), st);
  if (e != cudaSuccess) return e;
  const int vpr = C / 8;
  int R = 512 / vpr;
  if (R > HW) R = HW;
  const int threads = ((R * vpr + 31) / 32) * 32;
  // enough blocks to fill the chip, but keep >= 4 pixels per thread-row
  int splits = (592 + N - 1) / N;
  const int max_splits = (HW + 4 * R - 1) / (4 * R);
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  return launch_kernel_plain(gn_stats_kernel, dim3(dim3(splits, N)), dim3(threads), 0, st, x, HW, C, Ctot, c_off, groups, R, stats);
}

cudaError_t launch_gn_apply(const __half* x, int N, int HW, int C, int Ctot, int c_off, int groups, float eps, const float* stats,
                            const float* gamma, const float* beta, int silu, __half* out, int OCtot, int oc_off, cudaStream_t st) {
  if (C % groups != 0 || C % 8 != 0 || groups > 64 || (Ctot % 8) || (c_off % 8)) return cudaErrorInvalidValue;
  const size_t total_vec = (size_t)HW * (C / 8);
  int blocks = (int)((total_vec + 255) / 256);
  const int cap = (1184 + N - 1) / N;
  if (blocks > cap) blocks = cap;
  return launch_kernel_plain(gn_apply_kernel, dim3(dim3(blocks, N)), dim3(256), 2 * C * sizeof(float), st, x, HW, C, Ctot, c_off, groups, eps, stats, gamma, beta, silu, out, OCtot, oc_off, total_vec);
}

cudaError_t launch_groupnorm(const __half* x, int N, int HW, int C, int Ctot, int c_off, int groups, float eps, const float* gamma,
                             const float* beta, int silu, __half* out, int OCtot, int oc_off, float* stats_ws, cudaStream_t st) {
  cudaError_t e = launch_gn_stats(x, N, HW, C, Ctot, c_off, groups, stats_ws, st);
  if (e != cudaSuccess) return e;
  return launch_gn_apply(x, N, HW, C, Ctot, c_off, groups, eps, stats_ws, gamma, beta, silu, out, OCtot, oc_off, st);
}

// ------------------------------------------------------------------------------------------------ LayerNorm (warp per row)
constexpr int kLNMaxVec = 8;  // C <= 32*8*8 = 2048
__global__ void __launch_bounds__(256) layernorm_kernel(const __half* __restrict__ x, int rows, int C, float eps,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        __half* __restrict__ out) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int nvec = C / 8;
  const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)row * C);
  float v[kLNMaxVec][8];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < kLNMaxVec; ++k) {
    const int i = lane + k * 32;
    if (i < nvec) {
      const uint4 u = src[i];
      const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[k][j] = __half2float(h[j]);
        s += v[k][j];
      }
    }
  }
  const float mean = warp_sum(s) / C;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < kLNMaxVec; ++k) {
    const int i = lane + k * 32;
    if (i < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[k][j] - mean;
        q += d * d;
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
  uint4* dst = reinterpret_cast<uint4*>(out + (size_t)row * C);
#pragma unroll
  for (int k = 0; k < kLNMaxVec; ++k) {
    const int i = lane + k * 32;
    if (i < nvec) {
      uint4 o;
      __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
      for (int j = 0; j < 8; ++j) oh[j] = __float2half_rn((v[k][j] - mean) * rstd * __ldg(gamma + i * 8 + j) + __ldg(beta + i * 8 + j));
      dst[i] = o;
    }
  }
}

cudaError_t launch_layernorm(const __half* x, int rows, int C, float eps, const float* gamma, const float* beta, __half* out,
                             cudaStream_t st) {
  if (C % 8 != 0 || C > 32 * 8 * kLNMaxVec) return cudaErrorInvalidValue;
  return launch_kernel_plain(layernorm_kernel, dim3((rows + 7) / 8), dim3(256), 0, st, x, rows, C, eps, gamma, beta, out);
}

// ------------------------------------------------------------------------------------------------ softmax (warp per row)
// x: rows x ld fp16 logits; probabilities over the first `valid` columns of each row (scaled by `scale`), the padded
// columns [valid, cols) are written as 0 so that the P.V GEMM may run over the padded key count.
constexpr int kSMMaxVec = 6;  // cols <= 32*8*6 = 1536
__global__ void __launch_bounds__(256) softmax_kernel(const __half* __restrict__ x, int rows, int cols, int ld, int valid, float scale,
                                                      __half* __restrict__ out) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int nvec = cols / 8;
  const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)row * ld);
  float v[kSMMaxVec][8];
  float m = -INFINITY;
#pragma unroll
  for (int k = 0; k < kSMMaxVec; ++k) {
    const int i = lane + k * 32;
    if (i < nvec) {
      const uint4 u = src[i];
      const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const bool ok = (i * 8 + j) < valid;
        v[k][j] = ok ? __half2float(h[j]) * scale : -INFINITY;
        m = fmaxf(m, v[k][j]);
      }
    }
  }
  m = warp_max(m);
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < kSMMaxVec; ++k) {
    const int i = lane + k * 32;
    if (i < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[k][j] = (v[k][j] == -INFINITY) ? 0.f : __expf(v[k][j] - m);
        s += v[k][j];
      }
    }
  }
  const float inv = 1.f / warp_sum(s);
  uint4* dst = reinterpret_cast<uint4*>(out + (size_t)row * ld);
#pragma unroll
  for (int k = 0; k < kSMMaxVec; ++k) {
    const int i = lane + k * 32;
    if (i < nvec) {
      uint4 o;
      __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
      for (int j = 0; j < 8; ++j) oh[j] = __float2half_rn(v[k][j] * inv);
      dst[i] = o;
    }
  }
}

// Wide rows (cols > 1536: self-attention over the 64x64-latent maps of BASELINE configs[4], 4096 keys): one block per row,
// values in registers (cols <= 256*8*4 = 8192), block-wide max / sum through shared memory.
constexpr int kSMWideVec = 4;
__global__ void __launch_bounds__(256) softmax_wide_kernel(const __half* __restrict__ x, int cols, int ld, int valid, float scale,
                                                           __half* __restrict__ out) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  __shared__ float red[8];
  const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int nvec = cols / 8;
  const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)row * ld);
  float v[kSMWideVec][8];
  float m = -INFINITY;
#pragma unroll
  for (int k = 0; k < kSMWideVec; ++k) {
    const int i = tid + k * 256;
    if (i < nvec) {
      const uint4 u = src[i];
      const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const bool ok = (i * 8 + j) < valid;
        v[k][j] = ok ? __half2float(h[j]) * scale : -INFINITY;
        m = fmaxf(m, v[k][j]);
      }
    }
  }
  m = warp_max(m);
  if (lane == 0) red[w] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < kSMWideVec; ++k) {
    const int i = tid + k * 256;
    if (i < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[k][j] = (v[k][j] == -INFINITY) ? 0.f : __expf(v[k][j] - m);
        s += v[k][j];
      }
    }
  }
  s = warp_sum(s);
  if (lane == 0) red[w] = s;
  __syncthreads();
  s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += red[i];
  const float inv = 1.f / s;
  uint4* dst = reinterpret_cast<uint4*>(out + (size_t)row * ld);
#pragma unroll
  for (int k = 0; k < kSMWideVec; ++k) {
    const int i = tid + k * 256;
    if (i < nvec) {
      uint4 o;
      __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
      for (int j = 0; j < 8; ++j) oh[j] = __float2half_rn(v[k][j] * inv);
      dst[i] = o;
    }
  }
}

cudaError_t launch_softmax(const __half* x, int rows, int cols, int ld, int valid, float scale, __half* out, cudaStream_t st) {
  if (cols % 8 != 0 || cols > 256 * 8 * kSMWideVec || ld % 8 != 0 || valid > cols || valid < 1) return cudaErrorInvalidValue;
  if (cols > 32 * 8 * kSMMaxVec) return launch_kernel_plain(softmax_wide_kernel, dim3(rows), dim3(256), 0, st, x, cols, ld, valid, scale, out);
  return launch_kernel_plain(softmax_kernel, dim3((rows + 7) / 8), dim3(256), 0, st, x, rows, cols, ld, valid, scale, out);
}

// ------------------------------------------------------------------------------------------------ GEGLU / GELU / add
// h: rows x 2H  ->  out rows x H = h[:, :H] * gelu(h[:, H:])   (diffusers GEGLU: hidden, gate = proj(x).chunk(2))
__global__ void __launch_bounds__(256) geglu_kernel(const __half* __restrict__ h, size_t total_vec, int H, __half* __restrict__ out) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  const unsigned vpr = H / 8;
  for (unsigned i = blockIdx.x * 256u + threadIdx.x; i < (unsigned)total_vec; i += gridDim.x * 256u) {
    const size_t r = i / vpr;
    const int cv = (int)(i % vpr) * 8;
    const uint4 a = *reinterpret_cast<const uint4*>(h + r * 2 * H + cv);
    const uint4 g = *reinterpret_cast<const uint4*>(h + r * 2 * H + H + cv);
    const __half* ah = reinterpret_cast<const __half*>(&a);
    const __half* gh = reinterpret_cast<const __half*>(&g);
    uint4 o;
    __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
    for (int j = 0; j < 8; ++j) oh[j] = __float2half_rn(__half2float(ah[j]) * gelu_erf(__half2float(gh[j])));
    *reinterpret_cast<uint4*>(out + r * H + cv) = o;
  }
}
cudaError_t launch_geglu(const __half* h, size_t rows, int H, __half* out, cudaStream_t st) {
  if (H % 8 != 0) return cudaErrorInvalidValue;
  const size_t total = rows * (H / 8);
  int blocks = (int)((total + 255) / 256);
  if (blocks > 1184) blocks = 1184;
  return launch_kernel_plain(geglu_kernel, dim3(blocks), dim3(256), 0, st, h, total, H, out);
}

// elementwise: out = act(x (+ y broadcast over rows with period `period` vectors)) ; act 0 none, 1 gelu(erf), 2 silu
__global__ void __launch_bounds__(256) eltwise_kernel(const __half* __restrict__ x, const __half* __restrict__ y, size_t total_vec,
                                                      size_t period_vec, int act, __half* __restrict__ out) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  const unsigned tv = (unsigned)total_vec, pv = (unsigned)period_vec;
  for (unsigned i = blockIdx.x * 256u + threadIdx.x; i < tv; i += gridDim.x * 256u) {
    const uint4 a = reinterpret_cast<const uint4*>(x)[i];
    const __half* ah = reinterpret_cast<const __half*>(&a);
    uint4 b = make_uint4(0, 0, 0, 0);
    if (y) b = reinterpret_cast<const uint4*>(y)[i % pv];
    const __half* bh = reinterpret_cast<const __half*>(&b);
    uint4 o;
    __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float v = __half2float(ah[j]) + (y ? __half2float(bh[j]) : 0.f);
      if (act == 1) v = gelu_erf(v);
      if (act == 2) v = silu_f(v);
      oh[j] = __float2half_rn(v);
    }
    reinterpret_cast<uint4*>(out)[i] = o;
  }
}
cudaError_t launch_eltwise(const __half* x, const __half* y, size_t n, size_t period, int act, __half* out, cudaStream_t st) {
  if (n % 8 != 0 || (y && period % 8 != 0)) return cudaErrorInvalidValue;
  const size_t total = n / 8;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 1184) blocks = 1184;
  return launch_kernel_plain(eltwise_kernel, dim3(blocks), dim3(256), 0, st, x, y, total, y ? period / 8 : 1, act, out);
}

// ------------------------------------------------------------------------------------------------ layout helpers
__global__ void __launch_bounds__(256) upsample2x_kernel(const __half* __restrict__ x, int N, int H, int W, int C, __half* __restrict__ out) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  const unsigned vpp = C / 8;
  const unsigned total = (unsigned)N * (2 * H) * (2 * W) * vpp;   // < 2^32 for every tensor of the path
  for (unsigned i = blockIdx.x * 256u + threadIdx.x; i < total; i += gridDim.x * 256u) {
    const unsigned cv = i % vpp;
    unsigned p = i / vpp;
    const unsigned ox = p % (2u * W);
    p /= (2u * W);
    const unsigned oy = p % (2u * H);
    const unsigned n = p / (2u * H);
    reinterpret_cast<uint4*>(out)[i] =
        reinterpret_cast<const uint4*>(x)[(((size_t)n * H + (oy >> 1)) * W + (ox >> 1)) * vpp + cv];
  }
}
cudaError_t launch_upsample2x(const __half* x, int N, int H, int W, int C, __half* out, cudaStream_t st) {
  if (C % 8 != 0) return cudaErrorInvalidValue;
  const size_t total = (size_t)N * 4 * H * W * (C / 8);
  int blocks = (int)((total + 255) / 256);
  if (blocks > 2368) blocks = 2368;
  return launch_kernel_plain(upsample2x_kernel, dim3(blocks), dim3(256), 0, st, x, N, H, W, C, out);
}

__global__ void __launch_bounds__(256) copy_channels_kernel(const __half* __restrict__ src, size_t rows, int C, int SCtot, int sc_off,
                                                            __half* __restrict__ dst, int DCtot, int dc_off) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  const unsigned vpr = C / 8;
  const unsigned total = (unsigned)(rows * vpr);
  for (unsigned i = blockIdx.x * 256u + threadIdx.x; i < total; i += gridDim.x * 256u) {
    const size_t r = i / vpr;
    const int cv = (int)(i % vpr) * 8;
    *reinterpret_cast<uint4*>(dst + r * DCtot + dc_off + cv) = *reinterpret_cast<const uint4*>(src + r * SCtot + sc_off + cv);
  }
}
cudaError_t launch_copy_channels(const __half* src, size_t rows, int C, int SCtot, int sc_off, __half* dst, int DCtot, int dc_off,
                                 cudaStream_t st) {
  if ((C % 8) || (SCtot % 8) || (sc_off % 8) || (DCtot % 8) || (dc_off % 8)) return cudaErrorInvalidValue;
  const size_t total = rows * (C / 8);
  int blocks = (int)((total + 255) / 256);
  if (blocks > 2368) blocks = 2368;
  if (blocks < 1) blocks = 1;
  return launch_kernel_plain(copy_channels_kernel, dim3(blocks), dim3(256), 0, st, src, rows, C, SCtot, sc_off, dst, DCtot, dc_off);
}

// V [B, n_keys, Ctot] (head h = channels [c_off + h*d, +d))  ->  VT [B, heads, d, n_pad]  (zero for key >= n_keys)
__global__ void __launch_bounds__(256) transpose_heads_kernel(const __half* __restrict__ v, int n_keys, int Ctot, int c_off, int heads, int d,
                                                              int n_pad, __half* __restrict__ vt) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  __shared__ __half tile[32][33];
  const int bh = blockIdx.z, b = bh / heads, h = bh % heads;
  const int k0 = blockIdx.x * 32, j0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int r = ty; r < 32; r += 8) {
    const int key = k0 + r, j = j0 + tx;
    tile[r][tx] = (key < n_keys && j < d) ? v[((size_t)b * n_keys + key) * Ctot + c_off + h * d + j] : __float2half(0.f);
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int j = j0 + r, key = k0 + tx;
    if (j < d && key < n_pad) vt[(((size_t)b * heads + h) * d + j) * n_pad + key] = tile[tx][r];
  }
}
cudaError_t launch_transpose_heads(const __half* v, int B, int n_keys, int Ctot, int c_off, int heads, int d, int n_pad, __half* vt,
                                   cudaStream_t st) {
  dim3 grid((n_pad + 31) / 32, (d + 31) / 32, B * heads);
  return launch_kernel_plain(transpose_heads_kernel, dim3(grid), dim3(256), 0, st, v, n_keys, Ctot, c_off, heads, d, n_pad, vt);
}

// VAE decode post-processing (vae.py:104-107): (x/2+0.5).clamp(0,1) in fp16, *255, round-half-even, RGB->BGR, u8 NHWC
__global__ void __launch_bounds__(256) vae_post_kernel(const __half* __restrict__ x, size_t npix, int Ctot, uint8_t* __restrict__ out) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < npix; i += (size_t)gridDim.x * 256) {
    const __half* px = x + i * Ctot;
    uint8_t o[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      __half h = __hadd(__hmul(px[c], __float2half(0.5f)), __float2half(0.5f));
      float f = fminf(fmaxf(__half2float(h), 0.f), 1.f);
      o[2 - c] = (uint8_t)__float2int_rn(f * 255.f);
    }
    out[i * 3 + 0] = o[0];
    out[i * 3 + 1] = o[1];
    out[i * 3 + 2] = o[2];
  }
}
cudaError_t launch_vae_post(const __half* x, size_t npix, int Ctot, uint8_t* out, cudaStream_t st) {
  int blocks = (int)((npix + 255) / 256);
  if (blocks > 2368) blocks = 2368;
  return launch_kernel_plain(vae_post_kernel, dim3(blocks), dim3(256), 0, st, x, npix, Ctot, out);
}

// u8 BGR image [N,H,W,3] -> fp16 NHWC [N,H,W,16] RGB normalised to [-1,1] (channels 3..15 zero); upper-half mask optional
// (vae.py:51-82: BGR->RGB, /255, x*(mask>0.5) on the masked copy BEFORE Normalize(0.5,0.5))
__global__ void __launch_bounds__(256) vae_pre_kernel(const uint8_t* __restrict__ img, int N, int H, int W, int half_mask,
                                                      __half* __restrict__ out) {
  const size_t npix = (size_t)N * H * W;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < npix; i += (size_t)gridDim.x * 256) {
    const int y = (int)((i / W) % H);
    const bool keep = !half_mask || y < H / 2;
    uint4 o = make_uint4(0, 0, 0, 0);
    __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = (float)((double)img[i * 3 + (2 - c)] / 255.0);
      if (!keep) v = 0.f;
      oh[c] = __float2half_rn((v - 0.5f) / 0.5f);
    }
    reinterpret_cast<uint4*>(out)[i * 2] = o;
    reinterpret_cast<uint4*>(out)[i * 2 + 1] = make_uint4(0, 0, 0, 0);
  }
}
cudaError_t launch_vae_pre(const uint8_t* img, int N, int H, int W, int half_mask, __half* out, cudaStream_t st) {
  const size_t npix = (size_t)N * H * W;
  int blocks = (int)((npix + 255) / 256);
  if (blocks > 2368) blocks = 2368;
  vae_pre_kernel<<<blocks, 256, 0, st>>>(img, N, H, W, half_mask, out);
  return cudaGetLastError();
}

// gather rows by mirror index: out[i] = table[mirror_index(n, *d_index + i)]  (latent / asset gather for a batch)
__global__ void __launch_bounds__(256) gather_rows_kernel(const __half* __restrict__ table, int n, const int* __restrict__ d_index,
                                                          size_t row_vec, __half* __restrict__ out) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  const int i = blockIdx.y;
  const int index = *d_index + i;
  const int turn = index / n, res = index % n;
  const int idx = (turn % 2 == 0) ? res : n - res - 1;
  for (size_t v = (size_t)blockIdx.x * 256 + threadIdx.x; v < row_vec; v += (size_t)gridDim.x * 256)
    reinterpret_cast<uint4*>(out)[(size_t)i * row_vec + v] = reinterpret_cast<const uint4*>(table)[(size_t)idx * row_vec + v];
}
cudaError_t launch_gather_rows(const __half* table, int n, const int* d_index, int B, size_t row_elems, __half* out, cudaStream_t st) {
  if (row_elems % 8 != 0) return cudaErrorInvalidValue;
  const size_t rv = row_elems / 8;
  int bx = (int)((rv + 255) / 256);
  if (bx > 64) bx = 64;
  return launch_kernel_plain(gather_rows_kernel, dim3(dim3(bx, B)), dim3(256), 0, st, table, n, d_index, rv, out);
}

}  // namespace ltb
