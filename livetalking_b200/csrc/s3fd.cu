// S3FD face detector glue kernels (the wav2lip avatar generator, avatars/wav2lip/genavatar.py -> face_detection/detection/sfd):
// the convolutions run on the conv planner (ltb_op_conv2d); here are the pieces around them.
//   * s3fd_prep:     u8 BGR frames -> fp16 NHWC, RGB minus the per-channel means [104, 117, 123] (batch_detect, detect.py:58-65),
//                    zero-padded to 16 channels (both conv kernels need Cin >= 16)
//   * maxpool2x2:    F.max_pool2d(h, 2, 2) on NHWC fp16, floor semantics for odd maps
//   * l2norm_scale:  L2Norm (net_s3fd.py:6-19): x / (sqrt(sum_c x^2) + 1e-10) * w[c], fp32 sum of squares
//   * s3fd_select:   per image, the softmax face score of every anchor of the six heads, the arg-max, and the decoded box of the
//                    arg-max when its score is above the threshold.  This is what batch_detect + nms(0.3) + the score > 0.5 filter
//                    + d[0] of FaceAlignment.get_detections_for_batch reduce to (livetalking_b200/s3fd.py explains why).
#include "ltb_internal.h"
#include "ops.h"
#include "ptx_sm90.cuh"

namespace ltb {

// ------------------------------------------------------------------------------------------------ prep
// One thread = one pixel: three byte loads, two 16-byte stores (channels 0-7 and the zero channels 8-15).
__global__ void __launch_bounds__(256) s3fd_prep_kernel(const uint8_t* __restrict__ bgr, long long npix, __half* __restrict__ out) {
  pdl_launch_dependents();   // a PDL-launched successor (the conv kernels) may start its prologue now; it waits before reading
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < npix; i += (long long)gridDim.x * 256) {
    const uint8_t* p = bgr + i * 3;
    uint4 v;
    __half2* h = reinterpret_cast<__half2*>(&v);
    h[0] = __halves2half2(__int2half_rn((int)p[2] - 104), __int2half_rn((int)p[1] - 117));   // exact: integers in [-123, 151]
    h[1] = __halves2half2(__int2half_rn((int)p[0] - 123), __float2half(0.f));
    h[2] = h[3] = __float2half2_rn(0.f);
    uint4* o = reinterpret_cast<uint4*>(out + i * kS3fdInC);
    o[0] = v;
    o[1] = make_uint4(0, 0, 0, 0);
  }
}

cudaError_t launch_s3fd_prep(const uint8_t* bgr, int N, int H, int W, __half* out, cudaStream_t st) {
  if (N <= 0 || H <= 0 || W <= 0 || (reinterpret_cast<uintptr_t>(out) & 15)) return cudaErrorInvalidValue;
  const long long npix = (long long)N * H * W;
  long long blocks = (npix + 255) / 256;
  if (blocks > 132 * 64) blocks = 132 * 64;
  return launch_kernel_plain(s3fd_prep_kernel, dim3((unsigned)blocks), dim3(256), 0, st, bgr, npix, out);
}

// ------------------------------------------------------------------------------------------------ max-pool 2x2 / 2
// One thread = 8 channels of one output pixel: four 16-byte loads, one 16-byte store.  OH = IH / 2, OW = IW / 2 (floor: the last
// row / column of an odd map is dropped, as F.max_pool2d(h, 2, 2) does).
__global__ void __launch_bounds__(256) maxpool2x2_kernel(const __half* __restrict__ x, int N, int IH, int IW, int C, __half* __restrict__ out) {
  pdl_launch_dependents();
  const int OH = IH >> 1, OW = IW >> 1, cg = C >> 3;
  const long long total = (long long)N * OH * OW * cg;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int g = (int)(i % cg);
    const long long pix = i / cg;
    const int ox = (int)(pix % OW), oy = (int)((pix / OW) % OH);
    const long long n = pix / ((long long)OW * OH);
    const __half* src = x + (((n * IH + 2 * oy) * IW + 2 * ox) * C) + g * 8;
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(src));
    const uint4 b = __ldg(reinterpret_cast<const uint4*>(src + C));
    const uint4 c = __ldg(reinterpret_cast<const uint4*>(src + (long long)IW * C));
    const uint4 d = __ldg(reinterpret_cast<const uint4*>(src + (long long)IW * C + C));
    uint4 r;
    const __half2 *ha = reinterpret_cast<const __half2*>(&a), *hb = reinterpret_cast<const __half2*>(&b),
                  *hc = reinterpret_cast<const __half2*>(&c), *hd = reinterpret_cast<const __half2*>(&d);
    __half2* hr = reinterpret_cast<__half2*>(&r);
#pragma unroll
    for (int k = 0; k < 4; ++k) hr[k] = __hmax2(__hmax2(ha[k], hb[k]), __hmax2(hc[k], hd[k]));
    *reinterpret_cast<uint4*>(out + pix * C + g * 8) = r;
  }
}

cudaError_t launch_maxpool2x2(const __half* x, int N, int H, int W, int C, __half* out, cudaStream_t st) {
  if (N <= 0 || H < 2 || W < 2 || C <= 0 || (C & 7) || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(out) & 15))
    return cudaErrorInvalidValue;
  const long long total = (long long)N * (H >> 1) * (W >> 1) * (C >> 3);
  long long blocks = (total + 255) / 256;
  if (blocks > 132 * 64) blocks = 132 * 64;
  return launch_kernel_plain(maxpool2x2_kernel, dim3((unsigned)blocks), dim3(256), 0, st, x, N, H, W, C, out);
}

// ------------------------------------------------------------------------------------------------ L2Norm
// One warp = one pixel, lane l holds the 8-channel groups l and l + 32 (C <= 512).  The pixel is read completely before it is
// written, so out may equal x.
constexpr int kL2MaxGroups = 2;
__global__ void __launch_bounds__(256) l2norm_scale_kernel(const __half* x, long long npix, int C, const float* __restrict__ w, float eps,
                                                           __half* out) {
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31, cg = C >> 3;
  const long long warps = (long long)gridDim.x * 8;
  for (long long p = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); p < npix; p += warps) {
    uint4 v[kL2MaxGroups];
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < kL2MaxGroups; ++k) {
      const int g = lane + 32 * k;
      if (g < cg) {
        v[k] = *reinterpret_cast<const uint4*>(x + p * C + g * 8);
        const __half2* h = reinterpret_cast<const __half2*>(&v[k]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(h[j]);
          ss = fmaf(f.x, f.x, ss);
          ss = fmaf(f.y, f.y, ss);
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float norm = sqrtf(ss) + eps;
#pragma unroll
    for (int k = 0; k < kL2MaxGroups; ++k) {
      const int g = lane + 32 * k;
      if (g < cg) {
        const __half2* h = reinterpret_cast<const __half2*>(&v[k]);
        uint4 r;
        __half2* hr = reinterpret_cast<__half2*>(&r);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(h[j]);
          const int c = g * 8 + 2 * j;
          hr[j] = __floats2half2_rn(f.x / norm * __ldg(w + c), f.y / norm * __ldg(w + c + 1));
        }
        *reinterpret_cast<uint4*>(out + p * C + g * 8) = r;
      }
    }
  }
}

cudaError_t launch_l2norm_scale(const __half* x, long long npix, int C, const float* w, float eps, __half* out, cudaStream_t st) {
  if (npix <= 0 || C <= 0 || (C & 7) || C > 256 * kL2MaxGroups || (reinterpret_cast<uintptr_t>(x) & 15) ||
      (reinterpret_cast<uintptr_t>(out) & 15))
    return cudaErrorInvalidValue;
  long long blocks = (npix + 7) / 8;
  if (blocks > 132 * 64) blocks = 132 * 64;
  return launch_kernel_plain(l2norm_scale_kernel, dim3((unsigned)blocks), dim3(256), 0, st, x, npix, C, w, eps, out);
}

// ------------------------------------------------------------------------------------------------ selection
// Level l (stride 4 << l, anchor size 16 << l) reads head map heads.p[l] [N][h[l]][w[l]][pitch] fp16: level 0 holds the conf
// channels c0..c3 (background = max(c0, c1, c2), face = c3) then loc 4..7, the others conf c0 (background), c1 (face) then loc
// 2..5.  Anchors are numbered level by level in row-major order; the arg-max takes the highest score and, among equal scores,
// the lowest number.  out_i[n][6] = {found, x1, y1, x2, y2, anchor}, out_s[n] = score of the arg-max.
constexpr int kSelThreads = 1024;

__device__ __forceinline__ float face_score(const __half* px, int level) {
  float bg, fc;
  if (level == 0) {
    bg = fmaxf(fmaxf(__half2float(px[0]), __half2float(px[1])), __half2float(px[2]));
    fc = __half2float(px[3]);
  } else {
    bg = __half2float(px[0]);
    fc = __half2float(px[1]);
  }
  // F.softmax over (bg, face), fp32
  const float m = fmaxf(bg, fc);
  const float e0 = expf(bg - m), e1 = expf(fc - m);
  return e1 / (e0 + e1);
}

__global__ void __launch_bounds__(kSelThreads) s3fd_select_kernel(const S3fdHeads heads, float thresh, int* __restrict__ out_i,
                                                                  float* __restrict__ out_s) {
  pdl_launch_dependents();
  const int n = blockIdx.x;
  float best = -1.f;
  int best_i = 0x7fffffff;
  int base = 0;
#pragma unroll   // static indices into the parameter struct: no local-memory copy of it
  for (int l = 0; l < kS3fdLevels; ++l) {
    const int hw = heads.h[l] * heads.w[l];
    const __half* m = heads.p[l] + (size_t)n * hw * heads.pitch;
    for (int i = threadIdx.x; i < hw; i += kSelThreads) {
      const float s = face_score(m + (size_t)i * heads.pitch, l);
      if (s > best) {   // ascending i per thread: the first of equal scores is kept
        best = s;
        best_i = base + i;
      }
    }
    base += hw;
  }
  // block arg-max: higher score, then lower anchor number
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float s2 = __shfl_xor_sync(0xffffffffu, best, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, best_i, o);
    if (s2 > best || (s2 == best && i2 < best_i)) {
      best = s2;
      best_i = i2;
    }
  }
  __shared__ float ss[kSelThreads / 32];
  __shared__ int si[kSelThreads / 32];
  if ((threadIdx.x & 31) == 0) {
    ss[threadIdx.x >> 5] = best;
    si[threadIdx.x >> 5] = best_i;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int k = 1; k < kSelThreads / 32; ++k)
    if (ss[k] > best || (ss[k] == best && si[k] < best_i)) {
      best = ss[k];
      best_i = si[k];
    }
  if (best_i == 0x7fffffff) best_i = 0;   // every score NaN (NaN head inputs): decode anchor 0 rather than read past the maps
  int l = -1, i = best_i, mw = 1, mhw = 1;
  const __half* mp = nullptr;
#pragma unroll
  for (int k = 0; k < kS3fdLevels; ++k) {
    const int hw = heads.h[k] * heads.w[k];
    if (l < 0) {
      if (i < hw || k == kS3fdLevels - 1) {
        l = k;
        mp = heads.p[k];
        mw = heads.w[k];
        mhw = hw;
      } else {
        i -= hw;
      }
    }
  }
  const int y = i / mw, x = i % mw;
  const __half* px = mp + ((size_t)n * mhw + i) * heads.pitch + (l == 0 ? 4 : 2);
  // batch_decode (bbox.py) in fp32: centre + loc * 0.1 * size, size * exp(loc * 0.2), then corners
  const float stride = (float)(4 << l), size = 4.f * stride;
  const float cx = stride / 2.f + x * stride, cy = stride / 2.f + y * stride;
  const float bx = cx + __half2float(px[0]) * 0.1f * size;
  const float by = cy + __half2float(px[1]) * 0.1f * size;
  const float bw = size * expf(__half2float(px[2]) * 0.2f);
  const float bh = size * expf(__half2float(px[3]) * 0.2f);
  const float x1 = bx - bw / 2.f, y1 = by - bh / 2.f;
  const float x2 = bw + x1, y2 = bh + y1;
  int* o = out_i + n * 6;
  o[0] = best > thresh ? 1 : 0;
  // np.clip(d, 0, None) then int(): truncation of a non-negative value
  o[1] = (int)fmaxf(x1, 0.f);
  o[2] = (int)fmaxf(y1, 0.f);
  o[3] = (int)fmaxf(x2, 0.f);
  o[4] = (int)fmaxf(y2, 0.f);
  o[5] = best_i;
  out_s[n] = best;
}

cudaError_t launch_s3fd_select(const S3fdHeads& heads, int N, float thresh, int* out_i, float* out_s, cudaStream_t st) {
  if (N <= 0 || heads.pitch <= 0) return cudaErrorInvalidValue;
  for (int l = 0; l < kS3fdLevels; ++l)
    if (!heads.p[l] || heads.h[l] <= 0 || heads.w[l] <= 0) return cudaErrorInvalidValue;
  return launch_kernel_plain(s3fd_select_kernel, dim3(N), dim3(kSelThreads), 0, st, heads, thresh, out_i, out_s);
}

}  // namespace ltb
