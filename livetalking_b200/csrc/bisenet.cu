// BiSeNet face-parsing glue kernels (the MuseTalk avatar generator, avatars/musetalk/utils/face_parsing): the convolutions run on
// the conv planner (ltb_op_conv2d); here are the pieces around them (livetalking_b200/bisenet.py).
//   * bisenet_prep:            u8 RGB 512 x 512 -> fp16 ToTensor + Normalize, space-to-depth 2 x 2 into a zero-bordered 259 x 259 x 16
//                              map, which turns the 7 x 7 stride-2 pad-3 stem into a 4 x 4 valid stride-1 conv (16 taps)
//   * maxpool3x3s2:            MaxPool2d(3, 2, 1) on NHWC fp16 (padding never wins)
//   * chan_gate:               per image, the fp32 global average of an NHWC map, one or two fp32 mat-vecs and an activation: ARM's
//                              conv_atten + BN + sigmoid, conv_avg + BN + ReLU, FFM's 1x1 -> ReLU -> 1x1 -> sigmoid
//   * chan_scale_add:          out = x * g[n, c] + y, y a per-image vector, a tensor or x itself, in fp32 with one fp16 rounding
//   * bisenet_upsample_argmax: F.interpolate(bilinear, align_corners=True) of the logits to 512 x 512 and the arg-max over the real
//                              classes (exact ties: the lowest class, as numpy's argmax), without writing the interpolated logits
#include "ltb_internal.h"
#include "ops.h"
#include "ptx_sm90.cuh"

namespace ltb {

namespace {
constexpr long long kMaxBlocks = 132 * 64;

unsigned grid_for(long long items, int threads) {
  long long b = (items + threads - 1) / threads;
  if (b > kMaxBlocks) b = kMaxBlocks;
  return (unsigned)(b < 1 ? 1 : b);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
}  // namespace

// ------------------------------------------------------------------------------------------------ prep
// One thread = one pixel (j, i) of the space-to-depth map: it covers the input pixels (2 (j - 2) + by, 2 (i - 2) + bx), channel
// (2 by + bx) * 3 + c.  Pixels outside the image are 0 after normalisation (conv padding).  Each value follows torchvision's
// order in fp32: v / 255 (ToTensor), then (t - mean) / std (Normalize), IEEE divides, rounded to fp16 once.
__global__ void __launch_bounds__(256) bisenet_prep_kernel(const uint8_t* __restrict__ rgb, long long npix, __half* __restrict__ out) {
  pdl_launch_dependents();
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < npix; i += (long long)gridDim.x * 256) {
    const int x = (int)(i % kBisenetS2d), y = (int)((i / kBisenetS2d) % kBisenetS2d);
    const long long n = i / ((long long)kBisenetS2d * kBisenetS2d);
    alignas(16) __half v[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) v[k] = __float2half(0.f);
#pragma unroll
    for (int by = 0; by < 2; ++by)
#pragma unroll
      for (int bx = 0; bx < 2; ++bx) {
        const int sy = 2 * (y - 2) + by, sx = 2 * (x - 2) + bx;
        if (sy < 0 || sy >= kBisenetIn || sx < 0 || sx >= kBisenetIn) continue;
        const uint8_t* p = rgb + ((n * kBisenetIn + sy) * kBisenetIn + sx) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float t = __fdiv_rn((float)p[c], 255.f);
          v[(by * 2 + bx) * 3 + c] = __float2half_rn(__fdiv_rn(__fsub_rn(t, mean[c]), stdv[c]));
        }
      }
    uint4* o = reinterpret_cast<uint4*>(out + i * kBisenetInC);
    o[0] = *reinterpret_cast<const uint4*>(&v[0]);
    o[1] = *reinterpret_cast<const uint4*>(&v[8]);
  }
}

cudaError_t launch_bisenet_prep(const uint8_t* rgb, int N, __half* out, cudaStream_t st) {
  if (N <= 0 || !aligned16(out)) return cudaErrorInvalidValue;
  const long long npix = (long long)N * kBisenetS2d * kBisenetS2d;
  return launch_kernel_plain(bisenet_prep_kernel, dim3(grid_for(npix, 256)), dim3(256), 0, st, rgb, npix, out);
}

// ------------------------------------------------------------------------------------------------ max-pool 3x3 / 2, pad 1
// One thread = 8 channels of one output pixel: up to nine 16-byte loads, one 16-byte store.  Taps outside the map are skipped
// (MaxPool2d pads with -inf, which never wins).
__global__ void __launch_bounds__(256) maxpool3x3s2_kernel(const __half* __restrict__ x, int IH, int IW, int C, int OH, int OW, long long total,
                                                           __half* __restrict__ out) {
  pdl_launch_dependents();
  const int cg = C >> 3;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int g = (int)(i % cg);
    const long long pix = i / cg;
    const int ox = (int)(pix % OW), oy = (int)((pix / OW) % OH);
    const long long n = pix / ((long long)OW * OH);
    alignas(16) __half2 r[4];
    bool first = true;
    for (int dy = -1; dy <= 1; ++dy) {
      const int iy = 2 * oy + dy;
      if (iy < 0 || iy >= IH) continue;
      for (int dx = -1; dx <= 1; ++dx) {
        const int ix = 2 * ox + dx;
        if (ix < 0 || ix >= IW) continue;
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(x + ((n * IH + iy) * IW + ix) * C + g * 8));
        const __half2* ha = reinterpret_cast<const __half2*>(&a);
#pragma unroll
        for (int k = 0; k < 4; ++k) r[k] = first ? ha[k] : __hmax2(r[k], ha[k]);
        first = false;
      }
    }
    *reinterpret_cast<uint4*>(out + pix * C + g * 8) = *reinterpret_cast<const uint4*>(r);
  }
}

cudaError_t launch_maxpool3x3s2(const __half* x, int N, int H, int W, int C, __half* out, cudaStream_t st) {
  if (N <= 0 || H <= 0 || W <= 0 || C <= 0 || (C & 7) || !aligned16(x) || !aligned16(out)) return cudaErrorInvalidValue;
  const int OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1;
  const long long total = (long long)N * OH * OW * (C >> 3);
  return launch_kernel_plain(maxpool3x3s2_kernel, dim3(grid_for(total, 256)), dim3(256), 0, st, x, H, W, C, OH, OW, total, out);
}

// ------------------------------------------------------------------------------------------------ channel gate
// One CTA per image.  Thread t sums 8 channels (group t % G, G = C / 8) over the pixels t / G, t / G + T, ... (T = threads / G) in
// fp32; thread c then adds the T partials of channel c in slot order and divides by HW: a fixed summation order, so a replay is
// bit-identical.  Then h = act1(W1 avg + b1) and, with a second layer, out = act2(W2 h + b2), each an fp32 FMA chain in input order.
constexpr int kGateThreads = 512;

__device__ __forceinline__ float gate_act(float v, int act) {
  if (act == kActRelu) return fmaxf(v, 0.f);
  if (act == kActSigmoid) return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-v)));
  return v;
}

__global__ void __launch_bounds__(kGateThreads) chan_gate_kernel(const __half* __restrict__ x, int HW, int C, int pitch, int c_off,
                                                                 const float* __restrict__ w1t, const float* __restrict__ b1, int n1, int act1,
                                                                 const float* __restrict__ w2t, const float* __restrict__ b2, int n2, int act2,
                                                                 float* __restrict__ out) {
  pdl_launch_dependents();
  __shared__ float part[kGateThreads * 8];
  __shared__ float avg[kChanGateMax];
  __shared__ float hid[kChanGateMax];
  const int n = blockIdx.x, tid = threadIdx.x, G = C >> 3, T = kGateThreads / G;
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = 0.f;
  if (tid < T * G) {
    const int g = tid % G;
    const __half* base = x + (size_t)n * HW * pitch + c_off + g * 8;
    for (int px = tid / G; px < HW; px += T) {
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
  if (tid < C) {
    const int g = tid >> 3, k = tid & 7;
    float s = 0.f;
    for (int slot = 0; slot < T; ++slot) s += part[(slot * G + g) * 8 + k];
    avg[tid] = __fdiv_rn(s, (float)HW);
  }
  __syncthreads();
  if (tid < n1) {
    float a = b1 ? __ldg(b1 + tid) : 0.f;
    for (int j = 0; j < C; ++j) a = fmaf(__ldg(w1t + (size_t)j * n1 + tid), avg[j], a);
    hid[tid] = gate_act(a, act1);
  }
  __syncthreads();
  if (!w2t) {
    if (tid < n1) out[(size_t)n * n1 + tid] = hid[tid];
    return;
  }
  if (tid < n2) {
    float a = b2 ? __ldg(b2 + tid) : 0.f;
    for (int j = 0; j < n1; ++j) a = fmaf(__ldg(w2t + (size_t)j * n2 + tid), hid[j], a);
    out[(size_t)n * n2 + tid] = gate_act(a, act2);
  }
}

cudaError_t launch_chan_gate(const ChanGateArgs& a, cudaStream_t st) {
  if (a.N <= 0 || a.HW <= 0 || a.C < 8 || (a.C & 7) || a.C > kChanGateMax || (a.pitch & 7) || (a.c_off & 7) || a.c_off + a.C > a.pitch ||
      !aligned16(a.x) || !a.w1t || a.n1 <= 0 || a.n1 > kChanGateMax || (a.w2t && (a.n2 <= 0 || a.n2 > kChanGateMax)) ||
      a.act1 < kActNone || a.act1 > kActSigmoid || a.act2 < kActNone || a.act2 > kActSigmoid)
    return cudaErrorInvalidValue;
  return launch_kernel_plain(chan_gate_kernel, dim3(a.N), dim3(kGateThreads), 0, st, a.x, a.HW, a.C, a.pitch, a.c_off, a.w1t, a.b1, a.n1,
                             a.act1, a.w2t, a.b2, a.n2, a.act2, a.out);
}

// ------------------------------------------------------------------------------------------------ channel scale + add
// One thread = 8 channels of one pixel: out = fp16(fp32(x) * g[n, c] + y) with y = yvec[n, c] (kScaleAddVec), the fp16 tensor y
// (kScaleAddTensor) or x itself (kScaleAddSelf): torch.mul then +, both in fp32, one rounding to fp16.
__global__ void __launch_bounds__(256) chan_scale_add_kernel(const ChanScaleAddArgs a, long long total) {
  pdl_launch_dependents();
  const int cg = a.C >> 3;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int g = (int)(i % cg);
    const long long pix = i / cg;
    const long long n = pix / a.HW;
    const uint4 xv = __ldg(reinterpret_cast<const uint4*>(a.x + pix * a.xpitch + a.xoff + g * 8));
    uint4 yv = xv;
    if (a.mode == kScaleAddTensor) yv = __ldg(reinterpret_cast<const uint4*>(a.y + pix * a.ypitch + a.yoff + g * 8));
    const __half* xh = reinterpret_cast<const __half*>(&xv);
    const __half* yh = reinterpret_cast<const __half*>(&yv);
    const float* gp = a.g + n * a.C + g * 8;
    alignas(16) __half r[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float yk = a.mode == kScaleAddVec ? __ldg(a.yvec + n * a.C + g * 8 + k) : __half2float(yh[k]);
      r[k] = __float2half_rn(__fadd_rn(__fmul_rn(__half2float(xh[k]), __ldg(gp + k)), yk));
    }
    *reinterpret_cast<uint4*>(a.out + pix * a.opitch + a.ooff + g * 8) = *reinterpret_cast<const uint4*>(r);
  }
}

cudaError_t launch_chan_scale_add(const ChanScaleAddArgs& a, cudaStream_t st) {
  const bool bad_y = (a.mode == kScaleAddVec && !a.yvec) ||
                     (a.mode == kScaleAddTensor && (!a.y || (a.ypitch & 7) || (a.yoff & 7) || a.yoff + a.C > a.ypitch || !aligned16(a.y))) ||
                     a.mode < kScaleAddVec || a.mode > kScaleAddSelf;
  if (a.N <= 0 || a.HW <= 0 || a.C <= 0 || (a.C & 7) || (a.xpitch & 7) || (a.xoff & 7) || a.xoff + a.C > a.xpitch || (a.opitch & 7) ||
      (a.ooff & 7) || a.ooff + a.C > a.opitch || !aligned16(a.x) || !aligned16(a.out) || !a.g || bad_y)
    return cudaErrorInvalidValue;
  const long long total = (long long)a.N * a.HW * (a.C >> 3);
  return launch_kernel_plain(chan_scale_add_kernel, dim3(grid_for(total, 256)), dim3(256), 0, st, a, total);
}

// ------------------------------------------------------------------------------------------------ upsample + arg-max
// One thread = one output pixel.  Coordinates as torch's upsample_bilinear2d with align_corners=True in fp32:
// scale = (in - 1) / (out - 1), src = scale * dst, i0 = int(src), i1 = i0 + (i0 < in - 1), l1 = src - i0, l0 = 1 - l1, and
// val = l0y (l0x v00 + l1x v01) + l1y (l0x v10 + l1x v11).  The arg-max keeps the first of equal values (the lowest class).
__global__ void __launch_bounds__(256) bisenet_upsample_argmax_kernel(const __half* __restrict__ logits, int IH, int IW, int pitch, int ncls,
                                                                      int OH, int OW, long long total, uint8_t* __restrict__ out) {
  pdl_launch_dependents();
  const float sh = OH > 1 ? __fdiv_rn((float)(IH - 1), (float)(OH - 1)) : 0.f;
  const float sw = OW > 1 ? __fdiv_rn((float)(IW - 1), (float)(OW - 1)) : 0.f;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ox = (int)(i % OW), oy = (int)((i / OW) % OH);
    const long long n = i / ((long long)OW * OH);
    const float ry = __fmul_rn(sh, (float)oy), rx = __fmul_rn(sw, (float)ox);
    const int y0 = (int)ry, x0 = (int)rx;
    const int y1 = y0 + (y0 < IH - 1 ? 1 : 0), x1 = x0 + (x0 < IW - 1 ? 1 : 0);
    const float ly1 = __fsub_rn(ry, (float)y0), lx1 = __fsub_rn(rx, (float)x0);
    const float ly0 = __fsub_rn(1.f, ly1), lx0 = __fsub_rn(1.f, lx1);
    const __half* img = logits + n * IH * IW * pitch;
    const __half* p00 = img + ((long long)y0 * IW + x0) * pitch;
    const __half* p01 = img + ((long long)y0 * IW + x1) * pitch;
    const __half* p10 = img + ((long long)y1 * IW + x0) * pitch;
    const __half* p11 = img + ((long long)y1 * IW + x1) * pitch;
    float best = 0.f;
    int arg = 0;
    for (int c0 = 0; c0 < ncls; c0 += 8) {
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(p00 + c0)), b = __ldg(reinterpret_cast<const uint4*>(p01 + c0));
      const uint4 c = __ldg(reinterpret_cast<const uint4*>(p10 + c0)), d = __ldg(reinterpret_cast<const uint4*>(p11 + c0));
      const __half *ha = reinterpret_cast<const __half*>(&a), *hb = reinterpret_cast<const __half*>(&b);
      const __half *hc = reinterpret_cast<const __half*>(&c), *hd = reinterpret_cast<const __half*>(&d);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        if (c0 + k >= ncls) break;
        const float top = __fadd_rn(__fmul_rn(lx0, __half2float(ha[k])), __fmul_rn(lx1, __half2float(hb[k])));
        const float bot = __fadd_rn(__fmul_rn(lx0, __half2float(hc[k])), __fmul_rn(lx1, __half2float(hd[k])));
        const float v = __fadd_rn(__fmul_rn(ly0, top), __fmul_rn(ly1, bot));
        if (c0 + k == 0 || v > best) {
          best = v;
          arg = c0 + k;
        }
      }
    }
    out[i] = (uint8_t)arg;
  }
}

cudaError_t launch_bisenet_upsample_argmax(const __half* logits, int N, int IH, int IW, int pitch, int ncls, int OH, int OW, uint8_t* out,
                                           cudaStream_t st) {
  if (N <= 0 || IH <= 0 || IW <= 0 || OH <= 0 || OW <= 0 || ncls <= 0 || ncls > 255 || (pitch & 7) || (ncls + 7) / 8 * 8 > pitch ||
      !aligned16(logits))
    return cudaErrorInvalidValue;
  const long long total = (long long)N * OH * OW;
  return launch_kernel_plain(bisenet_upsample_argmax_kernel, dim3(grid_for(total, 256)), dim3(256), 0, st, logits, IH, IW, pitch, ncls, OH,
                             OW, total, out);
}

}  // namespace ltb
