// Small bandwidth-bound kernels around the wav2lip256 tensor-core convs.
//   prep_faces  : replaces the numpy batch assembly of LipReal.inference_batch
//                 (avatars/wav2lip_avatar.py:119-134: gather by mirror_index, zero lower half of the masked copy,
//                  concat (masked, full), /255, HWC->CHW, H2D) — faces stay resident on the GPU as u8.
//   audio_conv0 : first audio-encoder block, Conv2d(1,32,3,1,1)+BN+ReLU (wav2lip_v2.py:42) — K=9, CUDA cores.
//   head        : output_block.1 Conv2d(32,3,1) + Sigmoid (wav2lip_v2.py:90-91) and the "* 255" of
//                 wav2lip_avatar.py:138, emitting pred in the reference layout (B,256,256,3) f32 BGR.
#include "ltb_internal.h"
#include "ops.h"

namespace ltb {

__device__ __forceinline__ int mirror_index_dev(int size, int index) {
  // utils/image.py:26-32
  const int turn = index / size;
  const int res = index % size;
  return (turn % 2 == 0) ? res : size - res - 1;
}

constexpr int kPadH = 262;  // 256 + 3 + 3
constexpr int kPadW = 264;  // 256 + 3 + 5 (row pitch multiple of 8 pixels)

__global__ void __launch_bounds__(256) w2l_prep_faces_kernel(const uint8_t* __restrict__ faces, int nfaces,
                                                             const int* __restrict__ d_index,
                                                             __half* __restrict__ img_pad, const SlotDesc* __restrict__ slots) {
  const int b = blockIdx.y;
  const int pix = blockIdx.x * 256 + threadIdx.x;  // 0..65535
  const int y = pix >> 8, x = pix & 255;
  const uint8_t* src;
  if (slots) {   // cross-session batch: every slot names its own face crop
    src = slots[b].face + (size_t)pix * 3;
  } else {
    const int fidx = mirror_index_dev(nfaces, __ldg(d_index) + b);
    src = faces + ((size_t)fidx * 65536 + pix) * 3;
  }
  const float inv = 1.0f / 255.0f;
  const float c0 = src[0] * inv, c1 = src[1] * inv, c2 = src[2] * inv;
  const bool upper = y < 128;  // img_masked[:, face.shape[0]//2:] = 0
  uint4 o;
  __half2* oh = reinterpret_cast<__half2*>(&o);
  oh[0] = __floats2half2_rn(upper ? c0 : 0.f, upper ? c1 : 0.f);
  oh[1] = __floats2half2_rn(upper ? c2 : 0.f, c0);
  oh[2] = __floats2half2_rn(c1, c2);
  oh[3] = __floats2half2_rn(0.f, 0.f);
  uint4* dst = reinterpret_cast<uint4*>(img_pad + (((size_t)b * kPadH + (y + 3)) * kPadW + (x + 3)) * 8);
  *dst = o;
}

cudaError_t launch_w2l_prep_faces(const uint8_t* faces, int nfaces, const int* d_index, int B, __half* img_pad,
                                  cudaStream_t st, const SlotDesc* slots) {
  dim3 grid(256, B);
  w2l_prep_faces_kernel<<<grid, 256, 0, st>>>(faces, nfaces, d_index, img_pad, slots);
  return cudaGetLastError();
}

__global__ void __launch_bounds__(128) w2l_audio_conv0_kernel(const float* __restrict__ mel, const float* __restrict__ w,
                                                              const float* __restrict__ bias, __half* __restrict__ out,
                                                              int total) {
  __shared__ float sw[32 * 9];
  __shared__ float sb[32];
  for (int i = threadIdx.x; i < 288; i += 128) sw[i] = w[i];
  if (threadIdx.x < 32) sb[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const int pix = blockIdx.x * 128 + threadIdx.x;
  if (pix >= total) return;
  const int b = pix / 1280, rem = pix % 1280;
  const int y = rem / 16, x = rem % 16;
  float v[9];
#pragma unroll
  for (int kh = 0; kh < 3; ++kh)
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
      const int iy = y + kh - 1, ix = x + kw - 1;
      v[kh * 3 + kw] = (iy >= 0 && iy < 80 && ix >= 0 && ix < 16) ? mel[(size_t)b * 1280 + iy * 16 + ix] : 0.f;
    }
  __half2 o[16];
#pragma unroll
  for (int c = 0; c < 32; c += 2) {
    float a0 = sb[c], a1 = sb[c + 1];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      a0 = fmaf(v[t], sw[c * 9 + t], a0);
      a1 = fmaf(v[t], sw[(c + 1) * 9 + t], a1);
    }
    o[c / 2] = __floats2half2_rn(fmaxf(a0, 0.f), fmaxf(a1, 0.f));
  }
  uint4* dst = reinterpret_cast<uint4*>(out + (size_t)pix * 32);
  const uint4* so = reinterpret_cast<const uint4*>(o);
#pragma unroll
  for (int i = 0; i < 4; ++i) dst[i] = so[i];
}

cudaError_t launch_w2l_audio_conv0(const float* mel, const float* w9x32, const float* bias, __half* out, int B,
                                   cudaStream_t st) {
  const int total = B * 1280;
  w2l_audio_conv0_kernel<<<(total + 127) / 128, 128, 0, st>>>(mel, w9x32, bias, out, total);
  return cudaGetLastError();
}

// GRP: the block's image (hw % 256 == 0, so a block never straddles two) reads the weights of its group's slot
template <bool GRP>
__global__ void __launch_bounds__(256) w2l_head_kernel(const __half* __restrict__ x, const float* __restrict__ w,
                                                       const float* __restrict__ b, float* __restrict__ pred, int npix, int hw,
                                                       const WeightGroups grp) {
  __shared__ float sw[96];
  __shared__ float sb[3];
  if constexpr (GRP) {
    const int s = grp.slot[(int)((size_t)blockIdx.x * 256 / hw) / grp.images];
    w += s * grp.w_stride;
    b += s * grp.b_stride;
  }
  if (threadIdx.x < 96) sw[threadIdx.x] = w[threadIdx.x];
  if (threadIdx.x < 3) sb[threadIdx.x] = b[threadIdx.x];
  __syncthreads();
  const int pix = blockIdx.x * 256 + threadIdx.x;
  if (pix >= npix) return;
  const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)pix * 32);
  float a0 = sb[0], a1 = sb[1], a2 = sb[2];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint4 v = __ldg(src + i);
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 f = __half22float2(h[q]);
      const int c = i * 8 + q * 2;
      a0 = fmaf(f.x, sw[c], a0);
      a0 = fmaf(f.y, sw[c + 1], a0);
      a1 = fmaf(f.x, sw[32 + c], a1);
      a1 = fmaf(f.y, sw[32 + c + 1], a1);
      a2 = fmaf(f.x, sw[64 + c], a2);
      a2 = fmaf(f.y, sw[64 + c + 1], a2);
    }
  }
  float* o = pred + (size_t)pix * 3;
  o[0] = (1.f / (1.f + expf(-a0))) * 255.f;  // sigmoid, then "* 255." as wav2lip_avatar.py:138
  o[1] = (1.f / (1.f + expf(-a1))) * 255.f;
  o[2] = (1.f / (1.f + expf(-a2))) * 255.f;
}

cudaError_t launch_w2l_head(const __half* x, const float* w3x32, const float* b3, float* pred, int npix, cudaStream_t st) {
  w2l_head_kernel<false><<<(npix + 255) / 256, 256, 0, st>>>(x, w3x32, b3, pred, npix, 0, WeightGroups{});
  return cudaGetLastError();
}

cudaError_t launch_head_grouped(const __half* x, const float* w3x32, const float* b3, float* pred, int npix, int hw, const WeightGroups& grp,
                                cudaStream_t st) {
  if (hw <= 0 || hw % 256 || npix % hw || grp.images < 1 || (npix / hw) % grp.images) return cudaErrorInvalidValue;
  w2l_head_kernel<true><<<(npix + 255) / 256, 256, 0, st>>>(x, w3x32, b3, pred, npix, hw, grp);
  return cudaGetLastError();
}

__global__ void set_int_kernel(int* p, int v) { *p = v; }
cudaError_t launch_set_int(int* p, int v, cudaStream_t st) {
  set_int_kernel<<<1, 1, 0, st>>>(p, v);
  return cudaGetLastError();
}

}  // namespace ltb
