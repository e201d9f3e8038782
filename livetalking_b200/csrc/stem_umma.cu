// wav2lip256 stem on tensor cores: Conv2d(6,16,k7,s1,p3)+BN+ReLU (avatars/wav2lip/models/wav2lip_v2.py:13) over the
// zero-bordered 8-channel fp16 image written by w2l_prep_faces ([B,262,264,8]: 3 masked + 3 full + 2 zero channels).
//
// With 8 channels a pixel is exactly one 16-byte K chunk, so the im2col row of output pixel (y,x) for kernel row kh —
// 8 consecutive pixels x 8 channels = 64 K values (7 real taps + 1 zero-weighted) — is 128 CONTIGUOUS bytes of the image
// row, and the rows of neighbouring output pixels overlap by 112 bytes.  The SWIZZLE_NONE K-major wgmma descriptor
// expresses that directly: core-matrix rows 16 B apart (implicit), K chunks LBO = 16 B apart, 8-row groups (one image row
// of the 16x8 output tile) SBO = 256 B apart.  So ONE 22 x 16 pixel halo (5.6 KB, plain TMA box) feeds all 7 x 4 MMAs of a
// 128-pixel tile: 20x less operand traffic than gathering seven 16 KB im2col tiles.  Persistent CTAs, weights (14 KB)
// resident.  Warps 0-7: two consumer warpgroups (output rows 0-7 / 8-15 of the tile), warp 8: TMA producer.
#include <cuda.h>

#include <cstring>

#include "conv_tma.h"
#include "ltb_internal.h"
#include "ptx_sm90.cuh"
#include "stem_umma.h"

namespace ltb {

constexpr int kStemStages = 6;
constexpr int kStemABytes = 22 * 16 * 16;   // 5632 (halo: 22 rows x 16 px x 8 ch fp16)
constexpr int kStemAStride = 6144;          // stage pitch
constexpr int kStemWBytes = 7 * 16 * 128;   // 7 kernel rows x 16 cout x 64 k
constexpr int kStemThreads = 288;

__global__ void __launch_bounds__(kStemThreads, 1) stem_umma_kernel(const __grid_constant__ StemParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t a_full[kStemStages], a_empty[kStemStages];
  __shared__ __align__(8) uint64_t w_full;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t w_smem = smem0;                               // 14 KB, SWIZZLE_128B tiles of 16 rows
  const uint32_t a_smem = smem0 + kStemWBytes;                 // stages, SWIZZLE_NONE
  if (tid == 0) {
    for (int s = 0; s < kStemStages; ++s) {
      mbar_init(smem_u32(&a_full[s]), 1);
      mbar_init(smem_u32(&a_empty[s]), 8);   // one arrival per consumer warp
    }
    mbar_init(smem_u32(&w_full), 1);
    mbar_fence_init();
    tma_prefetch_desc(&p.tm_in);
    tma_prefetch_desc(&p.tm_w);
  }
  __syncthreads();
  const int tiles_per_img = 16 * 32;  // 256/16 x 256/8

  pdl_launch_dependents();   // PDL: weights (constants) before the wait, the padded image after it
  if (warp == 8 && lane == 0) {
    mbar_arrive_expect_tx(smem_u32(&w_full), kStemWBytes);
    tma_load_3d(w_smem, &p.tm_w, smem_u32(&w_full), 0, 0, 0);
  }
  pdl_wait();

  if (warp == 8) {
    if (lane == 0) {
      uint32_t ai = 0;
      for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x, ++ai) {
        const int img = t / tiles_per_img, r = t - img * tiles_per_img;
        const int ty = r >> 5, tx = r & 31;
        const uint32_t as = ai % kStemStages;
        mbar_wait(smem_u32(&a_empty[as]), ((ai / kStemStages) & 1u) ^ 1u);
        mbar_arrive_expect_tx(smem_u32(&a_full[as]), kStemABytes);
        // padded image coordinates: output (y,x) reads padded rows y..y+6, padded pixels x..x+7
        tma_load_4d(a_smem + as * kStemAStride, &p.tm_in, smem_u32(&a_full[as]), 0, tx * 8, ty * 16, img);
      }
    }
    return;
  }
  const int wg = warp >> 2, wq = warp & 3;
  // A: SWIZZLE_NONE, LBO = 16 B (next K chunk = next pixel), SBO = 256 B (next image row of the halo)
  constexpr uint32_t a_hi = 256u >> 4;
  constexpr uint32_t b_hi = wgmma_hi_128b(1024);
  float2 bias[2];
  const int cq = 2 * (lane & 3);
  bias[0] = __ldg(reinterpret_cast<const float2*>(p.bias + cq));
  bias[1] = __ldg(reinterpret_cast<const float2*>(p.bias + 8 + cq));
  mbar_wait(smem_u32(&w_full), 0);
  uint32_t ai = 0;
  for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x, ++ai) {
    const int img = t / tiles_per_img, r = t - img * tiles_per_img;
    const int ty = r >> 5, tx = r & 31;
    const uint32_t as = ai % kStemStages;
    mbar_wait(smem_u32(&a_full[as]), (ai / kStemStages) & 1u);
    const uint32_t a_base = a_smem + as * kStemAStride + wg * 8 * 256;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int kh = 0; kh < 7; ++kh) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t a_lo = (((a_base + kh * 256 + k * 32) & 0x3FFFFu) >> 4) | (1u << 16);   // LBO = 16 B
        const uint32_t b_lo = wgmma_lo(w_smem + kh * 2048 + k * 32);
        Wgmma<16>::ss(acc, wgmma_lohi(a_lo, a_hi), wgmma_lohi(b_lo, b_hi), 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&a_empty[as]));
    // rows of this thread: tile row 8*wg + 2*wq + hh, pixel lane/4 of the 8-pixel row
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const size_t pix = ((size_t)img * 256 + ty * 16 + wg * 8 + wq * 2 + hh) * 256 + tx * 8 + (lane >> 2);
      __half* optr = p.out + pix * p.OCtot + p.oc_off;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float x = fmaxf(acc[4 * i + 2 * hh] + bias[i].x, 0.f);
        const float y = fmaxf(acc[4 * i + 2 * hh + 1] + bias[i].y, 0.f);
        *reinterpret_cast<__half2*>(optr + 8 * i + cq) = __floats2half2_rn(fminf(x, 65504.f), fminf(y, 65504.f));
      }
    }
  }
}

int stem_make_plan(const __half* img_pad, int B, const __half* w_tap_major, const float* bias, __half* out, int OCtot, int oc_off,
                   StemParams* sp) {
  std::memset(sp, 0, sizeof(*sp));
  {
    cuuint64_t dims[4] = {8, 264, 262, (cuuint64_t)B};
    cuuint64_t strides[3] = {16, 264 * 16, (cuuint64_t)262 * 264 * 16};
    cuuint32_t box[4] = {8, 16, 22, 1};
    if (!encode_tmap_f16(&sp->tm_in, 4, img_pad, dims, strides, box, 1, CU_TENSOR_MAP_SWIZZLE_NONE)) return 2;
  }
  {
    cuuint64_t dims[3] = {64, 16, 7};
    cuuint64_t strides[2] = {128, 16 * 128};
    cuuint32_t box[3] = {64, 16, 7};
    if (!encode_tmap_f16(&sp->tm_w, 3, w_tap_major, dims, strides, box)) return 2;
  }
  sp->out = out;
  sp->bias = bias;
  sp->OCtot = OCtot;
  sp->oc_off = oc_off;
  sp->total_tiles = B * 16 * 32;
  return 0;
}

cudaError_t launch_stem(const StemParams& sp, cudaStream_t st) {
  static SmemConfigOnce once;
  constexpr int smem = kStemWBytes + kStemStages * kStemAStride + 1024;
  if (cudaError_t e = once.ensure(stem_umma_kernel, smem); e != cudaSuccess) return e;
  const int sms = device_sms();
  const int grid = sp.total_tiles < sms ? sp.total_tiles : sms;
  return launch_kernel_pdl(stem_umma_kernel, dim3(grid), dim3(kStemThreads), smem, st, sp);
}

}  // namespace ltb
