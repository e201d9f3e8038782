// Fused multi-head attention on Hopper wgmma (sm_90a): softmax(scale * Q K^T) V with the score matrix S living only in
// registers — replaces the three-kernel path (batched QK^T GEMM -> fp16 S in HBM -> softmax kernel -> batched PV GEMM)
// of the diffusers Attention blocks (UNet self / cross attention, avatars/musetalk/models/unet.py:29-48 -> diffusers
// BasicTransformerBlock) and the Whisper / HuBERT encoder layers (avatars/musetalk/whisper/audio2feature.py:106-117).
//
// One CTA = 128 queries of one (batch, head); each of the two consumer warpgroups owns 64 of them.  TWO passes over the keys
// instead of an online rescale of O:
//   pass 1: S_t = Q K_t^T (wgmma, M=64 queries per warpgroup, N=128 keys, K = head dim) in registers; every thread keeps the
//           running maximum m and the sum l = sum exp(scale*(s - m)) of its two query rows (merged over the four lanes of a row);
//   pass 2: S_t is recomputed (the head dim is 16..160: re-running 1..10 K steps is cheaper than keeping or rescaling
//           anything), P_t = exp(scale*(s - m)) / l is packed to fp16 straight into the A-operand register fragments of
//           O += P_t V_t (M=64, N = head dim, K=128 keys) — O accumulates in registers.
// Q / K tiles come by TMA straight out of the fused qkv (or q / kv) projection buffers (4-D maps (d, token, head, batch); the
// box is 64 channels wide and the tensor's channel extent is the head dim, so the padding up to 64 is zero-filled); V^T tiles from
// the [B*H][d][keys] buffer transpose_heads writes.  Roles (288 threads): warps 0-7 consumers, warp 8 TMA producer.
#include <cuda.h>

#include "conv_tma.h"
#include "ltb_internal.h"
#include "ops.h"
#include "ptx_sm90.cuh"

namespace ltb {

struct alignas(64) AttnParams {
  CUtensorMap tm_q;    // 4-D (d, nq, H, B), box (64, 128, 1, 1), SWIZZLE_128B
  CUtensorMap tm_k;    // 4-D (d, nk_rows, H, B), box (64, 128, 1, 1)
  CUtensorMap tm_vt;   // 3-D (n_pad, d, B*H), box (64, d, 1)
  __half* out;         // [B*nq][out_pitch], head h at columns [h*d, (h+1)*d)
  int out_pitch, nq, valid, d, H, kstages;
  float scale_log2e;   // scale * log2(e): probabilities are exp2((s - m) * scale_log2e)
};

constexpr int kAttnThreads = 288;
constexpr int kTileBytes = 128 * 128;   // 128 rows x 64 fp16

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int D>
__global__ void __launch_bounds__(kAttnThreads, 1) attn_fused_kernel(const __grid_constant__ AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t q_full, k_full[2], k_empty[2], v_full, v_empty;

  pdl_launch_dependents();   // the output projection (a PDL-launched conv kernel) may start its prologue under this kernel's tail
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.x * 128, bh = blockIdx.y, b = bh / p.H, h = bh - b * p.H;
  constexpr int chunks = (D + 63) / 64;               // 64-channel K chunks of the QK^T contraction
  const int nkt = (p.valid + 127) / 128;              // key tiles (keys >= valid are masked; rows beyond the tensor come back as zeros)
  const uint32_t KS = (uint32_t)p.kstages;            // K ring depth (1 when the head dim needs three chunks: shared memory)
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t q_smem = smem0;                                       // chunks x [128 x 128 B]
  const uint32_t k_smem = q_smem + chunks * kTileBytes;                // KS stages x chunks x [128 x 128 B]
  const uint32_t v_smem = k_smem + KS * chunks * kTileBytes;           // 2 key blocks x [d rows x 128 B]
  constexpr uint32_t v_blk = ((uint32_t)D * 128u + 1023u) & ~1023u;

  if (tid == 0) {
    mbar_init(smem_u32(&q_full), 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(smem_u32(&k_full[s]), 1);
      mbar_init(smem_u32(&k_empty[s]), 8);   // one arrival per consumer warp
    }
    mbar_init(smem_u32(&v_full), 1);
    mbar_init(smem_u32(&v_empty), 8);
    mbar_fence_init();
    tma_prefetch_desc(&p.tm_q);
    tma_prefetch_desc(&p.tm_k);
    tma_prefetch_desc(&p.tm_vt);
  }
  __syncthreads();

  if (warp == 8) {
    // =============================================================== TMA producer
    if (lane == 0) {
      mbar_arrive_expect_tx(smem_u32(&q_full), chunks * kTileBytes);
      for (int c = 0; c < chunks; ++c) tma_load_4d(q_smem + c * kTileBytes, &p.tm_q, smem_u32(&q_full), c * 64, q0, h, b);
      uint32_t ki = 0;
      for (int pass = 0; pass < 2; ++pass)
        for (int kt = 0; kt < nkt; ++kt, ++ki) {
          const uint32_t s = ki % KS;
          mbar_wait(smem_u32(&k_empty[s]), ((ki / KS) & 1u) ^ 1u);
          mbar_arrive_expect_tx(smem_u32(&k_full[s]), chunks * kTileBytes);
          for (int c = 0; c < chunks; ++c)
            tma_load_4d(k_smem + (s * chunks + c) * kTileBytes, &p.tm_k, smem_u32(&k_full[s]), c * 64, kt * 128, h, b);
          if (pass == 1) {
            mbar_wait(smem_u32(&v_empty), (kt & 1u) ^ 1u);
            mbar_arrive_expect_tx(smem_u32(&v_full), 2 * D * 128);
            for (int j = 0; j < 2; ++j) tma_load_3d(v_smem + j * v_blk, &p.tm_vt, smem_u32(&v_full), kt * 128 + j * 64, 0, bh);
          }
        }
    }
    return;
  }

  // =============================================================== consumers: warpgroup wg owns queries [64 wg, 64 wg + 64)
  const int wg = warp >> 2, wq = warp & 3;
  const int cq = 2 * (lane & 3);
  constexpr uint32_t kHi = wgmma_hi_128b(1024);   // SBO = 1024 B, SWIZZLE_128B
  constexpr int ksteps_last = ((D - 1) % 64) / 16 + 1;
  float s_acc[64];
  uint32_t ki = 0;
  // S = Q K^T of key tile kt into s_acc; hands the K stage back
  auto scores = [&]() {
    const uint32_t s = ki % KS;
    mbar_wait(smem_u32(&k_full[s]), (ki / KS) & 1u);
#pragma unroll
    for (int i = 0; i < 64; ++i) s_acc[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < chunks; ++c) {
      const uint32_t a_lo = wgmma_lo(q_smem + c * kTileBytes + wg * 64 * 128);
      const uint32_t b_lo = wgmma_lo(k_smem + (s * chunks + c) * kTileBytes);
      const int ks = (c == chunks - 1) ? ksteps_last : 4;
#pragma unroll
      for (int k = 0; k < ks; ++k) Wgmma<128>::ss(s_acc, wgmma_lohi(a_lo + k * 2, kHi), wgmma_lohi(b_lo + k * 2, kHi), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s_acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&k_empty[s]));
    ++ki;
  };
  mbar_wait(smem_u32(&q_full), 0);
  // ---- pass 1: running maximum and sum of the two rows (hh = 0, 1) of this thread
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  for (int kt = 0; kt < nkt; ++kt) {
    scores();
    const int lim = p.valid - kt * 128;   // key columns [0, lim) of this tile are real keys
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float tmax = -INFINITY;
#pragma unroll
      for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * i + cq + e < lim) tmax = fmaxf(tmax, s_acc[4 * i + 2 * hh + e]);
      tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
      tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 2));
      const float m_new = fmaxf(m[hh], tmax);   // finite: every tile holds at least one valid key
      float lsum = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * i + cq + e < lim) lsum += ex2f((s_acc[4 * i + 2 * hh + e] - m_new) * p.scale_log2e);
      lsum += __shfl_xor_sync(0xffffffffu, lsum, 1);
      lsum += __shfl_xor_sync(0xffffffffu, lsum, 2);
      l[hh] = l[hh] * ex2f((m[hh] - m_new) * p.scale_log2e) + lsum;   // m = -inf on the first tile: ex2(-inf) = 0
      m[hh] = m_new;
    }
  }
  const float inv_l[2] = {1.f / l[0], 1.f / l[1]};
  // ---- pass 2: probabilities (fp16 A fragments in registers) times V
  float o_acc[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o_acc[i] = 0.f;
  for (int kt = 0; kt < nkt; ++kt) {
    scores();
    const int lim = p.valid - kt * 128;
    uint32_t pf[32];   // 8 K steps x 4 registers: fragment of rows (l/4, l/4 + 8) x keys (16 kk + 2(l%4) (+8))
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int col = 8 * i + cq;
        const float a = (col < lim) ? ex2f((s_acc[4 * i + 2 * hh] - m[hh]) * p.scale_log2e) * inv_l[hh] : 0.f;
        const float c = (col + 1 < lim) ? ex2f((s_acc[4 * i + 2 * hh + 1] - m[hh]) * p.scale_log2e) * inv_l[hh] : 0.f;
        // key block i = 2 kk + half: register 4 kk + 2 half + hh
        pf[4 * (i >> 1) + 2 * (i & 1) + hh] = f32x2_to_f16x2_sat(a, c);
      }
    mbar_wait(smem_u32(&v_full), kt & 1u);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint32_t b_lo = wgmma_lo(v_smem + (kk >> 2) * v_blk + (kk & 3) * 32);
      Wgmma<D>::rs(o_acc, *reinterpret_cast<const uint32_t(*)[4]>(&pf[4 * kk]), wgmma_lohi(b_lo, kHi), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o_acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&v_empty));
  }
  // ---- epilogue: O (fp32 registers) -> fp16 rows of the output
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int qi = q0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * hh;
    if (qi >= p.nq) continue;
    __half* orow = p.out + ((size_t)b * p.nq + qi) * p.out_pitch + h * D;
#pragma unroll
    for (int i = 0; i < D / 8; ++i)
      *reinterpret_cast<uint32_t*>(orow + 8 * i + cq) = f32x2_to_f16x2_sat(o_acc[4 * i + 2 * hh], o_acc[4 * i + 2 * hh + 1]);
  }
}

// ------------------------------------------------------------------------------------------------ host side
bool attn_fused_supported(int d, int q_pitch, int kv_pitch, int n_pad) {
  return d >= 16 && d <= 160 && d % 16 == 0 && q_pitch % 8 == 0 && kv_pitch % 8 == 0 && n_pad % 8 == 0 && tma_encode_available();
}

// q: [B][nq] rows of q_pitch elements, head h at columns [h*d, (h+1)*d); k: [B][kv_rows] rows of kv_pitch elements, same head layout;
// vt: [B*H][d][n_pad] (transpose_heads: zero for key >= kv_rows); keys [valid, ..) get probability 0.
cudaError_t launch_attn_fused(const __half* q, int q_pitch, const __half* k, int kv_pitch, int kv_rows, const __half* vt, int n_pad, int B, int H,
                              int nq, int valid, int d, float scale, __half* out, int out_pitch, cudaStream_t st) {
  if (!attn_fused_supported(d, q_pitch, kv_pitch, n_pad) || nq < 1 || valid < 1 || valid > kv_rows || valid > n_pad || out_pitch % 8)
    return cudaErrorInvalidValue;
  const int nk = kv_rows;
  AttnParams p;
  {
    cuuint64_t dims[4] = {(cuuint64_t)d, (cuuint64_t)nq, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)q_pitch * 2, (cuuint64_t)d * 2, (cuuint64_t)nq * q_pitch * 2};
    cuuint32_t box[4] = {64, 128, 1, 1};
    if (!encode_tmap_f16(&p.tm_q, 4, q, dims, strides, box)) return cudaErrorInvalidValue;
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)d, (cuuint64_t)nk, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)kv_pitch * 2, (cuuint64_t)d * 2, (cuuint64_t)nk * kv_pitch * 2};
    cuuint32_t box[4] = {64, 128, 1, 1};
    if (!encode_tmap_f16(&p.tm_k, 4, k, dims, strides, box)) return cudaErrorInvalidValue;
  }
  {
    cuuint64_t dims[3] = {(cuuint64_t)n_pad, (cuuint64_t)d, (cuuint64_t)B * H};
    cuuint64_t strides[2] = {(cuuint64_t)n_pad * 2, (cuuint64_t)d * n_pad * 2};
    cuuint32_t box[3] = {64, (cuuint32_t)d, 1};
    if (!encode_tmap_f16(&p.tm_vt, 3, vt, dims, strides, box)) return cudaErrorInvalidValue;
  }
  p.out = out;
  p.out_pitch = out_pitch;
  p.nq = nq;
  p.valid = valid;
  p.d = d;
  p.H = H;
  p.scale_log2e = scale * 1.4426950408889634f;
  const int chunks = (d + 63) / 64;
  const int v_blk = (d * 128 + 1023) & ~1023;
  p.kstages = chunks <= 2 ? 2 : 1;
  const int smem = (1 + p.kstages) * chunks * kTileBytes + 2 * v_blk + 1024;
  constexpr int kMaxSmem = 200 * 1024;
  if (smem > kMaxSmem) return cudaErrorInvalidValue;
  const dim3 grid((nq + 127) / 128, B * H);
  switch (d) {
#define LTB_ATTN_CASE(DD)                                                            \
  case DD: {                                                                          \
    static SmemConfigOnce once;                                                       \
    if (cudaError_t e = once.ensure(attn_fused_kernel<DD>, kMaxSmem); e != cudaSuccess) return e; \
    attn_fused_kernel<DD><<<grid, kAttnThreads, smem, st>>>(p);                       \
    break;                                                                            \
  }
    LTB_ATTN_CASE(16) LTB_ATTN_CASE(32) LTB_ATTN_CASE(48) LTB_ATTN_CASE(64) LTB_ATTN_CASE(80)
    LTB_ATTN_CASE(96) LTB_ATTN_CASE(112) LTB_ATTN_CASE(128) LTB_ATTN_CASE(144) LTB_ATTN_CASE(160)
#undef LTB_ATTN_CASE
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace ltb
