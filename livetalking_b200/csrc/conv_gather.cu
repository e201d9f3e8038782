// Generic implicit-GEMM convolution on Hopper tensor cores (sm_90a wgmma).
//
//   A (im2col rows, 128 output pixels x KB channels of one tap) : gathered with cp.async (zero-fill = padding)
//                                                                 into the canonical K-major swizzled smem layout
//   B (weights, BN x KB)                                         : cp.async, same layout
//   D (128 x BN fp32)                                            : registers of two warpgroups (64 rows each), wgmma
//   epilogue                                                     : +bias (+residual) -> ReLU -> fp16 NHWC, written straight
//                                                                  into a channel slice of the destination (concat-free skips)
//
// This kernel handles EVERY conv geometry of the hot path (any stride / padding / kernel size, ConvTranspose
// sub-pixel phases, channel-sliced inputs/outputs).  conv_halo.cu is the TMA-fed fast path for the FLOP-heavy
// stride-1 layers.  Reference op being replaced: avatars/wav2lip/models/conv.py:5-19,33-44 (cuDNN conv + BN + add + ReLU).
#include "conv_params.h"
#include "ltb_internal.h"
#include "ptx_sm90.cuh"

namespace ltb {

constexpr int kGatherThreads = 256;   // two warpgroups: every thread gathers, each warpgroup owns 64 output rows

template <int BN, int KB>
struct GatherCfg {
  static constexpr int CH = KB / 8;                 // 16-byte chunks per smem row
  static constexpr int ROWB = KB * 2;               // bytes per smem row (= swizzle span)
  static constexpr int RSTEP = kGatherThreads / CH; // row step between the rows one thread fills
  static constexpr int RPT = 128 / RSTEP;           // rows per thread
  static constexpr int A_BYTES = 128 * ROWB;
  static constexpr int B_BYTES = (BN * ROWB < 1024) ? 1024 : BN * ROWB;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (STAGE_BYTES >= 32768) ? 3 : 4;
  static constexpr uint32_t LAYOUT = (KB == 64) ? 1u : (KB == 32) ? 2u : 3u;
  static constexpr uint32_t SBO = 8 * ROWB;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;
};

template <int KB>
__device__ __forceinline__ uint32_t swz_chunk(int row, int j) {
  if (KB == 64) return (uint32_t)(j ^ (row & 7));
  if (KB == 32) return (uint32_t)(j ^ ((row >> 1) & 3));
  return (uint32_t)(j ^ ((row >> 2) & 1));
}

// GRP: grouped weights (ConvParams::group_slot).  A CTA's 128 rows share one weight tile, so M-tiles are enumerated per group
// (blockIdx.x = group * tiles per group + tile) and rows past the group's end are neither gathered nor written.
template <int BN, int KB, bool GRP>
__global__ void __launch_bounds__(kGatherThreads) conv_gather_wgmma_kernel(const __grid_constant__ ConvParams p) {
  using C = GatherCfg<BN, KB>;
  extern __shared__ uint8_t smem_raw[];
  const int tid = threadIdx.x;
  const int wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const uint32_t tiles = (smem_u32(smem_raw) + 1023u) & ~1023u;

  const int zphase = (p.ksplit > 1) ? 0 : ((p.zbatch > 1) ? (int)(blockIdx.z % p.nphases) : (int)blockIdx.z);
  const ConvPhase& ph = p.ph[zphase];
  const __half* in_base = p.in;
  const __half* w_base = p.w;
  __half* out_base = p.out;
  if (p.zbatch > 1) {
    const int zb = blockIdx.z / p.nphases;
    const int zo = zb / p.zdiv, zi = zb - zo * p.zdiv;
    in_base += zo * p.in_zo + zi * p.in_zi;
    w_base += zo * p.w_zo + zi * p.w_zi;
    out_base += zo * p.out_zo + zi * p.out_zi;
  }
  const int g_rows = GRP ? p.group_images * p.GH * p.GW : 0, g_tiles = (g_rows + 127) / 128;
  const int group = GRP ? (int)blockIdx.x / g_tiles : 0;
  const int m0 = GRP ? group * g_rows + ((int)blockIdx.x - group * g_tiles) * 128 : blockIdx.x * 128;
  const int n0 = blockIdx.y * BN;
  const int cpt = p.Cin / KB;  // K chunks per tap
  int it_begin = 0, kiters = ph.ntaps * cpt;
  if (p.ksplit > 1) {  // split-K: this CTA owns K iterations [it_begin, it_begin + kiters)
    const int per = (kiters + p.ksplit - 1) / p.ksplit;
    it_begin = (int)blockIdx.z * per;
    kiters = min(per, kiters - it_begin);
  }
  // PDL: everything below touches activations
  pdl_launch_dependents();
  pdl_wait();
  const float* bias_g = nullptr;
  if constexpr (GRP) {   // the slot table is written by the stream before this kernel: read it after the wait
    const int slot = p.group_slot[group];
    w_base += slot * p.w_slot_stride;
    bias_g = p.bias + slot * p.bias_slot_stride;
  }
  // the ungrouped instantiation reads the parameters directly (same code as before grouping existed)
  const float* const bias = GRP ? bias_g : p.bias;
  const int M = GRP ? (group + 1) * g_rows : p.M;

  // per gathered row: input coordinates of tap (0,0) and the element offset of that pixel (+ this thread's 16-byte K chunk);
  // per K iteration only one uniform tap offset is added
  const int j = tid % C::CH;
  const int r0 = tid / C::CH;
  int riy[C::RPT], rix[C::RPT];
  long long rbase[C::RPT];
  const int gsz = p.GH * p.GW;
#pragma unroll
  for (int i = 0; i < C::RPT; ++i) {
    const int m = m0 + r0 + i * C::RSTEP;
    if (m < M) {
      const int b = m / gsz;
      const int rem = m - b * gsz;
      const int gy = rem / p.GW;
      const int gx = rem - gy * p.GW;
      riy[i] = gy * p.sy;
      rix[i] = gx * p.sx;
      rbase[i] = ((long long)(b * p.IH + riy[i]) * p.IW + rix[i]) * p.ICtot + p.ic_off + j * 8;
    } else {
      riy[i] = -(1 << 20);  // forces the bounds test to fail -> zero rows
      rix[i] = 0;
      rbase[i] = 0;
    }
  }
  auto load = [&](int it) {
    const int kk = it_begin + it;
    const int tap = kk / cpt, cc = kk - tap * cpt;
    const uint32_t a_base = tiles + (it % C::STAGES) * C::STAGE_BYTES;
    const uint32_t b_base = a_base + C::A_BYTES;
    const int dy = ph.dy[tap], dx = ph.dx[tap];
    const long long toff = (long long)(dy * p.IW + dx) * p.ICtot + cc * KB;   // uniform over the CTA
#pragma unroll
    for (int i = 0; i < C::RPT; ++i) {
      const int row = r0 + i * C::RSTEP;
      const int iy = riy[i] + dy, ix = rix[i] + dx;
      const bool inb = ((unsigned)iy < (unsigned)p.IH) && ((unsigned)ix < (unsigned)p.IW);
      const __half* src = inb ? (in_base + rbase[i] + toff) : in_base;
      cp_async16(a_base + row * C::ROWB + swz_chunk<KB>(row, j) * 16, src, inb ? 16u : 0u);
    }
    const size_t wk = (size_t)ph.koff + (size_t)tap * p.Cin + cc * KB + j * 8;
#pragma unroll
    for (int i = 0; i < C::RPT; ++i) {
      const int n = r0 + i * C::RSTEP;
      if (n < BN) cp_async16(b_base + n * C::ROWB + swz_chunk<KB>(n, j) * 16, w_base + (size_t)(n0 + n) * p.Ktot + wk, 16u);
    }
  };

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
#pragma unroll
  for (int s = 0; s < C::STAGES - 1; ++s) {
    if (s < kiters) load(s);
    cp_async_commit();
  }
  for (int it = 0; it < kiters; ++it) {
    cp_async_wait<C::STAGES - 2>();
    fence_proxy_async_smem();   // cp.async (generic proxy) writes -> wgmma operand reads (async proxy)
    __syncthreads();            // stage it is complete for every thread; every wgmma of iteration it-1 has retired
    if (it + C::STAGES - 1 < kiters) load(it + C::STAGES - 1);
    cp_async_commit();
    const uint32_t a_base = tiles + (it % C::STAGES) * C::STAGE_BYTES;
    const uint32_t b_base = a_base + C::A_BYTES;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KB / 16; ++k) {
      const uint64_t ad = wgmma_desc(a_base + wg * 64 * C::ROWB + k * 32, 16, C::SBO, C::LAYOUT);
      const uint64_t bd = wgmma_desc(b_base + k * 32, 16, C::SBO, C::LAYOUT);
      Wgmma<BN>::ss(acc, ad, bd, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
  }
  cp_async_wait<0>();

  // ------------------------------------------------------------------ epilogue straight from the accumulator fragments
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int m = m0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * hh;
    if (m >= M) continue;
    if (p.ksplit > 1) {
      // split-K: this CTA's fp32 partial goes to its own slice ws[split][m][co] (plain stores, no atomics)
      float* wrow = p.ws + ((size_t)blockIdx.z * p.M + m) * p.Cout + n0;
#pragma unroll
      for (int i = 0; i < BN / 8; ++i)
        *reinterpret_cast<float2*>(wrow + 8 * i + cq) = make_float2(acc[4 * i + 2 * hh], acc[4 * i + 2 * hh + 1]);
      continue;
    }
    const int b = m / gsz;
    const int rem = m - b * gsz;
    const int gy = rem / p.GW;
    const int gx = rem - gy * p.GW;
    const size_t opix = (size_t)(b * p.OH + gy * p.osy + ph.ooy) * p.OW + gx * p.osx + ph.oox;
    __half* optr = out_base + opix * p.OCtot + p.oc_off + n0;
    const __half* rptr = p.res ? (p.res + opix * p.RCtot + p.rc_off + n0) : nullptr;
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const int c = 8 * i + cq;
      const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + n0 + c));
      float x = acc[4 * i + 2 * hh] + bb.x, y = acc[4 * i + 2 * hh + 1] + bb.y;
      if (rptr) {
        const float2 rf = __half22float2(__ldcg(reinterpret_cast<const __half2*>(rptr + c)));
        x += rf.x;
        y += rf.y;
      }
      if (p.relu) {
        x = fmaxf(x, 0.f);
        y = fmaxf(y, 0.f);
      }
      x = fminf(fmaxf(x, -65504.f), 65504.f);
      y = fminf(fmaxf(y, -65504.f), 65504.f);
      *reinterpret_cast<__half2*>(optr + c) = __floats2half2_rn(x, y);
    }
  }
}

template <int BN, int KB, bool GRP>
static cudaError_t launch_grp(const ConvParams& p, cudaStream_t st) {
  using C = GatherCfg<BN, KB>;
  static SmemConfigOnce once;
  if (cudaError_t e = once.ensure(conv_gather_wgmma_kernel<BN, KB, GRP>, C::SMEM_BYTES); e != cudaSuccess) return e;
  const int mt = GRP ? (p.N / p.group_images) * ((p.group_images * p.GH * p.GW + 127) / 128) : (p.M + 127) / 128;
  dim3 grid(mt, p.Cout / BN, p.ksplit > 1 ? p.ksplit : p.nphases * (p.zbatch > 1 ? p.zbatch : 1));
  return launch_kernel_pdl(conv_gather_wgmma_kernel<BN, KB, GRP>, grid, dim3(kGatherThreads), C::SMEM_BYTES, st, p);
}

template <int BN, int KB>
static cudaError_t launch_one(const ConvParams& p, cudaStream_t st) {
  return p.group_slot ? launch_grp<BN, KB, true>(p, st) : launch_grp<BN, KB, false>(p, st);
}

template <int KB>
static cudaError_t launch_kb(const ConvParams& p, int bn, cudaStream_t st) {
  switch (bn) {
    case 128: return launch_one<128, KB>(p, st);
    case 64: return launch_one<64, KB>(p, st);
    case 32: return launch_one<32, KB>(p, st);
    case 16: return launch_one<16, KB>(p, st);
  }
  return cudaErrorInvalidValue;
}

static int conv_gather_pick_bn(const ConvParams& p) {
  int bn = 0;
  for (int c : {128, 64, 32, 16})
    if (p.Cout % c == 0) {
      bn = c;
      break;
    }
  if (!bn) return 0;
  // small-M layers are weight-bandwidth bound: prefer more, narrower CTAs until the grid fills the SMs
  const long mt = (p.M + 127) / 128;
  const long zb = p.zbatch > 1 ? p.zbatch : 1;
  while (bn > 32 && mt * (p.Cout / bn) * p.nphases * zb < 132) bn >>= 1;
  return bn;
}

// out[m, co] = act(sum_s ws[s][m][co] + bias[co] (+ res))
__global__ void __launch_bounds__(256) splitk_finalize_kernel(const float* __restrict__ ws, int ksplit, int M, int Cout,
                                                              const float* __restrict__ bias, const __half* __restrict__ res, int RCtot,
                                                              int rc_off, int relu, __half* __restrict__ out, int OCtot, int oc_off) {
  const unsigned vpr = Cout / 8;
  const unsigned total = (unsigned)M * vpr;
  const size_t slice = (size_t)M * Cout;
  pdl_launch_dependents();
  pdl_wait();   // the partial sums (and the residual) come from the predecessor kernels: coherent loads below, never .nc
  for (unsigned i = blockIdx.x * 256u + threadIdx.x; i < total; i += gridDim.x * 256u) {
    const size_t m = i / vpr;
    const int c = (int)(i % vpr) * 8;
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = __ldg(bias + c + j);
    for (int s = 0; s < ksplit; ++s) {
      const float4* w4 = reinterpret_cast<const float4*>(ws + s * slice + m * Cout + c);
      const float4 a = __ldcg(w4), b = __ldcg(w4 + 1);
      f[0] += a.x; f[1] += a.y; f[2] += a.z; f[3] += a.w;
      f[4] += b.x; f[5] += b.y; f[6] += b.z; f[7] += b.w;
    }
    if (res) {
      const uint4 rv = __ldcg(reinterpret_cast<const uint4*>(res + m * RCtot + rc_off + c));
      const __half* rh = reinterpret_cast<const __half*>(&rv);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] += __half2float(rh[j]);
    }
    uint4 ov;
    __half* oh = reinterpret_cast<__half*>(&ov);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float x = relu ? fmaxf(f[j], 0.f) : f[j];
      oh[j] = __float2half_rn(fminf(fmaxf(x, -65504.f), 65504.f));
    }
    *reinterpret_cast<uint4*>(out + m * OCtot + oc_off + c) = ov;
  }
}

bool conv_gather_pick(const ConvParams& p, bool have_ws, size_t splitk_ws_floats, int* bn_out, int* kb_out, int* ksplit_out) {
  if (p.Cout % 16 != 0 || p.Cin % 16 != 0 || (p.ICtot % 8) || (p.OCtot % 8) || (p.ic_off % 8) || (p.oc_off % 8) ||
      (p.Ktot % 8) || p.nphases < 1 || p.nphases > kMaxPhases)
    return false;
  if (p.res && ((p.RCtot % 8) || (p.rc_off % 8))) return false;
  int bn = conv_gather_pick_bn(p);
  if (!bn) return false;
  const int kb = (p.Cin % 64 == 0) ? 64 : (p.Cin % 32 == 0) ? 32 : 16;
  // split-K for small-M, deep-K layers (1x1..8x8 maps with 512..2560 channels): they are weight-streaming bound and a
  // handful of CTAs walking thousands of K blocks serially is latency-bound.
  int ksplit = 0;
  const int kiters = p.ph[0].ntaps * (p.Cin / kb);
  const long mt = (p.M + 127) / 128;
  if (have_ws && !p.group_slot && p.nphases == 1 && p.zbatch <= 1 && p.osy == 1 && p.osx == 1 && p.GH == p.OH && p.GW == p.OW && kiters >= 32 && mt <= 8) {
    int bn2 = 0;
    for (int c : {128, 64, 32, 16})
      if (p.Cout % c == 0) {
        bn2 = c;
        break;
      }
    const long tiles = mt * (p.Cout / bn2);
    if (tiles < 64) {
      int ks = (int)((264 + tiles - 1) / tiles);   // two CTAs per SM
      if (ks > kiters / 8) ks = kiters / 8;   // >= 8 K blocks per split
      if (ks > 32) ks = 32;
      while (ks >= 2 && (size_t)ks * p.M * p.Cout > splitk_ws_floats) --ks;
      if (ks >= 2) {
        const int per = (kiters + ks - 1) / ks;
        ksplit = (kiters + per - 1) / per;  // no empty splits
        bn = bn2;
      }
    }
  }
  *bn_out = bn;
  *kb_out = kb;
  *ksplit_out = ksplit;
  return true;
}

cudaError_t launch_conv_gather(const ConvParams& p_in, cudaStream_t st, float* splitk_ws, size_t splitk_ws_floats) {
  ConvParams p = p_in;
  int bn, kb;
  if (!conv_gather_pick(p, splitk_ws != nullptr, splitk_ws_floats, &bn, &kb, &p.ksplit)) return cudaErrorInvalidValue;
  p.ws = p.ksplit > 1 ? splitk_ws : nullptr;
  cudaError_t e;
  if (kb == 64) e = launch_kb<64>(p, bn, st);
  else if (kb == 32) e = launch_kb<32>(p, bn, st);
  else e = launch_kb<16>(p, bn, st);
  if (e != cudaSuccess || p.ksplit <= 1) return e;
  const size_t total = (size_t)p.M * (p.Cout / 8);
  int blocks = (int)((total + 255) / 256);
  if (blocks > 592) blocks = 592;
  return launch_kernel_pdl(splitk_finalize_kernel, dim3(blocks), dim3(256), 0, st, (const float*)p.ws, p.ksplit, p.M, p.Cout, p.bias, p.res,
                           p.RCtot, p.rc_off, p.relu, p.out, p.OCtot, p.oc_off);
}

}  // namespace ltb
