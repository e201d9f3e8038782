// Split-K conv for the wav2lip256 bottleneck: 512 - 1024 channel layers on 8x8, 4x4 and 1x1 grids (the engine routes L29 - L36).
//
// On these maps a 16 x 8 pixel halo tile holds one image and is mostly padding, and every image's tile streams the whole weight
// set from L2; the gather kernel walks thousands of K blocks on a few CTAs.  Here the operands swap roles, as in the ping-pong
// kernel:
//   A (wgmma M): 128 output channels per CTA, one m64 block per consumer warpgroup, TMA-loaded from the layer's K-major weight
//                rows [Cout][Ktot] (a 64-wide K box at the tap's column; ConvT phases start at their koff).
//   B (wgmma N): the pixels of `bimg` whole images (np = 256 on 8x8 grids, 64 on 4x4, 16 on 1x1): one 4-D TMA box (64 channels,
//                W, H, images) at the tap's shifted origin per K step.  TMA zero-fills the padding and images >= N; stride-2
//                convs use a traversal stride of 2.  Each pixel is one 128-byte SWIZZLE_128B row, the halo kernel's layout.
//   So each weight byte is read from L2 once per tile of np pixels instead of once per image.
// Split-K: the `ksplit` CTAs of one (channel block, pixel tile, phase) form a thread-block cluster; CTA z accumulates K steps
// [z per, (z + 1) per) of the phase.  After the loop every CTA parks its fp32 accumulators in its own shared memory, and CTA r
// of the cluster sums slice r of the tile over the ksplit CTAs in rank order through distributed shared memory (fixed order:
// deterministic, no atomics, no global workspace), adds the bias and the residual in fp32 and rounds once to fp16 (the gather
// kernel's split-K arithmetic), and stores into the output channel slice; ConvT phases scatter to (2y + a, 2x + b).
// Roles (288 threads): warpgroups 0 and 1 consume (MMAs), warp 8 is the TMA producer; all nine warps reduce.
#include <cuda.h>

#include <cstring>

#include "conv_smallmap.h"
#include "conv_tma.h"
#include "ltb_internal.h"
#include "ptx_sm90.cuh"

namespace ltb {

namespace {

constexpr int kThreads = 288;
constexpr int kStages = 4;
constexpr int kABytes = 128 * 128;   // 128 output channels x 64 input channels
constexpr int kMaxSplit = 8;         // portable cluster size

template <int NP>
struct SmCfg {
  static constexpr int B_BYTES = NP * 128;
  static constexpr int STAGE = kABytes + B_BYTES;
  static constexpr int RED = 256 * (NP / 2) * 4;   // fp32 accumulators of both consumer warpgroups
  static constexpr int SMEM = (kStages * STAGE > RED ? kStages * STAGE : RED) + 1024;
  static_assert(SMEM <= 227 * 1024, "shared memory overflow");
};

}  // namespace

template <int NP>
__global__ void __launch_bounds__(kThreads, 1) conv_smallmap_kernel(const __grid_constant__ SmallmapParams p) {
  using C = SmCfg<NP>;
  constexpr int NACC = NP / 2;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full[kStages], empty[kStages];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;

  const int cot = blockIdx.x;
  const int ptile = (int)blockIdx.y % p.ptiles, phase = (int)blockIdx.y / p.ptiles;
  const uint32_t split = cluster_ctarank();
  const ConvPhase& ph = p.ph[phase];
  const int cpt = p.Cin / 64;
  const int total = ph.ntaps * cpt;
  const int per = (total + p.ksplit - 1) / p.ksplit;
  const int it0 = (int)split * per;
  const int kiters = max(0, min(per, total - it0));
  const int co0 = cot * 128, img0 = ptile * p.bimg;

  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(smem_u32(&full[s]), 1);
      mbar_init(smem_u32(&empty[s]), 8);   // one arrival per consumer warp
    }
    mbar_fence_init();
    tma_prefetch_desc(&p.tm_in);
    tma_prefetch_desc(&p.tm_w);
  }
  __syncthreads();
  pdl_launch_dependents();

  if (warp == 8) {
    // =============================================================== TMA producer
    if (lane == 0) {
      auto load_a = [&](int it) {
        const int kk = it0 + it, tap = kk / cpt, cc = kk - tap * cpt;
        const uint32_t st = it % kStages;
        mbar_arrive_expect_tx(smem_u32(&full[st]), C::STAGE);
        tma_load_2d(smem0 + st * C::STAGE, &p.tm_w, smem_u32(&full[st]), ph.koff + tap * p.Cin + cc * 64, co0);
      };
      auto load_b = [&](int it) {
        const int kk = it0 + it, tap = kk / cpt, cc = kk - tap * cpt;
        const uint32_t st = it % kStages;
        tma_load_4d(smem0 + st * C::STAGE + kABytes, &p.tm_in, smem_u32(&full[st]), cc * 64, ph.dx[tap], ph.dy[tap], img0);
      };
      // the weights are constants: the first stages' weight boxes load before this kernel waits for its predecessor
      const int pre = min(kiters, kStages);
      for (int it = 0; it < pre; ++it) load_a(it);
      pdl_wait();
      for (int it = 0; it < pre; ++it) load_b(it);
      for (int it = kStages; it < kiters; ++it) {
        mbar_wait(smem_u32(&empty[it % kStages]), ((it / kStages) & 1u) ^ 1u);
        load_a(it);
        load_b(it);
      }
    } else {
      pdl_wait();
    }
  } else {
    pdl_wait();
  }

  float acc[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
  if (warp < 8) {
    // =============================================================== consumers: warpgroup wg owns channels co0 + 64 wg ..
    const int wg = warp >> 2;
    constexpr uint32_t kHi = wgmma_hi_128b(1024);   // 8-row groups of 128-byte rows
    for (int it = 0; it < kiters; ++it) {
      const uint32_t st = it % kStages;
      mbar_wait(smem_u32(&full[st]), (it / kStages) & 1u);
      const uint32_t a_lo = wgmma_lo(smem0 + st * C::STAGE + wg * 64 * 128);
      const uint32_t b_lo = wgmma_lo(smem0 + st * C::STAGE + kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) Wgmma<NP>::ss(acc, wgmma_lohi(a_lo + k * 2, kHi), wgmma_lohi(b_lo + k * 2, kHi), 1u);
      wgmma_commit();
      wgmma_wait<1>();   // the previous step's MMAs have read their stage
      if (it > 0 && lane == 0) mbar_arrive(smem_u32(&empty[(it - 1) % kStages]));
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    named_sync(1, 256);   // both warpgroups' MMAs have retired: the stages may be overwritten
    // park the accumulators in fragment order: floats 4q .. 4q + 3 of consumer thread t at red[q * 256 + t]
    float4* red = reinterpret_cast<float4*>(smem_raw + (smem0 - smem_u32(smem_raw)));
#pragma unroll
    for (int q = 0; q < NACC / 4; ++q) red[q * 256 + tid] = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
  }
  cluster_sync();

  // =============================================================== reduction of slice `split` over the cluster, epilogue
  {
    const int E = 64 * NACC, S = p.ksplit;   // float4 entries of the tile
    const int e0 = (int)split * (E / S), e1 = e0 + E / S;
    const int gsz = p.GH * p.GW;
    for (int e = e0 + tid; e < e1; e += kThreads) {
      // all ksplit loads in flight at once, then the sum in rank order
      float4 part[kMaxSplit];
#pragma unroll
      for (int s = 0; s < kMaxSplit; ++s)
        if (s < S) part[s] = dsmem_ld_f32x4(dsmem_map(smem0 + e * 16, (uint32_t)s));
      float4 v = part[0];
#pragma unroll
      for (int s = 1; s < kMaxSplit; ++s)
        if (s < S) {
          v.x += part[s].x;
          v.y += part[s].y;
          v.z += part[s].z;
          v.w += part[s].w;
        }
      const float vv[4] = {v.x, v.y, v.z, v.w};
      const int t = e & 255, q = e >> 8;
      const int wg = t >> 7, wq = (t >> 5) & 3, ln = t & 31;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int c = co0 + 64 * wg + 16 * wq + (ln >> 2) + 8 * (jj >> 1);
        const int n = 8 * q + 2 * (ln & 3) + (jj & 1);
        const int img = img0 + n / gsz, rem = n - (n / gsz) * gsz;
        if (img >= p.N) continue;
        const int gy = rem / p.GW, gx = rem - gy * p.GW;
        const size_t opix = ((size_t)img * p.OH + gy * p.osy + ph.ooy) * p.OW + gx * p.osx + ph.oox;
        float x = vv[jj] + __ldg(p.bias + c);
        if (p.res) x += __half2float(p.res[opix * p.RCtot + p.rc_off + c]);
        if (p.relu) x = fmaxf(x, 0.f);
        x = fminf(fmaxf(x, -65504.f), 65504.f);
        p.out[opix * p.OCtot + p.oc_off + c] = __float2half_rn(x);
      }
    }
  }
  cluster_sync();   // no CTA leaves while another still reads its shared memory
}

static int pick_np(const ConvParams& p) {
  const int g = p.GH * p.GW;
  return (p.GH == 8 && p.GW == 8) ? 256 : (p.GH == 4 && p.GW == 4) ? 64 : g == 1 ? 16 : 0;
}

bool conv_smallmap_supported(const ConvParams& p) {
  if (!p.smallmap || p.zbatch > 1 || p.group_slot || p.upconv) return false;
  if (!pick_np(p)) return false;
  const bool tr = p.nphases == 4 && p.osy == 2 && p.osx == 2 && p.sy == 1 && p.sx == 1 && p.IH == p.GH && p.IW == p.GW &&
                  p.OH == 2 * p.GH && p.OW == 2 * p.GW;
  const bool dense = p.nphases == 1 && p.osy == 1 && p.osx == 1 && p.OH == p.GH && p.OW == p.GW && p.sy == p.sx &&
                     (p.sy == 1 || (p.sy == 2 && p.GW > 1 && p.GH > 1));
  if (!tr && !dense) return false;
  if (p.Cin % 64 || p.Cout % 128) return false;
  // TMA: 16-byte aligned slice starts, pixel pitches and weight rows / tap columns
  if ((p.ICtot % 8) || (p.ic_off % 8) || (p.Ktot % 8) || (reinterpret_cast<uintptr_t>(p.in) % 16) ||
      (reinterpret_cast<uintptr_t>(p.w) % 16))
    return false;
  for (int i = 0; i < p.nphases; ++i)
    if (p.ph[i].koff % 8 || p.ph[i].ntaps < 1) return false;
  return ab_switch_on("LTB_CONV_SMALLMAP");   // 0 keeps these layers on the halo / gather kernels
}

int conv_smallmap_make_plan(const ConvParams& p, SmallmapParams* out) {
  if (!conv_smallmap_supported(p)) return 1;
  std::memset(out, 0, sizeof(*out));
  const int np = pick_np(p);
  out->np = np;
  out->bimg = np / (p.GH * p.GW);
  out->ptiles = (p.N + out->bimg - 1) / out->bimg;
  out->cotiles = p.Cout / 128;
  out->nphases = p.nphases;
  // split-K: the fewest splits (a power of two, at most a portable cluster of 8) that give >= 128 CTAs and at most 12 K steps
  // of the longest phase per CTA, with at least 128 K elements per split of the shortest phase
  int kmin = 1 << 30, kmax = 0;
  for (int i = 0; i < p.nphases; ++i) {
    kmin = kmin < p.ph[i].ntaps * p.Cin ? kmin : p.ph[i].ntaps * p.Cin;
    kmax = kmax > p.ph[i].ntaps * p.Cin ? kmax : p.ph[i].ntaps * p.Cin;
  }
  const long tiles = (long)out->cotiles * out->ptiles * p.nphases;
  int ks = 1;
  while (ks < kMaxSplit && 2 * ks * 128 <= kmin && (tiles * ks < 128 || (kmax / 64 + ks - 1) / ks > 12)) ks *= 2;
  out->ksplit = ks;
  {
    const int sx = p.nphases == 1 ? p.sx : 1;
    const cuuint32_t box[4] = {64, (cuuint32_t)((p.GW - 1) * sx + 1), (cuuint32_t)((p.GH - 1) * sx + 1), (cuuint32_t)out->bimg};
    if (!encode_nhwc_f16(&out->tm_in, p.in + p.ic_off, p.Cin, p.IW, p.IH, p.N, p.ICtot, box, sx)) return 2;
  }
  {
    const cuuint64_t dims[2] = {(cuuint64_t)p.Ktot, (cuuint64_t)p.Cout};
    const cuuint64_t strides[1] = {(cuuint64_t)p.Ktot * 2};
    const cuuint32_t box[2] = {64, 128};
    if (!encode_tmap_f16(&out->tm_w, 2, p.w, dims, strides, box)) return 2;
  }
  out->out = p.out;
  out->res = p.res;
  out->bias = p.bias;
  out->N = p.N;
  out->OH = p.OH;
  out->OW = p.OW;
  out->OCtot = p.OCtot;
  out->oc_off = p.oc_off;
  out->RCtot = p.RCtot;
  out->rc_off = p.rc_off;
  out->relu = p.relu;
  out->GH = p.GH;
  out->GW = p.GW;
  out->osy = p.osy;
  out->osx = p.osx;
  out->Cin = p.Cin;
  for (int i = 0; i < p.nphases; ++i) out->ph[i] = p.ph[i];
  return 0;
}

template <int NP>
static cudaError_t launch_np(const SmallmapParams& sp, cudaStream_t st) {
  static SmemConfigOnce once;
  if (cudaError_t e = once.ensure(conv_smallmap_kernel<NP>, SmCfg<NP>::SMEM); e != cudaSuccess) return e;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(sp.cotiles, sp.ptiles * sp.nphases, sp.ksplit);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = SmCfg<NP>::SMEM;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = sp.ksplit;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 2 : 1;
  return cudaLaunchKernelEx(&cfg, conv_smallmap_kernel<NP>, sp);
}

cudaError_t launch_conv_smallmap(const SmallmapParams& sp, cudaStream_t st) {
  switch (sp.np) {
    case 256: return launch_np<256>(sp, st);
    case 64: return launch_np<64>(sp, st);
    case 16: return launch_np<16>(sp, st);
  }
  return cudaErrorInvalidValue;
}

}  // namespace ltb
