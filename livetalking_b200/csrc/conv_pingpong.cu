// Ping-pong 3x3 conv for the 64 -> 64 channel residual blocks (wav2lip256 L18-L20 at 64x64 and L51/L52 at 256x256):
// stride 1, pad 1, Cin = Cout = 64, the residual is the conv's own input slice (HaloParams::res_halo semantics).
//
// The halo kernel (conv_halo.cu) puts the pixels on the wgmma M side and the 64 output channels on N, and both consumer
// warpgroups split one tile.  Every m64n64k16 then reads 2 KB of A and 2 KB of B from shared memory for 131 kFLOP (all of
// the SM's shared-memory bandwidth at full tensor rate), and both warpgroups run the epilogue at the same time while the
// tensor core idles.  Here the operands swap roles: A (M = 64) is the weights and B (N = 128) is one 16 x 8 pixel tile, so
// one warpgroup owns a whole tile (64 accumulator registers per thread) and each m64n128k16 reads 2 KB + 4 KB for 262 kFLOP.
// The two consumer warpgroups take alternate tiles of the CTA's persistent sequence, and an ordering barrier lets one issue
// its MMAs while the other runs its epilogue (the ping-pong schedule of CUTLASS's KernelTmaWarpSpecializedPingpong).
//
// Roles (384 threads): warpgroup 2 is the TMA producer (one thread), warpgroups 0 and 1 consume.  Shared memory holds the
// whole tap-major weight set (9 x 64 x 64 fp16, 72 KB, loaded once per CTA), a ring of (16+2) x 10 pixel halo stages and
// one 16 KB output staging tile per consumer warpgroup.
//   B (pixels): the nine im2col views of the halo, as in the halo kernel: start = halo + (dy * 10 + dx) rows, 8-pixel row
//               groups 1280 B apart (SWIZZLE_128B is a function of the absolute address, so shifted starts read what TMA
//               wrote).
//   A (weights): tap t is a K-major 64 x 64 block at weights + t * 8 KB.
//   Residual:   while the warpgroup holds the stage, ldmatrix.trans reads the centre view into the (channel x pixel)
//               accumulator fragment layout.
//   Epilogue:   the halo kernel's roundings in its order (fp16(acc + bias), then + residual in fp16 with the ReLU / finite
//               clamp), stmatrix.trans into the swizzled NHWC staging tile, one TMA store of the tile into the output channel
//               slice (TMA clips rows and columns past the map's edge).  A warpgroup waits for its previous store to have read
//               the staging tile only when it is about to refill it.
// The MMAs of a tile are issued in the halo kernel's order (tap row, K step, tap column), so every output element sees the
// same sequence of k16 partial sums as on conv_halo_wgmma_kernel<64, 2, 1, 9, 1>.
#include <cuda.h>

#include <cstring>

#include "conv_pingpong.h"
#include "conv_tma.h"
#include "ltb_internal.h"
#include "ptx_sm90.cuh"

namespace ltb {

namespace {

constexpr int kThreads = 384;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;   // 128 x 40 + 256 x 232 <= 64 K registers per SM
constexpr int kP = 10, kHR = 18;                         // halo pitch and rows of a 16 x 8 pixel tile
constexpr int kStages = 4;
constexpr int kABytesRaw = kHR * kP * 128;               // TMA transaction bytes per halo stage
constexpr int kABytes = (kABytesRaw + 1023) & ~1023;
constexpr int kTapBytes = 64 * 128;                      // one tap: 64 output channels x 64 input channels
constexpr int kWBytes = 9 * kTapBytes;
constexpr int kOutBytes = 128 * 128;                     // 128 pixels x 64 channels
constexpr int kSmemBytes = kWBytes + kStages * kABytes + 2 * kOutBytes + 1024;
static_assert(kSmemBytes + 1024 <= 227 * 1024, "shared memory overflow");
// named barriers: 1 + g = warpgroup g may issue its MMAs, 3 + g = warpgroup g's staging tile
constexpr uint32_t kBarOrder = 1, kBarStage = 3;

}  // namespace

__global__ void __launch_bounds__(kThreads, 1) conv_pingpong_kernel(const __grid_constant__ PingpongParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t a_full[kStages], a_empty[kStages], w_full;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t w_smem = smem0;
  const uint32_t a_smem = w_smem + kWBytes;
  const uint32_t o_smem = a_smem + kStages * kABytes;
  const int tiles_img = p.tiles_x * p.tiles_y;

  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(smem_u32(&a_full[s]), 1);
      mbar_init(smem_u32(&a_empty[s]), 4);   // one arrival per warp of the warpgroup that consumed the stage
    }
    mbar_init(smem_u32(&w_full), 1);
    mbar_fence_init();
    tma_prefetch_desc(&p.tm_in);
    tma_prefetch_desc(&p.tm_w);
    tma_prefetch_desc(&p.tm_out);
  }
  __syncthreads();

  // PDL: the weights are constants and load before this kernel waits for its predecessor; activations only after pdl_wait()
  pdl_launch_dependents();
  if (warp == 8 && lane == 0) {
    mbar_arrive_expect_tx(smem_u32(&w_full), kWBytes);
    for (int j = 0; j < 3; ++j) tma_load_3d(w_smem + 3 * j * kTapBytes, &p.tm_w, smem_u32(&w_full), 0, 0, 3 * j);
  }
  pdl_wait();

  if (warp >= 8) {
    // =============================================================== TMA producer
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 8 && lane == 0) {
      uint32_t s = 0;
      for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x, ++s) {
        const int img = t / tiles_img, r = t - img * tiles_img;
        const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
        const uint32_t st = s % kStages;
        mbar_wait(smem_u32(&a_empty[st]), ((s / kStages) & 1u) ^ 1u);
        mbar_arrive_expect_tx(smem_u32(&a_full[st]), kABytesRaw);
        tma_load_4d(a_smem + st * kABytes, &p.tm_in, smem_u32(&a_full[st]), 0, tx * 8 - 1, ty * 16 - 1, img);
      }
    }
    return;
  }

  // =============================================================== consumers: warpgroup wg takes tiles wg, wg + 2, ...
  setmaxnreg_inc<kConsumerRegs>();
  const int wg = warp >> 2, wq = warp & 3;
  const bool leader = (tid & 127) == 0;
  const uint32_t obuf = o_smem + wg * kOutBytes;
  constexpr uint32_t kWHi = wgmma_hi_128b(1024);          // weights: 8-row groups 1024 B apart
  constexpr uint32_t kXHi = wgmma_hi_128b(kP * 128);      // pixels: 8-pixel rows one halo row (1280 B) apart
  const uint32_t w_lo0 = wgmma_lo(w_smem);
  // accumulator rows (output channels) c0 and c0 + 8; columns 8i + 2(lane % 4) (+1) = pixel row i, pixels 2(lane % 4) (+1)
  const int c0 = 16 * wq + (lane >> 2);
  const float bias0 = __ldg(p.bias + c0), bias1 = __ldg(p.bias + c0 + 8);
  const __half2 hmax = __floats2half2_rn(65504.f, 65504.f);
  const __half2 hlo = p.relu ? __floats2half2_rn(0.f, 0.f) : __floats2half2_rn(-65504.f, -65504.f);
  // ldmatrix / stmatrix x4: lanes 8k..8k+7 address pixels 0..7 of pixel row i + (k >> 1), channel block 2 wq + (k & 1)
  const int lm_row = lane >> 4, lm_cb = 2 * wq + ((lane >> 3) & 1), lm_x = lane & 7;
  mbar_wait(smem_u32(&w_full), 0);

  uint32_t s = wg;   // position of the tile in the CTA's sequence (selects the halo stage)
  for (int t = blockIdx.x + wg * gridDim.x; t < p.total_tiles; t += 2 * gridDim.x, s += 2) {
    const int img = t / tiles_img, r = t - img * tiles_img;
    const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
    const uint32_t st = s % kStages;
    const uint32_t abase = a_smem + st * kABytes;
    if (s > 0) named_sync(kBarOrder + wg, 256);   // the other warpgroup has issued the MMAs of the previous tile
    mbar_wait(smem_u32(&a_full[st]), (s / kStages) & 1u);

    // residual: the centre view (halo row (y + 1) * 10 + x + 1), transposed into the accumulator layout
    uint32_t rh[16][2];
#pragma unroll
    for (int i = 0; i < 16; i += 2) {
      const int hr = (i + lm_row + 1) * kP + lm_x + 1;
      ldmatrix_x4_trans(rh[i][0], rh[i][1], rh[i + 1][0], rh[i + 1][1], abase + hr * 128 + ((lm_cb ^ (hr & 7)) << 4));
    }

    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    const uint32_t x_lo0 = wgmma_lo(abase);
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int tt = 0; tt < 3; ++tt)
          Wgmma<128>::ss(acc, wgmma_lohi(w_lo0 + (3 * j + tt) * (kTapBytes / 16) + k * 2, kWHi),
                         wgmma_lohi(x_lo0 + (j * kP + tt) * 8 + k * 2, kXHi), 1u);
    wgmma_commit();
    if (t + gridDim.x < p.total_tiles) named_arrive(kBarOrder + (wg ^ 1), 256);   // the other warpgroup's next tile may start
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&a_empty[st]));

    // ---------------------------------------------------------- epilogue: registers -> staging tile -> TMA store
    if (leader) bulk_wait_read<0>();   // this warpgroup's previous store has read the staging tile
    named_sync(kBarStage + wg, 128);
    auto out2 = [&](float f0, float f1, float b, uint32_t res) {
      const uint32_t v = f32x2_to_f16x2_sat(f0 + b, f1 + b);
      const __half2 o = __hmin2(__hmax2(__hadd2(*reinterpret_cast<const __half2*>(&v), *reinterpret_cast<const __half2*>(&res)), hlo), hmax);
      return *reinterpret_cast<const uint32_t*>(&o);
    };
#pragma unroll
    for (int i = 0; i < 16; i += 2) {
      const uint32_t o0 = out2(acc[4 * i], acc[4 * i + 1], bias0, rh[i][0]);
      const uint32_t o1 = out2(acc[4 * i + 2], acc[4 * i + 3], bias1, rh[i][1]);
      const uint32_t o2 = out2(acc[4 * i + 4], acc[4 * i + 5], bias0, rh[i + 1][0]);
      const uint32_t o3 = out2(acc[4 * i + 6], acc[4 * i + 7], bias1, rh[i + 1][1]);
      // staging row = pixel (i + lm_row) * 8 + lm_x, 128B swizzle on the 1024-aligned tile: chunk ^ (row & 7) = chunk ^ lm_x
      stmatrix_x4_trans(obuf + ((i + lm_row) * 8 + lm_x) * 128 + ((lm_cb ^ lm_x) << 4), o0, o1, o2, o3);
    }
    fence_proxy_async_smem();
    named_sync(kBarStage + wg, 128);
    if (leader) {
      tma_store_4d(&p.tm_out, obuf, 0, tx * 8, ty * 16, img);
      bulk_commit();
    }
  }
  if (leader) bulk_wait<0>();
}

bool conv_pingpong_supported(const ConvParams& p) {
  if (p.zbatch > 1 || p.group_slot || p.upconv || !conv_is_3x3_same(p)) return false;
  if (p.Cin != 64 || p.Cout != 64 || p.Ktot != 9 * 64) return false;
  // the residual is the input slice the halo tiles hold
  if (p.res != p.in || p.rc_off != p.ic_off || p.RCtot != p.ICtot) return false;
  // TMA: 16-byte aligned slice starts and pixel pitches
  if (!tma_slice_ok(p.in, p.ICtot, p.ic_off) || !tma_slice_ok(p.out, p.OCtot, p.oc_off)) return false;
  // The kernel clips tiles at any map edge, but only maps whose width is a multiple of the 8-pixel tile are routed here (the
  // wav2lip256 residual layers): other 64-channel maps keep the halo instance their callers were measured and tested on.
  if (p.GW % 8) return false;
  // at least three tiles per SM: each CTA's second warpgroup has a tile whose MMAs run under the first one's epilogue.  Smaller
  // layers stay on the halo kernel, which splits each tile over both warpgroups.
  const long tiles = (long)p.N * ((p.GH + 15) / 16) * ((p.GW + 7) / 8);
  if (tiles < 3L * device_sms()) return false;
  return ab_switch_on("LTB_CONV_PINGPONG");   // 0 runs these convs on the halo kernel
}

int conv_pingpong_make_plan(const ConvParams& p, const __half* w_tap_major, PingpongParams* out) {
  if (!conv_pingpong_supported(p) || !w_tap_major) return 1;
  std::memset(out, 0, sizeof(*out));
  const cuuint32_t in_box[4] = {64, kP, kHR, 1}, out_box[4] = {64, 8, 16, 1};
  if (!encode_nhwc_f16(&out->tm_in, p.in + p.ic_off, 64, p.IW, p.IH, p.N, p.ICtot, in_box)) return 2;
  if (!encode_nhwc_f16(&out->tm_out, p.out + p.oc_off, 64, p.OW, p.OH, p.N, p.OCtot, out_box)) return 2;
  {
    const cuuint64_t dims[3] = {64, 64, 9};
    const cuuint64_t strides[2] = {64 * 2, 64 * 64 * 2};
    const cuuint32_t box[3] = {64, 64, 3};
    if (!encode_tmap_f16(&out->tm_w, 3, w_tap_major, dims, strides, box)) return 2;
  }
  out->bias = p.bias;
  out->relu = p.relu;
  out->tiles_x = (p.GW + 7) / 8;
  out->tiles_y = (p.GH + 15) / 16;
  out->total_tiles = out->tiles_x * out->tiles_y * p.N;
  return 0;
}

cudaError_t launch_conv_pingpong(const PingpongParams& pp, cudaStream_t st) {
  static SmemConfigOnce once;
  if (cudaError_t e = once.ensure(conv_pingpong_kernel, kSmemBytes); e != cudaSuccess) return e;
  const int sms = device_sms();
  const int grid = pp.total_tiles < sms ? pp.total_tiles : sms;
  return launch_kernel_pdl(conv_pingpong_kernel, dim3(grid), dim3(kThreads), kSmemBytes, st, pp);
}

}  // namespace ltb
