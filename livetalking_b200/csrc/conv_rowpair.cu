// Row-pair 3x3 conv for the 80 -> 32 channel wav2lip256 output conv (L53 at 256x256): stride 1, pad 1, Cin = 80, Cout = 32,
// no residual, with the optional fused 1x1 head + sigmoid * 255 that writes the prediction.
//
// The halo kernel runs this layer on its BN = 32 instance: pixels on the wgmma M side and 32 output channels on N, so every
// m64n32k16 reads 2 KB + 1 KB of shared memory for 65 kFLOP, more than shared memory feeds at full tensor rate.  The ping-pong
// kernel's swap (conv_pingpong.cu: weights on M, pixels on N) would leave half of M = 64 empty with 32 output channels.  Here
// M packs two output rows: A rows 0-31 are the 32 output channels of an even tile row and rows 32-63 the same channels one row
// lower.  Since out(y + 1, x) = sum W[dy' - 1][dx] * in(y + dy', x + dx) for dy' = 1..3, one B view per (dy', dx), dy' = 0..3,
// feeds both rows:
//   B (pixels): the 16 (TH = 32) even rows of a TH x 8 pixel tile, N = 4 * TH, read from its (TH + 2) x 10 halo: start = halo
//               + (dy' * 10 + dx) pixels, 8-pixel groups two halo rows apart (SWIZZLE_128B and SWIZZLE_32B are functions of
//               the absolute address, so shifted starts read what TMA wrote).
//   A (weights, resident): per 64-channel chunk and tap column dx the 32-row blocks [0, W2, W1, W0, 0]; view dy' uses the
//               64-row window that starts at block 3 - dy'.  Neighbouring tap columns share their zero blocks.
// Each m64n128k16 reads 2 KB + 4 KB for 262 kFLOP; 12 views instead of 9 issue 4/3 of the useful products.
// K: chunk 0 is channels 0-63 (four K steps, 128-byte pixel rows); chunk 1, channels 64-79, is one K step stored with 32-byte
// pixel rows (SWIZZLE_32B) so that no zero-filled channels take shared memory or MMAs.
//
// Roles and schedule as conv_pingpong_kernel (384 threads): warpgroup 2 is the TMA producer (one thread), the two consumer
// warpgroups take alternate tiles and an ordering barrier lets one issue its MMAs while the other runs its epilogue; the weights
// load before pdl_wait().  Epilogue: the halo kernel's roundings in its order (fp16(acc + bias) with the ReLU / finite clamp),
// stmatrix.trans into an NHWC staging tile (warps 0-1 hold the even rows, warps 2-3 the odd rows), then
//   no head:   one TMA store of the tile into the output channel slice (TMA clips rows and columns past the map's edge);
//   head:      each thread reads one pixel's 32 channels back and sums the three outputs from the bias in channel order with
//              fmaf, as the halo kernel's fused head does, and stores the pred floats.
// The MMAs of a tile are issued in the halo kernel's order (chunk, tap row, K step, tap column).  The extra products of the
// views dy' = 0 and 3 are exact zeros, so every output element sees the same sequence of k16 partial sums as on
// conv_halo_wgmma_kernel<32, 2, 1, 9, 2>: the outputs are bit-identical.
#include <cuda.h>

#include <cstring>

#include "conv_rowpair.h"
#include "conv_tma.h"
#include "ltb_internal.h"
#include "ptx_sm90.cuh"

namespace ltb {

namespace {

constexpr int kThreads = 384;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;   // 128 x 40 + 256 x 232 <= 64 K registers per SM
constexpr int kTH = 32;                                   // tile rows (tile: kTH x 8 pixels)
constexpr int kN = 4 * kTH;                               // wgmma N: kTH / 2 row pairs x 8 pixels
constexpr int kP = 10, kHR = kTH + 2;                     // halo pitch and rows
// Two halo stages fit next to the weights and the staging tiles, so each warpgroup refills its own stage while the other issues
// its MMAs.  16 x 8 tiles (N = 64, four stages) hide more of the load latency but read more shared memory per MMA: L53 + head
// in the batch-16 forward took 110 us with them against 98 us here (H100 80GB HBM3, 700 W limit).
constexpr int kStages = 2;
constexpr int kX0Raw = kHR * kP * 128;                    // chunk 0 halo: 128-byte pixel rows
constexpr int kX1Raw = kHR * kP * 32;                     // chunk 1 halo: 32-byte pixel rows
constexpr int kX0Bytes = (kX0Raw + 1023) & ~1023;
constexpr int kX1Bytes = (kX1Raw + 1023) & ~1023;
constexpr int kStageBytes = kX0Bytes + kX1Bytes;
constexpr int kBlk0 = 32 * 128, kBlk1 = 32 * 32;          // one 32-row weight block of chunk 0 / chunk 1
constexpr int kBlocks = 13;                               // [0, W2, W1, W0] x 3 tap columns + a closing 0
constexpr int kW0Bytes = kBlocks * kBlk0, kW1Bytes = kBlocks * kBlk1;
constexpr int kWTxBytes = 9 * (kBlk0 + kBlk1);
constexpr int kOutBytes = kTH * 8 * 64;                   // kTH x 8 pixels x 32 channels
constexpr int kSmemBytes = kW0Bytes + kW1Bytes + kStages * kStageBytes + 2 * kOutBytes + 1024;
static_assert(kSmemBytes + 1024 <= 227 * 1024, "shared memory overflow");
// named barriers: 1 + g = warpgroup g may issue its MMAs, 3 + g = warpgroup g's staging tile
constexpr uint32_t kBarOrder = 1, kBarStage = 3;

}  // namespace

__global__ void __launch_bounds__(kThreads, 1) conv_rowpair_kernel(const __grid_constant__ RowpairParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t x_full[kStages], x_empty[kStages], w_full;
  __shared__ float head_sw[99];   // fused head: 3 x 32 weights + 3 biases
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* const smem = smem_raw + (smem0 - smem_u32(smem_raw));
  const uint32_t w0_smem = smem0;
  const uint32_t w1_smem = w0_smem + kW0Bytes;
  const uint32_t x_smem = w1_smem + kW1Bytes;
  const uint32_t o_smem = x_smem + kStages * kStageBytes;
  const int tiles_img = p.tiles_x * p.tiles_y;

  // the zero blocks 0, 4, 8, 12 of both weight chunks, written through the generic proxy and fenced for wgmma
  for (int i = tid; i < 4 * (kBlk0 + kBlk1) / 16; i += kThreads) {
    const int z = i / ((kBlk0 + kBlk1) / 16), r = i - z * ((kBlk0 + kBlk1) / 16);
    const int off = r < kBlk0 / 16 ? 4 * z * kBlk0 + r * 16 : kW0Bytes + 4 * z * kBlk1 + (r - kBlk0 / 16) * 16;
    *reinterpret_cast<uint4*>(smem + off) = make_uint4(0u, 0u, 0u, 0u);
  }
  fence_proxy_async_smem();
  if (p.head_out && tid < 99) head_sw[tid] = (tid < 96) ? p.head_w[tid] : p.head_b[tid - 96];
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(smem_u32(&x_full[s]), 1);
      mbar_init(smem_u32(&x_empty[s]), 4);   // one arrival per warp of the warpgroup that consumed the stage
    }
    mbar_init(smem_u32(&w_full), 1);
    mbar_fence_init();
    tma_prefetch_desc(&p.tm_x0);
    tma_prefetch_desc(&p.tm_x1);
    tma_prefetch_desc(&p.tm_w0);
    tma_prefetch_desc(&p.tm_w1);
    tma_prefetch_desc(&p.tm_out);
  }
  __syncthreads();

  // PDL: the weights are constants and load before this kernel waits for its predecessor; activations only after pdl_wait()
  pdl_launch_dependents();
  if (warp == 8 && lane == 0) {
    mbar_arrive_expect_tx(smem_u32(&w_full), kWTxBytes);
    for (int t = 0; t < 9; ++t) {
      const int b = 4 * (t % 3) + 3 - t / 3;   // tap (dy, dx) = W_dy of tap column dx: block 4 dx + 3 - dy
      tma_load_3d(w0_smem + b * kBlk0, &p.tm_w0, smem_u32(&w_full), 0, 0, t);
      tma_load_3d(w1_smem + b * kBlk1, &p.tm_w1, smem_u32(&w_full), 64, 0, t);
    }
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
        const uint32_t xb = x_smem + st * kStageBytes;
        mbar_wait(smem_u32(&x_empty[st]), ((s / kStages) & 1u) ^ 1u);
        mbar_arrive_expect_tx(smem_u32(&x_full[st]), kX0Raw + kX1Raw);
        tma_load_4d(xb, &p.tm_x0, smem_u32(&x_full[st]), 0, tx * 8 - 1, ty * kTH - 1, img);
        tma_load_4d(xb + kX0Bytes, &p.tm_x1, smem_u32(&x_full[st]), 64, tx * 8 - 1, ty * kTH - 1, img);
      }
    }
    return;
  }

  // =============================================================== consumers: warpgroup wg takes tiles wg, wg + 2, ...
  setmaxnreg_inc<kConsumerRegs>();
  const int wg = warp >> 2, wq = warp & 3;
  const bool leader = (tid & 127) == 0;
  const bool head = p.head_out != nullptr;
  const uint32_t obuf = o_smem + wg * kOutBytes;
  constexpr uint32_t kW0Hi = wgmma_hi_128b(8 * 128);        // weights: 8-row groups of 128-byte / 32-byte rows
  constexpr uint32_t kW1Hi = wgmma_hi_32b(8 * 32);
  constexpr uint32_t kX0Hi = wgmma_hi_128b(2 * kP * 128);   // pixels: 8-pixel groups two halo rows apart
  constexpr uint32_t kX1Hi = wgmma_hi_32b(2 * kP * 32);
  const uint32_t w0_lo = wgmma_lo(w0_smem), w1_lo = wgmma_lo(w1_smem);
  // accumulator rows 16 wq + lane / 4 (+8): output channel c0 (+8) of tile row 2i + par in column group i (pixels 2(lane % 4) (+1))
  const int par = wq >> 1, c0 = 16 * (wq & 1) + (lane >> 2);
  const float bias0 = __ldg(p.bias + c0), bias1 = __ldg(p.bias + c0 + 8);
  // stmatrix x4: lanes 8k..8k+7 address pixels 0..7 of tile row 2(i + (k >> 1)) + par, channel block 2(wq & 1) + (k & 1)
  const int sm_i = lane >> 4, sm_cb = 2 * (wq & 1) + ((lane >> 3) & 1), sm_x = lane & 7;
  // 64-byte pixel rows, SWIZZLE_64B on the 1024-aligned tile: 16-byte chunk ^ ((pixel >> 1) & 3)
  const uint32_t sm_off = (uint32_t)(sm_x * 64 + ((sm_cb ^ ((sm_x >> 1) & 3)) << 4));
  mbar_wait(smem_u32(&w_full), 0);

  uint32_t s = wg;   // position of the tile in the CTA's sequence (selects the halo stage)
  for (int t = blockIdx.x + wg * gridDim.x; t < p.total_tiles; t += 2 * gridDim.x, s += 2) {
    const int img = t / tiles_img, r = t - img * tiles_img;
    const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
    const uint32_t st = s % kStages;
    const uint32_t xb = x_smem + st * kStageBytes;
    if (s > 0) named_sync(kBarOrder + wg, 256);   // the other warpgroup has issued the MMAs of the previous tile
    mbar_wait(smem_u32(&x_full[st]), (s / kStages) & 1u);

    float acc[kN / 2];
#pragma unroll
    for (int i = 0; i < kN / 2; ++i) acc[i] = 0.f;
    const uint32_t x0_lo = wgmma_lo(xb), x1_lo = wgmma_lo(xb + kX0Bytes);
    wgmma_fence();
#pragma unroll
    for (int v = 0; v < 4; ++v)   // view dy': tap row dy' of the even rows, dy' - 1 of the odd rows
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx)
          Wgmma<kN>::ss(acc, wgmma_lohi(w0_lo + (4 * dx + 3 - v) * (kBlk0 / 16) + k * 2, kW0Hi),
                        wgmma_lohi(x0_lo + (v * kP + dx) * 8 + k * 2, kX0Hi), 1u);
#pragma unroll
    for (int v = 0; v < 4; ++v)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx)
        Wgmma<kN>::ss(acc, wgmma_lohi(w1_lo + (4 * dx + 3 - v) * (kBlk1 / 16), kW1Hi), wgmma_lohi(x1_lo + (v * kP + dx) * 2, kX1Hi), 1u);
    wgmma_commit();
    if (t + gridDim.x < p.total_tiles) named_arrive(kBarOrder + (wg ^ 1), 256);   // the other warpgroup's next tile may start
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&x_empty[st]));

    // ---------------------------------------------------------- epilogue: registers -> staging tile -> TMA store / head
    if (leader) bulk_wait_read<0>();   // this warpgroup's previous store has read the staging tile
    named_sync(kBarStage + wg, 128);   // (and, with the head, every thread has read its pixels back)
    auto cvt = [&](float f0, float f1, float b) { return p.relu ? f32x2_to_f16x2_sat_relu(f0 + b, f1 + b) : f32x2_to_f16x2_sat(f0 + b, f1 + b); };
#pragma unroll
    for (int i = 0; i < kTH / 2; i += 2) {
      const uint32_t o0 = cvt(acc[4 * i], acc[4 * i + 1], bias0);
      const uint32_t o1 = cvt(acc[4 * i + 2], acc[4 * i + 3], bias1);
      const uint32_t o2 = cvt(acc[4 * i + 4], acc[4 * i + 5], bias0);
      const uint32_t o3 = cvt(acc[4 * i + 6], acc[4 * i + 7], bias1);
      stmatrix_x4_trans(obuf + (2 * (i + sm_i) + par) * 8 * 64 + sm_off, o0, o1, o2, o3);
    }
    if (!head) fence_proxy_async_smem();
    named_sync(kBarStage + wg, 128);
    if (!head) {
      if (leader) {
        tma_store_4d(&p.tm_out, obuf, 0, tx * 8, ty * kTH, img);
        bulk_commit();
      }
      continue;
    }
#pragma unroll 1
    for (int pix = tid & 127; pix < kTH * 8; pix += 128) {
      const int gy = ty * kTH + (pix >> 3), gx = tx * 8 + (pix & 7);
      if (gy >= p.H || gx >= p.W) continue;
      uint32_t hv[16];   // channels 2j (+1)
#pragma unroll
      for (int cb = 0; cb < 4; ++cb) {
        const uint4 q = lds128(obuf + pix * 64 + ((cb ^ ((pix >> 1) & 3)) << 4));
        hv[4 * cb] = q.x;
        hv[4 * cb + 1] = q.y;
        hv[4 * cb + 2] = q.z;
        hv[4 * cb + 3] = q.w;
      }
      float ha0 = head_sw[96], ha1 = head_sw[97], ha2 = head_sw[98];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hv[j]));
        ha0 = fmaf(f.x, head_sw[2 * j], ha0);
        ha0 = fmaf(f.y, head_sw[2 * j + 1], ha0);
        ha1 = fmaf(f.x, head_sw[32 + 2 * j], ha1);
        ha1 = fmaf(f.y, head_sw[32 + 2 * j + 1], ha1);
        ha2 = fmaf(f.x, head_sw[64 + 2 * j], ha2);
        ha2 = fmaf(f.y, head_sw[64 + 2 * j + 1], ha2);
      }
      float* o = p.head_out + (((size_t)img * p.H + gy) * p.W + gx) * 3;
      o[0] = (1.f / (1.f + expf(-ha0))) * 255.f;
      o[1] = (1.f / (1.f + expf(-ha1))) * 255.f;
      o[2] = (1.f / (1.f + expf(-ha2))) * 255.f;
    }
  }
  if (leader) bulk_wait<0>();
}

bool conv_rowpair_supported(const ConvParams& p) {
  if (p.zbatch > 1 || p.group_slot || p.upconv || !conv_is_3x3_same(p)) return false;
  // The kernel takes any Cin in 65..80 (the second chunk is one K step of 16 channels), but only the wav2lip256 output conv's
  // 80 channels are routed here: other narrow convs keep the halo instances their callers were measured and tested on.
  if (p.Cin != 80 || p.Cout != 32 || p.Ktot != 9 * 80 || p.res) return false;
  // TMA: 16-byte aligned slice starts and pixel pitches
  if (!tma_slice_ok(p.in, p.ICtot, p.ic_off) || !tma_slice_ok(p.out, p.OCtot, p.oc_off)) return false;
  // at least three tiles per SM: each CTA's second warpgroup has a tile whose MMAs run under the first one's epilogue
  const long tiles = (long)p.N * ((p.GH + kTH - 1) / kTH) * ((p.GW + 7) / 8);
  if (tiles < 3L * device_sms()) return false;
  return ab_switch_on("LTB_CONV_ROWPAIR");   // 0 runs these convs on the halo kernel
}

int conv_rowpair_make_plan(const ConvParams& p, const __half* w_tap_major, RowpairParams* out) {
  if (!conv_rowpair_supported(p) || !w_tap_major) return 1;
  std::memset(out, 0, sizeof(*out));
  {
    const cuuint32_t box0[4] = {64, kP, kHR, 1}, box1[4] = {16, kP, kHR, 1};
    if (!encode_nhwc_f16(&out->tm_x0, p.in + p.ic_off, p.Cin, p.IW, p.IH, p.N, p.ICtot, box0)) return 2;
    if (!encode_nhwc_f16(&out->tm_x1, p.in + p.ic_off, p.Cin, p.IW, p.IH, p.N, p.ICtot, box1, 1, CU_TENSOR_MAP_SWIZZLE_32B)) return 2;
  }
  {
    const cuuint64_t dims[3] = {(cuuint64_t)p.Cin, 32, 9};
    const cuuint64_t strides[2] = {(cuuint64_t)p.Cin * 2, (cuuint64_t)32 * p.Cin * 2};
    const cuuint32_t box0[3] = {64, 32, 1}, box1[3] = {16, 32, 1};
    if (!encode_tmap_f16(&out->tm_w0, 3, w_tap_major, dims, strides, box0)) return 2;
    if (!encode_tmap_f16(&out->tm_w1, 3, w_tap_major, dims, strides, box1, 1, CU_TENSOR_MAP_SWIZZLE_32B)) return 2;
  }
  {
    const cuuint32_t box[4] = {32, 8, kTH, 1};
    if (!encode_nhwc_f16(&out->tm_out, p.out + p.oc_off, 32, p.OW, p.OH, p.N, p.OCtot, box, 1, CU_TENSOR_MAP_SWIZZLE_64B)) return 2;
  }
  out->bias = p.bias;
  out->relu = p.relu;
  out->H = p.GH;
  out->W = p.GW;
  out->tiles_x = (p.GW + 7) / 8;
  out->tiles_y = (p.GH + kTH - 1) / kTH;
  out->total_tiles = out->tiles_x * out->tiles_y * p.N;
  return 0;
}

cudaError_t launch_conv_rowpair(const RowpairParams& rp, cudaStream_t st) {
  static SmemConfigOnce once;
  if (cudaError_t e = once.ensure(conv_rowpair_kernel, kSmemBytes); e != cudaSuccess) return e;
  const int sms = device_sms();
  const int grid = rp.total_tiles < sms ? rp.total_tiles : sms;
  return launch_kernel_pdl(conv_rowpair_kernel, dim3(grid), dim3(kThreads), kSmemBytes, st, rp);
}

}  // namespace ltb
